"""The product columns of the permutation and lookup arguments two more ways, for the product tests: the reference's loops
restated with big integers (plonk/permutation/prover.rs:81-168, plonk/lookup/prover.rs:279-321), and a composition of
finer calls (Ast programs, batch_invert, running_product, the host's last_z)."""
from __future__ import annotations

from oracle import cref, pasta


# ---- the reference, restated -------------------------------------------------------------------------------------------
def oracle_permutation_product(columns, sigmas, beta, gamma, omega, delta, chunk_len, bf, blinding, m):
    """permutation/prover.rs:81-168 for every proof: columns[p][c] and sigmas[c] are lists of n ints, blinding the
    proofs x sets x bf values in the rng's order.  Returns z[p][a] (lists of n ints)."""
    n = len(sigmas[0])
    out, at = [], 0
    for cols in columns:
        last_z, deltaomega, sets = 1, 1, []
        for c0 in range(0, len(sigmas), chunk_len):
            mv = [1] * n
            for v, s in zip(cols[c0:c0 + chunk_len], sigmas[c0:c0 + chunk_len]):           # :101-116
                mv = [x * ((beta * s_i + gamma + v_i) % m) % m for x, s_i, v_i in zip(mv, s, v)]
            mv = [pasta.inv(x, m) if x else 0 for x in mv]                                   # :120 batch_invert
            for v in cols[c0:c0 + chunk_len]:                                                # :124-143
                cur = deltaomega
                for i in range(n):
                    mv[i] = mv[i] * ((cur * beta + gamma + v[i]) % m) % m
                    cur = cur * omega % m
                deltaomega = deltaomega * delta % m
            z = [last_z]
            for row in range(1, n):                                                          # :150-156
                z.append(z[row - 1] * mv[row - 1] % m)
            z[n - bf:] = blinding[at:at + bf]                                                # :158-161
            at += bf
            last_z = z[n - (bf + 1)]                                                         # :163
            sets.append(z)
        out.append(sets)
    return out


def oracle_lookup_product(a, s, a_perm, s_perm, beta, gamma, bf, blinding, m):
    """lookup/prover.rs:279-321 for one lookup: compressed input / table a, s and permuted a', s' (lists of n ints)."""
    n = len(a)
    lp = [(beta + x) * (gamma + y) % m for x, y in zip(a_perm, s_perm)]                     # :281-291
    lp = [pasta.inv(x, m) if x else 0 for x in lp]                                           # :295
    lp = [p * ((x + beta) % m) % m * ((y + gamma) % m) % m for p, x, y in zip(lp, a, s)]    # :299-309
    z, state = [], 1
    for cur in [1] + lp:                                                                     # :311-318
        state = state * cur % m
        z.append(state)
    return z[:n - bf] + list(blinding)                                                       # :319-321


# ---- the composition of finer calls ------------------------------------------------------------------------------------
def _close(*groups):
    for g in groups:
        for p in g:
            p.close()


def composition_permutation(eng, D, columns, sigmas, beta, gamma, delta, chunk_len, bf, blinding):
    """Per proof, per set: the Ast denominators, batch_invert, the Ast numerators, running_product from last_z, the blinding
    rows written, last_z read back.  Returns z[p][a] (resident)."""
    Ast, m, n = eng.Ast, D.m, D.n
    ev = eng.Evaluator(D, "lagrange")
    SL = [ev.register_poly(s) for s in sigmas]
    out, at, tmp = [], 0, []
    for cols in columns:
        CL = [ev.register_poly(c) for c in cols]
        sets, last_z = [], 1
        for c0 in range(0, len(sigmas), chunk_len):
            den = None
            for cl, sl in zip(CL[c0:c0 + chunk_len], SL[c0:c0 + chunk_len]):
                term = sl * beta + Ast.constant_term(gamma) + cl
                den = term if den is None else den * term
            inv_den = eng.batch_invert_resident(ev.evaluate(den, out=eng.ResidentPoly(D.field, n)))
            num = ev.register_poly(inv_den)
            for j, cl in enumerate(CL[c0:c0 + chunk_len]):
                num = num * (Ast.linear_term(pow(delta, c0 + j, m) * beta % m) + Ast.constant_term(gamma) + cl)
            mv = ev.evaluate(num, out=eng.ResidentPoly(D.field, n))
            z = eng.running_product_resident(mv, init=last_z, dst=eng.ResidentPoly(D.field, n))
            if bf:
                z.copy_from(eng.ResidentPoly(D.field, bf, cref.ints_to_bytes(blinding[at:at + bf])), bf, dst_off=n - bf)
            at += bf
            one = eng.ResidentPoly(D.field, 1).copy_from(z, 1, src_off=n - bf - 1)     # last_z: one element back to the host
            last_z = int.from_bytes(one.download(1)[0].tobytes(), "little")
            tmp += [inv_den, mv, one]
            sets.append(z)
        out.append(sets)
    _close(tmp)
    ev.close()
    return out


def composition_lookup(eng, D, lookups, beta, gamma, bf, blinding):
    Ast, n = eng.Ast, D.n
    ev = eng.Evaluator(D, "lagrange")
    out, tmp = [], []
    for b, (ci, ct, pi, pt) in enumerate(lookups):
        CI, CT, PI, PT = (ev.register_poly(p) for p in (ci, ct, pi, pt))
        inv_den = eng.batch_invert_resident(ev.evaluate((PI + Ast.constant_term(beta)) * (PT + Ast.constant_term(gamma)), out=eng.ResidentPoly(D.field, n)))
        num = ev.register_poly(inv_den) * (CI + Ast.constant_term(beta)) * (CT + Ast.constant_term(gamma))
        mv = ev.evaluate(num, out=eng.ResidentPoly(D.field, n))
        z = eng.running_product_resident(mv, init=1, dst=eng.ResidentPoly(D.field, n))
        if bf:
            z.copy_from(eng.ResidentPoly(D.field, bf, cref.ints_to_bytes(blinding[b * bf:(b + 1) * bf])), bf, dst_off=n - bf)
        tmp += [inv_den, mv]
        out.append(z)
    _close(tmp)
    ev.close()
    return out
