"""plonk::create_proof driven by a PINNED verifying key and the circuit's columns, through the oracle (test infrastructure).

Why it exists: the prover-side functions of the path -- lagrange_to_coeff / coeff_to_extended / extended_to_coeff (best_fft at
G = scalar), divide_by_vanishing_poly, permute_expression_pair, eval_polynomial, kate_division, commit / commit_lagrange, the
multi-point opening and the opening argument -- have no reference-held input -> output vector of their own.  The VERIFIER is
pinned on the reference's sixteen golden proofs (tests/plonk_verifier.py, tests/test_golden_proofs.py); so a REAL proof of the
reference's own test circuit, produced by the oracle's restatements of those functions under the reference's own golden
verifying key, and ACCEPTED by that pinned verifier, ties every one of them to the reference's verification equation: a wrong
butterfly, a wrong zeta power, a mis-ordered fold anywhere and the final multiexp is not the identity.

What is restated, in the reference's order (halo2_proofs/src/plonk):
  prover.rs:43-727               create_proof: instance / advice commitments, theta, lookups, beta / gamma, permutation and
                                 lookup products, the vanishing argument, y, h(X), x, every evaluation, the query list
  permutation/prover.rs:42-173   commit (the grand product over chunks of columns, last_z chaining, blinding rows),
                                 :176-283 construct (the expressions), :296-343 evaluate, :346-394 open
  lookup/prover.rs:63-203        commit_permuted, :206-300 commit_product, :303-383 construct, :386-425 evaluate, :428-470 open
  vanishing/prover.rs:41-60      commit (the random polynomial), :64-118 construct (h pieces), :121-150 evaluate, :153-175 open
  keygen.rs:306-325              l_0, l_blind, l_last
h(X) is evaluated point by point over the extended coset (2^extended_k points: 128 for the k = 5 test circuit) with the same
scalar formulas the verifier applies at x -- a rotation by r rows is a shift by r * 2^(extended_k - k) coset points.
The randomness (blinding rows, blinds, the random polynomial, the opening's) comes from a seeded generator.
"""
from __future__ import annotations

from typing import List

from oracle import pasta
from tests import plonk_verifier as PV


def create_proof(c: pasta.Curve, g, g_lagrange, w, u, vk: PV.PinnedKey, fixed: List[List[int]], sigma: List[List[int]],
                 advice: List[List[List[int]]], instances: List[List[List[int]]], rng, transcript, zeta: int, delta: int) -> None:
    """`fixed`, `sigma`: the circuit's fixed columns and permutation polynomials as Lagrange values (what keygen computes);
    `advice[proof][column]`: the witness, 2^k values each (the last blinding_factors + 1 rows are overwritten with randomness,
    prover.rs:276-282); `instances[proof][column]`: public inputs.  `transcript`: write_point / write_scalar / common_* /
    squeeze_challenge on affine tuples and ints."""
    m = vk.scalar_modulus
    k, n = vk.k, 1 << vk.k
    bf = vk.blinding_factors()
    usable = n - (bf + 1)
    cs_degree = vk.degree()
    chunk_len = cs_degree - 2
    D = pasta.EvaluationDomain(c.scalar, cs_degree, k, zeta)
    assert D.extended_k == vk.extended_k and D.omega == vk.omega
    L, step = D.extended_len(), 1 << (D.extended_k - k)
    num_proofs = len(advice)
    commit_l = lambda vals, blind: pasta.to_affine(c, pasta.best_multiexp(c, list(vals) + [blind], list(g_lagrange) + [w]))
    commit_c = lambda vals, blind: pasta.to_affine(c, pasta.best_multiexp(c, list(vals) + [blind], list(g) + [w]))
    to_coeff, to_ext = D.lagrange_to_coeff, D.coeff_to_extended
    evalp = lambda poly, x: pasta.eval_polynomial_mod(m, poly, x)

    transcript.common_scalar(vk.transcript_repr())                 # prover.rs:56  vk.hash_into
    # ---- instance columns, :73-126 ----
    inst_vals, inst_polys, inst_cosets = [], [], []
    for inst in instances:
        vals = []
        for col in inst:
            assert len(col) <= usable
            vals.append([v % m for v in col] + [0] * (n - len(col)))
        for v in vals:
            transcript.common_point(commit_l(v, 1))               # Blind::default()
        polys = [to_coeff(v) for v in vals]
        inst_vals.append(vals), inst_polys.append(polys), inst_cosets.append([to_ext(p) for p in polys])
    # ---- advice columns, :135-321 ----
    adv_vals, adv_polys, adv_cosets, adv_blinds = [], [], [], []
    for cols in advice:
        vals = [[v % m for v in col[:usable]] + [rng.scalar() for _ in range(n - usable)] for col in cols]     # :276-282
        blinds = [rng.scalar() for _ in vals]
        for v, b in zip(vals, blinds):
            transcript.write_point(commit_l(v, b))
        polys = [to_coeff(v) for v in vals]
        adv_vals.append(vals), adv_polys.append(polys), adv_cosets.append([to_ext(p) for p in polys]), adv_blinds.append(blinds)
    fixed_polys = [to_coeff(f) for f in fixed]
    fixed_cosets = [to_ext(p) for p in fixed_polys]
    sigma_polys = [to_coeff(s) for s in sigma]
    sigma_cosets = [to_ext(p) for p in sigma_polys]
    ind = lambda rows: to_ext(to_coeff([1 if r in rows else 0 for r in range(n)]))
    l0, l_blind, l_last = ind({0}), ind(set(range(n - bf, n))), ind({n - bf - 1})          # keygen.rs:306-325

    def rows_eval(expr, pr):                                       # an Expression over the Lagrange values, row by row (rotations wrap)
        out = []
        for row in range(n):
            at = lambda cols, qs: [cols[col][(row + r) % n] for col, r in qs]
            out.append(vk.evaluate(expr, m, at(fixed, vk.fixed_queries), at(adv_vals[pr], vk.advice_queries), at(inst_vals[pr], vk.instance_queries)))
        return out

    theta = transcript.squeeze_challenge()                         # :367
    # ---- lookups: permuted columns, lookup/prover.rs:63-203 ----
    lookups = []
    for pr in range(num_proofs):
        per = []
        for inp, tab in vk.lookups:
            def compress(exprs):
                acc = [0] * n
                for e in exprs:
                    ev = rows_eval(e, pr)
                    acc = [(a * theta + b) % m for a, b in zip(acc, ev)]
                return acc
            ci, ct = compress(inp), compress(tab)
            pi, pt = pasta.permute_expression_pair(c.scalar, ci, ct, usable)                # :563-647, usable rows
            pi = list(pi) + [rng.scalar() for _ in range(bf + 1)]                           # :623-624: the blinding rows, input first
            pt = list(pt) + [rng.scalar() for _ in range(bf + 1)]
            bi = rng.scalar()                                       # commit_values, :160-170: input then table
            cmi = commit_l(pi, bi)
            bt = rng.scalar()
            cmt = commit_l(pt, bt)
            transcript.write_point(cmi)
            transcript.write_point(cmt)
            per.append({"ci": ci, "ct": ct, "pi": pi, "pt": pt, "pi_poly": to_coeff(pi), "pt_poly": to_coeff(pt), "bi": bi, "bt": bt})
        lookups.append(per)
    beta = transcript.squeeze_challenge()                          # :405
    gamma = transcript.squeeze_challenge()                         # :408
    # ---- permutation products, permutation/prover.rs:42-173 ----
    perms = []
    col_vals = lambda pr, col: {"Advice": adv_vals[pr], "Fixed": fixed, "Instance": inst_vals[pr]}[col[0]][col[1]]
    for pr in range(num_proofs):
        sets, deltaomega, last_z = [], 1, 1
        for ci in range(0, len(vk.permutation_columns), chunk_len):
            cols = vk.permutation_columns[ci:ci + chunk_len]
            mod = [1] * n
            for col, sg in zip(cols, sigma[ci:ci + chunk_len]):     # :77-94
                v = col_vals(pr, col)
                mod = [a * ((beta * s + gamma + x) % m) % m for a, s, x in zip(mod, sg, v)]
            mod = [pasta.inv(a, m) if a else 0 for a in mod]        # batch_invert, :97
            for col in cols:                                        # :101-121
                v = col_vals(pr, col)
                cur = deltaomega
                for row in range(n):
                    mod[row] = mod[row] * ((cur * beta + gamma + v[row]) % m) % m
                    cur = cur * D.omega % m
                deltaomega = deltaomega * delta % m
            z = [last_z]
            for row in range(1, n):                                 # :126-133
                z.append(z[row - 1] * mod[row - 1] % m)
            for row in range(n - bf, n):                            # :136-138
                z[row] = rng.scalar()
            last_z = z[n - (bf + 1)]                                # :140
            blind = rng.scalar()
            transcript.write_point(commit_l(z, blind))              # :144-157
            zp = to_coeff(z)
            sets.append({"poly": zp, "coset": to_ext(zp), "blind": blind})
        perms.append(sets)
    # ---- lookup products, lookup/prover.rs:206-300 ----
    for pr in range(num_proofs):
        for lk in lookups[pr]:
            prod = [(beta + a) * (gamma + s) % m for a, s in zip(lk["pi"], lk["pt"])]
            prod = [pasta.inv(p, m) if p else 0 for p in prod]
            prod = [p * ((a + beta) % m) % m * ((s + gamma) % m) % m for p, a, s in zip(prod, lk["ci"], lk["ct"])]
            z, state = [], 1
            for cur in [1] + prod:                                  # :257-263: scan, take n - bf, then bf random values
                state = state * cur % m
                z.append(state)
            z = z[:n - bf] + [rng.scalar() for _ in range(bf)]
            assert z[0] == 1 and z[usable] == 1                     # the reference's sanity checks, :270, :290
            lk["zb"] = rng.scalar()
            transcript.write_point(commit_l(z, lk["zb"]))
            lk["z_poly"] = to_coeff(z)
    # ---- vanishing argument: the random polynomial, vanishing/prover.rs:41-60 ----
    random_poly = rng.poly(n)
    random_blind = rng.scalar()
    transcript.write_point(commit_c(random_poly, random_blind))
    y = transcript.squeeze_challenge()                             # :458
    # ---- h(X) over the extended coset: gates, permutation, lookups per proof, folded by y (prover.rs:460-564) ----
    xs, cur = [], D.g_coset
    for _ in range(L):
        xs.append(cur)
        cur = cur * D.extended_omega % m
    rot = lambda arr, i, r: arr[(i + r * step) % L]
    lk_cosets = [[{kk: to_ext(lk[kk + "_poly"]) for kk in ("pi", "pt", "z")} for lk in per] for per in lookups]
    lk_compressed = [[{kk: to_ext(to_coeff(lk[kk])) for kk in ("ci", "ct")} for lk in per] for per in lookups]
    last_rot = -(bf + 1)
    num = []
    for i in range(L):
        acc = 0
        active = (1 - (l_last[i] + l_blind[i])) % m
        for pr in range(num_proofs):
            at = lambda cosets, qs: [rot(cosets[col], i, r) for col, r in qs]
            fe, ae, ie = at(fixed_cosets, vk.fixed_queries), at(adv_cosets[pr], vk.advice_queries), at(inst_cosets[pr], vk.instance_queries)
            exprs = [vk.evaluate(gate, m, fe, ae, ie) for gate in vk.gates]
            sets = perms[pr]                                        # permutation/prover.rs:200-283
            if sets:
                zc = [s["coset"] for s in sets]
                exprs.append((1 - zc[0][i]) * l0[i] % m)
                exprs.append((zc[-1][i] * zc[-1][i] - zc[-1][i]) * l_last[i] % m)
                for a in range(1, len(sets)):
                    exprs.append((zc[a][i] - rot(zc[a - 1], i, last_rot)) * l0[i] % m)
                colc = lambda col: {"Advice": adv_cosets[pr], "Fixed": fixed_cosets, "Instance": inst_cosets[pr]}[col[0]][col[1]][i]
                for a, st in enumerate(sets):
                    cols = vk.permutation_columns[a * chunk_len:(a + 1) * chunk_len]
                    left = rot(zc[a], i, 1)
                    for col, sc in zip(cols, sigma_cosets[a * chunk_len:(a + 1) * chunk_len]):
                        left = left * ((colc(col) + beta * sc[i] + gamma) % m) % m
                    right = zc[a][i]
                    cur_delta = beta * xs[i] % m * pow(delta, a * chunk_len, m) % m
                    for col in cols:
                        right = right * ((colc(col) + cur_delta + gamma) % m) % m
                        cur_delta = cur_delta * delta % m
                    exprs.append((left - right) * active % m)
            for lc, lcc in zip(lk_cosets[pr], lk_compressed[pr]):   # lookup/prover.rs:318-372
                z_, a_, s_ = lc["z"], lc["pi"], lc["pt"]
                exprs.append((1 - z_[i]) * l0[i] % m)
                exprs.append((z_[i] * z_[i] - z_[i]) * l_last[i] % m)
                left = rot(z_, i, 1) * ((a_[i] + beta) % m) % m * ((s_[i] + gamma) % m) % m
                right = z_[i] * ((lcc["ci"][i] + beta) % m) % m * ((lcc["ct"][i] + gamma) % m) % m
                exprs.append((left - right) * active % m)
                exprs.append((a_[i] - s_[i]) * l0[i] % m)
                exprs.append((a_[i] - s_[i]) * (a_[i] - rot(a_, i, -1)) % m * active % m)
            for e in exprs:                                          # Ast::distribute_powers, vanishing/prover.rs:78
                acc = (acc * y + e) % m
        num.append(acc)
    h = D.extended_to_coeff(D.divide_by_vanishing_poly(num))       # vanishing/prover.rs:85-88
    assert len(h) == n * (cs_degree - 1)
    h_pieces = [h[a * n:(a + 1) * n] for a in range(cs_degree - 1)]
    h_blinds = [rng.scalar() for _ in h_pieces]
    for piece, b in zip(h_pieces, h_blinds):
        transcript.write_point(commit_c(piece, b))
    x = transcript.squeeze_challenge()                             # :566
    xn = pow(x, n, m)
    rotx = lambda r: D.rotate_omega(x, r)
    # ---- evaluations, :569-640 ----
    for pr in range(num_proofs):
        for col, r in vk.instance_queries:
            transcript.write_scalar(evalp(inst_polys[pr][col], rotx(r)))
    for pr in range(num_proofs):
        for col, r in vk.advice_queries:
            transcript.write_scalar(evalp(adv_polys[pr][col], rotx(r)))
    for col, r in vk.fixed_queries:
        transcript.write_scalar(evalp(fixed_polys[col], rotx(r)))
    h_poly, h_blind = [0] * n, 0                                   # vanishing/prover.rs:128-138
    for piece, b in zip(reversed(h_pieces), reversed(h_blinds)):
        h_poly = [(a * xn + p) % m for a, p in zip(h_poly, piece)]
        h_blind = (h_blind * xn + b) % m
    transcript.write_scalar(evalp(random_poly, x))
    for sp in sigma_polys:                                         # pk.permutation.evaluate, permutation/prover.rs:286-294
        transcript.write_scalar(evalp(sp, x))
    for pr in range(num_proofs):                                   # permutation/prover.rs:296-343
        sets = perms[pr]
        for a, st in enumerate(sets):
            transcript.write_scalar(evalp(st["poly"], x))
            transcript.write_scalar(evalp(st["poly"], rotx(1)))
            if a + 1 < len(sets):
                transcript.write_scalar(evalp(st["poly"], rotx(last_rot)))
    for pr in range(num_proofs):                                   # lookup/prover.rs:386-425
        for lk in lookups[pr]:
            for poly, r in ((lk["z_poly"], 0), (lk["z_poly"], 1), (lk["pi_poly"], 0), (lk["pi_poly"], -1), (lk["pt_poly"], 0)):
                transcript.write_scalar(evalp(poly, rotx(r)))
    # ---- the query list, :655-724, and the multi-point opening ----
    Q = pasta.ProverQuery
    queries = []
    for pr in range(num_proofs):
        for col, r in vk.instance_queries:
            queries.append(Q(rotx(r), inst_polys[pr][col], 1))
        for col, r in vk.advice_queries:
            queries.append(Q(rotx(r), adv_polys[pr][col], adv_blinds[pr][col]))
        sets = perms[pr]                                           # permutation/prover.rs:346-394
        for st in sets:
            queries.append(Q(x, st["poly"], st["blind"]))
            queries.append(Q(rotx(1), st["poly"], st["blind"]))
        for st in list(reversed(sets))[1:]:
            queries.append(Q(rotx(last_rot), st["poly"], st["blind"]))
        for lk in lookups[pr]:                                     # lookup/prover.rs:428-470
            queries += [Q(x, lk["z_poly"], lk["zb"]), Q(x, lk["pi_poly"], lk["bi"]), Q(x, lk["pt_poly"], lk["bt"]),
                        Q(rotx(-1), lk["pi_poly"], lk["bi"]), Q(rotx(1), lk["z_poly"], lk["zb"])]
    for col, r in vk.fixed_queries:
        queries.append(Q(rotx(r), fixed_polys[col], 1))
    for sp in sigma_polys:                                         # pk.permutation.open, permutation/prover.rs:397-409
        queries.append(Q(x, sp, 1))
    queries.append(Q(x, h_poly, h_blind))                          # vanishing/prover.rs:153-175
    queries.append(Q(x, random_poly, random_blind))
    pasta.multiopen_create_proof(c, g, w, u, rng, transcript, queries)                      # :726


# ------------------------------------------------------------------------------------------------------------------------
# The same prover composed from the engine's phase calls (halo2_b200: instance_commit / advice_commit, lookup_commit_permuted,
# permutation_commit, lookup_commit_product, vanishing_commit, the arguments' construct / evaluate / open, evaluate_columns /
# open_columns, multiopen.create_proof) -- the composition a patched plonk::create_proof would make, with each lookup
# compressed on the extended coset as lookup/prover.rs:172-176 does.  With the same seeded randomness it writes THE SAME PROOF
# BYTES as the oracle version above.  (tests/test_real_proof.py runs it over the ABI stand-in: transforms and group operations
# through the oracle, the device bodies on the host emulation.)
# ------------------------------------------------------------------------------------------------------------------------
def _to_ast(eng, e, fixed_l, advice_l, instance_l):
    """Expression::evaluate (circuit.rs:514-611) with the prover's closures (prover.rs:481-516): queries become leaves with rotations."""
    Ast = eng.Ast
    if e[0] == "struct":
        leaves = {"Fixed": fixed_l, "Advice": advice_l, "Instance": instance_l}[e[1]]
        return leaves[e[2]["column_index"]].with_rotation(e[2]["rotation"][2][0])
    name, args = e[1], e[2]
    if name == "Constant":
        return Ast.constant_term(args[0])
    if name == "Negated":
        return -_to_ast(eng, args[0], fixed_l, advice_l, instance_l)
    if name == "Sum":
        return _to_ast(eng, args[0], fixed_l, advice_l, instance_l) + _to_ast(eng, args[1], fixed_l, advice_l, instance_l)
    if name == "Product":
        return _to_ast(eng, args[0], fixed_l, advice_l, instance_l) * _to_ast(eng, args[1], fixed_l, advice_l, instance_l)
    if name == "Scaled":
        return _to_ast(eng, args[0], fixed_l, advice_l, instance_l) * args[1]
    raise ValueError(name)


# The Ast programs CrefProver evaluates, built from leaves alone so that a test can run exactly the prover's programs over
# columns of its own.  Column arguments are lists of leaves; a permutation or lookup argument's leaves come in its order.
def lookup_compression(eng, exprs, theta: int, fixed, advice, instance):
    """compress_expressions of lookup/prover.rs commit_permuted: a lookup's input or table expressions compressed by powers of theta (Lagrange basis)."""
    acc = eng.Ast.constant_term(0)
    for e in exprs:
        acc = acc * theta + _to_ast(eng, e, fixed, advice, instance)
    return acc


def vanishing_expressions(eng, vk: PV.PinnedKey, beta: int, gamma: int, delta: int, fixed, sigmas, lagrange, advice, instance, perm_z, lookups):
    """The h(X) constraints of one proof over the extended coset, in the reference's order (prover.rs:460-564): the gates, the
    permutation argument's (permutation/prover.rs construct), then each lookup's (lookup/prover.rs construct).  `lagrange`: the
    (l_0, l_blind, l_last) leaves; `perm_z`: one leaf per permutation set; `lookups`: (Z, A', S', A, S) leaves per lookup."""
    Ast = eng.Ast
    m = vk.scalar_modulus
    chunk_len = vk.degree() - 2
    last_rot = -(vk.blinding_factors() + 1)
    L0, LB, LL = lagrange
    one = Ast.constant_term(1)
    active = one - (LL + LB)
    exprs = [_to_ast(eng, gate, fixed, advice, instance) for gate in vk.gates]
    if perm_z:
        exprs.append((one - perm_z[0]) * L0)
        exprs.append((perm_z[-1] * perm_z[-1] - perm_z[-1]) * LL)
        for a in range(1, len(perm_z)):
            exprs.append((perm_z[a] - perm_z[a - 1].with_rotation(last_rot)) * L0)
        colc = lambda col: {"Advice": advice, "Fixed": fixed, "Instance": instance}[col[0]][col[1]]
        for a in range(len(perm_z)):
            cols = vk.permutation_columns[a * chunk_len:(a + 1) * chunk_len]
            left = perm_z[a].with_rotation(1)
            for col, sc in zip(cols, sigmas[a * chunk_len:(a + 1) * chunk_len]):
                left = left * (colc(col) + sc * beta + Ast.constant_term(gamma))
            right = perm_z[a]
            for j, col in enumerate(cols):
                right = right * (colc(col) + Ast.linear_term(beta * pow(delta, a * chunk_len + j, m) % m) + Ast.constant_term(gamma))
            exprs.append((left - right) * active)
    for Z_, A_, S_, CI_, CT_ in lookups:
        exprs.append((one - Z_) * L0)
        exprs.append((Z_ * Z_ - Z_) * LL)
        left = Z_.with_rotation(1) * (A_ + Ast.constant_term(beta)) * (S_ + Ast.constant_term(gamma))
        right = Z_ * (CI_ + Ast.constant_term(beta)) * (CT_ + Ast.constant_term(gamma))
        exprs.append((left - right) * active)
        exprs.append((A_ - S_) * L0)
        exprs.append((A_ - S_) * (A_ - A_.with_rotation(-1)) * active)
    return exprs


def proving_key(eng, D, fixed, sigma, blinding_factors: int):
    """A halo2_b200.ProvingKey of the Lagrange columns `fixed` and `sigma` (ints or (n, 32) uint8): every column, its
    coefficients and its extended coset, and l_0 / l_blind / l_last (keygen.rs:240-331).  The one key builder of the tests."""
    from halo2_b200.keygen import PermutationProvingKey
    n, bf = D.n, blinding_factors
    live = []

    def keep(p):
        live.append(p)
        return p

    def lag(vals):
        return keep(eng.ResidentPoly(D.field, n, vals if hasattr(vals, "dtype") else PV._ints_to_bytes([v % D.m for v in vals])))

    try:
        coeff = lambda p: D.lagrange_to_coeff_resident(p, out=keep(eng.ResidentPoly(D.field, n)))           # noqa: E731
        ext = lambda p: D.coeff_to_extended_resident(p, out=keep(eng.ResidentPoly(D.field, D.extended_len())))  # noqa: E731
        fv = [lag(f) for f in fixed]
        fp = [coeff(p) for p in fv]
        sv = [lag(s) for s in sigma]
        sp = [coeff(p) for p in sv]
        ls, tmp = [], []
        for rows in ({0}, set(range(n - bf, n)), {n - bf - 1}):
            co = coeff(lag([1 if r in rows else 0 for r in range(n)]))
            tmp += live[-2:]
            ls.append(ext(co))
        pk = eng.ProvingKey(fv, fp, [ext(p) for p in fp], PermutationProvingKey(sv, sp, [ext(p) for p in sp]), *ls)
    except BaseException:
        for p in live:
            p.close()
        raise
    for p in tmp:
        p.close()
    return pk


def close_proving_key(pk: dict) -> None:
    """Closes the key create_proof_engine stored in the dict `pk`, if it stored one."""
    key = pk.pop("key", None)
    if key is not None:
        key.close()


def prover_pk_bytes(pk) -> list:
    """The bytes of every polynomial of a halo2_b200.ProvingKey: fixed values, coefficients and cosets, then the permutation's,
    then l_0, l_blind and l_last."""
    return [p.download().tobytes() for p in pk._all()]


def create_proof_engine(eng, params, vk: PV.PinnedKey, fixed, sigma, advice, instances, rng, transcript, zeta: int, delta: int, pk=None,
                        on_construct=None) -> None:
    """plonk::create_proof (prover.rs:43-727) from the engine's phase calls.  `params`: halo2_b200.Params with u; `rng`:
    scalar() -> int, poly(n) -> (n, 32) bytes; `transcript`: tests/prover_replay.Blake2bTranscript (points as (64,) uint8).
    Columns are lists of ints or (n, 32) uint8 arrays; `advice[p]`, `instances[p]`: proof p's.

    `pk`: a halo2_b200.ProvingKey, used as it is (the caller closes it); None, for a key built from `fixed` and `sigma` and
    closed at the end; or a dict (see below).  `on_construct`, if given, is called as on_construct(extended evaluator,
    permuted lookups per proof, lookup expressions per proof over that evaluator, theta) once every argument is constructed,
    before anything is closed."""
    field = {pasta.P_MOD: "fp", pasta.Q_MOD: "fq"}[vk.scalar_modulus]
    bf = vk.blinding_factors()
    chunk_len = vk.degree() - 2
    D = eng.EvaluationDomain(field, vk.degree(), vk.k, zeta)
    assert D.extended_k == vk.extended_k and D.omega == vk.omega
    proofs = len(advice)
    owned = []                                                     # everything with a close(), freed at the end whatever happens

    def lookups_over(fixed_, adv_, inst_):
        ast = lambda e: _to_ast(eng, e, fixed_, adv_, inst_)       # noqa: E731
        return [([ast(e) for e in inp], [ast(e) for e in tab]) for inp, tab in vk.lookups]

    def columns_of(fixed_, adv_, inst_):
        return [{"Advice": adv_, "Fixed": fixed_, "Instance": inst_}[kind][i] for kind, i in vk.permutation_columns]

    try:
        if pk is None:
            pk = proving_key(eng, D, fixed, sigma, bf)
            owned.append(pk)
        elif isinstance(pk, dict):                                 # only for bench.py: it keeps the key between proofs in a dict
            if "key" not in pk:                                    # and frees it with close_proving_key
                pk["key"] = proving_key(eng, D, fixed, sigma, bf)
            pk = pk["key"]
        transcript.common_scalar(vk.transcript_repr())
        inst = eng.instance_commit(params, D, instances, bf)
        owned += [p for s in inst for p in s.values + s.polys + s.cosets]
        for s in inst:
            for cm in s.commitments:
                transcript.common_point(cm)
        adv = eng.advice_commit(params, D, advice, rng, bf)
        owned += [p for s in adv for p in s.values + s.polys + s.cosets]
        for s in adv:
            for cm in s.commitments:
                transcript.write_point(cm)
        ev_l = eng.Evaluator(D, "lagrange")
        FL = [ev_l.register_poly(p) for p in pk.fixed_values]
        AL = [[ev_l.register_poly(p) for p in s.values] for s in adv]
        IL = [[ev_l.register_poly(p) for p in s.values] for s in inst]
        theta = transcript.squeeze_challenge()
        permuted, cms = eng.lookup_commit_permuted(params, D, ev_l, [lookups_over(FL, AL[p], IL[p]) for p in range(proofs)], theta, bf, rng)
        owned += [q for per in permuted for lk in per for q in lk[:8]]
        for cm in cms:
            transcript.write_point(cm)
        beta = transcript.squeeze_challenge()
        gamma = transcript.squeeze_challenge()
        sets, cms = eng.permutation_commit(params, D, pk, [columns_of(pk.fixed_values, adv[p].values, inst[p].values) for p in range(proofs)],
                                           beta, gamma, delta, chunk_len, bf, rng)
        perm_committed = [eng.PermutationCommitted(per) for per in sets]
        owned += perm_committed
        for cm in cms:
            transcript.write_point(cm)
        products, cms = eng.lookup_commit_product(params, D, permuted, beta, gamma, bf, rng)
        lookup_committed = [eng.LookupCommitted(per, prods) for per, prods in zip(permuted, products)]
        owned += lookup_committed
        for cm in cms:
            transcript.write_point(cm)
        vanishing, cm = eng.vanishing_commit(params, D, rng)
        owned.append(vanishing)
        transcript.write_point(cm)
        y = transcript.squeeze_challenge()
        ev_e = eng.Evaluator(D, "extended")
        FC = [ev_e.register_poly(p) for p in pk.fixed_cosets]
        L0, LB, LL = (ev_e.register_poly(p) for p in (pk.l0, pk.l_blind, pk.l_last))
        exprs, perms, lookups, lookup_exprs = [], [], [], []
        for p in range(proofs):                                    # prover.rs:460-564: per proof the gates, the permutation, the lookups
            AC = [ev_e.register_poly(c) for c in adv[p].cosets]
            IC = [ev_e.register_poly(c) for c in inst[p].cosets]
            exprs += [_to_ast(eng, g, FC, AC, IC) for g in vk.gates]
            constructed, es = perm_committed[p].construct(ev_e, pk, columns_of(FC, AC, IC), L0, LB, LL, beta, gamma, delta, chunk_len, bf)
            perms.append(constructed)
            exprs += es
            lookup_exprs.append(lookups_over(FC, AC, IC))
            constructed, es = lookup_committed[p].construct(ev_e, lookup_exprs[-1], theta, beta, gamma, L0, LB, LL)
            owned.append(constructed)
            lookups.append(constructed)
            exprs += es
        if on_construct is not None:
            on_construct(ev_e, permuted, lookup_exprs, theta)
        vanishing, cms = vanishing.construct(params, D, ev_e, exprs, y, rng)
        owned.append(vanishing)
        for cm in cms:
            transcript.write_point(cm)
        x = transcript.squeeze_challenge()
        queries = ([s.polys for s in inst], [s.polys for s in adv], pk.fixed_polys, vk.instance_queries, vk.advice_queries, vk.fixed_queries)
        ie, ae, fe = eng.evaluate_columns(D, x, *queries)
        for e in [v for per in ie for v in per] + [v for per in ae for v in per] + fe:
            transcript.write_scalar(e)
        vanishing, random_eval = vanishing.evaluate(D, x)
        owned.append(vanishing)
        transcript.write_scalar(random_eval)
        for e in eng.permutation_key_evaluate(pk, D, x):
            transcript.write_scalar(e)
        perm_ev, lookup_ev = [], []
        for c in perms:
            ev, es = c.evaluate(D, x)
            perm_ev.append(ev)
            for e in es:
                transcript.write_scalar(e)
        for c in lookups:
            ev, es = c.evaluate(D, x)
            lookup_ev.append(ev)
            for e in es:
                transcript.write_scalar(e)
        iq, aq, fq = eng.open_columns(D, x, queries[0], queries[1], [s.blinds for s in adv], *queries[2:])
        opened = []
        for p in range(proofs):
            opened += iq[p] + aq[p] + perm_ev[p].open(x) + lookup_ev[p].open(x)
        opened += fq + eng.permutation_key_open(pk, x) + vanishing.open(x)
        eng.multiopen.create_proof(params, rng, transcript, opened)
    finally:
        for o in owned:
            o.close()


# ------------------------------------------------------------------------------------------------------------------------
# The same prover on the C RESTATEMENT of the reference algorithms (oracle/halo2_oracle.c through oracle/cref.py): the timed
# CPU arm for real proofs at benchmark sizes, where the big-integer version above would take minutes.  Same order, same
# randomness, THE SAME PROOF BYTES (tests/test_real_proof.py).  `hot_s` accumulates only the reference's hot-path calls --
# best_multiexp per commitment, the best_fft-based transforms, eval_polynomial, kate_division, the opening's round loop -- as
# tests/prover_replay.CpuArm does; the elementwise work (expressions, products, folds: Python integers or the C evaluator)
# is not counted.
# ------------------------------------------------------------------------------------------------------------------------
class CrefProver:
    def __init__(self, cref, curve: str, field: str, g, g_lagrange, w, u, threads: int):
        import numpy as np
        self.np, self.cref, self.curve, self.field, self.threads = np, cref, curve, field, threads
        self.bases = np.concatenate([g, w])
        self.bases_l = np.concatenate([g_lagrange, w])
        self.gwu = np.concatenate([g, w, u])
        self.hot_s, self.by_kind = 0.0, {}

    def _t(self, kind, t0):
        import time
        dt = time.time() - t0
        self.hot_s += dt
        self.by_kind[kind] = self.by_kind.get(kind, 0.0) + dt

    def commit(self, poly, blind: int, lagrange: bool):
        import time
        t0 = time.time()
        out = self.cref.best_multiexp(self.curve, self.np.concatenate([poly, self.cref.ints_to_bytes([blind])]),
                                      self.bases_l if lagrange else self.bases, self.threads)
        self._t("commit_lagrange" if lagrange else "commit", t0)
        return out

    def create_proof(self, vk: PV.PinnedKey, fixed, sigma, advice, instances, rng, transcript, zeta: int, delta: int) -> None:
        """plonk::create_proof; columns as (n, 32) uint8 arrays or int lists; `transcript`: tests/prover_replay.Blake2bTranscript."""
        import time
        from halo2_b200.evaluator import Ast, AstLeaf, compile_ast           # the pure-host flattener of the Ast (no GPU involved)
        np, cref, field = self.np, self.cref, self.field
        m = vk.scalar_modulus
        k, n = vk.k, 1 << vk.k
        bf = vk.blinding_factors()
        usable = n - (bf + 1)
        cs_degree = vk.degree()
        chunk_len = cs_degree - 2
        D = pasta.EvaluationDomain(field, cs_degree, k, zeta)
        L = D.extended_len()
        stride = 1 << (D.extended_k - k)
        B = lambda col: col if hasattr(col, "dtype") else cref.ints_to_bytes([v % m for v in col])
        I = cref.bytes_to_ints

        def timed(kind, fn, *a):
            t0 = time.time()
            out = fn(*a)
            self._t(kind, t0)
            return out

        l2c = lambda v: timed("lagrange_to_coeff", cref.ifft, field, v, D.omega_inv, k, D.ifft_divisor, self.threads)
        c2e = lambda p: timed("coeff_to_extended", cref.coeff_to_extended, field, p, k, D.extended_k, zeta, D.extended_omega, self.threads)
        evalp = lambda p, x: timed("eval_polynomial", cref.eval_polynomial, field, p, x)

        def run_ast(ast, polys, extended):                         # Evaluator::evaluate: the C evaluator, not counted as hot
            log_n = D.extended_k if extended else k
            code, consts = compile_ast(ast, m, stride if extended else 1)
            return cref.ast_eval(field, np.stack(polys), log_n, code, consts, D.extended_omega if extended else D.omega, zeta if extended else 1, self.threads)

        class Eng:                                                 # what _to_ast needs from an engine namespace
            pass
        Eng.Ast = Ast
        num_proofs = len(advice)
        transcript.common_scalar(vk.transcript_repr())
        inst_l, inst_p, inst_c = [], [], []
        for inst in instances:
            vals = [B(list(col) + [0] * (n - len(col))) for col in inst]
            for v in vals:
                transcript.common_point(self.commit(v, 1, True))
            polys = [l2c(v) for v in vals]
            inst_l.append(vals), inst_p.append(polys), inst_c.append([c2e(p) for p in polys])
        adv_l, adv_p, adv_c, adv_b = [], [], [], []
        for cols in advice:
            vals = []
            for col in cols:
                v = B(col).copy()
                v[usable:] = cref.ints_to_bytes([rng.scalar() for _ in range(n - usable)])
                vals.append(v)
            blinds = [rng.scalar() for _ in vals]
            for v, b in zip(vals, blinds):
                transcript.write_point(self.commit(v, b, True))
            polys = [l2c(v) for v in vals]
            adv_l.append(vals), adv_p.append(polys), adv_c.append([c2e(p) for p in polys]), adv_b.append(blinds)
        fixed_l = [B(f) for f in fixed]
        fixed_p = [cref.ifft(field, f, D.omega_inv, k, D.ifft_divisor, self.threads) for f in fixed_l]       # the proving key's: not per proof
        fixed_c = [cref.coeff_to_extended(field, p, k, D.extended_k, zeta, D.extended_omega, self.threads) for p in fixed_p]
        sigma_l = [B(s) for s in sigma]
        sigma_p = [cref.ifft(field, s, D.omega_inv, k, D.ifft_divisor, self.threads) for s in sigma_l]
        sigma_c = [cref.coeff_to_extended(field, p, k, D.extended_k, zeta, D.extended_omega, self.threads) for p in sigma_p]
        ind = lambda rows: cref.coeff_to_extended(field, cref.ifft(field, cref.ints_to_bytes([1 if r in rows else 0 for r in range(n)]), D.omega_inv, k,
                                                                 D.ifft_divisor, self.threads), k, D.extended_k, zeta, D.extended_omega, self.threads)
        l0_c, l_blind_c, l_last_c = ind({0}), ind(set(range(n - bf, n))), ind({n - bf - 1})
        # leaf numbering of the Lagrange-basis programs: fixed, then per proof advice and instance
        lag_polys = list(fixed_l)
        FL = [AstLeaf(i) for i in range(len(fixed_l))]
        AL, IL = [], []
        for pr in range(num_proofs):
            AL.append([AstLeaf(len(lag_polys) + i) for i in range(len(adv_l[pr]))])
            lag_polys += adv_l[pr]
            IL.append([AstLeaf(len(lag_polys) + i) for i in range(len(inst_l[pr]))])
            lag_polys += inst_l[pr]
        theta = transcript.squeeze_challenge()
        lookups = []
        for pr in range(num_proofs):
            per = []
            for inp, tab in vk.lookups:
                ci, ct = (run_ast(lookup_compression(Eng, exprs, theta, FL, AL[pr], IL[pr]), lag_polys, False) for exprs in (inp, tab))
                res = cref.permute_expression_pair(ci, ct, usable)
                assert res is not None, "an input value does not occur in the table"
                pi = np.concatenate([res[0], cref.ints_to_bytes([rng.scalar() for _ in range(bf + 1)])])
                pt = np.concatenate([res[1], cref.ints_to_bytes([rng.scalar() for _ in range(bf + 1)])])
                bi = rng.scalar()
                bt = rng.scalar()
                transcript.write_point(self.commit(pi, bi, True))
                transcript.write_point(self.commit(pt, bt, True))
                per.append({"ci": ci, "ct": ct, "pi": pi, "pt": pt, "pi_poly": l2c(pi), "pt_poly": l2c(pt), "bi": bi, "bt": bt})
            lookups.append(per)
        beta = transcript.squeeze_challenge()
        gamma = transcript.squeeze_challenge()
        omega_pows = [1] * n
        for i in range(1, n):
            omega_pows[i] = omega_pows[i - 1] * D.omega % m
        col_vals = lambda pr, col: {"Advice": adv_l[pr], "Fixed": fixed_l, "Instance": inst_l[pr]}[col[0]][col[1]]
        perms = []
        for pr in range(num_proofs):                               # permutation/prover.rs:42-173 on Python integers (elementwise: not counted)
            sets, last_z = [], 1
            for ci_ in range(0, len(vk.permutation_columns), chunk_len):
                cols = vk.permutation_columns[ci_:ci_ + chunk_len]
                mod = [1] * n
                vals_i = [I(col_vals(pr, col)) for col in cols]
                for v, sg in zip(vals_i, sigma_l[ci_:ci_ + chunk_len]):
                    mod = [a * ((beta * s_ + gamma + x_) % m) % m for a, s_, x_ in zip(mod, I(sg), v)]
                from halo2_b200.verifier import batch_invert         # pure host arithmetic (Montgomery's trick)
                mod = batch_invert(mod, m)
                for j, v in enumerate(vals_i):
                    d_j = pow(delta, ci_ + j, m) * beta % m
                    mod = [a * ((d_j * w_ + gamma + x_) % m) % m for a, w_, x_ in zip(mod, omega_pows, v)]
                z = [last_z]
                for row in range(1, n):
                    z.append(z[row - 1] * mod[row - 1] % m)
                for row in range(n - bf, n):
                    z[row] = rng.scalar()
                last_z = z[n - (bf + 1)]
                blind = rng.scalar()
                zb = cref.ints_to_bytes(z)
                transcript.write_point(self.commit(zb, blind, True))
                zp = l2c(zb)
                sets.append({"poly": zp, "coset": c2e(zp), "blind": blind})
            perms.append(sets)
        for pr in range(num_proofs):
            for lk in lookups[pr]:
                from halo2_b200.verifier import batch_invert
                pi_i, pt_i, ci_i, ct_i = I(lk["pi"]), I(lk["pt"]), I(lk["ci"]), I(lk["ct"])
                prod = batch_invert([(beta + a) * (gamma + s_) % m for a, s_ in zip(pi_i, pt_i)], m)
                prod = [p * ((a + beta) % m) % m * ((s_ + gamma) % m) % m for p, a, s_ in zip(prod, ci_i, ct_i)]
                z, state = [], 1
                for cur in [1] + prod:
                    state = state * cur % m
                    z.append(state)
                z = z[:n - bf] + [rng.scalar() for _ in range(bf)]
                lk["zb"] = rng.scalar()
                zbytes = cref.ints_to_bytes(z)
                transcript.write_point(self.commit(zbytes, lk["zb"], True))
                lk["z_poly"] = l2c(zbytes)
        random_poly = B(rng.poly(n))
        random_blind = rng.scalar()
        transcript.write_point(self.commit(random_poly, random_blind, False))
        y = transcript.squeeze_challenge()
        # ---- h(X): the same Ast as the engine version, evaluated by the C evaluator over the extended cosets ----
        ext_polys = list(fixed_c) + list(sigma_c) + [l0_c, l_blind_c, l_last_c]
        FC = [AstLeaf(i) for i in range(len(fixed_c))]
        SC = [AstLeaf(len(fixed_c) + i) for i in range(len(sigma_c))]
        L0, LB, LL = (AstLeaf(len(fixed_c) + len(sigma_c) + i) for i in range(3))

        def reg(p):
            ext_polys.append(p)
            return AstLeaf(len(ext_polys) - 1)

        exprs = []
        for pr in range(num_proofs):
            AC = [reg(p) for p in adv_c[pr]]
            IC = [reg(p) for p in inst_c[pr]]
            ZC = [reg(s_["coset"]) for s_ in perms[pr]]
            LK = [tuple(reg(c2e(lk[kk])) for kk in ("z_poly", "pi_poly", "pt_poly")) + tuple(reg(c2e(l2c(lk[kk]))) for kk in ("ci", "ct"))
                  for lk in lookups[pr]]
            exprs += vanishing_expressions(Eng, vk, beta, gamma, delta, FC, SC, (L0, LB, LL), AC, IC, ZC, LK)
        last_rot = -(bf + 1)
        h_ext = run_ast(Ast.distribute_powers(exprs, y), ext_polys, True)
        tev = cref.ints_to_bytes(D.t_evaluations)                  # divide_by_vanishing_poly (domain.rs:329-348) as an elementwise program
        tfull = tev[np.arange(L) % len(D.t_evaluations)]
        h_ext = cref.ast_eval(field, np.stack([h_ext, tfull]), D.extended_k, np.array([[0, 0, 0, 0], [0, 1, 0, 0], [4, 0, 0, 0]], dtype=np.uint32), [],
                              D.extended_omega, zeta, self.threads)
        h = timed("extended_to_coeff", cref.extended_to_coeff, field, h_ext, D.extended_k, D.extended_omega_inv, D.extended_ifft_divisor, zeta,
                  n * (cs_degree - 1), self.threads)
        h_pieces = [h[a * n:(a + 1) * n] for a in range(cs_degree - 1)]
        h_blinds = [rng.scalar() for _ in h_pieces]
        for piece, b in zip(h_pieces, h_blinds):
            transcript.write_point(self.commit(piece, b, False))
        x = transcript.squeeze_challenge()
        xn = pow(x, n, m)
        rotx = lambda r: D.rotate_omega(x, r)
        for pr in range(num_proofs):
            for col, r in vk.instance_queries:
                transcript.write_scalar(evalp(inst_p[pr][col], rotx(r)))
        for pr in range(num_proofs):
            for col, r in vk.advice_queries:
                transcript.write_scalar(evalp(adv_p[pr][col], rotx(r)))
        for col, r in vk.fixed_queries:
            transcript.write_scalar(evalp(fixed_p[col], rotx(r)))
        transcript.write_scalar(evalp(random_poly, x))
        for sp in sigma_p:
            transcript.write_scalar(evalp(sp, x))
        for pr in range(num_proofs):
            sets = perms[pr]
            for a, st in enumerate(sets):
                transcript.write_scalar(evalp(st["poly"], x))
                transcript.write_scalar(evalp(st["poly"], rotx(1)))
                if a + 1 < len(sets):
                    transcript.write_scalar(evalp(st["poly"], rotx(last_rot)))
        for pr in range(num_proofs):
            for lk in lookups[pr]:
                for poly, r in ((lk["z_poly"], 0), (lk["z_poly"], 1), (lk["pi_poly"], 0), (lk["pi_poly"], -1), (lk["pt_poly"], 0)):
                    transcript.write_scalar(evalp(poly, rotx(r)))
        h_poly, h_blind = [0] * n, 0                               # fold of the pieces by x^n: elementwise, Python integers
        for piece, b in zip(reversed(h_pieces), reversed(h_blinds)):
            h_poly = [(a * xn + p) % m for a, p in zip(h_poly, I(piece))]
            h_blind = (h_blind * xn + b) % m
        queries = []                                               # (point, key, polynomial bytes, blind)
        for pr in range(num_proofs):
            queries += [(rotx(r), ("i", pr, col), inst_p[pr][col], 1) for col, r in vk.instance_queries]
            queries += [(rotx(r), ("a", pr, col), adv_p[pr][col], adv_b[pr][col]) for col, r in vk.advice_queries]
            sets = perms[pr]
            for a, st in enumerate(sets):
                queries += [(x, ("z", pr, a), st["poly"], st["blind"]), (rotx(1), ("z", pr, a), st["poly"], st["blind"])]
            for a in reversed(range(len(sets) - 1)):
                queries.append((rotx(last_rot), ("z", pr, a), sets[a]["poly"], sets[a]["blind"]))
            for li, lk in enumerate(lookups[pr]):
                queries += [(x, ("lz", pr, li), lk["z_poly"], lk["zb"]), (x, ("li", pr, li), lk["pi_poly"], lk["bi"]), (x, ("lt", pr, li), lk["pt_poly"], lk["bt"]),
                            (rotx(-1), ("li", pr, li), lk["pi_poly"], lk["bi"]), (rotx(1), ("lz", pr, li), lk["z_poly"], lk["zb"])]
        queries += [(rotx(r), ("f", col), fixed_p[col], 1) for col, r in vk.fixed_queries]
        queries += [(x, ("s", i), sp, 1) for i, sp in enumerate(sigma_p)]
        queries.append((x, ("h",), cref.ints_to_bytes(h_poly), h_blind))
        queries.append((x, ("r",), random_poly, random_blind))
        self._multiopen(vk, rng, transcript, queries, m, k)

    def _multiopen(self, vk, rng, transcript, queries, m, k):
        """poly/multiopen/prover.rs:18-124 + poly/commitment/prover.rs:36-151: the folds on Python integers (elementwise, not counted), the
        divisions / evaluations / commitments / round loop on the C restatement."""
        import time
        np, cref, field = self.np, self.cref, self.field
        n = 1 << k
        I = cref.bytes_to_ints

        class Q:                                                   # pasta.construct_intermediate_sets wants objects with these members
            def __init__(self, point, key, poly, blind):
                self.point, self._k, self.poly, self.blind = point, key, poly, blind

            def key(self):
                return self._k

            def value(self):
                return (self.poly, self.blind)

        x1 = transcript.squeeze_challenge()
        x2 = transcript.squeeze_challenge()
        poly_map, point_sets = pasta.construct_intermediate_sets([Q(*q) for q in queries], prover=True)
        q_polys, q_blinds = [None] * len(point_sets), [0] * len(point_sets)
        for data in poly_map:
            s_ = data["set_index"]
            poly = I(data["commitment"])
            q_polys[s_] = poly if q_polys[s_] is None else [(a * x1 + b) % m for a, b in zip(q_polys[s_], poly)]
            q_blinds[s_] = (q_blinds[s_] * x1 + data["blind"]) % m
        q_prime = None
        for points, poly in zip(point_sets, q_polys):
            cur = cref.ints_to_bytes(poly)
            for pt in points:
                t0 = time.time()
                quo = cref.kate_division(field, cur, pt)
                self._t("kate_division", t0)
                cur = np.concatenate([quo, np.zeros((n - quo.shape[0], 32), dtype=np.uint8)])
            cur = I(cur)
            q_prime = cur if q_prime is None else [(a * x2 + b) % m for a, b in zip(q_prime, cur)]
        q_prime_blind = rng.scalar()
        transcript.write_point(self.commit(cref.ints_to_bytes(q_prime), q_prime_blind, False))
        x3 = transcript.squeeze_challenge()
        for q in q_polys:
            t0 = time.time()
            e = cref.eval_polynomial(field, cref.ints_to_bytes(q), x3)
            self._t("eval_polynomial", t0)
            transcript.write_scalar(e)
        x4 = transcript.squeeze_challenge()
        p_poly, p_blind = q_prime, q_prime_blind
        for poly, blind in zip(q_polys, q_blinds):
            p_poly = [(a * x4 + b) % m for a, b in zip(p_poly, poly)]
            p_blind = (p_blind * x4 + blind) % m
        # commitment::create_proof (poly/commitment/prover.rs:36-151)
        drawn = rng.poly(n)
        s = I(drawn) if hasattr(drawn, "dtype") else [v % m for v in drawn]
        sb = cref.ints_to_bytes(s)
        t0 = time.time()
        s_at = cref.eval_polynomial(field, sb, x3)
        self._t("eval_polynomial", t0)
        s[0] = (s[0] - s_at) % m
        s_blind = rng.scalar()
        transcript.write_point(self.commit(cref.ints_to_bytes(s), s_blind, False))
        xi = transcript.squeeze_challenge()
        z = transcript.squeeze_challenge()
        pp = [(a * xi + b) % m for a, b in zip(s, p_poly)]
        t0 = time.time()
        v = cref.eval_polynomial(field, cref.ints_to_bytes(pp), x3)
        self._t("eval_polynomial", t0)
        pp[0] = (pp[0] - v) % m
        f = (s_blind * xi + p_blind) % m
        rand = [(rng.scalar(), rng.scalar()) for _ in range(k)]
        us = []

        def challenge(j, l_xy, r_xy):
            transcript.write_point(l_xy)
            transcript.write_point(r_xy)
            us.append(transcript.squeeze_challenge())
            return us[-1]

        t0 = time.time()
        _, _, c_val = cref.ipa_rounds_transcript(self.curve, self.gwu, k, cref.ints_to_bytes(pp), x3, z, challenge,
                                                 cref.ints_to_bytes([a for a, _ in rand]), cref.ints_to_bytes([b for _, b in rand]), min(self.threads, 16))
        self._t("ipa", t0)
        for (lr, rr), uj in zip(rand, us):
            f = (f + lr * pow(uj, -1, m) + rr * uj) % m
        transcript.write_scalar(c_val)
        transcript.write_scalar(f)
