"""plonk::create_proof composed from package calls only, for the argument tests: instance_commit / advice_commit,
lookup_commit_permuted, permutation_commit, lookup_commit_product, vanishing_commit, the gates' expressions with the
permutation and lookup arguments' construct, vanishing construct, evaluate_columns and every argument's evaluate in the
reference's write order, the opens, and multiopen.create_proof.  Also:

- a proving key built from Lagrange columns with the same transforms create_proof_engine uses;
- a circuit whose lookup is not linear in the columns (a selector-gated input and table over two rows) with a pinned key,
  so that compressing on the coset and extending the compressed Lagrange column give different polynomials;
- the ABI stand-in with every entry point the composition reaches.
"""
from __future__ import annotations

import contextlib

import numpy as np

from oracle import cref, pasta
from tests import columns_cases as CC
from tests import fake_engine
from tests import plonk_prover as PP
from tests import vanishing_cases as VC
from tests.test_lookup_permuted_oracle import PermutedFake


# ---- the proving key ---------------------------------------------------------------------------------------------------
def proving_key(h2, D, fixed, sigma, blinding_factors: int):
    """A halo2_b200.ProvingKey of the Lagrange columns `fixed` and `sigma` (ints or (n, 32) uint8), every form made the
    way create_proof_engine makes its key, and l_0 / l_blind / l_last (keygen.rs:306-325)."""
    from halo2_b200.keygen import PermutationProvingKey
    n, bf = D.n, blinding_factors
    live = []

    def keep(p):
        live.append(p)
        return p

    def lag(vals):
        return keep(h2.ResidentPoly(D.field, n, vals if hasattr(vals, "dtype") else cref.ints_to_bytes([v % D.m for v in vals])))

    try:
        coeff = lambda p: D.lagrange_to_coeff_resident(p, out=keep(h2.ResidentPoly(D.field, n)))           # noqa: E731
        ext = lambda p: D.coeff_to_extended_resident(p, out=keep(h2.ResidentPoly(D.field, D.extended_len())))  # noqa: E731
        fv = [lag(f) for f in fixed]
        fp = [coeff(p) for p in fv]
        sv = [lag(s) for s in sigma]
        sp = [coeff(p) for p in sv]
        ls, tmp = [], []
        for rows in ({0}, set(range(n - bf, n)), {n - bf - 1}):
            co = coeff(lag([1 if r in rows else 0 for r in range(n)]))
            tmp += live[-2:]
            ls.append(ext(co))
        pk = h2.ProvingKey(fv, fp, [ext(p) for p in fp], PermutationProvingKey(sv, sp, [ext(p) for p in sp]), *ls)
    except BaseException:
        for p in live:
            p.close()
        raise
    for p in tmp:
        p.close()
    return pk


# ---- the composition ---------------------------------------------------------------------------------------------------
def create_proof_package(h2, params, D, pk, vk, advice, instances, rng, transcript, delta: int, on_construct=None) -> None:
    """plonk::create_proof (prover.rs:43-727) from package calls.  `pk`: a halo2_b200.ProvingKey; `advice[p]`, `instances[p]`:
    proof p's columns; `rng`: scalar() and poly(n); `transcript`: tests/prover_replay.Blake2bTranscript.  on_construct, if
    given, is called as on_construct(extended evaluator, permuted, lookups per proof over it, theta) once every argument is
    constructed, before anything is closed."""
    bf = vk.blinding_factors()
    chunk_len = vk.degree() - 2
    proofs = len(advice)
    owned = []                                                     # everything with a close(), freed at the end whatever happens

    def lookups_over(fixed, adv, inst):
        ast = lambda e: PP._to_ast(h2, e, fixed, adv, inst)       # noqa: E731
        return [([ast(e) for e in inp], [ast(e) for e in tab]) for inp, tab in vk.lookups]

    def columns_of(fixed, adv, inst):
        return [{"Advice": adv, "Fixed": fixed, "Instance": inst}[kind][i] for kind, i in vk.permutation_columns]

    try:
        transcript.common_scalar(vk.transcript_repr())
        inst = h2.instance_commit(params, D, instances, bf)
        owned += [p for s in inst for p in s.values + s.polys + s.cosets]
        for s in inst:
            for cm in s.commitments:
                transcript.common_point(cm)
        adv = h2.advice_commit(params, D, advice, rng, bf)
        owned += [p for s in adv for p in s.values + s.polys + s.cosets]
        for s in adv:
            for cm in s.commitments:
                transcript.write_point(cm)
        ev_l = h2.Evaluator(D, "lagrange")
        FL = [ev_l.register_poly(p) for p in pk.fixed_values]
        AL = [[ev_l.register_poly(p) for p in s.values] for s in adv]
        IL = [[ev_l.register_poly(p) for p in s.values] for s in inst]
        theta = transcript.squeeze_challenge()
        permuted, cms = h2.lookup_commit_permuted(params, D, ev_l, [lookups_over(FL, AL[p], IL[p]) for p in range(proofs)], theta, bf, rng)
        owned += [q for per in permuted for lk in per for q in lk[:8]]
        for cm in cms:
            transcript.write_point(cm)
        beta = transcript.squeeze_challenge()
        gamma = transcript.squeeze_challenge()
        sets, cms = h2.permutation_commit(params, D, pk, [columns_of(pk.fixed_values, adv[p].values, inst[p].values) for p in range(proofs)],
                                          beta, gamma, delta, chunk_len, bf, rng)
        perm_committed = [h2.PermutationCommitted(per) for per in sets]
        owned += perm_committed
        for cm in cms:
            transcript.write_point(cm)
        products, cms = h2.lookup_commit_product(params, D, permuted, beta, gamma, bf, rng)
        lookup_committed = [h2.LookupCommitted(per, prods) for per, prods in zip(permuted, products)]
        owned += lookup_committed
        for cm in cms:
            transcript.write_point(cm)
        vanishing, cm = h2.vanishing_commit(params, D, rng)
        owned.append(vanishing)
        transcript.write_point(cm)
        y = transcript.squeeze_challenge()
        ev_e = h2.Evaluator(D, "extended")
        FC = [ev_e.register_poly(p) for p in pk.fixed_cosets]
        L0, LB, LL = (ev_e.register_poly(p) for p in (pk.l0, pk.l_blind, pk.l_last))
        exprs, perms, lookups, lookup_exprs = [], [], [], []
        for p in range(proofs):                                    # prover.rs:460-564: per proof the gates, the permutation, the lookups
            AC = [ev_e.register_poly(c) for c in adv[p].cosets]
            IC = [ev_e.register_poly(c) for c in inst[p].cosets]
            exprs += [PP._to_ast(h2, g, FC, AC, IC) for g in vk.gates]
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
        ie, ae, fe = h2.evaluate_columns(D, x, *queries)
        for e in [v for per in ie for v in per] + [v for per in ae for v in per] + fe:
            transcript.write_scalar(e)
        vanishing, random_eval = vanishing.evaluate(D, x)
        owned.append(vanishing)
        transcript.write_scalar(random_eval)
        for e in h2.permutation_key_evaluate(pk, D, x):
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
        iq, aq, fq = h2.open_columns(D, x, queries[0], queries[1], [s.blinds for s in adv], *queries[2:])
        opened = []
        for p in range(proofs):
            opened += iq[p] + aq[p] + perm_ev[p].open(x) + lookup_ev[p].open(x)
        opened += fq + h2.permutation_key_open(pk, x) + vanishing.open(x)
        h2.multiopen.create_proof(params, rng, transcript, opened)
    finally:
        for o in owned:
            o.close()


# ---- a lookup that is not linear in the columns ------------------------------------------------------------------------
NL_ADVICE = 8                      # a, then b0 ... b6: copies of a, so that the permutation spans three sets
NL_BLINDING_FACTORS = 5            # a is queried at two rotations: max(3, 2) + 2
NL_DEGREE = 6                      # the lookup's: 2 + deg(q a) + deg(q t0)


def _hex(v: int) -> str:
    return "0x%064x" % v


def nonlinear_columns(k: int, m: int, omega: int, delta: int, base: int):
    """(fixed [q, t0, t1], sigma (10 columns), advice [a, b0 ... b6], instance [[base + 1]]) as Lagrange values.

    The lookup (q a, q a(omega X)) in (q t0, q t1) holds with a = t0 = base + row and t1 = base + row + 1, where the selector
    q is 1 on rows 0 ... usable - 2 and 0 elsewhere; a row with q = 0 looks up (0, 0), which row usable - 1 of the table
    holds.  The gate q (b0 - a) holds because every b_i equals a.  The permutation columns are a, b0 ... b6, the instance
    column and t0; the copies chain a, b0, ..., b6 on rows 1 ... 6, tie the instance's row 0 to a's row 1 and t0's row 2
    to a's row 2."""
    n = 1 << k
    usable = n - NL_BLINDING_FACTORS - 1
    q = [1 if r < usable - 1 else 0 for r in range(n)]
    t0 = [(base + r) % m for r in range(n)]
    t1 = [(base + r + 1) % m for r in range(n)]
    a = list(t0)
    advice = [list(a) for _ in range(NL_ADVICE)]
    ncols = NL_ADVICE + 2
    mapping = [[(i, j) for j in range(n)] for i in range(ncols)]
    aux = [[(i, j) for j in range(n)] for i in range(ncols)]
    sizes = [[1] * n for _ in range(ncols)]

    def copy(lc, lr, rc, rr):                                      # permutation/keygen.rs:45-100
        left, right = aux[lc][lr], aux[rc][rr]
        if left == right:
            return
        if sizes[left[0]][left[1]] < sizes[right[0]][right[1]]:
            left, right = right, left
        sizes[left[0]][left[1]] += sizes[right[0]][right[1]]
        i = right
        while True:
            aux[i[0]][i[1]] = left
            i = mapping[i[0]][i[1]]
            if i == right:
                break
        mapping[lc][lr], mapping[rc][rr] = mapping[rc][rr], mapping[lc][lr]

    for r in range(1, min(7, usable)):
        for i in range(NL_ADVICE - 1):
            copy(i, r, i + 1, r)
    copy(NL_ADVICE, 0, 0, 1)
    copy(NL_ADVICE + 1, 2, 0, 2)
    omega_powers = [1] * n
    for j in range(1, n):
        omega_powers[j] = omega_powers[j - 1] * omega % m
    sigma = [[pow(delta, mapping[i][j][0], m) * omega_powers[mapping[i][j][1]] % m for j in range(n)] for i in range(ncols)]
    return [q, t0, t1], sigma, advice, [[(base + 1) % m]]


def nonlinear_key_text(k: int, extended_k: int, base_modulus: int, scalar_modulus: int, omega: int, fixed_commitments,
                       permutation_commitments) -> str:
    """The pinned key of nonlinear_columns' circuit in the shape of `{:#?}` of PinnedVerificationKey."""
    def q(kind, qi, ci, rot=0):
        return f"{kind} {{\nquery_index: {qi},\ncolumn_index: {ci},\nrotation: Rotation(\n{rot},\n),\n}},"
    prod = lambda x, y: f"Product(\n{x}\n{y}\n),"                  # noqa: E731
    col = lambda idx, kind: f"Column {{\nindex: {idx},\ncolumn_type: {kind},\n}},"  # noqa: E731
    query = lambda idx, kind, rot=0: f"(\n{col(idx, kind)}\nRotation(\n{rot},\n),\n),"  # noqa: E731
    pts = lambda ps: "\n".join(f"({_hex(x)}, {_hex(y)})," for x, y in ps)  # noqa: E731
    sel, a, a_next, b0 = q("Fixed", 0, 0), q("Advice", 0, 0), q("Advice", 1, 0, 1), q("Advice", 2, 1)
    t0, t1 = q("Fixed", 1, 1), q("Fixed", 2, 2)
    gate = prod(sel, f"Sum(\n{b0}\nNegated(\n{a}\n),\n),")
    advice_queries = [query(0, "Advice"), query(0, "Advice", 1)] + [query(i, "Advice") for i in range(1, NL_ADVICE)]
    perm_cols = [col(i, "Advice") for i in range(NL_ADVICE)] + [col(0, "Instance"), col(1, "Fixed")]
    return "\n".join([
        "PinnedVerificationKey {",
        f'base_modulus: "0x{base_modulus:064x}",', f'scalar_modulus: "0x{scalar_modulus:064x}",',
        "domain: PinnedEvaluationDomain {", f"k: {k},", f"extended_k: {extended_k},", f"omega: {_hex(omega)},", "},",
        "cs: PinnedConstraintSystem {", "num_fixed_columns: 3,", f"num_advice_columns: {NL_ADVICE},", "num_instance_columns: 1,",
        "num_selectors: 0,",
        "gates: [", gate, "],",
        "advice_queries: [", *advice_queries, "],",
        "instance_queries: [", query(0, "Instance"), "],",
        "fixed_queries: [", query(0, "Fixed"), query(1, "Fixed"), query(2, "Fixed"), "],",
        "permutation: Argument {", "columns: [", *perm_cols, "],", "},",
        "lookups: [", "Argument {", "input_expressions: [", prod(sel, a), prod(sel, a_next), "],",
        "table_expressions: [", prod(sel, t0), prod(sel, t1), "],", "},", "],",
        "constants: [],", "minimum_degree: None,", "},",
        "fixed_commitments: [", pts(fixed_commitments), "],",
        "permutation: VerifyingKey {", "commitments: [", pts(permutation_commitments), "],", "},",
        "}"])


def nonlinear_case(h2, k: int, commit_lagrange, zeta: int, delta: int, base: int = 1000):
    """(vk, domain, fixed, sigma, advice, instance) of the circuit at k; commit_lagrange(values) -> (x, y) commits a column with
    Blind::default() for the key."""
    m = pasta.P_MOD
    omega = pasta.omega_for_k("fp", k)
    fixed, sigma, advice, instance = nonlinear_columns(k, m, omega, delta, base)
    D = h2.EvaluationDomain("fp", NL_DEGREE, k, zeta)
    vk_text = nonlinear_key_text(k, D.extended_k, pasta.Q_MOD, m, D.omega, [commit_lagrange(c) for c in fixed], [commit_lagrange(s) for s in sigma])
    from tests import plonk_verifier as PV
    vk = PV.PinnedKey(vk_text)
    assert (vk.degree(), vk.blinding_factors()) == (NL_DEGREE, NL_BLINDING_FACTORS)
    return vk, D, fixed, sigma, advice, instance


def coset_compression_differs(h2, D):
    """An on_construct hook for create_proof_package that records, per proof and lookup, whether the input and table
    compressed on the coset differ from the compressed Lagrange columns extended (the route for linear lookups only)."""
    from halo2_b200.arguments import _compress
    seen = []

    def hook(ev_e, permuted, lookup_exprs, theta):
        for per, exprs in zip(permuted, lookup_exprs):
            for lk, (inp, tab) in zip(per, exprs):
                for lag, ex in ((lk.compressed_input, inp), (lk.compressed_table, tab)):
                    co = D.lagrange_to_coeff_resident(lag, out=h2.ResidentPoly(D.field, D.n))
                    interpolated = D.coeff_to_extended_resident(co)
                    on_coset = ev_e.evaluate(_compress(ex, theta))
                    seen.append(not np.array_equal(interpolated.download(), on_coset.download()))
                    for p in (co, interpolated, on_coset):
                        p.close()
    return seen, hook


# ---- the ABI stand-in --------------------------------------------------------------------------------------------------
class ArgumentsFake(CC.ColumnsFake, VC.VanishingFake, PermutedFake):
    """The ABI stand-in with every entry point a package-composed proof reaches: the column-batched transforms and
    h2_poly_set_rows, the vanishing quotient, the lookup permutation, and the two product columns (the device bodies on the
    host emulation, emul_grandproduct.cpp)."""

    def h2_poly_permutation_product(self, z_out, proofs, columns, sigmas, cols, chunk_len, k, beta, gamma, omega, delta, blinding, bf, repr_):
        self._log("h2_poly_permutation_product")
        v = fake_engine._v
        proofs, cols, chunk_len, k, bf = v(proofs), v(cols), v(chunk_len), v(k), v(bf)
        n, sets = 1 << k, -(-cols // chunk_len)
        col = lambda h: self.polys[int(h)][1][:n]                  # noqa: E731
        f = self.polys[int(sigmas[0])][0]
        data = np.ascontiguousarray(np.concatenate([col(columns[i]) for i in range(proofs * cols)] + [col(sigmas[i]) for i in range(cols)]))
        out = np.zeros((proofs * sets * n, 32), dtype=np.uint8)
        rd = fake_engine._rd
        bl = rd(blinding, 32 * proofs * sets * bf) if bf else None
        self.emu.emu_permutation_product(cref.FIELD_ID[f], cref._p(data), proofs, cols, chunk_len, k, cref._p(rd(beta, 32)), cref._p(rd(gamma, 32)),
                                         cref._p(rd(omega, 32)), cref._p(rd(delta, 32)), cref._p(bl) if bf else None, bf, cref._p(out))
        for i in range(proofs * sets):
            self.polys[int(z_out[i])][1][:n] = out[i * n:(i + 1) * n]
        return 0

    def h2_poly_lookup_product(self, z_out, count, inputs, tables, permuted_inputs, permuted_tables, k, beta, gamma, blinding, bf, repr_):
        self._log("h2_poly_lookup_product")
        v = fake_engine._v
        count, k, bf = v(count), v(k), v(bf)
        if count == 0:
            return 0
        n = 1 << k
        col = lambda h: self.polys[int(h)][1][:n]                  # noqa: E731
        f = self.polys[int(inputs[0])][0]
        data = np.ascontiguousarray(np.concatenate([col(arr[b]) for b in range(count) for arr in (inputs, tables, permuted_inputs, permuted_tables)]))
        out = np.zeros((count * n, 32), dtype=np.uint8)
        rd = fake_engine._rd
        bl = rd(blinding, 32 * count * bf) if bf else None
        self.emu.emu_lookup_product(cref.FIELD_ID[f], cref._p(data), count, k, cref._p(rd(beta, 32)), cref._p(rd(gamma, 32)),
                                    cref._p(bl) if bf else None, bf, cref._p(out))
        for b in range(count):
            self.polys[int(z_out[b])][1][:n] = out[b * n:(b + 1) * n]
        return 0


@contextlib.contextmanager
def installed():
    """halo2_b200.lib bound to an ArgumentsFake for the duration of the block (and back to whatever it was afterwards)."""
    from halo2_b200 import lib as L
    saved = (L._lib, L._inited_device)
    fake = ArgumentsFake()
    L._lib, L._inited_device = fake, 0
    try:
        yield fake
    finally:
        L._lib, L._inited_device = saved


def params_for(h2, k: int, seed: int = 99):
    """Params over seeded generators, and a commit_lagrange(values) -> (x, y) with Blind::default() through the oracle."""
    n = 1 << k
    pts = cref.gen_points("vesta", seed, n + 2)
    A = cref.bytes_to_affine
    P = pasta.Params.from_generators(pasta.VESTA, k, [A(x) for x in pts[:n]], A(pts[n]), A(pts[n + 1]))
    gl = cref.affines_to_bytes(P.g_lagrange)
    prm = h2.Params("vesta", k, pts[:n], gl, pts[n:n + 1], u=pts[n + 1:n + 2])
    c = pasta.VESTA
    commit = lambda vals: pasta.to_affine(c, pasta.best_multiexp(c, [v % pasta.P_MOD for v in vals] + [1], P.g_lagrange + [P.w]))  # noqa: E731
    return prm, commit, (pts[:n], gl, pts[n:n + 1], pts[n + 1:n + 2])
