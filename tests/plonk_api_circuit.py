"""The fixed columns and the permutation polynomials of the reference's `plonk_api` test circuit
(/root/reference/halo2_proofs/tests/plonk_api.rs:21-420), rebuilt from its source so that the golden
commitments it pins (:958-982) can be recomputed: every one of them is
`params.commit_lagrange(column, Blind::default())` with `params = Params::<EqAffine>::new(5)`
(plonk/keygen.rs:233-236, plonk/permutation/keygen.rs:135-150) -- i.e. hash_to_curve -> EC-iFFT -> MSM.

Test infrastructure only.  The columns are pure integer bookkeeping (the caller supplies omega / delta / zeta); below them
are the circuit's golden case (key, Fp::ZETA, F::DELTA), its witness and copy constraints, and the provers the tests run on it.

Layout (SimpleFloorPlanner, circuit/floor_planner/single_pass.rs: a region starts at the first row free in all of
its columns): row 0 = public_input (sp = 1); then ten times a raw_multiply row (sa = sb = 0, sc = sm = 1) followed by
a raw_add row (sa = sb = sc = 1, sm = 0): rows 1..20.  Fixed columns in creation order (plonk_api.rs:293-307):
sf, sm, sa, sb, sc, sp, sl.  The table column sl holds [instance, a, a, 0] and is then filled with its row-0 value
up to the last usable row (circuit/table_layouter.rs:96, plonk/keygen.rs:152-173), usable rows = n - (blinding_factors
+ 1) with blinding_factors = max(3, 1) + 2 = 5 (plonk/circuit.rs:1435-1460).
Equality columns in enable_equality order (plonk_api.rs:299-301, :348-356): a, b, c, sf, e, d, p, sm, sa, sb, sc, sp;
per iteration copy(a0, a1) and copy(b1, c0) (plonk_api.rs:399-400), merged as plonk/permutation/keygen.rs:44-100.
"""
from oracle import pasta
from tests import multiopen_cases as MC
from tests import plonk_prover as PP
from tests import plonk_verifier as PV
from tests import prover_replay as R

K = 5
N = 1 << K
BLINDING_FACTORS = 5
USABLE_ROWS = N - (BLINDING_FACTORS + 1)
A_SMALL = 2834758237  # plonk_api.rs:421: a = Fp::from(2834758237) * Fp::ZETA


def fixed_columns(modulus: int, zeta: int):
    instance = 2
    a = A_SMALL * zeta % modulus
    mul_rows = [1 + 2 * i for i in range(10)]
    add_rows = [2 + 2 * i for i in range(10)]
    col = lambda rows: [1 if r in rows else 0 for r in range(N)]
    sf = [0] * N
    sm = col(mul_rows)
    sa = col(add_rows)
    sb = col(add_rows)
    sc = col(mul_rows + add_rows)
    sp = col([0])
    table = [instance, a, a, 0]
    sl = [0] * N
    for r in range(USABLE_ROWS):
        sl[r] = table[r] if r < len(table) else table[0]
    return [sf, sm, sa, sb, sc, sp, sl]


def permutation_columns(modulus: int, omega: int, delta: int):
    ncols = 12
    COL_A, COL_B, COL_C = 0, 1, 2
    mapping = [[(i, j) for j in range(N)] for i in range(ncols)]
    aux = [[(i, j) for j in range(N)] for i in range(ncols)]
    sizes = [[1] * N for _ in range(ncols)]

    def copy(lc, lr, rc, rr):
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

    for it in range(10):
        rm, ra = 1 + 2 * it, 2 + 2 * it
        for _ in range(2):                      # StandardCs::copy constrains twice (plonk_api.rs:216-217)
            copy(COL_A, rm, COL_A, ra)          # copy(a0, a1)
        for _ in range(2):
            copy(COL_B, ra, COL_C, rm)          # copy(b1, c0)

    omega_powers = [pow(omega, j, modulus) for j in range(N)]
    deltas = [pow(delta, i, modulus) for i in range(ncols)]
    return [[deltas[mapping[i][j][0]] * omega_powers[mapping[i][j][1]] % modulus for j in range(N)]
            for i in range(ncols)]


# ---- the golden case -----------------------------------------------------------------------------------------------------
FP_ZETA_INDEX = 1          # which primitive cube root pasta calls Fp::ZETA -- pinned by fixed_commitments[6]
CASE = PV.load_golden_proofs()[0]
M = pasta.P_MOD
DELTA = PV.scalar_delta(M)
ZETA = pasta.zeta_candidates("fp")[FP_ZETA_INDEX]                  # Fp::ZETA (pinned by the golden key's table-column commitment)


def golden_columns(goldens):
    """The fixed and permutation columns, and the 19 commitments the golden key pins for them (:958-982)."""
    vk = goldens["vk_plonk_api_k5"]
    cols = fixed_columns(M, ZETA) + permutation_columns(M, int(vk["omega"], 16), DELTA)
    want = [(int(x, 16), int(y, 16)) for x, y in vk["fixed_commitments"] + vk["permutation_commitments"]]
    assert len(cols) == len(want) == 19
    return cols, want


def plonk_api_copies():
    """The copy constraints in the order synthesis makes them (tests/plonk_api.rs:399-400, each twice by StandardCs::copy,
    :216-217): columns a = 0, b = 1, c = 2 of the permutation."""
    for it in range(10):
        rm, ra = 1 + 2 * it, 2 + 2 * it
        yield from [(0, rm, 0, ra)] * 2
        yield from [(1, ra, 2, rm)] * 2


def witness(break_row=None):
    """MyCircuit::synthesize (tests/plonk_api.rs:371-395) with a = 2834758237 * ZETA: row 0 the public input, then ten times a
    raw_multiply row (a, a, a^2; d = a^4, e = a^4) and a raw_add row (a, a^2, a^2 + a; d = a^4, e = a^8).  Advice columns in
    creation order: e, a, b, c, d (the permutation argument's column list, :880-930 of the pinned key)."""
    a = A_SMALL * ZETA % M
    a2 = a * a % M
    col = {name: [0] * N for name in "abcde"}
    col["a"][0] = 2
    for it in range(10):
        rm, ra = 1 + 2 * it, 2 + 2 * it
        col["a"][rm], col["b"][rm], col["c"][rm], col["d"][rm], col["e"][rm] = a, a, a2, pow(a, 4, M), pow(a, 4, M)
        col["a"][ra], col["b"][ra], col["c"][ra], col["d"][ra], col["e"][ra] = a, a2, (a2 + a) % M, pow(a, 4, M), pow(a2, 4, M)
    if break_row is not None:
        col["c"][break_row] = (col["c"][break_row] + 1) % M
    return [col["e"], col["a"], col["b"], col["c"], col["d"]]


def prove(setup, advice, instances, seed):
    """The oracle's prover; setup = (curve, Params, vk, fixed, sigma, generator bytes)."""
    c, P, vk, fixed, sigma, _ = setup
    W = R._WriteT(M)
    PP.create_proof(c, P.g, P.g_lagrange, P.w, P.u, vk, fixed, sigma, advice, instances, MC.SeededRng("fp", seed, False), W, ZETA, DELTA)
    return bytes(W.T.proof)


def plonk_api_key():
    return PV.PinnedKey(CASE["key_text"])


def plonk_api_proof(h2, prm):
    """create_proof_engine on the plonk_api circuit (k = 5, two proofs, seed 777) through `h2`, recording what the permuted
    and product commitments need.  Returns (proof bytes, record): record["theta"], the Lagrange columns registered by then
    ("cols"), the rng's draws ("draws", "draws_at_theta") and, per point written, the number of draws made before it."""
    vk = plonk_api_key()
    seen = {"point_draws": [], "challenges": []}
    rng = MC.RecordingRng(MC.SeededRng("fp", 777, True))

    class Eng:                                                     # the package, keeping the Lagrange-basis evaluator
        def __getattr__(self, name):
            return getattr(h2, name)

        def Evaluator(self, D, basis="extended"):
            ev = h2.Evaluator(D, basis)
            seen.setdefault(basis, ev)
            return ev

    class T(R.Blake2bTranscript):
        def squeeze_challenge(self):
            c = super().squeeze_challenge()
            seen["challenges"].append(c)
            if "theta" not in seen:
                seen.update(theta=c, draws_at_theta=len(rng.draws), points_at_theta=len(self.proof) // 32,
                            cols=[p.download() for p in seen["lagrange"].polys])
            return c

        def write_point(self, xy):
            seen["point_draws"].append(len(rng.draws))
            super().write_point(xy)

    tr = T(M)
    PP.create_proof_engine(Eng(), prm, vk, fixed_columns(M, ZETA), permutation_columns(M, vk.omega, DELTA),
                           [witness(), witness()], [[[2]], [[2]]], rng, tr, ZETA, DELTA)
    seen["draws"] = rng.draws
    return bytes(tr.proof), seen


def plonk_api_lookups(h2, seen):
    """The recorded Lagrange columns registered again in the prover's order (fixed, sigma, advice per proof, instance per
    proof) on a new evaluator, and the key's lookup expressions over it: (domain, evaluator, lookups[proof])."""
    vk = plonk_api_key()
    D = h2.EvaluationDomain("fp", vk.degree(), vk.k, ZETA)
    ev = h2.Evaluator(D, "lagrange")
    leaves = [ev.register_poly(h2.ResidentPoly("fp", D.n, c)) for c in seen["cols"]]
    nf, ns, na = len(fixed_columns(M, ZETA)), len(vk.permutation_columns), 5
    FL, AL = leaves[:nf], [leaves[nf + ns + p * na:nf + ns + (p + 1) * na] for p in range(2)]
    IL = [leaves[nf + ns + 2 * na + p:nf + ns + 2 * na + p + 1] for p in range(2)]
    ast = lambda e, p: PP._to_ast(h2, e, FL, AL[p], IL[p])
    return D, ev, [[([ast(e, p) for e in inp], [ast(e, p) for e in tab]) for inp, tab in vk.lookups] for p in range(2)]
