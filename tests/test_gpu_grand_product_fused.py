"""GPU tests of the product columns in one call per argument (h2_poly_permutation_product, h2_poly_lookup_product;
halo2_b200.permutation_commit / lookup_commit_product):

- the products equal the reference's loops restated with big integers (tests/grand_product_cases.py) element for
  element, both fields, k = 1, 4, 8, 11, several proofs, sets and lookups per call;
- at k = 14, 16, 18 and 20 the z columns and their commitments are byte-identical to a composition of finer calls (Ast
  programs, batch_invert, running_product, the host's last_z);
- a real proof of the benchmark circuit at k = 14 (tests/plonk_prover.create_proof_engine): permutation_commit, fed the
  challenges and draws the proof made, gives the permutation product commitments at their position in the proof bytes;
- sigma from a shared keygen_pk key on a lane, the z handles unknown elsewhere;
- every validation error, on the primary context and on a lane, fails with a message and leaves z_out untouched."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests import bench_circuit as BC  # noqa: E402
from tests import plonk_api_circuit as circ  # noqa: E402
from tests.abi_cases import _err, _run_parallel  # noqa: E402
from tests.bench_circuit import _bench_params, bench_copies  # noqa: E402
from tests.grand_product_cases import (_close, composition_lookup, composition_permutation, oracle_lookup_product,  # noqa: E402
                                       oracle_permutation_product)
from tests.plonk_api_circuit import ZETA  # noqa: E402
from tests.plonk_verifier import scalar_delta  # noqa: E402

SEED = 0x46555345


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


# ---- 1. against the restatement ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("k", [1, 4, 8, 11])
def test_permutation_product_against_the_restatement(eng, field, k):
    m, n = pasta.FIELDS[field], 1 << k
    D = eng.EvaluationDomain(field, 3, k, pasta.zeta_candidates(field)[0])
    for proofs, cols, chunk_len, bf in ((3, 7, 2, 0 if k == 1 else min(5, n - 2)), (2, 4, 1, n - 2), (1, 3, 3, 0)):
        seed = SEED + 100 * k + 10 * cols
        beta, gamma = pasta.gen_scalars(field, seed, 2)
        sig = [pasta.gen_scalars(field, seed + 1 + c, n) for c in range(cols)]
        val = [[pasta.gen_scalars(field, seed + 50 + 13 * p + c, n) for c in range(cols)] for p in range(proofs)]
        if n > 2:
            val[-1][0][n // 2] = (-(beta * sig[0][n // 2] + gamma)) % m          # a zero denominator
        sets = -(-cols // chunk_len)
        blinding = pasta.gen_scalars(field, seed + 9, proofs * sets * bf) if bf else []
        want = oracle_permutation_product(val, sig, beta, gamma, D.omega, scalar_delta(m), chunk_len, bf, blinding, m)
        S = [eng.ResidentPoly(field, n, cref.ints_to_bytes(s)) for s in sig]
        C = [[eng.ResidentPoly(field, n, cref.ints_to_bytes(v)) for v in per] for per in val]
        z = eng.permutation_product_resident(D, C, S, beta, gamma, scalar_delta(m), chunk_len, bf, blinding)
        got = [[cref.bytes_to_ints(q.download()) for q in per] for per in z]
        _close(S, *C, *z)
        assert got == want, (proofs, cols, chunk_len, bf)


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("k", [1, 4, 8, 11])
def test_lookup_product_against_the_restatement(eng, field, k):
    m, n = pasta.FIELDS[field], 1 << k
    D = eng.EvaluationDomain(field, 3, k, pasta.zeta_candidates(field)[0])
    bf = 0 if k == 1 else min(5, n - 2)
    seed = SEED + 7000 + k
    beta, gamma = pasta.gen_scalars(field, seed, 2)
    per_proof = (2, 3)
    vals = [[[pasta.gen_scalars(field, seed + 40 * p + 4 * b + j, n) for j in range(4)] for b in range(cnt)] for p, cnt in enumerate(per_proof)]
    if n > 2:
        vals[1][2][2][n // 2] = (-beta) % m                                      # a' = -beta: a zero denominator
    flat = [lk for per in vals for lk in per]
    blinding = pasta.gen_scalars(field, seed + 999, len(flat) * bf) if bf else []
    want = [oracle_lookup_product(*lk, beta, gamma, bf, blinding[b * bf:(b + 1) * bf], m) for b, lk in enumerate(flat)]
    R = [[tuple(eng.ResidentPoly(field, n, cref.ints_to_bytes(c)) for c in lk) for lk in per] for per in vals]
    z = eng.lookup_product_resident(D, R, beta, gamma, bf, blinding)
    assert [len(per) for per in z] == list(per_proof)
    got = [cref.bytes_to_ints(q.download()) for per in z for q in per]
    _close([p for per in R for lk in per for p in lk], *z)
    assert got == want


# ---- 2. byte-identical to the composition at prover sizes --------------------------------------------------------------
SHAPES = {"benchmark": (3, 3), "wide": (16, 3)}                             # (columns, chunk_len): 1 set; 6 sets, the last partial


@pytest.mark.parametrize("k", [14, 16, 18, 20])
def test_same_bytes_as_the_composition(eng, k):
    field, m, n, bf = "fp", pasta.P_MOD, 1 << k, BC.BLINDING_FACTORS
    D = eng.EvaluationDomain(field, BC.DEGREE, k, ZETA)
    prm = _bench_params(eng, k)
    delta = scalar_delta(m)
    beta, gamma = pasta.gen_scalars(field, SEED + k, 2)
    try:
        for name, (cols, chunk_len) in SHAPES.items():
            proofs = 2 if name == "benchmark" else 1
            sets = -(-cols // chunk_len)
            S = [eng.ResidentPoly(field, n, cref.gen_scalars(field, SEED + 10 * k + c, n)) for c in range(cols)]
            C = [[eng.ResidentPoly(field, n, cref.gen_scalars(field, SEED + 1000 * k + 40 * p + c, n)) for c in range(cols)] for p in range(proofs)]
            blinding = pasta.gen_scalars(field, SEED + 3 * k, proofs * sets * bf)
            blinds = pasta.gen_scalars(field, SEED + 5 * k, proofs * sets)
            want = [q for per in composition_permutation(eng, D, C, S, beta, gamma, delta, chunk_len, bf, blinding) for q in per]
            got = [q for per in eng.permutation_product_resident(D, C, S, beta, gamma, delta, chunk_len, bf, blinding) for q in per]
            assert len(got) == proofs * sets
            for a, b in zip(got, want):
                assert (a.download() == b.download()).all(), name
            cw = prm.commit_resident_affine(want, [eng.Blind(b) for b in blinds], lagrange=True)
            cg = prm.commit_resident_affine(got, [eng.Blind(b) for b in blinds], lagrange=True)
            assert (cw == cg).all()
            _close(S, *C, want, got)
        # 4 lookups
        L4 = [tuple(eng.ResidentPoly(field, n, cref.gen_scalars(field, SEED + 77 * k + 4 * b + j, n)) for j in range(4)) for b in range(4)]
        blinding = pasta.gen_scalars(field, SEED + 7 * k, 4 * bf)
        want = composition_lookup(eng, D, L4, beta, gamma, bf, blinding)
        got = eng.lookup_product_resident(D, [L4], beta, gamma, bf, blinding)[0]
        for a, b in zip(got, want):
            assert (a.download() == b.download()).all()
        assert (prm.commit_resident_affine(want, [eng.Blind(3)] * 4, lagrange=True) == prm.commit_resident_affine(got, [eng.Blind(3)] * 4, lagrange=True)).all()
        _close([p for lk in L4 for p in lk], want, got)
    finally:
        prm.close()


# ---- 3. real proofs -----------------------------------------------------------------------------------------------------
class RecordingTranscript:
    """Passes every call through; records the challenges."""
    def __init__(self, inner):
        self.inner, self.challenges = inner, []

    def squeeze_challenge(self):
        c = self.inner.squeeze_challenge()
        self.challenges.append(c)
        return c

    def __getattr__(self, name):
        return getattr(self.inner, name)


def test_benchmark_proof_k14_contains_the_permutation_commitments(eng):
    from tests import multiopen_cases as MC
    from tests import plonk_prover as PP
    from tests import plonk_verifier as PV
    from tests import prover_replay as R
    k, m = 14, pasta.P_MOD
    n, delta = 1 << k, scalar_delta(m)
    prm = _bench_params(eng, k)
    pk = None
    try:
        D = eng.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
        fixed, _, adv = BC.columns(k, m, D.omega, delta, circ.A_SMALL * ZETA % m)
        cc = eng.CopyConstraints(n, 3)
        cc.extend(np.array(list(bench_copies(k)), dtype=np.uint32))
        fc, pc = eng.keygen_vk(prm, D, fixed, cc, delta)
        A = cref.bytes_to_affine
        vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, pasta.Q_MOD, m, D.omega, [A(x) for x in fc], [A(x) for x in pc]))
        pk = eng.keygen_pk(prm, D, fixed, cc, delta, BC.BLINDING_FACTORS)
        rng = MC.RecordingRng(MC.SeededRng("fp", 11, True))
        T = RecordingTranscript(R.Blake2bTranscript(m))
        ab = [cref.ints_to_bytes(c) for c in adv]
        PP.create_proof_engine(eng, prm, vk, None, None, [ab], [[]], rng, T, ZETA, delta, pk=pk)
        proof = bytes(T.proof)
        assert not vk.lookups
        bf, usable, nadv = vk.blinding_factors(), n - (vk.blinding_factors() + 1), len(adv)
        # the advice columns as the prover committed them: its values, then the blinding rows it drew (prover.rs:276-282)
        adv_l = [eng.ResidentPoly("fp", n, cref.ints_to_bytes(list(c[:usable]) + rng.draws[j * (n - usable):(j + 1) * (n - usable)]))
                 for j, c in enumerate(adv)]
        cols = [{"Advice": adv_l, "Fixed": pk.fixed_values}[t][i] for t, i in vk.permutation_columns]
        beta, gamma = T.challenges[1], T.challenges[2]                          # theta, beta, gamma
        chunk_len = vk.degree() - 2
        sets, cm = eng.permutation_commit(prm, D, pk, [cols], beta, gamma, delta, chunk_len, bf, MC.ReplayRng(rng.draws[nadv * (n - usable) + nadv:]))
        at = 32 * nadv                                                          # the advice commitments come first
        assert proof[at:at + 32 * len(cm)] == R._encode(cm, m)
        assert len(sets) == 1 and len(sets[0]) == len(cm) == -(-len(vk.permutation_columns) // chunk_len)
        _close(adv_l, [q for s in sets[0] for q in s[:2]])
    finally:
        if pk is not None:
            pk.close()
        prm.close()


# ---- 4. a shared key's sigma on a lane ---------------------------------------------------------------------------------
def test_shared_key_sigma_on_a_lane(eng):
    from halo2_b200 import lib as L
    k, m = 10, pasta.P_MOD
    n, delta = 1 << k, scalar_delta(m)
    prm = _bench_params(eng, k)
    D = eng.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
    cc = eng.CopyConstraints(n, 3)
    cc.extend(np.array(list(bench_copies(k)), dtype=np.uint32))
    pk = eng.keygen_pk(prm, D, BC.columns(k, m, D.omega, delta, 7)[0], cc, delta, BC.BLINDING_FACTORS).share()
    sig = [cref.bytes_to_ints(p.download()) for p in pk.permutation.permutations]
    beta, gamma = pasta.gen_scalars("fp", SEED + 5, 2)
    bf = BC.BLINDING_FACTORS
    vals = [[pasta.gen_scalars("fp", SEED + 60 + 3 * p + c, n) for c in range(3)] for p in range(2)]
    blinding = pasta.gen_scalars("fp", SEED + 61, 2 * bf)
    want = oracle_permutation_product(vals, sig, beta, gamma, D.omega, delta, 3, bf, blinding, m)

    def go():
        with eng.Lane():
            C = [[eng.ResidentPoly("fp", n, cref.ints_to_bytes(v)) for v in per] for per in vals]
            z = eng.permutation_product_resident(D, C, pk.permutation.permutations, beta, gamma, delta, 3, bf, blinding)
            got = [[cref.bytes_to_ints(q.download()) for q in per] for per in z]
            handles = [q._h.value for per in z for q in per]
            _close(*C, *z)
            return got, handles
    try:
        got, handles = _run_parallel([go])[0]
        assert got == want
        for h in handles:                                       # the lane is gone, and its z handles are unknown here
            assert L.load().h2_poly_download(ctypes.c_uint64(h), None, ctypes.c_size_t(0), 0) != 0 and "unknown" in _err()
    finally:
        pk.close()
        prm.close()


# ---- 5. validation -----------------------------------------------------------------------------------------------------
def _error_cases(eng):
    from halo2_b200 import lib as L
    lib = L.load()
    k, n, field = 4, 16, "fp"
    D = eng.EvaluationDomain(field, 3, k, pasta.zeta_candidates(field)[0])
    mk = lambda seed, ln=n, f=field: eng.ResidentPoly(f, ln, cref.gen_scalars(f, SEED + seed, ln))
    cols = [mk(1), mk(2), mk(3)]
    sig = [mk(4), mk(5), mk(6)]
    z = [mk(7), mk(8)]
    fq, short, sh = mk(9, f="fq"), mk(10, n - 1), mk(11).share()
    gone = mk(12)
    gone_h = gone._h.value
    gone.close()
    fe = lambda x: L.ptr(L.fe_bytes(x))
    H = lambda ps: (ctypes.c_uint64 * len(ps))(*[p if isinstance(p, int) else p._h.value for p in ps])
    blind = cref.gen_scalars(field, SEED + 13, 4)
    before = [q.download() for q in z]

    def perm(zs=None, cs=None, ss=None, chunk=2, kk=k, bf=2, proofs=1, ncols=3):
        zs, cs, ss = zs or z, cs or cols, ss or sig
        return lib.h2_poly_permutation_product(H(zs), ctypes.c_size_t(proofs), H(cs), H(ss), ctypes.c_size_t(ncols), ctypes.c_uint32(chunk),
                                               ctypes.c_uint32(kk), fe(3), fe(5), fe(D.omega), fe(7), L.ptr(blind), ctypes.c_uint32(bf), 0)

    def look(zs=None, ins=None, kk=k, bf=2, count=2):
        zs, ins = zs or z, ins or [cols[0], cols[1], cols[2], sig[0], sig[1], sig[2], sh, cols[0]]
        return lib.h2_poly_lookup_product(H(zs), ctypes.c_size_t(count), H(ins[0::4]), H(ins[1::4]), H(ins[2::4]), H(ins[3::4]), ctypes.c_uint32(kk),
                                          fe(3), fe(5), L.ptr(blind), ctypes.c_uint32(bf), 0)

    def untouched():
        assert all((q.download() == b).all() for q, b in zip(z, before))

    try:
        cases = [
            (lambda: perm(zs=[z[0], 0xDEADBEEF]), "z_out[1]: unknown polynomial handle"), (lambda: perm(zs=[z[0], gone_h]), "z_out[1]: unknown polynomial handle"),
            (lambda: perm(cs=[cols[0], cols[1], 0xDEADBEEF]), "columns[2]: unknown polynomial handle"),
            (lambda: perm(ss=[sig[0], sig[1], fq]), "sigmas[2]: the polynomials live in different fields"),
            (lambda: perm(zs=[z[0], fq]), "z_out[1]: the polynomials live in different fields"),
            (lambda: perm(cs=[cols[0], short, cols[2]]), "columns[1]: a polynomial holds fewer than 2^k elements"),
            (lambda: perm(zs=[z[0], short]), "z_out[1]: a polynomial holds fewer than 2^k elements"),
            (lambda: perm(zs=[z[0], sh]), "z_out[1]: the polynomial is shared (read-only)"),
            (lambda: perm(zs=[z[0], z[0]]), "z_out[1] is also z_out[0]"), (lambda: perm(zs=[z[0], cols[1]]), "z_out[1] is also columns[1]"),
            (lambda: perm(zs=[sig[2], z[1]]), "z_out[0] is also sigmas[2]"), (lambda: perm(chunk=0), "chunk_len == 0"),
            (lambda: perm(bf=n - 1), "blinding_factors + 1 >= n"), (lambda: perm(kk=31), "k > 30"),
            (lambda: look(zs=[z[0], 0xDEADBEEF]), "z_out[1]: unknown polynomial handle"),
            (lambda: look(zs=[z[0], sh]), "z_out[1]: the polynomial is shared (read-only)"),
            (lambda: look(zs=[z[0], z[0]]), "z_out[1] is also z_out[0]"), (lambda: look(zs=[z[0], cols[2]]), "z_out[1] is also permuted_inputs[0]"),
            (lambda: look(ins=[cols[0], cols[1], fq, sig[0], sig[1], sig[2], sh, cols[0]]), "permuted_inputs[0]: the polynomials live in different fields"),
            (lambda: look(ins=[cols[0], cols[1], cols[2], short, sig[1], sig[2], sh, cols[0]]), "permuted_tables[0]: a polynomial holds fewer than 2^k elements"),
            (lambda: look(bf=n - 1), "blinding_factors + 1 >= n"), (lambda: look(kk=31), "k > 30"),
        ]
        for i, (call, msg) in enumerate(cases):
            assert call() != 0 and msg in _err(), (i, _err())
            untouched()
        assert perm(proofs=0) == 0 and perm(ncols=0) == 0 and look(count=0) == 0
        untouched()
        assert perm() == 0 and look() == 0                  # the same arguments, well formed, do run
        assert not all((q.download() == b).all() for q, b in zip(z, before))
    finally:
        _close(cols, sig, z, [fq, short, sh])


def test_errors_name_the_argument_on_the_primary_context(eng):
    _error_cases(eng)


def test_errors_name_the_argument_on_a_lane(eng):
    def go():
        with eng.Lane():
            _error_cases(eng)
    _run_parallel([go])
