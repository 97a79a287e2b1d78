"""GPU tests of the permutation argument from the list of copy constraints: h2_poly_permutation_sigma_copies
(csrc/assembly.cuh, then keygen.cuh's sigma kernels) and halo2_b200.CopyConstraints through keygen_vk / keygen_pk:

- keygen_vk of the plonk_api circuit's copies gives the 19 commitments the reference pins (tests/plonk_api.rs:958-982);
- sigma from copies is byte-identical to sigma from the reference's mapping through h2_poly_permutation_sigma, the mapping
  from the Python Assembly up to k = 16 and from orc_assembly at k = 18 and 20, in both fields with omega / delta in both
  representations: the benchmark circuit, random lists with large components, one cycle through every cell in increasing,
  decreasing and random copy order, and a star of degree 2^16;
- at k = 14 a proof made with the key from copies is the proof made with the Assembly's key, verifies, and is rejected
  after a flipped bit;
- every argument error, on the primary context and on a lane; a bad copy leaves dst unchanged;
- keys from copies on two lanes at once, with lane-local handles."""
import ctypes
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import assembly as orc  # noqa: E402
from oracle import cref, pasta  # noqa: E402
from tests import bench_circuit as BC  # noqa: E402
from tests import plonk_api_circuit as circ  # noqa: E402
from tests.abi_cases import _err, _lib, _run_parallel, _sigma_call  # noqa: E402
from tests.bench_circuit import _bench_assembly, _bench_params, bench_copies  # noqa: E402
from tests.keygen_cases import oracle_sigma  # noqa: E402
from tests.plonk_api_circuit import ZETA, golden_columns, plonk_api_copies  # noqa: E402
from tests.plonk_prover import prover_pk_bytes  # noqa: E402
from tests.plonk_verifier import scalar_delta  # noqa: E402

SEED = 0x41534D42


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


def _copies_call(polys, k: int, copies, omega: int, delta: int, repr_: int = 0, cols=None, m=None) -> int:
    """h2_poly_permutation_sigma_copies on raw handles / copies; omega and delta as given (already in `repr_`)."""
    from halo2_b200 import lib as L
    hs = [p if isinstance(p, int) else p._h.value for p in polys]
    arr = (ctypes.c_uint64 * max(len(hs), 1))(*hs)
    cp = None if copies is None else np.ascontiguousarray(np.asarray(copies, dtype=np.uint32).reshape(-1, 4))
    return _lib().h2_poly_permutation_sigma_copies(arr if hs else None, ctypes.c_size_t(len(hs) if cols is None else cols), ctypes.c_uint32(k),
                                                   None if cp is None else cp.ctypes.data_as(ctypes.c_void_p),
                                                   ctypes.c_size_t(cp.shape[0] if m is None else m), L.ptr(L.fe_bytes(omega)), L.ptr(L.fe_bytes(delta)),
                                                   repr_)


def _sigma_pair(eng, field: str, cols: int, k: int, copies, mapping, mont: bool):
    """The sigma columns from the copies and from the mapping, downloaded."""
    m = pasta.FIELDS[field]
    conv = (lambda x: (x << 256) % m) if mont else (lambda x: x)
    w, d = conv(pasta.omega_for_k(field, k)), conv(scalar_delta(m))
    a = [eng.ResidentPoly(field, 1 << k) for _ in range(cols)]
    b = [eng.ResidentPoly(field, 1 << k) for _ in range(cols)]
    try:
        assert _copies_call(a, k, copies, w, d, 1 if mont else 0) == 0, _err()
        assert _sigma_call(b, k, mapping, w, d, 1 if mont else 0) == 0, _err()
        return [p.download() for p in a], [p.download() for p in b]
    finally:
        for p in a + b:
            p.close()


def _cycle(rng, cols: int, k: int, order: str) -> np.ndarray:
    """One cycle through every cell: a path through a random cell order, closed, in increasing / decreasing / random copy
    order, so the walks' successor chains run through all cols * 2^k cells."""
    n = 1 << k
    perm = rng.permutation(cols * n).astype(np.int64)
    a, b = perm, np.roll(perm, -1)
    cp = np.stack([a >> k, a & (n - 1), b >> k, b & (n - 1)], axis=1)
    if order == "dec":
        cp = cp[::-1]
    elif order == "random":
        cp = cp[rng.permutation(cp.shape[0])]
    return np.ascontiguousarray(cp, dtype=np.uint32)


def _lists(rng, cols: int, k: int):
    n = 1 << k
    N = cols * n
    out = [("bench", np.array(list(bench_copies(k)), dtype=np.uint32).reshape(-1, 4))] if cols == 3 and k >= 3 else []
    few = rng.choice(N, size=max(2, N // 64), replace=False)             # large components over a few cells, duplicates
    x, y = rng.choice(few, size=2 * few.size + 5), rng.choice(few, size=2 * few.size + 5)
    out.append(("dense", np.stack([x >> k, x & (n - 1), y >> k, y & (n - 1)], axis=1).astype(np.uint32)))
    x, y = rng.integers(0, N, N), rng.integers(0, N, N)
    out.append(("random", np.stack([x >> k, x & (n - 1), y >> k, y & (n - 1)], axis=1).astype(np.uint32)))
    for order in ("inc", "dec", "random"):
        out.append((f"cycle-{order}", _cycle(rng, cols, k, order)))
    return out


def _python_mapping(eng, cols: int, k: int, copies) -> np.ndarray:
    asm = eng.Assembly(1 << k, cols)
    for c in copies.tolist():
        asm.copy(*c)
    return asm.mapping


# ---- the reference's golden verifying key -------------------------------------------------------------------------------
def test_keygen_vk_from_copies_reproduces_the_golden_commitments(eng, goldens):
    m = pasta.P_MOD
    _, want = golden_columns(goldens)
    prm = eng.Params.new("vesta", circ.K)
    try:
        D = eng.EvaluationDomain("fp", 4, circ.K, ZETA)
        cc = eng.CopyConstraints(circ.N, 12)
        for cp in plonk_api_copies():
            cc.copy(*cp)
        fc, pc = eng.keygen_vk(prm, D, circ.fixed_columns(m, ZETA), cc, scalar_delta(m))
        assert [cref.bytes_to_affine(x) for x in np.concatenate([fc, pc])] == want
    finally:
        prm.close()


# ---- sigma from copies against sigma from the mapping ------------------------------------------------------------------
@pytest.mark.parametrize("field", ["fp", "fq"])
def test_sigma_from_copies_python_assembly(eng, field):
    rng = np.random.default_rng(SEED)
    for k, cols in ((1, 1), (2, 3), (5, 8), (8, 3), (10, 2), (12, 3)):
        for name, cps in _lists(rng, cols, k):
            mp = _python_mapping(eng, cols, k, cps)
            for mont in (False, True):
                got, want = _sigma_pair(eng, field, cols, k, cps, mp, mont)
                assert all((g == w).all() for g, w in zip(got, want)), (k, cols, name, mont)
    k, cols = 16, 3
    for name, cps in _lists(rng, cols, k)[:3]:                           # bench, dense, random
        mp = _python_mapping(eng, cols, k, cps)
        assert (mp == orc.assembly(cps, cols, k)[0]).all()
        got, want = _sigma_pair(eng, field, cols, k, cps, mp, field == "fq")
        assert all((g == w).all() for g, w in zip(got, want)), (k, name)


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_sigma_from_copies_large(eng, field):
    rng = np.random.default_rng(SEED + 1)
    for k in (18, 20):
        for name, cps in _lists(rng, 3, k):
            mp, err = orc.assembly(cps, 3, k)
            assert err is None
            got, want = _sigma_pair(eng, field, 3, k, cps, mp, (k == 20) == (field == "fp"))
            assert all((g == w).all() for g, w in zip(got, want)), (k, name)
    k, cols = 18, 1                                                      # a star of degree 2^16 around one cell, random order
    leaves = rng.choice(np.arange(1, 1 << k), size=1 << 16, replace=False)
    centre = np.zeros_like(leaves)
    cps = np.stack([centre, centre + 77, centre, leaves], axis=1).astype(np.uint32)
    cps = cps[rng.permutation(cps.shape[0])]
    cps[::2] = cps[::2][:, [2, 3, 0, 1]]
    mp, err = orc.assembly(cps, cols, k)
    assert err is None
    got, want = _sigma_pair(eng, field, cols, k, cps, mp, field == "fq")
    assert (got[0] == want[0]).all()


# ---- errors ------------------------------------------------------------------------------------------------------------
def _error_cases(eng):
    field, k, n = "fp", 4, 16
    m = pasta.P_MOD
    omega, delta = pasta.omega_for_k(field, k), scalar_delta(m)
    ident = np.stack(np.meshgrid(np.arange(2), np.arange(n), indexing="ij"), axis=-1).astype(np.uint32)
    good = [(0, 1, 1, 2), (1, 2, 0, 5), (0, 5, 0, 5)]
    want = [cref.ints_to_bytes(col) for col in oracle_sigma(orc.assembly(good, 2, k)[0], n, omega, delta, m)]
    idw = [cref.ints_to_bytes(col) for col in oracle_sigma(ident, n, omega, delta, m)]
    a, b = eng.ResidentPoly(field, n), eng.ResidentPoly(field, n)
    fq, short = eng.ResidentPoly("fq", n), eng.ResidentPoly(field, n - 1)
    gone = eng.ResidentPoly(field, n)
    gone_h = gone._h.value
    gone.close()

    def works():
        a.upload(np.zeros((n, 32), dtype=np.uint8))
        assert _copies_call([a, b], k, good, omega, delta) == 0, _err()
        assert (a.download() == want[0]).all() and (b.download() == want[1]).all()

    try:
        works()
        for cps, msg in ((good + [(2, 0, 0, 0)] + good, "copy 3: a column"), (good + [(0, 0, 1, n)], "copy 3: a row"),
                         ([(0, n, 0, 0), (2, 0, 0, 0)], "copy 0: a row"), ([(0, 0, 0, 0), (0xFFFFFFFF, n, 0, 0)], "copy 1: a column")):
            sentinel = [np.full((n, 32), 7 + i, dtype=np.uint8) for i in range(2)]
            a.upload(sentinel[0])
            b.upload(sentinel[1])
            assert _copies_call([a, b], k, cps, omega, delta) != 0 and msg in _err(), _err()
            assert (a.download() == sentinel[0]).all() and (b.download() == sentinel[1]).all()     # dst unchanged
            works()
        cases = (([a, 0xDEADBEEF], "dst[1]: unknown polynomial handle"), ([a, gone_h], "dst[1]: unknown polynomial handle"),
                 ([a, fq], "dst[1]: the polynomials live in different fields"), ([short, a], "dst[0]: a polynomial holds fewer than 2^k elements"),
                 ([a, a], "dst[1] is also dst[0]"))
        for polys, msg in cases:
            assert _copies_call(polys, k, good, omega, delta) != 0 and msg in _err(), (polys, _err())
            works()
        assert _copies_call([a], 31, good, omega, delta) != 0 and "k > 30" in _err()
        assert _copies_call([a], k, good, omega, delta, cols=1 << 32) != 0 and "cols >= 2^32" in _err()
        assert _copies_call([a, b, fq, short], 30, good, omega, delta) != 0 and "cols * 2^k >= 2^32" in _err()
        assert _copies_call([a, b], k, good, omega, delta, m=1 << 32) != 0 and "m >= 2^32" in _err()
        assert _copies_call([a, b], k, None, omega, delta, m=3) != 0 and "null argument" in _err()
        works()
        assert _copies_call([a, b], k, None, omega, delta, m=0) == 0, _err()                # no copies: the identity
        assert (a.download() == idw[0]).all() and (b.download() == idw[1]).all()
        assert _copies_call([], k, None, omega, delta, cols=0, m=0) == 0, _err()
        works()
    finally:
        for p in (a, b, fq, short):
            p.close()


def test_errors_name_the_argument_on_the_primary_context(eng):
    _error_cases(eng)


def test_errors_name_the_argument_on_a_lane(eng):
    def go():
        with eng.Lane():
            _error_cases(eng)
    _run_parallel([go])


# ---- a real key at k = 14 ----------------------------------------------------------------------------------------------
def _bench_copy_constraints(eng, k: int):
    cc = eng.CopyConstraints(1 << k, 3)
    cc.extend(np.array(list(bench_copies(k)), dtype=np.uint32))
    return cc


def test_benchmark_circuit_proof_from_copies_k14(eng):
    from tests import multiopen_cases as MC
    from tests import plonk_prover as PP
    from tests import plonk_verifier as PV
    from tests import prover_replay as R
    k = 14
    m = pasta.P_MOD
    delta = scalar_delta(m)
    prm = _bench_params(eng, k)
    keys = []
    try:
        D = eng.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
        fixed, _, adv = BC.columns(k, m, D.omega, delta, circ.A_SMALL * ZETA % m)
        ab = [cref.ints_to_bytes(c_) for c_ in adv]
        cc, asm = _bench_copy_constraints(eng, k), _bench_assembly(eng, k)
        fc, pc = eng.keygen_vk(prm, D, fixed, cc, delta)
        fa, pa = eng.keygen_vk(prm, D, fixed, asm, delta)
        assert (fc == fa).all() and (pc == pa).all()
        A = cref.bytes_to_affine
        vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, pasta.Q_MOD, m, D.omega, [A(x) for x in fc], [A(x) for x in pc]))
        proofs = []
        for src in (cc, asm):
            keys.append(eng.keygen_pk(prm, D, fixed, src, delta, BC.BLINDING_FACTORS))
            T = R.Blake2bTranscript(m)
            PP.create_proof_engine(eng, prm, vk, None, None, [ab], [[]], MC.SeededRng("fp", 5, True), T, ZETA, delta, pk=keys[-1])
            proofs.append(bytes(T.proof))
        assert prover_pk_bytes(keys[0]) == prover_pk_bytes(keys[1])
        assert proofs[0] == proofs[1]
        arm = PV.EngineArm(eng, "vesta", k, params=prm)
        try:
            assert PV.verify_proof(arm, vk, proofs[0], [[]], delta)
            bad = bytearray(proofs[0])
            bad[len(bad) // 3] ^= 8
            assert not PV.verify_proof(arm, vk, bytes(bad), [[]], delta)
        finally:
            arm.close()
    finally:
        for pk in keys:
            pk.close()
        prm.close()


# ---- lanes -------------------------------------------------------------------------------------------------------------
def test_keygen_from_copies_on_two_lanes(eng):
    k = 12
    m = pasta.P_MOD
    delta = scalar_delta(m)
    prm = _bench_params(eng, k)
    D = eng.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
    fixed = BC.columns(k, m, D.omega, delta, 7)[0]
    cc = _bench_copy_constraints(eng, k)
    lib = _lib()
    pk0 = eng.keygen_pk(prm, D, fixed, _bench_assembly(eng, k), delta, BC.BLINDING_FACTORS)
    try:
        want = prover_pk_bytes(pk0)
        handles = {}
        meet = threading.Barrier(2, timeout=300)

        def on_lane(i):
            def go():
                with eng.Lane():
                    pk = eng.keygen_pk(prm, D, fixed, cc, delta, BC.BLINDING_FACTORS)
                    try:
                        got = prover_pk_bytes(pk)
                        handles[i] = pk.permutation.permutations[0]._h.value
                        meet.wait()
                        foreign = [lib.h2_poly_download(ctypes.c_uint64(h), None, ctypes.c_size_t(0), 0) != 0 and "unknown" in _err()
                                   for h in (handles[1 - i], pk0.l0._h.value)]
                        meet.wait()
                    finally:
                        pk.close()
                return got, foreign
            return go
        for got, foreign in _run_parallel([on_lane(0), on_lane(1)]):
            assert got == want
            assert foreign == [True, True]
    finally:
        pk0.close()
        prm.close()
