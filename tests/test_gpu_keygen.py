"""GPU tests of key generation: h2_poly_permutation_sigma (csrc/keygen.cuh) and halo2_b200.keygen (Assembly, keygen_vk,
keygen_pk) against the reference's own vectors and a restatement of permutation/keygen.rs:

- keygen_vk of the plonk_api circuit on Params::new(5) gives the 19 commitments the reference pins (tests/plonk_api.rs:958-982);
- the sigma polynomials equal the reference's serial omega-power loop and deltaomega gather, element for element up to
  k = 16 and on seeded samples at k = 18, 20 and 23 (two launches per column), in both fields, omega / delta given canonical
  or in Montgomery form;
- the benchmark circuit's key at k = 14 commits like the host path, proves byte for byte like the host-built sigma, and
  verifies;
- every argument error fails with a message and leaves the context usable;
- keygen_pk on two lanes at once gives the primary context's bytes, and a key's handles are unknown on other lanes."""
import ctypes
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests import bench_circuit as BC  # noqa: E402
from tests import plonk_api_circuit as circ  # noqa: E402
from tests.abi_cases import _err, _lib, _run_parallel, _sigma_call  # noqa: E402
from tests.bench_circuit import _bench_assembly, _bench_params  # noqa: E402
from tests.keygen_cases import oracle_sigma, random_mapping  # noqa: E402
from tests.plonk_api_circuit import ZETA, golden_columns, plonk_api_copies  # noqa: E402
from tests.plonk_prover import prover_pk_bytes, prover_pk_dict  # noqa: E402
from tests.plonk_verifier import scalar_delta  # noqa: E402

SEED = 0x4B455947


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


def _device_sigma(eng, field: str, mapping, k: int, omega: int, delta: int, mont: bool):
    m = pasta.FIELDS[field]
    conv = (lambda x: (x << 256) % m) if mont else (lambda x: x)
    polys = [eng.ResidentPoly(field, 1 << k) for _ in range(mapping.shape[0])]
    assert _sigma_call(polys, k, mapping, conv(omega), conv(delta), 1 if mont else 0) == 0, _err()
    return polys


# ---- the reference's golden verifying key -------------------------------------------------------------------------------
def test_keygen_vk_reproduces_the_golden_commitments(eng, goldens):
    m = pasta.P_MOD
    _, want = golden_columns(goldens)
    prm = eng.Params.new("vesta", circ.K)                                  # Params::<EqAffine>::new(5)
    try:
        D = eng.EvaluationDomain("fp", 4, circ.K, ZETA)
        assert D.omega == int(goldens["vk_plonk_api_k5"]["omega"], 16)
        asm = eng.Assembly(circ.N, 12)
        for cp in plonk_api_copies():
            asm.copy(*cp)
        fc, pc = eng.keygen_vk(prm, D, circ.fixed_columns(m, ZETA), asm, scalar_delta(m))
        assert fc.shape == (7, 64) and pc.shape == (12, 64)
        assert [cref.bytes_to_affine(x) for x in np.concatenate([fc, pc])] == want
    finally:
        prm.close()


# ---- sigma against the reference ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("field", ["fp", "fq"])
def test_sigma_every_element(eng, field):
    m = pasta.FIELDS[field]
    rng = np.random.default_rng(SEED)
    delta = scalar_delta(m)
    for k in range(1, 17):
        n = 1 << k
        omega = pasta.omega_for_k(field, k)
        cols = (1, 3, 12)[k % 3]
        mp = random_mapping(rng, cols, n)
        want = [cref.ints_to_bytes(col) for col in oracle_sigma(mp, n, omega, delta, m)]
        for mont in (False, True):
            polys = _device_sigma(eng, field, mp, k, omega, delta, mont)
            for i, p in enumerate(polys):
                assert (p.download() == want[i]).all(), (k, cols, mont, i)
                p.close()
    # the identity mapping: delta^i omega^j
    k, n = 16, 1 << 16
    omega = pasta.omega_for_k(field, k)
    ident = np.stack(np.meshgrid(np.arange(3), np.arange(n), indexing="ij"), axis=-1).astype(np.uint32)
    polys = _device_sigma(eng, field, ident, k, omega, delta, False)
    want = oracle_sigma(ident, n, omega, delta, m)
    for i, p in enumerate(polys):
        got = cref.bytes_to_ints(p.download())
        assert got[:3] == [pow(delta, i, m) * pow(omega, j, m) % m for j in range(3)] and got[-1] == pow(delta, i, m) * pow(omega, n - 1, m) % m
        assert got == want[i]
        p.close()


def _sampled(eng, field, k, cols, rng, mont, samples=4096):
    m = pasta.FIELDS[field]
    n = 1 << k
    omega, delta = pasta.omega_for_k(field, k), scalar_delta(m)
    perm = rng.permutation(cols * n)
    mp = np.stack([perm // n, perm % n], axis=-1).astype(np.uint32).reshape(cols, n, 2)
    polys = _device_sigma(eng, field, mp, k, omega, delta, mont)
    for i, p in enumerate(polys):
        rows = np.concatenate([[0, n - 1], rng.integers(0, n, samples - 2)])
        got = p.download()
        p.close()
        for j in rows:
            c, r = (int(x) for x in mp[i, j])
            assert int.from_bytes(got[j].tobytes(), "little") == pow(delta, c, m) * pow(omega, r, m) % m, (k, cols, i, j)


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_sigma_sampled_large(eng, field):
    rng = np.random.default_rng(SEED + 1)
    for k in (18, 20):
        for cols in (1, 3, 12):
            for mont in (False, True):
                _sampled(eng, field, k, cols, rng, mont)


def test_sigma_several_launches_per_column(eng):
    _sampled(eng, "fp", 23, 1, np.random.default_rng(SEED + 2), False)   # 2^23 rows: two pieces of 2^22


# ---- errors ------------------------------------------------------------------------------------------------------------
def _error_cases(eng):
    field, k, n = "fp", 4, 16
    m = pasta.P_MOD
    omega, delta = pasta.omega_for_k(field, k), scalar_delta(m)
    ident = np.stack(np.meshgrid(np.arange(2), np.arange(n), indexing="ij"), axis=-1).astype(np.uint32)
    want = [cref.ints_to_bytes(col) for col in oracle_sigma(ident, n, omega, delta, m)]
    a, b = eng.ResidentPoly(field, n), eng.ResidentPoly(field, n)
    fq, short = eng.ResidentPoly("fq", n), eng.ResidentPoly(field, n - 1)
    gone = eng.ResidentPoly(field, n)
    gone_h = gone._h.value
    gone.close()

    def works():
        a.upload(np.zeros((n, 32), dtype=np.uint8))
        assert _sigma_call([a, b], k, ident, omega, delta) == 0, _err()
        assert (a.download() == want[0]).all() and (b.download() == want[1]).all()

    try:
        works()
        for where, bad in (((1, 5), (2, 0)), ((0, 15), (0, n)), ((0, 0), (0xFFFFFFFF, 0))):
            mp = ident.copy()
            mp[where] = bad
            assert _sigma_call([a, b], k, mp, omega, delta) != 0 and "mapping entry" in _err()
            works()
        cases = (([a, 0xDEADBEEF], "dst[1]: unknown polynomial handle"), ([a, gone_h], "dst[1]: unknown polynomial handle"),
                 ([a, fq], "dst[1]: the polynomials live in different fields"), ([short, a], "dst[0]: a polynomial holds fewer than 2^k elements"),
                 ([a, a], "dst[1] is also dst[0]"))
        for polys, msg in cases:
            assert _sigma_call(polys, k, ident, omega, delta) != 0 and msg in _err(), (polys, _err())
            works()
        assert _sigma_call([a], 31, ident, omega, delta) != 0 and "k > 30" in _err()
        works()
        assert _sigma_call([], k, None, omega, delta, cols=0) == 0, _err()
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
def test_benchmark_circuit_key_and_proof_k14(eng):
    from tests import multiopen_cases as MC
    from tests import plonk_prover as PP
    from tests import plonk_verifier as PV
    from tests import prover_replay as R
    k = 14
    m = pasta.P_MOD
    delta = scalar_delta(m)
    prm = _bench_params(eng, k)
    pk = None
    try:
        D = eng.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
        fixed, sigma, adv = BC.columns(k, m, D.omega, delta, circ.A_SMALL * ZETA % m)
        asm = _bench_assembly(eng, k)
        fc, pc = eng.keygen_vk(prm, D, fixed, asm, delta)
        fb, sb, ab = ([cref.ints_to_bytes(c_) for c_ in cols] for cols in (fixed, sigma, adv))
        host = lambda col: eng.batch_normalize(prm.commit_lagrange(col, eng.Blind(1)).reshape(1, 96), "vesta")[0]   # the current path
        assert (fc == np.stack([host(c_) for c_ in fb])).all() and (pc == np.stack([host(c_) for c_ in sb])).all()
        A = cref.bytes_to_affine
        vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, pasta.Q_MOD, m, D.omega, [A(x) for x in fc], [A(x) for x in pc]))
        pk = eng.keygen_pk(prm, D, fixed, asm, delta, BC.BLINDING_FACTORS)
        T = R.Blake2bTranscript(m)
        PP.create_proof_engine(eng, prm, vk, fb, sb, [ab], [[]], MC.SeededRng("fp", 5, True), T, ZETA, delta)
        want = bytes(T.proof)
        T = R.Blake2bTranscript(m)
        PP.create_proof_engine(eng, prm, vk, None, None, [ab], [[]], MC.SeededRng("fp", 5, True), T, ZETA, delta, pk=prover_pk_dict(pk))
        got = bytes(T.proof)
        assert got == want
        arm = PV.EngineArm(eng, "vesta", k, params=prm)
        try:
            assert PV.verify_proof(arm, vk, got, [[]], delta)
            bad = bytearray(got)
            bad[len(bad) // 2] ^= 4
            assert not PV.verify_proof(arm, vk, bytes(bad), [[]], delta)
        finally:
            arm.close()
    finally:
        if pk is not None:
            pk.close()
        prm.close()


# ---- lanes -------------------------------------------------------------------------------------------------------------
def test_keygen_pk_on_two_lanes(eng):
    k = 12
    m = pasta.P_MOD
    delta = scalar_delta(m)
    prm = _bench_params(eng, k)
    D = eng.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
    fixed = BC.columns(k, m, D.omega, delta, 7)[0]
    asm = _bench_assembly(eng, k)
    lib = _lib()
    pk0 = eng.keygen_pk(prm, D, fixed, asm, delta, BC.BLINDING_FACTORS)
    try:
        want = prover_pk_bytes(pk0)
        handles = {}
        meet = threading.Barrier(2, timeout=300)

        def on_lane(i):
            def go():
                with eng.Lane():
                    pk = eng.keygen_pk(prm, D, fixed, asm, delta, BC.BLINDING_FACTORS)
                    try:
                        got = prover_pk_bytes(pk)
                        handles[i] = pk.permutation.cosets[0]._h.value
                        meet.wait()                                     # both keys exist
                        foreign = [lib.h2_poly_download(ctypes.c_uint64(h), None, ctypes.c_size_t(0), 0) != 0 and "unknown" in _err()
                                   for h in (handles[1 - i], pk0.l0._h.value)]
                        meet.wait()                                     # neither is freed before the other lane looked
                    finally:
                        pk.close()
                return got, foreign
            return go
        for got, foreign in _run_parallel([on_lane(0), on_lane(1)]):
            assert got == want
            assert foreign == [True, True]
        assert lib.h2_poly_download(ctypes.c_uint64(handles[0]), None, ctypes.c_size_t(0), 0) != 0 and "unknown" in _err()
    finally:
        pk0.close()
        prm.close()
