"""CPU checks of h2_poly_vanishing_quotient's pass bodies (csrc/ntt.cuh: NTT_IN_TABLE on the first pass, NTT_OUT_PIECES on
the last) on the host emulation: one transform gives the pieces of extended_to_coeff(divide_by_vanishing_poly(h)), against
the oracle's two steps chunked into n coefficients, and the size checks that reject a call before anything is launched."""
import ctypes

import numpy as np
import pytest

from oracle import cref, pasta
from tests import plonk_prover as PP
from tests.kernel_emul import build as emul_build


@pytest.fixture(scope="module")
def emu():
    lib = ctypes.CDLL(emul_build.build())
    lib.emu_vanishing_quotient_sizes.restype = ctypes.c_char_p
    return lib


def _quotient(emu, D, h, count, reverse=False, nthr=64):
    n = D.n
    out = np.zeros((count, n, 32), dtype=np.uint8)
    t = cref.ints_to_bytes(D.t_evaluations)
    rc = emu.emu_vanishing_quotient(cref.FIELD_ID[D.field], cref._p(h), D.k, D.extended_k, ctypes.c_uint64(count),
                                    cref._p(cref._fe(D.extended_omega_inv)), cref._p(cref._fe(D.extended_ifft_divisor)),
                                    cref._p(cref._fe(D.g_coset)), cref._p(t), len(D.t_evaluations), cref._p(out), int(reverse), nthr)
    return out, rc


def _want(D, h):
    """The oracle's divide_by_vanishing_poly then extended_to_coeff (every coefficient: out_len = 2^ext_k)."""
    div = cref.ints_to_bytes(D.divide_by_vanishing_poly(cref.bytes_to_ints(h)))
    return cref.extended_to_coeff(D.field, div, D.extended_k, D.extended_omega_inv, D.extended_ifft_divisor, D.g_coset, D.extended_len())


# cs degree j -> extended_k - k: quotient_poly_degree j - 1 rounds up to 2, 4 or 8 times n
_DEGREES = {1: 3, 2: 5, 3: 9}


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("ext", [1, 2, 3])
def test_pieces_equal_the_oracle(emu, field, ext):
    """k = 0 .. 10, extended_k = k + ext: for every count from 1 to 2^ext the pieces are the first count x n coefficients of
    the oracle's quotient, n at a time, and no store lands outside a piece.  Odd k visit every launch's tiles last-first."""
    j = _DEGREES[ext]
    for k in range(0, 11):
        D = pasta.EvaluationDomain(field, j, k)
        assert D.extended_k == k + ext
        h = cref.gen_scalars(field, 4000 + 100 * k + ext, D.extended_len())
        want = _want(D, h)
        passes = 1 if D.extended_k <= 10 else -(-D.extended_k // 7)       # ntt_plan
        for count in range(1, (1 << ext) + 1):
            got, rc = _quotient(emu, D, h, count, reverse=bool(k & 1), nthr=(7 if k < 4 else 64))
            assert rc == passes, (field, k, ext, count, rc)
            for i in range(count):
                assert (got[i] == want[i * D.n:(i + 1) * D.n]).all(), (field, k, ext, count, i)


def test_the_benchmark_circuits_degree(emu):
    """A degree whose quotient does not fill the extended domain (j = 4: 3 pieces of 4n): the pieces, then nothing."""
    D = pasta.EvaluationDomain("fp", 4, 9)
    assert (D.quotient_poly_degree, D.extended_k) == (3, 11)
    h = cref.gen_scalars("fp", 99, D.extended_len())
    want = _want(D, h)
    got, rc = _quotient(emu, D, h, 3)
    assert rc == 2
    assert (got.reshape(-1, 32) == want[:3 * D.n]).all()


@pytest.mark.parametrize("k, ext_k, count, t_len, reason", [
    (4, 31, 1, 1, b"ext_k > 30"),
    (5, 4, 1, 1, b"ext_k < k"),
    (4, 6, 0, 4, b"count must be at least 1 and count * 2^k at most 2^ext_k"),
    (4, 6, 5, 4, b"count must be at least 1 and count * 2^k at most 2^ext_k"),
    (0, 0, 2, 1, b"count must be at least 1 and count * 2^k at most 2^ext_k"),
    (4, 6, 1, 0, b"t_len must be a power of two <= 2^ext_k"),
    (4, 6, 1, 3, b"t_len must be a power of two <= 2^ext_k"),
    (4, 6, 1, 128, b"t_len must be a power of two <= 2^ext_k"),
])
def test_sizes_rejected_before_any_launch(emu, k, ext_k, count, t_len, reason):
    assert emu.emu_vanishing_quotient_sizes(k, ext_k, ctypes.c_uint64(count), t_len) == reason
    out = np.zeros((max(count, 1), 1, 32), dtype=np.uint8)
    h = np.zeros((2, 32), dtype=np.uint8)
    assert emu.emu_vanishing_quotient(0, cref._p(h), k, ext_k, ctypes.c_uint64(count), None, None, None, None, t_len, cref._p(out), 0, 1) == -1


@pytest.mark.parametrize("k, ext_k, count, t_len", [(0, 0, 1, 1), (4, 6, 4, 4), (4, 6, 1, 64), (10, 30, 1 << 20, 1 << 20), (30, 30, 1, 1)])
def test_sizes_accepted(emu, k, ext_k, count, t_len):
    assert emu.emu_vanishing_quotient_sizes(k, ext_k, ctypes.c_uint64(count), t_len) is None


def test_a_whole_proof_with_the_module_over_the_stand_in():
    """A proof whose vanishing argument comes from halo2_b200.vanishing (tests/arguments_cases.create_proof_package), over the
    ABI stand-in with the fused bodies on the host emulation: the same points, scalars, h_poly / random_poly queries and proof
    bytes as create_proof_engine on the plonk_api circuit under its golden key, one quotient call instead of the division,
    transform and copies, and every polynomial released."""
    import halo2_b200
    from tests import arguments_cases as AC
    from tests import fake_engine
    from tests import multiopen_cases as MC
    from tests import plonk_api_circuit as circ
    from tests import plonk_verifier as PV
    from tests import vanishing_cases as VC
    vk = circ.plonk_api_key()
    P = pasta.Params.new(pasta.VESTA, 5)
    gens = (cref.affines_to_bytes(P.g), cref.affines_to_bytes(P.g_lagrange), cref.affines_to_bytes([P.w]), cref.affines_to_bytes([P.u]))
    fixed, sigma = circ.fixed_columns(circ.M, circ.ZETA), circ.permutation_columns(circ.M, vk.omega, circ.DELTA)
    inst = [[[2]], [[2]]]
    adv = [circ.witness(), circ.witness()]
    with fake_engine.installed() as fake:
        prm = halo2_b200.Params("vesta", 5, *gens[:3], u=gens[3])
        D = halo2_b200.EvaluationDomain("fp", vk.degree(), vk.k, circ.ZETA)
        want = VC.record(halo2_b200, circ.M, lambda eng, t: PP.create_proof_engine(eng, prm, vk, fixed, sigma, adv, inst, MC.SeededRng("fp", 777, True),
                                                                                  t, circ.ZETA, circ.DELTA))
        pk = AC.proving_key(halo2_b200, D, fixed, sigma, vk.blinding_factors())
        fake.calls.clear()
        got = VC.record(halo2_b200, circ.M, lambda eng, t: AC.create_proof_package(eng, prm, D, pk, vk, adv, inst, MC.SeededRng("fp", 777, True), t,
                                                                                  circ.DELTA))
        assert fake.calls.count("h2_poly_vanishing_quotient") == 1
        assert "h2_poly_divide_by_vanishing" not in fake.calls and "h2_poly_extended_to_coeff" not in fake.calls
        assert len(got["points"]) == len(want["points"]) and all(np.array_equal(a, b) for a, b in zip(got["points"], want["points"]))
        assert got["scalars"] == want["scalars"]
        for (px, pa, pb), (wx, wa, wb) in zip(got["queries"], want["queries"]):
            assert px == wx and pb == wb and np.array_equal(pa, wa)
        assert got["proof"] == want["proof"] and len(got["proof"]) == 4160
        pk.close()
        assert not fake.polys
        earm = PV.EngineArm(halo2_b200, "vesta", 5, *gens)
        assert PV.verify_proof(earm, vk, got["proof"], inst, circ.DELTA)
        earm.close()
        prm.close()
