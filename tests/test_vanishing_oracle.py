"""CPU checks of h2_poly_vanishing_quotient's pass bodies (csrc/ntt.cuh: NTT_IN_TABLE on the first pass, NTT_OUT_PIECES on
the last) on the host emulation: one transform gives the pieces of extended_to_coeff(divide_by_vanishing_poly(h)), against
the oracle's two steps chunked into n coefficients, and the size checks that reject a call before anything is launched."""
import ctypes

import numpy as np
import pytest

from oracle import cref, pasta
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

