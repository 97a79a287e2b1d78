"""GPU tests of the stream contract of the two entry points that run on a caller's stream, h2_msm_dev and h2_ntt_dev
(include/halo2_b200.h): a call runs after the caller's earlier work on `stream` and after the calling context's earlier
calls, and the context's later calls run after it.  Both use the context's MSM / NTT scratch, twiddle cache and pow2 while
their kernels run on the caller's stream.  Every case issues its calls with no host synchronisation between them and checks
every result bit for bit against the oracle, on the primary context and on a lane.  Ordinary work whose results are checked:
nothing here tries to provoke a race, so a pass is evidence of the contract only together with the code."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402

SEED = 0x53545245414D
LOG_N = 20              # NTTs: several passes, so the transform runs through the NTT scratch
MSM_N = 1 << 18
FIELD, CURVE = "fp", "vesta"   # vesta's scalar field is fp


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


@pytest.fixture(params=["primary", "lane"])
def ctx(request, eng):
    if request.param == "lane":
        with eng.Lane():
            yield eng
    else:
        yield eng


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


def _lib():
    from halo2_b200 import lib as L
    return L


def _u8(a):
    return np.ascontiguousarray(a.cpu().numpy()).view(np.uint8)


def _ntt_dev(x, out, omega, stream, log_n=LOG_N):
    L = _lib()
    return L.load().h2_ntt_dev(L.FIELD_ID[FIELD], ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), L.ptr(L.fe_bytes(omega)),
                               L.REPR_CANONICAL, ctypes.c_uint32(log_n), ctypes.c_void_p(stream.cuda_stream))


def _msm_dev(sc, bases, out, stream, window_bits=0):
    L = _lib()
    return L.load().h2_msm_dev(L.CURVE_ID[CURVE], ctypes.c_void_p(sc.data_ptr()), L.REPR_CANONICAL, ctypes.c_void_p(bases.data_ptr()),
                               ctypes.c_size_t(sc.shape[0]), ctypes.c_uint32(window_bits), ctypes.c_void_p(out.data_ptr()),
                               ctypes.c_void_p(stream.cuda_stream))


def _lagrange_to_coeff(dst, src, omega):
    """The resident transform with divisor 1: best_fft of src with `omega`, on the context's stream, asynchronous."""
    L = _lib()
    L.check(L.load().h2_poly_lagrange_to_coeff(dst._h, src._h, ctypes.c_uint32(LOG_N), L.ptr(L.fe_bytes(omega)), L.ptr(L.fe_bytes(1)),
                                               L.REPR_CANONICAL))


def _canon_affine(xyz_mont: np.ndarray) -> np.ndarray:
    """h2_msm_dev's Montgomery Jacobian result as the oracle's canonical affine point."""
    m = pasta.CURVES[CURVE].p
    rinv = pow((1 << 256) % m, m - 2, m)
    canon = cref.ints_to_bytes([v * rinv % m for v in cref.bytes_to_ints(xyz_mont.reshape(3, 32))]).reshape(-1)
    return cref.jac_to_affine(CURVE, canon)


class Ntt:
    """Inputs of the NTT cases: `k` vectors of 2^LOG_N canonical elements, as host arrays, as device tensors (raw residues for
    h2_ntt_dev, which the transform treats linearly) and as resident polynomials, and the oracle's transforms."""

    def __init__(self, torch, eng, k, seed):
        n = 1 << LOG_N
        self.omega = pasta.omega_for_k(FIELD, LOG_N)
        self.host = [cref.gen_scalars(FIELD, seed + i, n) for i in range(k)]
        self.want = [cref.best_fft(FIELD, a, self.omega, LOG_N) for a in self.host]
        self.dev = [torch.from_numpy(a).cuda() for a in self.host]
        self.out = [torch.zeros_like(d) for d in self.dev]
        self.poly = [eng.ResidentPoly(FIELD, n, a) for a in self.host]
        self.res = []
        torch.cuda.synchronize()

    def result(self, eng):
        """A new zero-filled resident polynomial for one transform's output."""
        self.res.append(eng.ResidentPoly(FIELD, 1 << LOG_N))
        return self.res[-1]

    def close(self):
        for p in self.poly + self.res:
            p.close()


class Msm:
    """Inputs of the MSM cases: `k` scalar vectors against one set of bases, on the host (canonical) and on the device
    (scalars canonical, bases Montgomery as h2_msm_dev takes them), and the oracle's sums."""

    def __init__(self, torch, k, seed):
        L = _lib()
        self.bases = cref.gen_points(CURVE, seed, MSM_N)
        self.scalars = [cref.gen_scalars(FIELD, seed + 1 + i, MSM_N) for i in range(k)]
        self.want = [cref.best_multiexp(CURVE, s, self.bases) for s in self.scalars]
        self.d_bases = torch.from_numpy(self.bases).cuda()
        L.check(L.load().h2_dev_convert(L.FIELD_ID[L.BASE_FIELD[CURVE]], ctypes.c_void_p(self.d_bases.data_ptr()), ctypes.c_size_t(2 * MSM_N), 1,
                                        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
        self.d_scalars = [torch.from_numpy(s).cuda() for s in self.scalars]
        self.d_out = [torch.zeros(96, dtype=torch.uint8, device="cuda") for _ in self.scalars]
        torch.cuda.synchronize()


def test_cold_twiddles_built_on_the_caller_stream(ctx, torch):
    """h2_ntt_dev on a side stream builds a new twiddle entry there, and a resident transform right behind it on the context's
    stream reads that entry; then the same with the resident transform building it and h2_ntt_dev reading it."""
    L = _lib()
    side = torch.cuda.Stream()
    assert side.cuda_stream != torch.cuda.current_stream().cuda_stream
    d = Ntt(torch, ctx, 2, SEED)
    try:
        for first_dev in (True, False):
            res = d.result(ctx)
            d.out[0].zero_()
            L.check(L.load().h2_ntt_clear_cache())   # synchronises the device
            if first_dev:
                L.check(_ntt_dev(d.dev[0], d.out[0], d.omega, side))
                _lagrange_to_coeff(res, d.poly[1], d.omega)
            else:
                _lagrange_to_coeff(res, d.poly[1], d.omega)
                L.check(_ntt_dev(d.dev[0], d.out[0], d.omega, side))
            assert (res.download() == d.want[1]).all(), f"resident transform, h2_ntt_dev first: {first_dev}"
            side.synchronize()
            assert (_u8(d.out[0]).reshape(-1, 32) == d.want[0]).all(), f"h2_ntt_dev, h2_ntt_dev first: {first_dev}"
    finally:
        d.close()


def test_ntt_scratch_shared_with_the_context_stream(ctx, torch):
    """h2_ntt on the context's stream, h2_ntt_dev on a side stream, then a resident transform: all three through one NTT
    scratch and one twiddle entry."""
    side = torch.cuda.Stream()
    d = Ntt(torch, ctx, 3, SEED + 10)
    res = d.result(ctx)
    try:
        got = d.host[0].copy()
        ctx.best_fft(got, d.omega, LOG_N, FIELD)
        _lib().check(_ntt_dev(d.dev[1], d.out[1], d.omega, side))
        _lagrange_to_coeff(res, d.poly[2], d.omega)
        assert (got == d.want[0]).all(), "h2_ntt"
        assert (res.download() == d.want[2]).all(), "resident transform after h2_ntt_dev"
        side.synchronize()
        assert (_u8(d.out[1]).reshape(-1, 32) == d.want[1]).all(), "h2_ntt_dev"
    finally:
        d.close()


def test_msm_scratch_shared_with_the_context_stream(ctx, torch):
    """h2_msm on the context's stream, h2_msm_dev on a side stream, then h2_msm_registered: all three through one MSM scratch."""
    L = _lib()
    lib = L.load()
    side = torch.cuda.Stream()
    m = Msm(torch, 3, SEED + 20)
    h = ctypes.c_uint64(0)
    L.check(lib.h2_bases_register(L.CURVE_ID[CURVE], L.ptr(m.bases), ctypes.c_size_t(MSM_N), L.REPR_CANONICAL, ctypes.byref(h)))
    try:
        got0 = ctx.best_multiexp(m.scalars[0], m.bases, CURVE)
        L.check(_msm_dev(m.d_scalars[1], m.d_bases, m.d_out[1], side))
        got2 = np.zeros(96, dtype=np.uint8)
        L.check(lib.h2_msm_registered(h, L.ptr(m.scalars[2]), ctypes.c_size_t(MSM_N), None, L.REPR_CANONICAL, L.ptr(got2)))
        assert (cref.jac_to_affine(CURVE, got0) == m.want[0]).all(), "h2_msm"
        assert (cref.jac_to_affine(CURVE, got2) == m.want[2]).all(), "h2_msm_registered after h2_msm_dev"
        side.synchronize()
        assert (_canon_affine(_u8(m.d_out[1])) == m.want[1]).all(), "h2_msm_dev"
    finally:
        L.check(lib.h2_bases_release(h))


def test_caller_work_before_and_after_on_the_same_stream(ctx, torch):
    """A torch kernel on the side stream writes the input, the entry point runs on that stream, and a torch op on it reads
    the output."""
    L = _lib()
    side = torch.cuda.Stream()
    d = Ntt(torch, ctx, 1, SEED + 30)
    m = Msm(torch, 1, SEED + 40)
    x = torch.zeros_like(d.dev[0])
    sc = torch.zeros_like(m.d_scalars[0])
    torch.cuda.synchronize()
    try:
        with torch.cuda.stream(side):
            x.copy_(d.dev[0])
            L.check(_ntt_dev(x, d.out[0], d.omega, side))
            ntt_read = d.out[0].clone()
            sc.copy_(m.d_scalars[0])
            L.check(_msm_dev(sc, m.d_bases, m.d_out[0], side))
            msm_read = m.d_out[0].clone()
        side.synchronize()
        assert (_u8(ntt_read).reshape(-1, 32) == d.want[0]).all(), "h2_ntt_dev between torch ops on its stream"
        assert (_canon_affine(_u8(msm_read)) == m.want[0]).all(), "h2_msm_dev between torch ops on its stream"
    finally:
        d.close()


def test_argument_errors_leave_later_calls_ordered(ctx, torch):
    """h2_msm_dev with window_bits = 25 and h2_ntt_dev with log_n = 31 fail before any launch; the calls after them, on the
    side stream and on the context's stream, are still ordered and correct."""
    L = _lib()
    lib = L.load()
    side = torch.cuda.Stream()
    d = Ntt(torch, ctx, 2, SEED + 50)
    m = Msm(torch, 1, SEED + 60)
    res = d.result(ctx)
    try:
        launches = L.launch_count()
        assert _msm_dev(m.d_scalars[0], m.d_bases, m.d_out[0], side, window_bits=25) != 0
        assert lib.h2_last_error().decode() == "msm: window bits > 24"
        assert _ntt_dev(d.dev[0], d.out[0], d.omega, side, log_n=31) != 0
        assert lib.h2_last_error().decode() == "ntt: log_n > 30 not supported"
        assert L.launch_count() == launches
        L.check(_msm_dev(m.d_scalars[0], m.d_bases, m.d_out[0], side))
        L.check(_ntt_dev(d.dev[0], d.out[0], d.omega, side))
        _lagrange_to_coeff(res, d.poly[1], d.omega)
        assert (res.download() == d.want[1]).all(), "resident transform after the failed calls"
        side.synchronize()
        assert (_u8(d.out[0]).reshape(-1, 32) == d.want[0]).all(), "h2_ntt_dev after the failed calls"
        assert (_canon_affine(_u8(m.d_out[0])) == m.want[0]).all(), "h2_msm_dev after the failed calls"
    finally:
        d.close()
