"""GPU test of the curve id every entry point that takes one checks: an id other than H2_CURVE_PALLAS (0) or H2_CURVE_VESTA (1)
fails with "unknown curve id", launches no kernel and leaves the call's outputs unchanged.  Every row also succeeds with the
Vesta id (except the two multi-GPU calls, which need h2_multi_init and check the curve before they ask for it), so each row
fails for its curve id alone."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402

SEED = 0x43555256
N = 4
MARK = 0xA5
VESTA = 1


def _sz(n):
    return ctypes.c_size_t(n)


def _host(nbytes):
    return np.full(nbytes, MARK, dtype=np.uint8)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _rows(torch, lib):
    """name -> make(): a fresh (call(curve) -> rc, outputs, cleanup(rc)) for one entry point; outputs start as MARK bytes."""
    c = pasta.VESTA
    pts = cref.gen_points("vesta", SEED, N)                                         # affine, canonical
    jac = np.ascontiguousarray(np.concatenate([pts, np.tile(cref.ints_to_bytes([1]), (N, 1))], axis=1))   # z = 1
    scal = cref.gen_scalars(c.scalar, SEED + 1, N)
    omega = np.ascontiguousarray(cref.ints_to_bytes([pasta.omega_for_k(c.scalar, 2)])[0])
    canon = 0
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def dev(nbytes, fill=MARK):
        return torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda")

    def dptr(t):
        return ctypes.c_void_p(t.data_ptr())

    def release(fn, h):
        return lambda rc: fn(ctypes.c_uint64(h.value)) if rc == 0 else 0

    def msm():
        out = _host(96)
        return lambda cv: lib.h2_msm(cv, _p(scal), _p(pts), _sz(N), canon, _p(out)), [out], None

    def msm_dev():
        ds, db = torch.from_numpy(scal.copy()).cuda(), torch.from_numpy(pts.copy()).cuda()
        out = dev(96)
        return (lambda cv: lib.h2_msm_dev(cv, dptr(ds), canon, dptr(db), _sz(N), ctypes.c_uint32(0), dptr(out), stream)), [out], None

    def register():
        h = ctypes.c_uint64(MARK)
        return (lambda cv: lib.h2_bases_register(cv, _p(pts), _sz(N), canon, ctypes.byref(h))), [h], release(lib.h2_bases_release, h)

    def register_ex():
        h = ctypes.c_uint64(MARK)
        return ((lambda cv: lib.h2_bases_register_ex(cv, _p(pts), _sz(N), canon, ctypes.c_uint32(0), ctypes.c_uint32(1), ctypes.byref(h))),
                [h], release(lib.h2_bases_release, h))

    def point_sum():
        out = _host(96)
        return lambda cv: lib.h2_point_sum(cv, _p(jac), _sz(N), canon, _p(out)), [out], None

    def point_sum_dev():
        dj = dev(N * 96, 0)                                                          # N identities (z = 0), Montgomery in
        out = dev(96)
        return lambda cv: lib.h2_point_sum_dev(cv, dptr(dj), _sz(N), dptr(out), stream), [out], None

    def msm_multi_gpu():
        out = _host(96)
        return lambda cv: lib.h2_msm_multi_gpu(cv, _p(scal), _p(pts), _sz(N), canon, _p(out)), [out], None

    def multi_register():
        h = ctypes.c_uint64(MARK)
        return (lambda cv: lib.h2_multi_bases_register(cv, _p(pts), _sz(N), canon, ctypes.byref(h))), [h], release(lib.h2_multi_bases_release, h)

    def ec_fft():
        io = np.ascontiguousarray(jac.reshape(-1).copy())                            # in place: the points are the output
        return (lambda cv: lib.h2_ec_fft(cv, _p(io), _p(omega), ctypes.c_uint32(2), None, canon)), [io], None

    def params_lagrange():
        out = _host(N * 64)
        minv = np.ascontiguousarray(cref.ints_to_bytes([pow(4, -1, c.r)])[0])
        return lambda cv: lib.h2_params_lagrange(cv, _p(pts), ctypes.c_uint32(2), _p(omega), _p(minv), canon, _p(out)), [out], None

    def params_new():
        g, gl, w, u = _host(N * 64), _host(N * 64), _host(64), _host(64)
        return lambda cv: lib.h2_params_new(cv, ctypes.c_uint32(2), canon, _p(g), _p(gl), _p(w), _p(u)), [g, gl, w, u], None

    def hash_to_curve():
        out = _host(N * 64)
        msgs = np.arange(N * 8, dtype=np.uint8)
        return lambda cv: lib.h2_hash_to_curve(cv, b"curve-args", _p(msgs), _sz(8), _sz(N), canon, _p(out)), [out], None

    def batch_normalize():
        out = _host(N * 64)
        return lambda cv: lib.h2_batch_normalize(cv, _p(jac), _sz(N), canon, _p(out)), [out], None

    def compress():
        out = _host(N * 32)
        return lambda cv: lib.h2_points_compress(cv, _p(pts), _sz(N), canon, _p(out)), [out], None

    def decompress():
        enc = np.zeros(N * 32, dtype=np.uint8)                                       # the identity's encoding
        out = _host(N * 64)
        return lambda cv: lib.h2_points_decompress(cv, _p(enc), _sz(N), canon, _p(out)), [out], None

    def gen_points():
        out = dev(N * 64)
        return lambda cv: lib.h2_dev_gen_points(cv, ctypes.c_uint64(7), ctypes.c_uint64(0), _sz(N), dptr(out), stream), [out], None

    def curve_op():
        out = _host(N * 64)
        return lambda cv: lib.h2_test_curve_op(cv, 0, _p(pts), _p(pts[::-1].copy()), _sz(N), _p(out)), [out], None

    return {"h2_msm": msm, "h2_msm_dev": msm_dev, "h2_bases_register": register, "h2_bases_register_ex": register_ex,
            "h2_point_sum": point_sum, "h2_point_sum_dev": point_sum_dev, "h2_msm_multi_gpu": msm_multi_gpu,
            "h2_multi_bases_register": multi_register, "h2_ec_fft": ec_fft, "h2_params_lagrange": params_lagrange,
            "h2_params_new": params_new, "h2_hash_to_curve": hash_to_curve, "h2_batch_normalize": batch_normalize,
            "h2_points_compress": compress, "h2_points_decompress": decompress, "h2_dev_gen_points": gen_points,
            "h2_test_curve_op": curve_op}


def _snapshot(torch, outs):
    torch.cuda.synchronize()
    snap = []
    for o in outs:
        if isinstance(o, ctypes.c_uint64):
            snap.append(o.value)
        elif isinstance(o, np.ndarray):
            snap.append(o.tobytes())
        else:
            snap.append(o.cpu().numpy().tobytes())
    return snap


NEEDS_MULTI_INIT = {"h2_msm_multi_gpu", "h2_multi_bases_register"}


ENTRY_POINTS = ["h2_msm", "h2_msm_dev", "h2_bases_register", "h2_bases_register_ex", "h2_point_sum", "h2_point_sum_dev",
                "h2_msm_multi_gpu", "h2_multi_bases_register", "h2_ec_fft", "h2_params_lagrange", "h2_params_new", "h2_hash_to_curve",
                "h2_batch_normalize", "h2_points_compress", "h2_points_decompress", "h2_dev_gen_points", "h2_test_curve_op"]


@pytest.mark.parametrize("name", ENTRY_POINTS)
def test_unknown_curve_id_fails_before_any_launch(name):
    import torch
    from halo2_b200 import lib as L
    lib = L.init()
    make = _rows(torch, lib)[name]
    for bad in (2, -1):
        call, outs, _ = make()
        before = _snapshot(torch, outs)
        launches = lib.h2_launch_count()
        assert call(ctypes.c_int(bad)) != 0, (name, bad)
        assert lib.h2_last_error().decode() == "unknown curve id", (name, bad)
        assert lib.h2_launch_count() == launches, (name, bad)
        assert _snapshot(torch, outs) == before, (name, bad)
    if name not in NEEDS_MULTI_INIT:
        call, outs, cleanup = make()
        rc = call(ctypes.c_int(VESTA))
        assert rc == 0, (name, lib.h2_last_error().decode())
        if cleanup:
            L.check(cleanup(rc))
        torch.cuda.synchronize()
