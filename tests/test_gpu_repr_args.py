"""GPU tests of the encoding argument every entry point that takes host field elements or points checks (include/halo2_b200.h,
`repr`):

- a repr other than H2_REPR_CANONICAL (0) or H2_REPR_MONTGOMERY (1) fails with "<entry point>: unknown repr";
- a NULL host element or element array the call reads or writes fails with "<entry point>: null <parameter>"; the documented
  optional pointers, and the elements of a call with nothing to do (no lookups, columns or proofs, ...), may still be NULL;
- both failures launch no kernel and leave the call's outputs as they were (host bytes, resident polynomials, out handles);
- the same inputs give the same answer in either encoding: canonical inputs with repr 0 and their Montgomery forms
  (x 2^256 mod m, coordinate by coordinate for points) with repr 1.  Host results are compared after the same map, resident
  ones after a canonical download.  Jacobian results are compared as affine points: only the group element is defined."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests.abi_cases import _err  # noqa: E402

SEED = 0x52455052
K, N = 4, 1 << 4
MARK = 0xA5
VESTA, FP = 1, 0
S, B = "fp", "fq"                     # Vesta's scalar and base fields
R = 1 << 256


def _sz(n):
    return ctypes.c_size_t(n)


def _u32(n):
    return ctypes.c_uint32(n)


def _u64(n):
    return ctypes.c_uint64(n)


def _arr(hs):
    return (ctypes.c_uint64 * len(hs))(*hs)


def _fes(xs):
    return cref.ints_to_bytes(xs)


def _mark(nbytes):
    return np.full(nbytes, MARK, dtype=np.uint8)


def _conv(a, field, to_mont):
    """32-byte elements (or point coordinates) canonical -> Montgomery, or back."""
    m = pasta.FIELDS[field]
    f = R % m if to_mont else pow(R, -1, m)
    return cref.ints_to_bytes([x * f % m for x in cref.bytes_to_ints(a)]).reshape(np.shape(a))


class Enc:
    """The encoding of one run: enc() maps canonical host inputs into it, dec() maps host results back."""

    def __init__(self, repr):
        self.repr = repr

    def enc(self, a, field):
        return _conv(a, field, True) if self.repr else np.ascontiguousarray(a)

    def dec(self, a, field):
        return _conv(a, field, False) if self.repr else np.asarray(a).copy()


CANON, MONT = Enc(0), Enc(1)


def _affine(xyz):
    """Jacobian points (96 B each) -> affine bytes: a result is only defined up to the group element."""
    a = np.frombuffer(bytes(xyz), dtype=np.uint8).reshape(-1, 96)
    return b"".join(cref.jac_to_affine("vesta", p).tobytes() for p in a)


def _c(v):
    import torch
    if isinstance(v, np.ndarray):
        return ctypes.c_void_p(v.ctypes.data)
    if isinstance(v, torch.Tensor):
        return ctypes.c_void_p(v.data_ptr())
    return v


class Row:
    """One call of an entry point.  args: the arguments in order, by their header names (numpy arrays and tensors are passed
    as pointers); outs: what the call writes; result(): its answer, canonical; needs: the element pointers a NULL of which
    fails; optional: overrides (NULL pointers and what makes them optional) the call succeeds with; after(rc): cleanup."""

    def __init__(self, fn, args, outs, result, needs=(), optional=(), repr_arg="repr", after=None):
        self.fn, self.args, self.outs, self.result = fn, args, outs, result
        self.needs, self.optional, self.repr_arg, self.after = list(needs), list(optional), repr_arg, after

    def call(self, **over):
        return self.fn(*[_c(over.get(k, v)) for k, v in self.args.items()])


class Env:
    def __init__(self, lib, prm):
        import torch
        self.lib, self.prm, self.torch = lib, prm, torch
        self.polys = []
        self.stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def poly(self, values=None, n=N):
        import halo2_b200 as eng
        p = eng.ResidentPoly(S, n, values)
        self.polys.append(p)
        return p

    def close(self):
        for p in self.polys:
            p.close()
        self.polys = []


def _scal(seed, n=N):
    return cref.gen_scalars(S, SEED + seed, n)


def _rows(E):
    """entry point -> make(e): a fresh Row in the encoding e."""
    lib, prm, torch = E.lib, E.prm, E.torch
    pts = cref.gen_points("vesta", SEED, N)
    jac = np.ascontiguousarray(np.concatenate([pts, np.tile(_fes([1]), (N, 1))], axis=1))
    scal = _scal(1)
    fe = lambda x: _fes([x])[0]
    hs = lambda ps: _arr([p._h.value for p in ps])
    down = lambda ps: b"".join(p.download().tobytes() for p in ps)

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a).reshape(-1).copy()).cuda()

    def host_out(nbytes, field, e, jac=False):
        out = _mark(nbytes)
        return out, (lambda: (_affine if jac else bytes)(e.dec(out, field).tobytes()))

    # ---- MSM side --------------------------------------------------------------------------------------------------------
    def msm(e):
        out, res = host_out(96, B, e, True)
        return Row(lib.h2_msm, dict(curve=VESTA, scalars=e.enc(scal, S), bases_xy=e.enc(pts, B), n=_sz(N), repr=e.repr, out_xyz=out), [out], res,
                   ["scalars", "bases_xy", "out_xyz"])

    def msm_dev(e):
        ds, db, out = dev(e.enc(scal, S)), dev(MONT.enc(pts, B)), dev(_mark(96))

        def res():
            torch.cuda.synchronize()
            return _affine(MONT.dec(out.cpu().numpy(), B).tobytes())
        return Row(lib.h2_msm_dev, dict(curve=VESTA, d_scalars=ds, scalars_repr=e.repr, d_bases=db, n=_sz(N), window_bits=_u32(0), d_out_xyz=out,
                                        stream=E.stream), [out], res, repr_arg="scalars_repr")

    def register(ex):
        def make(e):
            h = _u64(MARK)
            out = _mark(96)

            def res():
                assert lib.h2_msm_registered(h, _c(scal), _sz(N), None, 0, _c(out)) == 0, _err()
                return _affine(out.tobytes())
            args = dict(curve=VESTA, bases_xy=e.enc(pts, B), n=_sz(N), repr=e.repr)
            args.update(dict(window_bits=_u32(0), flags=_u32(1)) if ex else {})
            args["handle"] = ctypes.byref(h)
            return Row(lib.h2_bases_register_ex if ex else lib.h2_bases_register, args, [h], res, ["bases_xy"],
                       after=lambda rc: rc == 0 and lib.h2_bases_release(h))
        return make

    def msm_registered(e):
        out, res = host_out(96, B, e, True)
        return Row(lib.h2_msm_registered, dict(handle=prm._h_g, scalars=e.enc(scal, S), n=_sz(N), extra_scalar=e.enc(_fes([7]), S), repr=e.repr,
                                               out_xyz=out), [out], res, ["scalars", "out_xyz"], [dict(extra_scalar=None)])

    def batch(affine):
        def make(e):
            name = "out_xy" if affine else "out_xyz"
            out, res = host_out(2 * (64 if affine else 96), B, e, not affine)
            fn = lib.h2_msm_registered_batch_affine if affine else lib.h2_msm_registered_batch
            return Row(fn, {"handle": prm._h_g, "scalars": e.enc(_scal(2, 2 * N), S), "n": _sz(N), "extra_scalars": e.enc(_fes([7, 8]), S),
                            "batch": _sz(2), "repr": e.repr, name: out}, [out], res, ["scalars", name], [dict(extra_scalars=None)])
        return make

    def point_sum(e):
        out, res = host_out(96, B, e, True)
        return Row(lib.h2_point_sum, dict(curve=VESTA, points_xyz=e.enc(jac, B), g=_sz(N), repr=e.repr, out_xyz=out), [out], res,
                   ["points_xyz", "out_xyz"])

    def multi_init():                                                                # only the multi-GPU rows need it: the one device
        assert lib.h2_multi_init(1) == 0, _err()

    def msm_multi_gpu(e):
        multi_init()
        out, res = host_out(96, B, e, True)
        return Row(lib.h2_msm_multi_gpu, dict(curve=VESTA, scalars=e.enc(scal, S), bases_xy=e.enc(pts, B), n=_sz(N), repr=e.repr, out_xyz=out),
                   [out], res, ["scalars", "bases_xy", "out_xyz"])

    def multi_register(e):
        multi_init()
        h = _u64(MARK)
        out = _mark(96)

        def res():
            assert lib.h2_msm_multi_registered(h, _c(scal), _sz(N), 0, _c(out)) == 0, _err()
            return _affine(out.tobytes())
        return Row(lib.h2_multi_bases_register, dict(curve=VESTA, bases_xy=e.enc(pts, B), n=_sz(N), repr=e.repr, handle=ctypes.byref(h)), [h],
                   res, ["bases_xy"], after=lambda rc: rc == 0 and lib.h2_multi_bases_release(h))

    def multi_registered(e):
        multi_init()
        h = _u64(0)
        assert lib.h2_multi_bases_register(VESTA, _c(pts), _sz(N), 0, ctypes.byref(h)) == 0, _err()
        out, res = host_out(96, B, e, True)
        return Row(lib.h2_msm_multi_registered, dict(handle=h, scalars=e.enc(scal, S), n=_sz(N), repr=e.repr, out_xyz=out), [out], res,
                   ["scalars", "out_xyz"], after=lambda rc: lib.h2_multi_bases_release(h))

    # ---- IPA: a session's remaining rounds run in canonical form, then it finishes --------------------------------------
    def rounds(sess, first, last):
        lrs = []
        for j in range(first, last):
            lr = np.zeros(192, dtype=np.uint8)
            u = 11 + j
            assert lib.h2_ipa_round(sess, _c(fe(3 + j)), _c(fe(5 + j)), _c(fe(9 + j)), 0, _c(lr)) == 0, _err()
            assert lib.h2_ipa_fold(sess, _c(fe(u)), _c(fe(pow(u, -1, pasta.FIELDS[S]))), 0) == 0, _err()
            lrs.append(_affine(lr.tobytes()))
        return b"".join(lrs)

    def finish(sess, state, first):
        state["open"] = False
        cb = np.zeros(64, dtype=np.uint8)
        lrs = rounds(sess, first, K)
        assert lib.h2_ipa_finish(sess, 0, _c(cb)) == 0, _err()
        return lrs + cb.tobytes()

    def open_session(n_rounds=0):
        sess = _u64(0)
        assert lib.h2_ipa_begin(prm._h_g, _u32(K), _c(_scal(3)), _c(fe(6)), 0, ctypes.byref(sess)) == 0, _err()
        rounds(sess, 0, n_rounds)
        return sess, {"open": True}

    def abort(sess, state):
        def after(rc):
            if state["open"]:
                assert lib.h2_ipa_finish(sess, 0, None) == 0, _err()
                state["open"] = False
        return after

    def ipa_begin(poly):
        def make(e):
            sess, state = _u64(MARK), {"open": True}
            args = {"bases_handle": prm._h_g, "k": _u32(K)}
            args.update({"p_prime_poly": E.poly(_scal(3))._h} if poly else {"p_prime": e.enc(_scal(3), S)})
            args.update({"x3": e.enc(fe(6), S), "repr": e.repr, "session": ctypes.byref(sess)})
            return Row(lib.h2_ipa_begin_poly if poly else lib.h2_ipa_begin, args, [sess], lambda: finish(sess, state, 0),
                       ["x3"] if poly else ["p_prime", "x3"], after=lambda rc: rc == 0 and abort(sess, state)(rc))
        return make

    def ipa_round(affine):
        def make(e):
            sess, state = open_session()
            name = "out_lr_xy" if affine else "out_lr_xyz"
            out, res = host_out(128 if affine else 192, B, e, not affine)
            fn = lib.h2_ipa_round_affine if affine else lib.h2_ipa_round
            return Row(fn, {"session": sess, "z": e.enc(fe(3), S), "l_rand": e.enc(fe(5), S), "r_rand": e.enc(fe(9), S), "repr": e.repr,
                            name: out}, [out], res, ["z", "l_rand", "r_rand", name], after=abort(sess, state))
        return make

    def ipa_fold(e):
        sess, state = open_session()
        lr = np.zeros(192, dtype=np.uint8)
        assert lib.h2_ipa_round(sess, _c(fe(3)), _c(fe(5)), _c(fe(9)), 0, _c(lr)) == 0, _err()
        u = 11
        return Row(lib.h2_ipa_fold, dict(session=sess, u=e.enc(fe(u), S), u_inv=e.enc(fe(pow(u, -1, pasta.FIELDS[S])), S), repr=e.repr), [],
                   lambda: finish(sess, state, 1), ["u", "u_inv"], after=abort(sess, state))

    def ipa_finish(e):
        sess, state = open_session(K)
        out = _mark(64)

        def res():
            state["open"] = False
            return e.dec(out, S).tobytes()

        def after(rc):
            state["open"] &= rc != 0
            abort(sess, state)(rc)
        return Row(lib.h2_ipa_finish, dict(session=sess, repr=e.repr, out_c_b=out), [out], res, [], [dict(out_c_b=None)], after=after)

    def polys_commit(affine):
        def make(e):
            name = "out_xy" if affine else "out_xyz"
            out, res = host_out(2 * (64 if affine else 96), B, e, not affine)
            fn = lib.h2_msm_registered_polys_affine if affine else lib.h2_msm_registered_polys
            return Row(fn, {"bases_handle": prm._h_g, "polys": hs([E.poly(_scal(4)), E.poly(_scal(5))]), "batch": _sz(2), "n": _sz(N),
                            "extra_scalars": e.enc(_fes([7, 8]), S), "repr": e.repr, name: out}, [out], res, [name], [dict(extra_scalars=None)])
        return make

    # ---- EC-FFT, hash_to_curve, Params::new, codec ------------------------------------------------------------------------
    def ec_fft(e):
        io = e.enc(jac, B).reshape(-1).copy()
        return Row(lib.h2_ec_fft, dict(curve=VESTA, points_xyz=io, omega=e.enc(fe(pasta.omega_for_k(S, K)), S), log_n=_u32(K),
                                       scale=e.enc(fe(3), S), repr=e.repr), [io], lambda: _affine(e.dec(io, B).tobytes()), ["points_xyz", "omega"],
                   [dict(scale=None)])

    def params_lagrange(e):
        out, res = host_out(N * 64, B, e)
        return Row(lib.h2_params_lagrange, dict(curve=VESTA, g_xy=e.enc(pts, B), k=_u32(K), omega_inv=e.enc(fe(pasta.inv(pasta.omega_for_k(S, K),
                                                                                                                       pasta.FIELDS[S])), S),
                                                minv=e.enc(fe(pasta.inv(N, pasta.FIELDS[S])), S), repr=e.repr, out_g_lagrange_xy=out), [out], res,
                   ["g_xy", "omega_inv", "minv", "out_g_lagrange_xy"])

    def hash_to_curve(e):
        out, res = host_out(N * 64, B, e)
        msgs = np.arange(N * 8, dtype=np.uint8)
        return Row(lib.h2_hash_to_curve, dict(curve=VESTA, domain_prefix=b"repr-args", messages=msgs, msg_len=_sz(8), n=_sz(N), repr=e.repr,
                                              out_xy=out), [out], res, ["out_xy"])

    def params_new(e):
        outs = [_mark(N * 64), _mark(N * 64), _mark(64), _mark(64)]
        names = ["out_g_xy", "out_g_lagrange_xy", "out_w_xy", "out_u_xy"]
        return Row(lib.h2_params_new, {"curve": VESTA, "k": _u32(K), "repr": e.repr, **dict(zip(names, outs))}, outs,
                   lambda: b"".join(e.dec(o, B).tobytes() for o in outs), names)

    def batch_normalize(e):
        out, res = host_out(N * 64, B, e)
        return Row(lib.h2_batch_normalize, dict(curve=VESTA, points_xyz=e.enc(jac, B), n=_sz(N), repr=e.repr, out_xy=out), [out], res,
                   ["points_xyz", "out_xy"])

    def compress(e):
        out = _mark(N * 32)                                                          # the wire format: not in repr
        return Row(lib.h2_points_compress, dict(curve=VESTA, points_xy=e.enc(pts, B), n=_sz(N), repr=e.repr, out_bytes=out), [out],
                   lambda: out.tobytes(), ["points_xy", "out_bytes"])

    def decompress(e):
        enc = np.zeros(N * 32, dtype=np.uint8)
        assert lib.h2_points_compress(VESTA, _c(pts), _sz(N), 0, _c(enc)) == 0, _err()
        out, res = host_out(N * 64, B, e)
        return Row(lib.h2_points_decompress, dict(curve=VESTA, bytes=enc, n=_sz(N), repr=e.repr, out_xy=out), [out], res, ["bytes", "out_xy"])

    # ---- NTT --------------------------------------------------------------------------------------------------------------
    def ntt(e):
        a = e.enc(_scal(6), S).reshape(-1).copy()
        return Row(lib.h2_ntt, dict(field=FP, a=a, omega=e.enc(fe(pasta.omega_for_k(S, K)), S), log_n=_u32(K), repr=e.repr), [a],
                   lambda: e.dec(a, S).tobytes(), ["a", "omega"])

    def intt_scaled(e):
        a = e.enc(_scal(6), S).reshape(-1).copy()
        return Row(lib.h2_intt_scaled, dict(field=FP, a=a, omega_inv=e.enc(fe(7), S), divisor=e.enc(fe(5), S), log_n=_u32(K), repr=e.repr), [a],
                   lambda: e.dec(a, S).tobytes(), ["a", "omega_inv", "divisor"])

    def coeff_to_extended(e):
        out, res = host_out(N * 32, S, e)
        return Row(lib.h2_coeff_to_extended, dict(field=FP, a=e.enc(_scal(6, N // 2), S), k=_u32(K - 1), ext_k=_u32(K), zeta=e.enc(fe(5), S),
                                                  ext_omega=e.enc(fe(7), S), out=out, repr=e.repr), [out], res, ["a", "zeta", "ext_omega", "out"])

    def extended_to_coeff(e):
        out, res = host_out(N // 2 * 32, S, e)
        return Row(lib.h2_extended_to_coeff, dict(field=FP, a=e.enc(_scal(6), S), ext_k=_u32(K), ext_omega_inv=e.enc(fe(7), S),
                                                  ext_divisor=e.enc(fe(3), S), zeta=e.enc(fe(5), S), out_len=_sz(N // 2), out=out, repr=e.repr),
                   [out], res, ["a", "ext_omega_inv", "ext_divisor", "zeta", "out"])

    def ntt_dev(e):
        d_in, d_out = dev(MONT.enc(_scal(6), S)), dev(_mark(N * 32))

        def res():
            torch.cuda.synchronize()
            return MONT.dec(d_out.cpu().numpy(), S).tobytes()
        return Row(lib.h2_ntt_dev, dict(field=FP, d_in=d_in, d_out=d_out, omega=e.enc(fe(7), S), omega_repr=e.repr, log_n=_u32(K), stream=E.stream),
                   [d_out], res, ["omega"], repr_arg="omega_repr")

    # ---- resident polynomials ---------------------------------------------------------------------------------------------
    def poly_row(fn, args, outs, needs, optional=()):
        return Row(fn, args, outs, lambda: down(outs), needs, optional)

    def upload(e):
        p = E.poly(_scal(7))
        return poly_row(lib.h2_poly_upload, dict(poly=p._h, src=e.enc(_scal(8), S), len=_sz(N), repr=e.repr), [p], ["src"])

    def download(e):
        out, res = host_out(N * 32, S, e)
        return Row(lib.h2_poly_download, dict(poly=E.poly(_scal(8))._h, dst=out, len=_sz(N), repr=e.repr), [out], res, ["dst"])

    def add_at(e):
        p = E.poly(_scal(7))
        return poly_row(lib.h2_poly_add_at, dict(poly=p._h, index=_sz(1), delta=e.enc(fe(5), S), repr=e.repr), [p], ["delta"])

    def lagrange_to_coeff(e):
        d = E.poly(_scal(7))
        return poly_row(lib.h2_poly_lagrange_to_coeff, dict(dst=d._h, src=E.poly(_scal(8))._h, k=_u32(K), omega_inv=e.enc(fe(7), S),
                                                            divisor=e.enc(fe(5), S), repr=e.repr), [d], ["omega_inv", "divisor"])

    def poly_coeff_to_extended(e):
        d = E.poly(_scal(7))
        return poly_row(lib.h2_poly_coeff_to_extended, dict(dst=d._h, src=E.poly(_scal(8))._h, k=_u32(K - 1), ext_k=_u32(K), zeta=e.enc(fe(5), S),
                                                            ext_omega=e.enc(fe(7), S), repr=e.repr), [d], ["zeta", "ext_omega"])

    def poly_extended_to_coeff(e):
        d = E.poly(_scal(7))
        return poly_row(lib.h2_poly_extended_to_coeff, dict(dst=d._h, src=E.poly(_scal(8))._h, ext_k=_u32(K), ext_omega_inv=e.enc(fe(7), S),
                                                            ext_divisor=e.enc(fe(3), S), zeta=e.enc(fe(5), S), out_len=_sz(N // 2), repr=e.repr),
                        [d], ["ext_omega_inv", "ext_divisor", "zeta"])

    def poly_eval(e):
        out, res = host_out(2 * 32, S, e)
        return Row(lib.h2_poly_eval, dict(polys=hs([E.poly(_scal(9)), E.poly(_scal(10))]), batch=_sz(2), n=_sz(N), points=e.enc(_fes([3, 5]), S),
                                          repr=e.repr, out=out), [out], res, ["points", "out"], [dict(n=_sz(0), points=None)])

    def inner_product(e):
        out, res = host_out(2 * 32, S, e)
        return Row(lib.h2_poly_inner_product, dict(a=hs([E.poly(_scal(9)), E.poly(_scal(10))]), b=hs([E.poly(_scal(11)), E.poly(_scal(12))]),
                                                   batch=_sz(2), n=_sz(N), repr=e.repr, out=out), [out], res, ["out"])

    def kate(e):
        d = [E.poly(_scal(7)), E.poly(_scal(8))]
        return poly_row(lib.h2_poly_kate_division, dict(dst=hs(d), src=hs([E.poly(_scal(9)), E.poly(_scal(10))]), batch=_sz(2), n=_sz(N),
                                                        points=e.enc(_fes([3, 5]), S), repr=e.repr), d, ["points"], [dict(n=_sz(1), points=None)])

    def eval_ast(e):
        d = E.poly(_scal(7))
        code = np.array([[0, 0, 0, 0], [2, 0, 0, 0], [3, 0, 0, 0], [1, 1, 0, 0], [4, 0, 0, 0]], dtype=np.uint32)   # (p0 + LINEAR c0) * c1
        plain = np.array([[0, 0, 0, 0], [1, 1, 0, 0], [4, 0, 0, 0]], dtype=np.uint32)                               # p0 * c1: no LINEAR
        return poly_row(lib.h2_poly_eval_ast, dict(out=d._h, polys=hs([E.poly(_scal(9))]), n_polys=_sz(1), log_n=_u32(K), code=code,
                                                   n_code=_sz(len(code)), consts=e.enc(_fes([3, 5]), S), n_consts=_sz(2), omega=e.enc(fe(7), S),
                                                   lin_base=e.enc(fe(11), S), repr=e.repr), [d], ["consts", "omega", "lin_base"],
                        [dict(omega=None, lin_base=None, code=plain, n_code=_sz(len(plain)))])

    def running_product(e):
        d = E.poly(_scal(7))
        return poly_row(lib.h2_poly_running_product, dict(dst=d._h, src=E.poly(_scal(9))._h, n=_sz(N), init=e.enc(fe(5), S), repr=e.repr), [d],
                        ["init"], [dict(n=_sz(0), init=None)])

    def divide_by_vanishing(e):
        p = E.poly(_scal(7))
        return poly_row(lib.h2_poly_divide_by_vanishing, dict(poly=p._h, ext_k=_u32(K), t_evals=e.enc(_fes([3, 5]), S), t_len=_u32(2),
                                                              repr=e.repr), [p], ["t_evals"])

    def lookup_permuted(e):
        table = _scal(13)
        inp = table.copy()
        inp[:N - 2] = table[:N - 2][::-1]                                            # every usable input row occurs in the table
        o = [E.poly(_scal(7)), E.poly(_scal(8))]
        return poly_row(lib.h2_poly_lookup_permuted, dict(out_inputs=hs(o[:1]), out_tables=hs(o[1:]), count=_sz(1), inputs=hs([E.poly(inp)]),
                                                          tables=hs([E.poly(table)]), k=_u32(K), blinding=e.enc(_fes([3, 5, 7, 9]), S),
                                                          blinding_factors=_u32(1), repr=e.repr), o, ["blinding"], [dict(count=_sz(0), blinding=None)])

    def compute_s(e):
        d = E.poly(_scal(7))
        return poly_row(lib.h2_poly_compute_s, dict(dst=d._h, u=e.enc(_fes([3, 5, 7, 9]), S), k=_u32(K), init=e.enc(fe(11), S), accumulate=1,
                                                    repr=e.repr), [d], ["u", "init"])

    def scale_add(e):
        d = E.poly(_scal(7))
        return poly_row(lib.h2_poly_scale_add, dict(dst=d._h, a=e.enc(fe(3), S), src=E.poly(_scal(9))._h, b=e.enc(fe(5), S), n=_sz(N), repr=e.repr),
                        [d], ["a", "b"], [dict(b=None, src=_u64(0))])

    ident = np.ascontiguousarray(np.stack(np.meshgrid(np.arange(2), np.arange(N), indexing="ij"), axis=-1).astype(np.uint32))

    def sigma(e):
        d = [E.poly(_scal(7)), E.poly(_scal(8))]
        return poly_row(lib.h2_poly_permutation_sigma, dict(dst=hs(d), cols=_sz(2), k=_u32(K), mapping=ident, omega=e.enc(fe(7), S),
                                                            delta=e.enc(fe(5), S), repr=e.repr), d, ["omega", "delta"],
                        [dict(cols=_sz(0), omega=None, delta=None)])

    def sigma_copies(e):
        d = [E.poly(_scal(7)), E.poly(_scal(8))]
        copies = np.array([[0, 1, 1, 2]], dtype=np.uint32)
        return poly_row(lib.h2_poly_permutation_sigma_copies, dict(dst=hs(d), cols=_sz(2), k=_u32(K), copies=copies, m=_sz(1),
                                                                   omega=e.enc(fe(7), S), delta=e.enc(fe(5), S), repr=e.repr), d, ["omega", "delta"],
                        [dict(cols=_sz(0), omega=None, delta=None)])

    def perm_product(e):
        z = [E.poly(_scal(7)), E.poly(_scal(8))]
        return poly_row(lib.h2_poly_permutation_product, dict(z_out=hs(z), proofs=_sz(1), columns=hs([E.poly(_scal(9)), E.poly(_scal(10))]),
                                                              sigmas=hs([E.poly(_scal(11)), E.poly(_scal(12))]), cols=_sz(2), chunk_len=_u32(1),
                                                              k=_u32(K), beta=e.enc(fe(3), S), gamma=e.enc(fe(5), S), omega=e.enc(fe(7), S),
                                                              delta=e.enc(fe(9), S), blinding=e.enc(_fes([13, 15]), S), blinding_factors=_u32(1),
                                                              repr=e.repr), z, ["beta", "gamma", "omega", "delta", "blinding"],
                        [dict(blinding=None, blinding_factors=_u32(0))] +
                        [{**empty, **dict.fromkeys(["beta", "gamma", "omega", "delta", "blinding"])} for empty in (dict(proofs=_sz(0)), dict(cols=_sz(0)))])

    def lookup_product(e):
        z = [E.poly(_scal(7)), E.poly(_scal(8))]
        p = [E.poly(_scal(9 + j)) for j in range(4)]
        return poly_row(lib.h2_poly_lookup_product, dict(z_out=hs(z), count=_sz(2), inputs=hs(p[0:2]), tables=hs(p[2:4]), permuted_inputs=hs(p[1:3]),
                                                         permuted_tables=hs([p[3], p[0]]), k=_u32(K), beta=e.enc(fe(3), S), gamma=e.enc(fe(5), S),
                                                         blinding=e.enc(_fes([13, 15]), S), blinding_factors=_u32(1), repr=e.repr), z,
                        ["beta", "gamma", "blinding"],
                        [dict(blinding=None, blinding_factors=_u32(0)), dict(count=_sz(0), beta=None, gamma=None, blinding=None)])

    return {
        "h2_msm": msm, "h2_msm_dev": msm_dev, "h2_bases_register": register(False), "h2_bases_register_ex": register(True),
        "h2_msm_registered": msm_registered, "h2_msm_registered_batch": batch(False), "h2_msm_registered_batch_affine": batch(True),
        "h2_point_sum": point_sum, "h2_msm_multi_gpu": msm_multi_gpu, "h2_multi_bases_register": multi_register,
        "h2_msm_multi_registered": multi_registered, "h2_ipa_begin": ipa_begin(False), "h2_ipa_begin_poly": ipa_begin(True),
        "h2_ipa_round": ipa_round(False), "h2_ipa_round_affine": ipa_round(True), "h2_ipa_fold": ipa_fold, "h2_ipa_finish": ipa_finish,
        "h2_msm_registered_polys": polys_commit(False), "h2_msm_registered_polys_affine": polys_commit(True),
        "h2_ec_fft": ec_fft, "h2_params_lagrange": params_lagrange, "h2_hash_to_curve": hash_to_curve, "h2_params_new": params_new,
        "h2_batch_normalize": batch_normalize, "h2_points_compress": compress, "h2_points_decompress": decompress,
        "h2_ntt": ntt, "h2_intt_scaled": intt_scaled, "h2_coeff_to_extended": coeff_to_extended, "h2_extended_to_coeff": extended_to_coeff,
        "h2_ntt_dev": ntt_dev, "h2_poly_upload": upload, "h2_poly_download": download, "h2_poly_add_at": add_at,
        "h2_poly_lagrange_to_coeff": lagrange_to_coeff, "h2_poly_coeff_to_extended": poly_coeff_to_extended,
        "h2_poly_extended_to_coeff": poly_extended_to_coeff, "h2_poly_eval": poly_eval, "h2_poly_inner_product": inner_product,
        "h2_poly_kate_division": kate, "h2_poly_eval_ast": eval_ast, "h2_poly_running_product": running_product,
        "h2_poly_divide_by_vanishing": divide_by_vanishing, "h2_poly_lookup_permuted": lookup_permuted, "h2_poly_compute_s": compute_s,
        "h2_poly_scale_add": scale_add, "h2_poly_permutation_sigma": sigma, "h2_poly_permutation_sigma_copies": sigma_copies,
        "h2_poly_permutation_product": perm_product, "h2_poly_lookup_product": lookup_product,
    }


ENTRY_POINTS = [
    "h2_msm", "h2_msm_dev", "h2_bases_register", "h2_bases_register_ex", "h2_msm_registered", "h2_msm_registered_batch",
    "h2_msm_registered_batch_affine", "h2_point_sum", "h2_msm_multi_gpu", "h2_multi_bases_register", "h2_msm_multi_registered",
    "h2_ipa_begin", "h2_ipa_begin_poly", "h2_ipa_round", "h2_ipa_round_affine", "h2_ipa_fold", "h2_ipa_finish", "h2_msm_registered_polys",
    "h2_msm_registered_polys_affine", "h2_ec_fft", "h2_params_lagrange", "h2_hash_to_curve", "h2_params_new", "h2_batch_normalize",
    "h2_points_compress", "h2_points_decompress", "h2_ntt", "h2_intt_scaled", "h2_coeff_to_extended", "h2_extended_to_coeff", "h2_ntt_dev",
    "h2_poly_upload", "h2_poly_download", "h2_poly_add_at", "h2_poly_lagrange_to_coeff", "h2_poly_coeff_to_extended",
    "h2_poly_extended_to_coeff", "h2_poly_eval", "h2_poly_inner_product", "h2_poly_kate_division", "h2_poly_eval_ast",
    "h2_poly_running_product", "h2_poly_divide_by_vanishing", "h2_poly_lookup_permuted", "h2_poly_compute_s", "h2_poly_scale_add",
    "h2_poly_permutation_sigma", "h2_poly_permutation_sigma_copies", "h2_poly_permutation_product", "h2_poly_lookup_product",
]


def _snapshot(torch, outs):
    torch.cuda.synchronize()
    snap = []
    for o in outs:
        if isinstance(o, ctypes.c_uint64):
            snap.append(o.value)
        elif isinstance(o, np.ndarray):
            snap.append(o.tobytes())
        elif isinstance(o, torch.Tensor):
            snap.append(o.cpu().numpy().tobytes())
        else:
            snap.append(o.download().tobytes())
    return snap


@pytest.fixture(scope="module")
def env():
    import halo2_b200 as eng
    from halo2_b200 import lib as L
    lib = L.init()
    pts = cref.gen_points("vesta", SEED + 100, N + 2)
    prm = eng.Params("vesta", K, pts[:N], eng.lagrange_generators("vesta", K, pts[:N]), pts[N:N + 1], u=pts[N + 1:])
    E = Env(lib, prm)
    try:
        yield E, _rows(E)
    finally:
        E.close()
        prm.close()


def _fails_cleanly(E, row, expect, **over):
    """row.call(**over) fails with `expect`, launches nothing and changes none of the row's outputs; '' when it does."""
    before = _snapshot(E.torch, row.outs)
    launches = E.lib.h2_launch_count()
    rc = row.call(**over)
    msg = _err() if rc else ""
    launched = E.lib.h2_launch_count() - launches
    changed = _snapshot(E.torch, row.outs) != before
    if row.after:
        row.after(rc)
    return "" if rc and msg == expect and not launched and not changed else f"rc {rc}, {launched} launches, changed {changed}: {msg!r}"


def _succeeds(E, row, **over):
    rc = row.call(**over)
    msg = _err() if rc else ""
    if row.after:
        row.after(rc)
    E.torch.cuda.synchronize()
    return msg


def test_every_entry_point_with_a_repr_has_a_row(env):
    E, rows = env
    assert sorted(rows) == sorted(ENTRY_POINTS) and len(ENTRY_POINTS) == 50


@pytest.mark.parametrize("name", ENTRY_POINTS)
def test_unknown_repr_fails_before_any_launch(env, name):
    E, rows = env
    try:
        for bad in (2, -1):
            row = rows[name](CANON)
            assert not (why := _fails_cleanly(E, row, f"{name}: unknown repr", **{row.repr_arg: bad})), (name, bad, why)
        assert not (why := _succeeds(E, rows[name](CANON))), (name, why)
    finally:
        E.close()


@pytest.mark.parametrize("name", ENTRY_POINTS)
def test_null_elements(env, name):
    E, rows = env
    try:
        for arg in rows[name](CANON).needs:
            row = rows[name](CANON)
            assert not (why := _fails_cleanly(E, row, f"{name}: null {arg}", **{arg: None})), (name, arg, why)
        for over in rows[name](CANON).optional:
            assert not (why := _succeeds(E, rows[name](CANON), **over)), (name, over, why)
    finally:
        E.close()


def test_ipa_finish_aborts_whatever_the_repr(env):
    E, rows = env
    for bad in (2, -1):
        assert not (why := _succeeds(E, rows["h2_ipa_finish"](CANON), repr=bad, out_c_b=None)), (bad, why)


@pytest.mark.parametrize("name", ENTRY_POINTS)
def test_both_encodings_agree(env, name):
    E, rows = env
    got = []
    try:
        for e in (CANON, MONT):
            row = rows[name](e)
            rc = row.call()
            assert rc == 0, (name, e.repr, _err())
            E.torch.cuda.synchronize()
            got.append(row.result())
            if row.after:
                row.after(rc)
    finally:
        E.close()
    assert got[0] == got[1], name
