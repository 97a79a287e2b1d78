"""TEST-ONLY stand-in for the CUDA library's ctypes handle, so that the HOST LOGIC of halo2_b200.verifier (the mirror of
poly/commitment/msm.rs and verifier.rs: term merging, the order of calls, what goes to which entry point) runs in the
`-m "not gpu"` suite.  It implements just the C-ABI entry points that mirror touches, with the ABI's own calling convention
(ctypes values, pointers and out-parameters exactly as halo2_b200/lib.py passes them): the two verifier kernels run as the
device bodies on the host emulation (tests/kernel_emul), the group operations through the oracle.  It is never importable from
the package: a test installs it with `installed()` and removes it again; the product has no CPU fallback."""
from __future__ import annotations

import contextlib
import ctypes

import numpy as np

from oracle import cref, pasta
from tests.kernel_emul import build as emul_build

_CURVES = {0: "pallas", 1: "vesta"}
_FIELDS = {0: "fp", 1: "fq"}


def _rd(p, nbytes: int) -> np.ndarray:
    addr = p.value if hasattr(p, "value") else p
    return np.frombuffer(ctypes.string_at(addr, nbytes), dtype=np.uint8).copy()


def _wr(p, arr: np.ndarray) -> None:
    data = np.ascontiguousarray(arr, dtype=np.uint8).tobytes()
    ctypes.memmove(p.value if hasattr(p, "value") else p, data, len(data))


def _v(x) -> int:
    return int(x.value) if hasattr(x, "value") else int(x)


def args(name: str, handles, out: bool) -> list:
    """The elements of one handle array as clash() takes them."""
    return [(f"{name}[{i}]", int(h), out) for i, h in enumerate(handles)]


def clash(looked_up, in_place=None):
    """The library's aliasing rule (PolyArgs::distinct, capi_core.cu) on (label, handle, is_output) in lookup order: the
    first argument that clashes with an earlier one, as "<a> is also <b>" with the output first, or None.  in_place:
    the (output, input) array names whose elements of one index may be the same polynomial."""
    paired = lambda o, x: in_place is not None and o[0] == in_place[0] + x[0][len(in_place[1]):] and x[0].startswith(in_place[1] + "[")
    seen = {}
    for a in looked_up:
        out, ins = seen.setdefault(a[1], [None, []])
        if a[2] and out:
            return f"{a[0]} is also {out[0]}"
        x = next((x for x in ins if not paired(a, x)), None) if a[2] else None
        if x:
            return f"{a[0]} is also {x[0]}"
        if not a[2] and out and not paired(out, a):
            return f"{out[0]} is also {a[0]}"
        if a[2]:
            seen[a[1]][0] = a
        else:
            ins.append(a)
    return None


def _jac_bytes(xy: np.ndarray) -> np.ndarray:
    out = np.zeros(96, dtype=np.uint8)
    if xy.any():
        out[:64] = xy
        out[64] = 1
    return out


class FakeLib:
    def __init__(self):
        self.emu = ctypes.CDLL(emul_build.build())
        self.polys, self.bases, self.next = {}, {}, 1
        self.err = b""
        self.calls = []

    def _fail(self, msg: str) -> int:
        self.err = msg.encode()
        return 1

    def _log(self, name):
        self.calls.append(name)

    # ---- plumbing ----
    def h2_init(self, device):
        return 0

    def h2_last_error(self):
        return self.err

    def h2_launch_count(self):
        return len(self.calls)

    # ---- base sets ----
    def h2_bases_register_ex(self, curve, bases, n, repr_, window_bits, flags, out_handle):
        h = self.next
        self.next += 1
        self.bases[h] = (_CURVES[_v(curve)], _rd(bases, 64 * _v(n)).reshape(-1, 64))
        out_handle._obj.value = h
        return 0

    def h2_bases_release(self, h):
        self.bases.pop(_v(h), None)
        return 0

    # ---- resident polynomials ----
    def h2_poly_alloc(self, field, length, out_handle):
        h = self.next
        self.next += 1
        self.polys[h] = [_FIELDS[_v(field)], np.zeros((_v(length), 32), dtype=np.uint8)]
        out_handle._obj.value = h
        return 0

    def h2_poly_free(self, h):
        self.polys.pop(_v(h), None)
        return 0

    def h2_poly_upload(self, h, src, length, repr_):
        self.polys[_v(h)][1][:_v(length)] = _rd(src, 32 * _v(length)).reshape(-1, 32)
        return 0

    def h2_poly_download(self, h, dst, length, repr_):
        _wr(dst, self.polys[_v(h)][1][:_v(length)])
        return 0

    def h2_poly_copy(self, dst, dst_off, src, src_off, length):
        d, s, n = self.polys[_v(dst)][1], self.polys[_v(src)][1], _v(length)
        d[_v(dst_off):_v(dst_off) + n] = s[_v(src_off):_v(src_off) + n]
        return 0

    def h2_poly_add_at(self, h, index, delta, repr_):
        f, a = self.polys[_v(h)]
        m = pasta.FIELDS[f]
        i = _v(index)
        cur = int.from_bytes(a[i].tobytes(), "little") + int.from_bytes(_rd(delta, 32).tobytes(), "little")
        a[i] = np.frombuffer((cur % m).to_bytes(32, "little"), dtype=np.uint8)
        return 0

    def h2_poly_compute_s(self, dst, u, k, init, accumulate, repr_):
        self._log("h2_poly_compute_s")
        if _v(dst) not in self.polys:
            return self._fail("h2_poly_compute_s: unknown polynomial handle")
        f, a = self.polys[_v(dst)]
        k = _v(k)
        if k == 0 or a.shape[0] < (1 << k):
            return self._fail("h2_poly_compute_s: bad size")
        ub, ib = _rd(u, 32 * k), _rd(init, 32)
        buf = np.ascontiguousarray(a[:1 << k])
        self.emu.emu_compute_s(cref.FIELD_ID[f], cref._p(ub), k, cref._p(ib), int(accumulate), cref._p(buf))
        a[:1 << k] = buf
        return 0

    def h2_poly_scale_add(self, dst, a, src, b, n, repr_):
        self._log("h2_poly_scale_add")
        n = _v(n)
        if _v(src) and _v(src) == _v(dst):
            return self._fail("h2_poly_scale_add: dst is also src")
        f, d = self.polys[_v(dst)]
        buf = np.ascontiguousarray(d[:n])
        sb = np.ascontiguousarray(self.polys[_v(src)][1][:n]) if _v(src) else None
        self.emu.emu_scale_add(cref.FIELD_ID[f], cref._p(buf), cref._p(_rd(a, 32)), cref._p(sb) if sb is not None else None,
                               cref._p(_rd(b, 32)) if sb is not None else None, ctypes.c_uint64(n))
        d[:n] = buf
        return 0

    # ---- group operations (through the oracle) ----
    def _registered(self, handle, polys, batch, n, extra, affine):
        curve, bases = self.bases[_v(handle)]
        n, batch = _v(n), _v(batch)
        blinds = _rd(extra, 32 * batch).reshape(-1, 32) if extra is not None else None
        out = []
        for i in range(batch):
            sc = self.polys[int(polys[i])][1][:n]
            bs = bases[:n]
            if blinds is not None:
                sc, bs = np.concatenate([sc, blinds[i:i + 1]]), bases[:n + 1]
            xy = cref.best_multiexp(curve, np.ascontiguousarray(sc), np.ascontiguousarray(bs), 2)
            out.append(xy if affine else _jac_bytes(xy))
        return np.stack(out)

    def h2_msm_registered_polys(self, handle, polys, batch, n, extra, repr_, out):
        self._log("h2_msm_registered_polys")
        _wr(out, self._registered(handle, polys, batch, n, extra, False))
        return 0

    def h2_msm_registered_polys_affine(self, handle, polys, batch, n, extra, repr_, out):
        self._log("h2_msm_registered_polys_affine")
        _wr(out, self._registered(handle, polys, batch, n, extra, True))
        return 0

    def h2_msm(self, curve, scalars, bases, n, repr_, out):
        self._log("h2_msm")
        n = _v(n)
        xy = cref.best_multiexp(_CURVES[_v(curve)], _rd(scalars, 32 * n).reshape(-1, 32), _rd(bases, 64 * n).reshape(-1, 64), 2)
        _wr(out, _jac_bytes(xy))
        return 0

    def h2_point_sum(self, curve, points, g, repr_, out):
        self._log("h2_point_sum")
        c = pasta.CURVES[_CURVES[_v(curve)]]
        acc = (0, 1, 0)
        for row in _rd(points, 96 * _v(g)).reshape(-1, 96):
            x, y, z = (int.from_bytes(row[i:i + 32].tobytes(), "little") for i in (0, 32, 64))
            acc = pasta.jac_add(c, acc, (x, y, z))
        _wr(out, _jac_bytes(cref.affines_to_bytes([pasta.to_affine(c, acc)])[0]))
        return 0

    def h2_msm_registered(self, handle, scalars, n, extra, repr_, out):
        self._log("h2_msm_registered")
        curve, bases = self.bases[_v(handle)]
        n = _v(n)
        sc, bs = _rd(scalars, 32 * n).reshape(-1, 32), bases[:n]
        if extra is not None:
            sc, bs = np.concatenate([sc, _rd(extra, 32).reshape(1, 32)]), bases[:n + 1]
        _wr(out, _jac_bytes(cref.best_multiexp(curve, np.ascontiguousarray(sc), np.ascontiguousarray(bs), 2)))
        return 0

    def h2_batch_normalize(self, curve, points, n, repr_, out):
        c = pasta.CURVES[_CURVES[_v(curve)]]
        rows = _rd(points, 96 * _v(n)).reshape(-1, 96)
        pts = [pasta.to_affine(c, tuple(int.from_bytes(row[i:i + 32].tobytes(), "little") for i in (0, 32, 64))) for row in rows]
        _wr(out, cref.affines_to_bytes(pts))
        return 0

    # ---- reductions on resident polynomials ----
    def h2_poly_eval(self, polys, batch, n, points, repr_, out):
        self._log("h2_poly_eval")
        n, batch = _v(n), _v(batch)
        pts = _rd(points, 32 * batch).reshape(-1, 32)
        res = []
        for i in range(batch):
            f, a = self.polys[int(polys[i])]
            res.append(cref.eval_polynomial(f, a[:n], int.from_bytes(pts[i].tobytes(), "little")))
        _wr(out, cref.ints_to_bytes(res))
        return 0

    def h2_poly_kate_division(self, dst, src, batch, n, points, repr_):
        self._log("h2_poly_kate_division")
        n, batch = _v(n), _v(batch)
        pts = _rd(points, 32 * batch).reshape(-1, 32)
        c = clash(args("dst", dst[:batch], True) + args("src", src[:batch], False))
        if c:
            return self._fail(f"h2_poly_kate_division: {c}")
        for i in range(batch):
            f, a = self.polys[int(src[i])]
            q = cref.kate_division(f, a[:n], int.from_bytes(pts[i].tobytes(), "little"))
            d = self.polys[int(dst[i])][1]
            d[:n - 1] = q
            if d.shape[0] >= n:
                d[n - 1] = 0
        return 0

    # ---- transforms (C restatement) and the elementwise programs / scans (the device bodies on the host emulation) ----
    def _fe_int(self, p):
        return int.from_bytes(_rd(p, 32).tobytes(), "little")

    def h2_poly_lagrange_to_coeff(self, dst, src, k, omega_inv, divisor, repr_):
        self._log("h2_poly_lagrange_to_coeff")
        f, a = self.polys[_v(src)]
        n = 1 << _v(k)
        self.polys[_v(dst)][1][:n] = cref.ifft(f, np.ascontiguousarray(a[:n]), self._fe_int(omega_inv), _v(k), self._fe_int(divisor), 2)
        return 0

    def h2_poly_coeff_to_extended(self, dst, src, k, ext_k, zeta, ext_omega, repr_):
        self._log("h2_poly_coeff_to_extended")
        f, a = self.polys[_v(src)]
        self.polys[_v(dst)][1][:1 << _v(ext_k)] = cref.coeff_to_extended(f, np.ascontiguousarray(a[:1 << _v(k)]), _v(k), _v(ext_k), self._fe_int(zeta),
                                                                        self._fe_int(ext_omega), 2)
        return 0

    def h2_poly_extended_to_coeff(self, dst, src, ext_k, ext_omega_inv, ext_divisor, zeta, out_len, repr_):
        self._log("h2_poly_extended_to_coeff")
        f, a = self.polys[_v(src)]
        self.polys[_v(dst)][1][:_v(out_len)] = cref.extended_to_coeff(f, np.ascontiguousarray(a[:1 << _v(ext_k)]), _v(ext_k), self._fe_int(ext_omega_inv),
                                                                     self._fe_int(ext_divisor), self._fe_int(zeta), _v(out_len), 2)
        return 0

    def h2_poly_divide_by_vanishing(self, poly, ext_k, t_evals, t_len, repr_):
        self._log("h2_poly_divide_by_vanishing")
        f, a = self.polys[_v(poly)]
        m = pasta.FIELDS[f]
        t = cref.bytes_to_ints(_rd(t_evals, 32 * _v(t_len)).reshape(-1, 32))
        vals = cref.bytes_to_ints(a[:1 << _v(ext_k)])
        a[:1 << _v(ext_k)] = cref.ints_to_bytes([x * t[i % len(t)] % m for i, x in enumerate(vals)])
        return 0

    def h2_poly_eval_ast(self, out, polys, n_polys, log_n, code, n_code, consts, n_consts, omega, lin_base, repr_):
        self._log("h2_poly_eval_ast")
        n_polys, log_n, n_code, n_consts = _v(n_polys), _v(log_n), _v(n_code), _v(n_consts)
        n = 1 << log_n
        if n_code == 0 or n_code > 1 << 20:
            return self._fail("h2_poly_eval_ast: empty or oversized program")
        prog = np.frombuffer(ctypes.string_at(_v(code), 16 * n_code), dtype=np.uint32).reshape(-1, 4).copy()
        depth = 0                                                 # the library's own validation (capi_poly.cu): operand stack of 24
        for op, arg, _, _ in prog:
            if op in (0, 1, 2):
                depth += 1
            elif op in (3, 4):
                depth -= 1
            if depth > 24 or depth < 1:
                return self._fail("h2_poly_eval_ast: operand stack out of range")
        if depth != 1:
            return self._fail("h2_poly_eval_ast: the program leaves more than one value")
        if self.polys[_v(out)][1].shape[0] < n:
            return self._fail("h2_poly_eval_ast: a polynomial holds fewer than 2^log_n elements")
        short = [i for i in range(n_polys) if self.polys[int(polys[i])][1].shape[0] < n]
        if short:
            return self._fail(f"h2_poly_eval_ast: polys[{short[0]}]: a polynomial holds fewer than 2^log_n elements")
        c = clash([("out", _v(out), True)] + args("polys", polys[:n_polys], False))
        if c:
            return self._fail(f"h2_poly_eval_ast: {c}")
        f = self.polys[_v(out)][0]
        stack = np.ascontiguousarray(np.stack([self.polys[int(polys[i])][1][:n] for i in range(n_polys)])) if n_polys else np.zeros((1, n, 32), dtype=np.uint8)
        cs = _rd(consts, 32 * n_consts) if n_consts else np.zeros(32, dtype=np.uint8)
        res = np.zeros((n, 32), dtype=np.uint8)
        self.emu.emu_ast_eval(cref.FIELD_ID[f], cref._p(stack), n_polys, log_n, prog.ctypes.data_as(ctypes.c_void_p), n_code, cref._p(cs), n_consts,
                              cref._p(_rd(omega, 32)), cref._p(_rd(lin_base, 32)), cref._p(res))
        self.polys[_v(out)][1][:n] = res
        return 0

    def h2_poly_batch_invert(self, poly, n):
        self._log("h2_poly_batch_invert")
        f, a = self.polys[_v(poly)]
        n = _v(n)
        res = np.zeros((n, 32), dtype=np.uint8)
        self.emu.emu_grand_product(cref.FIELD_ID[f], 0, cref._p(np.ascontiguousarray(a[:n])), ctypes.c_uint64(n), None, cref._p(res))
        a[:n] = res
        return 0

    def h2_poly_running_product(self, dst, src, n, init, repr_):
        self._log("h2_poly_running_product")
        if _v(dst) == _v(src):
            return self._fail("h2_poly_running_product: dst is also src")
        f, a = self.polys[_v(src)]
        n = _v(n)
        res = np.zeros((n, 32), dtype=np.uint8)
        self.emu.emu_grand_product(cref.FIELD_ID[f], 1, cref._p(np.ascontiguousarray(a[:n])), ctypes.c_uint64(n), cref._p(_rd(init, 32)), cref._p(res))
        self.polys[_v(dst)][1][:n] = res
        return 0

    def h2_poly_lookup_permute(self, inp, tab, usable, out_in, out_tab):
        self._log("h2_poly_lookup_permute")
        f, a = self.polys[_v(inp)]
        t = self.polys[_v(tab)][1]
        n, u = a.shape[0], _v(usable)
        oa, ot = np.ascontiguousarray(self.polys[_v(out_in)][1][:n]), np.ascontiguousarray(self.polys[_v(out_tab)][1][:n])
        rc = self.emu.emu_lookup_permute(cref.FIELD_ID[f], cref._p(np.ascontiguousarray(a)), cref._p(np.ascontiguousarray(t[:n])), ctypes.c_size_t(n),
                                         ctypes.c_size_t(u), cref._p(oa), cref._p(ot))
        if rc != 0:
            return self._fail("h2_poly_lookup_permute: an input value does not occur in the table")
        self.polys[_v(out_in)][1][:n], self.polys[_v(out_tab)][1][:n] = oa, ot
        return 0

    # ---- the opening's round loop: the reference's own folding loop, one round per call (poly/commitment/prover.rs:100-142) ----
    def h2_ipa_begin_poly(self, bases_handle, k, poly, x3, repr_, out_session):
        f, a = self.polys[_v(poly)]
        return self._ipa_begin(bases_handle, k, cref.bytes_to_ints(a[:1 << _v(k)]), x3, out_session)

    def h2_ipa_begin(self, bases_handle, k, p_prime, x3, repr_, out_session):
        return self._ipa_begin(bases_handle, k, cref.bytes_to_ints(_rd(p_prime, 32 << _v(k)).reshape(-1, 32)), x3, out_session)

    def _ipa_begin(self, bases_handle, k, p_prime, x3, out_session):
        self._log("h2_ipa_begin")
        curve, bases = self.bases[_v(bases_handle)]
        c = pasta.CURVES[curve]
        k = _v(k)
        n = 1 << k
        x = int.from_bytes(_rd(x3, 32).tobytes(), "little")
        b = [1] * n
        for i in range(1, n):
            b[i] = b[i - 1] * x % c.r
        pts = [cref.bytes_to_affine(row) for row in bases[:n + 2]]
        h = self.next
        self.next += 1
        self.sessions = getattr(self, "sessions", {})
        self.sessions[h] = {"c": c, "g": pts[:n], "w": pts[n], "u": pts[n + 1], "p": list(p_prime), "b": b}
        out_session._obj.value = h
        return 0

    def h2_ipa_round_affine(self, session, z, l_rand, r_rand, repr_, out):
        self._log("h2_ipa_round")
        S = self.sessions[_v(session)]
        c, r = S["c"], S["c"].r
        zi, lr, rr = (int.from_bytes(_rd(x, 32).tobytes(), "little") for x in (z, l_rand, r_rand))
        half = len(S["p"]) // 2
        p, b, g = S["p"], S["b"], S["g"]
        l_j = pasta.best_multiexp(c, p[half:] + [pasta.compute_inner_product(r, p[half:], b[:half]) * zi % r, lr], g[:half] + [S["u"], S["w"]])
        r_j = pasta.best_multiexp(c, p[:half] + [pasta.compute_inner_product(r, p[:half], b[half:]) * zi % r, rr], g[half:] + [S["u"], S["w"]])
        _wr(out, cref.affines_to_bytes([pasta.to_affine(c, l_j), pasta.to_affine(c, r_j)]))
        return 0

    def h2_ipa_fold(self, session, u, u_inv, repr_):
        S = self.sessions[_v(session)]
        c, r = S["c"], S["c"].r
        uj, ui = (int.from_bytes(_rd(x, 32).tobytes(), "little") for x in (u, u_inv))
        half = len(S["p"]) // 2
        S["p"] = [(S["p"][i] + S["p"][i + half] * ui) % r for i in range(half)]
        S["b"] = [(S["b"][i] + S["b"][i + half] * uj) % r for i in range(half)]
        S["g"] = pasta.parallel_generator_collapse(c, S["g"], uj)
        return 0

    def h2_ipa_finish(self, session, repr_, out):
        S = self.sessions.pop(_v(session))
        if out is not None:
            _wr(out, cref.ints_to_bytes([S["p"][0], S["b"][0]]))
        return 0

    def h2_params_lagrange(self, curve, g_xy, k, omega_inv, minv, repr_, out):
        k = _v(k)
        gl = cref.params_lagrange(_CURVES[_v(curve)], _rd(g_xy, 64 << k).reshape(-1, 64), k, int.from_bytes(_rd(omega_inv, 32).tobytes(), "little"),
                                  int.from_bytes(_rd(minv, 32).tobytes(), "little"))
        _wr(out, gl)
        return 0

    def h2_params_new(self, curve, k, repr_, out_g, out_gl, out_w, out_u):
        name = _CURVES[_v(curve)]
        c = pasta.CURVES[name]
        k = _v(k)
        g, w, u = pasta.params_generators(c, k)
        gb = cref.affines_to_bytes(g)
        r = c.r
        gl = cref.params_lagrange(name, gb, k, pasta.inv(pasta.omega_for_k(c.scalar, k), r), pow(pasta.inv(2, r), k, r))
        _wr(out_g, gb), _wr(out_gl, gl), _wr(out_w, cref.affines_to_bytes([w])), _wr(out_u, cref.affines_to_bytes([u]))
        return 0

    def h2_points_compress(self, curve, points, n, repr_, out):
        rows = _rd(points, 64 * _v(n)).reshape(-1, 64)
        _wr(out, np.frombuffer(b"".join(pasta.compress(cref.bytes_to_affine(r)) for r in rows), dtype=np.uint8))
        return 0

    def h2_points_decompress(self, curve, data, n, repr_, out):
        self._log("h2_points_decompress")
        c = pasta.CURVES[_CURVES[_v(curve)]]
        rows = _rd(data, 32 * _v(n)).reshape(-1, 32)
        try:
            pts = [pasta.decompress(c, r.tobytes()) for r in rows]
        except Exception as e:
            return self._fail(f"h2_points_decompress: {e}")
        _wr(out, cref.affines_to_bytes(pts))
        return 0


@contextlib.contextmanager
def installed():
    """halo2_b200.lib bound to a FakeLib for the duration of the block (and back to whatever it was afterwards)."""
    from halo2_b200 import lib as L
    saved = (L._lib, L._inited_device)
    fake = FakeLib()
    L._lib, L._inited_device = fake, 0
    try:
        yield fake
    finally:
        L._lib, L._inited_device = saved
