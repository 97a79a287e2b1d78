"""TEST-ONLY stand-in for the CUDA library's ctypes handle, so that the HOST LOGIC of the package (the verifier's mirror of
poly/commitment/msm.rs and verifier.rs, the prover's phases, key generation: the order of calls, what goes to which entry
point) runs in the `-m "not gpu"` suite.  It implements the C-ABI entry points that logic touches, with the ABI's own calling
convention (ctypes values, pointers and out-parameters exactly as halo2_b200/lib.py passes them): the kernels run as the device
bodies on the host emulation (tests/kernel_emul), the transforms and group operations through the oracle.  Each call that a
test may count is logged in `calls`.  It is never importable from the package: a test installs it with `installed()` and
removes it again; the product has no CPU fallback."""
from __future__ import annotations

import contextlib
import ctypes

import numpy as np

from oracle import cref, pasta
from tests.kernel_emul import build as emul_build

_CURVES = {0: "pallas", 1: "vesta"}
_FIELDS = {0: "fp", 1: "fq"}
KEYGEN_CHUNK = 1 << 22                                             # rows per launch in capi_poly.cu (H2_KEYGEN_CHUNK)
NONE = 0xFFFFFFFF                                                  # emu_lookup_permuted's status when no lookup misses


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


def emu_assembly(emu, copies, cols: int, k: int):
    """The copy-cycle bodies on the host emulation: (rc, mapping (cols, 2^k, 2), first-bad code, Borůvka rounds, |F|)."""
    cp = np.ascontiguousarray(np.asarray(copies, dtype=np.uint32).reshape(-1, 4))
    out = np.zeros((cols, 1 << k, 2), dtype=np.uint32)
    bad, rounds, forest = ctypes.c_ulonglong(), ctypes.c_uint32(), ctypes.c_uint32()
    rc = emu.emu_assembly(cp.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint64(cp.shape[0]), ctypes.c_uint32(cols), ctypes.c_uint32(k),
                          out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(bad), ctypes.byref(rounds), ctypes.byref(forest))
    return rc, out, bad.value, rounds.value, forest.value


def _jac_bytes(xy: np.ndarray) -> np.ndarray:
    out = np.zeros(96, dtype=np.uint8)
    if xy.any():
        out[:64] = xy
        out[64] = 1
    return out


class FakeLib:
    def __init__(self):
        self.emu = ctypes.CDLL(emul_build.build())
        self.emu.emu_lookup_permuted.restype = ctypes.c_uint32
        self.polys, self.bases, self.next = {}, {}, 1
        self.err = b""
        self.calls = []
        self.shared, self.share_calls, self.freed = set(), [], []       # h2_poly_share's handles, each call's, every h2_poly_free's

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
        self.freed.append(_v(h))
        self.shared.discard(_v(h))
        self.polys.pop(_v(h), None)
        return 0

    def h2_poly_share(self, polys, n):
        """The library's all-or-nothing rule: the calling context's or already shared handles only."""
        hs = [int(x) for x in polys[:_v(n)]]
        self.share_calls.append(hs)
        if any(h not in self.polys for h in hs):
            return self._fail("h2_poly_share: unknown polynomial handle")
        self.shared.update(hs)
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
        if _v(batch) > 64:
            return self._fail("h2_msm_registered_polys: batch > 64")
        _wr(out, self._registered(handle, polys, batch, n, extra, False))
        return 0

    def h2_msm_registered_polys_affine(self, handle, polys, batch, n, extra, repr_, out):
        self._log("h2_msm_registered_polys_affine")
        if _v(batch) > 64:
            return self._fail("h2_msm_registered_polys: batch > 64")
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

    # ---- the prover phases' batched calls (the device bodies on the host emulation, after the library's checks the host
    # mirror can reach) ----
    def _transform_batch(self, who, mode, dst, src, count, in_log, log_n, omega, zeta, divisor):
        self._log(who)
        count = _v(count)
        if count == 0:
            return 0
        d, s = [int(dst[i]) for i in range(count)], [int(src[i]) for i in range(count)]
        c = clash(args("dst", d, True) + args("src", s, False), in_place=("dst", "src"))
        if c:
            return self._fail(f"{who}: {c}")
        f = self.polys[s[0]][0]
        in_log, log_n = _v(in_log), _v(log_n)
        stack = np.ascontiguousarray(np.stack([self.polys[h][1][:1 << in_log] for h in s]))
        out = np.zeros((count, 1 << log_n, 32), dtype=np.uint8)
        self.emu.emu_ntt_batch(cref.FIELD_ID[f], mode, cref._p(stack), ctypes.c_uint64(count), in_log, log_n, cref._p(_rd(omega, 32)),
                               cref._p(_rd(zeta, 32)) if zeta is not None else None, cref._p(_rd(divisor, 32)) if divisor is not None else None,
                               cref._p(out), ctypes.c_uint64(0), 0, 64)
        for i, h in enumerate(d):
            self.polys[h][1][:1 << log_n] = out[i]
        return 0

    def h2_poly_lagrange_to_coeff_batch(self, dst, src, count, k, omega_inv, divisor, repr_):
        return self._transform_batch("h2_poly_lagrange_to_coeff_batch", 1, dst, src, count, k, k, omega_inv, None, divisor)

    def h2_poly_coeff_to_extended_batch(self, dst, src, count, k, ext_k, zeta, ext_omega, repr_):
        return self._transform_batch("h2_poly_coeff_to_extended_batch", 2, dst, src, count, k, ext_k, ext_omega, zeta, None)

    def h2_poly_set_rows(self, polys, count, start, rows, values, repr_):
        self._log("h2_poly_set_rows")
        count, start, rows = _v(count), _v(start), _v(rows)
        if count == 0 or rows == 0:
            return 0
        hs = [int(polys[i]) for i in range(count)]
        short = [i for i, h in enumerate(hs) if start + rows > self.polys[h][1].shape[0]]
        if short:
            return self._fail(f"h2_poly_set_rows: polys[{short[0]}]: a polynomial holds fewer than start + rows elements")
        c = clash(args("polys", hs, True))
        if c:
            return self._fail(f"h2_poly_set_rows: {c}")
        vals = _rd(values, 32 * count * rows).reshape(count, rows, 32)
        for i, h in enumerate(hs):
            self.polys[h][1][start:start + rows] = vals[i]
        return 0

    def h2_poly_lookup_permuted(self, out_inputs, out_tables, count, inputs, tables, k, blinding, bf, repr_):
        self._log("h2_poly_lookup_permuted")
        count, k, bf = _v(count), _v(k), _v(bf)
        n, rows = 1 << k, bf + 1
        outs = [int(out_inputs[b]) for b in range(count)] + [int(out_tables[b]) for b in range(count)]
        ins = [int(inputs[b]) for b in range(count)] + [int(tables[b]) for b in range(count)]
        c = clash(args("out_inputs", outs[:count], True) + args("out_tables", outs[count:], True) +
                  args("inputs", ins[:count], False) + args("tables", ins[count:], False))
        if c:
            return self._fail(f"h2_poly_lookup_permuted: {c}")
        if count == 0:
            return 0
        f = self.polys[ins[0]][0]
        col = lambda hs: np.ascontiguousarray(np.concatenate([self.polys[h][1][:n] for h in hs]))  # noqa: E731
        oa, ot = col(outs[:count]), col(outs[count:])
        bl = _rd(blinding, 32 * count * 2 * rows)
        rc = self.emu.emu_lookup_permuted(cref.FIELD_ID[f], cref._p(col(ins[:count])), cref._p(col(ins[count:])), ctypes.c_uint32(count), ctypes.c_size_t(n),
                                          ctypes.c_size_t(n - rows), cref._p(bl), ctypes.c_size_t(rows), cref._p(oa), cref._p(ot))
        if rc != NONE:
            return self._fail(f"h2_poly_lookup_permuted: lookup {rc}: an input value does not occur in the table")
        for b in range(count):
            self.polys[outs[b]][1][:n] = oa[b * n:(b + 1) * n]
            self.polys[outs[count + b]][1][:n] = ot[b * n:(b + 1) * n]
        return 0

    def h2_poly_permutation_product(self, z_out, proofs, columns, sigmas, cols, chunk_len, k, beta, gamma, omega, delta, blinding, bf, repr_):
        self._log("h2_poly_permutation_product")
        proofs, cols, chunk_len, k, bf = _v(proofs), _v(cols), _v(chunk_len), _v(k), _v(bf)
        n, sets = 1 << k, -(-cols // chunk_len)
        col = lambda h: self.polys[int(h)][1][:n]                  # noqa: E731
        f = self.polys[int(sigmas[0])][0]
        data = np.ascontiguousarray(np.concatenate([col(columns[i]) for i in range(proofs * cols)] + [col(sigmas[i]) for i in range(cols)]))
        out = np.zeros((proofs * sets * n, 32), dtype=np.uint8)
        bl = _rd(blinding, 32 * proofs * sets * bf) if bf else None
        self.emu.emu_permutation_product(cref.FIELD_ID[f], cref._p(data), proofs, cols, chunk_len, k, cref._p(_rd(beta, 32)), cref._p(_rd(gamma, 32)),
                                         cref._p(_rd(omega, 32)), cref._p(_rd(delta, 32)), cref._p(bl) if bf else None, bf, cref._p(out))
        for i in range(proofs * sets):
            self.polys[int(z_out[i])][1][:n] = out[i * n:(i + 1) * n]
        return 0

    def h2_poly_lookup_product(self, z_out, count, inputs, tables, permuted_inputs, permuted_tables, k, beta, gamma, blinding, bf, repr_):
        self._log("h2_poly_lookup_product")
        count, k, bf = _v(count), _v(k), _v(bf)
        if count == 0:
            return 0
        n = 1 << k
        col = lambda h: self.polys[int(h)][1][:n]                  # noqa: E731
        f = self.polys[int(inputs[0])][0]
        data = np.ascontiguousarray(np.concatenate([col(arr[b]) for b in range(count) for arr in (inputs, tables, permuted_inputs, permuted_tables)]))
        out = np.zeros((count * n, 32), dtype=np.uint8)
        bl = _rd(blinding, 32 * count * bf) if bf else None
        self.emu.emu_lookup_product(cref.FIELD_ID[f], cref._p(data), count, k, cref._p(_rd(beta, 32)), cref._p(_rd(gamma, 32)),
                                    cref._p(bl) if bf else None, bf, cref._p(out))
        for b in range(count):
            self.polys[int(z_out[b])][1][:n] = out[b * n:(b + 1) * n]
        return 0

    def h2_poly_vanishing_quotient(self, pieces, count, src, k, ext_k, ext_omega_inv, ext_divisor, zeta, t_evals, t_len, repr_):
        who = "h2_poly_vanishing_quotient"
        self._log(who)
        count, src, k, ext_k, t_len = (_v(x) for x in (count, src, k, ext_k, t_len))
        why = self.emu.emu_vanishing_quotient_sizes(k, ext_k, ctypes.c_uint64(count), t_len)
        if why:
            return self._fail(f"{who}: {ctypes.string_at(why).decode()}")
        hs = [int(pieces[i]) for i in range(count)]
        short = [i for i, h in enumerate(hs) if self.polys[h][1].shape[0] < 1 << k]
        if short:
            return self._fail(f"{who}: pieces[{short[0]}]: a polynomial holds fewer than 2^k elements")
        c = clash(args("pieces", hs, True) + [("src", src, False)])
        if c:
            return self._fail(f"{who}: {c}")
        f, a = self.polys[src]
        out = np.zeros((count, 1 << k, 32), dtype=np.uint8)
        rc = self.emu.emu_vanishing_quotient(cref.FIELD_ID[f], cref._p(np.ascontiguousarray(a[:1 << ext_k])), k, ext_k, ctypes.c_uint64(count),
                                             cref._p(_rd(ext_omega_inv, 32)), cref._p(_rd(ext_divisor, 32)), cref._p(_rd(zeta, 32)),
                                             cref._p(_rd(t_evals, 32 * t_len)), t_len, cref._p(out), 0, 64)
        assert rc > 0, rc
        for i, h in enumerate(hs):
            self.polys[h][1][:1 << k] = out[i]
        return 0

    # ---- key generation: the sigma bodies, and the copy-cycle bodies before them, on the host emulation ----
    def h2_poly_permutation_sigma(self, dst, cols, k, mapping, omega, delta, repr_):
        self._log("h2_poly_permutation_sigma")
        cols, k = _v(cols), _v(k)
        if k > 30:
            return self._fail("h2_poly_permutation_sigma: k > 30")
        if cols == 0:
            return 0
        hs = [int(dst[i]) for i in range(cols)]
        unknown = [i for i, h in enumerate(hs) if h not in self.polys]
        if unknown:
            return self._fail(f"h2_poly_permutation_sigma: dst[{unknown[0]}]: unknown polynomial handle")
        c = clash(args("dst", hs, True))
        if c:
            return self._fail(f"h2_poly_permutation_sigma: {c}")
        field = self.polys[hs[0]][0]
        n = 1 << k
        if any(self.polys[h][0] != field or self.polys[h][1].shape[0] < n for h in hs):
            return self._fail("h2_poly_permutation_sigma: a polynomial of another field or shorter than 2^k")
        mp = np.frombuffer(ctypes.string_at(_v(mapping), 8 * cols * n), dtype=np.uint32).copy()
        out = np.zeros((cols * n, 32), dtype=np.uint8)
        rc = self.emu.emu_permutation_sigma(cref.FIELD_ID[field], mp.ctypes.data_as(ctypes.c_void_p), cols, k, cref._p(_rd(omega, 32)),
                                            cref._p(_rd(delta, 32)), ctypes.c_uint64(KEYGEN_CHUNK), cref._p(out))
        if rc:
            return self._fail("h2_poly_permutation_sigma: a mapping entry is outside the permutation's columns or the domain's rows")
        for i, h in enumerate(hs):
            self.polys[h][1][:n] = out[i * n:(i + 1) * n]
        return 0

    def h2_poly_permutation_sigma_copies(self, dst, cols, k, copies, m, omega, delta, repr_):
        self._log("h2_poly_permutation_sigma_copies")
        cols, k, m = _v(cols), _v(k), _v(m)
        if k > 30:
            return self._fail("h2_poly_permutation_sigma_copies: k > 30")
        if cols == 0:
            return 0
        if (cols << k) >= 1 << 32 or m >= 1 << 32:
            return self._fail("h2_poly_permutation_sigma_copies: too many cells or copies")
        hs = [int(dst[i]) for i in range(cols)]
        if any(h not in self.polys for h in hs) or len(set(hs)) != cols:
            return self._fail("h2_poly_permutation_sigma_copies: unknown or repeated polynomial handle")
        field = self.polys[hs[0]][0]
        n = 1 << k
        if any(self.polys[h][0] != field or self.polys[h][1].shape[0] < n for h in hs):
            return self._fail("h2_poly_permutation_sigma_copies: a polynomial of another field or shorter than 2^k")
        cp = np.frombuffer(ctypes.string_at(_v(copies), 16 * m), dtype=np.uint32).reshape(-1, 4) if m else np.zeros((0, 4), np.uint32)
        rc, mapping, bad, _, _ = emu_assembly(self.emu, cp, cols, k)
        if rc:
            return self._fail(f"h2_poly_permutation_sigma_copies: copy {bad >> 1}: a {'row' if bad & 1 else 'column'} is out of range")
        out = np.zeros((cols * n, 32), dtype=np.uint8)
        rc = self.emu.emu_permutation_sigma(cref.FIELD_ID[field], mapping.ctypes.data_as(ctypes.c_void_p), cols, k, cref._p(_rd(omega, 32)),
                                            cref._p(_rd(delta, 32)), ctypes.c_uint64(KEYGEN_CHUNK), cref._p(out))
        assert rc == 0
        for i, h in enumerate(hs):
            self.polys[h][1][:n] = out[i * n:(i + 1) * n]
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
