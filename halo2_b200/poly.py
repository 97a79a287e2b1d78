"""Host-side mirror of poly::commitment::Params::{commit, commit_lagrange}
(/root/reference/halo2_proofs/src/poly/commitment.rs:119-150) and
poly::EvaluationDomain::{new, lagrange_to_coeff, coeff_to_extended, extended_to_coeff}
(poly/domain.rs:40-146, :227-255, :303-325) over the C ABI.

The domain constants are derived on the host exactly as domain.rs:40-146 does (they are a few
field elements); the transforms run on the GPU.
"""
from __future__ import annotations

import contextlib
import ctypes
from typing import List, Optional, Sequence

import numpy as np

from . import lib as _l

FIELDS = {
    "fp": 0x40000000000000000000000000000000224698FC094CF91B992D30ED00000001,
    "fq": 0x40000000000000000000000000000000224698FC0994A8DD8C46EB2100000001,
}
S = 32  # two-adicity of both fields
_MSM_BATCH = 64  # the most polynomials one h2_msm_registered_batch* / h2_msm_registered_polys* call takes (csrc/capi_msm.cu)
DIRECT_DEFAULT: Optional[bool] = None  # None: window tables (Params(direct=True) opts into digit-multiples tables; tests flip this)


class Blind:
    """poly/commitment.rs:210-216: newtype over a scalar; default = 1."""

    def __init__(self, value: int = 1):
        self.value = int(value)


def lagrange_generators(curve: str, k: int, g) -> np.ndarray:
    """g -> g_lagrange, poly/commitment.rs:74-101 (h2_params_lagrange: nothing but g goes up and g_lagrange comes back)."""
    m = FIELDS[_l.SCALAR_FIELD[curve]]
    alpha_inv = pow(pow(5, (m - 1) >> S, m), m - 2, m)  # ROOT_OF_UNITY_INV
    for _ in range(k, S):
        alpha_inv = alpha_inv * alpha_inv % m  # commitment.rs:77-80
    minv = pow(pow(2, m - 2, m), k, m)  # TWO_INV^k, :83
    gb = _l.as_u8(g, 64)
    assert gb.shape[0] == 1 << k
    out = np.zeros((1 << k, 64), dtype=np.uint8)
    _l.check(_l.init().h2_params_lagrange(_l.CURVE_ID[curve], _l.ptr(gb), ctypes.c_uint32(k), _l.ptr(_l.fe_bytes(alpha_inv)),
                                          _l.ptr(_l.fe_bytes(minv)), _l.REPR_CANONICAL, _l.ptr(out)))
    return out


def hash_to_curve(curve: str, domain_prefix: str):
    """C::CurveExt::hash_to_curve(domain_prefix) (call sites poly/commitment.rs:52,102; benches/hashtocurve.rs:15,18):
    returns the closure message -> affine point (64 bytes, canonical; identity = zeros).  The closure also takes a LIST of
    equal-length messages and hashes them in one launch -> (n, 64)."""
    dom = domain_prefix.encode()

    def hasher(message):
        single = isinstance(message, (bytes, bytearray))
        msgs = [bytes(message)] if single else [bytes(m) for m in message]
        n = len(msgs)
        ml = len(msgs[0]) if n else 0
        assert all(len(m) == ml for m in msgs), "batched messages must have equal length"
        buf = np.frombuffer(b"".join(msgs), dtype=np.uint8).copy() if n * ml else None
        out = np.zeros((n, 64), dtype=np.uint8)
        _l.check(_l.init().h2_hash_to_curve(_l.CURVE_ID[curve], ctypes.c_char_p(dom), _l.ptr(buf), ctypes.c_size_t(ml), ctypes.c_size_t(n),
                                            _l.REPR_CANONICAL, _l.ptr(out)))
        return out[0] if single else out

    return hasher


def compress_points(points_xy, curve: str) -> np.ndarray:
    """C::to_bytes for a batch (book/src/background/curves.md:203-225): (n, 64) affine -> (n, 32) uint8."""
    p = _l.as_u8(points_xy, 64)
    out = np.zeros((p.shape[0], 32), dtype=np.uint8)
    _l.check(_l.init().h2_points_compress(_l.CURVE_ID[curve], _l.ptr(p), ctypes.c_size_t(p.shape[0]), _l.REPR_CANONICAL, _l.ptr(out)))
    return out


def decompress_points(data, curve: str) -> np.ndarray:
    """C::from_bytes for a batch (curves.md:227-240): (n, 32) uint8 -> (n, 64) affine.  Raises H2Error on an invalid
    encoding (the reference's C::read returns io::Error)."""
    b = _l.as_u8(data, 32)
    out = np.zeros((b.shape[0], 64), dtype=np.uint8)
    _l.check(_l.init().h2_points_decompress(_l.CURVE_ID[curve], _l.ptr(b), ctypes.c_size_t(b.shape[0]), _l.REPR_CANONICAL, _l.ptr(out)))
    return out


class Params:
    """poly/commitment.rs:26-33.  g / g_lagrange / w are uploaded once and stay resident in HBM
    (they are immutable for the life of a Params); commit / commit_lagrange only ship the
    polynomial.  Params.new(curve, k) is Params::new (:38-114) whole -- hash_to_curve generators and
    g_lagrange derived on the device; Params.read (:185-205) / the constructor take existing generators."""

    def __init__(self, curve: str, k: int, g, g_lagrange, w, u=None, precompute: bool = True, window_bits: int = 0,
                 direct: Optional[bool] = None):
        assert k < 32  # commitment.rs:41
        self.curve, self.k, self.n = curve, k, 1 << k
        self.g = _l.as_u8(g, 64)
        self.g_lagrange = _l.as_u8(g_lagrange, 64)
        self.w = _l.as_u8(w, 64)
        self.u = None if u is None else _l.as_u8(u, 64)
        assert self.g.shape[0] == self.n and self.g_lagrange.shape[0] == self.n
        lib = _l.init()
        self._h_g = ctypes.c_uint64(0)
        self._h_gl = ctypes.c_uint64(0)
        cid = _l.CURVE_ID[curve]
        # tmp_bases = g ++ [w]  (:126-127); u rides along at index n + 1 for the IPA rounds (prover.rs:118-119)
        both = np.concatenate([self.g, self.w] + ([] if self.u is None else [self.u]))
        flags = 1 if precompute else 0   # H2_BASES_PRECOMPUTE: window tables, fixed-base MSM
        # H2_BASES_DIRECT: digit-multiples tables (256 KiB per generator) for small sets -- commits and IPA rounds become
        # plain sums of table entries (csrc/fixedbase.cuh).
        if direct is None:
            direct = DIRECT_DEFAULT
        if direct is None:
            direct = False   # no faster than the window table on commits, slower on openings -- opt-in only (DESIGN.md K12)
        if direct:
            assert precompute and k <= 15, "direct tables need precompute=True and k <= 15"
            flags |= 2
        self.direct = bool(direct)
        self._has_table = bool(precompute)
        _l.check(lib.h2_bases_register_ex(cid, _l.ptr(both), ctypes.c_size_t(both.shape[0]), _l.REPR_CANONICAL,
                                          ctypes.c_uint32(window_bits), ctypes.c_uint32(flags), ctypes.byref(self._h_g)))
        both = np.concatenate([self.g_lagrange, self.w])   # g_lagrange ++ [w]     (:146-147)
        _l.check(lib.h2_bases_register_ex(cid, _l.ptr(both), ctypes.c_size_t(self.n + 1), _l.REPR_CANONICAL,
                                          ctypes.c_uint32(window_bits), ctypes.c_uint32(flags), ctypes.byref(self._h_gl)))

    @classmethod
    def new(cls, curve: str, k: int, **kw) -> "Params":
        """Params::new(k) (commitment.rs:38-114), whole, on the device (h2_params_new): the generators g[i], w, u from
        hash_to_curve("Halo2-Parameters") (:46-58, :102-105), g_lagrange by EC-iFFT, * 2^-k, batch_normalize (:74-101)."""
        assert k < 32  # commitment.rs:41
        n = 1 << k
        g = np.zeros((n, 64), dtype=np.uint8)
        gl = np.zeros((n, 64), dtype=np.uint8)
        w = np.zeros((1, 64), dtype=np.uint8)
        u = np.zeros((1, 64), dtype=np.uint8)
        _l.check(_l.init().h2_params_new(_l.CURVE_ID[curve], ctypes.c_uint32(k), _l.REPR_CANONICAL, _l.ptr(g), _l.ptr(gl), _l.ptr(w), _l.ptr(u)))
        return cls(curve, k, g, gl, w, u, **kw)

    @classmethod
    def from_generators(cls, curve: str, k: int, g, w, u=None, **kw) -> "Params":
        """Params::new (commitment.rs:38-114) from its generators on: g_lagrange is derived on the device exactly as
        :74-101 does -- EC-iFFT of g with alpha_inv = ROOT_OF_UNITY_INV^(2^(S-k)), every output times 2^-k,
        batch_normalize.  (The hash_to_curve calls that produce g, w, u, :46-58 and :103-105, live in the un-vendored
        pasta_curves crate: the caller supplies them, e.g. from Params::read, :185-205.)"""
        assert k < 32  # commitment.rs:41
        n = 1 << k
        gb = _l.as_u8(g, 64)
        assert gb.shape[0] == n
        return cls(curve, k, gb, lagrange_generators(curve, k, gb), w, u, **kw)

    def write(self, writer) -> None:
        """Params::write (commitment.rs:168-181): k as u32 LE, then g, g_lagrange, w, u as compressed points."""
        if self.u is None:
            raise _l.H2Error("Params.write needs u")
        writer.write(int(self.k).to_bytes(4, "little"))
        writer.write(compress_points(np.concatenate([self.g, self.g_lagrange, self.w, self.u]), self.curve).tobytes())

    @classmethod
    def read(cls, curve: str, reader, **kw) -> "Params":
        """Params::read (commitment.rs:183-205).  A short file raises EOFError (read_exact), an invalid point H2Error."""
        head = reader.read(4)
        if len(head) != 4:
            raise EOFError("failed to fill whole buffer")
        k = int.from_bytes(head, "little")
        assert k < 32
        n = 1 << k
        body = reader.read(32 * (2 * n + 2))
        if len(body) != 32 * (2 * n + 2):
            raise EOFError("failed to fill whole buffer")
        pts = decompress_points(np.frombuffer(body, dtype=np.uint8).reshape(-1, 32), curve)
        return cls(curve, k, pts[:n], pts[n:2 * n], pts[2 * n:2 * n + 1], pts[2 * n + 1:], **kw)

    def _commit(self, handle, poly, r: Blind) -> np.ndarray:
        p = _l.as_u8(poly, 32)
        assert p.shape[0] == self.n, "polynomial length != params.n"
        out = np.zeros(96, dtype=np.uint8)
        _l.check(_l.init().h2_msm_registered(handle, _l.ptr(p), ctypes.c_size_t(self.n), _l.ptr(_l.fe_bytes(r.value)),
                                              _l.REPR_CANONICAL, _l.ptr(out)))
        return out

    def commit(self, poly, r: Blind) -> np.ndarray:
        """<poly, g> + r * w   (commitment.rs:119-130)."""
        return self._commit(self._h_g, poly, r)

    def commit_lagrange(self, poly, r: Blind) -> np.ndarray:
        """<poly, g_lagrange> + r * w   (commitment.rs:135-150)."""
        return self._commit(self._h_gl, poly, r)

    def _commit_batched(self, polys, blinds: Sequence[Blind], lagrange: bool, affine: bool, resident: bool) -> np.ndarray:
        """Every batched commit: the blinds encoded once, then one MSM pass per _MSM_BATCH polynomials (host arrays, or
        ResidentPolys with resident=True).  Returns (batch, 64) affine or (batch, 96) Jacobian points."""
        assert len(polys) == len(blinds)
        lib, handle, n = _l.init(), self._h_gl if lagrange else self._h_g, ctypes.c_size_t(self.n)
        bl = _l.fe_array([b.value for b in blinds], FIELDS[_l.SCALAR_FIELD[self.curve]])
        out = np.zeros((len(polys), 64 if affine else 96), dtype=np.uint8)
        for lo in range(0, len(polys), _MSM_BATCH):
            part = polys[lo:lo + _MSM_BATCH]
            count, b, o = ctypes.c_size_t(len(part)), _l.ptr(bl[lo:lo + _MSM_BATCH]), _l.ptr(out[lo:lo + _MSM_BATCH])
            if resident:
                fn = lib.h2_msm_registered_polys_affine if affine else lib.h2_msm_registered_polys
                _l.check(fn(handle, _handles(part), count, n, b, _l.REPR_CANONICAL, o))
            else:
                stack = np.ascontiguousarray(np.stack([_l.as_u8(p, 32) for p in part]))
                assert stack.shape[1] == self.n, "polynomial length != params.n"
                fn = lib.h2_msm_registered_batch_affine if affine else lib.h2_msm_registered_batch
                _l.check(fn(handle, _l.ptr(stack), n, b, count, _l.REPR_CANONICAL, o))
        return out

    def commit_many_affine(self, polys, blinds: Sequence[Blind], lagrange: bool = False) -> np.ndarray:
        """commit_many / commit_lagrange_many followed by C::Curve::batch_normalize on the device: the affine points
        the prover writes to the transcript (plonk/prover.rs:305-316), (batch, 64) uint8."""
        return self._commit_batched(polys, blinds, lagrange, affine=True, resident=False)

    def commit_many(self, polys, blinds: Sequence[Blind]) -> np.ndarray:
        """[commit(p, r) for p, r in zip(polys, blinds)] in one pass over the resident table -- the shape
        of the prover's per-column loops (plonk/prover.rs:305-309, vanishing/prover.rs:102-106)."""
        return self._commit_batched(polys, blinds, lagrange=False, affine=False, resident=False)

    def commit_lagrange_many(self, polys, blinds: Sequence[Blind]) -> np.ndarray:
        return self._commit_batched(polys, blinds, lagrange=True, affine=False, resident=False)

    def commit_resident(self, polys: Sequence["ResidentPoly"], blinds: Sequence[Blind], lagrange: bool = False) -> np.ndarray:
        """[commit(p, r)] (or commit_lagrange with lagrange=True) for device-resident polynomials: nothing but the
        blinds goes up, nothing but the points comes back."""
        return self._commit_batched(polys, blinds, lagrange, affine=False, resident=True)

    def commit_resident_affine(self, polys: Sequence["ResidentPoly"], blinds: Sequence[Blind], lagrange: bool = False) -> np.ndarray:
        """commit_resident + C::Curve::batch_normalize on the device: (batch, 64) affine points, ready for write_point."""
        return self._commit_batched(polys, blinds, lagrange, affine=True, resident=True)

    def _ipa_rounds(self, begin, width: int, x3: int, z: int, challenge, l_rand: Sequence[int], r_rand: Sequence[int]):
        """The round loop of ipa_rounds / ipa_rounds_transcript: `begin(lib, x3, session)` opens the session on p', and the
        rounds return L_j / R_j as Jacobian (width 96) or affine (width 64) points."""
        if self.u is None or not self._has_table:
            raise _l.H2Error("ipa_rounds needs Params(u=..., precompute=True)")
        m = FIELDS[_l.SCALAR_FIELD[self.curve]]
        lib = _l.init()
        assert len(l_rand) == self.k and len(r_rand) == self.k
        sess = ctypes.c_uint64(0)
        _l.check(begin(lib, _l.ptr(_l.fe_bytes(x3 % m)), ctypes.byref(sess)))
        round_call = lib.h2_ipa_round_affine if width == 64 else lib.h2_ipa_round
        ls = np.zeros((self.k, width), dtype=np.uint8)
        rs = np.zeros((self.k, width), dtype=np.uint8)
        lr = np.zeros((2, width), dtype=np.uint8)
        zb = _l.fe_bytes(z % m)
        try:
            for j in range(self.k):
                _l.check(round_call(sess, _l.ptr(zb), _l.ptr(_l.fe_bytes(l_rand[j] % m)), _l.ptr(_l.fe_bytes(r_rand[j] % m)),
                                    _l.REPR_CANONICAL, _l.ptr(lr)))
                ls[j], rs[j] = lr[0], lr[1]
                u_j = int(challenge(j, ls[j], rs[j])) % m
                _l.check(lib.h2_ipa_fold(sess, _l.ptr(_l.fe_bytes(u_j)), _l.ptr(_l.fe_bytes(pow(u_j, -1, m))), _l.REPR_CANONICAL))
            cb = np.zeros((2, 32), dtype=np.uint8)
            _l.check(lib.h2_ipa_finish(sess, _l.REPR_CANONICAL, _l.ptr(cb)))
            sess.value = 0
        finally:
            if sess.value:
                lib.h2_ipa_finish(sess, _l.REPR_CANONICAL, None)
        return ls, rs, int.from_bytes(cb[0].tobytes(), "little")

    def _begin_host(self, p_prime):
        def begin(lib, x3, sess):
            pp = _l.as_u8(p_prime, 32)
            assert pp.shape[0] == self.n
            return lib.h2_ipa_begin(self._h_g, ctypes.c_uint32(self.k), _l.ptr(pp), x3, _l.REPR_CANONICAL, sess)
        return begin

    def ipa_rounds_transcript(self, p_prime, x3: int, z: int, challenge, l_rand: Sequence[int], r_rand: Sequence[int]):
        """ipa_rounds for a transcript-driven caller: `p_prime` may be a ResidentPoly (nothing is uploaded), L_j / R_j come back
        as the AFFINE points the reference writes to the transcript (prover.rs:120-125), and `challenge(j, l_xy, r_xy) -> u_j`.
        Returns (L (k, 64), R (k, 64), c)."""
        if isinstance(p_prime, ResidentPoly):
            def begin(lib, x3, sess):
                return lib.h2_ipa_begin_poly(self._h_g, ctypes.c_uint32(self.k), p_prime._h, x3, _l.REPR_CANONICAL, sess)
        else:
            begin = self._begin_host(p_prime)
        return self._ipa_rounds(begin, 64, x3, z, challenge, l_rand, r_rand)

    def ipa_rounds(self, p_prime, x3: int, z: int, challenge, l_rand: Sequence[int], r_rand: Sequence[int]):
        """The round loop of commitment::create_proof (poly/commitment/prover.rs:100-142) on the device.
        `p_prime` (:80) is the blinded polynomial with P(x3) removed; `challenge(j, L_j, R_j) -> u_j` is the
        caller's transcript (write L_j, R_j; squeeze u_j); l_rand / r_rand are the per-round blinds (:112-113).
        Returns (L (k, 96), R (k, 96), c) -- c is what :147 writes to the transcript."""
        return self._ipa_rounds(self._begin_host(p_prime), 96, x3, z, challenge, l_rand, r_rand)

    def close(self) -> None:
        lib = _l.load()
        for h in (self._h_g, self._h_gl):
            if h.value:
                lib.h2_bases_release(h)
                h.value = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ResidentPoly:
    """A polynomial kept in HBM (Montgomery form) between transforms and commits -- SURVEY.md section 8(f) row 3.
    The reference keeps every Polynomial<F, B> in host memory (poly.rs:56-71); this is the handle a patched prover
    would hold instead while a column travels lagrange -> coeff -> extended.

    It belongs to the lane (or the primary context) that allocated it until share() makes it read-only and readable from
    every lane."""

    _shared = False

    def __init__(self, field: str, length: int, values=None):
        self.field, self.len = field, int(length)
        self._h = ctypes.c_uint64(0)
        _l.check(_l.init().h2_poly_alloc(_l.FIELD_ID[field], ctypes.c_size_t(self.len), ctypes.byref(self._h)))
        if values is not None:
            self.upload(values)

    def upload(self, values) -> None:
        arr = _l.as_u8(values, 32)
        assert arr.shape[0] <= self.len
        _l.check(_l.init().h2_poly_upload(self._h, _l.ptr(arr), ctypes.c_size_t(arr.shape[0]), _l.REPR_CANONICAL))

    def download(self, length: Optional[int] = None) -> np.ndarray:
        n = self.len if length is None else int(length)
        out = np.zeros((n, 32), dtype=np.uint8)
        _l.check(_l.init().h2_poly_download(self._h, _l.ptr(out), ctypes.c_size_t(n), _l.REPR_CANONICAL))
        return out

    @classmethod
    def from_tensor(cls, field: str, t, length: Optional[int] = None, repr: str = "canonical", stream=None) -> "ResidentPoly":
        """A polynomial of `length` elements (default: the tensor's rows) filled from a CUDA tensor on the device, without
        a trip through host memory (h2_poly_upload_dev).  `t`: contiguous torch.uint8 of shape (rows, 32), one element per
        row in `repr` ("canonical" or "montgomery").  Asynchronous on `stream` (default: torch's current stream on t's
        device), ordered before every later call of the calling thread's lane."""
        rows = _tensor_rows(t, "t")
        with freed_on_failure() as fresh:
            p = fresh.keep(cls(field, rows if length is None else length))
            p.upload_tensor(t, repr=repr, stream=stream)
        return p

    def upload_tensor(self, t, repr: str = "canonical", stream=None) -> None:
        """Rows [0, t.shape[0]) <- a CUDA tensor (see from_tensor)."""
        upload_tensors_resident([self], [t], repr=repr, stream=stream)

    def to_tensor(self, length: Optional[int] = None, repr: str = "canonical", out=None, stream=None):
        """The first `length` elements (default: out's rows, else the polynomial's length) as a (length, 32) torch.uint8
        CUDA tensor in `repr`, into `out` when given.  Asynchronous on `stream` (default: torch's current stream), after
        every earlier call of the calling thread's lane (h2_poly_download_dev)."""
        return download_tensors_resident([self], None if length is None else [length], repr=repr, out=None if out is None else [out],
                                         stream=stream)[0]

    def copy_from(self, src: "ResidentPoly", length: int, src_off: int = 0, dst_off: int = 0) -> "ResidentPoly":
        """self[dst_off : dst_off + length] = src[src_off : src_off + length] on the device (`h_poly.chunks_exact(n)`)."""
        _l.check(_l.init().h2_poly_copy(self._h, ctypes.c_size_t(int(dst_off)), src._h, ctypes.c_size_t(int(src_off)), ctypes.c_size_t(int(length))))
        return self

    def add_at(self, index: int, delta: int) -> None:
        """a[index] += delta in place (poly/commitment/prover.rs:51, :78: `poly[0] -= value`)."""
        _l.check(_l.init().h2_poly_add_at(self._h, ctypes.c_size_t(int(index)), _l.ptr(_l.fe_bytes(int(delta) % FIELDS[self.field])), _l.REPR_CANONICAL))

    def share(self) -> "ResidentPoly":
        """h2_poly_share: from now on every lane and the primary context can read the polynomial, and none can write it."""
        share_resident([self])
        return self

    @property
    def shared(self) -> bool:
        return self._shared

    def close(self) -> None:
        """Frees the polynomial.  A shared one may be closed from any thread: the call waits for reads in progress on every lane."""
        if self._h.value:
            _l.load().h2_poly_free(self._h)
            self._h.value = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _Fresh(list):
    """The resident polynomials a call makes for its result (see freed_on_failure)."""

    def keep(self, poly: ResidentPoly) -> ResidentPoly:
        self.append(poly)
        return poly


@contextlib.contextmanager
def freed_on_failure():
    """`with freed_on_failure() as fresh:` -- the polynomials handed to fresh.keep(poly) (which returns poly) are closed if the
    block raises and kept if it returns, so a call that fails leaves none of its outputs allocated."""
    fresh = _Fresh()
    try:
        yield fresh
    except BaseException:
        for p in fresh:
            p.close()
        raise


def _split(flat: list, sizes: Sequence[int]) -> List[list]:
    """flat cut into consecutive lists of sizes[0], sizes[1], ... items: one list per proof."""
    out, at = [], 0
    for s in sizes:
        out.append(flat[at:at + s])
        at += s
    return out


def _handles(polys: Sequence["ResidentPoly"]):
    return (ctypes.c_uint64 * len(polys))(*[p._h.value for p in polys])


_REPRS = {"canonical": _l.REPR_CANONICAL, "montgomery": _l.REPR_MONTGOMERY}


def _repr_id(repr: str) -> int:
    if repr not in _REPRS:
        raise ValueError(f"repr must be 'canonical' or 'montgomery', not {repr!r}")
    return _REPRS[repr]


def is_device_tensor(x) -> bool:
    """x is a CUDA torch tensor (told without importing torch: a package that never sees one never loads it)."""
    return getattr(x, "is_cuda", False) is True and hasattr(x, "data_ptr")


def _tensor_rows(t, name: str, limit: Optional[int] = None) -> int:
    """The rows of a column tensor the device transfers take: contiguous, torch.uint8, shape (rows, 32), at most `limit`
    rows, a CUDA tensor on the library's device.  Anything else is refused; nothing is reinterpreted."""
    import torch
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name}: expected a torch.Tensor, got {type(t).__name__}")
    if t.dtype != torch.uint8:
        raise ValueError(f"{name}: dtype {t.dtype}, expected torch.uint8 (32 bytes per element)")
    if t.dim() != 2 or t.shape[1] != 32:
        raise ValueError(f"{name}: shape {tuple(t.shape)}, expected (rows, 32)")
    if not t.is_contiguous():
        raise ValueError(f"{name}: not contiguous")
    if limit is not None and t.shape[0] > limit:
        raise ValueError(f"{name}: {t.shape[0]} rows, the polynomial holds {limit}")
    if not t.is_cuda:
        raise ValueError(f"{name}: a CPU tensor; host columns go through ResidentPoly(values) / upload()")
    _l.init()
    if t.device.index != _l._inited_device:
        raise ValueError(f"{name}: on {t.device}, the library runs on cuda:{_l._inited_device}")
    return int(t.shape[0])


def _stream_handle(stream, device) -> int:
    import torch
    s = torch.cuda.current_stream(device) if stream is None else stream
    return int(s.cuda_stream)


def upload_dev_resident(polys: Sequence["ResidentPoly"], ptrs: Sequence[int], lens: Sequence[int], repr_id: int, stream: int) -> None:
    """h2_poly_upload_dev: polys[i][0 .. lens[i]) <- the device address ptrs[i], one call for every column, on the CUDA stream
    handle `stream` (0: the legacy default stream)."""
    _dev_io("h2_poly_upload_dev", polys, ptrs, lens, repr_id, stream)


def download_dev_resident(polys: Sequence["ResidentPoly"], ptrs: Sequence[int], lens: Sequence[int], repr_id: int, stream: int) -> None:
    """h2_poly_download_dev: the device address ptrs[i] <- polys[i][0 .. lens[i]), one call for every column."""
    _dev_io("h2_poly_download_dev", polys, ptrs, lens, repr_id, stream)


def _dev_io(name, polys, ptrs, lens, repr_id, stream) -> None:
    count = len(polys)
    if len(ptrs) != count or len(lens) != count:
        raise ValueError("one pointer and one length per polynomial")
    fn = getattr(_l.init(), name)
    _l.check(fn(_handles(polys), ctypes.c_size_t(count), (ctypes.c_void_p * count)(*[int(p) for p in ptrs]),
                (ctypes.c_size_t * count)(*[int(n) for n in lens]), ctypes.c_int(int(repr_id)), ctypes.c_void_p(int(stream))))


def upload_tensors_resident(polys: Sequence["ResidentPoly"], tensors: Sequence, repr: str = "canonical", stream=None) -> None:
    """polys[i][0 .. rows_i) <- tensors[i] (CUDA tensors as ResidentPoly.from_tensor takes them), every column in one
    h2_poly_upload_dev on `stream` (default: torch's current stream on the tensors' device)."""
    if len(polys) != len(tensors):
        raise ValueError("one tensor per polynomial")
    if not polys:
        return
    rid = _repr_id(repr)
    rows = [_tensor_rows(t, f"tensors[{i}]", p.len) for i, (p, t) in enumerate(zip(polys, tensors))]
    upload_dev_resident(polys, [t.data_ptr() for t in tensors], rows, rid, _stream_handle(stream, tensors[0].device))


def download_tensors_resident(polys: Sequence["ResidentPoly"], lengths: Optional[Sequence[int]] = None, repr: str = "canonical",
                              out: Optional[Sequence] = None, stream=None) -> list:
    """[the first lengths[i] elements of polys[i]] as (lengths[i], 32) torch.uint8 CUDA tensors, every column in one
    h2_poly_download_dev on `stream` (default: torch's current stream).  lengths default to out's rows, else to the
    polynomials' lengths; `out` (optional) are the destination tensors, which must not overlap."""
    import torch
    count = len(polys)
    if (lengths is not None and len(lengths) != count) or (out is not None and len(out) != count):
        raise ValueError("one length and one output tensor per polynomial")
    rid = _repr_id(repr)
    rows = [_tensor_rows(t, f"out[{i}]") for i, t in enumerate(out)] if out is not None else None
    if lengths is None:
        lengths = rows if rows is not None else [p.len for p in polys]
    lengths = [int(n) for n in lengths]
    for i, (p, n) in enumerate(zip(polys, lengths)):
        if n < 0 or n > p.len:
            raise ValueError(f"lengths[{i}] = {n}: the polynomial holds {p.len}")
        if rows is not None and rows[i] < n:
            raise ValueError(f"out[{i}]: {rows[i]} rows, fewer than the {n} requested")
    if not polys:
        return []
    _l.init()
    device = out[0].device if out is not None else torch.device("cuda", _l._inited_device)
    if out is None:
        s = torch.cuda.current_stream(device) if stream is None else stream
        with torch.cuda.stream(s):                     # allocated for the stream that writes it
            out = [torch.empty((n, 32), dtype=torch.uint8, device=device) for n in lengths]
    download_dev_resident(polys, [t.data_ptr() for t in out], lengths, rid, _stream_handle(stream, device))
    return list(out)


def share_resident(polys: Sequence["ResidentPoly"]) -> None:
    """h2_poly_share of all `polys` in one call, all or none: each must belong to the calling thread's lane (or be shared)."""
    _l.check(_l.init().h2_poly_share(_handles(polys), ctypes.c_size_t(len(polys))))
    for p in polys:
        p._shared = True


def set_rows_resident(polys: Sequence["ResidentPoly"], start: int, values) -> None:
    """Rows [start, start + rows) of every polynomial <- values[i] (a (count, rows, 32) uint8 array, or one list of ints per
    polynomial), in one upload and one kernel (h2_poly_set_rows): the blinding rows of resident advice columns."""
    count = len(polys)
    if count == 0:
        return
    if isinstance(values, np.ndarray):
        arr = np.ascontiguousarray(values, dtype=np.uint8)
    else:
        arr = _l.fe_array((v for col in values for v in col), FIELDS[polys[0].field])
    arr = arr.reshape(count, -1, 32) if arr.size else np.zeros((count, 0, 32), dtype=np.uint8)
    _l.check(_l.init().h2_poly_set_rows(_handles(polys), ctypes.c_size_t(count), ctypes.c_size_t(int(start)), ctypes.c_size_t(arr.shape[1]),
                                        _l.ptr(arr) if arr.size else None, _l.REPR_CANONICAL))


def eval_polynomial_resident(polys: Sequence["ResidentPoly"], points: Sequence[int], n: Optional[int] = None) -> list:
    """[eval_polynomial(p, x)] (arithmetic.rs:297-303) for device-resident coefficient vectors, one launch tree for the batch."""
    batch = len(polys)
    assert batch == len(points) and batch >= 1
    n = polys[0].len if n is None else int(n)
    pts = _l.fe_array(points, FIELDS[polys[0].field])
    out = np.zeros((batch, 32), dtype=np.uint8)
    _l.check(_l.init().h2_poly_eval(_handles(polys), ctypes.c_size_t(batch), ctypes.c_size_t(n), _l.ptr(pts), _l.REPR_CANONICAL, _l.ptr(out)))
    return [int.from_bytes(r.tobytes(), "little") for r in out]


def inner_product_resident(a: Sequence["ResidentPoly"], b: Sequence["ResidentPoly"], n: Optional[int] = None) -> list:
    """[compute_inner_product(a_i, b_i)] (arithmetic.rs:308-319); panics (AssertionError) on unequal lengths like assert_eq! :311."""
    batch = len(a)
    assert batch == len(b) and batch >= 1
    if n is None:
        assert all(x.len == y.len for x, y in zip(a, b)), "compute_inner_product: a.len() != b.len()"
        n = a[0].len
    out = np.zeros((batch, 32), dtype=np.uint8)
    _l.check(_l.init().h2_poly_inner_product(_handles(a), _handles(b), ctypes.c_size_t(batch), ctypes.c_size_t(int(n)), _l.REPR_CANONICAL, _l.ptr(out)))
    return [int.from_bytes(r.tobytes(), "little") for r in out]


def kate_division_resident(src: Sequence["ResidentPoly"], points: Sequence[int], dst: Optional[Sequence["ResidentPoly"]] = None,
                           n: Optional[int] = None) -> list:
    """[kate_division(a, b)] (arithmetic.rs:322-341): quotients by (X - b), n - 1 coefficients each, left on the device."""
    batch = len(src)
    assert batch == len(points) and batch >= 1
    n = src[0].len if n is None else int(n)
    pts = _l.fe_array(points, FIELDS[src[0].field])
    with freed_on_failure() as fresh:
        if dst is None:
            dst = [fresh.keep(ResidentPoly(src[0].field, max(n - 1, 1))) for _ in range(batch)]
        _l.check(_l.init().h2_poly_kate_division(_handles(dst), _handles(src), ctypes.c_size_t(batch), ctypes.c_size_t(n), _l.ptr(pts), _l.REPR_CANONICAL))
    return list(dst)


def batch_invert_resident(a: "ResidentPoly", n: Optional[int] = None) -> "ResidentPoly":
    """`values.batch_invert()` (ff::BatchInvert) in place on a resident vector: zeros stay zero (plonk/permutation/prover.rs:120)."""
    _l.check(_l.init().h2_poly_batch_invert(a._h, ctypes.c_size_t(a.len if n is None else int(n))))
    return a


def running_product_resident(src: "ResidentPoly", init: int = 1, dst: Optional["ResidentPoly"] = None, n: Optional[int] = None) -> "ResidentPoly":
    """z[0] = init, z[i] = z[i-1] * src[i-1] (plonk/permutation/prover.rs:150-156), left on the device."""
    n = src.len if n is None else int(n)
    with freed_on_failure() as fresh:
        dst = fresh.keep(ResidentPoly(src.field, n)) if dst is None else dst
        _l.check(_l.init().h2_poly_running_product(dst._h, src._h, ctypes.c_size_t(n), _l.ptr(_l.fe_bytes(int(init) % FIELDS[src.field])), _l.REPR_CANONICAL))
    return dst


def permute_expression_pair_resident(input_expression: "ResidentPoly", table_expression: "ResidentPoly", usable_rows: int,
                                     out_input: Optional["ResidentPoly"] = None, out_table: Optional["ResidentPoly"] = None):
    """permute_expression_pair (plonk/lookup/prover.rs:563-647) on resident Lagrange-basis columns: returns (A', S') with
    A'[:usable_rows] the sorted input values and S'[:usable_rows] the table values arranged so that S'[r] == A'[r] on the first
    row of every run of equal inputs.  The blinding rows from `usable_rows` on (:625-627) are the caller's: write them with
    `upload_at`-style calls or `add_at`.  An input value missing from the table raises H2Error (the reference returns
    Error::ConstraintSystemFailure, :605-608)."""
    with freed_on_failure() as fresh:
        out_input = fresh.keep(ResidentPoly(input_expression.field, input_expression.len)) if out_input is None else out_input
        out_table = fresh.keep(ResidentPoly(input_expression.field, input_expression.len)) if out_table is None else out_table
        _l.check(_l.init().h2_poly_lookup_permute(input_expression._h, table_expression._h, ctypes.c_size_t(int(usable_rows)), out_input._h, out_table._h))
    return out_input, out_table


class EvaluationDomain:
    """poly/domain.rs:20-146.  `zeta` is F::ZETA (domain.rs:85): pasta_curves' choice of cube root
    is not pinned by any in-tree golden, so the caller supplies it."""

    def __init__(self, field: str, j: int, k: int, zeta: int):
        m = FIELDS[field]
        self.field, self.m, self.k, self.n = field, m, k, 1 << k
        self.quotient_poly_degree = j - 1
        ext_k = k
        while (1 << ext_k) < self.n * self.quotient_poly_degree:
            ext_k += 1
        assert ext_k <= S  # domain.rs:56
        self.extended_k = ext_k
        ew = pow(5, (m - 1) >> S, m)  # ROOT_OF_UNITY
        for _ in range(ext_k, S):
            ew = ew * ew % m
        self.extended_omega = ew
        w = ew
        for _ in range(k, ext_k):
            w = w * w % m
        self.omega = w
        self.omega_inv = pow(w, -1, m)
        self.extended_omega_inv = pow(ew, -1, m)
        assert pow(zeta, 3, m) == 1 and zeta != 1, "zeta must be a primitive cube root of unity"
        self.g_coset = zeta
        self.g_coset_inv = zeta * zeta % m
        self.ifft_divisor = pow((1 << k) % m, -1, m)
        self.extended_ifft_divisor = pow((1 << ext_k) % m, -1, m)
        # t(X) = X^n - 1 over the coset, inverted (domain.rs:86-128): 2^(ext_k - k) values, then it repeats
        orig, step = pow(zeta, self.n, m), pow(ew, self.n, m)
        t, cur = [], orig
        while True:
            t.append(cur)
            cur = cur * step % m
            if cur == orig:
                break
        assert len(t) == 1 << (ext_k - k)
        self.t_evaluations = [pow((x - 1) % m, m - 2, m) for x in t]

    def extended_len(self) -> int:
        return 1 << self.extended_k

    def rotate_omega(self, value: int, rotation: int) -> int:
        """domain.rs:408-418: value * omega^rotation (a handful of scalars per proof: host arithmetic)."""
        return value * pow(self.omega if rotation >= 0 else self.omega_inv, abs(rotation), self.m) % self.m

    def l_i_range(self, x: int, xn: int, rotations) -> list:
        """domain.rs:447-472: l_i(x) for every rotation i in `rotations` (xn = x^n), l_i(omega^i) = 1:
        l_i(x) = omega^i (x^n - 1) / (n (x - omega^i)); the reference batch-inverts the denominators, and panics (division by
        zero in the inversion's unwrap-free path gives 0) only for x on the domain, which a challenge never is."""
        m = self.m
        rotations = list(rotations)
        common = (xn - 1) * self.ifft_divisor % m                 # (x^n - 1) * barycentric_weight, :465
        out = []
        for r in rotations:
            d = (x - self.rotate_omega(1, r)) % m
            out.append(self.rotate_omega((pow(d, -1, m) if d else 0) * common % m, r))
        return out

    def lagrange_to_coeff(self, a) -> np.ndarray:
        """domain.rs:227-237 (+ ifft :375-383)."""
        arr = _l.as_u8(a, 32).copy()
        assert arr.shape[0] == 1 << self.k
        _l.check(_l.init().h2_intt_scaled(_l.FIELD_ID[self.field], _l.ptr(arr), _l.ptr(_l.fe_bytes(self.omega_inv)),
                                          _l.ptr(_l.fe_bytes(self.ifft_divisor)), ctypes.c_uint32(self.k), _l.REPR_CANONICAL))
        return arr

    def coeff_to_extended(self, a) -> np.ndarray:
        """domain.rs:241-255: zeta-scale, zero-pad and transform, fused in the first NTT pass."""
        arr = _l.as_u8(a, 32)
        assert arr.shape[0] == 1 << self.k
        out = np.zeros((self.extended_len(), 32), dtype=np.uint8)
        _l.check(_l.init().h2_coeff_to_extended(_l.FIELD_ID[self.field], _l.ptr(arr), ctypes.c_uint32(self.k),
                                                ctypes.c_uint32(self.extended_k), _l.ptr(_l.fe_bytes(self.g_coset)),
                                                _l.ptr(_l.fe_bytes(self.extended_omega)), _l.ptr(out), _l.REPR_CANONICAL))
        return out

    def extended_to_coeff(self, a) -> np.ndarray:
        """domain.rs:303-325: inverse transform, coset un-scale and truncate, fused in the last pass."""
        arr = _l.as_u8(a, 32)
        assert arr.shape[0] == self.extended_len()
        out_len = self.n * self.quotient_poly_degree
        out = np.zeros((out_len, 32), dtype=np.uint8)
        _l.check(_l.init().h2_extended_to_coeff(_l.FIELD_ID[self.field], _l.ptr(arr), ctypes.c_uint32(self.extended_k),
                                                _l.ptr(_l.fe_bytes(self.extended_omega_inv)),
                                                _l.ptr(_l.fe_bytes(self.extended_ifft_divisor)),
                                                _l.ptr(_l.fe_bytes(self.g_coset)), ctypes.c_size_t(out_len), _l.ptr(out),
                                                _l.REPR_CANONICAL))
        return out

    def divide_by_vanishing_poly(self, a) -> np.ndarray:
        """domain.rs:329-348 on a host vector of extended-domain evaluations (through a temporary resident polynomial)."""
        arr = _l.as_u8(a, 32)
        assert arr.shape[0] == self.extended_len()
        r = ResidentPoly(self.field, self.extended_len(), arr)
        try:
            return self.divide_by_vanishing_poly_resident(r).download()
        finally:
            r.close()

    def divide_by_vanishing_poly_resident(self, a: "ResidentPoly") -> "ResidentPoly":
        """In place on a resident extended-domain polynomial (the step between the AST evaluation and extended_to_coeff,
        plonk/vanishing/prover.rs:81-88)."""
        assert a.len >= self.extended_len()
        t = _l.fe_array(self.t_evaluations, self.m)
        _l.check(_l.init().h2_poly_divide_by_vanishing(a._h, ctypes.c_uint32(self.extended_k), _l.ptr(t), ctypes.c_uint32(len(self.t_evaluations)),
                                                       _l.REPR_CANONICAL))
        return a

    # ---- device-resident forms (SURVEY.md section 8(f) row 3): asynchronous, no host copies
    def lagrange_to_coeff_resident(self, a: "ResidentPoly", out: Optional["ResidentPoly"] = None) -> "ResidentPoly":
        out = a if out is None else out
        _l.check(_l.init().h2_poly_lagrange_to_coeff(out._h, a._h, ctypes.c_uint32(self.k), _l.ptr(_l.fe_bytes(self.omega_inv)),
                                                     _l.ptr(_l.fe_bytes(self.ifft_divisor)), _l.REPR_CANONICAL))
        return out

    def coeff_to_extended_resident(self, a: "ResidentPoly", out: Optional["ResidentPoly"] = None) -> "ResidentPoly":
        with freed_on_failure() as fresh:
            out = fresh.keep(ResidentPoly(self.field, self.extended_len())) if out is None else out
            _l.check(_l.init().h2_poly_coeff_to_extended(out._h, a._h, ctypes.c_uint32(self.k), ctypes.c_uint32(self.extended_k),
                                                         _l.ptr(_l.fe_bytes(self.g_coset)), _l.ptr(_l.fe_bytes(self.extended_omega)),
                                                         _l.REPR_CANONICAL))
        return out

    def extended_to_coeff_resident(self, a: "ResidentPoly", out: Optional["ResidentPoly"] = None) -> "ResidentPoly":
        out_len = self.n * self.quotient_poly_degree
        with freed_on_failure() as fresh:
            out = fresh.keep(ResidentPoly(self.field, out_len)) if out is None else out
            _l.check(_l.init().h2_poly_extended_to_coeff(out._h, a._h, ctypes.c_uint32(self.extended_k),
                                                         _l.ptr(_l.fe_bytes(self.extended_omega_inv)),
                                                         _l.ptr(_l.fe_bytes(self.extended_ifft_divisor)), _l.ptr(_l.fe_bytes(self.g_coset)),
                                                         ctypes.c_size_t(out_len), _l.REPR_CANONICAL))
        return out

    def lagrange_to_coeff_batch_resident(self, polys: Sequence["ResidentPoly"], out: Optional[Sequence["ResidentPoly"]] = None) -> list:
        """lagrange_to_coeff of every column in one call (h2_poly_lagrange_to_coeff_batch): each NTT pass is one launch for all
        of them.  out=None transforms in place."""
        out = list(polys) if out is None else list(out)
        assert len(out) == len(polys)
        _l.check(_l.init().h2_poly_lagrange_to_coeff_batch(_handles(out), _handles(polys), ctypes.c_size_t(len(polys)), ctypes.c_uint32(self.k),
                                                           _l.ptr(_l.fe_bytes(self.omega_inv)), _l.ptr(_l.fe_bytes(self.ifft_divisor)),
                                                           _l.REPR_CANONICAL))
        return out

    def coeff_to_extended_batch_resident(self, polys: Sequence["ResidentPoly"], out: Optional[Sequence["ResidentPoly"]] = None) -> list:
        """coeff_to_extended of every column in one call (h2_poly_coeff_to_extended_batch).  out=None allocates the cosets."""
        with freed_on_failure() as fresh:
            out = [fresh.keep(ResidentPoly(self.field, self.extended_len())) for _ in polys] if out is None else list(out)
            assert len(out) == len(polys)
            _l.check(_l.init().h2_poly_coeff_to_extended_batch(_handles(out), _handles(polys), ctypes.c_size_t(len(polys)), ctypes.c_uint32(self.k),
                                                               ctypes.c_uint32(self.extended_k), _l.ptr(_l.fe_bytes(self.g_coset)),
                                                               _l.ptr(_l.fe_bytes(self.extended_omega)), _l.REPR_CANONICAL))
        return out
