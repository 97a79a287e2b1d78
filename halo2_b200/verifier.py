"""Host-side mirror of the verifier's side of the polynomial commitment scheme over the C ABI:

  * `MSM`          poly::commitment::MSM<C>                  (/root/reference/halo2_proofs/src/poly/commitment/msm.rs:9-178)
  * `verify_proof` poly::commitment::verify_proof            (poly/commitment/verifier.rs:67-141)
  * `Guard`        poly::commitment::Guard                   (poly/commitment/verifier.rs:13-63)
  * `compute_b`    (verifier.rs:145-153)

Same names, argument meaning and panics as the reference.  The verifier's hot path is `MSM::eval` (msm.rs:138-177): one
best_multiexp over params.g (2^k bases) plus w, u and the proof's commitments.  Here `g_scalars` is a ResidentPoly in HBM:
compute_s (verifier.rs:156-171) is built on the device straight into it (`h2_poly_compute_s`), `scale` / `add_msm` are one
elementwise pass (`h2_poly_scale_add`), and `eval` commits the resident vector against the resident generator table
(`h2_msm_registered_polys`, w_scalar on base index n), runs the few dozen other terms through `h2_msm` and adds the two
(`h2_point_sum`).  The `other` map, w_scalar, u_scalar and the k round challenges are a few dozen scalars and stay on the host,
as does the transcript (the caller's: any object with read_point() -> (64,) uint8 affine x||y, read_scalar() -> int,
squeeze_challenge() -> int).  No CPU fallback: every group operation and every O(n) loop runs through the CUDA library.

Elements: scalars are Python ints (canonical), points (64,) uint8 affine x||y little-endian, identity = zeros.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import lib as _l
from .arithmetic import best_multiexp
from .poly import FIELDS, Blind, Params, ResidentPoly


class VerifyError(Exception):
    """Error::OpeningError / Error::SamplingError (poly/commitment/verifier.rs:77, :86-87, :126-128)."""


def compute_b(x: int, u: Sequence[int], modulus: int) -> int:
    """verifier.rs:145-153: prod_{i<k} (1 + u_{k-1-i} x^(2^i)) -- k multiplications, on the host like the challenges."""
    tmp, cur = 1, x % modulus
    for u_j in reversed(list(u)):
        tmp = tmp * (1 + u_j * cur) % modulus
        cur = cur * cur % modulus
    return tmp


def batch_invert(values: Sequence[int], modulus: int) -> List[int]:
    """ff::BatchInvert (verifier.rs:95-98): all inverses from ONE modular inversion (Montgomery's trick); zeros stay zero."""
    prefix, acc = [], 1
    for v in values:
        prefix.append(acc)
        if v % modulus:
            acc = acc * v % modulus
    inv = pow(acc, -1, modulus)
    out = [0] * len(values)
    for i in range(len(values) - 1, -1, -1):
        v = values[i] % modulus
        if v:
            out[i] = inv * prefix[i] % modulus
            inv = inv * v % modulus
    return out


def _is_identity_xy(xy: np.ndarray) -> bool:
    return not xy.any()


class MSM:
    """msm.rs:9-178.  `params` must carry u (Params(..., u=...)): eval needs all of g, w, u."""

    def __init__(self, params: Params):
        if params.u is None:
            raise _l.H2Error("MSM needs Params(u=...)")
        self.params = params
        self.field = _l.SCALAR_FIELD[params.curve]
        self.r = FIELDS[self.field]
        self.p = FIELDS[_l.BASE_FIELD[params.curve]]
        self.g_scalars: Optional[ResidentPoly] = None
        self.w_scalar: Optional[int] = None
        self.u_scalar: Optional[int] = None
        self.other: Dict[bytes, Tuple[int, bytes]] = {}      # x -> (scalar, y), the reference's BTreeMap<C::Base, (C::Scalar, C::Base)>

    # ---- structure ------------------------------------------------------------------------------------------------------
    def clone(self) -> "MSM":
        o = MSM(self.params)
        if self.g_scalars is not None:
            o.g_scalars = ResidentPoly(self.field, self.params.n).copy_from(self.g_scalars, self.params.n)
        o.w_scalar, o.u_scalar, o.other = self.w_scalar, self.u_scalar, dict(self.other)
        return o

    def close(self) -> None:
        if self.g_scalars is not None:
            self.g_scalars.close()
            self.g_scalars = None

    def _merge(self, x: bytes, y: bytes, scalar: int) -> None:   # msm.rs:40-50, :73-83
        if x in self.other:
            ours, our_y = self.other[x]
            if our_y == y:
                self.other[x] = ((ours + scalar) % self.r, our_y)
            else:
                assert int.from_bytes(our_y, "little") == (-int.from_bytes(y, "little")) % self.p, "MSM: same x, unrelated y"
                self.other[x] = ((ours - scalar) % self.r, our_y)
        else:
            self.other[x] = (scalar % self.r, y)

    def _g(self) -> ResidentPoly:
        if self.g_scalars is None:
            self.g_scalars = ResidentPoly(self.field, self.params.n)      # zero-filled on the device (h2_poly_alloc)
        return self.g_scalars

    # ---- the reference's methods ----------------------------------------------------------------------------------------
    def add_msm(self, other: "MSM") -> None:
        """msm.rs:37-62."""
        for x, (scalar, y) in other.other.items():
            self._merge(x, y, scalar)
        if other.g_scalars is not None:
            self.add_to_g_scalars(other.g_scalars)
        if other.w_scalar is not None:
            self.add_to_w_scalar(other.w_scalar)
        if other.u_scalar is not None:
            self.add_to_u_scalar(other.u_scalar)

    def append_term(self, scalar: int, point) -> None:
        """msm.rs:65-84 (the identity is skipped, :66)."""
        xy = np.ascontiguousarray(point, dtype=np.uint8).reshape(64)
        if not _is_identity_xy(xy):
            self._merge(bytes(xy[:32]), bytes(xy[32:]), int(scalar))

    def add_constant_term(self, constant: int) -> None:
        """msm.rs:87-95: g_scalars[0] += constant."""
        self._g().add_at(0, int(constant) % self.r)

    def add_to_g_scalars(self, scalars) -> None:
        """msm.rs:99-109; `scalars` is a ResidentPoly or an (n, 32) host array.  Panics unless its length is params.n (:100)."""
        n = self.params.n
        if isinstance(scalars, ResidentPoly):
            assert scalars.len == n, "add_to_g_scalars: scalars.len() != params.n"
            src, tmp = scalars, None
        else:
            arr = _l.as_u8(scalars, 32)
            assert arr.shape[0] == n, "add_to_g_scalars: scalars.len() != params.n"
            src = tmp = ResidentPoly(self.field, n, arr)
        try:
            if self.g_scalars is None:
                self.g_scalars = ResidentPoly(self.field, n).copy_from(src, n)
            else:
                one = _l.fe_bytes(1)
                _l.check(_l.init().h2_poly_scale_add(self.g_scalars._h, _l.ptr(one), src._h, _l.ptr(one), ctypes.c_size_t(n), _l.REPR_CANONICAL))
        finally:
            if tmp is not None:
                tmp.close()

    def add_compute_s(self, u: Sequence[int], init: int) -> None:
        """`self.add_to_g_scalars(&compute_s(u, init))` (verifier.rs:36-38) in one pass on the device: s is never materialised."""
        k = len(u)
        assert k > 0 and (1 << k) == self.params.n, "compute_s: u.len() != params.k"
        accumulate = 0 if self.g_scalars is None else 1
        ub = _l.fe_array(u, self.r)
        _l.check(_l.init().h2_poly_compute_s(self._g()._h, _l.ptr(ub), ctypes.c_uint32(k), _l.ptr(_l.fe_bytes(int(init) % self.r)), accumulate,
                                             _l.REPR_CANONICAL))

    def add_to_w_scalar(self, scalar: int) -> None:
        """msm.rs:112-114."""
        self.w_scalar = scalar % self.r if self.w_scalar is None else (self.w_scalar + scalar) % self.r

    def add_to_u_scalar(self, scalar: int) -> None:
        """msm.rs:117-119."""
        self.u_scalar = scalar % self.r if self.u_scalar is None else (self.u_scalar + scalar) % self.r

    def scale(self, factor: int) -> None:
        """msm.rs:122-135."""
        factor = int(factor) % self.r
        if self.g_scalars is not None:
            _l.check(_l.init().h2_poly_scale_add(self.g_scalars._h, _l.ptr(_l.fe_bytes(factor)), ctypes.c_uint64(0), None,
                                                 ctypes.c_size_t(self.params.n), _l.REPR_CANONICAL))
        self.other = {x: (s * factor % self.r, y) for x, (s, y) in self.other.items()}
        if self.w_scalar is not None:
            self.w_scalar = self.w_scalar * factor % self.r
        if self.u_scalar is not None:
            self.u_scalar = self.u_scalar * factor % self.r

    def scale_add_msm(self, factor: int, other: "MSM") -> None:
        """`self.scale(factor); self.add_msm(other)` -- BatchVerifier's accumulate_msm (plonk/verifier/batch.rs:83-93) -- with the
        two passes over g_scalars fused into one when both sides have the vector."""
        if self.g_scalars is not None and other.g_scalars is not None:
            factor = int(factor) % self.r
            _l.check(_l.init().h2_poly_scale_add(self.g_scalars._h, _l.ptr(_l.fe_bytes(factor)), other.g_scalars._h, _l.ptr(_l.fe_bytes(1)),
                                                 ctypes.c_size_t(self.params.n), _l.REPR_CANONICAL))
            mine, self.g_scalars = self.g_scalars, None          # the rest of scale / add_msm without touching the vector again
            theirs, other.g_scalars = other.g_scalars, None
            try:
                self.scale(factor)
                self.add_msm(other)
            finally:
                self.g_scalars, other.g_scalars = mine, theirs
        else:
            self.scale(factor)
            self.add_msm(other)

    def evaluate(self) -> np.ndarray:
        """The group element of eval's multiexp (msm.rs:142-175) as a Jacobian point (96 bytes, z = 0 for the identity)."""
        P = self.params
        parts: List[np.ndarray] = []
        scalars = [s for s, _ in self.other.values()]
        bases = [np.frombuffer(x + y, dtype=np.uint8) for x, (_, y) in self.other.items()]
        if self.u_scalar is not None:
            scalars.append(self.u_scalar)
            bases.append(P.u.reshape(64))
        if self.g_scalars is not None:
            # <g_scalars, g> + w_scalar * w over the resident table: g ++ [w] is what commit runs on (poly/commitment.rs:126-127)
            parts.append(P.commit_resident([self.g_scalars], [Blind(self.w_scalar or 0)])[0])
        elif self.w_scalar is not None:
            scalars.append(self.w_scalar)
            bases.append(P.w.reshape(64))
        if scalars:
            sc = _l.fe_array(scalars, self.r)
            parts.append(best_multiexp(sc, np.ascontiguousarray(np.stack(bases)), curve=P.curve))
        if not parts:
            return np.zeros(96, dtype=np.uint8)                  # the empty multiexp: the identity
        if len(parts) == 1:
            return parts[0]
        out = np.zeros(96, dtype=np.uint8)
        pts = np.ascontiguousarray(np.stack(parts))
        _l.check(_l.init().h2_point_sum(_l.CURVE_ID[P.curve], _l.ptr(pts), ctypes.c_size_t(len(parts)), _l.REPR_CANONICAL, _l.ptr(out)))
        return out

    def eval(self) -> bool:
        """msm.rs:138-177: `bool::from(best_multiexp(&scalars, &bases).is_identity())`."""
        return not self.evaluate()[64:96].any()


class Guard:
    """verifier.rs:13-63: what verify_proof returns; the caller either supplies the challenges' s vector (use_challenges)
    or a purported G (use_g)."""

    def __init__(self, msm: MSM, neg_c: int, u: List[int]):
        self.msm, self.neg_c, self.u = msm, neg_c, list(u)

    def clone(self) -> "Guard":
        return Guard(self.msm.clone(), self.neg_c, self.u)

    def use_challenges(self) -> MSM:
        """verifier.rs:36-41: g_scalars += compute_s(u, -c)."""
        self.msm.add_compute_s(self.u, self.neg_c)
        return self.msm

    def use_g(self, g) -> Tuple[MSM, Tuple[np.ndarray, List[int]]]:
        """verifier.rs:45-55: appends [-c] G; returns the MSM and the accumulator (g, u)."""
        g = np.ascontiguousarray(g, dtype=np.uint8).reshape(64)
        self.msm.append_term(self.neg_c, g)
        return self.msm, (g, list(self.u))

    def compute_g(self) -> np.ndarray:
        """verifier.rs:58-62: G = <compute_s(u, 1), params.g> as an affine point."""
        m = MSM(self.msm.params)
        try:
            m.add_compute_s(self.u, 1)
            return self.msm.params.commit_resident_affine([m.g_scalars], [Blind(0)])[0]
        finally:
            m.close()


def verify_proof(params: Params, msm: MSM, transcript, x: int, v: int) -> Guard:
    """commitment::verify_proof (verifier.rs:67-141): checks that the proof in `transcript` opens the commitment `msm`
    evaluates to, at `x`, to the value `v`; returns the Guard whose MSM must evaluate to the identity."""
    r = msm.r
    k = params.k
    msm.add_constant_term((-v) % r)                              # :76  P' = P - [v] G_0 + [xi] S
    try:
        s_poly_commitment = transcript.read_point()              # :77
    except Exception as e:
        raise VerifyError("OpeningError") from e
    xi = transcript.squeeze_challenge()                          # :78
    msm.append_term(xi, s_poly_commitment)                       # :79
    z = transcript.squeeze_challenge()                           # :81
    rounds = []
    for _ in range(k):                                           # :84-93
        try:
            l = transcript.read_point()
            rr = transcript.read_point()
        except Exception as e:
            raise VerifyError("OpeningError") from e
        rounds.append((l, rr, transcript.squeeze_challenge()))
    u: List[int] = []
    u_inv = batch_invert([u_j for _, _, u_j in rounds], r)       # :95-98
    for (l, rr, u_j), u_j_inv in zip(rounds, u_inv):             # :104-111
        msm.append_term(u_j_inv, l)
        msm.append_term(u_j, rr)
        u.append(u_j)
    try:
        c = transcript.read_scalar()                             # :126
        f = transcript.read_scalar()                             # :128
    except Exception as e:
        raise VerifyError("SamplingError") from e
    neg_c = (-c) % r
    b = compute_b(x, u, r)                                       # :129
    msm.add_to_u_scalar(neg_c * b % r * z % r)                   # :131
    msm.add_to_w_scalar((-f) % r)                                # :132
    return Guard(msm, neg_c, u)
