"""Host-side mirror of poly::commitment::create_proof, the opening prover of the polynomial commitment scheme
(/root/reference/halo2_proofs/src/poly/commitment/prover.rs:36-151), on device-resident polynomials over the C ABI.

Every O(n) step runs on the GPU: the blinding polynomial's evaluation (`h2_poly_eval`), its commitment over the resident
generator table (`h2_msm_registered_polys_affine`), p' = s * xi + p in one elementwise pass (`h2_poly_scale_add`), and the
k rounds (`h2_ipa_*`: fold-free L_j / R_j over the original generators, csrc/ipa.cuh).  The transcript, the k challenges
and their inverses and the running blind f are a handful of scalars and stay with the caller's host code.

Randomness: the reference draws s_poly (n scalars), its blind and two scalars per round from `rng` in that order
(prover.rs:46-54, :112-113).  Here `rng` is any object with `poly(n)` -> a ResidentPoly or (n, 32) uint8 array the callee may
keep, and `scalar()` -> int.  halo2_b200.ChaCha20Rng draws s_poly on the device, the scalars a ChaCha20Rng with the same seed
and position gives (h2_poly_random); any other rng hands over its own draws.
"""
from __future__ import annotations

import ctypes
from typing import Union

from . import lib as _l
from .poly import FIELDS, Blind, Params, ResidentPoly, eval_polynomial_resident


def _scale_add(dst: ResidentPoly, a: int, src: ResidentPoly, b: int, n: int) -> None:
    """dst = a * dst + b * src on the device (one pass)."""
    m = FIELDS[dst.field]
    _l.check(_l.init().h2_poly_scale_add(dst._h, _l.ptr(_l.fe_bytes(int(a) % m)), src._h, _l.ptr(_l.fe_bytes(int(b) % m)), ctypes.c_size_t(n),
                                         _l.REPR_CANONICAL))


def create_proof(params: Params, rng, transcript, p_poly: ResidentPoly, p_blind: Union[Blind, int], x_3: int) -> None:
    """commitment::create_proof (prover.rs:36-151): writes the opening of `p_poly` (blind `p_blind`) at `x_3` to `transcript`
    (write_point((64,) uint8 affine), write_scalar(int), squeeze_challenge() -> int).  `p_poly` is left untouched."""
    n, k = params.n, params.k
    assert p_poly.len == n, "create_proof: p_poly.len() != params.n"          # :41
    field = _l.SCALAR_FIELD[params.curve]
    m = FIELDS[field]
    p_blind = p_blind.value if isinstance(p_blind, Blind) else int(p_blind)
    s = rng.poly(n)                                                            # :46-49
    own = not isinstance(s, ResidentPoly)
    if own:
        s = ResidentPoly(field, n, s)
    try:
        assert s.len == n
        s_at_x3 = eval_polynomial_resident([s], [x_3], n=n)[0]                 # :51
        s.add_at(0, -s_at_x3)                                                  # :52
        s_poly_blind = rng.scalar() % m                                        # :54
        transcript.write_point(params.commit_resident_affine([s], [Blind(s_poly_blind)])[0])   # :57-58
        xi = transcript.squeeze_challenge()                                    # :63
        z = transcript.squeeze_challenge()                                     # :67
        _scale_add(s, xi, p_poly, 1, n)                                        # :71  p' = s * xi + p  (in s's buffer)
        v = eval_polynomial_resident([s], [x_3], n=n)[0]                       # :72
        s.add_at(0, -v)                                                        # :73
        f = (s_poly_blind * xi + p_blind) % m                                  # :74-76
        rand = [(rng.scalar() % m, rng.scalar() % m) for _ in range(k)]        # :112-113, drawn in the reference's order
        us = []

        def challenge(j, l_xy, r_xy):                                          # :119-122
            transcript.write_point(l_xy)
            transcript.write_point(r_xy)
            us.append(transcript.squeeze_challenge())
            return us[-1]

        _, _, c = params.ipa_rounds_transcript(s, x_3, z, challenge, [a for a, _ in rand], [b for _, b in rand])   # :100-142
        for (l_r, r_r), u_j in zip(rand, us):                                  # :140-141
            f = (f + l_r * pow(u_j, -1, m) + r_r * u_j) % m
        transcript.write_scalar(c)                                             # :148
        transcript.write_scalar(f)                                             # :149
    finally:
        if own:
            s.close()
