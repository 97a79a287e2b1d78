"""The vanishing argument over the C ABI: plonk::vanishing::Argument::commit and Committed::construct / Constructed::evaluate /
Evaluated::open (/root/reference/halo2_proofs/src/plonk/vanishing/prover.rs:38-175) on device-resident polynomials.

construct evaluates h(X) once on the extended domain and then makes one h2_poly_vanishing_quotient call, which divides by
X^n - 1, transforms back to coefficients and splits into the quotient_poly_degree pieces of n coefficients in one transform
(csrc/ntt.cuh, K24).  The h(X) expressions are the caller's, as in the reference (plonk/prover.rs:460-586 builds them).

The library has no transcript: commit and construct return the commitments and evaluate returns random_eval, and the caller
writes them in the reference's order.  `rng` is any object with poly(n) -> a ResidentPoly or (n, 32) uint8 array the callee
keeps, and scalar() -> int.
"""
from __future__ import annotations

import ctypes
from typing import List, NamedTuple, Optional, Tuple

import numpy as np

from . import lib as _l
from .evaluator import Ast
from .multiopen import ProverQuery
from .opening import _scale_add
from .poly import Blind, EvaluationDomain, Params, ResidentPoly, _handles, eval_polynomial_resident, freed_on_failure


def vanishing_quotient_resident(domain: EvaluationDomain, h_ext: ResidentPoly, out: Optional[List[ResidentPoly]] = None) -> List[ResidentPoly]:
    """`divide_by_vanishing_poly`, `extended_to_coeff` and `chunks_exact(n)` (vanishing/prover.rs:84-100) of the extended-domain
    evaluations `h_ext` in one device call (h2_poly_vanishing_quotient): the quotient_poly_degree pieces of n coefficients.
    `h_ext` is only read.  out=None allocates the pieces (and frees them again if the call fails)."""
    with freed_on_failure() as fresh:
        pieces = [fresh.keep(ResidentPoly(domain.field, domain.n)) for _ in range(domain.quotient_poly_degree)] if out is None else list(out)
        t = _l.fe_array(domain.t_evaluations, domain.m)
        _l.check(_l.init().h2_poly_vanishing_quotient(
            _handles(pieces), ctypes.c_size_t(len(pieces)), h_ext._h, ctypes.c_uint32(domain.k), ctypes.c_uint32(domain.extended_k),
            _l.ptr(_l.fe_bytes(domain.extended_omega_inv)), _l.ptr(_l.fe_bytes(domain.extended_ifft_divisor)),
            _l.ptr(_l.fe_bytes(domain.g_coset)), _l.ptr(t), ctypes.c_uint32(len(domain.t_evaluations)), _l.REPR_CANONICAL))
    return pieces


class Committed(NamedTuple):
    """vanishing::prover::Committed (:23-26): the random polynomial (coefficient form, n coefficients) and its blind."""
    random_poly: ResidentPoly
    random_blind: int

    def construct(self, params: Params, domain: EvaluationDomain, evaluator, expressions, y: int, rng) -> Tuple["Constructed", np.ndarray]:
        """Committed::construct (:65-122): h(X) = Ast.distribute_powers(expressions, y) evaluated once on the extended
        `evaluator`, divided, transformed back and split in one h2_poly_vanishing_quotient call; then quotient_poly_degree
        rng.scalar() blinds and one commitment pass of every piece.  Returns (Constructed, the (pieces, 64) affine commitments
        in the order the reference writes them).  The extended h(X) is freed before returning, and nothing stays allocated
        when the call fails."""
        h_ext = ResidentPoly(domain.field, domain.extended_len())
        try:
            evaluator.evaluate(Ast.distribute_powers(list(expressions), y), out=h_ext)
            pieces = vanishing_quotient_resident(domain, h_ext)
        finally:
            h_ext.close()
        with freed_on_failure() as fresh:
            fresh.extend(pieces)
            blinds = [rng.scalar() for _ in pieces]
            cm = params.commit_resident_affine(pieces, [Blind(b) for b in blinds])
        return Constructed(pieces, blinds, self), cm

    def close(self) -> None:
        self.random_poly.close()


class Constructed(NamedTuple):
    """vanishing::prover::Constructed (:28-32): the pieces of h(X) in coefficient form, their blinds, and Committed."""
    h_pieces: List[ResidentPoly]
    h_blinds: List[int]
    committed: Committed

    def evaluate(self, domain: EvaluationDomain, x: int) -> Tuple["Evaluated", int]:
        """Constructed::evaluate (:125-150): h_poly = sum_i h_pieces[i] x^(n i), folded from the last piece with one
        h2_poly_scale_add pass per piece, the blinds folded alike, and random_eval = random_poly(x), which the caller writes
        (:144-145).  Returns (Evaluated, random_eval)."""
        n, m = domain.n, domain.m
        xn = pow(int(x), n, m)
        with freed_on_failure() as fresh:
            h_poly = fresh.keep(ResidentPoly(domain.field, n))
            h_poly.copy_from(self.h_pieces[-1], n)
            for piece in reversed(self.h_pieces[:-1]):
                _scale_add(h_poly, xn, piece, 1, n)
            random_eval = eval_polynomial_resident([self.committed.random_poly], [int(x) % m], n=n)[0]
        h_blind = 0
        for b in reversed(self.h_blinds):
            h_blind = (h_blind * xn + b) % m
        return Evaluated(h_poly, h_blind, self.committed), random_eval

    def close(self) -> None:
        for p in self.h_pieces:
            p.close()
        self.committed.close()


class Evaluated(NamedTuple):
    """vanishing::prover::Evaluated (:34-37): h(X) folded into one polynomial of n coefficients, its blind, and Committed."""
    h_poly: ResidentPoly
    h_blind: int
    committed: Committed

    def open(self, x: int) -> List[ProverQuery]:
        """Evaluated::open (:156-175): h_poly with h_blind, then random_poly with random_blind, both at x."""
        return [ProverQuery(x, self.h_poly, Blind(self.h_blind)),
                ProverQuery(x, self.committed.random_poly, Blind(self.committed.random_blind))]

    def close(self) -> None:
        self.h_poly.close()
        self.committed.close()


def vanishing_commit(params: Params, domain: EvaluationDomain, rng) -> Tuple[Committed, np.ndarray]:
    """vanishing::Argument::commit (:38-60): the random polynomial from rng.poly(n), its blind from one rng.scalar(), and its
    commitment over g (params.commit, :53).  Returns (Committed, the (64,) affine commitment the caller writes)."""
    n = domain.n
    rp = rng.poly(n)
    with freed_on_failure() as fresh:
        rp = fresh.keep(rp if isinstance(rp, ResidentPoly) else ResidentPoly(domain.field, n, rp))
        blind = rng.scalar()
        cm = params.commit_resident_affine([rp], [Blind(blind)])[0]
    return Committed(rp, blind), cm
