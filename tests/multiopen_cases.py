"""Shared scenarios for the multi-point opening tests (test infrastructure): the reference's own test inputs
(poly/multiopen.rs:278-481) and a plonk-shaped query list with rotations, a seeded stand-in for the prover's RNG, and one
driver that runs prover and verifier through either the oracle or the engine's host mirror."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import cref, pasta
from tests import prover_replay as R

SEED = 0x48414C4F32


class SeededRng:
    """The draws multiopen::create_proof / commitment::create_proof make from their RNG, from the seeded generator of
    SURVEY.md section 8(d): scalar() -> int; poly(n) -> [int] (oracle) or an (n, 32) uint8 array (engine)."""

    def __init__(self, field: str, seed: int, as_bytes: bool):
        self.field, self.seed, self.as_bytes, self.i = field, seed, as_bytes, 0

    def scalar(self) -> int:
        self.i += 1
        return cref.bytes_to_ints(cref.gen_scalars(self.field, self.seed + self.i, 1))[0]

    def poly(self, n: int):
        self.i += 1
        b = cref.gen_scalars(self.field, self.seed + self.i, n)
        return b if self.as_bytes else cref.bytes_to_ints(b)


class RecordingRng:
    """Passes every draw through and keeps the scalars drawn."""

    def __init__(self, inner):
        self.inner, self.draws = inner, []

    def scalar(self):
        x = self.inner.scalar()
        self.draws.append(x)
        return x

    def poly(self, n):
        return self.inner.poly(n)


class ReplayRng:
    """Gives back recorded scalar draws in order."""

    def __init__(self, draws):
        self.draws = list(draws)

    def scalar(self):
        return self.draws.pop(0)


def reference_roundtrip_polys(n: int):
    """multiopen.rs:294-307: ax = 10 + i, bx = 100 + i, cx = 100 + i."""
    return [10 + i for i in range(n)], [100 + i for i in range(n)], [100 + i for i in range(n)]


def plonk_shaped(field: str, k: int, seed: int):
    """Four columns queried the way a PLONK prover queries (rotations share points): returns (polys, blinds, [(poly index, point)]).
    Sets that arise: {x, x w} (columns 0 and 3 -- queried in different orders), {x}, {x, x w, x w^-1}."""
    m = pasta.FIELDS[field]
    n = 1 << k
    polys = [cref.bytes_to_ints(cref.gen_scalars(field, seed + i, n)) for i in range(4)]
    blinds = cref.bytes_to_ints(cref.gen_scalars(field, seed + 10, 4))
    x = cref.bytes_to_ints(cref.gen_scalars(field, seed + 11, 1))[0]
    w = pasta.omega_for_k(field, k)
    xw, xwi = x * w % m, x * pow(w, -1, m) % m
    plan = [(0, x), (1, x), (2, x), (0, xw), (2, xw), (2, xwi), (3, xw), (3, x)]
    return polys, blinds, plan


class OracleSide:
    """Prover and verifier through oracle/pasta.py."""

    def __init__(self, curve: str, k: int, g, w, u):
        self.c = pasta.CURVES[curve]
        self.k, self.curve = k, curve
        self.g, self.w, self.u = [cref.bytes_to_affine(x) for x in g], cref.bytes_to_affine(np.asarray(w).reshape(64)), cref.bytes_to_affine(np.asarray(u).reshape(64))

    def commit(self, poly, blind):
        return pasta.to_affine(self.c, pasta.best_multiexp(self.c, list(poly) + [blind], self.g + [self.w]))

    def prove(self, polys, blinds, plan, rng_seed) -> bytes:
        W = R._WriteT(self.c.r)
        qs = [pasta.ProverQuery(pt, polys[i], blinds[i]) for i, pt in plan]
        pasta.multiopen_create_proof(self.c, self.g, self.w, self.u, SeededRng(self.c.scalar, rng_seed, False), W, qs)
        return bytes(W.T.proof)

    def verify(self, proof: bytes, commitments, plan_with_evals):
        """plan_with_evals: [(commitment index, point, eval)]; returns the final msm.eval()."""
        T = R.Blake2bRead(proof, lambda b32: cref.affines_to_bytes([pasta.decompress(self.c, b32)])[0], self.c.r)
        qs = [pasta.VerifierQuery.new_commitment(commitments[i], pt, ev) for i, pt, ev in plan_with_evals]
        guard = pasta.multiopen_verify_proof(self.k, R._TupleTranscript(T, cref), qs, pasta.MSM(self.c, self.g, self.w, self.u))
        assert T.pos == len(proof)
        return guard.use_challenges().eval()


class EngineSide:
    """Prover and verifier through halo2_b200.multiopen (the CUDA library, or tests/fake_engine.py standing in for its ABI)."""

    def __init__(self, eng, curve: str, k: int, g, w, u, g_lagrange=None):
        self.eng, self.curve, self.k = eng, curve, k
        self.c = pasta.CURVES[curve]
        self.params = eng.Params(curve, k, g, g if g_lagrange is None else g_lagrange, w, u=u)

    def commit(self, poly, blind) -> np.ndarray:
        p = self.eng.ResidentPoly(self.c.scalar, 1 << self.k, cref.ints_to_bytes(poly))
        try:
            return self.params.commit_resident_affine([p], [self.eng.Blind(blind)])[0]
        finally:
            p.close()

    def prove(self, polys, blinds, plan, rng_seed) -> bytes:
        eng = self.eng
        W = R.Blake2bTranscript(self.c.r)
        res = [eng.ResidentPoly(self.c.scalar, 1 << self.k, cref.ints_to_bytes(p)) for p in polys]
        try:
            qs = [eng.multiopen.ProverQuery(pt, res[i], eng.Blind(blinds[i])) for i, pt in plan]
            eng.multiopen.create_proof(self.params, SeededRng(self.c.scalar, rng_seed, True), W, qs)
            for r_, p in zip(res, polys):                        # the prover leaves the caller's polynomials as they were
                assert cref.bytes_to_ints(r_.download()) == [x % self.c.r for x in p]
        finally:
            for r_ in res:
                r_.close()
        return bytes(W.proof)

    def verify(self, proof: bytes, commitments, plan_with_evals):
        eng = self.eng
        T = R.Blake2bRead(proof, lambda b32: eng.decompress_points(np.frombuffer(b32, dtype=np.uint8).reshape(1, 32), self.curve)[0], self.c.r)
        qs = [eng.multiopen.VerifierQuery.new_commitment(commitments[i], pt, ev) for i, pt, ev in plan_with_evals]
        guard = eng.multiopen.verify_proof(self.params, T, qs, eng.MSM(self.params))
        assert T.pos == len(proof)
        msm = guard.use_challenges()
        try:
            return msm.eval()
        finally:
            msm.close()

    def close(self):
        self.params.close()


def evals_for(field: str, polys, plan):
    m = pasta.FIELDS[field]
    return [(i, pt, pasta.eval_polynomial_mod(m, polys[i], pt)) for i, pt in plan]


def roundtrip(side, field):
    """multiopen.rs:278-373 and :375-481 on `side`."""
    m = pasta.FIELDS[field]
    n = 1 << side.k
    ax, bx, cx = reference_roundtrip_polys(n)
    blind, x, y, bvx_bad = cref.bytes_to_ints(cref.gen_scalars(field, SEED + 20, 4))
    a, b, c = (side.commit(p, blind) for p in (ax, bx, cx))
    avx, bvx, cvy = (pasta.eval_polynomial_mod(m, p, pt) for p, pt in ((ax, x), (bx, x), (cx, y)))
    polys = [ax, bx, cx]
    proof = side.prove(polys, [blind] * 3, [(0, x), (1, x), (2, y)], SEED + 30)
    assert not side.verify(proof, [a, b, c], [(0, x, avx), (1, x, avx), (2, y, cvy)])        # "NB: wrong!" (:347): should fail
    assert side.verify(proof, [a, b, c], [(0, x, avx), (1, x, bvx), (2, y, cvy)])            # should succeed (:360-371)
    # test_identical_queries (:464-479): the same commitment at the same point with two different evaluations
    VerifyError = pasta.VerifyError if isinstance(side, OracleSide) else side.eng.VerifyError
    with pytest.raises(VerifyError):
        side.verify(proof, [a, b, c], [(0, x, avx), (1, x, bvx_bad), (1, x, bvx), (2, y, cvy)])
    # bx and cx have the same coefficients but are different polynomials (different pointers): b == c as points, two queries
    assert np.array_equal(np.asarray(b), np.asarray(c)) if not isinstance(b, tuple) else b == c
    return proof
