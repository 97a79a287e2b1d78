"""What a proof's vanishing argument leaves behind, for the vanishing tests: record() runs a prover -- create_proof_engine,
whose own lines build the random polynomial, h(X) and its pieces, or tests/arguments_cases.create_proof_package, which
takes them from halo2_b200.vanishing's vanishing_commit / construct / evaluate / open -- and returns the points and scalars
it wrote, its proof bytes, and the last two queries (h_poly with h_blind, random_poly with random_blind) as bytes."""
from __future__ import annotations

import numpy as np

from tests import prover_replay as R


def record(h2, modulus: int, prove) -> dict:
    """Runs prove(eng, transcript), a prover with every other argument bound, over `eng`: the package `h2` with
    multiopen.create_proof recording its queries."""
    rec = {"points": [], "scalars": [], "queries": []}

    class T(R.Blake2bTranscript):
        def write_point(self, xy):
            rec["points"].append(np.array(xy, dtype=np.uint8).reshape(64).copy())
            super().write_point(xy)

        def write_scalar(self, v):
            rec["scalars"].append(int(v))
            super().write_scalar(v)

    class Multiopen:
        def __getattr__(self, name):
            return getattr(h2.multiopen, name)

        def create_proof(self, params_, rng_, transcript, queries):
            rec["queries"] = [(q.point, q.poly.download(), q.blind.value) for q in queries[-2:]]
            return h2.multiopen.create_proof(params_, rng_, transcript, queries)

    class Eng:
        multiopen = Multiopen()

        def __getattr__(self, name):
            return getattr(h2, name)

    t = T(modulus)
    prove(Eng(), t)
    rec["proof"] = bytes(t.proof)
    return rec
