"""The instance and advice phases of plonk::create_proof two ways, for the column tests: create_proof_engine's per-column
composition (run up to its first challenge) and halo2_b200.instance_commit / advice_commit.  Both return the same record:
the points in transcript order and the bytes of every column's values, coefficient form and coset."""
from __future__ import annotations

import numpy as np

from oracle import cref, pasta
from tests import multiopen_cases as MC
from tests import plonk_prover as PP
from tests import prover_replay as R


class _Stop(Exception):
    pass


class ShapeKey:
    """What create_proof_engine reads from a key before its first challenge, for a circuit shape without a pinned key."""

    def __init__(self, field: str, k: int, degree: int, blinding_factors: int, zeta: int):
        self.scalar_modulus, self.k, self._deg, self._bf = pasta.FIELDS[field], k, degree, blinding_factors
        d = pasta.EvaluationDomain(field, degree, k, zeta)
        self.extended_k, self.omega = d.extended_k, d.omega

    def blinding_factors(self) -> int:
        return self._bf

    def degree(self) -> int:
        return self._deg

    def transcript_repr(self) -> int:
        return 0


def _skip_key():
    """A proving-key dict that makes create_proof_engine skip its keygen part (the phases here do not read it)."""
    return {"fixed_l": [], "fixed_p": [], "fixed_c": [], "sigma_l": [], "sigma_p": [], "sigma_c": [], "l": [None, None, None]}


def engine_phases(h2, prm, vk, advice, instances, seed: int, zeta: int) -> dict:
    """create_proof_engine through its instance and advice phases, under SeededRng(seed)."""
    field = {pasta.P_MOD: "fp", pasta.Q_MOD: "fq"}[vk.scalar_modulus]
    rec = {"common": [], "written": [], "values": [], "polys": [], "cosets": []}

    class D(h2.EvaluationDomain):
        def lagrange_to_coeff_resident(self, a, out=None):
            rec["values"].append(a.download(self.n))
            r = super().lagrange_to_coeff_resident(a, out)
            rec["polys"].append(r.download(self.n))
            return r

        def coeff_to_extended_resident(self, a, out=None):
            r = super().coeff_to_extended_resident(a, out)
            rec["cosets"].append(r.download(self.extended_len()))
            return r

    class Eng:
        EvaluationDomain = D

        def __getattr__(self, name):
            return getattr(h2, name)

    class T(R.Blake2bTranscript):
        def common_point(self, xy):
            rec["common"].append(np.array(xy, dtype=np.uint8).reshape(64))
            super().common_point(xy)

        def write_point(self, xy):
            rec["written"].append(np.array(xy, dtype=np.uint8).reshape(64))
            super().write_point(xy)

        def squeeze_challenge(self):
            raise _Stop()

    try:
        PP.create_proof_engine(Eng(), prm, vk, [], [], advice, instances, MC.SeededRng(field, seed, True), T(vk.scalar_modulus), zeta, 0,
                               pk=_skip_key())
    except _Stop:
        pass
    return rec


def batched_phases(h2, prm, vk, advice, instances, seed: int, zeta: int) -> dict:
    """instance_commit and advice_commit on the same inputs under SeededRng(seed); closes what they made."""
    field = {pasta.P_MOD: "fp", pasta.Q_MOD: "fq"}[vk.scalar_modulus]
    D = h2.EvaluationDomain(field, vk.degree(), vk.k, zeta)
    bf = vk.blinding_factors()
    inst = h2.instance_commit(prm, D, instances, bf)
    adv = h2.advice_commit(prm, D, advice, MC.SeededRng(field, seed, True), bf)
    rec = {"common": [c for s in inst for c in s.commitments], "written": [c for s in adv for c in s.commitments],
           "values": [], "polys": [], "cosets": []}
    for s in list(inst) + list(adv):
        rec["values"] += [p.download(D.n) for p in s.values]
        rec["polys"] += [p.download(D.n) for p in s.polys]
        rec["cosets"] += [p.download(D.extended_len()) for p in s.cosets]
        for p in s.values + s.polys + s.cosets:
            p.close()
    return rec


def assert_same(want: dict, got: dict) -> None:
    for key in ("common", "written", "values", "polys", "cosets"):
        assert len(want[key]) == len(got[key]), key
        for i, (a, b) in enumerate(zip(want[key], got[key])):
            assert np.array_equal(np.asarray(a, dtype=np.uint8), np.asarray(b, dtype=np.uint8)), (key, i)


def random_columns(field: str, seed: int, proofs: int, columns: int, n: int):
    return [[cref.gen_scalars(field, seed + 100 * p + c, n) for c in range(columns)] for p in range(proofs)]
