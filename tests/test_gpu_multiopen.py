"""GPU tests of the multi-point opening argument through the engine (halo2_b200.multiopen / opening on resident polynomials):
the reference's `test_roundtrip` and `test_identical_queries` (poly/multiopen.rs:278-481), a PLONK-shaped query list with
rotations -- the same proof bytes as the oracle's restatement of poly/multiopen/prover.rs at the small sizes, accepted by the
engine's verifier and by the restated reference verifier, wrong evaluations / commitments / flipped bits rejected -- and a
k = 12 round trip."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests import multiopen_cases as MC  # noqa: E402
from tests import prover_replay as R  # noqa: E402

SEED = MC.SEED


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


def test_roundtrip_and_identical_queries_device(eng):
    """multiopen.rs:278-373, :375-481 with Params::<EqAffine>::new(4) derived on the device."""
    prm = eng.Params.new("vesta", 4)
    g, gl, w, u = prm.g, prm.g_lagrange, prm.w, prm.u
    prm.close()
    side = MC.EngineSide(eng, "vesta", 4, g, w, u, g_lagrange=gl)
    try:
        got = MC.roundtrip(side, "fp")
        want = MC.roundtrip(MC.OracleSide("vesta", 4, g, w, u), "fp")
        assert got == want
        p = eng.ResidentPoly("fp", 16, cref.ints_to_bytes(list(range(16))))
        with pytest.raises(ValueError):
            eng.multiopen.create_proof(side.params, MC.SeededRng("fp", 1, True), R.Blake2bTranscript(),
                                       [eng.multiopen.ProverQuery(5, p, eng.Blind(1)), eng.multiopen.ProverQuery(5, p, eng.Blind(1))])
        p.close()
    finally:
        side.close()


@pytest.mark.parametrize("curve,k", [("vesta", 3), ("pallas", 2), ("vesta", 12)])
def test_plonk_shaped_queries_device(eng, curve, k):
    c = pasta.CURVES[curve]
    n = 1 << k
    pts = cref.gen_points(curve, SEED + 1, n + 2)
    g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    polys, blinds, plan = MC.plonk_shaped(c.scalar, k, SEED + 40)
    esd = MC.EngineSide(eng, curve, k, g, w, u)
    try:
        proof = esd.prove(polys, blinds, plan, SEED + 50)
        assert len(proof) == 32 * (1 + 3 + 1 + 2 * k + 2)
        assert esd.prove(polys, blinds, plan, SEED + 50) == proof          # again: pooled buffers, replayed graphs
        ec = [esd.commit(p, b) for p, b in zip(polys, blinds)]
        good = MC.evals_for(c.scalar, polys, plan)
        assert esd.verify(proof, ec, good)
        if k <= 3:                                                         # the oracle's prover writes the same bytes; its verifier agrees
            osd = MC.OracleSide(curve, k, g, w, u)
            assert osd.prove(polys, blinds, plan, SEED + 50) == proof
            oc = [osd.commit(p, b) for p, b in zip(polys, blinds)]
            assert [cref.bytes_to_affine(x) for x in ec] == oc
            assert osd.verify(proof, oc, good)
        for j in (0, 3, 5, 7):
            bad = list(good)
            bad[j] = (bad[j][0], bad[j][1], (bad[j][2] + 1) % c.r)
            assert not esd.verify(proof, ec, bad), j
        assert not esd.verify(proof, [ec[1], ec[0]] + ec[2:], good)
        flip = bytearray(proof)
        flip[32 * 2 + 1] ^= 4
        assert not esd.verify(bytes(flip), ec, good)
        # CommitmentReference::MSM (verifier.rs:62-66): column 1 as 2 * half + 3 * column 0
        r = c.r
        half = [(p1 - 3 * p0) * pow(2, -1, r) % r for p0, p1 in zip(polys[0], polys[1])]
        hc = esd.commit(half, (blinds[1] - 3 * blinds[0]) * pow(2, -1, r) % r)
        m_e = eng.MSM(esd.params)
        m_e.append_term(2, hc)
        m_e.append_term(3, ec[0])
        assert esd.verify(proof, [ec[0], m_e] + ec[2:], good)
        with pytest.raises(eng.VerifyError):
            esd.verify(proof[:32 * 3], ec, good)                           # the proof ends inside the q evaluations: SamplingError
    finally:
        esd.close()
