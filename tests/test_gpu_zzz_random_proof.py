"""GPU test (runs last): real proofs whose random polynomials are drawn on the device by halo2_b200.ChaCha20Rng
(h2_poly_random) equal, byte for byte, the proofs of the host provers drawing the same ChaCha20Rng stream
(oracle/chacha.HostChaCha20Rng): the benchmark circuit at k = 14 and 16 against the C restatement's prover
(tests/plonk_prover.CrefProver), and the reference's plonk_api circuit against the big-integer oracle prover.  Both verifiers
accept, and a flipped bit is rejected."""
import os

import pytest

pytestmark = pytest.mark.gpu

from oracle import chacha as C  # noqa: E402
from oracle import cref, pasta  # noqa: E402
from tests import plonk_api_circuit as circ  # noqa: E402
from tests import plonk_prover as PP  # noqa: E402
from tests import plonk_verifier as PV  # noqa: E402
from tests import prover_replay as R  # noqa: E402


def test_plonk_api_proof_with_the_device_rng():
    import halo2_b200 as h2
    from halo2_b200 import lib as L
    L.init()
    c = pasta.VESTA
    vk = PV.PinnedKey(circ.CASE["key_text"])
    prm = h2.Params.new("vesta", 5)
    try:
        gens = (prm.g, prm.g_lagrange, prm.w, prm.u)
        P = pasta.Params.from_generators(c, 5, [cref.bytes_to_affine(x) for x in prm.g], cref.bytes_to_affine(prm.w[0]), cref.bytes_to_affine(prm.u[0]))
        fixed = circ.fixed_columns(circ.M, circ.ZETA)
        sigma = circ.permutation_columns(circ.M, vk.omega, circ.DELTA)
        inst, seed = [[[2]], [[2]]], bytes(range(7, 39))
        W = R._WriteT(circ.M)
        PP.create_proof(c, P.g, P.g_lagrange, P.w, P.u, vk, fixed, sigma, [circ.witness(), circ.witness()], inst, C.HostChaCha20Rng(seed, "fp", False),
                        W, circ.ZETA, circ.DELTA)
        want = bytes(W.T.proof)
        T = R.Blake2bTranscript(circ.M)
        with h2.ChaCha20Rng(seed, "fp") as rng:
            PP.create_proof_engine(h2, prm, vk, fixed, sigma, [circ.witness(), circ.witness()], inst, rng, T, circ.ZETA, circ.DELTA)
        got = bytes(T.proof)
        assert len(got) == 4160 and got == want
        earm = PV.EngineArm(h2, "vesta", 5, *gens)
        try:
            assert PV.verify_proof(earm, vk, got, inst, circ.DELTA)
            bad = bytearray(got)
            bad[2000] ^= 1
            assert not PV.verify_proof(earm, vk, bytes(bad), inst, circ.DELTA)
        finally:
            earm.close()
        assert PV.verify_proof(PV.OracleArm("vesta", 5, *gens), vk, got, inst, circ.DELTA)
    finally:
        prm.close()


@pytest.mark.parametrize("k", [14, 16])
def test_benchmark_circuit_proof_with_the_device_rng(k):
    import halo2_b200 as h2
    from halo2_b200 import lib as L
    from tests import bench_circuit as BC
    L.init()
    n, m = 1 << k, circ.M
    pts = cref.gen_points("vesta", 99, n + 2)
    g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    gl = h2.lagrange_generators("vesta", k, g)
    prm = h2.Params("vesta", k, g, gl, w, u=u)
    pk = {}
    try:
        D = h2.EvaluationDomain("fp", BC.DEGREE, k, circ.ZETA)
        fixed, sigma, adv = BC.columns(k, m, D.omega, circ.DELTA, circ.A_SMALL * circ.ZETA % m)
        fb, sb, ab = ([cref.ints_to_bytes(c_) for c_ in cols] for cols in (fixed, sigma, adv))
        xy = lambda col: cref.bytes_to_affine(h2.batch_normalize(prm.commit_lagrange(col, h2.Blind(1)).reshape(1, 96), "vesta")[0])  # noqa: E731
        vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, pasta.Q_MOD, m, D.omega, [xy(c_) for c_ in fb], [xy(c_) for c_ in sb]))
        seed = bytes([k]) * 32
        T = R.Blake2bTranscript(m)
        with h2.ChaCha20Rng(seed, "fp", stream=5) as rng:
            PP.create_proof_engine(h2, prm, vk, fb, sb, [ab], [[]], rng, T, circ.ZETA, circ.DELTA, pk=pk)
        got = bytes(T.proof)
        cp = PP.CrefProver(cref, "vesta", "fp", g, gl, w, u, os.cpu_count() or 1)
        Tc = R.Blake2bTranscript(m)
        cp.create_proof(vk, fb, sb, [ab], [[]], C.HostChaCha20Rng(seed, "fp", True, stream=5), Tc, circ.ZETA, circ.DELTA)
        assert got == bytes(Tc.proof)
        arm = PV.EngineArm(h2, "vesta", k, params=prm)
        assert PV.verify_proof(arm, vk, got, [[]], circ.DELTA)
        bad = bytearray(got)
        bad[len(bad) // 3] ^= 8
        assert not PV.verify_proof(arm, vk, bytes(bad), [[]], circ.DELTA)
        arm.close()
        assert PV.verify_proof(PV.OracleArm("vesta", k, g, gl, w, u), vk, got, [[]], circ.DELTA)
    finally:
        PP.close_proving_key(pk)
        prm.close()
