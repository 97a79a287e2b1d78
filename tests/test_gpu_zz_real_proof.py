"""GPU test (runs last): a REAL PLONK proof of the reference's own test circuit (halo2_proofs/tests/plonk_api.rs:21-420, k = 5,
two instances) is produced ON THE DEVICE by plonk::create_proof composed from the engine's reference-facing API
(tests/plonk_prover.create_proof_engine: the instance and advice commitments, the lookups' permuted and product columns, the
permutation products, the vanishing argument, the arguments' construct / evaluate / open, the multi-point opening and the
opening argument) under the reference's GOLDEN verifying key -- the same 4 160 bytes as the oracle's prover with the same randomness --
and is accepted by the engine's verifier and by the restated reference verifier that the reference's sixteen golden proofs pin.

This composition was validated without a GPU (tests/test_real_proof.py: the same code over the ABI stand-in, device bodies on the
host emulation, identical bytes); every entry point it calls has its own GPU parity test."""
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests import multiopen_cases as MC  # noqa: E402
from tests import plonk_api_circuit as circ  # noqa: E402
from tests import plonk_prover as PP  # noqa: E402
from tests import plonk_verifier as PV  # noqa: E402
from tests import prover_replay as R  # noqa: E402


def test_real_proof_on_the_device():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    c = pasta.VESTA
    vk = PV.PinnedKey(circ.CASE["key_text"])
    prm = halo2_b200.Params.new("vesta", 5)                          # Params::<EqAffine>::new(5) on the device
    try:
        gens = (prm.g, prm.g_lagrange, prm.w, prm.u)
        P = pasta.Params.from_generators(c, 5, [cref.bytes_to_affine(x) for x in prm.g], cref.bytes_to_affine(prm.w[0]), cref.bytes_to_affine(prm.u[0]))
        fixed = circ.fixed_columns(circ.M, circ.ZETA)
        sigma = circ.permutation_columns(circ.M, vk.omega, circ.DELTA)
        inst = [[[2]], [[2]]]
        want = circ.prove((c, P, vk, fixed, sigma, gens), [circ.witness(), circ.witness()], inst, 777)
        T = R.Blake2bTranscript(circ.M)
        PP.create_proof_engine(halo2_b200, prm, vk, fixed, sigma, [circ.witness(), circ.witness()], inst, MC.SeededRng("fp", 777, True), T, circ.ZETA, circ.DELTA)
        got = bytes(T.proof)
        assert len(got) == 4160
        assert got == want                                           # bit-identical to the oracle's proof
        earm = PV.EngineArm(halo2_b200, "vesta", 5, *gens)
        try:
            assert PV.verify_proof(earm, vk, got, inst, circ.DELTA)
            bad = bytearray(got)
            bad[2000] ^= 1
            assert not PV.verify_proof(earm, vk, bytes(bad), inst, circ.DELTA)
        finally:
            earm.close()
        assert PV.verify_proof(PV.OracleArm("vesta", 5, *gens), vk, got, inst, circ.DELTA)
        # a witness that breaks a gate: the device prover still runs, the verifier rejects
        T2 = R.Blake2bTranscript(circ.M)
        PP.create_proof_engine(halo2_b200, prm, vk, fixed, sigma, [circ.witness(break_row=5)], [[[2]]], MC.SeededRng("fp", 901, True), T2, circ.ZETA, circ.DELTA)
        assert not PV.verify_proof(PV.OracleArm("vesta", 5, *gens), vk, bytes(T2.proof), [[[2]]], circ.DELTA)
    finally:
        prm.close()


def test_benchmark_circuit_real_proof_on_the_device():
    """The reference's benchmark circuit (benches/plonk.rs, tests/bench_circuit.py) at k = 8: key generated on the device, a
    real proof through the engine's phase calls with the proving key's polynomials resident between two proofs (in a dict, as
    bench.py keeps them), THE SAME BYTES as the same prover on the C restatement (tests/plonk_prover.CrefProver), accepted by
    the engine's verifier -- the workload of bench.py's extra.create_proof_k14_real."""
    _benchmark_circuit_proofs(8)


def test_benchmark_circuit_k14_real_proof_on_the_device():
    """The same at bench.py's own k = 14."""
    _benchmark_circuit_proofs(14)


def _benchmark_circuit_proofs(k):
    import os

    import halo2_b200 as h2
    from halo2_b200 import lib as L
    from tests import bench_circuit as BC
    L.init()
    n = 1 << k
    m = circ.M
    pts = cref.gen_points("vesta", 99, n + 2)
    g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    gl = h2.lagrange_generators("vesta", k, g)
    prm = h2.Params("vesta", k, g, gl, w, u=u)
    pk = {}
    try:
        D = h2.EvaluationDomain("fp", BC.DEGREE, k, circ.ZETA)
        fixed, sigma, adv = BC.columns(k, m, D.omega, circ.DELTA, circ.A_SMALL * circ.ZETA % m)
        fb, sb, ab = ([cref.ints_to_bytes(c_) for c_ in cols] for cols in (fixed, sigma, adv))
        xy = lambda col: cref.bytes_to_affine(h2.batch_normalize(prm.commit_lagrange(col, h2.Blind(1)).reshape(1, 96), "vesta")[0])
        vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, pasta.Q_MOD, m, D.omega, [xy(c_) for c_ in fb], [xy(c_) for c_ in sb]))
        proofs = []
        for seed in (5, 6):
            T = R.Blake2bTranscript(m)
            PP.create_proof_engine(h2, prm, vk, fb, sb, [ab], [[]], MC.SeededRng("fp", seed, True), T, circ.ZETA, circ.DELTA, pk=pk)
            proofs.append(bytes(T.proof))
        cp = PP.CrefProver(cref, "vesta", "fp", g, gl, w, u, os.cpu_count() or 1)
        Tc = R.Blake2bTranscript(m)
        cp.create_proof(vk, fb, sb, [ab], [[]], MC.SeededRng("fp", 6, True), Tc, circ.ZETA, circ.DELTA)
        assert proofs[1] == bytes(Tc.proof) and proofs[0] != proofs[1]
        arm = PV.EngineArm(h2, "vesta", k, params=prm)
        assert PV.verify_proof(arm, vk, proofs[0], [[]], circ.DELTA) and PV.verify_proof(arm, vk, proofs[1], [[]], circ.DELTA)
        bad = bytearray(proofs[1])
        bad[len(bad) // 3] ^= 8
        assert not PV.verify_proof(arm, vk, bytes(bad), [[]], circ.DELTA)
    finally:
        PP.close_proving_key(pk)
        prm.close()
