"""GPU test: the proof-shaped replay of create_proof's hot path (tests/prover_replay.py) produces THE SAME PROOF BYTES through
the engine (device-resident polynomials, fixed-base MSMs over the resident generators, fold-free IPA rounds) and through the
C restatement of the reference algorithm, with the reference's Blake2b transcript (transcript.rs:160-219) in both arms and
the challenges fed back into the computation.  BASELINE.json's north star: "bit-identical proof transcripts".
k = 14 and 16 are the sizes bench.py replays; from k = 16 the opening's rounds accumulate with a thread per work item and the
evaluations run 4-level reduction trees."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests import prover_replay as R  # noqa: E402

SEED = 0x48414C4F32


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


@pytest.mark.parametrize("k,real_params", [(5, True), (8, False), (10, False), (14, False), (16, False), (17, False)])
def test_replay_transcript_identical(eng, k, real_params):
    n = 1 << k
    c = pasta.VESTA
    if real_params:      # Params::new(5) proper: hash_to_curve generators, g_lagrange by EC-iFFT, all on the device
        prm = eng.Params.new("vesta", k)
        g, gl, w, u = prm.g, prm.g_lagrange, prm.w, prm.u
        prm.close()
    else:
        pts = cref.gen_points("vesta", SEED + 1, n + 2)
        g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
        gl = eng.lagrange_generators("vesta", k, g)
    inp = R.replay_inputs(cref, k, SEED + k)
    omega = pasta.omega_for_k("fp", k)
    cpu = R.CpuArm(cref, pasta, k, g, gl, w, u, threads=8)
    want = R.run(cpu, inp, k, omega)
    gpu = R.GpuArm(eng, k, g, gl, w, u)
    try:
        got = R.run(gpu, inp, k, omega)
        gpu.free()
        again = R.run(gpu, inp, k, omega)        # second pass: pooled buffers, replayed graphs
    finally:
        gpu.close()
    # 3 + 1 + 1 + 4 + 1 + 1 + 2k points, 14 + 2 + 2 scalars
    assert len(want) == 32 * (11 + 2 * k) + 32 * 18
    assert got == want
    assert again == want
    # a different seed gives a different proof (the check is not vacuous)
    inp2 = R.replay_inputs(cref, k, SEED + k + 1)
    assert R.run(cpu, inp2, k, omega) != want
