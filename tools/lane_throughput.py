"""Throughput of independent provers on one GPU, one prover lane each (halo2_b200.Lane; DESIGN.md section 9.1).

  python tools/lane_throughput.py [commit] [replay] [real] [--ks 14,16] [--real-ks 16,18] [--lanes 1,2,4,8] [--rounds 3]
                                  [--out results/lane_throughput.json]

Three workloads (commit and replay when none is named), each from 1, 2, 4 and 8 host threads, every thread bound to a lane
of its own:
  commit  a single commit of a 2^k host column against resident generators (h2_msm_registered_batch_affine, batch 1):
          a plain ctypes loop, so the GIL is released for the whole device call;
  replay  the proof-shaped k-replay of tests/prover_replay.py (GpuArm), whose host glue holds the GIL between calls;
  real    real proofs of the benchmark circuit through tests/plonk_prover.create_proof_engine, once with a private proving
          key per lane (each lane runs keygen_pk) and once with one key built on the primary context and shared
          (ProvingKey.share).  Besides the rate it reports the key's bytes, computed from its shapes, and the device's free
          memory (cudaMemGetInfo) before the keys exist and while they all do; other tenants of the GPU can move the latter.
Every result is checked: each commit against the same commit run serially on the primary context, each proof byte for byte
against a serial run with the same seed (for real: with a private key).  commit and replay alternate their runs -- 1 lane,
then N lanes, for every N, `rounds` times -- and report the medians; real runs every lane count once per key mode.  The
GPU's name and power limit are read in the same run."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import halo2_b200 as h2  # noqa: E402
from halo2_b200 import lib as L  # noqa: E402
from oracle import cref, pasta  # noqa: E402
from tests import prover_replay as R  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", str(L._inited_device or 0), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    f = [x.strip() for x in q.stdout.strip().split(",")]
    return {"name": f[0], "power_limit": f[1], "sm_max_clock": f[2]} if len(f) == 3 else {"raw": q.stdout.strip()}


def timed(nlanes, make, reps, warm=2, probe=None):
    """Runs make(i) -> step on nlanes threads, each on its own lane; every thread warms up with `warm` steps, then all run
    `reps` steps at once.  Returns steps per second over the wall time of the timed window.  probe(), when given, runs on
    the calling thread after the window, while every lane still holds what make() built."""
    start, done, held = threading.Barrier(nlanes + 1), threading.Barrier(nlanes + 1), threading.Barrier(nlanes + 1)
    t_end, errs = [0.0] * nlanes, []

    def run(i):
        try:
            with h2.Lane():
                step, close = make(i)
                try:
                    for _ in range(warm):
                        step()
                    start.wait()
                    for _ in range(reps):
                        step()
                    t_end[i] = time.perf_counter()
                    done.wait()
                    held.wait()
                finally:
                    close()
        except BaseException as e:  # noqa: BLE001
            errs.append(e)
            start.abort()
            done.abort()
            held.abort()
    th = [threading.Thread(target=run, args=(i,)) for i in range(nlanes)]
    for t in th:
        t.start()
    try:
        start.wait()
    except threading.BrokenBarrierError:
        pass
    t0 = time.perf_counter()
    try:
        done.wait()
        if probe:
            try:
                probe()
            except BaseException as e:  # noqa: BLE001
                errs.append(e)          # raised below, once the lanes have closed and joined
        held.wait()
    except threading.BrokenBarrierError:
        pass
    for t in th:
        t.join()
    if errs:
        raise next((e for e in errs if not isinstance(e, threading.BrokenBarrierError)), errs[0])
    return nlanes * reps / (max(t_end) - t0)


def commit_bench(k, lanes, rounds, reps):
    n = 1 << k
    lib = L.load()
    pts = cref.gen_points("vesta", 14 + k, n + 1)
    prm = h2.Params("vesta", k, pts[:n], pts[:n], pts[n:n + 1])
    cols = [cref.gen_scalars("fp", 100 * k + i, n) for i in range(max(lanes))]
    blind = np.stack([L.fe_bytes(12345)])
    want = [prm.commit_many_affine([c], [h2.Blind(12345)]) for c in cols]     # serially, on the primary context

    def make(i):
        out = np.zeros((1, 64), dtype=np.uint8)
        col = cols[i]

        def step():
            L.check(lib.h2_msm_registered_batch_affine(prm._h_g, L.ptr(col), ctypes.c_size_t(n), L.ptr(blind), ctypes.c_size_t(1),
                                                        L.REPR_CANONICAL, L.ptr(out)))
            if not (out == want[i]).all():
                raise AssertionError(f"commit k={k} lane {i}: result differs from the serial run")
        return step, lambda: None
    res = sweep(lanes, rounds, lambda nl: timed(nl, make, reps))
    prm.close()
    return res


def replay_bench(k, lanes, rounds, reps):
    n = 1 << k
    pts = cref.gen_points("vesta", 40 + k, n + 2)
    g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    gl = h2.lagrange_generators("vesta", k, g)
    omega = pasta.omega_for_k("fp", k)
    inputs = [R.replay_inputs(cref, k, 1000 * k + i) for i in range(max(lanes))]
    arm = R.GpuArm(h2, k, g, gl, w, u)
    want = []
    for inp in inputs:                                          # serially, on the primary context
        want.append(R.run(arm, inp, k, omega))
        arm.free()
    gv = R.GpuVerifierArm(h2, k, g, gl, w, u, params=arm.params)
    if not all(R.verify(gv, p, k, omega) for p in want[:2]):
        raise AssertionError("the serial proofs do not verify")
    arm.close()

    def make(i):
        a = R.GpuArm(h2, k, g, gl, w, u)

        def step():
            proof = R.run(a, inputs[i], k, omega)
            a.free()
            if proof != want[i]:
                raise AssertionError(f"replay k={k} lane {i}: proof differs from the serial replay")
        return step, a.close
    return sweep(lanes, rounds, lambda nl: timed(nl, make, reps))


def real_bench(k, lanes, reps):
    """Real proofs on N lanes, with a private key per lane and with one shared key.  Each lane proves with a seed of its
    own; every proof must equal the serial proof with that seed under a private key on the primary context."""
    import torch
    from tests import bench_circuit as BC
    from tests import multiopen_cases as MC
    from tests import plonk_api_circuit as circ
    from tests import plonk_prover as PP
    from tests import plonk_verifier as PV
    from tests.bench_circuit import bench_copies
    from tests.plonk_api_circuit import ZETA
    n, m = 1 << k, pasta.P_MOD
    delta = PV.scalar_delta(m)
    dev = L._inited_device or 0
    free = lambda: int(torch.cuda.mem_get_info(dev)[0])
    pts = cref.gen_points("vesta", 99, n + 2)
    prm = h2.Params("vesta", k, pts[:n], h2.lagrange_generators("vesta", k, pts[:n]), pts[n:n + 1], u=pts[n + 1:])
    D = h2.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
    fixed, _, adv = BC.columns(k, m, D.omega, delta, circ.A_SMALL * ZETA % m)
    ab = [cref.ints_to_bytes(c) for c in adv]
    cc = h2.CopyConstraints(n, 3)
    cc.extend(np.array(list(bench_copies(k)), dtype=np.uint32))
    fc, pc = h2.keygen_vk(prm, D, fixed, cc, delta)
    A = cref.bytes_to_affine
    vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, pasta.Q_MOD, m, D.omega, [A(x) for x in fc], [A(x) for x in pc]))
    keygen = lambda: h2.keygen_pk(prm, D, fixed, cc, delta, BC.BLINDING_FACTORS)

    def prove(pk, seed):
        T = R.Blake2bTranscript(m)
        PP.create_proof_engine(h2, prm, vk, None, None, [ab], [[]], MC.SeededRng("fp", seed, True), T, ZETA, delta, pk=pk)
        return bytes(T.proof)
    seeds = [3000 * k + i for i in range(max(lanes))]
    pk = keygen()
    want = [prove(pk, s) for s in seeds]                         # serially, private key, primary context
    key_bytes = 32 * sum(p.len + 1 for p in pk._all())           # len + 1 slots per resident polynomial
    arm = PV.EngineArm(h2, "vesta", k, params=prm)
    if not all(PV.verify_proof(arm, vk, p, [[]], delta) for p in want[:2]):
        raise AssertionError("the serial proofs do not verify")
    arm.close()
    pk.close()
    free()                                                        # torch's own context exists before the first reading
    res = {"key_bytes": key_bytes, "key_field_elements_per_n": round(key_bytes / 32 / n, 3)}
    for mode in ("private", "shared"):
        res[mode] = {}
        for nl in lanes:
            mem = {"free_before_keys": free()}
            shared = keygen().share() if mode == "shared" else None

            def make(i):
                key = shared or keygen()

                def step():
                    if prove(key, seeds[i]) != want[i]:
                        raise AssertionError(f"real k={k} {mode} lane {i}: proof differs from the serial proof")
                return step, (lambda: None) if shared else key.close
            rate = timed(nl, make, reps, warm=1, probe=lambda: mem.update(free_with_keys=free()))
            if shared:
                shared.close()
            mem["keys_and_lanes_bytes"] = mem["free_before_keys"] - mem["free_with_keys"]
            res[mode][str(nl)] = {"per_s": round(rate, 3), **mem}
            print(f"real k={k} {mode} {nl} lanes: " + json.dumps(res[mode][str(nl)]), flush=True)
    prm.close()
    return res


def sweep(lanes, rounds, run):
    """1 lane and N lanes alternated, `rounds` times; medians of the rates."""
    rates = {nl: [] for nl in lanes}
    for _ in range(rounds):
        for nl in lanes:
            if nl == 1:
                continue
            rates[1].append(run(1))
            rates[nl].append(run(nl))
    if len(lanes) == 1:
        rates[1] = [run(1) for _ in range(rounds)]
    med = {nl: statistics.median(v) for nl, v in rates.items()}
    return {str(nl): {"per_s": round(med[nl], 2), "speedup_vs_1": round(med[nl] / med[1], 3), "runs": [round(x, 2) for x in rates[nl]]}
            for nl in lanes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", help="commit, replay and / or real (default: commit replay)")
    ap.add_argument("--ks", default="14,16")
    ap.add_argument("--real-ks", default="16,18")
    ap.add_argument("--lanes", default="1,2,4,8")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--commit-reps", type=int, default=200)
    ap.add_argument("--replay-reps", type=int, default=6)
    ap.add_argument("--real-reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    a.workloads = a.workloads or ["commit", "replay"]
    if set(a.workloads) - {"commit", "replay", "real"}:
        ap.error("workloads are commit, replay and real")
    L.init()
    ks = [int(x) for x in a.ks.split(",")]
    lanes = sorted({1} | {int(x) for x in a.lanes.split(",")})
    res = {"gpu": gpu_info(), "lanes": lanes, "rounds": a.rounds}
    for w in a.workloads:
        res[w] = {}
    if "commit" in a.workloads:
        for k in ks:
            res["commit"][str(k)] = commit_bench(k, lanes, a.rounds, a.commit_reps)
            print(f"commit k={k}: " + json.dumps(res["commit"][str(k)]), flush=True)
    if "replay" in a.workloads:
        for k in ks:
            res["replay"][str(k)] = replay_bench(k, lanes, a.rounds, a.replay_reps)
            print(f"replay k={k}: " + json.dumps(res["replay"][str(k)]), flush=True)
    if "real" in a.workloads:
        for k in (int(x) for x in a.real_ks.split(",")):
            res["real"][str(k)] = real_bench(k, lanes, a.real_reps)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
