"""Throughput of independent provers on one GPU, one prover lane each (halo2_b200.Lane; DESIGN.md section 9.1).

  python tools/lane_throughput.py [--ks 14,16] [--lanes 1,2,4,8] [--rounds 3] [--out results/lane_throughput.json]

Two workloads, each from 1, 2, 4 and 8 host threads, every thread bound to a lane of its own:
  commit  a single commit of a 2^k host column against resident generators (h2_msm_registered_batch_affine, batch 1):
          a plain ctypes loop, so the GIL is released for the whole device call;
  replay  the proof-shaped k-replay of tests/prover_replay.py (GpuArm), whose host glue holds the GIL between calls.
Every result is checked: each commit against the same commit run serially on the primary context, each proof byte for byte
against a serial replay with the same seed.  Runs are alternated -- 1 lane, then N lanes, for every N, `rounds` times -- and the
medians are reported, with the GPU's name and power limit read in the same run."""
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


def timed(nlanes, make, reps):
    """Runs make(i) -> step on nlanes threads, each on its own lane; every thread warms up with 2 steps, then all run `reps`
    steps at once.  Returns steps per second over the wall time of the timed window."""
    start, done = threading.Barrier(nlanes + 1), threading.Barrier(nlanes + 1)
    t_end, errs = [0.0] * nlanes, []

    def run(i):
        try:
            with h2.Lane():
                step, close = make(i)
                try:
                    step()
                    step()
                    start.wait()
                    for _ in range(reps):
                        step()
                    t_end[i] = time.perf_counter()
                    done.wait()
                finally:
                    close()
        except BaseException as e:  # noqa: BLE001
            errs.append(e)
            start.abort()
            done.abort()
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
    ap.add_argument("--ks", default="14,16")
    ap.add_argument("--lanes", default="1,2,4,8")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--commit-reps", type=int, default=200)
    ap.add_argument("--replay-reps", type=int, default=6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L.init()
    ks = [int(x) for x in a.ks.split(",")]
    lanes = sorted({1} | {int(x) for x in a.lanes.split(",")})
    res = {"gpu": gpu_info(), "lanes": lanes, "rounds": a.rounds, "commit": {}, "replay": {}}
    for k in ks:
        res["commit"][str(k)] = commit_bench(k, lanes, a.rounds, a.commit_reps)
        print(f"commit k={k}: " + json.dumps(res["commit"][str(k)]), flush=True)
    for k in ks:
        res["replay"][str(k)] = replay_bench(k, lanes, a.rounds, a.replay_reps)
        print(f"replay k={k}: " + json.dumps(res["replay"][str(k)]), flush=True)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
