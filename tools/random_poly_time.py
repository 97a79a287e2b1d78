"""Time of the prover's random polynomials drawn on the device (h2_poly_random, csrc/chacha.cuh) against what a patched Rust
prover does without it: draw n scalars on one host thread, then upload them.

  python tools/random_poly_time.py [--ks 14,16,18,20,22] [--proof-ks 18,20] [--reps 5] [--out random_poly_time.json]

Per k, n = 2^k draws:
  device    h2_poly_random into a resident polynomial, ending in a device synchronise;
  host      the C oracle's single-thread ChaCha20Rng + Field::random loop (oracle/chacha_oracle.c) plus the upload of its
            canonical bytes from pageable memory (h2_poly_upload).  A lower bound for OsRng, whose eight next_u64 per scalar
            each read the OS random source: this tool cannot measure that.
The two results are compared byte for byte.  Then whole proofs of the benchmark circuit (tests/bench_circuit.py) at
--proof-ks through tests/plonk_prover.create_proof_engine, the proving key resident between proofs, with the seeded host rng
of the test suite (tests/multiopen_cases.SeededRng: C-drawn polynomials, uploaded) and with halo2_b200.ChaCha20Rng, the
two alternating; timing only, their bytes differ.  Medians of `reps` runs after one warm-up.  The GPU's name and power
limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import halo2_b200 as h2  # noqa: E402
from halo2_b200 import lib as L  # noqa: E402
from halo2_b200.rng import fill_random  # noqa: E402
from oracle import chacha as C  # noqa: E402
from oracle import cref, pasta  # noqa: E402

SEED = bytes(range(0x20, 0x40))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", str(L._inited_device or 0), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    f = [x.strip() for x in q.stdout.strip().split(",")]
    return {"name": f[0], "power_limit": f[1], "sm_max_clock": f[2]} if len(f) == 3 else {"raw": q.stdout.strip()}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def draw_row(k, reps):
    n = 1 << k
    p = h2.ResidentPoly("fp", n)
    q = h2.ResidentPoly("fp", n)
    try:
        def host():
            b = C.draws("fp", SEED, 0, 16, n)
            q.upload(b)
            return b
        t_dev, t_host, t_cpu = [], [], []
        for r in range(reps + 1):                                    # run 0 warms both paths up
            t, _ = timed(lambda: fill_random([p], [n], SEED, 0, 16))
            t_dev.append(t)
            t0 = time.perf_counter()
            C.draws("fp", SEED, 0, 16, n)
            t_cpu.append(time.perf_counter() - t0)
            t, _ = timed(host)
            t_host.append(t)
        if not (p.download() == q.download()).all():
            raise SystemExit(f"k = {k}: the device draws differ from the oracle's")
    finally:
        p.close()
        q.close()
    med = lambda ts: 1e3 * statistics.median(ts[1:])                # noqa: E731
    return {"k": k, "draws": n, "device_ms": med(t_dev), "host_draw_ms": med(t_cpu), "host_draw_upload_ms": med(t_host),
            "device_all_ms": [round(1e3 * t, 3) for t in t_dev[1:]], "host_draw_upload_all_ms": [round(1e3 * t, 3) for t in t_host[1:]]}


def proof_row(k, reps):
    from tests import bench_circuit as BC
    from tests import multiopen_cases as MC
    from tests import plonk_api_circuit as circ
    from tests import plonk_prover as PP
    from tests import plonk_verifier as PV
    from tests import prover_replay as R
    n, m = 1 << k, circ.M
    pts = cref.gen_points("vesta", 99, n + 2)
    g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    prm = h2.Params("vesta", k, g, h2.lagrange_generators("vesta", k, g), w, u=u)
    pk = {}
    try:
        D = h2.EvaluationDomain("fp", BC.DEGREE, k, circ.ZETA)
        fixed, sigma, adv = BC.columns(k, m, D.omega, circ.DELTA, circ.A_SMALL * circ.ZETA % m)
        fb, sb, ab = ([cref.ints_to_bytes(c_) for c_ in cols] for cols in (fixed, sigma, adv))
        xy = lambda col: cref.bytes_to_affine(h2.batch_normalize(prm.commit_lagrange(col, h2.Blind(1)).reshape(1, 96), "vesta")[0])  # noqa: E731
        vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, pasta.Q_MOD, m, D.omega, [xy(c_) for c_ in fb], [xy(c_) for c_ in sb]))

        def prove(rng):
            T = R.Blake2bTranscript(m)
            PP.create_proof_engine(h2, prm, vk, fb, sb, [ab], [[]], rng, T, circ.ZETA, circ.DELTA, pk=pk)
            return bytes(T.proof)

        def seeded(i):
            return prove(MC.SeededRng("fp", 1000 + i, True))

        def device(i):
            with h2.ChaCha20Rng(SEED, "fp", stream=i) as rng:
                return prove(rng)
        t_seeded, t_device = [], []
        for r in range(reps + 1):
            for fn, acc in ((seeded, t_seeded), (device, t_device)):
                t, proof = timed(lambda: fn(r))
                acc.append(t)
        arm = PV.EngineArm(h2, "vesta", k, params=prm)
        accepted = PV.verify_proof(arm, vk, proof, [[]], circ.DELTA)
        arm.close()
    finally:
        PP.close_proving_key(pk)
        prm.close()
    med = lambda ts: 1e3 * statistics.median(ts[1:])                # noqa: E731
    return {"k": k, "proof_seeded_rng_ms": med(t_seeded), "proof_device_rng_ms": med(t_device), "device_rng_proof_accepted": bool(accepted),
            "seeded_all_ms": [round(1e3 * t, 1) for t in t_seeded[1:]], "device_all_ms": [round(1e3 * t, 1) for t in t_device[1:]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="14,16,18,20,22")
    ap.add_argument("--proof-ks", default="18,20")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    L.init()
    info = gpu_info()
    print(json.dumps({"gpu": info}), flush=True)
    rows = []
    for k in (int(x) for x in a.ks.split(",") if x):
        rows.append(draw_row(k, a.reps))
        print(json.dumps(rows[-1]), flush=True)
    for k in (int(x) for x in a.proof_ks.split(",") if x):
        rows.append(proof_row(k, a.reps))
        print(json.dumps(rows[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
