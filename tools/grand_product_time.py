"""Time of the permutation and lookup product columns on the GPU: one call per argument (h2_poly_permutation_product /
h2_poly_lookup_product, csrc/grandproduct.cuh) against a composition of finer calls (tests/grand_product_cases.py: per
column set two Ast programs, batch_invert, running_product, the blinding rows uploaded, last_z read back to the host).

  python tools/grand_product_time.py [--ks 14,16,18,20] [--reps 5] [--out grand_product_time.json]

Shapes: the benchmark circuit's permutation (3 columns, chunk_len 3: 1 set), a wide permutation (16 columns, chunk_len 3:
6 sets, the last one partial) and 4 lookups, one proof each, blinding_factors = 5.  Each timed run starts from resident
inputs, allocates its z columns and ends in a device synchronise; medians of `reps` runs after one warm-up.  Every run's
z columns are compared byte for byte between the two paths.  The GPU's name and power limit are read in the same run."""
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
from oracle import cref, pasta  # noqa: E402
from tests.grand_product_cases import composition_lookup, composition_permutation  # noqa: E402

M = pasta.P_MOD
ZETA = pow(5, (M - 1) // 3, M)
DELTA = pow(5, 1 << 32, M)                                         # F::DELTA
BF = 5
SHAPES = [("benchmark", 3, 3), ("wide", 16, 3), ("lookups", 4, None)]


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


def flat(z):
    return [q for per in z for q in per] if z and isinstance(z[0], list) else list(z)


def run_shape(D, name, count, chunk_len, reps, seed):
    n = D.n
    beta, gamma = pasta.gen_scalars("fp", seed, 2)
    col = lambda s: h2.ResidentPoly("fp", n, cref.gen_scalars("fp", s, n))
    if chunk_len is None:                                            # `count` lookups
        ins = [tuple(col(seed + 10 + 4 * b + j) for j in range(4)) for b in range(count)]
        blinding = pasta.gen_scalars("fp", seed + 1, count * BF)
        new = lambda: h2.lookup_product_resident(D, [ins], beta, gamma, BF, blinding)
        old = lambda: composition_lookup(h2, D, ins, beta, gamma, BF, blinding)
        inputs = [p for lk in ins for p in lk]
    else:                                                            # a permutation of `count` columns
        sig = [col(seed + 10 + c) for c in range(count)]
        cols = [[col(seed + 100 + c) for c in range(count)]]
        blinding = pasta.gen_scalars("fp", seed + 1, -(-count // chunk_len) * BF)
        new = lambda: h2.permutation_product_resident(D, cols, sig, beta, gamma, DELTA, chunk_len, BF, blinding)
        old = lambda: composition_permutation(h2, D, cols, sig, beta, gamma, DELTA, chunk_len, BF, blinding)
        inputs = sig + cols[0]
    t_new, t_old = [], []
    for r in range(reps + 1):                                        # run 0 warms both paths up
        for fn, acc in ((new, t_new), (old, t_old)):
            t, z = timed(fn)
            if r:
                acc.append(t)
            if fn is new:
                z_new = flat(z)
            else:
                z_old = flat(z)
        if not all((a.download() == b.download()).all() for a, b in zip(z_new, z_old)) or len(z_new) != len(z_old):
            raise SystemExit(f"{name}: the z columns differ from the composition's")
        for p in z_new + z_old:
            p.close()
    for p in inputs:
        p.close()
    return {"shape": name, "columns": len(z_new), "one_call_ms": 1e3 * statistics.median(t_new), "composition_ms": 1e3 * statistics.median(t_old),
            "one_call_all_ms": [round(1e3 * t, 3) for t in t_new], "composition_all_ms": [round(1e3 * t, 3) for t in t_old]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="14,16,18,20")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    L.init()
    info = gpu_info()
    print(json.dumps({"gpu": info}), flush=True)
    rows = []
    for k in (int(x) for x in a.ks.split(",")):
        D = h2.EvaluationDomain("fp", 5, k, ZETA)
        for i, (name, count, chunk_len) in enumerate(SHAPES):
            r = {"k": k, **run_shape(D, name, count, chunk_len, a.reps, 0x5449 + 100 * k + i)}
            print(json.dumps(r), flush=True)
            rows.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
