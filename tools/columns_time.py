"""Time of the instance / advice columns' domain transforms on the GPU: lagrange_to_coeff then coeff_to_extended of `count`
resident columns, one call per column per step (this tool's own per-column composition) against one column-batched call
per step (h2_poly_lagrange_to_coeff_batch / h2_poly_coeff_to_extended_batch).

  python tools/columns_time.py [--cases 11x10,14x1,14x4,14x16,17x1,...] [--reps 7] [--out columns_time.json]

A case KxC is C columns of 2^K rows with extended_k = K + 3 for K = 11 (the reference's stored k = 11 proofs: extended_k = 14),
else K + 2 (the benchmark circuit's degree 5).  Each timed run starts from resident Lagrange columns and ends in a device
synchronise; the two arms alternate, medians of `reps` runs after one warm-up of each, and the last run's outputs of the two
arms are compared byte for byte.  The GPU's name and power limit are read in the same run."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_CASES = "11x10," + ",".join(f"{k}x{c}" for k in (14, 17, 20) for c in (1, 4, 16))


def gpu_info(L):
    q = subprocess.run(["nvidia-smi", "-i", str(L._inited_device or 0), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    f = [x.strip() for x in q.stdout.strip().split(",")]
    return {"name": f[0], "power_limit": f[1], "sm_max_clock": f[2]} if len(f) == 3 else {"raw": q.stdout.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=DEFAULT_CASES)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch
    import halo2_b200 as h2
    from halo2_b200 import lib as L
    from oracle import cref, pasta
    if not torch.cuda.is_available():
        raise SystemExit("columns_time.py needs a GPU")
    L.init(0)
    info = gpu_info(L)
    print(json.dumps({"gpu": info}), flush=True)
    rows = []
    for case in a.cases.split(","):
        k, count = (int(x) for x in case.split("x"))
        ext_k = k + (3 if k == 11 else 2)
        D = h2.EvaluationDomain("fp", (1 << (ext_k - k)) + 1, k, pasta.zeta_candidates("fp")[0])
        assert D.extended_k == ext_k
        vals = [h2.ResidentPoly("fp", D.n, cref.gen_scalars("fp", 0xC0 + 97 * k + c, D.n)) for c in range(count)]
        arms = {}
        for name in ("per_column", "batched"):
            arms[name] = ([h2.ResidentPoly("fp", D.n) for _ in range(count)], [h2.ResidentPoly("fp", D.extended_len()) for _ in range(count)])

        def per_column():
            P, E = arms["per_column"]
            for v, p, e in zip(vals, P, E):
                D.lagrange_to_coeff_resident(v, out=p)
                D.coeff_to_extended_resident(p, out=e)

        def batched():
            P, E = arms["batched"]
            D.lagrange_to_coeff_batch_resident(vals, out=P)
            D.coeff_to_extended_batch_resident(P, out=E)

        fns = {"per_column": per_column, "batched": batched}
        times = {name: [] for name in fns}
        for r in range(a.reps + 1):
            for name, fn in fns.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                if r:
                    times[name].append(time.perf_counter() - t0)
        digest = {}
        for name, (P, E) in arms.items():
            h = hashlib.sha256()
            for p in P:
                h.update(p.download().tobytes())
            for e in E:
                h.update(e.download().tobytes())
            digest[name] = h.hexdigest()
        row = {"k": k, "extended_k": ext_k, "columns": count,
               "per_column_ms": round(1e3 * statistics.median(times["per_column"]), 4),
               "batched_ms": round(1e3 * statistics.median(times["batched"]), 4),
               "per_column_all_ms": [round(1e3 * x, 4) for x in times["per_column"]],
               "batched_all_ms": [round(1e3 * x, 4) for x in times["batched"]],
               "identical": digest["per_column"] == digest["batched"]}
        row["speedup"] = round(row["per_column_ms"] / row["batched_ms"], 3)
        print(json.dumps(row), flush=True)
        rows.append(row)
        for p in vals + [q for P, E in arms.values() for q in P + E]:
            p.close()
        if not row["identical"]:
            raise SystemExit(f"outputs differ at {case}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
