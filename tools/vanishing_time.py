"""Time of the vanishing argument's quotient on the GPU: h(X) on the extended domain -> its quotient_poly_degree pieces of n
coefficients, the existing sequence (h2_poly_divide_by_vanishing in place, h2_poly_extended_to_coeff into a temporary of
n (d - 1) coefficients, d - 1 h2_poly_copy calls; the composition of tests/plonk_prover.create_proof_engine) against one
h2_poly_vanishing_quotient call.

  python tools/vanishing_time.py [--ks 11,14,17,20] [--degrees 3,5] [--reps 15] [--out vanishing_time.json]

d is the constraint system's degree (quotient_poly_degree = d - 1); every k runs with each of --degrees, and k = 14 also with
the benchmark circuit's own degree (tests/bench_circuit.DEGREE).  Both arms start from the same resident random extended
array: the existing sequence divides in place, so its input is restored from the source before each of its runs, outside
the timed window.  Each timed run ends in a device synchronise; the two arms alternate, medians of `reps` runs after one
warm-up of each, and the last run's pieces of the two arms are compared byte for byte.  The GPU's name and power limit are
read in the same run."""
import argparse
import hashlib
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.columns_time import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="11,14,17,20")
    ap.add_argument("--degrees", default="3,5")
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import halo2_b200 as h2
    from halo2_b200 import lib as L
    from halo2_b200.vanishing import vanishing_quotient_resident
    from oracle import cref, pasta
    from tests import bench_circuit as BC
    if not torch.cuda.is_available():
        raise SystemExit("vanishing_time.py needs a GPU")
    L.init(0)
    info = gpu_info(L)
    print(json.dumps({"gpu": info}), flush=True)
    cases = [(int(k), int(d), "") for k in a.ks.split(",") for d in a.degrees.split(",")]
    cases.append((14, BC.DEGREE, "benchmark circuit"))
    rows = []
    for k, degree, label in cases:
        D = h2.EvaluationDomain("fp", degree, k, pasta.zeta_candidates("fp")[0])
        n, N, parts = D.n, D.extended_len(), D.quotient_poly_degree
        src = h2.ResidentPoly("fp", N, cref.gen_scalars("fp", 0x7A + 31 * k + degree, N))
        work = h2.ResidentPoly("fp", N)
        flat = h2.ResidentPoly("fp", n * parts)
        old = [h2.ResidentPoly("fp", n) for _ in range(parts)]
        new = [h2.ResidentPoly("fp", n) for _ in range(parts)]

        def existing():
            D.divide_by_vanishing_poly_resident(work)
            D.extended_to_coeff_resident(work, out=flat)
            for i, p in enumerate(old):
                p.copy_from(flat, n, src_off=i * n)

        def fused():
            vanishing_quotient_resident(D, src, out=new)

        fns = {"existing": existing, "fused": fused}
        times = {name: [] for name in fns}
        for r in range(a.reps + 1):
            for name, fn in fns.items():
                if name == "existing":
                    work.copy_from(src, N)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                if r:
                    times[name].append(time.perf_counter() - t0)
        digest = {}
        for name, ps in (("existing", old), ("fused", new)):
            hsh = hashlib.sha256()
            for p in ps:
                hsh.update(p.download().tobytes())
            digest[name] = hsh.hexdigest()
        row = {"k": k, "degree": degree, "extended_k": D.extended_k, "pieces": parts, "case": label,
               "existing_ms": round(1e3 * statistics.median(times["existing"]), 4),
               "fused_ms": round(1e3 * statistics.median(times["fused"]), 4),
               "existing_all_ms": [round(1e3 * x, 4) for x in times["existing"]],
               "fused_all_ms": [round(1e3 * x, 4) for x in times["fused"]],
               "identical": digest["existing"] == digest["fused"]}
        row["speedup"] = round(row["existing_ms"] / row["fused_ms"], 3)
        print(json.dumps(row), flush=True)
        rows.append(row)
        for p in [src, work, flat] + old + new:
            p.close()
        if not row["identical"]:
            raise SystemExit(f"outputs differ at k = {k}, degree {degree}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
