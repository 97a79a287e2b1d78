"""Time of the lookup argument's permuted columns on the GPU, from compressed columns to committed permuted columns: one call
for every lookup (h2_poly_lookup_permuted + one batched commit, csrc/lookup.cuh) against a per-lookup composition
(tests/lookup_permuted_cases.py: per lookup h2_poly_lookup_permute, the blinding rows uploaded, one commit of its two
columns).

  python tools/lookup_permuted_time.py [--ks 14,16,18,20] [--counts 1,4,16] [--reps 5] [--out lookup_permuted_time.json]
  python tools/lookup_permuted_time.py --single [--pkg DIR]    # h2_poly_lookup_permute alone, one lookup

Inputs: a full-width random table, the input drawn from its usable rows uniformly or with 90 % of the rows on one value;
blinding_factors = 5.  Each timed run starts from resident compressed columns and ends in a device synchronise; medians of
`reps` alternated runs after one warm-up, every run's outputs and commitments compared byte for byte between the two paths.
--single times h2_poly_lookup_permute of the package found in DIR (default: this tree), so two builds of the library can be
compared by running it once on each.  The GPU's name and power limit are read in the same run."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF = 5


def gpu_info(L):
    q = subprocess.run(["nvidia-smi", "-i", str(L._inited_device or 0), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    f = [x.strip() for x in q.stdout.strip().split(",")]
    return {"name": f[0], "power_limit": f[1], "sm_max_clock": f[2]} if len(f) == 3 else {"raw": q.stdout.strip()}


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def run_single(h2, torch, reps, ks):
    from tests.lookup_permuted_cases import columns
    rows = []
    for k in ks:
        n = 1 << k
        u = n - BF - 1
        for hot in (False, True):
            a, t = (h2.ResidentPoly("fp", n, c) for c in columns("fp", n, u, 0x51 + k, hot))
            oa, ot = h2.ResidentPoly("fp", n), h2.ResidentPoly("fp", n)
            ts = []
            for r in range(reps + 1):
                dt, _ = timed(torch, lambda: h2.permute_expression_pair_resident(a, t, u, oa, ot))
                if r:
                    ts.append(dt)
            row = {"k": k, "hot": hot, "permute_ms": 1e3 * statistics.median(ts), "all_ms": [round(1e3 * x, 3) for x in ts],
                   "sha256": hashlib.sha256(oa.download().tobytes() + ot.download().tobytes()).hexdigest()}
            print(json.dumps(row), flush=True)
            rows.append(row)
            for p in (a, t, oa, ot):
                p.close()
    return rows


def run_fused(h2, torch, reps, ks, counts):
    from oracle import pasta
    from tests.bench_circuit import _bench_params
    from tests.lookup_permuted_cases import columns, composition
    rows = []
    for k in ks:
        n = 1 << k
        u = n - BF - 1
        prm = _bench_params(h2, k)
        D = h2.EvaluationDomain("fp", 3, k, pasta.zeta_candidates("fp")[0])
        for count in counts:
            for hot in (False, True):
                pairs = [tuple(h2.ResidentPoly("fp", n, c) for c in columns("fp", n, u, 0x1000 + 100 * k + b, hot)) for b in range(count)]
                blinding = pasta.gen_scalars("fp", 0x77 + k, count * 2 * (BF + 1))
                blinds = pasta.gen_scalars("fp", 0x78 + k, 2 * count)

                def new():
                    out = [q for pr in h2.lookup_permute_resident(D, pairs, BF, blinding) for q in pr]
                    return out, prm.commit_resident_affine(out, [h2.Blind(b) for b in blinds], lagrange=True)

                def old_path():
                    out, cms = [], []
                    for b in range(count):
                        pi, pt = composition(h2, D, [pairs[b]], BF, blinding[2 * (BF + 1) * b:2 * (BF + 1) * (b + 1)])[0]
                        out += [pi, pt]
                        cms.append(prm.commit_resident_affine([pi, pt], [h2.Blind(x) for x in blinds[2 * b:2 * b + 2]], lagrange=True))
                    return out, cms

                t_new, t_old = [], []
                for r in range(reps + 1):                            # run 0 warms both paths up; the order alternates
                    got = {}
                    for name, fn, acc in ((("new", new, t_new), ("old", old_path, t_old)) if r % 2 else (("old", old_path, t_old), ("new", new, t_new))):
                        dt, res = timed(torch, fn)
                        got[name] = res
                        if r:
                            acc.append(dt)
                    (on, cn), (oo, co) = got["new"], got["old"]
                    if not all((x.download() == y.download()).all() for x, y in zip(on, oo)) or not all(
                            (cn[2 * b:2 * b + 2] == co[b]).all() for b in range(count)):
                        raise SystemExit(f"k={k} count={count} hot={hot}: the one call differs from the composition")
                    for p in on + oo:
                        p.close()
                for pr in pairs:
                    for p in pr:
                        p.close()
                row = {"k": k, "lookups": count, "hot": hot, "one_call_ms": 1e3 * statistics.median(t_new),
                       "composition_ms": 1e3 * statistics.median(t_old), "one_call_all_ms": [round(1e3 * x, 3) for x in t_new],
                       "composition_all_ms": [round(1e3 * x, 3) for x in t_old]}
                print(json.dumps(row), flush=True)
                rows.append(row)
        prm.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="14,16,18,20")
    ap.add_argument("--counts", default="1,4,16")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--single", action="store_true")
    ap.add_argument("--pkg", default=ROOT)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.abspath(a.pkg))
    import torch
    import halo2_b200 as h2
    from halo2_b200 import lib as L
    L.init()
    info = gpu_info(L)
    print(json.dumps({"gpu": info, "lib": L.lib_path()}), flush=True)
    ks = [int(x) for x in a.ks.split(",")]
    if a.single:
        rows = run_single(h2, torch, a.reps, ks)
    else:
        rows = run_fused(h2, torch, a.reps, ks, [int(x) for x in a.counts.split(",")])
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
