"""Time of filling resident polynomials from columns that already live on the GPU as torch tensors: (a) the host route,
tensor -> .cpu().numpy() -> ResidentPoly(values), against (b) the device route, ResidentPoly.from_tensor for one column or one
upload_tensors_resident call for all of them (h2_poly_upload_dev, K25).

  python tools/device_columns_time.py [--ks 14,15,...,20] [--counts 1,10] [--reps 9] [--out device_columns_time.json]

Each arm allocates its polynomials and fills them; a run is timed with a host clock from the first call to a device
synchronise.  The two arms alternate, medians and ranges of `reps` runs after one warm-up of each, and the resident bytes of
the two arms are compared after the last run.  The GPU's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_info(L):
    q = subprocess.run(["nvidia-smi", "-i", str(L._inited_device or 0), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    f = [x.strip() for x in q.stdout.strip().split(",")]
    return {"name": f[0], "power_limit": f[1], "sm_max_clock": f[2]} if len(f) == 3 else {"raw": q.stdout.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="14,15,16,17,18,19,20")
    ap.add_argument("--counts", default="1,10")
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import halo2_b200 as h2
    from halo2_b200 import lib as L
    if not torch.cuda.is_available():
        raise SystemExit("device_columns_time.py needs a GPU")
    L.init(0)
    info = gpu_info(L)
    print(json.dumps({"gpu": info}), flush=True)
    rows = []
    for k in (int(x) for x in a.ks.split(",")):
        n = 1 << k
        for count in (int(x) for x in a.counts.split(",")):
            g = torch.Generator(device="cuda").manual_seed(k * 100 + count)
            cols = [torch.randint(0, 256, (n, 32), dtype=torch.uint8, device="cuda", generator=g) for _ in range(count)]
            for c in cols:
                c[:, 31] &= 0x3F                                   # canonical values
            torch.cuda.synchronize()
            kept = {}

            def host():
                ps = [h2.ResidentPoly("fp", n, c.cpu().numpy()) for c in cols]
                torch.cuda.synchronize()
                return ps

            def device():
                if count == 1:
                    ps = [h2.ResidentPoly.from_tensor("fp", cols[0])]
                else:
                    ps = [h2.ResidentPoly("fp", n) for _ in cols]
                    h2.upload_tensors_resident(ps, cols)
                torch.cuda.synchronize()
                return ps

            times = {"host": [], "device": []}
            for rep in range(a.reps + 1):
                for name, fn in (("host", host), ("device", device)) if rep % 2 == 0 else (("device", device), ("host", host)):
                    t0 = time.perf_counter()
                    ps = fn()
                    dt = time.perf_counter() - t0
                    if rep:
                        times[name].append(dt * 1e3)
                    for p in kept.get(name, []):
                        p.close()
                    kept[name] = ps
            same = all(np.array_equal(x.download(), y.download()) for x, y in zip(kept["host"], kept["device"]))
            for ps in kept.values():
                for p in ps:
                    p.close()
            row = {"k": k, "columns": count, "identical": same}
            for name, ts in times.items():
                row[name + "_ms"] = {"median": statistics.median(ts), "min": min(ts), "max": max(ts)}
            row["ratio"] = row["host_ms"]["median"] / row["device_ms"]["median"]
            rows.append(row)
            print(json.dumps(row), flush=True)
            del cols
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
