"""Key generation time for the reference's benchmark circuit (benches/plonk.rs, rebuilt in tests/bench_circuit.py: 4 fixed
columns, 3 permutation columns) on the GPU, the engine's keygen against the path the tests and bench.py take today.

  python tools/keygen_time.py [--ks 14,16,18,20] [--reps 3] [--cycle-k 20] [--out keygen_time.json]

engine   host Assembly (halo2_b200.Assembly, the reference's copy bookkeeping) | sigma (build_permutation_polys: the mapping
         array, its upload and the kernel, one synchronous call) | the rest of keygen_vk + keygen_pk (fixed-column uploads, one
         batched commit pass, the transforms, l_0 / l_blind / l_last) = keygen_vk + keygen_pk - 2 sigma
current  sigma in Python from the same mapping (the serial omega-power loop and the gather of permutation/keygen.rs:108-143, as
         tests/bench_circuit.py does it) | an upload and a commit_lagrange + batch_normalize per column (bench.py's keygen) | an
         upload and the two transforms per column, and the three indicator columns from host arrays (tests/plonk_prover.py)
copies   the copy list instead of the Assembly (halo2_b200.CopyConstraints, h2_poly_permutation_sigma_copies): the whole
         sigma call (copy-list upload, the assembly kernels of csrc/assembly.cuh, sigma), keygen_vk + keygen_pk from it, and
         the host baselines on the same (m, 4) copy array: the Python Assembly and the C oracle's sequential loop
         (orc_assembly of oracle/assembly_oracle.c, compiled -O3).  The copy arrays are generated vectorised; the baselines replay them row by row.
A separate torch.profiler pass per k gives the device time of the sigma kernels and of the mapping's host-to-device copies,
and for the copies path that of the copy-list upload, the assembly kernels and sigma.  --cycle-k adds a synthetic list:
one cycle through every cell of 3 columns, copies in random order, the longest pointer-jumping chains there are.
Medians of `reps` runs after one warm-up (the host baselines of the synthetic list run once); both paths' commitments and
sigma columns are compared.  The GPU's name and power limit are read in the same run."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import halo2_b200 as h2  # noqa: E402
from halo2_b200 import lib as L  # noqa: E402
from tests import bench_circuit as BC  # noqa: E402

M = h2.poly.FIELDS["fp"]
ZETA = pow(5, (M - 1) // 3, M)
DELTA = pow(5, 1 << 32, M)                                         # F::DELTA


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", str(L._inited_device or 0), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    f = [x.strip() for x in q.stdout.strip().split(",")]
    return {"name": f[0], "power_limit": f[1], "sm_max_clock": f[2]} if len(f) == 3 else {"raw": q.stdout.strip()}


def gen_points(n: int) -> np.ndarray:
    """n seeded Vesta points, generated on the device (affine, canonical)."""
    lib = L.init()
    t = torch.empty((n, 16), dtype=torch.int32, device="cuda")
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.h2_dev_gen_points(L.CURVE_ID["vesta"], ctypes.c_uint64(0x4B47), ctypes.c_uint64(0), ctypes.c_size_t(n), ctypes.c_void_p(t.data_ptr()), s))
    L.check(lib.h2_dev_convert(L.FIELD_ID[L.BASE_FIELD["vesta"]], ctypes.c_void_p(t.data_ptr()), ctypes.c_size_t(2 * n), 0, s))
    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint8).reshape(n, 64).copy()


def to_bytes(col) -> np.ndarray:
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in col), dtype=np.uint8).reshape(-1, 32)


def python_sigma(mapping: np.ndarray, n: int, omega: int, delta: int):
    omega_powers = [1] * n
    for j in range(1, n):
        omega_powers[j] = omega_powers[j - 1] * omega % M
    deltas = [pow(delta, i, M) for i in range(mapping.shape[0])]
    return [[deltas[c] * omega_powers[r] % M for c, r in col.tolist()] for col in mapping]


def median_of(fn, reps):
    """Median wall time of fn() up to the end of its device work (a device-wide synchronise: the engine's streams included)."""
    fn()                                                           # warm-up
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def sigma_profile(D, asm):
    """Device time (ms) of the sigma kernels and of the host-to-device copies inside one build_permutation_polys."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for p in h2.build_permutation_polys(D, asm, DELTA):
            p.close()
        torch.cuda.synchronize()
    out = {"sigma_kernel_ms": 0.0, "tables_kernel_ms": 0.0, "h2d_copy_ms": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        t = (ev.cuda_time_total if t is None else t) / 1e3
        if "keygen_sigma_kernel" in ev.key:
            out["sigma_kernel_ms"] += t
        elif "keygen_tables_kernel" in ev.key:
            out["tables_kernel_ms"] += t
        elif "HtoD" in ev.key:
            out["h2d_copy_ms"] += t
    return out


def copies_profile(D, cc):
    """Device time (ms) inside one build_permutation_polys from CopyConstraints: the copy-list upload, the assembly kernels
    (as_*), the sigma and table kernels."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for p in h2.build_permutation_polys(D, cc, DELTA):
            p.close()
        torch.cuda.synchronize()
    out = {"copies_upload_ms": 0.0, "copies_assembly_kernels_ms": 0.0, "copies_sigma_kernels_ms": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        t = (ev.cuda_time_total if t is None else t) / 1e3
        if "keygen_sigma_kernel" in ev.key or "keygen_tables_kernel" in ev.key:
            out["copies_sigma_kernels_ms"] += t
        elif "HtoD" in ev.key:
            out["copies_upload_ms"] += t
        elif "as_" in ev.key or "scan_" in ev.key:
            out["copies_assembly_kernels_ms"] += t
    return out


def copies_path(D, copies: np.ndarray, cols: int, reps: int, host_reps: int) -> dict:
    """The sigma call from the copy list, its profile, and the host baselines on the same array; checks the sigma columns
    against those from the Assembly's mapping."""
    from oracle import assembly as orc
    k, n = D.k, D.n
    res = {"copies": int(copies.shape[0])}
    cc = h2.CopyConstraints(n, cols)
    cc.extend(copies)

    def sigma():
        for p in h2.build_permutation_polys(D, cc, DELTA):
            p.close()
    res["copies_sigma_call_s"] = median_of(sigma, reps)
    res.update(copies_profile(D, cc))
    rows = copies.tolist()

    def py_assembly():
        a = h2.Assembly(n, cols)
        for c in rows:
            a.copy(*c)
        return a
    timed = (lambda fn: median_of(fn, reps)) if host_reps > 1 else once
    res["python_assembly_s"] = timed(py_assembly)
    res["orc_assembly_s"] = timed(lambda: orc.assembly(copies, cols, k))
    mapping, err = orc.assembly(copies, cols, k)
    assert err is None
    a = [p for p in h2.build_permutation_polys(D, cc, DELTA)]
    asm = h2.Assembly(n, cols)
    asm._mapping = (mapping[..., 0].astype(np.int64) * n + mapping[..., 1]).reshape(-1)   # the oracle's mapping, no second replay
    b = h2.build_permutation_polys(D, asm, DELTA)
    res["copies_sigma_identical"] = all((x.download() == y.download()).all() for x, y in zip(a, b))
    for p in a + b:
        p.close()
    return res


def once(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def run_cycle(k: int, reps: int) -> dict:
    """The synthetic list: one cycle through all 3 * 2^k cells, copies in random order."""
    n = 1 << k
    D = h2.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
    rng = np.random.default_rng(20)
    perm = rng.permutation(3 * n).astype(np.int64)
    nxt = np.roll(perm, -1)
    cp = np.stack([perm >> k, perm & (n - 1), nxt >> k, nxt & (n - 1)], axis=1)[rng.permutation(3 * n)].astype(np.uint32)
    res = {"k": k, "list": "one cycle through every cell, random copy order"}
    res.update(copies_path(D, np.ascontiguousarray(cp), 3, reps, 1))
    return res


def run_k(k: int, reps: int) -> dict:
    n = 1 << k
    D = h2.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
    pts = gen_points(n + 2)
    prm = h2.Params("vesta", k, pts[:n], pts[:n], pts[n:n + 1], u=pts[n + 1:])   # any generators: both paths commit to the same ones
    fixed, _, _ = BC.columns(k, M, D.omega, DELTA, 7)
    fixed_b = [to_bytes(c) for c in fixed]
    copies = [(0, 2 * i, 0, 2 * i + 1, 1, 2 * i + 1, 2, 2 * i) for i in range((1 << (k - 1)) - 3)]
    res = {"k": k, "columns": {"fixed": len(fixed), "permutation": 3}}
    try:
        def assembly():
            a = h2.Assembly(n, 3)
            for c in copies:
                a.copy(*c[:4])
                a.copy(*c[4:])
            return a
        asm = assembly()
        res["assembly_s"] = median_of(assembly, reps)
        res["mapping_array_s"] = median_of(lambda: asm.mapping, reps)

        def sigma():
            for p in h2.build_permutation_polys(D, asm, DELTA):
                p.close()
        res["sigma_call_s"] = median_of(sigma, reps)
        res["keygen_vk_s"] = median_of(lambda: h2.keygen_vk(prm, D, fixed_b, asm, DELTA), reps)
        res["keygen_pk_s"] = median_of(lambda: h2.keygen_pk(prm, D, fixed_b, asm, DELTA, BC.BLINDING_FACTORS).close(), reps)
        res["engine_rest_s"] = res["keygen_vk_s"] + res["keygen_pk_s"] - 2 * res["sigma_call_s"]
        res["engine_total_s"] = res["assembly_s"] + res["keygen_vk_s"] + res["keygen_pk_s"]
        res.update(sigma_profile(D, asm))
        elems = 3 * n
        res["sigma_bytes"] = 40 * elems                            # 8 B of mapping read, 32 B of result written per element
        if res["sigma_kernel_ms"] > 0:
            res["sigma_kernel_GBps"] = res["sigma_bytes"] / (res["sigma_kernel_ms"] * 1e-3) / 1e9

        # the current path
        mapping = asm.mapping
        t0 = time.perf_counter()
        sig = python_sigma(mapping, n, D.omega, DELTA)
        res["current_python_sigma_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        sig_b = [to_bytes(c) for c in sig]
        res["current_sigma_to_bytes_s"] = time.perf_counter() - t0
        xy = lambda col: h2.batch_normalize(prm.commit_lagrange(col, h2.Blind(1)).reshape(1, 96), "vesta")[0]

        def current_vk():
            return [xy(c) for c in fixed_b], [xy(c) for c in sig_b]

        def current_pk():
            keep = []
            for col in fixed_b + sig_b:
                lag = h2.ResidentPoly("fp", n, col)
                co = D.lagrange_to_coeff_resident(lag, out=h2.ResidentPoly("fp", n))
                keep += [lag, co, D.coeff_to_extended_resident(co)]
            bf = BC.BLINDING_FACTORS
            for rows in ([0], range(n - bf, n), [n - bf - 1]):
                host = np.zeros((n, 32), dtype=np.uint8)
                for r in rows:
                    host[r, 0] = 1
                lag = h2.ResidentPoly("fp", n, host)
                D.lagrange_to_coeff_resident(lag)
                keep.append(D.coeff_to_extended_resident(lag))
                lag.close()
            torch.cuda.synchronize()
            for p in keep:
                p.close()
        res["current_vk_commits_s"] = median_of(current_vk, reps)
        res["current_pk_s"] = median_of(current_pk, reps)
        res["current_total_s"] = (res["assembly_s"] + res["current_python_sigma_s"] + res["current_sigma_to_bytes_s"] + res["current_vk_commits_s"]
                                  + res["current_pk_s"])

        fc, pc = h2.keygen_vk(prm, D, fixed_b, asm, DELTA)
        cf, cs = current_vk()
        res["commitments_identical"] = bool((fc == np.stack(cf)).all() and (pc == np.stack(cs)).all())
        pk = h2.keygen_pk(prm, D, fixed_b, asm, DELTA, BC.BLINDING_FACTORS)
        res["sigma_identical"] = all((p.download() == s).all() for p, s in zip(pk.permutation.permutations, sig_b))
        pk.close()

        # the copy-list path
        arr = np.empty((2 * len(copies), 4), dtype=np.uint32)
        it = np.arange(len(copies), dtype=np.uint32)
        arr[0::2] = np.stack([0 * it, 2 * it, 0 * it, 2 * it + 1], axis=1)          # copy(a0, a1) ...
        arr[1::2] = np.stack([0 * it + 1, 2 * it + 1, 0 * it + 2, 2 * it], axis=1)  # ... copy(b1, c0), as assembly() replays them
        res.update(copies_path(D, arr, 3, reps, reps))
        cc = h2.CopyConstraints(n, 3)
        cc.extend(arr)
        res["copies_keygen_vk_s"] = median_of(lambda: h2.keygen_vk(prm, D, fixed_b, cc, DELTA), reps)
        res["copies_keygen_pk_s"] = median_of(lambda: h2.keygen_pk(prm, D, fixed_b, cc, DELTA, BC.BLINDING_FACTORS).close(), reps)
        res["copies_engine_total_s"] = res["copies_keygen_vk_s"] + res["copies_keygen_pk_s"]
        fcc, pcc = h2.keygen_vk(prm, D, fixed_b, cc, DELTA)
        res["copies_commitments_identical"] = bool((fcc == fc).all() and (pcc == pc).all())
    finally:
        prm.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="14,16,18,20")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cycle-k", type=int, default=20, help="k of the synthetic one-cycle list (0: none)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L.init()
    out = {"gpu": gpu_info(), "results": []}
    for k in (int(x) for x in a.ks.split(",")):
        r = run_k(k, a.reps)
        out["results"].append(r)
        print(json.dumps(r), flush=True)
    if a.cycle_k:
        r = run_cycle(a.cycle_k, a.reps)
        out["results"].append(r)
        print(json.dumps(r), flush=True)
    out["gpu_after"] = gpu_info()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out["gpu"]))


if __name__ == "__main__":
    main()
