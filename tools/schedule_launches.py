"""Kernel launches and output bytes of the entry points whose scratch comes from a host-side plan (the chunk trees of
polyops.cuh, lk_plan, the copy cycles' layouts): eval, inner product, kate division, running product, permutation
product, lookup product, lookup permutation and sigma from copies, at each k, on seeded inputs.

  python tools/schedule_launches.py [--ks 1,5,10,14,20] [--out FILE]

Each row has the h2_launch_count() difference of one call and the SHA-256 of its outputs; the rows go to stdout as JSON
lines, and with --out also to FILE as one JSON list.  Run it on two builds of the library (each from its own tree) and
compare the outputs: a change to how the plans are written must leave both the same.  One count is not fixed by the build:
sigma from copies repeats its in-place pointer-jumping pass until a pass changes nothing, and how many passes that takes
depends on thread timing, so at large k its launch count can differ by a pass or two between runs of one build (its
output bytes do not)."""
import argparse
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FIELD = "fp"
SEED = 0x5C4ED


def digest(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def run(ks):
    import halo2_b200 as h2
    from halo2_b200 import keygen, lib, products
    from oracle import cref, pasta
    lib.init(0)
    rows = []

    def measure(name, k, fn):
        before = lib.launch_count()
        out = fn()
        rows.append({"k": k, "call": name, "launches": lib.launch_count() - before, "sha256": digest(*out)})
        print(json.dumps(rows[-1]), flush=True)

    for k in ks:
        n = 1 << k
        seed = SEED + 97 * k
        D = h2.EvaluationDomain(FIELD, 3, k, pasta.zeta_candidates(FIELD)[0])
        col = lambda i: h2.ResidentPoly(FIELD, n, cref.gen_scalars(FIELD, seed + i, n))
        a = [col(i) for i in range(3)]
        b = [col(10 + i) for i in range(3)]
        pts = cref.bytes_to_ints(cref.gen_scalars(FIELD, seed + 20, 3))
        measure("h2_poly_eval", k, lambda: [np.array(h2.eval_polynomial_resident(a, pts), dtype=object).astype(str)])
        measure("h2_poly_inner_product", k, lambda: [np.array(h2.inner_product_resident(a, b), dtype=object).astype(str)])
        if n > 1:
            q = h2.kate_division_resident(a, pts)
            measure("h2_poly_kate_division", k, lambda: [p.download() for p in h2.kate_division_resident(a, pts, dst=q)])
        z = h2.running_product_resident(a[0], 5)
        measure("h2_poly_running_product", k, lambda: [h2.running_product_resident(a[0], 5, dst=z).download()])
        bf = min(5, n - 2)
        rnd = cref.bytes_to_ints(cref.gen_scalars(FIELD, seed + 30, 64))
        beta, gamma, delta = rnd[:3]
        if bf >= 0:
            sigmas = [col(40 + i) for i in range(3)]
            proofs = [[a[0], a[1], b[0]], [b[1], b[2], a[2]]]
            blind = rnd[3:3 + 2 * 2 * bf]
            measure("h2_poly_permutation_product", k, lambda: [p.download() for per in products.permutation_product_resident(
                D, proofs, sigmas, beta, gamma, delta, 2, bf, blind) for p in per])
            # lookups: each input's rows are drawn from its table's usable rows
            u = n - bf - 1
            rng = np.random.default_rng(seed)
            tabs = [cref.gen_scalars(FIELD, seed + 50 + i, n) for i in range(4)]
            pairs = [(h2.ResidentPoly(FIELD, n, t[rng.integers(0, u, n)]), h2.ResidentPoly(FIELD, n, t)) for t in tabs]
            lblind = cref.bytes_to_ints(cref.gen_scalars(FIELD, seed + 60, 4 * 2 * (bf + 1)))
            perm = []

            def permute():
                perm.extend(products.lookup_permute_resident(D, pairs, bf, lblind))
                return [p.download() for pr in perm for p in pr]
            measure("h2_poly_lookup_permuted", k, permute)
            lk = [[(pairs[i][0], pairs[i][1], perm[i][0], perm[i][1]) for i in range(4)]]
            measure("h2_poly_lookup_product", k, lambda: [p.download() for per in products.lookup_product_resident(
                D, lk, beta, gamma, bf, rnd[3:3 + 4 * bf]) for p in per])
        cols, copies = 3, 2 * n
        rng = np.random.default_rng(seed + 1)
        cc = keygen.CopyConstraints(n, cols)
        cc.extend(np.stack([rng.integers(0, cols, copies), rng.integers(0, n, copies), rng.integers(0, cols, copies),
                            rng.integers(0, n, copies)], axis=1).astype(np.uint32))
        measure("h2_poly_permutation_sigma_copies", k, lambda: [p.download() for p in keygen.build_permutation_polys(D, cc, delta)])
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,5,10,14,20")
    ap.add_argument("--out", help="also write the rows to this file")
    args = ap.parse_args()
    rows = run([int(x) for x in args.ks.split(",")])
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
