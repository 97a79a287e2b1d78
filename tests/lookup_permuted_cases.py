"""Lookup columns for the batched lookup permutation's tests and timings: input / table pairs with a full-width or a hot
input, and the per-lookup composition create_proof_engine uses (h2_poly_lookup_permute, then the blinding rows)."""
from __future__ import annotations

import numpy as np

from oracle import cref


def columns(field, n, u, seed, hot):
    """(input, table) as (n, 32) canonical bytes: a full-width table, the input drawn from its usable rows (hot: 90 % of
    the rows on its first value), random rows past u."""
    rnd = np.random.default_rng(seed)
    tab = cref.gen_scalars(field, seed, n)
    pick = rnd.integers(0, u, size=n)
    if hot:
        pick[rnd.random(n) < 0.9] = 0
    inp = tab[pick].copy()
    inp[u:] = cref.gen_scalars(field, seed + 1, n - u)
    return np.ascontiguousarray(inp), np.ascontiguousarray(tab)


def composition(eng, D, pairs, bf, blinding):
    """What tests/plonk_prover.create_proof_engine does per lookup: h2_poly_lookup_permute over the usable rows, then the
    blinding rows uploaded into rows [u, n)."""
    rows, n = bf + 1, D.n
    out = []
    for b, (a, t) in enumerate(pairs):
        pi, pt = eng.permute_expression_pair_resident(a, t, n - rows, eng.ResidentPoly(D.field, n), eng.ResidentPoly(D.field, n))
        for q, vals in ((pi, blinding[2 * rows * b:2 * rows * b + rows]), (pt, blinding[2 * rows * b + rows:2 * rows * (b + 1)])):
            tmp = eng.ResidentPoly(D.field, rows, cref.ints_to_bytes(vals))
            q.copy_from(tmp, rows, src_off=0, dst_off=n - rows)
            tmp.close()
        out.append((pi, pt))
    return out
