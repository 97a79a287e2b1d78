"""GPU tests of the prover's phase calls at production sizes (k = 15 to 20), each compared exactly with the C oracle
(oracle/cref.py), never with another device path:

- K21, h2_poly_permutation_product / h2_poly_lookup_product: the benchmark shape (3 columns, chunk_len 3, 2 proofs), the wide
  shape (16 columns, chunk_len 3: 6 sets, the last partial) and 2 proofs x 3-4 lookups, with blinding rows and zero
  denominators planted at the chunk-tree boundaries, against cref.permutation_product / cref.lookup_product.  A zero
  denominator makes the rest of its column zero, so each zero gets a column of its own that ends its chain: the permutation
  call takes rows 32767 and 32768 (where the third level's chunks start; at k = 15, where they are blinding rows, row
  n / 2), the lookup call rows 0, 31, 32, 1023 and 1024, both row n - bf - 1, whose zero reaches only the blinding row after
  it.  The columns without such a zero are asserted nonzero up to row n - bf - 1, so every row of every level is compared
  with values that depend on it.  Every call also asserts, from its launch count, that it ran the number of chunk-tree
  levels gp_scan_plan gives for its size, so a later change of the plan fails here instead of moving these tests off the
  levels they are meant to cover;
- K23, the column-batched transforms at (k, extended_k) = (16, 18), (18, 20), (20, 22) with 3 and 17 columns, against
  cref.ifft / cref.coeff_to_extended column by column, and h2_poly_set_rows at k = 20;
- K24, h2_poly_vanishing_quotient at k = 15 ... 20 with extended_k - k = 1, 2, 3 (at most 2^23 elements), against
  cref.divide_by_vanishing_poly, cref.extended_to_coeff and the split into pieces, on a random and a structured h(X).

The C restatements of the product loops and of the division are checked against the big-integer loops in
tests/test_grand_product_oracle.py."""
import ctypes
import functools
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests import bench_circuit as BC  # noqa: E402
from tests.plonk_verifier import scalar_delta  # noqa: E402

SEED = 0x5048415345
PRODUCT_RULE = 3                                                # emu_chunk_tree's rule of the product columns (gp_scan_plan, level 1 forced)
LEVELS = {5: 1, 15: 2, 16: 3, 18: 3, 20: 3}                    # the chunk-tree levels of a 2^k product column


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


def _close(*groups):
    for g in groups:
        for p in g:
            p.close()


def _first_diff(got, want):
    """The first row where two (n, 32) arrays differ, or None."""
    rows = np.flatnonzero((got != want).any(axis=1))
    return int(rows[0]) if rows.size else None


def _where(row):
    """A row's chunk index at every level of the product columns' chunk tree: where a wrong carry came from."""
    return None if row is None else [row >> (5 * l) for l in range(4)]


@functools.lru_cache(maxsize=None)
def _plan_levels(n):
    """gp_scan_plan's level count of a product column of n rows, through the host emulation's copy of the plan."""
    from tests.kernel_emul import build as emul_build
    emu = ctypes.CDLL(emul_build.build())
    m = np.zeros(8, dtype=np.uint64)
    off = np.zeros(8, dtype=np.uint64)
    L, total = ctypes.c_uint32(), ctypes.c_uint64()
    assert emu.emu_chunk_tree(PRODUCT_RULE, ctypes.c_uint64(n), ctypes.c_uint64(1), m.ctypes.data_as(ctypes.c_void_p),
                              off.ctypes.data_as(ctypes.c_void_p), ctypes.byref(L), ctypes.byref(total)) == 0
    return L.value


def _launches(call):
    from halo2_b200 import lib as L
    before = L.launch_count()
    out = call()
    return out, L.launch_count() - before


# ---- K21: the product columns ------------------------------------------------------------------------------------------
SHAPES = {"benchmark": (2, 3, 3), "wide": (1, 16, 3)}          # (proofs, columns, chunk_len)


def _perm_zeros(name, n, bf):
    """(proof, column, row) whose denominator term is planted to zero.  A zero makes the rest of its product column zero, and
    of every later set of its proof through last_z, so the rows spread over the columns: row n - bf - 1 (its zero only reaches
    the blinding row n - bf, so the carry is untouched) in sets that hand over, the others in columns that are last in their
    chain."""
    late = [r for r in (32767, 32768) if r < n - bf - 1] or [n // 2]
    if name == "benchmark":
        return [(0, 2, n - bf - 1), (1, 1, late[-1])]
    return [(0, 1, n - bf - 1), (0, 8, n - bf - 1), (0, 15, late[0])]


LOOKUP_PER_PROOF = (3, 4)
# (lookup, 2: beta + a' = 0 / 3: gamma + s' = 0, row): the first rows of level-1 and level-2 chunks and the rows before them,
# one per lookup, and lookups 2 and 6 (one per proof) with a zero only at n - bf - 1
LOOKUP_ZEROS = [(0, 2, 0), (1, 3, 31), (3, 2, 32), (4, 3, 1023), (5, 2, 1024)]
LOOKUP_CLEAN = (2, 6)


def _perm_case(eng, field, k, name):
    m, n, bf = pasta.FIELDS[field], 1 << k, BC.BLINDING_FACTORS
    proofs, cols, chunk_len = SHAPES[name]
    sets = -(-cols // chunk_len)
    seed = SEED + 1000 * k + 100 * (field == "fq") + cols
    beta, gamma = pasta.gen_scalars(field, seed, 2)
    omega = pasta.omega_for_k(field, k)
    delta = scalar_delta(m)
    sig = np.stack([cref.gen_scalars(field, seed + 1 + c, n) for c in range(cols)])
    val = np.stack([np.stack([cref.gen_scalars(field, seed + 50 + 20 * p + c, n) for c in range(cols)]) for p in range(proofs)])
    for p, c, r in _perm_zeros(name, n, bf):
        s = int.from_bytes(sig[c, r].tobytes(), "little")
        val[p, c, r] = cref.ints_to_bytes([(-(beta * s + gamma)) % m])[0]
    blinding = pasta.gen_scalars(field, seed + 9, proofs * sets * bf)
    want = cref.permutation_product(field, val, sig, chunk_len, beta, gamma, omega, delta, cref.ints_to_bytes(blinding), bf)
    D = eng.EvaluationDomain(field, BC.DEGREE, k, pasta.zeta_candidates(field)[0])
    assert D.omega == omega
    S = [eng.ResidentPoly(field, n, s) for s in sig]
    C = [[eng.ResidentPoly(field, n, v) for v in per] for per in val]
    try:
        z, launches = _launches(lambda: eng.permutation_product_resident(D, C, S, beta, gamma, delta, chunk_len, bf, blinding))
        try:
            for p in range(proofs):
                for a in range(sets):
                    got = z[p][a].download()
                    row = _first_diff(got, want[p, a])
                    assert row is None, (field, k, name, "proof", p, "set", a, "row", row, "chunks by level", _where(row))
        finally:
            _close(*z)
    finally:
        _close(S, *C)
    killed = set()
    for p, c, r in _perm_zeros(name, n, bf):                   # the planted zeros did reach the product where they can
        if r + 1 < n - bf:
            assert not want[p, c // chunk_len, r + 1].any() and want[p, c // chunk_len, r].any()
            killed.add((p, c // chunk_len))
    for p in range(proofs):                                     # and every other column is nonzero on every row that carries
        for a in range(sets):
            if (p, a) not in killed:
                assert want[p, a, :n - bf].any(axis=1).all(), (field, k, name, p, a)
    assert len(killed) == 1
    return launches


@pytest.fixture(scope="module")
def small_launches(eng):
    """The launch count of each call shape at k = 5, where the product columns have one chunk-tree level: the count at
    level L is this plus two launches per level above the first (one up, one down)."""
    assert _plan_levels(1 << 5) == LEVELS[5]
    out = {name: _perm_case(eng, "fp", 5, name) for name in SHAPES}
    out["lookup"] = _lookup_case(eng, "fp", 5)
    return out


def _lookup_case(eng, field, k):
    m, n, bf = pasta.FIELDS[field], 1 << k, BC.BLINDING_FACTORS
    seed = SEED + 7000 + 10 * k + (field == "fq")
    beta, gamma = pasta.gen_scalars(field, seed, 2)
    per_proof = LOOKUP_PER_PROOF
    flat = [[cref.gen_scalars(field, seed + 1 + 4 * b + j, n) for j in range(4)] for b in range(sum(per_proof))]
    for b, which, r in LOOKUP_ZEROS + [(b, 2 + b % 2, n - bf - 1) for b in LOOKUP_CLEAN]:
        if r < n:
            flat[b][which][r] = cref.ints_to_bytes([(-(beta if which == 2 else gamma)) % m])[0]
    blinding = pasta.gen_scalars(field, seed + 99, len(flat) * bf)
    want = [cref.lookup_product(field, *lk, beta, gamma, cref.ints_to_bytes(blinding[b * bf:(b + 1) * bf]), bf) for b, lk in enumerate(flat)]
    D = eng.EvaluationDomain(field, BC.DEGREE, k, pasta.zeta_candidates(field)[0])
    R, at = [], 0
    for cnt in per_proof:
        R.append([tuple(eng.ResidentPoly(field, n, c) for c in lk) for lk in flat[at:at + cnt]])
        at += cnt
    try:
        z, launches = _launches(lambda: eng.lookup_product_resident(D, R, beta, gamma, bf, blinding))
        try:
            assert [len(per) for per in z] == list(per_proof)
            for b, q in enumerate(q for per in z for q in per):
                row = _first_diff(q.download(), want[b])
                assert row is None, (field, k, "lookup", b, "row", row, "chunks by level", _where(row))
        finally:
            _close(*z)
    finally:
        _close([p for per in R for lk in per for p in lk])
    for b, which, r in LOOKUP_ZEROS:                           # the planted zeros did reach the product where they can
        if r + 1 < n - bf:
            assert not want[b][r + 1].any()
    for b in LOOKUP_CLEAN:                                      # and the other lookups are nonzero on every row that carries
        assert want[b][:n - bf].any(axis=1).all(), (field, k, b)
    return launches


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("k", [15, 16, 18, 20])
def test_permutation_products_against_the_oracle(eng, small_launches, field, k):
    L = _plan_levels(1 << k)
    assert L == LEVELS[k], (k, L)
    for name in SHAPES:
        launches = _perm_case(eng, field, k, name)
        assert launches == small_launches[name] + 2 * (L - LEVELS[5]), (name, k, launches)


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("k", [15, 16, 18, 20])
def test_lookup_products_against_the_oracle(eng, small_launches, field, k):
    L = _plan_levels(1 << k)
    assert L == LEVELS[k], (k, L)
    launches = _lookup_case(eng, field, k)
    assert launches == small_launches["lookup"] + 2 * (L - LEVELS[5]), (k, launches)


# ---- K23: the column-batched transforms and set_rows -------------------------------------------------------------------
def _domain(eng, field, k, ext_k):
    D = eng.EvaluationDomain(field, (1 << (ext_k - k)) + 1, k, pasta.zeta_candidates(field)[0])
    assert D.extended_k == ext_k
    return D


def _sample(count, seed):
    """Column 0, the last column and a seeded sample of the columns between them."""
    inner = list(range(1, count - 1))
    return sorted({0, count - 1, *random.Random(seed).sample(inner, min(3, len(inner)))})


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("k,ext_k", [(16, 18), (18, 20), (20, 22)])
def test_batched_transforms_against_the_oracle(eng, field, k, ext_k):
    D = _domain(eng, field, k, ext_k)
    n, N = D.n, D.extended_len()
    for count in (3, 17):
        seed = SEED + 300 * k + count + (field == "fq")
        vals = [cref.gen_scalars(field, seed + c, n) for c in range(count)]
        src = [eng.ResidentPoly(field, n, v) for v in vals]
        co, ext = [], []
        try:
            co = D.lagrange_to_coeff_batch_resident(src, out=[eng.ResidentPoly(field, n) for _ in src])
            ext = D.coeff_to_extended_batch_resident(co)
            for c in _sample(count, seed):
                want_co = cref.ifft(field, vals[c], D.omega_inv, k, D.ifft_divisor)
                row = _first_diff(co[c].download(), want_co)
                assert row is None, (field, k, count, "lagrange_to_coeff column", c, "row", row)
                want_ext = cref.coeff_to_extended(field, want_co, k, ext_k, D.g_coset, D.extended_omega)
                row = _first_diff(ext[c].download(N), want_ext)
                assert row is None, (field, k, ext_k, count, "coeff_to_extended column", c, "row", row)
        finally:
            _close(src, co, ext)


def test_set_rows_at_k20(eng):
    from halo2_b200 import lib as L
    field, k, count, bf = "fp", 20, 17, BC.BLINDING_FACTORS
    n = 1 << k
    start = n - bf
    cols = [cref.gen_scalars(field, SEED + 40 + c, n) for c in range(count)]
    P = [eng.ResidentPoly(field, n, c) for c in cols]
    try:
        vals = np.stack([cref.gen_scalars(field, SEED + 90 + c, bf) for c in range(count)])
        before = L.launch_count()
        eng.set_rows_resident(P, start, vals)
        assert L.launch_count() - before == 1
        for c, p in enumerate(P):
            got = p.download()
            assert np.array_equal(got[start:], vals[c]), c                             # the blinding rows written
            assert np.array_equal(got[:start], cols[c][:start]), c                     # the rows below them, n - bf - 1 included, untouched
    finally:
        _close(P)


# ---- K24: the vanishing quotient ---------------------------------------------------------------------------------------
_DEGREES = {1: 3, 2: 5, 3: 9}                                   # cs degree j -> extended_k - k
MAX_EXTENDED = 1 << 23


def _structured_h(field, N, n, seed):
    """A random h(X) with runs of 0, 1 and m - 1 and one full-size value alone among zeros."""
    m = pasta.FIELDS[field]
    h = cref.gen_scalars(field, seed, N)
    h[:n // 2] = 0
    h[n // 2:n] = cref.ints_to_bytes([1])[0]
    h[N - n // 2:] = cref.ints_to_bytes([m - 1])[0]
    h[N // 2 - 64:N // 2 + 64] = 0
    h[N // 2] = cref.gen_scalars(field, seed + 1, 1)[0]
    return h


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("k", [15, 16, 17, 18, 19, 20])
def test_vanishing_quotient_against_the_oracle(eng, field, k):
    from halo2_b200 import vanishing as V
    for ext, j in _DEGREES.items():
        if (1 << (k + ext)) > MAX_EXTENDED:
            continue
        D = eng.EvaluationDomain(field, j, k, pasta.zeta_candidates(field)[0])
        assert D.extended_k == k + ext
        n, N, d = D.n, D.extended_len(), D.quotient_poly_degree
        inputs = {"random": cref.gen_scalars(field, SEED + 10 * k + ext, N), "structured": _structured_h(field, N, n, SEED + 20 * k + ext)}
        for name, h in inputs.items():
            div = cref.divide_by_vanishing_poly(field, h, D.t_evaluations)
            want = cref.extended_to_coeff(field, div, D.extended_k, D.extended_omega_inv, D.extended_ifft_divisor, D.g_coset, d * n)
            h_ext = eng.ResidentPoly(field, N, h)
            pieces = []
            try:
                pieces = V.vanishing_quotient_resident(D, h_ext)
                assert len(pieces) == d
                for i, p in enumerate(pieces):
                    row = _first_diff(p.download(), want[i * n:(i + 1) * n])
                    assert row is None, (field, k, D.extended_k, name, "piece", i, "row", row)
                assert np.array_equal(h_ext.download(), h)                          # the source is only read
            finally:
                _close(pieces, [h_ext])
