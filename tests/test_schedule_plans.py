"""CPU checks of the host-side plans that size and lay out the scratch of the multi-launch schedules on resident
polynomials, through the host emulation (tests/kernel_emul), which runs the schedules on the same plans:

- the chunk trees of polyops.cuh (gp_reduce_plan: eval, inner product, kate division; gp_scan_plan: the running product
  and, with level 1, K21's product columns), against each rule's level loop written out here;
- the lookup permutation's plan (lookup.cuh lk_plan);
- the copy cycles' scratch layouts (assembly.cuh as_edge_layout, as_slot_layout).
"""
import ctypes

import numpy as np
import pytest

from tests.kernel_emul import build as emul_build

CHUNK = 32
MAX_LEVELS = 8
REDUCE, INNER, SCAN, PRODUCT = 0, 1, 2, 3                  # emu_chunk_tree's rules
SIZES = sorted(set(range(65)) | {32 ** j + d for j in range(1, 7) for d in (-1, 0, 1)})
BATCHES = (1, 3, 256)


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emul_build.build())


def _ceil(m):
    return (m + CHUNK - 1) // CHUNK


def _reference(rule, n, batch):
    """The level arrays (m, off) of each rule as a plain loop: the reductions, the running product (one column), the
    product columns (level 1 always present)."""
    if rule in (REDUCE, INNER):
        m, off = [n], [0]
        while m[-1] > 1:
            off.append(off[-1] + (m[-1] * batch if len(m) > 1 else 0))
            m.append(_ceil(m[-1]))
        if rule == INNER and len(m) == 1:                         # a length-1 inner product's product level
            off.append(0)
            m.append(1)
        return m, off
    if rule == SCAN:
        assert batch == 1
        m, off = [n], [0]
        while m[-1] > CHUNK:
            off.append(off[-1] + (m[-1] if len(m) > 1 else 0))
            m.append(_ceil(m[-1]))
        return m, off
    m, off = [n, _ceil(n)], [0, 0]
    while m[-1] > CHUNK:
        off.append(off[-1] + m[-1] * batch)
        m.append(_ceil(m[-1]))
    return m, off


def _plan(emu, rule, n, batch):
    m = np.zeros(MAX_LEVELS, dtype=np.uint64)
    off = np.zeros(MAX_LEVELS, dtype=np.uint64)
    L, total = ctypes.c_uint32(), ctypes.c_uint64()
    rc = emu.emu_chunk_tree(rule, ctypes.c_uint64(n), ctypes.c_uint64(batch), m.ctypes.data_as(ctypes.c_void_p),
                            off.ctypes.data_as(ctypes.c_void_p), ctypes.byref(L), ctypes.byref(total))
    if rc:
        return None
    return [int(x) for x in m[:L.value + 1]], [int(x) for x in off[:L.value + 1]], total.value


def _disjoint_within(regions, end):
    """regions: (start, length); every one inside [0, end), none overlapping another."""
    at = 0
    for start, length in sorted(regions):
        assert start >= at, regions
        at = start + length
    assert at <= end, (regions, end)
    return at


@pytest.mark.parametrize("rule", [REDUCE, INNER, SCAN, PRODUCT], ids=["reduce", "inner_product", "running_product", "product_columns"])
def test_chunk_tree_plans(emu, rule):
    stop = 1 if rule in (REDUCE, INNER) else CHUNK
    forced = rule in (INNER, PRODUCT)                             # level 1 even when n <= stop
    for batch in (1,) if rule == SCAN else BATCHES:
        for n in SIZES:
            m, off, total = _plan(emu, rule, n, batch)
            L = len(m) - 1
            assert m[0] == n
            for l in range(L):                                    # the ceil-divide rule; a length-0 inner product's level holds 1
                assert m[l + 1] == (_ceil(m[l]) or (1 if rule == INNER else 0)), (rule, n, batch, l)
            assert m[L] <= stop and all(m[l] > stop for l in range(L) if not (forced and l == 0)), (rule, n, m)
            assert L >= 1 or not forced
            end = _disjoint_within([(off[l], m[l] * batch) for l in range(1, L + 1)], total)
            assert end == total, (rule, n, batch)                 # the scratch is exactly the levels
            assert (m, off) == _reference(rule, n, batch), (rule, n, batch)


def test_chunk_tree_plans_refuse_what_does_not_fit(emu):
    m, _, _ = _plan(emu, REDUCE, 2 ** 32 - 1, 256)               # every size the reductions accept: all 8 entries
    assert len(m) == MAX_LEVELS and m[-1] == 1
    assert _plan(emu, REDUCE, 2 ** 36, 1) is None
    m, _, _ = _plan(emu, SCAN, 2 ** 40, 1)
    assert len(m) == MAX_LEVELS and m[-1] == CHUNK
    assert _plan(emu, SCAN, 2 ** 40 + 1, 1) is None
    assert _plan(emu, PRODUCT, 2 ** 41, 3) is None


@pytest.mark.parametrize("count", [1, 3, 256, 65535])
def test_lookup_plan(emu, count):
    for u in (1, 2, 3, 4, 5, 31, 32, 33, 1023, 1024, 1025, 2 ** 20 - 6, 2 ** 30 - 6):
        out = np.zeros(8, dtype=np.uint64)
        emu.emu_lookup_plan(ctypes.c_uint64(u), ctypes.c_uint64(count), out.ctypes.data_as(ctypes.c_void_p))
        N, w, keys, keys_end, sc, left, err, u32_end = (int(x) for x in out)
        assert N & (N - 1) == 0 and max(u, 2) <= N < 2 * max(u, 2), (u, N)
        assert w == u + 1
        assert _disjoint_within([(keys, count * N)], keys_end) == keys_end
        assert _disjoint_within([(sc, 2 * w * count), (left, u * count), (err, 1)], u32_end) == u32_end


@pytest.mark.parametrize("m", [0, 1, 2, 7, 1000, 2 ** 31 - 1])
def test_assembly_layouts(emu, m):
    for S in (0, 1, 2, 255, 256, 257, 2 ** 20, 2 ** 32 - 2):
        edge = np.zeros(13, dtype=np.uint64)
        slot = np.zeros(8, dtype=np.uint64)
        emu.emu_assembly_layouts(ctypes.c_uint64(m), ctypes.c_uint64(S), edge.ctypes.data_as(ctypes.c_void_p), slot.ctypes.data_as(ctypes.c_void_p))
        err, changed, copies, ea, eb, flag, live0, live1, ra, rb, keep, fl, end = (int(x) for x in edge)
        assert err % 2 == 0                                       # a u64
        regions = [(err, 2), (changed, 2), (copies, 4 * m), (ea, m), (eb, m), (flag, m + 1), (live0, m), (live1, m), (ra, m),
                   (rb, m), (keep, m + 1), (fl, m)]
        assert _disjoint_within(regions, end) == end
        ntiles, scell, order0, order1, nxt0, nxt1, counts, send = (int(x) for x in slot)
        assert ntiles == (S + 255) // 256
        regions = [(scell, S), (order0, S), (order1, S), (nxt0, S), (nxt1, S), (counts, 256 * ntiles + 1)]
        assert _disjoint_within(regions, send) == send
