"""The batched lookup permutation (csrc/lookup.cuh, h2_poly_lookup_permuted) without a GPU: its kernel bodies run on the host
emulation in capi_poly.cu's launch schedule and must give permute_expression_pair (plonk/lookup/prover.rs:563-647,
oracle/pasta.py) for every lookup of a call, plus the caller's blinding rows; a miss is reported at the lowest failing lookup
and changes nothing.  Then halo2_b200.lookup_commit_permuted, the whole of commit_permuted for every proof, runs over the ABI
stand-in on the reference's plonk_api circuit and gives the permuted commitments of a real proof at their offsets."""
import ctypes
import random

import pytest

from oracle import cref, pasta
from tests import fake_engine
from tests import multiopen_cases as MC
from tests import plonk_api_circuit as circ
from tests import prover_replay as R
from tests.fake_engine import NONE
from tests.kernel_emul import build as emul_build


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emul_build.build())


def emu_permuted(emu, field, inputs, tables, k, bf, blinding, marker):
    """One emulated call over len(inputs) lookups: returns (status, permuted inputs, permuted tables) as ints per lookup."""
    count, n, rows = len(inputs), 1 << k, bf + 1
    flat = lambda cols: cref.ints_to_bytes([x for c in cols for x in c])
    oa, ot = flat([marker] * count), flat([marker] * count)
    emu.emu_lookup_permuted.restype = ctypes.c_uint32
    rc = emu.emu_lookup_permuted(cref.FIELD_ID[field], cref._p(flat(inputs)), cref._p(flat(tables)), ctypes.c_uint32(count), ctypes.c_size_t(n),
                                 ctypes.c_size_t(n - rows), cref._p(cref.ints_to_bytes(blinding)), ctypes.c_size_t(rows), cref._p(oa), cref._p(ot))
    a, t = cref.bytes_to_ints(oa), cref.bytes_to_ints(ot)
    return rc, [a[b * n:(b + 1) * n] for b in range(count)], [t[b * n:(b + 1) * n] for b in range(count)]


def _lookup(rnd, m, u, n, kind):
    """(input column, table column) of n rows whose usable rows [0, u) satisfy the lookup."""
    if kind == "one_value":                                        # every row one value (a selector that is off)
        tab = [rnd.randrange(m) for _ in range(u)]
        inp = [tab[0]] * u
    elif kind == "hot":                                            # 90 % of the rows on one value
        tab = [rnd.randrange(1 << 8) for _ in range(u)]
        inp = [tab[0] if rnd.random() < 0.9 else rnd.choice(tab) for _ in range(u)]
    elif kind == "dup_table":                                      # a table of few distinct values, each many times
        pool = [rnd.randrange(m) for _ in range(max(1, u // 8))]
        tab = [rnd.choice(pool) for _ in range(u)]
        inp = [rnd.choice(tab) for _ in range(u)]
    elif kind == "no_leftover":                                    # the input is a permutation of the table: every value consumed
        tab = [rnd.randrange(m) for _ in range(u)]
        inp = list(tab)
        rnd.shuffle(inp)
    elif kind == "small":                                          # small integers: the high limbs of every key tie
        tab = [rnd.randrange(1 << 10) for _ in range(u)]
        inp = [rnd.choice(tab) for _ in range(u)]
    else:                                                          # full width, with p - 1 (the largest key below the padding)
        tab = [rnd.randrange(m) for _ in range(u)]
        tab[rnd.randrange(u)] = m - 1
        inp = [rnd.choice(tab) for _ in range(u)]
        inp[rnd.randrange(u)] = m - 1
    tail = [rnd.randrange(m) for _ in range(n - u)]
    return inp + tail, tab + tail


KINDS = ["one_value", "hot", "dup_table", "no_leftover", "small", "full"]


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("k,bf", [(1, 0), (2, 1), (3, 2), (6, 5), (7, 0), (9, 5), (11, 12)])   # u = 1, 2, 5, 58, 127, 506, 2035
def test_emulated_bodies_equal_the_reference(emu, field, k, bf):
    m = pasta.FIELDS[field]
    rnd = random.Random(k * 31 + bf)
    n, rows = 1 << k, bf + 1
    u = n - rows
    pairs = [_lookup(rnd, m, u, n, kind) for kind in KINDS]
    blinding = [rnd.randrange(m) for _ in range(len(pairs) * 2 * rows)]
    marker = [424242 + i for i in range(n)]
    rc, ga, gt = emu_permuted(emu, field, [p[0] for p in pairs], [p[1] for p in pairs], k, bf, blinding, marker)
    assert rc == NONE
    for b, (inp, tab) in enumerate(pairs):
        want_a, want_s = pasta.permute_expression_pair(field, inp[:u], tab[:u], u)
        blind = blinding[b * 2 * rows:(b + 1) * 2 * rows]
        assert ga[b] == want_a + blind[:rows], (KINDS[b], k)
        assert gt[b] == want_s + blind[rows:], (KINDS[b], k)


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_a_miss_names_the_lowest_lookup_and_writes_nothing(emu, field):
    m = pasta.FIELDS[field]
    rnd = random.Random(3)
    k, bf = 6, 3
    n, u = 1 << k, (1 << k) - bf - 1
    pairs = [_lookup(rnd, m, u, n, "small") for _ in range(5)]
    marker = [99 + i for i in range(n)]
    blinding = [rnd.randrange(m) for _ in range(5 * 2 * (bf + 1))]
    for bad in ([3], [1, 4], [0, 2, 3], [4]):
        inputs = [list(p[0]) for p in pairs]
        for b in bad:
            inputs[b][rnd.randrange(u)] = (1 << 10) + 5              # no table holds it
        rc, ga, gt = emu_permuted(emu, field, inputs, [p[1] for p in pairs], k, bf, blinding, marker)
        assert rc == min(bad)
        assert all(col == marker for col in ga + gt)                # the blinding rows too
    # a value only in a row past the usable ones is no miss
    inputs = [list(p[0]) for p in pairs]
    inputs[2][u] = (1 << 10) + 5
    assert emu_permuted(emu, field, inputs, [p[1] for p in pairs], k, bf, blinding, marker)[0] == NONE


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_rank_form_equals_the_two_sort_form(emu, field):
    """h2_poly_lookup_permute's shape (any usable_rows, no blinding rows, rows past usable_rows untouched): the rank form, one
    lookup, gives the bytes of K17's two-sort bodies (emu_lookup_permute), and both fail on the same miss."""
    m = pasta.FIELDS[field]
    rnd = random.Random(17)
    emu.emu_lookup_permuted.restype = ctypes.c_uint32
    for n, u in ((4, 1), (4, 3), (8, 8), (40, 33), (300, 257), (1024, 1000)):
        for kind in KINDS:
            inp, tab = _lookup(rnd, m, u, n, kind)
            marker = cref.ints_to_bytes([31337 + i for i in range(n)])
            two = [marker.copy(), marker.copy()]
            rank = [marker.copy(), marker.copy()]
            a, t = cref.ints_to_bytes(inp), cref.ints_to_bytes(tab)
            rc2 = emu.emu_lookup_permute(cref.FIELD_ID[field], cref._p(a), cref._p(t), ctypes.c_size_t(n), ctypes.c_size_t(u), cref._p(two[0]), cref._p(two[1]))
            rc1 = emu.emu_lookup_permuted(cref.FIELD_ID[field], cref._p(a), cref._p(t), ctypes.c_uint32(1), ctypes.c_size_t(n), ctypes.c_size_t(u), None,
                                          ctypes.c_size_t(0), cref._p(rank[0]), cref._p(rank[1]))
            assert rc2 == 0 and rc1 == NONE
            assert (two[0] == rank[0]).all() and (two[1] == rank[1]).all(), (n, u, kind)
            missing = (max(tab[:u]) + 1) % m
            bad = list(inp)
            bad[rnd.randrange(u)] = missing
            b = cref.ints_to_bytes(bad)
            rc2 = emu.emu_lookup_permute(cref.FIELD_ID[field], cref._p(b), cref._p(t), ctypes.c_size_t(n), ctypes.c_size_t(u), cref._p(two[0]), cref._p(two[1]))
            rc1 = emu.emu_lookup_permuted(cref.FIELD_ID[field], cref._p(b), cref._p(t), ctypes.c_uint32(1), ctypes.c_size_t(n), ctypes.c_size_t(u), None,
                                          ctypes.c_size_t(0), cref._p(rank[0]), cref._p(rank[1]))
            assert (rc2 == 1) == (rc1 == 0) == (missing not in set(tab[:u]))


def test_commit_permuted_of_the_plonk_api_proof():
    """create_proof_engine (its per-lookup composition) proves the plonk_api circuit (k = 5, two proofs, one lookup each) over
    the stand-in while the Lagrange columns, theta and the rng's draws are recorded.  lookup_commit_permuted, fed the same,
    makes one permute call and gives the four permuted commitments the proof holds at their offsets, and draws as many values."""
    import halo2_b200
    vk = circ.plonk_api_key()
    bf = vk.blinding_factors()
    with fake_engine.installed() as fake:
        g, gl, w, u = _gens()
        prm = halo2_b200.Params("vesta", 5, g, gl, w, u=u)
        proof, seen = circ.plonk_api_proof(halo2_b200, prm)
        assert fake.calls.count("h2_poly_lookup_permute") == 2 and len(vk.lookups) == 1
        assert "h2_poly_lookup_permuted" not in fake.calls
        D, ev, lookups = circ.plonk_api_lookups(halo2_b200, seen)
        replay = MC.ReplayRng(seen["draws"][seen["draws_at_theta"]:])
        before = len(replay.draws)
        perm, cm = halo2_b200.lookup_commit_permuted(prm, D, ev, lookups, seen["theta"], bf, replay)
        assert fake.calls.count("h2_poly_lookup_permuted") == 1
        assert before - len(replay.draws) == 2 * (2 * (bf + 1) + 2)
        at = 32 * seen["points_at_theta"]
        assert len(cm) == 4 and proof[at:at + 32 * len(cm)] == R._encode(cm, circ.M)
        assert [len(per) for per in perm] == [1, 1] and isinstance(perm[0][0], halo2_b200.Permuted)
        for per in perm:
            for q in per:
                for p in q[:8]:
                    p.close()
        for p in ev.polys:
            p.close()
        prm.close()


def _gens():
    c = pasta.VESTA
    P = pasta.Params.new(c, 5)
    return cref.affines_to_bytes(P.g), cref.affines_to_bytes(P.g_lagrange), cref.affines_to_bytes([P.w]), cref.affines_to_bytes([P.u])
