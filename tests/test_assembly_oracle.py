"""CPU checks of the copy-cycle computation from the list of copy constraints (csrc/assembly.cuh, oracle/assembly_oracle.c's
orc_assembly, halo2_b200.CopyConstraints) against the restated reference Assembly::copy (permutation/keygen.rs:45-100):

- the closed form the kernels compute, restated here in Python (the applied copies are Kruskal's spanning forest with
  weight = copy index, and the mapping is the product of its transpositions in copy order, read off by a walk), equals the
  sequential copy loop on random lists, stars, paths in every copy order, cycle-closing and cross-column copies;
- orc_assembly equals the restated loop on the same lists and on the plonk_api and benchmark circuits, first bad copy
  included;
- the device bodies on the host emulation, in the host driver's order, give the same mapping for k = 1 ... 12 and 1 to 8
  columns, including a list that needs every one of the floor(log2 cells) Borůvka rounds, and name the same first bad copy;
- keygen_vk / keygen_pk from CopyConstraints over an ABI stand-in reproduce the test prover's key values."""
import ctypes
import random

import numpy as np
import pytest

from oracle import assembly as orc
from oracle import cref, pasta
from tests import bench_circuit as BC
from tests import fake_engine
from tests import plonk_api_circuit as circ
from tests.bench_circuit import _bench_setup, bench_copies
from tests.fake_engine import emu_assembly
from tests.keygen_cases import oracle_assembly, oracle_copy, oracle_sigma
from tests.kernel_emul import build as emul_build
from tests.plonk_api_circuit import ZETA, plonk_api_copies
from tests.plonk_prover import prover_pk_dict
from tests.plonk_verifier import scalar_delta


# ---- copy lists --------------------------------------------------------------------------------------------------------
def _ordered(copies, order: str, rng):
    copies = list(copies)
    if order == "dec":
        copies.reverse()
    elif order == "shuffle":
        rng.shuffle(copies)
    return copies


def path_copies(cells, cols: int, n: int, order: str, rng):
    """A path through `cells` (flat ids c * n + r), one copy per consecutive pair, in increasing / decreasing / shuffled
    copy order; the ends alternate sides so both (left, right) orientations occur."""
    cps = []
    for j in range(len(cells) - 1):
        a, b = (cells[j], cells[j + 1]) if j % 2 else (cells[j + 1], cells[j])
        cps.append((a // n, a % n, b // n, b % n))
    return _ordered(cps, order, rng)


def star_copies(center: int, leaves, n: int, order: str, rng):
    return _ordered([(center // n, center % n, v // n, v % n) if j % 3 else (v // n, v % n, center // n, center % n)
                     for j, v in enumerate(leaves)], order, rng)


def halving_path(N: int):
    """A path over the first 2^floor(log2 N) cells whose copy order makes Borůvka merge exactly pairs every round: the copy
    between cells p and p + 1 comes in the order of the trailing zeros of p + 1, so the forest takes floor(log2 N) rounds."""
    P = 1 << (N.bit_length() - 1)
    edges = sorted(range(P - 1), key=lambda p: (((p + 1) & -(p + 1)).bit_length(), p))
    return [(p, p + 1) for p in edges]


def copy_lists(rng, cols: int, k: int):
    """(name, list of (lc, lr, rc, rr)) for a permutation of `cols` columns of 2^k rows."""
    n = 1 << k
    N = cols * n
    cell = lambda v: (v // n, v % n)
    out = []
    m = rng.randint(1, 2 * N + 2)
    rnd = [(rng.randrange(cols), rng.randrange(n), rng.randrange(cols), rng.randrange(n)) for _ in range(m)]
    for _ in range(max(1, m // 8)):                                     # duplicates (either orientation) and self-copies
        c = rng.choice(rnd)
        rnd.insert(rng.randrange(len(rnd) + 1), c if rng.random() < 0.5 else (c[2], c[3], c[0], c[1]))
        v = rng.randrange(N)
        rnd.insert(rng.randrange(len(rnd) + 1), cell(v) + cell(v))
    out.append(("random", rnd))
    few = max(2, N // 4)                                                 # large components: copies among a few cells
    pool = rng.sample(range(N), min(N, few))
    out.append(("dense", [cell(rng.choice(pool)) + cell(rng.choice(pool)) for _ in range(2 * len(pool) + 3)]))
    perm = list(range(N))
    rng.shuffle(perm)
    for order in ("inc", "dec", "shuffle"):
        out.append((f"path-{order}", path_copies(perm, cols, n, order, rng)))
        out.append((f"star-{order}", star_copies(perm[0], perm[1:], n, order, rng)))
    closing = path_copies(perm, cols, n, "shuffle", rng) + [cell(perm[-1]) + cell(perm[0])]
    chords = [cell(rng.choice(perm)) + cell(rng.choice(perm)) for _ in range(max(1, N // 8))]
    out.append(("cycle-closing", closing + chords))
    if cols > 1:
        cross = []
        for _ in range(N):
            c0 = rng.randrange(cols)
            c1 = (c0 + rng.randrange(1, cols)) % cols
            cross.append((c0, rng.randrange(n), c1, rng.randrange(n)))
        out.append(("cross-column", cross))
    out.append(("halving", [cell(a) + cell(b) for a, b in halving_path(N)]))
    return out


def restated_mapping(n: int, cols: int, copies):
    """The sequential loop (tests/keygen_cases.oracle_copy) as a (cols, n, 2) uint32 array."""
    asm = oracle_assembly(n, cols)
    for c in copies:
        oracle_copy(asm, *c)
    return np.array(asm[0], dtype=np.uint32).reshape(cols, n, 2)


# ---- 1. the closed form ------------------------------------------------------------------------------------------------
def characterized_mapping(n: int, cols: int, copies):
    """Steps 1-4 of DESIGN.md K20: the applied copies are Kruskal's forest F (weight = copy index: a copy is applied iff
    its two cells are not yet connected), and M(v) is the end of the walk that leaves v by its largest F-edge and then, at
    each cell, by the largest F-edge below the one it arrived by."""
    N = cols * n
    parent = list(range(N))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    slots = [[] for _ in range(N)]                                       # per cell: (copy index, other end), in copy order
    for i, (lc, lr, rc, rr) in enumerate(copies):
        a, b = lc * n + lr, rc * n + rr
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[ra] = rb
            slots[a].append((i, b))
            slots[b].append((i, a))
    out = list(range(N))
    for v in range(N):
        if not slots[v]:
            continue
        i, x = slots[v][-1]
        while True:
            below = [s for s in slots[x] if s[0] < i]
            if not below:
                break
            i, x = below[-1]
        out[v] = x
    return np.array([(x // n, x % n) for x in out], dtype=np.uint32).reshape(cols, n, 2)


def test_closed_form_equals_the_sequential_loop():
    rng = random.Random(20)
    for trial in range(300):
        cols, k = rng.randint(1, 5), rng.randint(0, 5)
        for name, cps in copy_lists(rng, cols, k):
            assert (characterized_mapping(1 << k, cols, cps) == restated_mapping(1 << k, cols, cps)).all(), (trial, name, cols, k)


def test_closed_form_on_tiny_exhaustive_lists():
    """Every list of up to 4 copies over 2 columns of 2 rows."""
    import itertools
    cells = [(c, r) for c in range(2) for r in range(2)]
    copies = [a + b for a in cells for b in cells]
    for m in range(5):
        for cps in itertools.product(copies, repeat=m):
            assert (characterized_mapping(2, 2, cps) == restated_mapping(2, 2, cps)).all(), cps


# ---- 2. orc_assembly ---------------------------------------------------------------------------------------------------
def test_orc_assembly_equals_the_sequential_loop():
    rng = random.Random(21)
    for trial in range(60):
        cols, k = rng.randint(1, 6), rng.randint(0, 7)
        for name, cps in copy_lists(rng, cols, k):
            got, err = orc.assembly(np.array(cps, dtype=np.uint32).reshape(-1, 4), cols, k)
            assert err is None and (got == restated_mapping(1 << k, cols, cps)).all(), (trial, name)


def test_orc_assembly_on_the_test_circuits():
    got, err = orc.assembly(list(plonk_api_copies()), 12, circ.K)
    assert err is None and (got == restated_mapping(circ.N, 12, plonk_api_copies())).all()
    m = pasta.P_MOD
    for k in (5, 8, 10):
        n = 1 << k
        omega = pasta.omega_for_k("fp", k)
        got, err = orc.assembly(list(bench_copies(k)), 3, k)
        assert err is None
        assert oracle_sigma(got, n, omega, scalar_delta(m), m) == BC.columns(k, m, omega, scalar_delta(m), 7)[1]


def _bad_lists(cols: int, n: int):
    """(copies, (kind, first bad index)): the column check comes before the row check within a copy, as in the reference."""
    ok = [(0, 0, cols - 1, n - 1), (0, 1 % n, 0, 0)]
    return [
        (ok + [(cols, 0, 0, 0)] + ok, ("column", 2)),
        (ok + [(0, 0, cols, 0)], ("column", 2)),
        (ok + [(0, n, 0, 0), (cols, 0, 0, 0)], ("row", 2)),
        (ok + [(0, 0, 0, n)], ("row", 2)),
        (ok + [(cols, n, 0, 0)], ("column", 2)),                        # both out of range: the column is reported
        ([(0xFFFFFFFF, 0, 0, 0)] + ok, ("column", 0)),
        (ok * 3 + [(0, 0xFFFFFFFF, 0, 0)], ("row", 6)),
    ]


def test_orc_assembly_first_bad_copy():
    for cols, k in ((1, 0), (3, 4), (8, 2)):
        n = 1 << k
        for cps, want in _bad_lists(cols, n):
            assert orc.assembly(np.array(cps, dtype=np.uint32), cols, k) == (None, want)
            asm = oracle_assembly(n, cols)
            with pytest.raises((IndexError, ValueError)):                    # the restated loop fails at the same copy
                for j, c in enumerate(cps):
                    if c[0] >= cols or c[2] >= cols:
                        raise ValueError(j)
                    oracle_copy(asm, *c)
            assert j == want[1]


# ---- 3. the device bodies on the host emulation ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emul_build.build())


@pytest.mark.parametrize("k", range(1, 13))
def test_emul_assembly_matches_the_oracle(emu, k):
    rng = random.Random(100 + k)
    for cols in ((1, 2, 3, 5, 8) if k <= 8 else (1, 3, 8)):
        N = cols << k
        for name, cps in copy_lists(rng, cols, k):
            want, err = orc.assembly(np.array(cps, dtype=np.uint32).reshape(-1, 4), cols, k)
            assert err is None
            if N <= 512:
                assert (want == restated_mapping(1 << k, cols, cps)).all()
            rc, got, _, rounds, forest = emu_assembly(emu, cps, cols, k)
            assert rc == 0 and (got == want).all(), (k, cols, name)
            assert rounds <= N.bit_length() - 1
            if name == "halving":
                assert rounds == N.bit_length() - 1 and forest == (1 << (N.bit_length() - 1)) - 1
            if name.startswith(("path", "star")):
                assert forest == N - 1


def test_emul_assembly_edge_cases(emu):
    for cols, k in ((1, 0), (2, 0), (1, 1), (4, 3)):
        n = 1 << k
        N = cols * n
        ident = np.stack(np.meshgrid(np.arange(cols), np.arange(n), indexing="ij"), axis=-1).astype(np.uint32)
        for cps in ([], [(0, 0, 0, 0)] * 3):                              # no copies, only self-copies: the identity
            rc, got, _, rounds, forest = emu_assembly(emu, cps, cols, k)
            assert rc == 0 and (got == ident).all() and rounds == forest == 0
        if N > 1:
            cps = [(0, 0, (N - 1) // n, (N - 1) % n)] * 4                  # one copy, repeated: one transposition
            rc, got, _, rounds, forest = emu_assembly(emu, cps, cols, k)
            assert rc == 0 and (got == restated_mapping(n, cols, cps)).all() and rounds == forest == 1
    # a star of degree 2^12 - 1 around a cell in the middle, copied in random order
    k, cols = 12, 1
    rng = random.Random(7)
    leaves = [v for v in range(1 << k) if v != 1000]
    cps = star_copies(1000, leaves, 1 << k, "shuffle", rng)
    rc, got, _, _, forest = emu_assembly(emu, cps, cols, k)
    assert rc == 0 and forest == len(leaves) and (got == orc.assembly(cps, cols, k)[0]).all()


def test_emul_assembly_first_bad_copy(emu):
    for cols, k in ((1, 0), (3, 4), (8, 2)):
        for cps, (kind, idx) in _bad_lists(cols, 1 << k):
            rc, _, bad, _, _ = emu_assembly(emu, cps, cols, k)
            assert rc == 1 and bad == 2 * idx + (kind == "row"), (cps, bad)


# ---- 4. CopyConstraints ------------------------------------------------------------------------------------------------
def test_copy_constraints_checks_and_records():
    import halo2_b200 as h2
    cc = h2.CopyConstraints(8, 3)
    cc.copy(0, 7, 2, 0)
    for bad in ((0, 8, 1, 0), (0, 0, 1, 8), (0, -1, 1, 0)):
        with pytest.raises(IndexError):
            cc.copy(*bad)
    for bad in ((3, 0, 1, 0), (0, 0, -1, 0), (3, 9, 1, 0)):               # a bad column is reported before a bad row
        with pytest.raises(ValueError):
            cc.copy(*bad)
    cc.extend(np.array([[1, 2, 1, 3], [2, 5, 0, 0]], dtype=np.int64))
    cc.copy(1, 1, 1, 1)
    with pytest.raises(IndexError, match="copy 1"):
        cc.extend([[0, 0, 0, 0], [0, 8, 0, 0], [5, 0, 0, 0]])
    with pytest.raises(ValueError, match="copy 2"):
        cc.extend(np.array([[0, 0, 0, 0], [0, 1, 0, 0], [5, 9, 0, 0]], dtype=np.uint32))
    with pytest.raises(TypeError):
        cc.extend(np.zeros((2, 3), dtype=np.int64))
    cc.extend(np.zeros((0, 4), dtype=np.int64))
    assert len(cc) == 4
    assert cc.copies.tolist() == [[0, 7, 2, 0], [1, 2, 1, 3], [2, 5, 0, 0], [1, 1, 1, 1]] and cc.copies.dtype == np.uint32


def test_keygen_from_copy_constraints_reproduces_the_test_provers_key():
    """keygen_vk / keygen_pk given CopyConstraints at k = 5: the same commitments and key values as from the Assembly
    (which test_keygen_oracle ties to the test prover's own key), through one copies call each, and the same proof bytes."""
    import halo2_b200 as h2
    from tests import multiopen_cases as MC
    from tests import plonk_prover as PP
    from tests import plonk_verifier as PV
    from tests import prover_replay as R
    k = 5
    c, m, gens, fixed, sigma, adv, copies = _bench_setup(k)
    n = 1 << k
    delta = scalar_delta(m)
    with fake_engine.installed() as fake:
        prm = h2.Params("vesta", k, *gens[:3], u=gens[3])
        D = h2.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
        cc = h2.CopyConstraints(n, 3)
        cc.extend(np.array(copies[:7]))
        for cp in copies[7:]:
            cc.copy(*cp)
        fc, pc = h2.keygen_vk(prm, D, fixed, cc, delta)
        assert fake.calls.count("h2_poly_permutation_sigma_copies") == 1 and "h2_poly_permutation_sigma" not in fake.calls
        assert not fake.polys
        A = cref.bytes_to_affine
        cl = lambda v: pasta.to_affine(c, pasta.best_multiexp(c, list(v) + [1], [A(x) for x in gens[1]] + [A(gens[2][0])]))
        assert [A(x) for x in fc] == [cl(f) for f in fixed] and [A(x) for x in pc] == [cl(s) for s in sigma]
        vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, c.p, m, D.omega, [A(x) for x in fc], [A(x) for x in pc]))
        asm = h2.Assembly(n, 3)
        for cp in copies:
            asm.copy(*cp)
        fake.calls.clear()
        pk = h2.keygen_pk(prm, D, fixed, cc, delta, BC.BLINDING_FACTORS)
        ref = h2.keygen_pk(prm, D, fixed, asm, delta, BC.BLINDING_FACTORS)
        assert fake.calls.count("h2_poly_permutation_sigma_copies") == 1 and fake.calls.count("h2_poly_permutation_sigma") == 1
        mine, theirs = prover_pk_dict(pk), prover_pk_dict(ref)
        for key in ("fixed_l", "fixed_p", "fixed_c", "sigma_l", "sigma_p", "sigma_c", "l"):
            for a, b in zip(mine[key], theirs[key]):
                assert (a.download() == b.download()).all(), key
        assert [cref.bytes_to_ints(p.download()) for p in pk.permutation.permutations] == sigma
        adv_bytes = [cref.ints_to_bytes(col) for col in adv]
        proofs = []
        for key in (mine, theirs):
            T = R.Blake2bTranscript(m)
            PP.create_proof_engine(h2, prm, vk, None, None, [adv_bytes], [[]], MC.SeededRng("fp", 5, True), T, ZETA, delta, pk=key)
            proofs.append(bytes(T.proof))
        assert proofs[0] == proofs[1]
        pk.close()
        ref.close()
        # a bad copy that reached the library (bypassing CopyConstraints' own checks) fails the call and frees its outputs
        bad = h2.CopyConstraints(n, 3)
        bad._arrays.append(np.array([[0, 0, 1, 1], [0, n, 1, 1]], dtype=np.uint32))
        with pytest.raises(h2.H2Error, match="copy 1: a row"):
            h2.build_permutation_polys(D, bad, delta)
        assert not fake.polys
        prm.close()


def test_plonk_api_copies_through_copy_constraints():
    """The plonk_api circuit's copies give the sigma columns the test circuit pins (the golden commitments on the GPU)."""
    import halo2_b200 as h2
    m = pasta.P_MOD
    omega, delta = pasta.omega_for_k("fp", circ.K), scalar_delta(m)
    with fake_engine.installed():
        D = h2.EvaluationDomain("fp", 4, circ.K, ZETA)
        assert D.omega == omega
        cc = h2.CopyConstraints(circ.N, 12)
        cc.extend(np.array(list(plonk_api_copies())))
        polys = h2.build_permutation_polys(D, cc, delta)
        got = [cref.bytes_to_ints(p.download()) for p in polys]
        for p in polys:
            p.close()
    assert got == circ.permutation_columns(m, omega, delta)
