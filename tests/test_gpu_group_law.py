"""The device group law on its degenerate cases, against the oracle (oracle/pasta.py), exactly, as canonical affine bytes.

Element by element (h2_test_curve_op ops 3 - 13): every XYZZ form -- serial, lane-cooperative and the EC-FFT's warp-uniform
ones -- on operands rescaled to ZZ != 1 (ZZ = 1 on every 4th element), so that its P + P, P + (-P) and identity branches
compare the projective quantities they are meant to compare.  The cases are interleaved with a period of 11, so the quads and
pairs of one warp take different branches; whole warps of a single case follow, and the element count leaves the last warp
partly filled.  The cooperative ops also check that the lanes of a quad or pair end with equal values.

Whole MSMs (one-shot on every accumulation path, fixed-base on both tables, batched commits, IPA rounds) over bases drawn
from a small support S = {P, -P, 2P, Q, -Q, O}: a bucket then holds many copies of a few points and their negatives, its
running sum walks over small combinations aP + bQ (and their phi images under GLV) and often equals +-the next point, so the
degenerate branches run with non-trivial ZZ in the accumulation kernels, the partial merges and the reduce -- whatever order
the atomics produce.  That is a probability argument; how often each branch runs is not counted on the device.  The expected
value sum_j (sum_{i: base_i = S_j} k_i mod r) S_j = aP + bQ is two oracle scalar multiplications at any n.  Each MSM case
asserts through h2_test_last_msm_plan / h2_test_last_msm_flags that it ran the path it is meant to cover."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402

SEED = 0x4C4157
CURVES = ["pallas", "vesta"]
ADD_OPS = (3, 4, 7, 8, 9, 11)       # a + b: xyzz_add, xyzz_add_mixed, the quad / mixed quad / pair forms, xyzz_addsub_q's sum
SUB_OP = 12                         # xyzz_addsub_q's difference a - b
DBL_OPS = (5, 13)                   # xyzz_double, xyzz_double_q
SHIFT_OPS = (6, 10)                 # xyzz_shift, xyzz_shift_quad
PLAN_KEYS = ("mode", "c", "W", "sets", "accum", "natural", "fast", "rerun")


def _ways(ways, log2_refs=20):
    """h2_test_set_accum_ways: lanes per work item, and up to how many references (2^20 by default) lanes cooperate."""
    return ways | (log2_refs << 8)


ACCUM_WAYS_DEFAULT = _ways(12)


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


def _lib():
    from halo2_b200 import lib as L
    return L, L.init()


def _curve_op(curve, op, a, b):
    L, lib = _lib()
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    out = np.zeros_like(a)
    L.check(lib.h2_test_curve_op(L.CURVE_ID[curve], op, L.ptr(a), L.ptr(b), ctypes.c_size_t(a.shape[0]), L.ptr(out)))
    return out


def _plan():
    L, lib = _lib()
    out = (ctypes.c_uint32 * 8)()
    L.check(lib.h2_test_last_msm_plan(out))
    return dict(zip(PLAN_KEYS, list(out)))


def _flags():
    L, lib = _lib()
    f = ctypes.c_uint32(0)
    L.check(lib.h2_test_last_msm_flags(ctypes.byref(f)))
    return f.value


def _neg(c, p):
    return None if p is None else (p[0], (c.p - p[1]) % c.p)


def _add(c, a, b):
    return pasta.to_affine(c, pasta.jac_add(c, pasta.to_jac(a), pasta.to_jac(b)))


def _dbl(c, a):
    return pasta.to_affine(c, pasta.jac_double(c, pasta.to_jac(a)))


def _points(curve, seed, n):
    return [cref.bytes_to_affine(p) for p in cref.gen_points(curve, seed, n)]


def _check(got, want, what, labels):
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, (what, int(bad.size), [(int(i), labels[i]) for i in bad[:8]])


# ------------------------------------------------------------------------------------------ element by element
KINDS = ("P+Q", "P+P", "P-P", "O+P", "P+O", "O+O", "P+2P", "2P+P", "G+G", "G-G", "G+Q")   # 11: not a multiple of 2, 4 or 8


def _pair(c, kind, p, q):
    g = pasta.generator(c)
    return {"P+Q": (p, q), "P+P": (p, p), "P-P": (p, _neg(c, p)), "O+P": (None, p), "P+O": (p, None), "O+O": (None, None),
            "P+2P": (p, _dbl(c, p)), "2P+P": (_dbl(c, p), p), "G+G": (g, g), "G-G": (g, _neg(c, g)), "G+Q": (g, q)}[kind]


def _add_cases(curve):
    """(a, b, labels): 11 interleaved kinds x 40, 16 elements (a whole warp of pairs, two of quads) of each kind in turn, a few
    thousand random pairs; 3 + 440 + 176 + 3000 elements, not a multiple of 8."""
    c = pasta.CURVES[curve]
    pts = _points(curve, SEED + 1, 2 * (440 + 176) + 2 * 3000 + 6)
    it = iter(pts)
    a, b, labels = [], [], []

    def put(kind):
        x, y = _pair(c, kind, next(it), next(it)) if kind != "random" else (next(it), next(it))
        a.append(x)
        b.append(y)
        labels.append(kind)
    for kind in ("P+P", "P-P", "O+P"):
        put(kind)
    for i in range(440):
        put(KINDS[i % len(KINDS)])
    for kind in KINDS:
        for _ in range(16):
            put(kind)
    for _ in range(3000):
        put("random")
    assert len(a) % 8 != 0
    return a, b, labels


@pytest.mark.parametrize("curve", CURVES)
def test_group_law_add_double(eng, curve):
    """a + b (ops 3, 4, 7, 8, 9, 11), a - b (op 12) and 2a (ops 5, 13) on every case kind, against pasta's Jacobian law."""
    c = pasta.CURVES[curve]
    a, b, labels = _add_cases(curve)
    A, B = cref.affines_to_bytes(a), cref.affines_to_bytes(b)
    want_sum = cref.affines_to_bytes([_add(c, x, y) for x, y in zip(a, b)])
    want_diff = cref.affines_to_bytes([_add(c, x, _neg(c, y)) for x, y in zip(a, b)])
    want_dbl = cref.affines_to_bytes([_dbl(c, x) for x in a])
    for op in ADD_OPS:
        _check(_curve_op(curve, op, A, B), want_sum, (curve, op), labels)
    _check(_curve_op(curve, SUB_OP, A, B), want_diff, (curve, SUB_OP), labels)
    for op in DBL_OPS:
        _check(_curve_op(curve, op, A, B), want_dbl, (curve, op), labels)


SHIFTS = [0, 1, 2, 3] + list(range(4, 21)) + [31, 32, 63, 64, 100, 127, 128, 254, 255, 256, 269, 270]   # 33 counts


@pytest.mark.parametrize("curve", CURVES)
def test_group_law_shift(eng, curve):
    """2^k a (ops 6, 10): k = 0 - 3 (the doubling loop), 4 - 20 and the window-combine range up to 270 (the Jacobian chain), on
    random points, the generator and the identity; interleaved, then whole warps of one count."""
    c = pasta.CURVES[curve]
    g = pasta.generator(c)
    pts = iter(_points(curve, SEED + 2, 500))
    a, ks = [], []
    for i in range(3 * len(SHIFTS) * 4 - 1):
        ks.append(SHIFTS[i % len(SHIFTS)])
        form = (i // len(SHIFTS)) % 4
        a.append(next(pts) if form == 0 else g if form == 1 else None if form == 2 else _neg(c, next(pts)))
    for k in (2, 5, 270):
        for _ in range(16):
            ks.append(k)
            a.append(next(pts))
    B = np.zeros((len(a), 64), dtype=np.uint8)
    B[:, :4] = np.array(ks, dtype="<u4").view(np.uint8).reshape(-1, 4)
    want = cref.affines_to_bytes([pasta.to_affine(c, pasta.scalar_mul(c, pow(2, k, c.r), p)) for p, k in zip(a, ks)])
    labels = [("k", k, "O" if p is None else "G" if p == g else "P") for p, k in zip(a, ks)]
    for op in SHIFT_OPS:
        _check(_curve_op(curve, op, cref.affines_to_bytes(a), B), want, (curve, op), labels)


def test_group_law_unknown_op(eng):
    L, lib = _lib()
    a = np.zeros((4, 64), dtype=np.uint8)
    out = np.zeros_like(a)
    for op in (-1, 14, 99):
        assert lib.h2_test_curve_op(L.CURVE_ID["pallas"], op, L.ptr(a), L.ptr(a), ctypes.c_size_t(4), L.ptr(out)) != 0, op
        assert b"op must be" in lib.h2_last_error(), op


@pytest.mark.parametrize("curve", CURVES)
def test_point_sum_projective_partials(eng, curve):
    """h2_point_sum on Jacobian partials with Z != 1 (converted to XYZZ inside the kernel): equal, opposite and identity partials,
    and running sums that meet +-the next partial."""
    L, lib = _lib()
    c = pasta.CURVES[curve]
    p, q, *rest = _points(curve, SEED + 3, 8)
    zs = iter(pasta.gen_scalars(c.base, SEED + 4, 64))
    pq = _add(c, p, q)

    def jac(pt):
        if pt is None:
            return (3, 7, 0)                              # any x, y with z = 0 is the identity
        z = next(zs) or 1
        return (pt[0] * z * z % c.p, pt[1] * z * z * z % c.p, z)
    seqs = [[p, p], [p, _neg(c, p)], [None, p, None], [p, p, _neg(c, _dbl(c, p))], [p, q, pq], [p, q, _neg(c, pq), p],
            [None, None], [p, _neg(c, p), p, p], rest]
    for seq in seqs:
        want = None
        for pt in seq:
            want = _add(c, want, pt)
        parts = cref.ints_to_bytes([v for pt in seq for v in jac(pt)]).reshape(-1, 96)
        out = np.zeros(96, dtype=np.uint8)
        L.check(lib.h2_point_sum(L.CURVE_ID[curve], L.ptr(parts), ctypes.c_size_t(len(seq)), L.REPR_CANONICAL, L.ptr(out)))
        assert cref.bytes_to_affine(cref.jac_to_affine(curve, out)) == want, (curve, len(seq))


# ------------------------------------------------------------------------------------------ whole MSMs over a small support
class Support:
    """S = {P, -P, 2P, Q, -Q, O}; a term (k, S_j) contributes k * coef_j to a in aP + bQ."""

    def __init__(self, curve, seed):
        self.curve, self.c = curve, pasta.CURVES[curve]
        p, q = _points(curve, seed, 2)
        self.p, self.q = p, q
        self.points = [p, _neg(self.c, p), _dbl(self.c, p), q, _neg(self.c, q), None]
        self.coef = [(1, 0), (-1, 0), (2, 0), (0, 1), (0, -1), (0, 0)]
        self.bytes = cref.affines_to_bytes(self.points)

    def bases(self, idx):
        return np.ascontiguousarray(self.bytes[idx])

    def want(self, scalars, idx):
        """The affine point sum_i k_i S_{idx_i}."""
        r = self.c.r
        ks = cref.bytes_to_ints(scalars)
        sums = [0] * len(self.points)
        for k, j in zip(ks, np.asarray(idx).tolist()):
            sums[j] += k
        a = sum(s * cp for s, (cp, _) in zip(sums, self.coef)) % r
        b = sum(s * cq for s, (_, cq) in zip(sums, self.coef)) % r
        return pasta.to_affine(self.c, pasta.jac_add(self.c, pasta.scalar_mul(self.c, a, self.p), pasta.scalar_mul(self.c, b, self.q)))


def _affine(curve, xyz):
    return cref.bytes_to_affine(cref.jac_to_affine(curve, xyz))


def _columns(curve, n, seed):
    """Uniform scalars, and a skewed column (small integers and one repeated value: its bins overflow)."""
    c = pasta.CURVES[curve]
    one = pasta.gen_scalars(c.scalar, seed + 1, 1)[0]
    return {"uniform": cref.gen_scalars(c.scalar, seed, n), "skewed": cref.ints_to_bytes([one if i % 3 else i % 7 for i in range(n)])}


# (name, accum_ways hook, batched-affine rounds, exact sort, accumulation: 0 cooperating lanes / 1 thread per item)
ONE_SHOT_PATHS = [
    ("split2", _ways(12), 0, 0, 0), ("split4", _ways(14), 0, 0, 0), ("pair", _ways(0), 0, 0, 0), ("quad1", _ways(1), 0, 0, 0),
    ("quad2", _ways(2), 0, 0, 0), ("quad4", _ways(4), 0, 0, 0), ("thread", _ways(12, 8), 0, 0, 1), ("ba1", _ways(12, 8), 1, 0, 1),
    ("ba2", _ways(12, 8), 2, 0, 1), ("ba3", _ways(12, 8), 3, 0, 1), ("exact", _ways(12), 0, 1, 0),
]


@pytest.mark.parametrize("curve", CURVES)
def test_msm_small_support_one_shot(eng, curve):
    """h2_msm at n = 4099 over the support, uniform and skewed scalars, GLV on and off, on every accumulation of small MSMs (2 / 4
    independent lanes, a cooperating pair, 1 / 2 / 4 quads), a thread per work item, 1 - 3 batched-affine rounds and the exact sort;
    then chunked upload (forced at this n)."""
    L, lib = _lib()
    n = 4099
    S = Support(curve, SEED + 10)
    idx = np.random.default_rng(SEED + 11).integers(0, len(S.points), n)
    pb = S.bases(idx)
    cols = _columns(curve, n, SEED + 12)
    wants = {name: S.want(kb, idx) for name, kb in cols.items()}
    try:
        for name, ways, ba, exact, accum in ONE_SHOT_PATHS:
            L.check(lib.h2_test_set_accum_ways(ways))
            L.check(lib.h2_test_set_batched_affine(ba, 32))
            L.check(lib.h2_set_sort_mode(exact))
            for glv in (1, 0):
                L.check(lib.h2_set_glv(glv))
                for col, kb in cols.items():
                    assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == wants[col], (name, glv, col)
                    p = _plan()
                    assert (p["mode"], p["accum"]) == (0, accum), (name, glv, col, p)
                    if exact:
                        assert _flags() & 2, (name, glv, col)
                    elif ba and col == "uniform":
                        assert not _flags() & 2, ("the exact sort ran: the batched-affine rounds were skipped", name, glv)
        L.check(lib.h2_test_set_accum_ways(ACCUM_WAYS_DEFAULT))
        L.check(lib.h2_test_set_batched_affine(0, 32))
        L.check(lib.h2_set_sort_mode(0))
        for thr in (4, 11):                               # 4 and 3 upload chunks
            L.check(lib.h2_test_set_chunk_threshold(thr))
            for glv in (1, 0):
                L.check(lib.h2_set_glv(glv))
                for col, kb in cols.items():
                    assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == wants[col], ("chunked", thr, glv, col)
                    assert _plan()["mode"] == 0
    finally:
        L.check(lib.h2_test_set_accum_ways(ACCUM_WAYS_DEFAULT))
        L.check(lib.h2_test_set_batched_affine(0, 32))
        L.check(lib.h2_set_sort_mode(0))
        L.check(lib.h2_set_glv(1))
        L.check(lib.h2_test_set_chunk_threshold(19))


def test_msm_small_support_production_size(eng):
    """n = 2^20 + 1 with the default settings: chunked upload and a thread per work item."""
    curve = "pallas"
    n = (1 << 20) + 1
    S = Support(curve, SEED + 20)
    idx = np.random.default_rng(SEED + 21).integers(0, len(S.points), n)
    kb = cref.gen_scalars(pasta.CURVES[curve].scalar, SEED + 22, n)
    assert _affine(curve, eng.best_multiexp(kb, S.bases(idx), curve)) == S.want(kb, idx)
    p = _plan()
    assert (p["mode"], p["accum"]) == (0, 1), p


@pytest.mark.parametrize("curve", CURVES)
def test_msm_small_support_fixed_base(eng, curve):
    """Params whose g, g_lagrange, w and u are drawn from the support: commits on the window table's fast pass (buckets in index
    order, and sorted work items under 4 quads per item) and its re-run (skewed column), on the digit-multiples table (direct
    sum), commit_many, and the IPA round loop against the oracle's."""
    L, lib = _lib()
    c = pasta.CURVES[curve]
    k = 10
    n = 1 << k
    S = Support(curve, SEED + 30)
    rng = np.random.default_rng(SEED + 31)
    gi, gli = rng.integers(0, len(S.points), n), rng.integers(0, len(S.points), n)
    wi, ui = 2, 3                                         # w = 2P, u = Q
    cols = _columns(curve, n, SEED + 32)
    polys = [cols["uniform"], cols["skewed"], cref.gen_scalars(c.scalar, SEED + 33, n)]
    blinds = pasta.gen_scalars(c.scalar, SEED + 34, len(polys))
    idx_g, idx_gl = np.concatenate([gi, [wi]]), np.concatenate([gli, [wi]])
    want = [S.want(np.concatenate([p, cref.ints_to_bytes([b])]), idx_g) for p, b in zip(polys, blinds)]
    want_l = [S.want(np.concatenate([p, cref.ints_to_bytes([b])]), idx_gl) for p, b in zip(polys, blinds)]
    bases = S.bases(np.concatenate([gi, [wi, ui]]))
    ch = pasta.gen_scalars(c.scalar, SEED + 35, k)
    lr = pasta.gen_scalars(c.scalar, SEED + 36, k)
    rr = pasta.gen_scalars(c.scalar, SEED + 37, k)
    x3, z = pasta.gen_scalars(c.scalar, SEED + 38, 2)
    ipa_l, ipa_r, ipa_c = cref.ipa_rounds(curve, bases, k, polys[0], x3, z, cref.ints_to_bytes(ch), cref.ints_to_bytes(lr), cref.ints_to_bytes(rr))
    try:
        for direct in (False, True):
            params = eng.Params(curve, k, S.bases(gi), S.bases(gli), S.bases([wi]), u=S.bases([ui]), direct=direct)
            try:
                for ways, natural in ((ACCUM_WAYS_DEFAULT, 1), (_ways(4), 0)):
                    L.check(lib.h2_test_set_accum_ways(ways))
                    for rep in range(3):                  # eager, captured, replayed
                        for i, (poly, b) in enumerate(zip(polys, blinds)):
                            assert _affine(curve, params.commit(poly, eng.Blind(b))) == want[i], (direct, ways, rep, i)
                            p = _plan()
                            if direct:
                                assert p["mode"] == 2, p
                            else:
                                skewed = i == 1
                                assert (p["mode"], p["fast"], p["rerun"]) == ((1, 0, 1) if skewed else (1, 1, 0)), (i, p)
                                assert skewed or p["natural"] == natural, (i, ways, p)
                            assert _affine(curve, params.commit_lagrange(poly, eng.Blind(b))) == want_l[i], (direct, ways, rep, i)
                    many = params.commit_many(polys, [eng.Blind(b) for b in blinds])
                    assert [_affine(curve, m) for m in many] == want, (direct, ways)
                    assert _plan()["sets"] == len(polys)
                L.check(lib.h2_test_set_accum_ways(ACCUM_WAYS_DEFAULT))
                got_l, got_r, got_c = params.ipa_rounds(polys[0], x3, z, lambda j, a, b: ch[j], lr, rr)
                assert got_c == ipa_c, direct
                for j in range(k):
                    assert (cref.jac_to_affine(curve, got_l[j]) == ipa_l[j]).all(), (direct, j)
                    assert (cref.jac_to_affine(curve, got_r[j]) == ipa_r[j]).all(), (direct, j)
                assert _plan()["mode"] == (2 if direct else 1)
            finally:
                params.close()
    finally:
        L.check(lib.h2_test_set_accum_ways(ACCUM_WAYS_DEFAULT))
