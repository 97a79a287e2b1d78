"""GPU tests at production sizes (k = 15 to 20): the kernels, plans and table shapes the engine picks by size only above the
k <= 14 of the other GPU tests, each compared exactly with the C oracle (oracle/cref.py).

Every MSM case also asserts, through h2_test_last_msm_plan (and h2_test_last_msm_flags where the sort matters), that the pass
took the path it is meant to cover: window size and window count of the default table, thread-per-item accumulation where a
pass has more than 2 x 2^20 references, the digit-multiples table, the exact-sort fallback of skewed columns.  A later change
of a threshold then fails here instead of silently moving these tests off their paths.

The cases are ordered so that the largest allocation (the 8.6 GB digit-multiples table at k = 15) comes before the scratch of
the large bucket sets has grown."""
import ctypes
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402

SEED = 0x4C41524745
THREAD_PER_ITEM_REFS = 2 << 20      # fixed-base passes with more references accumulate with a thread per work item
TABLE_WINDOW = {15: 16, 16: 16, 17: 17, 18: 17, 19: 20, 20: 20}   # default window of a k-sized set of generators
PLAN_KEYS = ("mode", "c", "W", "sets", "accum", "natural", "fast", "rerun")


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


def _lib():
    from halo2_b200 import lib as L
    return L, L.init()


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


def _windows(c):
    return (256 + c - 1) // c


@functools.lru_cache(maxsize=2)
def _points(curve):
    """2^20 + 2 seeded points; a set of 2^k generators is a prefix, w and u follow it."""
    return cref.gen_points(curve, SEED + (1 if curve == "pallas" else 2), (1 << 20) + 2)


def _gens(curve, k, extra):
    pts = _points(curve)
    n = 1 << k
    return np.ascontiguousarray(np.concatenate([pts[:n], pts[1 << 20:(1 << 20) + extra]]))


def _small_ints(vals):
    out = np.zeros((len(vals), 32), dtype=np.uint8)
    out[:, :8] = np.ascontiguousarray(vals, dtype="<u8").view(np.uint8).reshape(-1, 8)
    return out


def _const(x, n):
    return np.ascontiguousarray(np.tile(cref.ints_to_bytes([x]), (n, 1)))


def _columns(curve, n, seed):
    """Uniform and skewed columns of n scalars: name -> (bytes, skewed)."""
    r = pasta.CURVES[curve].r
    f = pasta.CURVES[curve].scalar
    i = np.arange(n, dtype=np.uint64)
    return {
        "random": (cref.gen_scalars(f, seed, n), False),
        "sel01": (_small_ints(i & 1), True),
        "const": (_const(pasta.gen_scalars(f, seed + 1, 1)[0], n), True),
        "r-1": (_const(r - 1, n), True),
        "small": (_small_ints(i % 251), True),        # n / 251 references per low bucket: above the bin capacity from k = 15 on
    }


def _want(curve, poly, blind, bases):
    kb = np.concatenate([poly, cref.ints_to_bytes([blind])]) if blind is not None else poly
    return cref.best_multiexp(curve, np.ascontiguousarray(kb), bases[:kb.shape[0]])


def _aff(curve, xyz):
    return cref.jac_to_affine(curve, xyz)


def _register(curve, pts, flags, window_bits=0):
    L, lib = _lib()
    h = ctypes.c_uint64(0)
    L.check(lib.h2_bases_register_ex(L.CURVE_ID[curve], L.ptr(pts), ctypes.c_size_t(pts.shape[0]), L.REPR_CANONICAL,
                                     ctypes.c_uint32(window_bits), ctypes.c_uint32(flags), ctypes.byref(h)))
    return h


def _commit(h, poly, blind):
    L, lib = _lib()
    out = np.zeros(96, dtype=np.uint8)
    L.check(lib.h2_msm_registered(h, L.ptr(poly), ctypes.c_size_t(poly.shape[0]), L.ptr(L.fe_bytes(blind)), L.REPR_CANONICAL, L.ptr(out)))
    return out


def _commit_batch(h, polys, blinds):
    L, lib = _lib()
    stack = np.ascontiguousarray(np.stack(polys))
    bl = np.ascontiguousarray(np.stack([L.fe_bytes(b) for b in blinds]))
    out = np.zeros((len(polys), 96), dtype=np.uint8)
    L.check(lib.h2_msm_registered_batch(h, L.ptr(stack), ctypes.c_size_t(stack.shape[1]), L.ptr(bl), ctypes.c_size_t(len(polys)),
                                        L.REPR_CANONICAL, L.ptr(out)))
    return out


def _ipa(curve, h, k, pp, x3, z, ch, lr, rr):
    """The IPA round loop over a raw base-set handle (g || w || u); returns (L, R, c, the plan of every round's pass)."""
    L, lib = _lib()
    r = pasta.CURVES[curve].r
    sess = ctypes.c_uint64(0)
    L.check(lib.h2_ipa_begin(h, ctypes.c_uint32(k), L.ptr(pp), L.ptr(L.fe_bytes(x3)), L.REPR_CANONICAL, ctypes.byref(sess)))
    ls, rs, plans = np.zeros((k, 64), dtype=np.uint8), np.zeros((k, 64), dtype=np.uint8), []
    lr_out = np.zeros((2, 96), dtype=np.uint8)
    try:
        for j in range(k):
            L.check(lib.h2_ipa_round(sess, L.ptr(L.fe_bytes(z)), L.ptr(L.fe_bytes(lr[j])), L.ptr(L.fe_bytes(rr[j])), L.REPR_CANONICAL,
                                     L.ptr(lr_out)))
            plans.append(_plan())
            ls[j], rs[j] = _aff(curve, lr_out[0]), _aff(curve, lr_out[1])
            L.check(lib.h2_ipa_fold(sess, L.ptr(L.fe_bytes(ch[j])), L.ptr(L.fe_bytes(pow(ch[j], -1, r))), L.REPR_CANONICAL))
        cb = np.zeros((2, 32), dtype=np.uint8)
        L.check(lib.h2_ipa_finish(sess, L.REPR_CANONICAL, L.ptr(cb)))
        sess.value = 0
    finally:
        if sess.value:
            lib.h2_ipa_finish(sess, L.REPR_CANONICAL, None)
    return ls, rs, int.from_bytes(cb[0].tobytes(), "little"), plans


# ------------------------------------------------------------------------------------------ IPA rounds
@pytest.mark.parametrize("curve,k,flags", [("vesta", 15, 3), ("pallas", 15, 1), ("vesta", 16, 1), ("pallas", 17, 1), ("vesta", 18, 1)])
def test_ipa_rounds_production_k(eng, curve, k, flags):
    """Params::ipa_rounds against the oracle's loop (poly/commitment/prover.rs:100-142), every L_j, R_j and c.  k = 15 runs on the
    window table and on the digit-multiples table at its largest size (2^15 + 2 points, 8.6 GB); from k = 16 a round's two sets
    over n + 2 scalars pass 2^21 references and accumulate with a thread per work item."""
    c = pasta.CURVES[curve]
    n = 1 << k
    bases = _gens(curve, k, 2)
    pp = cref.gen_scalars(c.scalar, SEED + 10 + k, n)
    ch = pasta.gen_scalars(c.scalar, SEED + 20 + k, k)
    lr = pasta.gen_scalars(c.scalar, SEED + 30 + k, k)
    rr = pasta.gen_scalars(c.scalar, SEED + 40 + k, k)
    x3, z = pasta.gen_scalars(c.scalar, SEED + 50 + k, 2)
    want_l, want_r, want_c = cref.ipa_rounds(curve, bases, k, pp, x3, z, cref.ints_to_bytes(ch), cref.ints_to_bytes(lr), cref.ints_to_bytes(rr))
    L, lib = _lib()
    h = _register(curve, bases, flags)
    try:
        got_l, got_r, got_c, plans = _ipa(curve, h, k, pp, x3, z, ch, lr, rr)
        assert got_c == want_c
        for j in range(k):
            assert (got_l[j] == want_l[j]).all() and (got_r[j] == want_r[j]).all(), (curve, k, j)
        for p in plans:
            assert p["sets"] == 2, p
            if flags & 2:
                assert p["mode"] == 2 and p["accum"] == 2, p
            else:
                cw = TABLE_WINDOW[k]
                assert (p["mode"], p["c"], p["W"]) == (1, cw, _windows(cw)), p
                assert p["accum"] == int(2 * (n + 2) * _windows(cw) > THREAD_PER_ITEM_REFS), p
                assert p["fast"] == 1 and p["rerun"] == 0, p
        if k >= 16:
            assert all(p["accum"] == 1 for p in plans)
        # the same set still commits (w at index n)
        poly = pp
        assert (_aff(curve, _commit(h, poly, lr[0])) == _want(curve, poly, lr[0], bases)).all()
    finally:
        L.check(lib.h2_bases_release(h))


# ------------------------------------------------------------------------------------------ commits at production k
@pytest.mark.parametrize("k", [15, 16, 17, 18, 19, 20])
def test_commits_production_k(eng, k):
    """Single, batched and resident commits on Params with the default window table, against the oracle, on uniform and skewed
    columns (0/1, constant, r - 1, small integers) with blinds: the window is the table's size class, batches accumulate with a
    thread per work item, the skewed columns take the exact sort (after the fast pass is re-run) and the uniform ones do not."""
    curve = "vesta" if k % 2 else "pallas"
    c = pasta.CURVES[curve]
    n = 1 << k
    bases = _gens(curve, k, 1)
    cols = _columns(curve, n, SEED + 100 + k)
    names = list(cols) + ["random2", "zero", "random3"]
    polys = [cols[nm][0] for nm in cols] + [cref.gen_scalars(c.scalar, SEED + 110 + k, n), np.zeros((n, 32), dtype=np.uint8),
                                            cref.gen_scalars(c.scalar, SEED + 120 + k, n)]
    skewed = [cols[nm][1] for nm in cols]
    blinds = pasta.gen_scalars(c.scalar, SEED + 130 + k, len(polys))
    wants = [_want(curve, p, b, bases) for p, b in zip(polys, blinds)]
    cw = TABLE_WINDOW[k]
    W = _windows(cw)
    params = eng.Params(curve, k, bases[:n], bases[:n], bases[n:n + 1])
    try:
        for i in range(5):
            got = _aff(curve, params.commit(polys[i], eng.Blind(blinds[i])))
            assert (got == wants[i]).all(), (k, names[i])
            p = _plan()
            assert (p["mode"], p["c"], p["W"], p["sets"]) == (1, cw, W, 1), (names[i], p)
            assert p["accum"] == int((n + 1) * W > THREAD_PER_ITEM_REFS), (names[i], p)
            if skewed[i]:
                assert _flags() & 2 and p["rerun"] == 1 and p["fast"] == 0, (names[i], p)
            else:
                assert not _flags() & 2 and p["rerun"] == 0 and p["fast"] == 1, (names[i], p)
        # eight mixed columns in one pass: thread per work item, the exact sort (skewed members)
        many = params.commit_many(polys, [eng.Blind(b) for b in blinds])
        for i in range(len(polys)):
            assert (_aff(curve, many[i]) == wants[i]).all(), (k, "commit_many", names[i])
        p = _plan()
        assert (p["mode"], p["c"], p["sets"], p["accum"], p["rerun"]) == (1, cw, 8, 1, 1), p
        assert _flags() & 2
        # three uniform columns: the fast pass holds
        uni = [0, 5, 7]
        many = params.commit_many([polys[i] for i in uni], [eng.Blind(blinds[i]) for i in uni])
        assert all((_aff(curve, m) == wants[i]).all() for m, i in zip(many, uni)), k
        p = _plan()
        assert (p["sets"], p["accum"], p["fast"], p["rerun"]) == (3, int(3 * (n + 1) * W > THREAD_PER_ITEM_REFS), 1, 0), p
        assert not _flags() & 2
        # resident columns, batch_normalize on the device
        res = [eng.ResidentPoly(c.scalar, n, p_) for p_ in polys]
        try:
            aff = params.commit_resident_affine(res, [eng.Blind(b) for b in blinds])
            for i in range(len(polys)):
                assert (aff[i] == wants[i]).all(), (k, "commit_resident_affine", names[i])
            p = _plan()
            assert (p["c"], p["sets"], p["accum"]) == (cw, 8, 1), p
        finally:
            for r_ in res:
                r_.close()
    finally:
        params.close()


# ------------------------------------------------------------------------------------------ reductions in the default tree
@pytest.mark.parametrize("n", [(1 << 15) + 1, 1 << 16, (1 << 17) + 31, 1 << 20, (1 << 20) + 1])
def test_poly_reductions_large(eng, n):
    """eval_polynomial, kate_division and compute_inner_product (arithmetic.rs:297-341) on batches of three resident
    polynomials in the default level tree -- 4 and 5 levels at these sizes -- at x random, 0 and 1."""
    L, lib = _lib()
    L.check(lib.h2_test_set_poly_cta(0))
    field = "fp" if n & 1 else "fq"
    m = pasta.FIELDS[field]
    polys = [cref.gen_scalars(field, SEED + 200 + b + n, n) for b in range(3)]
    others = [cref.gen_scalars(field, SEED + 210 + b + n, n) for b in range(3)]
    pts = [pasta.gen_scalars(field, SEED + 220 + n, 1)[0], 0, 1]
    res = [eng.ResidentPoly(field, n, p) for p in polys]
    oth = [eng.ResidentPoly(field, n, p) for p in others]
    dst = [eng.ResidentPoly(field, n, _const(7, n)) for _ in range(3)]        # stale contents: slot n - 1 must come back zero
    try:
        assert eng.eval_polynomial_resident(res, pts) == [cref.eval_polynomial(field, p, x) for p, x in zip(polys, pts)], n
        eng.kate_division_resident(res, pts, dst=dst)
        for b in range(3):
            q = dst[b].download(n)
            assert (q[:n - 1] == cref.kate_division(field, polys[b], pts[b])).all(), (n, b)
            assert not q[n - 1].any(), (n, b)
        want_ip = [sum(x * y for x, y in zip(cref.bytes_to_ints(a), cref.bytes_to_ints(b))) % m for a, b in zip(polys, others)]
        assert eng.inner_product_resident(res, oth) == want_ip, n
    finally:
        for r_ in res + oth + dst:
            r_.close()


# ------------------------------------------------------------------------------------------ grand product
@pytest.mark.parametrize("n", [(1 << 15) + 1, 1 << 16, (1 << 18) + 5])
def test_grand_product_large(eng, n):
    """batch_invert (zeros stay zero) and the running product (plonk/permutation/prover.rs:120, :150-156) on resident vectors
    whose level trees have 3 or more levels."""
    field = "fq" if n & 1 else "fp"
    m = pasta.FIELDS[field]
    vals = cref.gen_scalars(field, SEED + 300 + n, n)
    zeros = np.r_[0, 1, 31, 32, 1023, np.arange(777, n, 4099), n - 1]
    vals[zeros] = 0
    a = eng.ResidentPoly(field, n, vals)
    src = cref.gen_scalars(field, SEED + 310 + n, n)
    s = eng.ResidentPoly(field, n, src)
    try:
        eng.batch_invert_resident(a, n)
        want = [pow(x, -1, m) if x else 0 for x in cref.bytes_to_ints(vals)]
        assert cref.bytes_to_ints(a.download(n)) == want, n
        init = pasta.gen_scalars(field, SEED + 320 + n, 1)[0]
        z = eng.running_product_resident(s, init)
        acc, want = init, []
        for x in cref.bytes_to_ints(src):
            want.append(acc)
            acc = acc * x % m
        assert cref.bytes_to_ints(z.download(n)) == want, n
        z.close()
    finally:
        a.close()
        s.close()


# ------------------------------------------------------------------------------------------ lookup
@pytest.mark.parametrize("n,small", [(1 << 16, True), (1 << 16, False), (1 << 18, True), (1 << 18, False)])
def test_lookup_permute_large(eng, n, small):
    """permute_expression_pair (plonk/lookup/prover.rs:563-647) at 2^16 and 2^18 rows (u = n - 6), where the bitonic sort runs
    global stages, with small and full-width values, against the oracle; the blinding rows stay untouched."""
    field = "fp"
    u = n - 6
    rng = np.random.default_rng(SEED + n + small)
    if small:
        pool = cref.ints_to_bytes(list(range(1 << 12)))
    else:
        pool = cref.gen_scalars(field, SEED + 400 + n, n // 4)
    tab = pool[rng.integers(0, pool.shape[0], u)]
    tab[:pool.shape[0]] = pool                                              # every pool value is in the table
    tab = tab[rng.permutation(u)]
    inp = tab[rng.integers(0, u, u)]
    tail = cref.gen_scalars(field, SEED + 410 + n, n - u)
    marker = cref.gen_scalars(field, SEED + 420 + n, n)
    a = eng.ResidentPoly(field, n, np.concatenate([inp, tail]))
    t = eng.ResidentPoly(field, n, np.concatenate([tab, tail]))
    oa = eng.ResidentPoly(field, n, marker)
    ot = eng.ResidentPoly(field, n, marker)
    try:
        eng.permute_expression_pair_resident(a, t, u, oa, ot)
        want_a, want_s = cref.permute_expression_pair(inp, tab, u)
        got_a, got_s = oa.download(n), ot.download(n)
        assert (got_a[:u] == want_a).all() and (got_s[:u] == want_s).all(), (n, small)
        assert (got_a[u:] == marker[u:]).all() and (got_s[u:] == marker[u:]).all()
    finally:
        for p in (a, t, oa, ot):
            p.close()


# ------------------------------------------------------------------------------------------ NTT
@pytest.mark.parametrize("log_n,field", [(17, "fp"), (21, "fq"), (22, "fp"), (23, "fq")])
def test_ntt_plans_large(eng, log_n, field):
    """best_fft at the plan sizes no other test reaches (22 and 23 are the uneven 4-pass splits), with the classic pass kernel
    and the bulk-copy (TMA) one, against the oracle."""
    L, lib = _lib()
    a = cref.gen_scalars(field, SEED + 500 + log_n, 1 << log_n)
    w = pasta.omega_for_k(field, log_n)
    want = cref.best_fft(field, a, w, log_n)
    try:
        for tma in (0, 1):
            L.check(lib.h2_test_set_ntt_tma(tma))
            got = a.copy()
            eng.best_fft(got, w, log_n, field)
            assert (got == want).all(), (log_n, tma)
    finally:
        L.check(lib.h2_test_set_ntt_tma(0))


@pytest.mark.parametrize("field,j,k", [("fp", 5, 16), ("fq", 9, 17), ("fp", 5, 20)])
def test_domain_transforms_large(eng, field, j, k):
    """lagrange_to_coeff, coeff_to_extended (zero padding from 2^k to 2^ext_k) and extended_to_coeff at (k, ext_k) = (16, 18),
    (17, 20) and (20, 22), against the oracle."""
    d = pasta.EvaluationDomain(field, j, k)
    dom = eng.EvaluationDomain(field, j, k, d.g_coset)
    assert dom.extended_k == d.extended_k == {16: 18, 17: 20, 20: 22}[k]
    a = cref.gen_scalars(field, SEED + 600 + k, 1 << k)
    co = cref.ifft(field, a, d.omega_inv, k, d.ifft_divisor)
    assert (dom.lagrange_to_coeff(a) == co).all()
    ext = cref.coeff_to_extended(field, co, k, d.extended_k, d.g_coset, d.extended_omega)
    assert (dom.coeff_to_extended(co) == ext).all()
    back = cref.extended_to_coeff(field, ext, d.extended_k, d.extended_omega_inv, d.extended_ifft_divisor, d.g_coset, (1 << k) * (j - 1))
    assert (dom.extended_to_coeff(ext) == back).all()


def test_quotient_pipeline_k16(eng):
    """The quotient pipeline of plonk/vanishing/prover.rs:81-88 on resident polynomials at k = 16 (extended_k = 18):
    coeff_to_extended of four columns, an h(X)-shaped Ast with rotations, divide_by_vanishing_poly, extended_to_coeff -- against
    the same steps on the oracle."""
    from halo2_b200.evaluator import Ast, compile_ast
    field, j, k = "fp", 5, 16
    d_or = pasta.EvaluationDomain(field, j, k)
    d = eng.EvaluationDomain(field, j, k, d_or.g_coset)
    m = d.m
    y, theta = pasta.gen_scalars(field, SEED + 700, 2)

    def expr(a, b, c_, q):
        gate0 = (a * b - c_) * q
        gate1 = (a.with_rotation(1) - a) * (b.with_rotation(-1) + Ast.constant_term(7)) * 3
        perm = (c_ + Ast.linear_term(theta) + Ast.constant_term(11)) * (a.with_rotation(-2) + b * theta)
        return Ast.distribute_powers([gate0, gate1, -perm, q.with_rotation(3)], y)

    cols = [cref.gen_scalars(field, SEED + 710 + i, d.n) for i in range(4)]
    res = [eng.ResidentPoly(field, d.n, c_) for c_ in cols]
    ext = [d.coeff_to_extended_resident(r) for r in res]
    ev = eng.Evaluator(d, "extended")
    leaves = [ev.register_poly(e) for e in ext]
    h = ev.evaluate(expr(*leaves))
    ext_or = np.stack([cref.coeff_to_extended(field, c_, k, d.extended_k, d.g_coset, d.extended_omega) for c_ in cols])
    for i in range(4):
        assert (ext[i].download() == ext_or[i]).all(), i
    code, consts = compile_ast(expr(*[eng.AstLeaf(i) for i in range(4)]), m, 1 << (d.extended_k - k))
    h_or = cref.ast_eval(field, ext_or, d.extended_k, code, consts, d.extended_omega, d.g_coset)
    assert (h.download() == h_or).all()
    d.divide_by_vanishing_poly_resident(h)
    h_div = cref.ints_to_bytes(d_or.divide_by_vanishing_poly(cref.bytes_to_ints(h_or)))
    assert (h.download() == h_div).all()
    got = d.extended_to_coeff_resident(h).download()
    want = cref.extended_to_coeff(field, h_div, d.extended_k, d.extended_omega_inv, d.extended_ifft_divisor, d.g_coset, d.n * (j - 1))
    assert (got == want).all()
    ev.close()
    for r_ in res + ext + [h]:
        r_.close()


# ------------------------------------------------------------------------------------------ window sweep (last: large bucket sets)
@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_window_table_sweep(eng, curve):
    """A window table of every size from c = 4 to 24 over 2^10 + 2 bases: single commits and batches of three on uniform, 0/1,
    constant, r - 1 and power-of-two columns, against the oracle.  Every c has its own top-window capacity rule in
    msm_make_plan (tb = 254 - (W - 1) c).  At c = 24 the batch holds two vectors: the scratch of a pass grows with its
    2^23 buckets per vector (bins, bucket sums, partial slots: about 5.5 GB each), and three would take the device past 16 GB."""
    c = pasta.CURVES[curve]
    n = (1 << 10) + 2
    bases = cref.gen_points(curve, SEED + 800 + (curve == "vesta"), n)
    m = n - 1                                                                   # scalars + the blind on bases[n - 1]
    cols = _columns(curve, m, SEED + 810)
    polys = [cols["random"][0], cols["sel01"][0], cols["const"][0], cols["r-1"][0],
             cref.ints_to_bytes([(1 << (i * 7 % 254)) % c.r for i in range(m)])]
    blinds = pasta.gen_scalars(c.scalar, SEED + 820, len(polys))
    wants = [_want(curve, p, b, bases) for p, b in zip(polys, blinds)]
    L, lib = _lib()
    for cb in range(4, 25):
        h = _register(curve, bases, 1, cb)
        try:
            for i, (p, b) in enumerate(zip(polys, blinds)):
                assert (_aff(curve, _commit(h, p, b)) == wants[i]).all(), (curve, cb, i)
                pl = _plan()
                assert (pl["mode"], pl["c"], pl["W"], pl["sets"]) == (1, cb, _windows(cb), 1), (cb, pl)
            for sel in ((0, 1, 2), (3, 4, 0)):
                sel = sel if cb < 24 else sel[:2]
                out = _commit_batch(h, [polys[i] for i in sel], [blinds[i] for i in sel])
                for o, i in zip(out, sel):
                    assert (_aff(curve, o) == wants[i]).all(), (curve, cb, "batch", i)
                pl = _plan()
                assert (pl["c"], pl["sets"]) == (cb, len(sel)), (cb, pl)
        finally:
            L.check(lib.h2_bases_release(h))
