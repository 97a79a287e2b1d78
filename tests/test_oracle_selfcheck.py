"""The two independent restatements (pasta.py big-int, halo2_oracle.c limbs) agree with each
other and with the naive definitions -- mirrors the reference's own property tests
(arithmetic.rs:440-458, poly/commitment.rs:258-302, poly/commitment/msm.rs:179-219,
poly/domain.rs:500-569).  CPU only."""
import numpy as np
import pytest

from oracle import cref, pasta

SEED = 0x48414C4F32


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_field_ops(field):
    m = pasta.FIELDS[field]
    xs = pasta.gen_scalars(field, SEED, 40) + [0, 1, 2, m - 1, m - 2]
    assert cref.bytes_to_ints(cref.gen_scalars(field, SEED, 40)) == xs[:40]
    for a, b in zip(xs, xs[1:] + xs[:1]):
        assert cref.field_op(field, "add", a, b) == (a + b) % m
        assert cref.field_op(field, "sub", a, b) == (a - b) % m
        assert cref.field_op(field, "mul", a, b) == a * b % m
        if a:
            assert cref.field_op(field, "inv", a) == pow(a, m - 2, m)


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_multiexp_matches_naive(curve):
    """arithmetic.rs:440-458 (test_multiexp), plus n that exercise c = 1, 3, ceil(ln n)."""
    c = pasta.CURVES[curve]
    for n in (1, 2, 3, 5, 31, 40, 256):
        ks = pasta.gen_scalars(c.scalar, SEED + n, n)
        kb = cref.ints_to_bytes(ks)
        pb = cref.gen_points(curve, SEED + 7 * n, n)
        want = cref.bytes_to_affine(cref.naive_msm(curve, kb, pb))
        if n <= 40:
            pts = [cref.bytes_to_affine(r) for r in pb]
            assert pts == pasta.gen_points(c, SEED + 7 * n, n)
            assert pasta.to_affine(c, pasta.naive_msm(c, ks, pts)) == want
            assert pasta.to_affine(c, pasta.best_multiexp(c, ks, pts, num_threads=4)) == want
            assert pasta.to_affine(c, pasta.best_multiexp(c, ks, pts, num_threads=1000)) == want
        for threads in (1, 8, 1000):  # parallel branch and serial-Horner branch
            assert cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb, threads)) == want


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_multiexp_edge_cases(curve):
    """Duplicates, negations, cancelling terms, identity bases -- cf. msm.rs:179-219."""
    c = pasta.CURVES[curve]
    g = pasta.generator(c)
    ng = (g[0], c.p - g[1])
    p3 = pasta.gen_points(c, SEED, 4)[3]
    pts = [g, g, ng, None, p3, p3]
    ks = [5, 7, 12, 99, c.r - 1, 1]
    for threads in (2, 64):
        out = cref.best_multiexp(curve, cref.ints_to_bytes(ks), cref.affines_to_bytes(pts), threads)
        assert cref.bytes_to_affine(out) is None
    assert pasta.to_affine(c, pasta.best_multiexp(c, ks, pts)) is None
    ks[0] = 6  # now the sum is 1*g
    out = cref.best_multiexp(curve, cref.ints_to_bytes(ks), cref.affines_to_bytes(pts), 2)
    assert cref.bytes_to_affine(out) == g
    # length mismatch panics (arithmetic.rs:144)
    with pytest.raises(AssertionError):
        cref.best_multiexp(curve, cref.ints_to_bytes(ks), cref.affines_to_bytes(pts[:3]))


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_fft_network(field):
    m = pasta.FIELDS[field]
    for log_n in (1, 2, 3, 6, 9):
        n = 1 << log_n
        a = pasta.gen_scalars(field, SEED + log_n, n)
        w = pasta.omega_for_k(field, log_n)
        x = list(a)
        pasta.best_fft(field, x, w, log_n)
        if log_n <= 6:  # true root of unity: the network is the DFT
            assert x == [sum(a[j] * pow(w, j * k, m) for j in range(n)) % m for k in range(n)]
        y = list(a)
        pasta.best_fft_recursive(field, y, w, log_n)
        assert x == y
        wr = pasta.gen_scalars(field, SEED + 99, 1)[0]  # benches/fft.rs:17: random omega
        xr = list(a)
        pasta.best_fft(field, xr, wr, log_n)
        for threads in (1, 8, 4096):  # recursive and iterative branches of arithmetic.rs:223-254
            assert cref.bytes_to_ints(cref.best_fft(field, cref.ints_to_bytes(a), w, log_n, threads)) == x
            assert cref.bytes_to_ints(cref.best_fft(field, cref.ints_to_bytes(a), wr, log_n, threads)) == xr
    with pytest.raises(AssertionError):
        cref.best_fft(field, cref.ints_to_bytes([1, 2, 3]), 1, 2)


@pytest.mark.parametrize("field,j,k", [("fp", 5, 5), ("fq", 3, 6), ("fp", 4, 3)])
def test_domain_transforms(field, j, k):
    """domain.rs:500-569 style: iFFT output evaluates back to the Lagrange samples; coset
    round trip; C restatement == Python."""
    m = pasta.FIELDS[field]
    d = pasta.EvaluationDomain(field, j, k)
    n = 1 << k
    a = pasta.gen_scalars(field, SEED, n)
    co = d.lagrange_to_coeff(a)
    assert [pasta.eval_polynomial(field, co, pow(d.omega, i, m)) for i in range(n)] == a
    assert cref.bytes_to_ints(cref.ifft(field, cref.ints_to_bytes(a), d.omega_inv, k, d.ifft_divisor)) == co
    ext = d.coeff_to_extended(co)
    for i in (0, 1, 5, (1 << d.extended_k) - 1):
        assert ext[i] == pasta.eval_polynomial(field, co, d.g_coset * pow(d.extended_omega, i, m) % m)
    got = cref.coeff_to_extended(field, cref.ints_to_bytes(co), k, d.extended_k, d.g_coset, d.extended_omega)
    assert cref.bytes_to_ints(got) == ext
    back = d.extended_to_coeff(ext)
    assert back[:n] == co and not any(back[n:])
    got = cref.extended_to_coeff(field, cref.ints_to_bytes(ext), d.extended_k, d.extended_omega_inv,
                                 d.extended_ifft_divisor, d.g_coset, len(back))
    assert cref.bytes_to_ints(got) == back


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_commit_lagrange_equals_commit(curve):
    """poly/commitment.rs:258-302 at k=4 (synthetic generators, reference EC-FFT)."""
    c = pasta.CURVES[curve]
    k = 4
    params = pasta.Params(c, k)
    d = pasta.EvaluationDomain(c.scalar, 2, k)
    a = pasta.gen_scalars(c.scalar, SEED + 3, 1 << k)
    alpha = pasta.gen_scalars(c.scalar, SEED + 4, 1)[0]
    lhs = params.commit_lagrange(a, alpha)
    rhs = params.commit(d.lagrange_to_coeff(a), alpha)
    assert pasta.to_affine(c, lhs) == pasta.to_affine(c, rhs)
    # and through the C restatement
    kb = cref.ints_to_bytes(list(a) + [alpha])
    pb = cref.affines_to_bytes(list(params.g_lagrange) + [params.w])
    assert cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb)) == pasta.to_affine(c, lhs)


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_ipa_rounds_c_vs_python(curve):
    """The two restatements of the IPA round loop (prover.rs:100-142) agree bit for bit."""
    from oracle import cref
    c = pasta.CURVES[curve]
    for k in (1, 3, 5):
        n = 1 << k
        pts = pasta.gen_points(c, 900 + k, n + 2)
        pp = pasta.gen_scalars(c.scalar, 910 + k, n)
        ch = pasta.gen_scalars(c.scalar, 920 + k, k)
        lr = pasta.gen_scalars(c.scalar, 930 + k, k)
        rr = pasta.gen_scalars(c.scalar, 940 + k, k)
        x3, z = pasta.gen_scalars(c.scalar, 950 + k, 2)
        L, R, cc, _ = pasta.ipa_rounds(c, pts[:n], pts[n], pts[n + 1], pp, x3, z, ch, lr, rr)
        gl, gr, gc = cref.ipa_rounds(curve, cref.affines_to_bytes(pts), k, cref.ints_to_bytes(pp), x3, z, cref.ints_to_bytes(ch),
                                     cref.ints_to_bytes(lr), cref.ints_to_bytes(rr), threads=3)
        assert gc == cc
        assert [cref.bytes_to_affine(x) for x in gl] == L
        assert [cref.bytes_to_affine(x) for x in gr] == R


def test_eval_and_kate_division_restatements_agree():
    """arithmetic.rs:297-341 in C and in Python, and kate_division's defining identity q(X) (X - b) + a(b) == a(X)."""
    for field in ("fp", "fq"):
        m = pasta.FIELDS[field]
        for n in (1, 2, 3, 64, 257):
            a = cref.gen_scalars(field, 40 + n, n)
            ai = cref.bytes_to_ints(a)
            b, z = pasta.gen_scalars(field, 41 + n, 2)
            assert cref.eval_polynomial(field, a, b) == pasta.eval_polynomial(field, ai, b)
            q = pasta.kate_division(field, ai, b)
            assert cref.bytes_to_ints(cref.kate_division(field, a, b)) == q and len(q) == n - 1
            assert (pasta.eval_polynomial(field, q, z) * (z - b) + pasta.eval_polynomial(field, ai, b)) % m == pasta.eval_polynomial(field, ai, z)


def test_ast_evaluate_restatements_agree():
    """Evaluator::evaluate (poly/evaluator.rs:129-228): the recursive big-int walk and the C interpreter of the flattened program
    agree in both bases, for any thread count (chunk boundaries, evaluator.rs:16-32)."""
    from halo2_b200.evaluator import Ast, AstLeaf, compile_ast     # the flattening only: no GPU, no engine call
    from tests.ast_cases import _ast_tuple, _quotient_like_ast
    field = "fq"
    for basis, j, k in (("extended", 3, 3), ("lagrange", 2, 6), ("extended", 5, 2)):
        d = pasta.EvaluationDomain(field, j, k, pasta.zeta_candidates(field)[1])
        log_n = k if basis == "lagrange" else d.extended_k
        polys = [pasta.gen_scalars(field, 70 + i, 1 << log_n) for i in range(4)]
        y, theta = pasta.gen_scalars(field, 75, 2)
        ast = _quotient_like_ast([AstLeaf(i) for i in range(4)], y, theta)
        code, consts = compile_ast(ast, d.m, 1 if basis == "lagrange" else 1 << (d.extended_k - d.k))
        want = pasta.ast_evaluate(d, basis, _ast_tuple(ast), polys)
        pb = np.stack([cref.ints_to_bytes(p) for p in polys])
        for threads in (1, 3, 64):
            got = cref.ast_eval(field, pb, log_n, code, consts, d.omega if basis == "lagrange" else d.extended_omega,
                                1 if basis == "lagrange" else d.g_coset, threads)
            assert cref.bytes_to_ints(got) == want, (basis, threads)


def test_permute_expression_pair_properties():
    """The restated permute_expression_pair against what the reference's own sanity check demands (plonk/lookup/prover.rs:630-641:
    where A' and S' differ, A' repeats the previous row) plus the multiset equalities, and the failure case (:605-608)."""
    import random
    rnd = random.Random(11)
    m = pasta.FIELDS["fp"]
    for u, vals in ((1, 1), (7, 3), (200, 16), (257, 300), (64, 1)):
        table = [rnd.randrange(m) for _ in range(vals)]
        tab_col = [table[i % vals] if i < vals else rnd.choice(table) for i in range(u)]
        rnd.shuffle(tab_col)
        inp = [rnd.choice(tab_col) for _ in range(u)]
        a, s = pasta.permute_expression_pair("fp", inp + [5, 6], tab_col + [7, 8], u)
        assert a == sorted(inp) and sorted(s) == sorted(tab_col)
        ca, cs = cref.permute_expression_pair(cref.ints_to_bytes(inp + [5, 6]), cref.ints_to_bytes(tab_col + [7, 8]), u)   # the C restatement agrees
        assert cref.bytes_to_ints(ca) == a and cref.bytes_to_ints(cs) == s
        last = None
        for x, y in zip(a, s):
            if x != y:
                assert x == last
            last = x
    assert pasta.permute_expression_pair("fp", [1, 2, 3], [1, 2, 4], 3) is None
    assert cref.permute_expression_pair(cref.ints_to_bytes([1, 2, 3]), cref.ints_to_bytes([1, 2, 4]), 3) is None
    assert pasta.permute_expression_pair("fp", [1, 2, 9], [1, 2, 4], 2) == ([1, 2], [1, 2])     # rows past usable_rows are ignored
