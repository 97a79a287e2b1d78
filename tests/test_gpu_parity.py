"""GPU parity tests: the sm_90a path, called through the C ABI, against the CPU oracle on the
same seeded inputs.  Bit-exact (integer arithmetic): scalars compare as canonical 32-byte
elements, MSM results as affine canonical bytes.  Mirrors SURVEY.md section 4.1."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests.ast_cases import _ast_tuple  # noqa: E402
from tests.poseidon_kat import permute  # noqa: E402

SEED = 0x48414C4F32


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


@pytest.fixture(params=["direct", "buckets"])
def table_mode(request):
    """Fixed-base MSMs over resident generators run either on the digit-multiples table (direct sum, csrc/fixedbase.cuh:
    the default up to k = 14) or on the window table with one shared bucket set; both must give the oracle's points."""
    from halo2_b200 import poly
    poly.DIRECT_DEFAULT = request.param == "direct"
    yield request.param
    poly.DIRECT_DEFAULT = None


def _field_op(field, op, a, b=None):
    from halo2_b200 import lib as L
    lib = L.init()
    a = cref.ints_to_bytes(a)
    b = cref.ints_to_bytes(b if b is not None else [0] * len(a))
    out = np.zeros_like(a)
    L.check(lib.h2_test_field_op(L.FIELD_ID[field], op, L.ptr(a), L.ptr(b), ctypes.c_size_t(a.shape[0]), L.ptr(out)))
    return cref.bytes_to_ints(out)


def _curve_op(curve, op, a, b):
    from halo2_b200 import lib as L
    lib = L.init()
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b)
    out = np.zeros_like(a)
    L.check(lib.h2_test_curve_op(L.CURVE_ID[curve], op, L.ptr(a), L.ptr(b), ctypes.c_size_t(a.shape[0]), L.ptr(out)))
    return out


def _affine(curve, xyz):
    return cref.bytes_to_affine(cref.jac_to_affine(curve, xyz))


# ------------------------------------------------------------------------------------------ K0
def _structured_limbs(m):
    import random
    rnd = random.Random(6)
    raws = [0, 1, m - 1, m - 2, 1 << 254, (1 << 254) - 1, (1 << 254) + 1, m >> 1]
    for mask in range(256):
        v = sum(0xFFFFFFFF << (32 * i) for i in range(8) if (mask >> i) & 1)
        raws += [v % m, v & ((1 << 254) - 1)]
    for _ in range(1500):
        raws.append(sum(rnd.choice([0, 0xFFFFFFFF, 1, 0x80000000, 0x7FFFFFFF, rnd.getrandbits(32)]) << (32 * i) for i in range(8)) % m)
    return raws


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_device_field_ops(eng, field):
    m = pasta.FIELDS[field]
    xs = pasta.gen_scalars(field, SEED, 2000) + [0, 1, 2, m - 1, m - 2, 1 << 254, (1 << 254) - 1, m - (1 << 32),
                                                 0xFFFFFFFF, 1 << 32, (1 << 224) - 1, m >> 1, (1 << 255) % m]
    ys = xs[7:] + xs[:7]
    assert _field_op(field, 0, xs, ys) == [(a + b) % m for a, b in zip(xs, ys)]
    assert _field_op(field, 1, xs, ys) == [(a - b) % m for a, b in zip(xs, ys)]
    assert _field_op(field, 2, xs, ys) == [a * b % m for a, b in zip(xs, ys)]
    assert _field_op(field, 4, xs) == [a * a % m for a in xs]
    nz = [x for x in xs if x][:300]
    assert _field_op(field, 3, nz) == [pow(a, m - 2, m) for a in nz]
    # the divsteps inversion the kernels use (fe_inv_gcd): all samples, 0 -> 0, and the structured Montgomery residues below
    assert _field_op(field, 5, xs) == [pow(a, m - 2, m) if a else 0 for a in xs]
    # structured MONTGOMERY operands (all-ones / zero / single-bit limbs): the carry edges of the dedicated squaring
    raws = _structured_limbs(m)
    rinv = pow(1 << 256, -1, m)
    zs = [x * rinv % m for x in raws]              # to_mont(z) == x
    assert _field_op(field, 4, zs) == [a * a % m for a in zs]
    assert _field_op(field, 2, zs, zs[5:] + zs[:5]) == [a * b % m for a, b in zip(zs, zs[5:] + zs[:5])]
    assert _field_op(field, 5, zs) == [pow(a, m - 2, m) if a else 0 for a in zs]


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_device_poseidon_kat(eng, goldens, field):
    """halo2_poseidon/src/test_vectors.rs reproduced with the DEVICE add/mul (field-layer KAT)."""
    g = goldens["poseidon"][field]
    rc = [int(x, 16) for x in g["round_constants"]]
    mds = [int(x, 16) for x in g["mds"]]
    add = lambda a, b: _field_op(field, 0, [a], [b])[0]  # noqa: E731
    mul = lambda a, b: _field_op(field, 2, [a], [b])[0]  # noqa: E731
    pow5 = lambda a: mul(mul(mul(a, a), mul(a, a)), a)   # noqa: E731
    for tv in g["permute"][:2]:
        out = permute([int(x, 16) for x in tv["initial_state"]], rc, mds, add, mul, pow5)
        assert out == [int(x, 16) for x in tv["final_state"]]


# ------------------------------------------------------------------------------------------ K1
@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_device_curve_ops(eng, curve):
    c = pasta.CURVES[curve]
    n = 64
    pts = cref.gen_points(curve, SEED, n)
    other = cref.gen_points(curve, SEED + 1, n)
    g = pasta.generator(c)
    a_list = [cref.bytes_to_affine(p) for p in pts]
    b_list = [cref.bytes_to_affine(p) for p in other]
    # edge cases: P+P, P+(-P), identity operands
    a_list[0], b_list[0] = g, g
    a_list[1], b_list[1] = g, (g[0], c.p - g[1])
    a_list[2], b_list[2] = None, b_list[2]
    a_list[3], b_list[3] = a_list[3], None
    a_list[4], b_list[4] = None, None
    a = cref.affines_to_bytes(a_list)
    b = cref.affines_to_bytes(b_list)
    got = _curve_op(curve, 0, a, b)
    for i in range(n):
        assert cref.bytes_to_affine(got[i]) == cref.bytes_to_affine(cref.point_add(curve, a[i], b[i])), i
    got = _curve_op(curve, 1, a, b)
    for i in range(n):
        assert cref.bytes_to_affine(got[i]) == cref.bytes_to_affine(cref.point_add(curve, a[i], a[i])), i
    ks = pasta.gen_scalars(c.scalar, SEED + 2, n - 4) + [0, 1, 2, c.r - 1]
    kb = np.zeros((n, 64), dtype=np.uint8)
    kb[:, :32] = cref.ints_to_bytes(ks)
    got = _curve_op(curve, 2, a, kb)
    for i in range(0, n, 3):
        assert cref.bytes_to_affine(got[i]) == cref.bytes_to_affine(cref.scalar_mul(curve, ks[i], a[i])), i


# ------------------------------------------------------------------------------------------ K7-K9
@pytest.mark.parametrize("field", ["fp", "fq"])
def test_best_fft_parity(eng, field):
    """Direct best_fft parity (the reference has no such test): log_n = 0..16, true root and a
    random omega (benches/fft.rs:17)."""
    for log_n in list(range(0, 15)) + [16]:
        n = 1 << log_n
        a = cref.gen_scalars(field, SEED + log_n, n)
        for w in (pasta.omega_for_k(field, log_n), pasta.gen_scalars(field, SEED + 77, 1)[0]):
            want = cref.best_fft(field, a, w, log_n)
            got = a.copy()
            eng.best_fft(got, w, log_n, field)
            assert (got == want).all(), (field, log_n)
    with pytest.raises(AssertionError):  # arithmetic.rs:205
        eng.best_fft(cref.gen_scalars(field, 1, 3), 1, 2, field)


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_best_fft_2pow20(eng, field):
    """BASELINE.json config 2 at full size against the C restatement."""
    log_n = 20
    a = cref.gen_scalars(field, SEED + 2, 1 << log_n)
    w = pasta.omega_for_k(field, log_n)
    want = cref.best_fft(field, a, w, log_n)
    got = a.copy()
    eng.best_fft(got, w, log_n, field)
    assert (got == want).all()
    # Montgomery-form round trip through the same entry point: encode, transform, decode
    from halo2_b200 import lib as L
    R = (1 << 256) % pasta.FIELDS[field]
    m = pasta.FIELDS[field]
    small = cref.bytes_to_ints(a[:4096])
    am = cref.ints_to_bytes([x * R % m for x in small])
    wm = w * R % m
    eng.best_fft(am, pasta.omega_for_k(field, 12) * R % m, 12, field, repr=L.REPR_MONTGOMERY)
    want12 = cref.bytes_to_ints(cref.best_fft(field, a[:4096], pasta.omega_for_k(field, 12), 12))
    assert cref.bytes_to_ints(am) == [x * R % m for x in want12]
    del wm


@pytest.mark.parametrize("field,j,k", [("fp", 5, 14), ("fp", 4, 5), ("fq", 9, 11), ("fq", 3, 8), ("fp", 2, 3)])
def test_domain_transforms(eng, field, j, k):
    """lagrange_to_coeff / coeff_to_extended / extended_to_coeff vs the restated
    poly/domain.rs:227-255,303-325 for (k, ext_k) = (14,16), (5,7), (11,14), ..."""
    zeta = pasta.zeta_candidates(field)[1]
    d_or = pasta.EvaluationDomain(field, j, k, zeta)
    d = eng.EvaluationDomain(field, j, k, zeta)
    assert (d.omega, d.extended_omega, d.extended_k) == (d_or.omega, d_or.extended_omega, d_or.extended_k)
    a = cref.gen_scalars(field, SEED + k, 1 << k)
    co = cref.ifft(field, a, d_or.omega_inv, k, d_or.ifft_divisor)
    assert (d.lagrange_to_coeff(a) == co).all()
    ext = cref.coeff_to_extended(field, co, k, d_or.extended_k, zeta, d_or.extended_omega)
    assert (d.coeff_to_extended(co) == ext).all()
    out_len = (1 << k) * (j - 1)
    back = cref.extended_to_coeff(field, ext, d_or.extended_k, d_or.extended_omega_inv, d_or.extended_ifft_divisor, zeta, out_len)
    got = d.extended_to_coeff(ext)
    assert got.shape == back.shape and (got == back).all()
    # round trip: truncation keeps the low 2^k coefficients, the rest are zero
    assert (got[: 1 << k] == co).all() and not got[1 << k:].any()


def test_rotate_property(eng):
    """poly/domain.rs:500-540 (test_rotate) with lagrange_to_coeff on the device: for Lagrange values a over the k = 3 domain of
    the Pallas scalar field, p(x) == p_cur(x), p(x w) == p_next(x), p(x / w) == p_prev(x) -- and the iNTT output evaluates
    back to the samples on the domain (the Horner check of SURVEY.md section 4.1)."""
    field, k = "fq", 3
    m, n = pasta.FIELDS[field], 8
    d = eng.EvaluationDomain(field, 1 + 1, k, pasta.zeta_candidates(field)[0])
    a = cref.gen_scalars(field, SEED + 900, n)
    rot = {0: a, 1: np.roll(a, -1, axis=0), -1: np.roll(a, 1, axis=0)}          # Polynomial::rotate, poly.rs:157-171
    co = {r: cref.bytes_to_ints(d.lagrange_to_coeff(v)) for r, v in rot.items()}
    x = pasta.gen_scalars(field, SEED + 901, 1)[0]
    ev = lambda c_, at: pasta.eval_polynomial(field, c_, at)                    # noqa: E731
    assert ev(co[0], x) == ev(co[0], x)
    assert ev(co[0], x * d.omega % m) == ev(co[1], x)
    assert ev(co[0], x * d.omega_inv % m) == ev(co[-1], x)
    assert [ev(co[0], pow(d.omega, i, m)) for i in range(n)] == cref.bytes_to_ints(a)


# ------------------------------------------------------------------------------------------ K2-K5
@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_best_multiexp_parity(eng, curve):
    """arithmetic.rs:440-458 widened: n = 1 .. 2^14+1 (the commit size at k=14)."""
    c = pasta.CURVES[curve]
    for n in (1, 2, 3, 4, 31, 32, 33, 256, 1024, 4097, 16385):
        kb = cref.gen_scalars(c.scalar, SEED + n, n)
        pb = cref.gen_points(curve, SEED + 3 * n, n)
        want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
        assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == want, (curve, n)
    with pytest.raises(AssertionError):  # arithmetic.rs:144
        eng.best_multiexp(kb[:5], pb[:4], curve)
    # empty input: identity
    assert _affine(curve, eng.best_multiexp(kb[:0], pb[:0], curve)) is None


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_best_multiexp_edge_and_skew(eng, curve):
    """Duplicates, negations, identity bases (msm.rs:179-219) and the skewed scalar
    distributions real provers produce (SURVEY.md section 7)."""
    from halo2_b200 import lib as L
    c = pasta.CURVES[curve]
    r = c.r
    g = pasta.generator(c)
    pts = [cref.bytes_to_affine(x) for x in cref.gen_points(curve, SEED, 8)]
    pts2 = [g, g, (g[0], c.p - g[1]), None, pts[3], pts[3], pts[4], (pts[4][0], c.p - pts[4][1]), None, g] * 40
    ks = pasta.gen_scalars(c.scalar, SEED + 4, len(pts2))
    ks[0] = ks[1] = ks[2] = 5
    ks[6] = ks[7]
    kb, pb = cref.ints_to_bytes(ks), cref.affines_to_bytes(pts2)
    assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
    out = eng.best_multiexp(cref.ints_to_bytes([5, 7, 12, 99, r - 1, 1]),
                            cref.affines_to_bytes([g, g, (g[0], c.p - g[1]), None, pts[3], pts[3]]), curve)
    assert _affine(curve, out) is None
    n = 5000
    pb = cref.gen_points(curve, SEED + 9, n)
    one = pasta.gen_scalars(c.scalar, 1, 1)[0]
    cases = {
        "zeros": [0] * n, "ones": [1] * n, "equal": [one] * n, "mix01": [i & 1 for i in range(n)],
        "rminus1": [r - 1] * n, "topheavy": [(r - 1) - (i << 3) for i in range(n)], "small": [i % 1000 for i in range(n)],
        "pow2": [(1 << (i % 255)) % r for i in range(n)], "half": [(1 << 254) - 1 + i for i in range(n)],
    }
    lib = L.init()
    try:
        for name, ks in cases.items():
            kb = cref.ints_to_bytes(ks)
            want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
            for cbits in (0, 7, 13):
                L.check(lib.h2_set_window_bits(cbits))
                assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == want, (name, cbits)
    finally:
        lib.h2_set_window_bits(0)


def test_glv_on_off_agree(eng):
    """The GLV split (default) and the plain 255-bit path give the same point, also on skewed scalars."""
    from halo2_b200 import lib as L
    curve, c = "vesta", pasta.VESTA
    n = 3000
    pb = cref.gen_points(curve, SEED + 40, n)
    lam = 0x2d33357cb532458ed3552a23a8554e5005270d29d19fc7d27b7fd22f0201b547
    sets = [cref.gen_scalars(c.scalar, SEED + 41, n), cref.ints_to_bytes([lam] * n), cref.ints_to_bytes([c.r - lam + (i % 3) for i in range(n)]),
            cref.ints_to_bytes([(1 << 128) - 1 + (i & 1) for i in range(n)])]
    lib = L.init()
    try:
        for kb in sets:
            want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
            for on in (1, 0):
                L.check(lib.h2_set_glv(on))
                for cbits in (0, 5, 12):
                    L.check(lib.h2_set_window_bits(cbits))
                    assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == want, (on, cbits)
    finally:
        lib.h2_set_glv(1)
        lib.h2_set_window_bits(0)


def test_window_sweep_and_montgomery_inputs(eng):
    """BASELINE.json config 3's sweep dimension: every window size gives the same point;
    Montgomery-encoded inputs (pasta's in-memory form) give the same point too."""
    from halo2_b200 import lib as L
    curve, c = "pallas", pasta.PALLAS
    n = 4096
    kb = cref.gen_scalars(c.scalar, SEED + 5, n)
    pb = cref.gen_points(curve, SEED + 6, n)
    want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
    lib = L.init()
    try:
        for cbits in list(range(1, 21)):
            L.check(lib.h2_set_window_bits(cbits))
            assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == want, cbits
    finally:
        lib.h2_set_window_bits(0)
    Rr, Rp = (1 << 256) % c.r, (1 << 256) % c.p
    km = cref.ints_to_bytes([k * Rr % c.r for k in cref.bytes_to_ints(kb)])
    coords = cref.bytes_to_ints(pb.reshape(-1, 32))
    pm = cref.ints_to_bytes([v * Rp % c.p for v in coords]).reshape(-1, 64)
    out = eng.best_multiexp(km, pm, curve, repr=L.REPR_MONTGOMERY)
    Rinv = pow(Rp, c.p - 2, c.p)
    xyz = cref.ints_to_bytes([v * Rinv % c.p for v in cref.bytes_to_ints(out.reshape(3, 32))]).reshape(-1)
    assert _affine(curve, xyz) == want


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_commit_lagrange_equals_commit(eng, curve, table_mode):
    """poly/commitment.rs:258-302 at k=6: commit(lagrange_to_coeff(a)) == commit_lagrange(a), with
    g_lagrange from the oracle's EC-FFT (commitment.rs:77-94) -- ties NTT, MSM and resident bases."""
    c = pasta.CURVES[curve]
    k = 6
    po = pasta.Params(c, k)
    params = eng.Params(curve, k, cref.affines_to_bytes(po.g), cref.affines_to_bytes(po.g_lagrange),
                        cref.affines_to_bytes([po.w]))
    zeta = pasta.zeta_candidates(c.scalar)[0]
    dom = eng.EvaluationDomain(c.scalar, 2, k, zeta)
    a = cref.gen_scalars(c.scalar, SEED + 8, 1 << k)
    alpha = pasta.gen_scalars(c.scalar, SEED + 9, 1)[0]
    lhs = _affine(curve, params.commit_lagrange(a, eng.Blind(alpha)))
    rhs = _affine(curve, params.commit(dom.lagrange_to_coeff(a), eng.Blind(alpha)))
    assert lhs == rhs
    assert lhs == pasta.to_affine(c, po.commit_lagrange(cref.bytes_to_ints(a), alpha))
    # Blind::default() == 1 (commitment.rs:212-216): all-zero column commits to w
    zero = np.zeros((1 << k, 32), dtype=np.uint8)
    assert _affine(curve, params.commit_lagrange(zero, eng.Blind())) == po.w
    params.close()


@pytest.mark.parametrize("curve,k", [("vesta", 14), ("pallas", 10)])
def test_resident_bases_with_window_table(eng, curve, k):
    """Params::commit on resident generators with the precomputed window table (fixed-base MSM) ==
    the reference algorithm on the same n+1 terms (poly/commitment.rs:119-130); with and without the
    table, several window sizes, skewed polynomials (0/1 selector columns, constant columns)."""
    import ctypes
    from halo2_b200 import lib as L
    c = pasta.CURVES[curve]
    n = 1 << k
    g = cref.gen_points(curve, SEED + 21, n + 1)      # g_0..g_(n-1), w
    lib = L.init()
    polys = {
        "random": cref.gen_scalars(c.scalar, SEED + 22, n),
        "zero": np.zeros((n, 32), dtype=np.uint8),
        "sel01": cref.ints_to_bytes([i & 1 for i in range(n)]),
        "const": cref.ints_to_bytes([pasta.gen_scalars(c.scalar, 5, 1)[0]] * n),
        "small": cref.ints_to_bytes([i % 251 for i in range(n)]),
    }
    blind = pasta.gen_scalars(c.scalar, SEED + 23, 1)[0]
    wants = {}
    for name, poly in polys.items():
        kb = np.concatenate([poly, cref.ints_to_bytes([blind])])
        wants[name] = cref.bytes_to_affine(cref.best_multiexp(curve, kb, g))
    for flags, wbits in ((1, 0), (3, 0), (1, 9), (1, 13), (0, 0)):   # 3 = + H2_BASES_DIRECT: digit-multiples table, direct sum
        h = ctypes.c_uint64(0)
        L.check(lib.h2_bases_register_ex(L.CURVE_ID[curve], L.ptr(g), ctypes.c_size_t(n + 1), L.REPR_CANONICAL,
                                         ctypes.c_uint32(wbits), ctypes.c_uint32(flags), ctypes.byref(h)))
        try:
            for name, poly in polys.items():
                out = np.zeros(96, dtype=np.uint8)
                L.check(lib.h2_msm_registered(h, L.ptr(poly), ctypes.c_size_t(n), L.ptr(L.fe_bytes(blind)), L.REPR_CANONICAL, L.ptr(out)))
                assert _affine(curve, out) == wants[name], (name, flags, wbits)
            # fewer scalars than bases (IPA-style prefix) and no blind
            out = np.zeros(96, dtype=np.uint8)
            L.check(lib.h2_msm_registered(h, L.ptr(polys["random"]), ctypes.c_size_t(n // 2), None, L.REPR_CANONICAL, L.ptr(out)))
            assert _affine(curve, out) == cref.bytes_to_affine(cref.best_multiexp(curve, polys["random"][: n // 2], g[: n // 2]))
        finally:
            L.check(lib.h2_bases_release(h))


def test_commit_many_batched(eng, table_mode):
    """Batched commits (one pass, one bucket set per polynomial) == the individual commits == the oracle."""
    curve, c, k = "vesta", pasta.VESTA, 12
    n = 1 << k
    g = cref.gen_points(curve, SEED + 31, n + 1)
    params = eng.Params(curve, k, g[:n], g[:n], g[n:n + 1])
    polys = [cref.gen_scalars(c.scalar, SEED + 32 + i, n) for i in range(4)]
    polys[2] = cref.ints_to_bytes([i & 1 for i in range(n)])
    polys[3] = np.zeros((n, 32), dtype=np.uint8)
    blinds = [eng.Blind(pasta.gen_scalars(c.scalar, SEED + 40 + i, 1)[0]) for i in range(4)]
    many = params.commit_many(polys, blinds)
    for i in range(4):
        single = params.commit(polys[i], blinds[i])
        want = cref.bytes_to_affine(cref.best_multiexp(curve, np.concatenate([polys[i], cref.ints_to_bytes([blinds[i].value])]), g))
        assert _affine(curve, many[i]) == want == _affine(curve, single), i
    # ... followed by batch_normalize on the device (plonk/prover.rs:305-311); an all-zero column with a zero blind is the identity
    aff = params.commit_many_affine(polys + [polys[3]], blinds + [eng.Blind(0)])
    assert [cref.bytes_to_affine(a) for a in aff] == [_affine(curve, m) for m in many] + [None]
    assert (params.commit_many_affine(polys[:2], blinds[:2], lagrange=True) == aff[:2]).all()   # same generators registered twice here
    params.close()


def test_ipa_rounds(eng, table_mode):
    """The device IPA round loop (fold-free, resident generators) == the reference loop restated in the oracle
    (poly/commitment/prover.rs:100-142): every L_j, R_j and the final c, on both curves; commit() keeps working
    on the same base set (w at index n, u at n + 1)."""
    for curve, k in (("vesta", 10), ("pallas", 7), ("vesta", 1)):
        c = pasta.CURVES[curve]
        n, r = 1 << k, c.r
        bases = cref.gen_points(curve, SEED + 200 + k, n + 2)
        params = eng.Params(curve, k, bases[:n], bases[:n], bases[n:n + 1], u=bases[n + 1:n + 2])
        pp = cref.gen_scalars(c.scalar, SEED + 210 + k, n)
        ch = pasta.gen_scalars(c.scalar, SEED + 220 + k, k)
        lr = pasta.gen_scalars(c.scalar, SEED + 230 + k, k)
        rr = pasta.gen_scalars(c.scalar, SEED + 240 + k, k)
        x3, z = pasta.gen_scalars(c.scalar, SEED + 250 + k, 2)
        want_l, want_r, want_c = cref.ipa_rounds(curve, bases, k, pp, x3, z, cref.ints_to_bytes(ch), cref.ints_to_bytes(lr),
                                                 cref.ints_to_bytes(rr))
        seen = []
        def challenge(j, l_j, r_j):
            seen.append((l_j.copy(), r_j.copy()))
            return ch[j]
        got_l, got_r, got_c = params.ipa_rounds(pp, x3, z, challenge, lr, rr)
        assert got_c == want_c
        for j in range(k):
            assert cref.jac_to_affine(curve, got_l[j]).tobytes() == want_l[j].tobytes(), (curve, k, j)
            assert cref.jac_to_affine(curve, got_r[j]).tobytes() == want_r[j].tobytes(), (curve, k, j)
        assert len(seen) == k
        blind = eng.Blind(lr[0])
        want = cref.bytes_to_affine(cref.best_multiexp(curve, np.concatenate([pp, cref.ints_to_bytes([blind.value])]), bases[:n + 1]))
        assert _affine(curve, params.commit(pp, blind)) == want
        params.close()


def test_ipa_errors(eng):
    """Misuse fails loudly: no u / no table, fold without round, round without fold."""
    import ctypes
    from halo2_b200 import lib as L
    curve, k = "vesta", 4
    n = 1 << k
    bases = cref.gen_points(curve, SEED + 260, n + 2)
    params = eng.Params(curve, k, bases[:n], bases[:n], bases[n:n + 1])
    with pytest.raises(L.H2Error):
        params.ipa_rounds(np.zeros((n, 32), dtype=np.uint8), 1, 1, lambda j, a, b: 1, [1] * k, [1] * k)
    params.close()
    params = eng.Params(curve, k, bases[:n], bases[:n], bases[n:n + 1], u=bases[n + 1:n + 2])
    lib = L.init()
    sess = ctypes.c_uint64(0)
    one = L.fe_bytes(1)
    L.check(lib.h2_ipa_begin(params._h_g, ctypes.c_uint32(k), L.ptr(np.zeros((n, 32), dtype=np.uint8)), L.ptr(one), L.REPR_CANONICAL, ctypes.byref(sess)))
    assert lib.h2_ipa_fold(sess, L.ptr(one), L.ptr(one), L.REPR_CANONICAL) != 0
    out = np.zeros((2, 96), dtype=np.uint8)
    L.check(lib.h2_ipa_round(sess, L.ptr(one), L.ptr(one), L.ptr(one), L.REPR_CANONICAL, L.ptr(out)))
    assert lib.h2_ipa_round(sess, L.ptr(one), L.ptr(one), L.ptr(one), L.REPR_CANONICAL, L.ptr(out)) != 0
    cb = np.zeros((2, 32), dtype=np.uint8)
    assert lib.h2_ipa_finish(sess, L.REPR_CANONICAL, L.ptr(cb)) != 0          # rounds incomplete: error, session freed
    assert lib.h2_ipa_finish(sess, L.REPR_CANONICAL, None) != 0               # already gone
    assert lib.h2_ipa_begin(params._h_gl, ctypes.c_uint32(k), L.ptr(np.zeros((n, 32), dtype=np.uint8)), L.ptr(one), L.REPR_CANONICAL, ctypes.byref(sess)) != 0
    params.close()


def _msm_flags():
    from halo2_b200 import lib as L
    f = ctypes.c_uint32(0)
    L.check(L.init().h2_test_last_msm_flags(ctypes.byref(f)))
    return f.value


def test_msm_sort_paths(eng):
    """Uniform scalars take the single-pass binned sort (no bin overflows at the automatic capacity -- at 2^12, 2^16
    and, in test_best_multiexp_2pow20, at 2^20); all-equal scalars overflow and fall back to the exact sort; forcing
    the exact sort gives the same point."""
    from halo2_b200 import lib as L
    lib = L.init()
    curve, c = "pallas", pasta.PALLAS
    for k in (12, 16):
        n = 1 << k
        kb = cref.gen_scalars(c.scalar, SEED + 300 + k, n)
        pb = cref.gen_points(curve, SEED + 310 + k, n)
        want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
        for glv in (1, 0):
            L.check(lib.h2_set_glv(glv))
            try:
                assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == want
                assert _msm_flags() & 2 == 0, ("uniform scalars overflowed a bin", k, glv)
                L.check(lib.h2_set_sort_mode(1))
                assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == want
                assert _msm_flags() & 2 == 2
            finally:
                L.check(lib.h2_set_sort_mode(0))
                L.check(lib.h2_set_glv(1))
    n = 1 << 12
    pb = cref.gen_points(curve, SEED + 320, n)
    kb = cref.ints_to_bytes([pasta.gen_scalars(c.scalar, 5, 1)[0]] * n)
    assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
    assert _msm_flags() & 2 == 2          # every reference of a window in one bucket: overflow -> exact sort
    # resident (fixed-base) path: commits of uniform polynomials stay on the fast path
    k = 12
    g = cref.gen_points("vesta", SEED + 330, (1 << k) + 1)
    params = eng.Params("vesta", k, g[:-1], g[:-1], g[-1:])
    poly = cref.gen_scalars("fp", SEED + 331, 1 << k)
    want = cref.bytes_to_affine(cref.best_multiexp("vesta", np.concatenate([poly, cref.ints_to_bytes([9])]), g))
    assert _affine("vesta", params.commit(poly, eng.Blind(9))) == want
    assert _msm_flags() & 2 == 0
    params.close()


def test_msm_chunked_upload(eng):
    """h2_msm with the bases uploaded, sorted and accumulated in chunks (forced at small n): same point, including
    skewed scalars (exact-sort fallback per chunk), sizes that do not divide by the chunk count, and both curves."""
    from halo2_b200 import lib as L
    lib = L.init()
    try:
        # 4, 3, 2, 3, 1, 1 chunks (growing sizes: 1/16, 3/16, 6/16, 6/16 | 1/8, 3/8, 1/2 | 1/4, 3/4)
        for curve, n, thr in (("pallas", 4099, 4), ("vesta", 1 << 12, 11), ("vesta", 3000, 11), ("pallas", 70, 4), ("pallas", 17, 4),
                              ("vesta", 5, 1)):
            L.check(lib.h2_test_set_chunk_threshold(thr))
            c = pasta.CURVES[curve]
            pb = cref.gen_points(curve, SEED + 400 + n, n)
            for name, kb in (("random", cref.gen_scalars(c.scalar, SEED + 401 + n, n)),
                             ("equal", cref.ints_to_bytes([pasta.gen_scalars(c.scalar, 3, 1)[0]] * n)),
                             ("mix01", cref.ints_to_bytes([i & 1 for i in range(n)]))):
                want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
                for glv in (1, 0):
                    L.check(lib.h2_set_glv(glv))
                    assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == want, (curve, n, name, glv)
    finally:
        L.check(lib.h2_set_glv(1))
        L.check(lib.h2_test_set_chunk_threshold(19))


def test_resident_polynomials(eng, table_mode):
    """The device-resident pipeline (upload once; lagrange -> coeff -> extended -> coeff and commits on handles) gives
    exactly what the host-buffer calls -- and therefore the oracle -- give."""
    field, curve, k, j = "fp", "vesta", 9, 5
    n = 1 << k
    zeta = pasta.zeta_candidates(field)[0]
    dom = eng.EvaluationDomain(field, j, k, zeta)
    g = cref.gen_points(curve, SEED + 500, n + 1)
    params = eng.Params(curve, k, g[:n], g[:n], g[n:])
    vals = [cref.gen_scalars(field, SEED + 501 + i, n) for i in range(3)]
    vals[2] = cref.ints_to_bytes([i & 1 for i in range(n)])
    blinds = [eng.Blind(3 + i) for i in range(3)]
    res = [eng.ResidentPoly(field, n, v) for v in vals]
    assert (res[0].download() == vals[0]).all()
    # commit_lagrange on the values, then to coefficients in place, commit again, extend, come back
    # (Jacobian coordinates depend on the order the atomics hand out bin slots: compare the points)
    want = params.commit_lagrange_many(vals, blinds)
    got = params.commit_resident(res, blinds, lagrange=True)
    assert [_affine(curve, x) for x in got] == [_affine(curve, x) for x in want]
    for r in res:
        dom.lagrange_to_coeff_resident(r)
    coeffs = [dom.lagrange_to_coeff(v) for v in vals]
    for r, cf in zip(res, coeffs):
        assert (r.download() == cf).all()
    assert [_affine(curve, x) for x in params.commit_resident(res, blinds)] == [_affine(curve, x) for x in params.commit_many(coeffs, blinds)]
    assert _affine(curve, params.commit_resident(res[:1], blinds[:1])[0]) == _affine(curve, params.commit(coeffs[0], blinds[0]))
    want0 = cref.bytes_to_affine(cref.best_multiexp(curve, np.concatenate([coeffs[0], cref.ints_to_bytes([blinds[0].value])]), g))
    assert _affine(curve, params.commit_resident(res[:1], blinds[:1])[0]) == want0        # ... and the oracle
    ext = dom.coeff_to_extended_resident(res[0])
    want_ext = dom.coeff_to_extended(coeffs[0])
    assert (ext.download() == want_ext).all()
    back = dom.extended_to_coeff_resident(ext)
    assert (back.download() == dom.extended_to_coeff(want_ext)).all()
    o = pasta.EvaluationDomain(field, j, k, zeta)
    assert cref.bytes_to_ints(res[1].download()) == o.lagrange_to_coeff(cref.bytes_to_ints(vals[1]))   # and the oracle
    # misuse fails loudly
    from halo2_b200 import lib as L
    with pytest.raises(L.H2Error):
        dom.lagrange_to_coeff_resident(eng.ResidentPoly(field, n // 2))
    with pytest.raises(L.H2Error):
        params.commit_resident([eng.ResidentPoly("fq", n)], blinds[:1])
    for r in res + [ext, back]:
        r.close()
    params.close()


def test_fixed_base_graph_replay(eng, table_mode):
    """Fixed-base MSMs replay a captured CUDA graph from their third call with the same parameters: six different
    polynomials in a row (and batches of them) still each give their own commitment; switching the replay off gives
    the same points."""
    from halo2_b200 import lib as L
    lib = L.init()
    curve, c, k = "vesta", pasta.VESTA, 11
    n = 1 << k
    g = cref.gen_points(curve, SEED + 600, n + 1)
    params = eng.Params(curve, k, g[:n], g[:n], g[n:])
    polys = [cref.gen_scalars(c.scalar, SEED + 601 + i, n) for i in range(6)]
    polys[4] = cref.ints_to_bytes([i % 3 for i in range(n)])          # overflows the bins: exact sort inside the graph
    blinds = [eng.Blind(11 + i) for i in range(6)]
    want = [cref.bytes_to_affine(cref.best_multiexp(curve, np.concatenate([p, cref.ints_to_bytes([b.value])]), g)) for p, b in zip(polys, blinds)]
    try:
        for on in (1, 0, 1):
            L.check(lib.h2_test_set_graphs(on))
            for rep in range(2):
                for i in range(6):
                    assert _affine(curve, params.commit(polys[i], blinds[i])) == want[i], (on, rep, i)
            for i in range(0, 6, 3):
                many = params.commit_many(polys[i:i + 3], blinds[i:i + 3])
                assert [_affine(curve, x) for x in many] == want[i:i + 3], (on, i)
                many = params.commit_many(polys[i:i + 3][::-1], blinds[i:i + 3][::-1])
                assert [_affine(curve, x) for x in many] == want[i:i + 3][::-1]
    finally:
        L.check(lib.h2_test_set_graphs(1))
        params.close()


def test_best_multiexp_2pow20(eng):
    """BASELINE.json config 3 at full size (Pallas) against the C restatement."""
    curve, c = "pallas", pasta.PALLAS
    n = 1 << 20
    kb = cref.gen_scalars(c.scalar, SEED + 3, n)
    pb = cref.gen_points(curve, SEED + 33, n)
    want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
    assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == want
    assert _msm_flags() & 2 == 0          # the binned single-pass sort held (no bin overflow)


def test_point_sum(eng):
    """The multi-GPU combine step: sum of per-shard Jacobian partials == MSM of the whole."""
    from halo2_b200 import lib as L
    curve, c = "vesta", pasta.VESTA
    n, shards = 3000, 4
    kb = cref.gen_scalars(c.scalar, SEED + 11, n)
    pb = cref.gen_points(curve, SEED + 12, n)
    parts = np.zeros((shards, 96), dtype=np.uint8)
    step = n // shards
    for s in range(shards):
        lo, hi = s * step, n if s == shards - 1 else (s + 1) * step
        parts[s] = eng.best_multiexp(kb[lo:hi], pb[lo:hi], curve)
    out = np.zeros(96, dtype=np.uint8)
    lib = L.init()
    L.check(lib.h2_point_sum(L.CURVE_ID[curve], L.ptr(parts), ctypes.c_size_t(shards), L.REPR_CANONICAL, L.ptr(out)))
    assert _affine(curve, out) == cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))


# ------------------------------------------------------------------------------------------ K10 / K11
def _ecfft_inputs(curve, k, seed):
    n = 1 << k
    g = cref.gen_points(curve, seed, n)
    if n > 4:
        g[3] = 0                                   # an identity among the inputs
        g[n - 1] = g[1]                            # and a repeated point
    return g


@pytest.fixture(params=[1, 0], ids=["quad", "thread"])
def ecfft_form(request):
    from halo2_b200 import lib as L
    L.check(L.init().h2_test_set_ecfft_quad(request.param))
    yield request.param
    L.check(L.init().h2_test_set_ecfft_quad(-1))


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
@pytest.mark.parametrize("k", [0, 1, 2, 5, 8, 10])
def test_ec_fft_and_lagrange_generators(eng, curve, k, ecfft_form):
    """best_fft at G = curve point (arithmetic.rs:192-295 via FftGroup :17-27) and the g -> g_lagrange derivation of
    Params::new (poly/commitment.rs:74-101), against the oracle's restatement; batch_normalize on its own."""
    c = pasta.CURVES[curve]
    r, n = c.r, 1 << k
    g = _ecfft_inputs(curve, k, 300 + k)
    omega_inv = pasta.inv(pasta.omega_for_k(c.scalar, k), r) if k else 1
    minv = pow(pasta.inv(2, r), k, r)
    want_gl = cref.params_lagrange(curve, g, k, omega_inv, minv)
    assert (eng.lagrange_generators(curve, k, g) == want_gl).all()
    # the bare network with a random (non-root) omega like benches/fft.rs:17, Jacobian in / out
    w = pasta.gen_scalars(c.scalar, 17 + k, 1)[0]
    jac = cref.affine_to_jacobian_bytes(g)
    got = eng.best_fft_curve(jac.copy(), w, k, curve)
    want = cref.batch_normalize(curve, cref.ec_fft(curve, jac, w, k))
    assert (cref.batch_normalize(curve, got) == want).all()
    assert (eng.batch_normalize(got, curve) == want).all()
    if k == 5:
        with pytest.raises(AssertionError):      # arithmetic.rs:205
            eng.best_fft_curve(jac.copy(), w, k + 1, curve)


def test_params_from_generators_commit_lagrange(eng):
    """Params built from g alone (g_lagrange derived on the device) satisfies the reference's own property
    poly/commitment.rs:258-302: commit_lagrange(a) == commit(lagrange_to_coeff(a)); the Montgomery ABI form agrees."""
    from halo2_b200 import lib as L
    curve, c, k = "vesta", pasta.VESTA, 9
    g = cref.gen_points(curve, SEED + 40, 1 << k)
    wu = cref.gen_points(curve, SEED + 41, 2)
    params = eng.Params.from_generators(curve, k, g, wu[:1], wu[1:])
    dom = eng.EvaluationDomain(c.scalar, 2, k, pasta.zeta_candidates(c.scalar)[0])
    a = cref.gen_scalars(c.scalar, SEED + 42, 1 << k)
    alpha = pasta.gen_scalars(c.scalar, SEED + 43, 1)[0]
    lhs = _affine(curve, params.commit_lagrange(a, eng.Blind(alpha)))
    assert lhs == _affine(curve, params.commit(dom.lagrange_to_coeff(a), eng.Blind(alpha)))
    assert lhs == cref.bytes_to_affine(cref.best_multiexp(curve, np.concatenate([a, cref.ints_to_bytes([alpha])]),
                                                          np.concatenate([params.g_lagrange, wu[:1]])))
    # Montgomery repr at the ABI (pasta's in-memory form): same points
    m, R = pasta.FIELDS[c.base], 1 << 256
    gm = cref.ints_to_bytes([v * R % m for v in cref.bytes_to_ints(g.reshape(-1, 32))]).reshape(-1, 64)
    ms = pasta.FIELDS[c.scalar]
    omega_inv = pasta.inv(pasta.omega_for_k(c.scalar, k), ms)
    minv = pow(pasta.inv(2, ms), k, ms)
    out = np.zeros((1 << k, 64), dtype=np.uint8)
    lib = L.init()
    L.check(lib.h2_params_lagrange(L.CURVE_ID[curve], L.ptr(gm), ctypes.c_uint32(k), L.ptr(L.fe_bytes(omega_inv * R % ms)),
                                   L.ptr(L.fe_bytes(minv * R % ms)), L.REPR_MONTGOMERY, L.ptr(out)))
    back = cref.ints_to_bytes([v * pasta.inv(R, m) % m for v in cref.bytes_to_ints(out.reshape(-1, 32))]).reshape(-1, 64)
    assert (back == params.g_lagrange).all()
    params.close()


def test_small_multiexp_and_batch_normalize(eng):
    """arithmetic.rs:116-136 (benches/arithmetic.rs:29 uses 2 terms) and the prover's normalisation of its commitments
    (plonk/prover.rs:305-311): a batch of commits -> affine, identity included."""
    curve, c = "pallas", pasta.PALLAS
    kb = cref.gen_scalars(c.scalar, SEED + 50, 5)
    pb = cref.gen_points(curve, SEED + 51, 5)
    for m in (0, 1, 2, 5):
        got = _affine(curve, eng.small_multiexp(kb[:m], pb[:m], curve))
        assert got == pasta.to_affine(c, pasta.small_multiexp(c, cref.bytes_to_ints(kb[:m]), [cref.bytes_to_affine(p) for p in pb[:m]]))
    pts = np.stack([eng.best_multiexp(kb[:m], pb[:m], curve) for m in (0, 1, 2, 5, 0, 3)] * 7)   # 42 points: 3 chunks of 16
    want = np.stack([cref.jac_to_affine(curve, p) for p in pts])
    assert (eng.batch_normalize(pts, curve) == want).all()
    assert eng.batch_normalize(np.zeros((0, 96), dtype=np.uint8), curve).shape == (0, 64)


def test_accum_ways(eng):
    """Small MSMs accumulate with 1, 2 or 4 quads of lanes per work item (msm_accum0_multi_kernel) or one pair of lanes
    (ways = 0, msm_accum0_pair_kernel): same points -- incl. a 0/1/2 column and a constant column, which crowd the references
    into a few buckets.  The window-table entries of distinct generators are distinct, so those buckets still sum distinct
    points; the P + P / P + (-P) branches of the pair and quad formulas are run by tests/test_gpu_group_law.py."""
    from halo2_b200 import lib as L
    lib = L.init()
    curve, c, k = "vesta", pasta.VESTA, 10
    n = 1 << k
    g = cref.gen_points(curve, SEED + 600, n + 1)
    polys = [cref.gen_scalars(c.scalar, SEED + 601, n), cref.ints_to_bytes([i % 3 for i in range(n)]), cref.ints_to_bytes([5] * n)]
    blind = eng.Blind(9)
    kb = cref.gen_scalars(c.scalar, SEED + 602, 3000)
    pb = cref.gen_points(curve, SEED + 603, 3000)
    want_one = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
    wants = [cref.bytes_to_affine(cref.best_multiexp(curve, np.concatenate([p, cref.ints_to_bytes([9])]), g)) for p in polys]
    try:
        for ways in (1, 2, 4, 0, 12, 14):     # 12 / 14: 2 / 4 independent lanes per item (msm_accum0_split_kernel)
            L.check(lib.h2_test_set_accum_ways(ways))
            params = eng.Params(curve, k, g[:n], g[:n], g[n:])
            for rep in range(3):     # eager, captured, replayed
                assert [_affine(curve, params.commit(p, blind)) for p in polys] == wants, (ways, rep)
            assert [_affine(curve, m) for m in params.commit_many(polys, [blind] * 3)] == wants, ways
            params.close()
            assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == want_one, ways
        assert lib.h2_test_set_accum_ways(3) != 0
    finally:
        L.check(lib.h2_test_set_accum_ways(12))


# ------------------------------------------------------------------------------------------ K13
def test_point_codec_and_params_io(eng, goldens):
    """C::to_bytes / C::from_bytes on the device (book/src/background/curves.md:203-240) against the oracle and the
    reference's golden commitments; Params::{write, read} (poly/commitment.rs:168-205) byte-for-byte and round trip; invalid
    encodings and short files fail like C::read / read_exact."""
    import io
    from halo2_b200 import lib as L
    for curve in ("pallas", "vesta"):
        c = pasta.CURVES[curve]
        pts = [cref.bytes_to_affine(p) for p in cref.gen_points(curve, SEED + 700, 300)] + [None, pasta.generator(c)]
        if curve == "vesta":
            for vk in (goldens["vk_plonk_api_k5"], goldens["vk_lookup_range_check_k11"]):
                pts += [(int(x, 16), int(y, 16)) for x, y in vk["fixed_commitments"] + vk["permutation_commitments"]]
        xy = cref.affines_to_bytes(pts)
        enc = eng.compress_points(xy, curve)
        assert enc.tobytes() == b"".join(pasta.compress(p) for p in pts)
        assert (eng.decompress_points(enc, curve) == xy).all()
        flipped = enc.copy()
        flipped[:300, 31] ^= 0x80
        assert [cref.bytes_to_affine(b) for b in eng.decompress_points(flipped[:300], curve)] == [(p[0], c.p - p[1]) for p in pts[:300]]
        nonres = next(x for x in range(2, 200) if pasta.fe_sqrt(c.base, (x ** 3 + 5) % c.p) is None)
        for bad_val in (nonres, c.p, (1 << 255) - 1, 1 << 255):
            batch = enc[:9].copy()
            batch[7] = np.frombuffer(bad_val.to_bytes(32, "little"), dtype=np.uint8)
            with pytest.raises(L.H2Error, match="index 7"):
                eng.decompress_points(batch, curve)
        assert eng.compress_points(np.zeros((0, 64), dtype=np.uint8), curve).shape == (0, 32)
    curve, c, k = "vesta", pasta.VESTA, 5
    po = pasta.Params(c, k)
    params = eng.Params(curve, k, cref.affines_to_bytes(po.g), cref.affines_to_bytes(po.g_lagrange), cref.affines_to_bytes([po.w]),
                        u=cref.affines_to_bytes([po.u]))
    buf = io.BytesIO()
    params.write(buf)
    assert buf.getvalue() == pasta.params_to_bytes(k, po.g, po.g_lagrange, po.w, po.u)
    back = eng.Params.read(curve, io.BytesIO(buf.getvalue()))
    assert back.k == k and (back.g == params.g).all() and (back.g_lagrange == params.g_lagrange).all() and (back.w == params.w).all() and (back.u == params.u).all()
    a = cref.gen_scalars(c.scalar, SEED + 710, 1 << k)
    assert _affine(curve, back.commit_lagrange(a, eng.Blind(4))) == pasta.to_affine(c, po.commit_lagrange(cref.bytes_to_ints(a), 4))
    with pytest.raises(EOFError):
        eng.Params.read(curve, io.BytesIO(buf.getvalue()[:-1]))
    corrupt = bytearray(buf.getvalue())
    corrupt[4 + 32 * 3: 4 + 32 * 4] = (c.p).to_bytes(32, "little")
    with pytest.raises(L.H2Error):
        eng.Params.read(curve, io.BytesIO(bytes(corrupt)))
    params.close()
    back.close()


# ------------------------------------------------------------------------------------------ K14
@pytest.mark.parametrize("field", ["fp", "fq"])
def test_poly_reductions(eng, field):
    """eval_polynomial / compute_inner_product / kate_division (arithmetic.rs:297-341) on resident and host polynomials against
    the restated loops, at the chunk-tree's edge sizes and at k = 14; kate_division's defining identity; misuse fails."""
    from halo2_b200 import lib as L
    m = pasta.FIELDS[field]
    lib = L.init()
    try:
        for cta in (1, 0):      # one CTA per polynomial (n <= 2^16) / the level tree: same values
            L.check(lib.h2_test_set_poly_cta(cta))
            for n in (1, 2, 3, 32, 33, 511, 1025, 1 << 14) + ((1000, 1 << 16, (1 << 16) + 1) if cta else ()):
                a = cref.gen_scalars(field, SEED + 800 + n, n)
                c = cref.gen_scalars(field, SEED + 801 + n, n)
                ai, ci = cref.bytes_to_ints(a), cref.bytes_to_ints(c)
                for x in (pasta.gen_scalars(field, SEED + 802 + n, 1)[0], 0, 1):
                    assert eng.eval_polynomial(a, x, field) == pasta.eval_polynomial(field, ai, x), (cta, n, x)
                    q = eng.kate_division(a, x, field)
                    assert cref.bytes_to_ints(q) == pasta.kate_division(field, ai, x), (cta, n, x)
                assert eng.compute_inner_product(a, c, field) == pasta.compute_inner_product(m, ai, ci)
    finally:
        L.check(lib.h2_test_set_poly_cta(0))
    # a batch of resident polynomials, each at its own point (the prover's evaluation loop, plonk/prover.rs: eval_polynomial per
    # column and rotation), x = 0 and x = 1 included; the quotients stay on the device and evaluate to (a(z) - a(x)) / (z - x)
    n, batch = 1 << 12, 5
    polys = [cref.gen_scalars(field, SEED + 810 + b, n) for b in range(batch)]
    res = [eng.ResidentPoly(field, n, p) for p in polys]
    pts = pasta.gen_scalars(field, SEED + 820, batch - 2) + [0, 1]
    want = [pasta.eval_polynomial(field, cref.bytes_to_ints(p), x) for p, x in zip(polys, pts)]
    assert eng.eval_polynomial_resident(res, pts) == want
    assert eng.inner_product_resident(res, res[1:] + res[:1]) == [pasta.compute_inner_product(m, cref.bytes_to_ints(p), cref.bytes_to_ints(q_))
                                                                   for p, q_ in zip(polys, polys[1:] + polys[:1])]
    quot = eng.kate_division_resident(res, pts)
    z = pasta.gen_scalars(field, SEED + 830, 1)[0]
    qz = eng.eval_polynomial_resident(quot, [z] * batch, n=n - 1)
    az = eng.eval_polynomial_resident(res, [z] * batch)
    for b in range(batch):
        assert qz[b] * (z - pts[b]) % m == (az[b] - want[b]) % m, b
        assert (quot[b].download(n - 1) == cref.ints_to_bytes(pasta.kate_division(field, cref.bytes_to_ints(polys[b]), pts[b]))).all()
    # divide_by_vanishing_poly (poly/domain.rs:329-348) on host and resident extended evaluations; the quotient pipeline of
    # plonk/vanishing/prover.rs:81-88 end to end on the device: coeff_to_extended -> (h = a * a here) -> divide -> extended_to_coeff
    zeta = pasta.zeta_candidates(field)[0]
    for j, k in ((3, 5), (5, 9)):
        d_or = pasta.EvaluationDomain(field, j, k, zeta)
        d = eng.EvaluationDomain(field, j, k, zeta)
        assert d.t_evaluations == d_or.t_evaluations
        ext = cref.gen_scalars(field, SEED + 840 + k, d.extended_len())
        want_div = cref.ints_to_bytes(d_or.divide_by_vanishing_poly(cref.bytes_to_ints(ext)))
        assert (d.divide_by_vanishing_poly(ext) == want_div).all()
        r = eng.ResidentPoly(field, d.extended_len(), ext)
        d.divide_by_vanishing_poly_resident(r)
        assert (r.download() == want_div).all()
        assert (d.extended_to_coeff_resident(r).download() == d.extended_to_coeff(want_div)).all()
        r.close()
    with pytest.raises(L.H2Error):      # the quotient cannot overwrite its dividend
        eng.kate_division_resident(res[:1], pts[:1], dst=res[:1])
    with pytest.raises(AssertionError):  # arithmetic.rs:311
        eng.compute_inner_product(polys[0], polys[1][:-1], field)
    for r in res + quot:
        r.close()


# ------------------------------------------------------------------------------------------ K15
@pytest.mark.parametrize("field", ["fp", "fq"])
def test_ast_evaluator_and_quotient_pipeline(eng, field):
    """Evaluator::evaluate (poly/evaluator.rs:129-228) on the device against the restated tree walk, in both bases; then the
    quotient pipeline of plonk/vanishing/prover.rs:81-88 without leaving HBM: coeff_to_extended of four columns, an h(X)-shaped
    Ast over them, divide_by_vanishing_poly, extended_to_coeff -- against the same steps on the oracle."""
    from halo2_b200 import lib as L
    from halo2_b200.evaluator import Ast
    zeta = pasta.zeta_candidates(field)[0]
    y, theta = pasta.gen_scalars(field, SEED + 1010, 2)

    def expr(a, b, c, q):
        gate0 = (a * b - c) * q
        gate1 = (a.with_rotation(1) - a) * (b.with_rotation(-1) + Ast.constant_term(7)) * 3
        perm = (c + Ast.linear_term(theta) + Ast.constant_term(11)) * (a.with_rotation(-2) + b * theta)
        return Ast.distribute_powers([gate0, gate1, -perm, q.with_rotation(3)], y) + Ast.constant_term(0) * 5

    for basis, j, k in (("extended", 5, 6), ("lagrange", 2, 7), ("extended", 3, 10)):
        d_or = pasta.EvaluationDomain(field, j, k, zeta)
        d = eng.EvaluationDomain(field, j, k, zeta)
        n = d.n if basis == "lagrange" else d.extended_len()
        polys = [cref.gen_scalars(field, SEED + 1000 + i + k, n) for i in range(4)]
        ev = eng.Evaluator(d, basis)
        leaves = [ev.register_poly(p) for p in polys]
        ast = expr(*leaves)
        want = pasta.ast_evaluate(d_or, basis, _ast_tuple(ast), [cref.bytes_to_ints(p) for p in polys])
        got = ev.evaluate(ast)
        assert cref.bytes_to_ints(got.download()) == want, (basis, k)
        for node in (Ast.constant_term(0), Ast.linear_term(0), Ast.linear_term(9), leaves[2].with_rotation(-1)):   # evaluator.rs:625-660
            assert cref.bytes_to_ints(ev.evaluate(node, out=got).download()) == pasta.ast_evaluate(d_or, basis, _ast_tuple(node),
                                                                                                     [cref.bytes_to_ints(p) for p in polys])
        with pytest.raises(L.H2Error):       # the output cannot be an operand
            ev.evaluate(leaves[0], out=ev.polys[0])
        got.close()
        ev.close()
    # resident quotient pipeline at k = 8, degree 5 (extended_k = 10)
    j, k = 5, 8
    d_or = pasta.EvaluationDomain(field, j, k, zeta)
    d = eng.EvaluationDomain(field, j, k, zeta)
    cols = [cref.gen_scalars(field, SEED + 1100 + i, d.n) for i in range(4)]          # coefficient form
    res = [eng.ResidentPoly(field, d.n, c_) for c_ in cols]
    ext = [d.coeff_to_extended_resident(r) for r in res]
    ev = eng.Evaluator(d, "extended")
    h = ev.evaluate(expr(*[ev.register_poly(e) for e in ext]))
    d.divide_by_vanishing_poly_resident(h)
    got = d.extended_to_coeff_resident(h).download()
    ext_or = [d_or.coeff_to_extended(cref.bytes_to_ints(c_)) for c_ in cols]
    h_or = d_or.divide_by_vanishing_poly(pasta.ast_evaluate(d_or, "extended", _ast_tuple(expr(*[eng.AstLeaf(i) for i in range(4)])), ext_or))
    assert cref.bytes_to_ints(got) == d_or.extended_to_coeff(h_or)
    # misuse: malformed programs are rejected before anything is launched
    lib = L.init()
    out = eng.ResidentPoly(field, d.extended_len())
    hs = (ctypes.c_uint64 * 1)(ext[0]._h.value)
    for bad in ([[3, 0, 0, 0]], [[0, 0, 0, 0], [0, 0, 0, 0]], [[0, 5, 0, 0]], [[1, 0, 0, 0]], [[9, 0, 0, 0]], [[0, 0, 0, 0]] * 30):
        code = np.array(bad, dtype=np.uint32)
        assert lib.h2_poly_eval_ast(out._h, hs, ctypes.c_size_t(1), ctypes.c_uint32(d.extended_k), code.ctypes.data_as(ctypes.c_void_p),
                                    ctypes.c_size_t(code.shape[0]), None, ctypes.c_size_t(0), None, None, L.REPR_CANONICAL) != 0, bad
    for r in res + ext + [h, out]:
        r.close()
