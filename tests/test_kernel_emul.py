"""CPU checks of the DEVICE code's logic: halo2_b200/csrc/*.cuh compiled for the host
(tests/kernel_emul, PTX carry flag emulated) and run serially against the oracle.  Covers the
Montgomery multiply, the XYZZ group law, the NTT pass geometry (single and multi-pass, all fused
modes) and the whole MSM pipeline (digits, counting sort, chunked accumulation with multi-level
partial merging, hierarchical bucket reduce) including skewed scalars and degenerate bases."""
import ctypes

import numpy as np
import pytest

from oracle import cref, pasta
from tests.ast_cases import _ast_tuple, _quotient_like_ast
from tests.kernel_emul import build as emul_build

SEED = 0x48414C4F32


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emul_build.build())


def _fop(emu, f, op, a, b=0):
    out = np.zeros(32, dtype=np.uint8)
    emu.emu_field_op(cref.FIELD_ID[f], op, cref._p(cref._fe(a)), cref._p(cref._fe(b)), cref._p(out))
    return int.from_bytes(out.tobytes(), "little")


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_emul_field(emu, field):
    m = pasta.FIELDS[field]
    xs = pasta.gen_scalars(field, SEED, 200) + [0, 1, 2, m - 1, m - 2, 1 << 254, (1 << 254) - 1, m - (1 << 32),
                                                0xFFFFFFFF, 1 << 32, (1 << 224) - 1, m >> 1]
    for i, a in enumerate(xs):
        b = xs[(i * 7 + 3) % len(xs)]
        assert _fop(emu, field, 0, a, b) == (a + b) % m
        assert _fop(emu, field, 1, a, b) == (a - b) % m
        assert _fop(emu, field, 2, a, b) == a * b % m
        assert _fop(emu, field, 4, a) == a * a % m
        assert _fop(emu, field, 5, a) == (-a) % m
    for a in xs[:10] + xs[-6:]:
        if a:
            assert _fop(emu, field, 3, a) == pow(a, m - 2, m)
    # the divsteps inversion (fe_inv_gcd): every sample, the structured values, small and near-modulus inputs; 0 -> 0
    for a in xs + [3, 5, 1 << 30, (1 << 30) - 1, 1 << 60, m - 3, (m + 1) // 2, pow(2, 256, m), pow(2, 512, m), (1 << 253) + 12345]:
        assert _fop(emu, field, 7, a) == (pow(a, m - 2, m) if a else 0), hex(a)


def _cop(emu, curve, op, a, b, i=0):
    out = np.zeros(64, dtype=np.uint8)
    emu.emu_curve_op(cref.CURVE_ID[curve], op, cref._p(np.ascontiguousarray(a)), cref._p(np.ascontiguousarray(b)), ctypes.c_uint64(i),
                     cref._p(out))
    return cref.bytes_to_affine(out)


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_curve(emu, curve):
    """The serial XYZZ group law against the oracle: on affine operands (ZZ = 1, ops 0 - 2) and, as h2_test_curve_op's ops 3 - 6
    run it on the device, on operands rescaled to ZZ != 1 (element index i % 4 != 0; i % 4 == 0 keeps ZZ = 1)."""
    c = pasta.CURVES[curve]
    pts = pasta.gen_points(c, 5, 8)
    g = pasta.generator(c)
    two = lambda p: pasta.to_affine(c, pasta.jac_double(c, pasta.to_jac(p)))   # noqa: E731
    cases = [(pts[0], pts[1]), (pts[2], pts[2]), (pts[3], (pts[3][0], c.p - pts[3][1])), (None, pts[4]), (pts[5], None),
             (None, None), (g, g), (g, (g[0], c.p - g[1])), (pts[6], two(pts[6])), (two(pts[6]), pts[6])]
    for j, (a, b) in enumerate(cases):
        A, B = cref.affines_to_bytes([a])[0], cref.affines_to_bytes([b])[0]
        want = pasta.to_affine(c, pasta.jac_add(c, pasta.to_jac(a), pasta.to_jac(b)))
        dbl = pasta.to_affine(c, pasta.jac_double(c, pasta.to_jac(a)))
        assert _cop(emu, curve, 0, A, B) == want
        assert _cop(emu, curve, 1, A, B) == want
        assert _cop(emu, curve, 2, A, B) == dbl
        for i in (4 * j, 4 * j + 1, 4 * j + 2, 4 * j + 7):
            assert _cop(emu, curve, 3, A, B, i) == want, (j, i)
            assert _cop(emu, curve, 4, A, B, i) == want, (j, i)
            assert _cop(emu, curve, 5, A, B, i) == dbl, (j, i)
    for j, k in enumerate(list(range(0, 21)) + [63, 64, 255, 256, 270]):
        for a in (pts[7], g, None):
            kb = np.zeros(64, dtype=np.uint8)
            kb[:4] = np.frombuffer(int(k).to_bytes(4, "little"), dtype=np.uint8)
            want = pasta.to_affine(c, pasta.scalar_mul(c, pow(2, k, c.r), a))
            for i in (4 * j, 4 * j + 3):
                assert _cop(emu, curve, 6, cref.affines_to_bytes([a])[0], kb, i) == want, (k, i)
    for k in pasta.gen_scalars(c.scalar, 3, 3) + [0, 1, c.r - 1]:
        kb = np.zeros(64, dtype=np.uint8)
        kb[:32] = cref._fe(k)
        assert _cop(emu, curve, 8, cref.affines_to_bytes([pts[7]])[0], kb) == pasta.to_affine(c, pasta.scalar_mul(c, k, pts[7]))


def _ntt(emu, f, mode, a, in_log, log_n, omega, zeta=None, div=None, out_len=None, nthr=64):
    n = 1 << log_n
    out_len = n if out_len is None else out_len
    out = np.zeros((out_len, 32), dtype=np.uint8)
    emu.emu_ntt(cref.FIELD_ID[f], mode, cref._p(np.ascontiguousarray(a)), in_log, log_n, cref._p(cref._fe(omega)),
                cref._p(cref._fe(zeta)) if zeta is not None else None, cref._p(cref._fe(div)) if div is not None else None,
                ctypes.c_uint64(out_len), cref._p(out), nthr)
    return out


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_emul_ntt(emu, field):
    for log_n in (1, 2, 3, 5, 8, 10, 11, 12, 13, 15):
        a = cref.gen_scalars(field, 100 + log_n, 1 << log_n)
        for w in (pasta.omega_for_k(field, log_n), pasta.gen_scalars(field, 77, 1)[0]):
            got = _ntt(emu, field, 0, a, log_n, log_n, w, nthr=(7 if log_n < 8 else 64))
            assert (got == cref.best_fft(field, a, w, log_n)).all(), (field, log_n)
    # odd thread counts select the dense shared-memory layout of the bulk-copy (TMA) pass kernel (emul_ntt.cpp): row /
    # column spans, zero padding, the row-major output staging of the last pass, in_scale / out_scale inside the steps
    for log_n in (11, 12, 14, 15):
        a = cref.gen_scalars(field, 200 + log_n, 1 << log_n)
        for w in (pasta.omega_for_k(field, log_n), pasta.gen_scalars(field, 78, 1)[0]):
            assert (_ntt(emu, field, 0, a, log_n, log_n, w, nthr=63) == cref.best_fft(field, a, w, log_n)).all(), (field, log_n)
    for (j, k) in ((4, 9), (5, 11), (5, 12)):
        d = pasta.EvaluationDomain(field, j, k)
        a = cref.gen_scalars(field, 6, 1 << k)
        co = cref.ifft(field, a, d.omega_inv, k, d.ifft_divisor)
        assert (_ntt(emu, field, 1, a, k, k, d.omega_inv, div=d.ifft_divisor, nthr=63) == co).all()
        ext = cref.coeff_to_extended(field, co, k, d.extended_k, d.g_coset, d.extended_omega)
        assert (_ntt(emu, field, 2, co, k, d.extended_k, d.extended_omega, zeta=d.g_coset, nthr=63) == ext).all()
        ol = (1 << k) * (j - 1)
        back = cref.extended_to_coeff(field, ext, d.extended_k, d.extended_omega_inv, d.extended_ifft_divisor, d.g_coset, ol)
        got = _ntt(emu, field, 3, ext, d.extended_k, d.extended_k, d.extended_omega_inv, zeta=d.g_coset,
                   div=d.extended_ifft_divisor, out_len=ol, nthr=63)
        assert (got == back).all()
    for (j, k) in ((5, 5), (3, 6), (4, 9), (5, 11)):
        d = pasta.EvaluationDomain(field, j, k)
        a = cref.gen_scalars(field, 5, 1 << k)
        co = cref.ifft(field, a, d.omega_inv, k, d.ifft_divisor)
        assert (_ntt(emu, field, 1, a, k, k, d.omega_inv, div=d.ifft_divisor) == co).all()
        ext = cref.coeff_to_extended(field, co, k, d.extended_k, d.g_coset, d.extended_omega)
        assert (_ntt(emu, field, 2, co, k, d.extended_k, d.extended_omega, zeta=d.g_coset) == ext).all()
        ol = (1 << k) * (j - 1)
        back = cref.extended_to_coeff(field, ext, d.extended_k, d.extended_omega_inv, d.extended_ifft_divisor, d.g_coset, ol)
        got = _ntt(emu, field, 3, ext, d.extended_k, d.extended_k, d.extended_omega_inv, zeta=d.g_coset,
                   div=d.extended_ifft_divisor, out_len=ol)
        assert (got == back).all()


def _msm(emu, curve, kb, pb, c=0, mont=0, k0=0, gs=0, glv=False):
    # k0 = forced references per work item (T), gs = forced merge-level chunk
    out = np.zeros(96, dtype=np.uint8)
    r = (emu.emu_msm_glv if glv else emu.emu_msm)(cref.CURVE_ID[curve], cref._p(np.ascontiguousarray(kb)), cref._p(np.ascontiguousarray(pb)),
                    ctypes.c_size_t(kb.shape[0]), c, mont, k0, gs, cref._p(out))
    assert r > 0, r
    return cref.bytes_to_affine(cref.jac_to_affine(curve, out))


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_msm(emu, curve):
    c = pasta.CURVES[curve]
    for n in (1, 2, 3, 7, 33, 100, 257):
        kb = cref.gen_scalars(c.scalar, n, n)
        pb = cref.gen_points(curve, n + 1, n)
        want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
        for cb, k0, gs in ((0, 0, 0), (1, 0, 0), (5, 3, 4), (11, 5, 8), (16, 0, 0), (2, 4, 4), (9, 2, 4), (3, 1, 4)):
            assert _msm(emu, curve, kb, pb, cb, 0, k0, gs) == want, (n, cb, k0, gs)
            assert _msm(emu, curve, kb, pb, cb, 0, k0, gs, glv=True) == want, ("glv", n, cb, k0, gs)
        assert _msm(emu, curve, kb, pb, 0, 1, 0) == want   # Montgomery-encoded scalars
        assert _msm(emu, curve, kb, pb, 0, 1, 0, glv=True) == want
    n, r = 200, c.r
    pb = cref.gen_points(curve, 9, n)
    cases = {"zeros": [0] * n, "ones": [1] * n, "equal": [pasta.gen_scalars(c.scalar, 1, 1)[0]] * n,
             "mix01": [i & 1 for i in range(n)], "rminus1": [r - 1] * n, "pow2": [(1 << (i % 255)) % r for i in range(n)],
             "half": [(1 << 254) - 1 + i for i in range(n)]}
    for name, ks in cases.items():
        kb = cref.ints_to_bytes(ks)
        want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
        for cb, k0, gs in ((0, 0, 0), (4, 3, 4), (16, 4, 8), (7, 2, 4), (6, 1, 4)):
            assert _msm(emu, curve, kb, pb, cb, 0, k0, gs) == want, (name, cb, k0, gs)
            assert _msm(emu, curve, kb, pb, cb, 0, k0, gs, glv=True) == want, ("glv", name, cb, k0, gs)
    g = pasta.generator(c)
    pts = [cref.bytes_to_affine(x) for x in pb[:6]]
    pts2 = [g, g, (g[0], c.p - g[1]), None, pts[3], pts[3], pts[4], (pts[4][0], c.p - pts[4][1]), None, g] * 5
    ks = pasta.gen_scalars(c.scalar, 4, len(pts2))
    ks[0] = ks[1] = ks[2] = 5
    ks[6] = ks[7]
    kb, pb2 = cref.ints_to_bytes(ks), cref.affines_to_bytes(pts2)
    want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb2))
    for cb, k0, gs in ((0, 0, 0), (3, 2, 4), (13, 0, 0)):
        assert _msm(emu, curve, kb, pb2, cb, 0, k0, gs) == want
        assert _msm(emu, curve, kb, pb2, cb, 0, k0, gs, glv=True) == want


def _msm_fixed(emu, curve, kb, pb, c=0, t=0, kn=0):
    out = np.zeros(96, dtype=np.uint8)
    r = emu.emu_msm_fixed(cref.CURVE_ID[curve], cref._p(np.ascontiguousarray(kb)), cref._p(np.ascontiguousarray(pb)),
                          ctypes.c_size_t(kb.shape[0]), c, t, kn, cref._p(out))
    assert r > 0, r
    return cref.bytes_to_affine(cref.jac_to_affine(curve, out))


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_msm_fixed_base_table(emu, curve):
    """Resident-bases path: precomputed table T[w][i] = 2^(c w) G_i, one shared bucket set."""
    c = pasta.CURVES[curve]
    g = pasta.generator(c)
    for n in (1, 2, 9, 65, 130):
        kb = cref.gen_scalars(c.scalar, 40 + n, n)
        pts = [cref.bytes_to_affine(x) for x in cref.gen_points(curve, 41 + n, n)]
        if n >= 9:
            pts[3] = None            # identity base
            pts[5] = pts[4]          # duplicate
            pts[7] = (g[0], c.p - g[1])
        pb = cref.affines_to_bytes(pts)
        want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
        # 15 / 16 / 17 / 20: the default table windows from k = 14 on; 24 (2^23 buckets, seconds on the host) at one size only
        for cb, t, kn in ((0, 0, 0), (4, 2, 4), (7, 0, 0), (13, 3, 8), (15, 0, 0), (16, 0, 0), (17, 0, 0), (20, 0, 0)) + (((24, 0, 0),) if n == 130 else ()):
            assert _msm_fixed(emu, curve, kb, pb, cb, t, kn) == want, (n, cb, t, kn)
    n = 64
    pb = cref.gen_points(curve, 9, n)
    for ks in ([0] * n, [1] * n, [c.r - 1] * n, [i & 1 for i in range(n)], [(1 << (i * 4 % 255)) % c.r for i in range(n)]):
        kb = cref.ints_to_bytes(ks)
        want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
        for cb in (5, 15, 16, 17, 20):
            assert _msm_fixed(emu, curve, kb, pb, cb) == want, cb


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_msm_fixed_batch(emu, curve):
    """Several scalar vectors against one table in a single pass (bucket set = vector index): a uniform, a 0/1 and an r - 1
    column, at small windows and at the default table windows of production sizes (15, 17, 20) and the largest (24)."""
    c = pasta.CURVES[curve]
    n, sets = 70, 3
    pb = cref.gen_points(curve, 77, n)
    kbs = [cref.gen_scalars(c.scalar, 80 + k, n) for k in range(sets)]
    kbs[1] = cref.ints_to_bytes([i & 1 for i in range(n)])
    kbs[2] = cref.ints_to_bytes([c.r - 1] * n)
    out = np.zeros(96 * sets, dtype=np.uint8)
    for cb in (5, 13, 15, 17, 20, 24):
        r = emu.emu_msm_fixed_batch(cref.CURVE_ID[curve], cref._p(np.ascontiguousarray(np.concatenate(kbs))), cref._p(pb),
                                    ctypes.c_size_t(n), sets, cb, cref._p(out))
        assert r > 0
        for k in range(sets):
            got = cref.bytes_to_affine(cref.jac_to_affine(curve, out[96 * k:96 * k + 96]))
            assert got == cref.bytes_to_affine(cref.best_multiexp(curve, kbs[k], pb)), (cb, k)


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_ipa_rounds(emu, curve):
    """The fold-free IPA round loop (ipa.cuh: resident generators, challenge products folded into the scalars,
    L_j / R_j as a 2-set fixed-base MSM) yields the reference loop's L_j, R_j and c (prover.rs:100-142)."""
    c = pasta.CURVES[curve]
    r = c.r
    for k, cb in ((1, 5), (4, 6), (6, 9)):
        n = 1 << k
        bases = cref.gen_points(curve, 300 + k, n + 2)
        pp = cref.gen_scalars(c.scalar, 310 + k, n)
        ch = pasta.gen_scalars(c.scalar, 320 + k, k)
        lr = cref.gen_scalars(c.scalar, 330 + k, k)
        rr = cref.gen_scalars(c.scalar, 340 + k, k)
        x3, z = pasta.gen_scalars(c.scalar, 350 + k, 2)
        want_l, want_r, want_c = cref.ipa_rounds(curve, bases, k, pp, x3, z, cref.ints_to_bytes(ch), lr, rr, threads=2)
        out_l = np.zeros((k, 96), dtype=np.uint8)
        out_r = np.zeros((k, 96), dtype=np.uint8)
        out_c = np.zeros(32, dtype=np.uint8)
        rc = emu.emu_ipa(cref.CURVE_ID[curve], cref._p(bases), k, cref._p(pp), cref._p(cref._fe(x3)), cref._p(cref._fe(z)),
                         cref._p(cref.ints_to_bytes(ch)), cref._p(cref.ints_to_bytes([pow(u, r - 2, r) for u in ch])),
                         cref._p(lr), cref._p(rr), cb, cref._p(out_l), cref._p(out_r), cref._p(out_c))
        assert rc == 0
        assert int.from_bytes(out_c.tobytes(), "little") == want_c
        for j in range(k):
            assert cref.jac_to_affine(curve, out_l[j]).tobytes() == want_l[j].tobytes(), (k, j)
            assert cref.jac_to_affine(curve, out_r[j]).tobytes() == want_r[j].tobytes(), (k, j)


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_glv_split_bounds(emu, curve):
    """glv_decompose: k1 + k2 lambda = k (mod r) and |k1|, |k2| < 2^127 -- the bound the plan's W = ceil(128 / c) and
    the 4-limb stored halves rely on -- on random scalars and on scalars placed at the rounding boundaries of c1 / c2
    (k b / r within one unit of a half-integer), where the device's 2^384 fixed-point rounding could differ from exact."""
    import random
    import sys
    sys.path.insert(0, "tools")
    import gen_glv_constants as gg
    c = pasta.CURVES[curve]
    r = c.r
    lam, _ = gg.find_lambda_zeta(c)
    (a1, b1), (a2, b2) = gg.lattice(r, lam)
    # rigorous: |k1| <= (1/2 + eps)(a1 + a2), |k2| <= (1/2 + eps)(|b1| + b2), eps < 2^-130
    assert (a1 + a2) * 1001 // 2000 < 1 << 127 and (abs(b1) + b2) * 1001 // 2000 < 1 << 127
    rnd = random.Random(99)
    ks = [0, 1, 2, r - 1, r - 2, lam, r - lam, (r - 1) // 2, (r + 1) // 2]
    ks += [rnd.randrange(r) for _ in range(3000)]
    for b in (b2, abs(b1)):
        for _ in range(300):
            j = rnd.randrange(b)
            k0 = ((2 * j + 1) * r) // (2 * b)          # k b / r ~ j + 1/2
            ks += [(k0 + d) % r for d in (-2, -1, 0, 1, 2)]
    out = np.zeros(66, dtype=np.uint8)
    worst = 0
    for k in ks:
        emu.emu_glv(cref.CURVE_ID[curve], cref._p(cref._fe(k)), cref._p(out))
        k1 = int.from_bytes(out[:32].tobytes(), "little") * (-1 if out[64] else 1)
        k2 = int.from_bytes(out[32:64].tobytes(), "little") * (-1 if out[65] else 1)
        assert (k1 + k2 * lam - k) % r == 0
        worst = max(worst, abs(k1).bit_length(), abs(k2).bit_length())
    assert worst <= 127, worst


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_emul_field_structured_limbs(emu, field):
    """fe_sqr (dedicated squaring: 36 products + product-free reduction rounds) and fe_mul on operands whose MONTGOMERY
    limbs are all-ones / zero / single-bit patterns -- the carry edges random inputs never reach."""
    import random
    m = pasta.FIELDS[field]
    rnd = random.Random(6)
    raws = [0, 1, m - 1, m - 2, 1 << 254, (1 << 254) - 1, (1 << 254) + 1, m >> 1]
    for mask in range(256):
        v = sum(0xFFFFFFFF << (32 * i) for i in range(8) if (mask >> i) & 1)
        raws += [v % m, v & ((1 << 254) - 1)]
    for _ in range(1500):
        raws.append(sum(rnd.choice([0, 0xFFFFFFFF, 1, 0x80000000, 0x7FFFFFFF, rnd.getrandbits(32)]) << (32 * i) for i in range(8)) % m)
    rinv = pow(1 << 256, -1, m)
    for i, x in enumerate(raws):
        a = x * rinv % m                     # to_mont(a) == x
        b = raws[(i * 7 + 3) % len(raws)] * rinv % m
        assert _fop(emu, field, 4, a) == a * a % m, hex(x)
        assert _fop(emu, field, 2, a, b) == a * b % m, hex(x)


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_msm_batched_affine(emu, curve):
    """Batched-affine rounds before the XYZZ chain (msm.cuh ba_round_body / accum0_pts_body): 1-3 halving rounds, batches of
    every size (items per thread from the target, sub-batches of 8 in this build), odd list lengths, split buckets (T = 8, 16),
    and every degenerate pair -- P + P, P + (-P), identity operands, all-equal scalars -- give the oracle's point."""
    c = pasta.CURVES[curve]
    g = pasta.generator(c)

    def run(kb, pb, cb, k0, glv, rounds, target, expect_ba=True):
        emu.emu_msm_set_ba(rounds, target)
        try:
            got = _msm(emu, curve, kb, pb, cb, 0, k0, 4 if k0 else 0, glv=glv)
            if expect_ba:
                assert emu.emu_msm_last_ba() == rounds
            return got
        finally:
            emu.emu_msm_set_ba(0, 0)

    for n in (40, 97, 300):
        kb = cref.gen_scalars(c.scalar, 70 + n, n)
        pb = cref.gen_points(curve, 71 + n, n)
        want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
        for cb, k0 in ((3, 0), (2, 8), (4, 16), (5, 0)):
            for glv in (False, True):
                for rounds, target in ((1, 64), (2, 5), (3, 1), (3, 20)):
                    dense = ((2 * n if glv else n) >> (cb - 1)) >= 4      # under 4 references per bucket there is nothing to pair up
                    assert run(kb, pb, cb, k0, glv, rounds, target, expect_ba=dense) == want, (n, cb, k0, glv, rounds, target)
    # degenerate inputs: repeated / opposite / identity bases under equal scalars put P + P, P - P and O + P into the pairs
    pts = [cref.bytes_to_affine(x) for x in cref.gen_points(curve, 5, 6)]
    neg = lambda q: (q[0], c.p - q[1])  # noqa: E731
    pts2 = [g, g, neg(g), None, pts[3], pts[3], pts[4], neg(pts[4]), None, g, None, None, pts[5], neg(pts[5]), pts[5], pts[5]] * 6
    n2 = len(pts2)
    pb2 = cref.affines_to_bytes(pts2)
    for name, ks in (("equal", [5] * n2), ("ones", [1] * n2), ("rminus1", [c.r - 1] * n2), ("mix", [(i % 3) + 1 for i in range(n2)]),
                     ("random", pasta.gen_scalars(c.scalar, 4, n2))):
        kb = cref.ints_to_bytes(ks)
        want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb2))
        for cb, k0 in ((3, 0), (4, 8), (13, 0)):
            for glv in (False, True):
                for rounds, target in ((1, 4), (3, 64), (2, 9)):
                    # (sparse plans -- under 4 references per bucket -- keep the classic accumulation: nothing to pair up)
                    assert run(kb, pb2, cb, k0, glv, rounds, target, expect_ba=False) == want, (name, cb, k0, glv, rounds, target)
    # a forced odd bin capacity or item size cannot be halved in place: the plan falls back to the classic accumulation
    kb = cref.gen_scalars(c.scalar, 3, 64)
    pb = cref.gen_points(curve, 4, 64)
    want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
    emu.emu_msm_set_ba(3, 64)
    try:
        assert _msm(emu, curve, kb, pb, 3, 0, 5, 4) == want and emu.emu_msm_last_ba() == 0
    finally:
        emu.emu_msm_set_ba(0, 0)


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_msm_sort_paths(emu, curve):
    """The single-pass binned sort, its overflow fallback to the exact sort, and the exact sort alone give the same
    point; splits of oversized buckets (forced T < bin capacity) work in the binned layout too."""
    NO_BINS = 0xFFFFFFFF
    c = pasta.CURVES[curve]
    n = 300
    kb = cref.gen_scalars(c.scalar, 41, n)
    pb = cref.gen_points(curve, 42, n)
    want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
    skew = cref.ints_to_bytes([7] * n)                      # every digit of every scalar lands in the same buckets
    want_skew = cref.bytes_to_affine(cref.best_multiexp(curve, skew, pb))

    def run(kbytes, cb, cap, k0=0, gs=0, glv=False):
        emu.emu_msm_set_cap(cap)
        try:
            out = np.zeros(96, dtype=np.uint8)
            fn = emu.emu_msm_glv if glv else emu.emu_msm
            r = fn(cref.CURVE_ID[curve], cref._p(kbytes), cref._p(pb), ctypes.c_size_t(n), cb, 0, k0, gs, cref._p(out))
            assert r > 0, r
            return r, cref.bytes_to_affine(cref.jac_to_affine(curve, out))
        finally:
            emu.emu_msm_set_cap(0)

    for glv in (False, True):
        for cb in ((4, 8, 7) if glv else (3, 5, 7)):        # full and sparse (c = 7) top windows
            r, got = run(kb, cb, 0, glv=glv)                # automatic capacity: random digits never overflow
            assert r < 1000 and got == want, (glv, cb)
            r, got = run(kb, cb, NO_BINS, glv=glv)          # exact sort only
            assert r >= 1000 and got == want
            r, got = run(kb, cb, 8, 3, 4, glv=glv)          # tiny bins: overflow -> fallback (with splits)
            assert got == want
            r, got = run(skew, cb, 0, glv=glv)              # all-equal scalars: n references in one bucket
            plan = (ctypes.c_uint64 * 8)()
            emu.emu_msm_plan(ctypes.c_size_t(n), cb, 0, int(glv), 1, 0, plan)
            assert got == want_skew and (r >= 1000) == (plan[4] < n), (glv, cb, list(plan))   # 7 = low digits only: lower windows
            r, got = run(kb, cb, 512, 4, 4, glv=glv)        # roomy bins, T = 4 < sizes: splits in the binned layout
            assert r < 1000 and (r % 1000 >= 100 or cb >= 7) and got == want


# ---- K10 / K11: EC-FFT (best_fft with G = curve point), scaling, batch_normalize -------------------------------------
def _ecfft_inputs(curve, k, seed):
    n = 1 << k
    g = cref.gen_points(curve, seed, n)
    if n > 4:
        g[3] = 0                                   # an identity among the inputs
        g[n - 1] = g[1]                            # and a repeated point
    return g


@pytest.mark.parametrize("quad", [0, 1])
@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_glv_scalar_mul_projective(emu, curve, quad):
    """xyzz_scalar_mul_glv (the EC butterfly's `tw * b`) on a projective operand against the oracle's double-and-add."""
    c = pasta.CURVES[curve]
    base = cref.gen_points(curve, 91, 1)[0]
    three_b = cref.affines_to_bytes([pasta.to_affine(c, pasta.scalar_mul(c, 3, cref.bytes_to_affine(base)))])[0]
    ks = pasta.gen_scalars(c.scalar, SEED + 5, 12) + [0, 1, 2, c.r - 1, c.r - 2, (1 << 127) - 1, 1 << 127, 1 << 254, (c.r - 1) // 2]
    for kk in ks:
        out = np.zeros(64, dtype=np.uint8)
        emu.emu_glv_mul3(cref.CURVE_ID[curve], quad, cref._p(np.ascontiguousarray(base)), cref._p(cref._fe(kk)), cref._p(out))
        assert (out == cref.scalar_mul(curve, kk, three_b)).all(), hex(kk)


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_addsub_butterfly(emu, curve):
    """xyzz_addsub_q: (3a + 5b, 3a - 5b) including b = ±a multiples, identities and equal points."""
    c = pasta.CURVES[curve]
    pts = [cref.bytes_to_affine(p) for p in cref.gen_points(curve, 93, 3)]
    five_inv_three = 3 * pasta.inv(5, c.r) % c.r        # 5 * (3/5 a) = 3 a: the sum / difference degenerate
    same = pasta.to_affine(c, pasta.scalar_mul(c, five_inv_three, pts[0]))
    opp = (same[0], c.p - same[1])
    for a, b in [(pts[0], pts[1]), (pts[0], same), (pts[0], opp), (None, pts[1]), (pts[0], None), (None, None), (pts[2], pts[2])]:
        out = np.zeros(128, dtype=np.uint8)
        emu.emu_addsub35(cref.CURVE_ID[curve], cref._p(cref.affines_to_bytes([a])[0]), cref._p(cref.affines_to_bytes([b])[0]), cref._p(out))
        A = pasta.scalar_mul(c, 3, a) if a else pasta.JAC_ID
        B = pasta.scalar_mul(c, 5, b) if b else pasta.JAC_ID
        assert cref.bytes_to_affine(out[:64]) == pasta.to_affine(c, pasta.jac_add(c, A, B))
        assert cref.bytes_to_affine(out[64:]) == pasta.to_affine(c, pasta.jac_add(c, A, pasta.jac_neg(c, B)))


@pytest.mark.parametrize("quad", [0, 1])
@pytest.mark.parametrize("curve", ["pallas", "vesta"])
@pytest.mark.parametrize("k", [0, 1, 2, 4, 6])
def test_emul_ec_fft_and_params_lagrange(emu, curve, k, quad):
    c = pasta.CURVES[curve]
    r = c.r
    n = 1 << k
    g = _ecfft_inputs(curve, k, 300 + k)
    omega_inv = pasta.inv(pasta.omega_for_k(c.scalar, k), r) if k else 1
    minv = pow(pasta.inv(2, r), k, r)
    # mode 1: poly/commitment.rs:74-101 (affine g -> affine g_lagrange)
    out = np.zeros((n, 64), dtype=np.uint8)
    emu.emu_ec_fft(cref.CURVE_ID[curve], 1, quad, cref._p(g), k, cref._p(cref._fe(omega_inv)), cref._p(cref._fe(minv)), cref._p(out))
    assert (out == cref.params_lagrange(curve, g, k, omega_inv, minv, threads=4)).all()
    # mode 0: the bare network on Jacobian points, random (non-root) omega like benches/fft.rs:17, no scaling
    w = pasta.gen_scalars(c.scalar, 17 + k, 1)[0]
    jac = cref.affine_to_jacobian_bytes(g)
    o = np.zeros((n, 96), dtype=np.uint8)
    emu.emu_ec_fft(cref.CURVE_ID[curve], 0, quad, cref._p(jac), k, cref._p(cref._fe(w)), None, cref._p(o))
    want = cref.batch_normalize(curve, cref.ec_fft(curve, jac, w, k, threads=2))
    assert (cref.batch_normalize(curve, o) == want).all()
    # K11 on its own (Jacobian in, including identities) -- and through a second chunk when n > H2_NORM_CHUNK
    got = np.zeros((n, 64), dtype=np.uint8)
    emu.emu_batch_normalize(cref.CURVE_ID[curve], cref._p(o), ctypes.c_uint64(n), cref._p(got))
    assert (got == want).all()


# ---- K12: direct-sum fixed-base MSM (multiples table, signed base-256 digits, quad reduce tree) -----------------------
@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_direct_fixed_base(emu, curve):
    c = pasta.CURVES[curve]
    r = c.r
    n = 36
    bases = cref.gen_points(curve, 700, n)
    bases[5] = 0                                                   # an identity generator
    bases[9] = bases[8]                                            # a repeated one (equal partial sums meet in the tree)
    rnd = cref.gen_scalars(c.scalar, 701, n)
    edge = cref.ints_to_bytes([0, 1, 128, 129, 255, 256, 0x80, 0x7F80, r - 1, r - 2, (1 << 254), (1 << 248) * 0x40, 0x8080808080808080,
                               int("81" * 31, 16), int("80" * 31, 16), int("ff" * 31, 16)] + [7] * (n - 16))
    same = cref.ints_to_bytes([3] * n)
    for total, sets, split, name, kb in ((n, 1, 0, "random", rnd), (n, 1, 1, "random/1", rnd), (n, 1, 2, "edge/2", edge), (n, 1, 8, "edge/8", edge),
                                          (n - 3, 1, 4, "same", same[:n - 3]), (1, 1, 0, "one", rnd[:1]),
                                          (n // 2, 2, 0, "two sets", rnd)):
        out = np.zeros((sets, 64), dtype=np.uint8)
        emu.emu_msm_direct(cref.CURVE_ID[curve], cref._p(np.ascontiguousarray(kb)), cref._p(bases), ctypes.c_size_t(n), ctypes.c_size_t(total),
                           sets, split, 0, cref._p(out))
        for s_ in range(sets):
            want = cref.best_multiexp(curve, np.ascontiguousarray(kb[s_ * total:(s_ + 1) * total]), np.ascontiguousarray(bases[:total]))
            assert (out[s_] == want).all(), (name, s_)
    # Montgomery scalars (the IPA session's form)
    R = 1 << 256
    km = cref.ints_to_bytes([v * R % r for v in cref.bytes_to_ints(rnd)])
    out = np.zeros((1, 64), dtype=np.uint8)
    emu.emu_msm_direct(cref.CURVE_ID[curve], cref._p(km), cref._p(bases), ctypes.c_size_t(n), ctypes.c_size_t(n), 1, 0, 1, cref._p(out))
    assert (out[0] == cref.best_multiexp(curve, rnd, bases)).all()


# ---- K13: point compression (C::to_bytes / C::from_bytes, book/src/background/curves.md:203-240) ----------------------
@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_point_codec(emu, curve):
    c = pasta.CURVES[curve]
    pts = [cref.bytes_to_affine(p) for p in cref.gen_points(curve, 800, 40)] + [None, pasta.generator(c)]
    xy = cref.affines_to_bytes(pts)
    n = len(pts)
    enc = np.zeros((n, 32), dtype=np.uint8)
    emu.emu_compress(cref.CURVE_ID[curve], cref._p(xy), ctypes.c_uint64(n), cref._p(enc))
    assert enc.tobytes() == b"".join(pasta.compress(p) for p in pts)
    back = np.zeros((n, 64), dtype=np.uint8)
    emu.emu_decompress.restype = ctypes.c_uint32
    assert emu.emu_decompress(cref.CURVE_ID[curve], cref._p(enc), ctypes.c_uint64(n), cref._p(back)) == 0xFFFFFFFF
    assert (back == xy).all()
    # the other sign gives the negated point
    flipped = enc.copy()
    flipped[:40, 31] ^= 0x80
    emu.emu_decompress(cref.CURVE_ID[curve], cref._p(flipped), ctypes.c_uint64(40), cref._p(back))
    assert [cref.bytes_to_affine(b) for b in back[:40]] == [(p[0], c.p - p[1]) for p in pts[:40]]
    # invalid encodings: x^3 + 5 not a square, x >= p, x = 0 with the sign bit -- reported by first index, decoded as identity
    nonres = next(x for x in range(2, 200) if pasta.fe_sqrt(c.base, (x ** 3 + 5) % c.p) is None)
    for bad_val in (nonres, c.p, c.p + 1, (1 << 255) - 1, 1 << 255):
        batch = enc[:6].copy()
        batch[4] = np.frombuffer(bad_val.to_bytes(32, "little"), dtype=np.uint8)
        with pytest.raises(ValueError):
            pasta.decompress(c, batch[4].tobytes())
        out = np.ones((6, 64), dtype=np.uint8)
        assert emu.emu_decompress(cref.CURVE_ID[curve], cref._p(batch), ctypes.c_uint64(6), cref._p(out)) == 4
        assert not out[4].any() and (out[:4] == xy[:4]).all() and (out[5] == xy[5]).all()


# ---- K14: eval_polynomial / compute_inner_product / kate_division as chunk trees --------------------------------------
@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 1024, 1025, 2500])
def test_emul_polyops(emu, field, n):
    m = pasta.FIELDS[field]
    batch = 3
    a = [pasta.gen_scalars(field, 900 + b, n) for b in range(batch)]
    c = [pasta.gen_scalars(field, 910 + b, n) for b in range(batch)]
    a[2] = [0] * n if n > 1 else a[2]
    pts = [pasta.gen_scalars(field, 920, 1)[0], 0, 1]
    ab = np.concatenate([cref.ints_to_bytes(v) for v in a])
    cb = np.concatenate([cref.ints_to_bytes(v) for v in c])
    pb = cref.ints_to_bytes(pts)
    out = np.zeros((batch, 32), dtype=np.uint8)
    emu.emu_polyops(cref.FIELD_ID[field], 0, cref._p(ab), None, batch, ctypes.c_uint64(n), cref._p(pb), cref._p(out))
    assert cref.bytes_to_ints(out) == [pasta.eval_polynomial(field, a[b], pts[b]) for b in range(batch)]
    emu.emu_polyops(cref.FIELD_ID[field], 1, cref._p(ab), cref._p(cb), batch, ctypes.c_uint64(n), None, cref._p(out))
    assert cref.bytes_to_ints(out) == [pasta.compute_inner_product(m, a[b], c[b]) for b in range(batch)]
    if n >= 2:
        q = np.zeros((batch, n - 1, 32), dtype=np.uint8)
        emu.emu_polyops(cref.FIELD_ID[field], 2, cref._p(ab), cref._p(cb), batch, ctypes.c_uint64(n), cref._p(pb), cref._p(q))
        for b in range(batch):
            want = pasta.kate_division(field, a[b], pts[b])
            assert cref.bytes_to_ints(q[b]) == want, b
            # the defining property: q(X) (X - b) + a(b) == a(X), checked at a random point
            z = pasta.gen_scalars(field, 930 + b, 1)[0]
            assert (pasta.eval_polynomial(field, want, z) * (z - pts[b]) + pasta.eval_polynomial(field, a[b], pts[b])) % m == pasta.eval_polynomial(field, a[b], z)


# ---- K15: Evaluator::evaluate over an Ast (poly/evaluator.rs:129-228) as one postfix program ----------------------------
@pytest.mark.parametrize("basis,j,k", [("extended", 3, 4), ("extended", 5, 3), ("lagrange", 2, 5), ("lagrange", 2, 0)])
def test_emul_ast_evaluator(emu, basis, j, k):
    from halo2_b200.evaluator import AstLeaf, compile_ast
    field = "fp"
    d = pasta.EvaluationDomain(field, j, k, pasta.zeta_candidates(field)[0])
    log_n = k if basis == "lagrange" else d.extended_k
    n = 1 << log_n
    polys = [pasta.gen_scalars(field, 1000 + i, n) for i in range(4)]
    y, theta = pasta.gen_scalars(field, 1010, 2)
    ast = _quotient_like_ast([AstLeaf(i) for i in range(4)], y, theta)
    want = pasta.ast_evaluate(d, basis, _ast_tuple(ast), polys)
    stride = 1 if basis == "lagrange" else 1 << (d.extended_k - d.k)
    code, consts = compile_ast(ast, d.m, stride)
    pb = np.concatenate([cref.ints_to_bytes(p) for p in polys])
    cb = cref.ints_to_bytes(consts)
    omega = d.omega if basis == "lagrange" else d.extended_omega
    lin = 1 if basis == "lagrange" else d.g_coset
    out = np.zeros((n, 32), dtype=np.uint8)
    emu.emu_ast_eval(cref.FIELD_ID[field], cref._p(pb), 4, log_n, code.ctypes.data_as(ctypes.c_void_p), code.shape[0], cref._p(cb), len(consts),
                     cref._p(cref._fe(omega)), cref._p(cref._fe(lin)), cref._p(out))
    assert cref.bytes_to_ints(out) == want
    # the reference's own regression cases (evaluator.rs:625-660): a bare ConstantTerm / LinearTerm of zero
    from halo2_b200.evaluator import Ast
    for node in (Ast.constant_term(0), Ast.linear_term(0), Ast.linear_term(9)):
        code, consts = compile_ast(node, d.m, stride)
        emu.emu_ast_eval(cref.FIELD_ID[field], cref._p(pb), 4, log_n, code.ctypes.data_as(ctypes.c_void_p), code.shape[0], cref._p(cref.ints_to_bytes(consts)),
                         len(consts), cref._p(cref._fe(omega)), cref._p(cref._fe(lin)), cref._p(out))
        assert cref.bytes_to_ints(out) == pasta.ast_evaluate(d, basis, _ast_tuple(node), polys)


# ---- the permutation argument's grand product: batch_invert and the running product (plonk/permutation/prover.rs:98-157) ----
@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("n", [1, 2, 16, 17, 32, 33, 1024, 1057])
def test_emul_grand_product(emu, field, n):
    m = pasta.FIELDS[field]
    a = pasta.gen_scalars(field, 1100 + n, n)
    if n > 3:
        a[1] = 0                    # batch_invert leaves zeros alone; a zero factor zeroes the rest of the running product
    ab = cref.ints_to_bytes(a)
    out = np.zeros((n, 32), dtype=np.uint8)
    emu.emu_grand_product(cref.FIELD_ID[field], 0, cref._p(ab), ctypes.c_uint64(n), None, cref._p(out))
    assert cref.bytes_to_ints(out) == [pasta.inv(x, m) if x else 0 for x in a]
    init = pasta.gen_scalars(field, 1101, 1)[0]
    for vals in (a, [x or 5 for x in a]):
        emu.emu_grand_product(cref.FIELD_ID[field], 1, cref._p(cref.ints_to_bytes(vals)), ctypes.c_uint64(n), cref._p(cref._fe(init)), cref._p(out))
        z = [init]
        for row in range(1, n):      # permutation/prover.rs:150-156
            z.append(z[row - 1] * vals[row - 1] % m)
        assert cref.bytes_to_ints(out) == z


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_emul_hash_to_curve(emu, curve):
    """h2c.cuh on the host: BLAKE2b core vs hashlib, expand_message_xmd / SWU / isogeny vs the oracle (itself pinned on the
    reference's golden commitments, tests/test_oracle_golden.py), generator messages of Params::new."""
    import hashlib
    import random
    rnd = random.Random(5)
    for ln in (0, 1, 5, 63, 64, 127, 128, 129, 180, 255, 256, 257, 1000):
        d = bytes(rnd.getrandbits(8) for _ in range(ln))
        out = (ctypes.c_uint8 * 64)()
        emu.emu_blake2b(d, ln, out)
        assert bytes(out) == hashlib.blake2b(d).digest()
    c = pasta.CURVES[curve]
    n = 12
    out = np.zeros((n, 64), dtype=np.uint8)
    assert emu.emu_hash_to_curve(cref.CURVE_ID[curve], b"Halo2-Parameters", None, 0, 1, ctypes.c_uint64(3), ctypes.c_uint64(n), cref._p(out)) == 0
    g, w, u = pasta.params_generators(c, 4)
    assert [cref.bytes_to_affine(o) for o in out] == g[3:3 + n]
    msgs = np.frombuffer(b"\x01\x02", dtype=np.uint8).copy()
    out = np.zeros((2, 64), dtype=np.uint8)
    assert emu.emu_hash_to_curve(cref.CURVE_ID[curve], b"Halo2-Parameters", cref._p(msgs), 1, 0, ctypes.c_uint64(0), ctypes.c_uint64(2), cref._p(out)) == 0
    assert [cref.bytes_to_affine(o) for o in out] == [w, u]
    h = pasta.hash_to_curve(c, "z.cash:test")
    for ml in (0, 44, 84, 85, 200):
        ms = [bytes(rnd.getrandbits(8) for _ in range(ml)) for _ in range(2)]
        buf = np.frombuffer(b"".join(ms) or b"\0", dtype=np.uint8).copy()
        out = np.zeros((2, 64), dtype=np.uint8)
        assert emu.emu_hash_to_curve(cref.CURVE_ID[curve], b"z.cash:test", cref._p(buf), ml, 0, ctypes.c_uint64(0), ctypes.c_uint64(2), cref._p(out)) == 0
        assert [cref.bytes_to_affine(o) for o in out] == [h(m) for m in ms]
    assert emu.emu_hash_to_curve(cref.CURVE_ID[curve], b"p" * 250, None, 0, 1, ctypes.c_uint64(0), ctypes.c_uint64(1), cref._p(out)) == 1


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_emul_lookup_permute(emu, field):
    """The lookup permutation's kernel bodies (lookup.cuh) run serially == the oracle's permute_expression_pair
    (plonk/lookup/prover.rs:563-647): sizes around the powers of two of the bitonic network, one / few / all-distinct table
    values, small integers (the high limbs of the keys tie), rows past usable_rows untouched, a missing value fails."""
    import random
    m = pasta.FIELDS[field]
    rnd = random.Random(9)
    for n, u, distinct, small in ((4, 1, 1, True), (4, 2, 2, False), (8, 5, 3, True), (20, 16, 16, False), (40, 33, 7, True), (70, 64, 1, False),
                                  (300, 257, 100, True), (300, 290, 290, False)):
        pool = [rnd.randrange(1 << 10) if small else rnd.randrange(m) for _ in range(distinct)]
        tab = (pool + [rnd.choice(pool) for _ in range(u)])[:u]
        rnd.shuffle(tab)
        inp = [rnd.choice(tab) for _ in range(u)]
        tail = [rnd.randrange(m) for _ in range(n - u)]
        marker = [7000 + i for i in range(n)]
        oa, ot = cref.ints_to_bytes(marker), cref.ints_to_bytes(marker)
        rc = emu.emu_lookup_permute(cref.FIELD_ID[field], cref._p(cref.ints_to_bytes(inp + tail)), cref._p(cref.ints_to_bytes(tab + tail)),
                                    ctypes.c_size_t(n), ctypes.c_size_t(u), cref._p(oa), cref._p(ot))
        assert rc == 0
        want_a, want_s = pasta.permute_expression_pair(field, inp, tab, u)
        ga, gs = cref.bytes_to_ints(oa), cref.bytes_to_ints(ot)
        assert ga[:u] == want_a and gs[:u] == want_s, (n, u, distinct)
        assert ga[u:] == marker[u:] and gs[u:] == marker[u:]
        bad = list(inp)
        bad[u // 2] = (max(tab) + 1) % m
        if bad[u // 2] not in set(tab):
            rc = emu.emu_lookup_permute(cref.FIELD_ID[field], cref._p(cref.ints_to_bytes(bad + tail)), cref._p(cref.ints_to_bytes(tab + tail)),
                                        ctypes.c_size_t(n), ctypes.c_size_t(u), cref._p(oa), cref._p(ot))
            assert rc == 1
