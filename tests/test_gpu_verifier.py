"""GPU tests of the verifier's side of the path: compute_s / scale_add on resident polynomials (verifier.cuh) against the
oracle, the host mirror of MSM / verify_proof / Guard (halo2_b200.verifier) against the reference's own tests
(`msm_arithmetic`, poly/commitment/msm.rs:179-219; `test_opening_proof`, poly/commitment.rs:304-379), and the prove ->
verify round trip of the proof-shaped replay: what the engine proves, the engine and the restated reference verifier accept,
and nothing else."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests import prover_replay as R  # noqa: E402

SEED = 0x48414C4F32


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


def _seeded_params(eng, curve, k):
    n = 1 << k
    pts = cref.gen_points(curve, SEED + 1, n + 2)
    g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    return eng.Params(curve, k, g, eng.lagrange_generators(curve, k, g), w, u=u), g, w, u


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_compute_s_and_scale_add_device(eng, field):
    from halo2_b200 import lib as L
    lib = L.init()
    m = pasta.FIELDS[field]
    for k in (1, 2, 3, 7, 10, 14, 17):
        n = 1 << k
        u = cref.bytes_to_ints(cref.gen_scalars(field, SEED + k, k))
        if k == 7:
            u[2] = 0
        init = cref.bytes_to_ints(cref.gen_scalars(field, SEED + 100 + k, 1))[0]
        want = cref.compute_s(field, u, init)
        ub = cref.ints_to_bytes(u)
        p = eng.ResidentPoly(field, n)
        L.check(lib.h2_poly_compute_s(p._h, L.ptr(ub), ctypes.c_uint32(k), L.ptr(L.fe_bytes(init)), 0, L.REPR_CANONICAL))
        assert np.array_equal(p.download(), want), k
        # accumulate on top of a random vector, twice
        base = cref.gen_scalars(field, SEED + 200 + k, n)
        p.upload(base)
        L.check(lib.h2_poly_compute_s(p._h, L.ptr(ub), ctypes.c_uint32(k), L.ptr(L.fe_bytes(init)), 1, L.REPR_CANONICAL))
        L.check(lib.h2_poly_compute_s(p._h, L.ptr(ub), ctypes.c_uint32(k), L.ptr(L.fe_bytes(1)), 1, L.REPR_CANONICAL))
        if k <= 10:
            s1 = pasta.compute_s(m, u, 1)
            exp = [(b + init * s + s) % m for b, s in zip(cref.bytes_to_ints(base), s1)]
            assert cref.bytes_to_ints(p.download()) == exp, k
        # dst = a dst + b src, and the scale-only form
        if k <= 10:
            q = eng.ResidentPoly(field, n, want)
            a, b = cref.bytes_to_ints(cref.gen_scalars(field, SEED + 300 + k, 2))
            cur = cref.bytes_to_ints(p.download())
            L.check(lib.h2_poly_scale_add(p._h, L.ptr(L.fe_bytes(a)), q._h, L.ptr(L.fe_bytes(b)), ctypes.c_size_t(n), L.REPR_CANONICAL))
            exp = [(a * x + b * y) % m for x, y in zip(cur, cref.bytes_to_ints(want))]
            assert cref.bytes_to_ints(p.download()) == exp
            L.check(lib.h2_poly_scale_add(p._h, L.ptr(L.fe_bytes(b)), ctypes.c_uint64(0), None, ctypes.c_size_t(n - 1), L.REPR_CANONICAL))
            exp = [x * b % m for x in exp[:-1]] + exp[-1:]
            assert cref.bytes_to_ints(p.download()) == exp
            assert lib.h2_poly_scale_add(p._h, L.ptr(L.fe_bytes(a)), p._h, L.ptr(L.fe_bytes(b)), ctypes.c_size_t(n), L.REPR_CANONICAL) != 0
            q.close()
        p.close()
    # errors: no challenges (assert!(!u.is_empty())), a polynomial that is too short, an unknown handle
    p = eng.ResidentPoly(field, 7)
    one = L.fe_bytes(1)
    assert lib.h2_poly_compute_s(p._h, L.ptr(one), ctypes.c_uint32(0), L.ptr(one), 0, L.REPR_CANONICAL) != 0
    assert lib.h2_poly_compute_s(p._h, L.ptr(cref.ints_to_bytes([1, 2, 3])), ctypes.c_uint32(3), L.ptr(one), 0, L.REPR_CANONICAL) != 0
    assert lib.h2_poly_compute_s(ctypes.c_uint64(1 << 60), L.ptr(one), ctypes.c_uint32(1), L.ptr(one), 0, L.REPR_CANONICAL) != 0
    p.close()


def test_msm_arithmetic_device(eng):
    """poly/commitment/msm.rs:179-219, statement by statement, on halo2_b200.verifier.MSM (Pallas, Params of k = 4)."""
    c = pasta.PALLAS
    r = c.r
    prm, g, w, u = _seeded_params(eng, "pallas", 4)
    base_t = (c.p - 1, 2)
    viol_t = pasta.to_affine(c, pasta.jac_double(c, pasta.to_jac(base_t)))
    B = lambda pt: cref.affines_to_bytes([pt])[0]
    neg = lambda pt: (pt[0], (-pt[1]) % c.p)
    base, base_viol = B(base_t), B(viol_t)
    new = lambda: eng.MSM(prm)
    try:
        a = new()
        a.append_term(1, base)
        assert not a.clone().eval()
        a.append_term(1, base)
        assert not a.clone().eval()
        a.append_term(r - 1, base_viol)
        assert a.clone().eval()
        b = a.clone()
        a.append_term(4, B(neg(base_t)))
        assert not a.clone().eval()
        a.append_term(2, base_viol)
        assert a.clone().eval()
        a.scale(3)
        a.add_msm(b)
        assert a.clone().eval()
        cc = new()
        cc.append_term(2, base)
        cc.append_term(1, B(neg(viol_t)))
        assert cc.clone().eval()
        a.add_msm(cc)
        assert a.eval()
        assert new().eval()                                       # the empty MSM is the identity
        a.append_term(5, np.zeros(64, dtype=np.uint8))            # the identity is skipped (msm.rs:66)
        assert a.eval()
        # g_scalars / w / u against the oracle's MSM through the same operations; the group element itself is compared
        gt, wt, ut = [cref.bytes_to_affine(x) for x in g], cref.bytes_to_affine(w[0]), cref.bytes_to_affine(u[0])
        d, od = new(), pasta.MSM(c, gt, wt, ut)
        sc = cref.gen_scalars("fq", SEED + 7, 16)
        sci = cref.bytes_to_ints(sc)
        for mm, arg in ((d, sc), (od, sci)):
            mm.add_to_g_scalars(arg)
            mm.add_constant_term(5)
            mm.add_to_w_scalar(9)
            mm.add_to_u_scalar(11)
        d.append_term(77, base)
        od.append_term(77, base_t)
        same = lambda: cref.bytes_to_affine(cref.jac_to_affine("pallas", d.evaluate())) == pasta.to_affine(c, pasta.best_multiexp(c, *od.terms()))
        assert same() and not d.clone().eval()
        e, oe = d.clone(), od.clone()
        d.scale(12345)
        od.scale(12345)
        assert same()
        d.add_msm(e)
        od.add_msm(oe)
        assert same()
        d.add_to_g_scalars(eng.ResidentPoly("fq", 16, sc))
        od.add_to_g_scalars(sci)
        assert same()
        d.scale_add_msm(424242, e)                                # BatchVerifier's accumulate_msm, fused
        od.scale(424242)
        od.add_msm(oe)
        assert same()
        us = cref.bytes_to_ints(cref.gen_scalars("fq", SEED + 8, 4))
        d.add_compute_s(us, 31337)
        od.add_to_g_scalars(pasta.compute_s(r, us, 31337))
        assert same()
        assert cref.bytes_to_ints(d.g_scalars.download()) == od.g_scalars
        total = pasta.to_affine(c, pasta.best_multiexp(c, *od.terms()))
        d.append_term(r - 1, B(total))
        assert d.eval()
        with pytest.raises(AssertionError):
            new().add_to_g_scalars(sc[:15])                       # assert_eq!(scalars.len(), params.n), msm.rs:100
    finally:
        prm.close()


def _gpu_create_proof(eng, prm, T, px, blind, x3, s_poly, s_blind, l_rand, r_rand, r):
    """commitment::create_proof (poly/commitment/prover.rs:36-151) through the engine: commit, the device round loop."""
    s = list(s_poly)
    s[0] = (s[0] - pasta.eval_polynomial_mod(r, s, x3)) % r
    T.write_point(eng.batch_normalize(prm.commit(cref.ints_to_bytes(s), eng.Blind(s_blind)).reshape(1, 96), prm.curve)[0])
    xi = T.squeeze_challenge()
    z = T.squeeze_challenge()
    pp = [(a * xi + b) % r for a, b in zip(s, px)]
    pp[0] = (pp[0] - pasta.eval_polynomial_mod(r, pp, x3)) % r
    f = (s_blind * xi + blind) % r
    us = []

    def challenge(j, l_xy, r_xy):
        T.write_point(l_xy)
        T.write_point(r_xy)
        us.append(T.squeeze_challenge())
        return us[-1]

    _, _, c_val = prm.ipa_rounds_transcript(cref.ints_to_bytes(pp), x3, z, challenge, l_rand, r_rand)
    for j, uj in enumerate(us):
        f = (f + l_rand[j] * pow(uj, -1, r) + r_rand[j] * uj) % r
    T.write_scalar(c_val)
    T.write_scalar(f)


@pytest.mark.parametrize("curve,k", [("pallas", 6), ("vesta", 4), ("vesta", 1)])
def test_opening_proof_device(eng, curve, k):
    """poly/commitment.rs:304-379 (`test_opening_proof`, K = 6, EpAffine) through the engine end to end: Params::new on the device,
    write / read of the parameters, commit, create_proof, verify_proof, both uses of the Guard -- and, at the small sizes, the same
    proof bytes as the oracle's create_proof."""
    import io
    c = pasta.CURVES[curve]
    r = c.r
    n = 1 << k
    prm0 = eng.Params.new(curve, k)
    buf = io.BytesIO()
    prm0.write(buf)
    prm0.close()
    prm = eng.Params.read(curve, io.BytesIO(buf.getvalue()))
    try:
        px = list(range(n))
        blind, s_blind = cref.bytes_to_ints(cref.gen_scalars(c.scalar, SEED + 1, 2))
        s_poly = cref.bytes_to_ints(cref.gen_scalars(c.scalar, SEED + 2, n))
        l_rand = cref.bytes_to_ints(cref.gen_scalars(c.scalar, SEED + 3, k))
        r_rand = cref.bytes_to_ints(cref.gen_scalars(c.scalar, SEED + 4, k))
        p = eng.batch_normalize(prm.commit(cref.ints_to_bytes(px), eng.Blind(blind)).reshape(1, 96), curve)[0]
        W = R.Blake2bTranscript(r)
        W.write_point(p)
        x = W.squeeze_challenge()
        v = pasta.eval_polynomial_mod(r, px, x)
        W.write_scalar(v)
        _gpu_create_proof(eng, prm, W, px, blind, x, s_poly, s_blind, l_rand, r_rand, r)
        ch_prover = W.squeeze_challenge()
        proof = bytes(W.proof)
        if k <= 4:                                                # the oracle's prover writes the same bytes
            OW = R._WriteT(r)
            gt = [cref.bytes_to_affine(x_) for x_ in prm.g]
            OW.write_point(cref.bytes_to_affine(p))
            assert OW.squeeze_challenge() == x
            OW.write_scalar(v)
            pasta.ipa_create_proof(c, gt, cref.bytes_to_affine(prm.w[0]), cref.bytes_to_affine(prm.u[0]), OW, px, blind, x, s_poly, s_blind,
                                   l_rand, r_rand)
            assert bytes(OW.T.proof) == proof

        def reader(data):
            return R.Blake2bRead(data, lambda b32: eng.decompress_points(np.frombuffer(b32, dtype=np.uint8).reshape(1, 32), curve)[0], r)

        T = reader(proof)
        assert np.array_equal(T.read_point(), p)
        assert T.squeeze_challenge() == x
        assert T.read_scalar() == v
        msm = eng.MSM(prm)
        msm.append_term(1, p)
        guard = eng.verify_proof(prm, msm, T, x, v)
        assert T.squeeze_challenge() == ch_prover and T.pos == len(proof)
        g_pt = guard.compute_g()
        s1 = cref.compute_s(c.scalar, guard.u, 1)
        assert cref.bytes_to_affine(g_pt) == cref.bytes_to_affine(cref.best_multiexp(curve, s1, prm.g))
        keep = guard.clone()
        assert guard.use_challenges().eval()
        msm_g, acc = keep.use_g(g_pt)
        assert msm_g.eval() and np.array_equal(acc[0], g_pt) and acc[1] == guard.u
        if k > 1:
            keep2 = eng.Guard(msm_g.clone(), keep.neg_c, keep.u)
            m2, _ = keep2.use_g(prm.g[1])                         # a G that is not <s, g>: [-c] G no longer cancels
            assert not m2.eval()
        for bad_x, bad_v in ((x, (v + 1) % r), ((x + 1) % r, v)):
            T = reader(proof)
            T.read_point(), T.squeeze_challenge(), T.read_scalar()
            msm = eng.MSM(prm)
            msm.append_term(1, p)
            assert not eng.verify_proof(prm, msm, T, bad_x, bad_v).use_challenges().eval()
        for cut in (32 * 3 + 16, len(proof) - 32):
            T = reader(proof[:cut])
            T.read_point(), T.squeeze_challenge(), T.read_scalar()
            msm = eng.MSM(prm)
            msm.append_term(1, p)
            with pytest.raises(eng.VerifyError):
                eng.verify_proof(prm, msm, T, x, v)
    finally:
        prm.close()


@pytest.mark.parametrize("k,real_params", [(5, True), (10, False), (14, False)])
def test_replay_prove_verify_round_trip(eng, k, real_params):
    """The engine's proof (tests/prover_replay.run, GPU arm) is accepted by the engine's verifier AND by the restated reference
    verifier (C multiexp); the C restatement's proof is accepted by the engine; flipped bits are rejected by both."""
    n = 1 << k
    if real_params:
        prm = eng.Params.new("vesta", k)
        g, gl, w, u = prm.g, prm.g_lagrange, prm.w, prm.u
        prm.close()
    else:
        pts = cref.gen_points("vesta", SEED + 1, n + 2)
        g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
        gl = eng.lagrange_generators("vesta", k, g)
    inp = R.replay_inputs(cref, k, SEED + k)
    omega = pasta.omega_for_k("fp", k)
    gpu = R.GpuArm(eng, k, g, gl, w, u)
    try:
        proof = R.run(gpu, inp, k, omega)
        gpu.free()
        gv = R.GpuVerifierArm(eng, k, g, gl, w, u, params=gpu.params)
        cv = R.CpuVerifierArm(cref, pasta, k, g, gl, w, u, 8)
        assert R.verify(gv, proof, k, omega)
        assert R.verify(gv, proof, k, omega)                      # again: pooled buffers, replayed graphs
        assert R.verify(cv, proof, k, omega)
        if k <= 10:
            cpu = R.CpuArm(cref, pasta, k, g, gl, w, u, threads=8)
            proof_c = R.run(cpu, R.replay_inputs(cref, k, SEED + k + 1), k, omega)
            assert proof_c != proof and R.verify(gv, proof_c, k, omega)
        npts = 9
        off = {"advice": 0, "h": 32 * 6, "eval adv@x": 32 * npts, "eval z@xw": 32 * (npts + 7), "f commitment": 32 * (npts + 14),
               "q eval": 32 * (npts + 15), "s commitment": 32 * (npts + 17), "L_0": 32 * (npts + 18), "R_last": 32 * (npts + 18 + 2 * k - 1),
               "c": len(proof) - 64, "f": len(proof) - 32}
        for name, o in off.items():
            bad = bytearray(proof)
            bad[o + 3] ^= 0x10
            assert not R.verify(gv, bytes(bad), k, omega), name
            if name in ("advice", "q eval", "c"):
                assert not R.verify(cv, bytes(bad), k, omega), name
        assert not R.verify(gv, proof[:-32], k, omega)
    finally:
        gpu.close()


def test_batch_verifier_accumulation(eng):
    """BatchVerifier::finalize's shape (plonk/verifier/batch.rs:83-131): every proof's MSM (after use_challenges) scaled by a
    random factor and added into one accumulator, ONE eval for the batch; a single bad proof fails the batch."""
    k = 8
    n = 1 << k
    c = pasta.VESTA
    r = c.r
    prm, g, w, u = _seeded_params(eng, "vesta", k)
    try:
        def one_proof(seed, lie=0):
            px = cref.bytes_to_ints(cref.gen_scalars("fp", seed, n))
            blind, s_blind = cref.bytes_to_ints(cref.gen_scalars("fp", seed + 1, 2))
            s_poly = cref.bytes_to_ints(cref.gen_scalars("fp", seed + 2, n))
            l_rand = cref.bytes_to_ints(cref.gen_scalars("fp", seed + 3, k))
            r_rand = cref.bytes_to_ints(cref.gen_scalars("fp", seed + 4, k))
            p = eng.batch_normalize(prm.commit(cref.ints_to_bytes(px), eng.Blind(blind)).reshape(1, 96), "vesta")[0]
            W = R.Blake2bTranscript(r)
            W.write_point(p)
            x = W.squeeze_challenge()
            v = pasta.eval_polynomial_mod(r, px, x)
            W.write_scalar(v)
            _gpu_create_proof(eng, prm, W, px, blind, x, s_poly, s_blind, l_rand, r_rand, r)
            T = R.Blake2bRead(bytes(W.proof), lambda b32: eng.decompress_points(np.frombuffer(b32, dtype=np.uint8).reshape(1, 32), "vesta")[0], r)
            T.read_point(), T.squeeze_challenge(), T.read_scalar()
            msm = eng.MSM(prm)
            msm.append_term(1, p)
            return eng.verify_proof(prm, msm, T, x, (v + lie) % r).use_challenges()

        factors = cref.bytes_to_ints(cref.gen_scalars("fp", SEED + 99, 3))
        for lie_at in (None, 1):
            acc = eng.MSM(prm)                                    # params.empty_msm()
            for i in range(3):
                m_i = one_proof(SEED + 1000 * (i + 1), lie=1 if lie_at == i else 0)
                acc.scale_add_msm(factors[i], m_i)
                m_i.close()
            assert acc.eval() == (lie_at is None)
            acc.close()
    finally:
        prm.close()
