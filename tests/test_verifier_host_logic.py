"""CPU checks of the HOST LOGIC of halo2_b200.verifier (the mirror of poly/commitment/msm.rs and verifier.rs) with the C ABI
replaced by tests/fake_engine.py -- the same flows tests/test_gpu_verifier.py runs against the CUDA library.  What this
covers is the mirror's own code (term merging, clone / scale / add_msm bookkeeping, which entry point gets what, the
transcript order of verify_proof); the device code is covered by the host emulation and the GPU tests."""
import numpy as np
import pytest

from oracle import cref, pasta
from tests import fake_engine, prover_replay as R

SEED = 0x48414C4F32


@pytest.fixture()
def eng():
    import halo2_b200
    with fake_engine.installed() as fake:
        halo2_b200._fake = fake
        yield halo2_b200
        del halo2_b200._fake


def _params(eng, curve, k, g=None, w=None, u=None):
    n = 1 << k
    if g is None:
        pts = cref.gen_points(curve, SEED + 1, n + 2)
        g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    return eng.Params(curve, k, g, g, w, u=u), g, w, u          # g_lagrange plays no part on the verifier's side


def test_no_fake_outside_the_fixture():
    from halo2_b200 import lib as L
    assert not isinstance(L._lib, fake_engine.FakeLib)


def test_msm_arithmetic_host_logic(eng):
    """poly/commitment/msm.rs:179-219 on halo2_b200.verifier.MSM, then g_scalars / w / u against the oracle's MSM."""
    c = pasta.PALLAS
    r = c.r
    prm, g, w, u = _params(eng, "pallas", 4)
    base_t = (c.p - 1, 2)
    viol_t = pasta.to_affine(c, pasta.jac_double(c, pasta.to_jac(base_t)))
    B = lambda pt: cref.affines_to_bytes([pt])[0]
    neg = lambda pt: (pt[0], (-pt[1]) % c.p)
    base, base_viol = B(base_t), B(viol_t)
    new = lambda: eng.MSM(prm)
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
    assert new().eval()
    a.append_term(5, np.zeros(64, dtype=np.uint8))
    assert a.eval()
    with pytest.raises(AssertionError):
        a.append_term(1, B((base_t[0], 3)))                       # same x, a y that is neither ours nor its negation (msm.rs:47, :79)
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
    before = list(eng._fake.calls)
    d.scale_add_msm(424242, e)
    assert eng._fake.calls[len(before):] == ["h2_poly_scale_add"]  # ONE pass over the vector for scale + add_msm
    assert e.g_scalars is not None and d.g_scalars is not None
    od.scale(424242)
    od.add_msm(oe)
    assert same()
    us = cref.bytes_to_ints(cref.gen_scalars("fq", SEED + 8, 4))
    d.add_compute_s(us, 31337)
    od.add_to_g_scalars(pasta.compute_s(r, us, 31337))
    assert same()
    assert cref.bytes_to_ints(d.g_scalars.download()) == od.g_scalars
    d.append_term(r - 1, B(pasta.to_affine(c, pasta.best_multiexp(c, *od.terms()))))
    assert d.eval()
    # an MSM with only w / u / other terms never touches the generator table
    f = new()
    f.add_to_w_scalar(3)
    f.add_to_u_scalar(4)
    f.append_term(r - 1, B(pasta.to_affine(c, pasta.best_multiexp(c, [3, 4], [wt, ut]))))
    before = len(eng._fake.calls)
    assert f.eval() and eng._fake.calls[before:] == ["h2_msm"]
    with pytest.raises(AssertionError):
        new().add_to_g_scalars(sc[:15])
    with pytest.raises(eng.H2Error):
        eng.MSM(eng.Params("pallas", 4, g, g, w))                 # no u: eval could not be formed


@pytest.mark.parametrize("curve,k", [("pallas", 4), ("vesta", 1)])
def test_opening_proof_host_logic(eng, curve, k):
    """`test_opening_proof` (poly/commitment.rs:304-379) with the oracle as the prover and halo2_b200.verifier as the verifier."""
    c = pasta.CURVES[curve]
    r = c.r
    n = 1 << k
    gt, wt, ut = pasta.params_generators(c, k)
    prm, g, w, u = _params(eng, curve, k, cref.affines_to_bytes(gt), cref.affines_to_bytes([wt]), cref.affines_to_bytes([ut]))
    px = list(range(n))
    blind, s_blind = pasta.gen_scalars(c.scalar, SEED + 1, 2)
    s_poly = pasta.gen_scalars(c.scalar, SEED + 2, n)
    l_rand, r_rand = pasta.gen_scalars(c.scalar, SEED + 3, k), pasta.gen_scalars(c.scalar, SEED + 4, k)
    p_t = pasta.to_affine(c, pasta.best_multiexp(c, px + [blind], gt + [wt]))
    W = R._WriteT(r)
    W.write_point(p_t)
    x = W.squeeze_challenge()
    v = pasta.eval_polynomial_mod(r, px, x)
    W.write_scalar(v)
    pasta.ipa_create_proof(c, gt, wt, ut, W, px, blind, x, s_poly, s_blind, l_rand, r_rand)
    ch_prover = W.squeeze_challenge()
    proof = bytes(W.T.proof)
    p = cref.affines_to_bytes([p_t])[0]

    def reader(data):
        return R.Blake2bRead(data, lambda b32: eng.decompress_points(np.frombuffer(b32, dtype=np.uint8).reshape(1, 32), curve)[0], r)

    T = reader(proof)
    assert np.array_equal(T.read_point(), p) and T.squeeze_challenge() == x and T.read_scalar() == v
    msm = eng.MSM(prm)
    msm.append_term(1, p)
    guard = eng.verify_proof(prm, msm, T, x, v)
    assert T.squeeze_challenge() == ch_prover and T.pos == len(proof)
    # the same Guard as the oracle's verifier builds
    OT = R._TupleTranscript(reader(proof), cref)
    OT.read_point(), OT.squeeze_challenge(), OT.read_scalar()
    om = pasta.MSM(c, gt, wt, ut)
    om.append_term(1, p_t)
    og = pasta.ipa_verify_proof(k, om, OT, x, v)
    assert (guard.neg_c, guard.u) == (og.neg_c, og.u) and (guard.msm.w_scalar, guard.msm.u_scalar) == (og.msm.w_scalar, og.msm.u_scalar)
    assert {int.from_bytes(kx, "little"): (s, int.from_bytes(y, "little")) for kx, (s, y) in guard.msm.other.items()} == og.msm.other
    g_pt = guard.compute_g()
    assert cref.bytes_to_affine(g_pt) == og.compute_g()
    keep = guard.clone()
    assert guard.use_challenges().eval()
    msm_g, acc = keep.use_g(g_pt)
    assert msm_g.eval() and np.array_equal(acc[0], g_pt) and acc[1] == guard.u
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


def test_replay_verify_host_logic(eng):
    """tests/prover_replay.verify with the GPU verifier arm's code path (batched decompression, resident g_scalars, fused
    compute_s) on the C restatement's proof; flips are rejected; a batch of proofs accumulates into one eval."""
    k = 5
    n = 1 << k
    pts = cref.gen_points("vesta", SEED + 1, n + 2)
    g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    P = pasta.Params.from_generators(pasta.VESTA, k, [cref.bytes_to_affine(x) for x in g], cref.bytes_to_affine(w[0]), cref.bytes_to_affine(u[0]))
    gl = cref.affines_to_bytes(P.g_lagrange)
    omega = pasta.omega_for_k("fp", k)
    cpu = R.CpuArm(cref, pasta, k, g, gl, w, u, threads=4)
    proof = R.run(cpu, R.replay_inputs(cref, k, SEED + k), k, omega)
    gv = R.GpuVerifierArm(eng, k, g, gl, w, u)
    before = len(eng._fake.calls)
    assert R.verify(gv, proof, k, omega)
    calls = eng._fake.calls[before:]
    assert calls.count("h2_points_decompress") == 1 and calls.count("h2_poly_compute_s") == 1
    assert calls.count("h2_msm_registered_polys") == 1 and calls.count("h2_msm") == 1 and calls.count("h2_point_sum") == 1
    for o in (0, 32 * 9, 32 * (9 + 14), 32 * (9 + 15), 32 * (9 + 18), len(proof) - 64, len(proof) - 32):
        bad = bytearray(proof)
        bad[o + 3] ^= 0x10
        assert not R.verify(gv, bytes(bad), k, omega), o
    assert not R.verify(gv, proof[:-32], k, omega)
    gv.close()
