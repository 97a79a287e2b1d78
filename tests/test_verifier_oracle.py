"""CPU checks of the verifier's side of the path (no GPU): the oracle's restatement of MSM / verify_proof / Guard /
compute_s / compute_b (oracle/pasta.py, oracle/halo2_oracle.c) against the reference's own tests --
`msm_arithmetic` (poly/commitment/msm.rs:179-219) and `test_opening_proof` (poly/commitment.rs:304-379) mirrored step by
step -- the device bodies of verifier.cuh on the host emulation, and the proof-shaped replay verified end to end."""
import ctypes

import numpy as np
import pytest

from oracle import cref, pasta
from tests import prover_replay as R
from tests.kernel_emul import build as emul_build

SEED = 0x48414C4F32


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emul_build.build())


def _closed_form(m, u, init):
    k = len(u)
    out = []
    for i in range(1 << k):
        v = init % m
        for j in range(k):
            if (i >> j) & 1:
                v = v * u[k - 1 - j] % m
        out.append(v)
    return out


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_compute_s_every_form(emu, field):
    """The doubling loop of verifier.rs:156-171 (Python and C restatements) = init * prod of the challenges the set bits of
    the index select = the device body (one thread per four elements), with and without accumulation."""
    m = pasta.FIELDS[field]
    for k in list(range(1, 10)) + [11]:
        u = pasta.gen_scalars(field, SEED + k, k)
        if k == 4:
            u[1] = 0                                          # a zero challenge wipes half of the vector
        if k == 5:
            u[0], u[4] = 1, m - 1
        init = pasta.gen_scalars(field, SEED + 100 + k, 1)[0]
        want = pasta.compute_s(m, u, init)
        assert want == _closed_form(m, u, init)
        assert cref.bytes_to_ints(cref.compute_s(field, u, init)) == want
        base = pasta.gen_scalars(field, SEED + 200 + k, 1 << k)
        for accumulate in (0, 1):
            buf = cref.ints_to_bytes(base)
            emu.emu_compute_s(cref.FIELD_ID[field], cref._p(cref.ints_to_bytes(u)), k, cref._p(cref._fe(init)), accumulate, cref._p(buf))
            got = cref.bytes_to_ints(buf)
            assert got == ([(a + b) % m for a, b in zip(base, want)] if accumulate else want), (k, accumulate)
    with pytest.raises(AssertionError):
        pasta.compute_s(m, [], 1)                             # assert!(!u.is_empty())
    with pytest.raises(AssertionError):
        cref.compute_s(field, [], 1)


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_compute_b_is_g_at_x(field):
    """compute_b (verifier.rs:145-153) is g(X) = sum_i s_i X^i at x, s = compute_s(u, 1)."""
    m = pasta.FIELDS[field]
    for k in (1, 2, 5, 8):
        u = pasta.gen_scalars(field, SEED + 300 + k, k)
        x = pasta.gen_scalars(field, SEED + 400 + k, 1)[0]
        assert pasta.compute_b(m, x, u) == pasta.eval_polynomial_mod(m, pasta.compute_s(m, u, 1), x)
    from halo2_b200.verifier import compute_b          # the host mirror's copy (pure host arithmetic, no GPU involved)
    assert compute_b(x, u, m) == pasta.compute_b(m, x, u)


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_emul_scale_add(emu, field):
    m = pasta.FIELDS[field]
    for n in (1, 5, 256, 777):
        d = pasta.gen_scalars(field, SEED + n, n)
        s = pasta.gen_scalars(field, SEED + n + 1, n)
        a, b = pasta.gen_scalars(field, SEED + n + 2, 2)
        for fa, fb, src in ((a, b, s), (1, 1, s), (a, 0, None), (0, 1, s), (m - 1, m - 1, s)):
            buf = cref.ints_to_bytes(d)
            emu.emu_scale_add(cref.FIELD_ID[field], cref._p(buf), cref._p(cref._fe(fa)), cref._p(cref.ints_to_bytes(src)) if src else None,
                              cref._p(cref._fe(fb)), ctypes.c_uint64(n))
            want = [(fa * x + (fb * y if src else 0)) % m for x, y in zip(d, src or d)]
            assert cref.bytes_to_ints(buf) == want


def test_msm_arithmetic_oracle():
    """poly/commitment/msm.rs:179-219, statement by statement, on the oracle's MSM."""
    c = pasta.PALLAS
    r = c.r
    base = (c.p - 1, 2)                                       # EpAffine::from_xy(-Fp::one(), Fp::from(2))
    assert pasta.on_curve(c, base)
    base_viol = pasta.to_affine(c, pasta.jac_double(c, pasta.to_jac(base)))
    neg = lambda pt: (pt[0], (-pt[1]) % c.p)
    pts = pasta.gen_points(c, SEED, 18)
    new = lambda: pasta.MSM(c, pts[:16], pts[16], pts[17])    # Params::new(4): the generators play no part in this test
    a = new()
    a.append_term(1, base)
    assert not a.clone().eval()
    a.append_term(1, base)
    assert not a.clone().eval()
    a.append_term(r - 1, base_viol)
    assert a.clone().eval()
    b = a.clone()
    a.append_term(4, neg(base))
    assert not a.clone().eval()
    a.append_term(2, base_viol)
    assert a.clone().eval()
    a.scale(3)
    a.add_msm(b)
    assert a.clone().eval()
    cc = new()
    cc.append_term(2, base)
    cc.append_term(1, neg(base_viol))
    assert cc.clone().eval()
    a.add_msm(cc)
    assert a.eval()
    # beyond the reference's test: g_scalars / w / u terms cancel against explicit terms on the same points
    d = new()
    sc = pasta.gen_scalars("fq", SEED + 7, 16)
    d.add_to_g_scalars(sc)
    d.add_constant_term(5)
    d.add_to_w_scalar(9)
    d.add_to_u_scalar(11)
    assert not d.clone().eval()
    total = pasta.naive_msm(c, [(sc[0] + 5) % r] + sc[1:] + [9, 11], pts)
    d.append_term(r - 1, pasta.to_affine(c, total))
    assert d.clone().eval()
    d.scale(12345)
    assert d.eval()
    with pytest.raises(AssertionError):
        new().add_to_g_scalars(sc[:15])                        # assert_eq!(scalars.len(), params.n), msm.rs:100


@pytest.mark.parametrize("curve,k", [("pallas", 4), ("vesta", 3)])
def test_opening_proof_oracle(curve, k):
    """poly/commitment.rs:304-379 (`test_opening_proof`, K = 6 there) through the oracle: commit, create_proof, read the
    proof back, verify_proof, the prover's and the verifier's next challenge agree, and both uses of the Guard evaluate to
    the identity; a wrong claimed value does not."""
    c = pasta.CURVES[curve]
    r = c.r
    n = 1 << k
    g, w, u = pasta.params_generators(c, k)                   # Params::new(k): hash_to_curve generators
    px = list(range(n))                                       # *a = Fq::from(i as u64)
    blind, s_blind = pasta.gen_scalars(c.scalar, SEED + 1, 2)
    s_poly = pasta.gen_scalars(c.scalar, SEED + 2, n)
    l_rand, r_rand = pasta.gen_scalars(c.scalar, SEED + 3, k), pasta.gen_scalars(c.scalar, SEED + 4, k)
    p = pasta.to_affine(c, pasta.best_multiexp(c, px + [blind], g + [w]))
    W = R._WriteT(r)
    W.write_point(p)
    x = W.squeeze_challenge()
    v = pasta.eval_polynomial_mod(r, px, x)
    W.write_scalar(v)
    pasta.ipa_create_proof(c, g, w, u, W, px, blind, x, s_poly, s_blind, l_rand, r_rand)
    ch_prover = W.squeeze_challenge()
    proof = bytes(W.T.proof)
    assert len(proof) == 32 * (1 + 1 + 1 + 2 * k + 2)

    def read_side(data):
        T = R.Blake2bRead(data, lambda b32: cref.affines_to_bytes([pasta.decompress(c, b32)])[0], r)
        return T, R._TupleTranscript(T, cref)

    T, TT = read_side(proof)
    assert TT.read_point() == p
    assert TT.squeeze_challenge() == x
    assert TT.read_scalar() == v
    msm = pasta.MSM(c, g, w, u)
    msm.append_term(1, p)
    guard = pasta.ipa_verify_proof(k, msm, TT, x, v)
    assert TT.squeeze_challenge() == ch_prover
    assert T.pos == len(proof)
    g_pt = guard.compute_g()
    keep = pasta.Guard(guard.msm.clone(), guard.neg_c, guard.u)
    assert guard.use_challenges().eval()
    msm_g, acc = keep.use_g(g_pt)
    assert msm_g.eval() and acc[0] == g_pt and acc[1] == guard.u
    # the same proof does not open to another value, nor at another point
    for bad_x, bad_v in ((x, (v + 1) % r), ((x + 1) % r, v)):
        T, TT = read_side(proof)
        TT.read_point(), TT.squeeze_challenge(), TT.read_scalar()
        msm = pasta.MSM(c, g, w, u)
        msm.append_term(1, p)
        assert not pasta.ipa_verify_proof(k, msm, TT, bad_x, bad_v).use_challenges().eval()
    # a truncated proof: Error::OpeningError / SamplingError
    for cut in (32 * 3 + 16, len(proof) - 32, len(proof) - 1):
        T, TT = read_side(proof[:cut])
        TT.read_point(), TT.squeeze_challenge(), TT.read_scalar()
        msm = pasta.MSM(c, g, w, u)
        msm.append_term(1, p)
        with pytest.raises(pasta.VerifyError):
            pasta.ipa_verify_proof(k, msm, TT, x, v)


def _replay_setup(k, real_params=False):
    n = 1 << k
    c = pasta.VESTA
    if real_params:
        P = pasta.Params.new(c, k)
        g, w, u = cref.affines_to_bytes(P.g), cref.affines_to_bytes([P.w]), cref.affines_to_bytes([P.u])
        gl = cref.affines_to_bytes(P.g_lagrange)
    else:
        pts = cref.gen_points("vesta", SEED + 1, n + 2)
        g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
        P = pasta.Params.from_generators(c, k, [cref.bytes_to_affine(x) for x in g], cref.bytes_to_affine(w[0]), cref.bytes_to_affine(u[0]))
        gl = cref.affines_to_bytes(P.g_lagrange)
    return g, gl, w, u


@pytest.mark.parametrize("k,real_params", [(3, False), (5, True), (6, False)])
def test_replay_proof_verifies(k, real_params):
    """The proof-shaped replay's bytes (tests/prover_replay.run, CPU arm) are accepted by the restated verifier -- the
    multiopen MSM from the proof's commitments and evaluations, the opening, the final multiexp over all generators -- and
    a flip anywhere in the proof is rejected."""
    g, gl, w, u = _replay_setup(k, real_params)
    inp = R.replay_inputs(cref, k, SEED + k)
    omega = pasta.omega_for_k("fp", k)
    cpu = R.CpuArm(cref, pasta, k, g, gl, w, u, threads=4)
    proof = R.run(cpu, inp, k, omega)
    assert len(proof) == 32 * (11 + 2 * k) + 32 * 18
    ver = R.CpuVerifierArm(cref, pasta, k, g, gl, w, u, 4)
    assert R.verify(ver, proof, k, omega)
    assert ver.hot_s > 0
    # one flipped bit per region of the proof: an advice commitment, the permutation product's, an h piece, an evaluation that is
    # opened, f's commitment, a q evaluation, the s commitment, an L_j, an R_j, c, f
    npts = 9
    off = {"advice": 0, "z": 32 * 3, "h": 32 * 6, "eval adv@x": 32 * npts, "eval z@xw": 32 * (npts + 7), "eval rnd@x": 32 * (npts + 13),
           "f commitment": 32 * (npts + 14), "q eval": 32 * (npts + 15), "s commitment": 32 * (npts + 17), "L_0": 32 * (npts + 18),
           "R_last": 32 * (npts + 18 + 2 * k - 1), "c": len(proof) - 64, "f": len(proof) - 32}
    for name, o in off.items():
        bad = bytearray(proof)
        bad[o + 3] ^= 0x10
        assert not R.verify(ver, bytes(bad), k, omega), name
    # evaluations that are in the proof but not opened (z at x and at x omega^-1) only enter the transcript: still rejected,
    # because every later challenge changes
    bad = bytearray(proof)
    bad[32 * (npts + 6) + 1] ^= 1
    assert not R.verify(ver, bytes(bad), k, omega)
    assert not R.verify(ver, proof[:-32], k, omega)
    # another witness gives another proof, which verifies too
    proof2 = R.run(cpu, R.replay_inputs(cref, k, SEED + k + 1), k, omega)
    assert proof2 != proof and R.verify(ver, proof2, k, omega)
