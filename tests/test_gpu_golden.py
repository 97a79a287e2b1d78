"""GPU tests whose EXPECTED VALUES ARE LITERALS FROM THE REFERENCE TREE: the 19 golden commitments of the `plonk_api`
verifying key (/root/reference/halo2_proofs/tests/plonk_api.rs:958-982, carried in tests/golden/reference_goldens.json).
Each is `Params::<EqAffine>::new(5).commit_lagrange(column, Blind::default())`, so reproducing them on the device pins, on
reference-held vectors and through the C ABI, the whole chain: hash_to_curve (h2c.cuh) -> EC-iFFT at G = curve point
(best_fft through FftGroup, ecfft.cuh) -> batch_normalize -> best_multiexp / commit_lagrange (msm.cuh)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests.plonk_api_circuit import golden_columns  # noqa: E402


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


def _affine(curve, xyz):
    return cref.bytes_to_affine(cref.jac_to_affine(curve, xyz))


def test_params_new_k5_reproduces_reference_golden_commitments(eng, goldens):
    cols, want = golden_columns(goldens)
    prm = eng.Params.new("vesta", 5)
    assert cref.bytes_to_affine(prm.w[0]) == want[0]                 # fixed_commitments[0] = 1 * w
    # one by one through h2_msm_registered (fixed-base path over the resident g_lagrange || w table)
    for col, pt in zip(cols, want):
        assert _affine("vesta", prm.commit_lagrange(cref.ints_to_bytes(col), eng.Blind())) == pt
    # all 19 in one batched pass + device batch_normalize (the shape of keygen's loops, plonk/keygen.rs:233-236)
    aff = prm.commit_many_affine([cref.ints_to_bytes(c) for c in cols], [eng.Blind()] * len(cols), lagrange=True)
    assert [cref.bytes_to_affine(a) for a in aff] == want
    # and through the one-shot variable-base best_multiexp (arithmetic.rs:143-180) over g_lagrange ++ [w] (commitment.rs:140-149)
    bases = np.concatenate([prm.g_lagrange, prm.w])
    for col, pt in list(zip(cols, want))[::3]:
        out = eng.best_multiexp(cref.ints_to_bytes(list(col) + [1]), bases, "vesta")
        assert _affine("vesta", out) == pt
    # without the precomputed window table (bucket path over resident bases)
    prm2 = eng.Params("vesta", 5, prm.g, prm.g_lagrange, prm.w, prm.u, precompute=False)
    for col, pt in list(zip(cols, want))[1::4]:
        assert _affine("vesta", prm2.commit_lagrange(cref.ints_to_bytes(col), eng.Blind())) == pt


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_hash_to_curve_vs_oracle(eng, curve):
    c = pasta.CURVES[curve]
    h_dev = eng.hash_to_curve(curve, "z.cash:test")                  # benches/hashtocurve.rs:15,18
    h_orc = pasta.hash_to_curve(c, "z.cash:test")
    import random
    rnd = random.Random(11)
    for ml in (0, 1, 5, 43, 44, 45, 83, 84, 85, 127, 128, 129, 200, 300):   # block-boundary lengths of both BLAKE2b inputs
        msgs = [bytes(rnd.getrandbits(8) for _ in range(ml)) for _ in range(3)]
        out = h_dev(msgs)
        assert [cref.bytes_to_affine(o) for o in out] == [h_orc(m) for m in msgs]
    assert cref.bytes_to_affine(h_dev(b"Trans rights now!")) == h_orc(b"Trans rights now!")
    # other domain prefixes (the DST changes length: different padding of every BLAKE2b input)
    for dom in ("Halo2-Parameters", "z.cash:SinsemillaS", "x"):
        assert cref.bytes_to_affine(eng.hash_to_curve(curve, dom)(b"\x07\x00\x00\x00")) == pasta.hash_to_curve(c, dom)(b"\x07\x00\x00\x00")
    with pytest.raises(eng.H2Error):
        eng.hash_to_curve(curve, "p" * 250)(b"")


@pytest.mark.parametrize("curve,k", [("pallas", 6), ("vesta", 3), ("pallas", 0)])
def test_params_new_vs_oracle(eng, curve, k):
    c = pasta.CURVES[curve]
    po = pasta.Params.new(c, k)
    prm = eng.Params.new(curve, k)
    assert [cref.bytes_to_affine(x) for x in prm.g] == po.g
    assert [cref.bytes_to_affine(x) for x in prm.g_lagrange] == po.g_lagrange
    assert cref.bytes_to_affine(prm.w[0]) == po.w and cref.bytes_to_affine(prm.u[0]) == po.u
    poly = pasta.gen_scalars(c.scalar, 77 + k, 1 << k)
    assert _affine(curve, prm.commit(cref.ints_to_bytes(poly), eng.Blind(5))) == pasta.to_affine(c, po.commit(poly, 5))
