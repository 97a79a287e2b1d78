"""Pins the oracle against every known-answer datum the reference's tests hold for the path
(SURVEY.md section 8(c)).  CPU only."""
import numpy as np
import pytest

from oracle import cref, pasta
from tests.plonk_api_circuit import FP_ZETA_INDEX, golden_columns
from tests.poseidon_kat import permute


def test_moduli_and_omegas(goldens):
    vk5 = goldens["vk_plonk_api_k5"]
    vk11 = goldens["vk_lookup_range_check_k11"]
    # EqAffine = Vesta: base field Fq, scalar field Fp (tests/plonk_api.rs:591-592)
    for vk in (vk5, vk11):
        assert int(vk["base_modulus"], 16) == pasta.Q_MOD
        assert int(vk["scalar_modulus"], 16) == pasta.P_MOD
    # domain.rs:58-78 with ROOT_OF_UNITY = 5^T reproduces the pinned omegas
    assert pasta.omega_for_k("fp", 5) == int(vk5["omega"], 16)
    assert pasta.omega_for_k("fp", 11) == int(vk11["omega"], 16)
    d = pasta.EvaluationDomain("fp", 4, 5)  # plonk_api circuit: extended_k = 7
    assert d.omega == int(vk5["omega"], 16)
    for f in ("fp", "fq"):
        m = pasta.FIELDS[f]
        w = pasta.root_of_unity(f)
        assert pow(w, 1 << 32, m) == 1 and pow(w, 1 << 31, m) == m - 1
        for z in pasta.zeta_candidates(f):
            assert z != 1 and pow(z, 3, m) == 1


def test_golden_commitments_on_vesta(goldens):
    """commit_lagrange outputs pinned by the reference lie on y^2 = x^3 + 5 over Fq."""
    n = 0
    for key in ("vk_plonk_api_k5", "vk_lookup_range_check_k11"):
        vk = goldens[key]
        for x, y in vk["fixed_commitments"] + vk["permutation_commitments"]:
            pt = (int(x, 16), int(y, 16))
            assert pasta.on_curve(pasta.VESTA, pt)
            assert not pasta.on_curve(pasta.PALLAS, pt)
            assert cref.on_curve("vesta", cref.affines_to_bytes([pt])[0])
            n += 1
    assert n >= 19
    # the all-zero column's commitment (= params.w, blind 1) recurs at k=5 and k=11
    assert goldens["vk_plonk_api_k5"]["fixed_commitments"][0] in goldens["vk_lookup_range_check_k11"]["fixed_commitments"]


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_poseidon_permutation_kat_python(goldens, field):
    m = pasta.FIELDS[field]
    g = goldens["poseidon"][field]
    rc = [int(x, 16) for x in g["round_constants"]]
    mds = [int(x, 16) for x in g["mds"]]
    assert len(g["permute"]) == 11
    for tv in g["permute"]:
        out = permute([int(x, 16) for x in tv["initial_state"]], rc, mds,
                      lambda a, b: (a + b) % m, lambda a, b: a * b % m, lambda a: pow(a, 5, m))
        assert out == [int(x, 16) for x in tv["final_state"]]


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_poseidon_permutation_kat_c(goldens, field):
    g = goldens["poseidon"][field]
    rc = [int(x, 16) for x in g["round_constants"]]
    mds = [int(x, 16) for x in g["mds"]]
    for tv in g["permute"][:4]:
        out = permute([int(x, 16) for x in tv["initial_state"]], rc, mds,
                      lambda a, b: cref.field_op(field, "add", a, b),
                      lambda a, b: cref.field_op(field, "mul", a, b),
                      lambda a: cref.field_op(field, "pow5", a))
        assert out == [int(x, 16) for x in tv["final_state"]]


def test_generator_order():
    """(-1, 2) (poly/commitment/msm.rs:181) has prime order r on both curves."""
    for c in (pasta.PALLAS, pasta.VESTA):
        g = pasta.generator(c)
        assert pasta.on_curve(c, g)
        assert pasta.to_affine(c, pasta.scalar_mul(c, c.r - 1, g)) == (g[0], c.p - g[1])
        gb = cref.affines_to_bytes([g])[0]
        assert cref.bytes_to_affine(cref.scalar_mul(c.name, c.r - 1, gb)) == (g[0], c.p - g[1])


def test_point_compression_on_golden_commitments(goldens):
    """C::to_bytes / C::from_bytes as specified in book/src/background/curves.md:203-240, on the reference's golden
    commitments (tests/plonk_api.rs:958-982, circuit_data/vk_lookup_range_check.rdata): decompressing the encoding of (x, y)
    must find exactly the golden y -- pins the square root and the sign rule of the oracle; the device path is checked against
    the oracle (tests/test_kernel_emul.py::test_emul_point_codec, tests/test_gpu_parity.py::test_point_codec_and_params_io)."""
    c = pasta.VESTA
    n = 0
    for vk in (goldens["vk_plonk_api_k5"], goldens["vk_lookup_range_check_k11"]):
        for x, y in vk["fixed_commitments"] + vk["permutation_commitments"]:
            x, y = int(x, 16), int(y, 16)
            enc = pasta.compress((x, y))
            assert len(enc) == 32 and enc[31] >> 7 == (y & 1)
            assert pasta.decompress(c, enc) == (x, y)
            flipped = bytearray(enc)
            flipped[31] ^= 0x80
            assert pasta.decompress(c, bytes(flipped)) == (x, c.p - y)
            n += 1
    assert n == 26
    assert pasta.compress(None) == b"\0" * 32 and pasta.decompress(c, b"\0" * 32) is None
    # Params::{write, read} (poly/commitment.rs:168-205) round trip on a tiny synthetic parameter set
    po = pasta.Params(c, 2)
    data = pasta.params_to_bytes(po.k, po.g, po.g_lagrange, po.w, po.u)
    assert len(data) == 4 + 32 * (2 * 4 + 2) and data[:4] == (2).to_bytes(4, "little")
    assert pasta.params_from_bytes(c, data) == (2, po.g, po.g_lagrange, po.w, po.u)
    with pytest.raises(ValueError):
        pasta.params_from_bytes(c, data[:-1])


# ------------------------------------------------------------------------------------------------------------------
# hash_to_curve -> Params::new -> commit_lagrange, pinned on the reference's golden commitments.
# Every one of the 19 points at tests/plonk_api.rs:958-982 is commit_lagrange(column, Blind::default()) over
# Params::<EqAffine>::new(5): fixed_commitments[0] is an all-zero column, i.e. the point w = hash_to_curve(..)(&[1]);
# the others are MSMs over g_lagrange = 2^-5 * EC-iFFT(32 hashed generators) -- so they pin hash_to_curve, the EC-FFT
# (best_fft at G = curve point) and best_multiexp together.  tests/plonk_api_circuit.py rebuilds the columns.
# ------------------------------------------------------------------------------------------------------------------


def test_hash_to_curve_w_is_golden(goldens):
    vk = goldens["vk_plonk_api_k5"]
    h = pasta.hash_to_curve(pasta.VESTA, "Halo2-Parameters")
    w = h(b"\x01")
    assert w == (int(vk["fixed_commitments"][0][0], 16), int(vk["fixed_commitments"][0][1], 16))
    # the same point is the all-zero column's commitment of the k = 11 verifying key
    assert [hex(w[0]), hex(w[1])] in [[hex(int(a, 16)), hex(int(b, 16))]
                                      for a, b in goldens["vk_lookup_range_check_k11"]["fixed_commitments"]]
    # the iso curves and the isogeny are what Velu's formulas say, on both curves; outputs lie on the curve
    for c in (pasta.PALLAS, pasta.VESTA):
        k = pasta.iso_constants(c)
        assert k["B"] == 1265 and (k["A"] * k["A"] * k["A"] * 4 + 27 * 1265 * 1265) % c.p != 0
        hc = pasta.hash_to_curve(c, "z.cash:test")          # benches/hashtocurve.rs:15,18
        for msg in (b"", b"Trans rights now!", bytes(range(200))):
            pt = hc(msg)
            assert pt is not None and pasta.on_curve(c, pt)
            assert pasta.jac_eq(c, pasta.scalar_mul(c, c.r, pt), pasta.JAC_ID)


def test_golden_commitments_python_oracle(goldens):
    """All 19 golden commitments through oracle/pasta.py: hash_to_curve, ec_fft, best_multiexp."""
    cols, want = golden_columns(goldens)
    prm = pasta.Params.new(pasta.VESTA, 5)
    for col, pt in zip(cols, want):
        assert pasta.to_affine(pasta.VESTA, prm.commit_lagrange(col, 1)) == pt
    # the other ZETA would not do: the lookup-table column contains a = 2834758237 * ZETA
    from tests import plonk_api_circuit as circ
    other = circ.fixed_columns(pasta.P_MOD, pasta.zeta_candidates("fp")[1 - FP_ZETA_INDEX])[6]
    assert pasta.to_affine(pasta.VESTA, prm.commit_lagrange(other, 1)) != want[6]


def test_golden_commitments_c_oracle(goldens):
    """The same 19 points through oracle/halo2_oracle.c (the timed CPU baseline): its EC-FFT from the hashed generators
    and its threaded best_multiexp."""
    cols, want = golden_columns(goldens)
    c = pasta.VESTA
    g, w, _u = pasta.params_generators(c, 5)
    r = c.r
    alpha_inv = pasta.inv(pasta.omega_for_k(c.scalar, 5), r)
    gl = cref.params_lagrange("vesta", cref.affines_to_bytes(g), 5, alpha_inv, pow(pasta.inv(2, r), 5, r))
    bases = np.concatenate([gl, cref.affines_to_bytes([w])])
    for col, pt in zip(cols, want):
        out = cref.best_multiexp("vesta", cref.ints_to_bytes(list(col) + [1]), bases)
        assert cref.bytes_to_affine(out) == pt          # cref.best_multiexp returns the affine canonical bytes
