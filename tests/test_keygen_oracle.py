"""CPU checks of key generation (halo2_b200/keygen.py, csrc/keygen.cuh) against a restatement of the reference
(plonk/permutation/keygen.rs:24-211, plonk/keygen.rs:240-336, poly.rs:135-180):

- the mirror's Assembly, fed the copy sequences of the plonk_api and benchmark circuits, gives the mappings whose sigma
  polynomials the test circuits pin;
- the device bodies of the sigma kernel and its power tables, on the host emulation, equal the reference's serial
  omega-power loop and deltaomega gather;
- keygen_pk / keygen_vk / batch_invert_assigned_resident run their calls, in their order, over an ABI stand-in (the
  sigma kernel on the emulation), and reproduce the test prover's proving-key values."""
import ctypes
import random

import numpy as np
import pytest

from oracle import cref, pasta
from tests import bench_circuit as BC
from tests import fake_engine
from tests import plonk_api_circuit as circ
from tests.bench_circuit import _bench_setup, bench_copies
from tests.fake_engine import KEYGEN_CHUNK
from tests.keygen_cases import oracle_assembly, oracle_copy, oracle_sigma, random_mapping
from tests.kernel_emul import build as emul_build
from tests.plonk_api_circuit import ZETA, plonk_api_copies
from tests.plonk_prover import prover_pk_dict
from tests.plonk_verifier import scalar_delta


# ---- the reference, restated -------------------------------------------------------------------------------------------
def oracle_batch_invert_assigned(numerators, denominators, m: int):
    """batch_invert_assigned (poly.rs:135-180): numerator * denominator^-1, with BatchInvert leaving a zero denominator 0."""
    return [[a * (pow(d, -1, m) if d % m else 0) % m for a, d in zip(nums, dens)] for nums, dens in zip(numerators, denominators)]


# ---- 1. the mirror's Assembly ------------------------------------------------------------------------------------------
def test_assembly_plonk_api_circuit():
    import halo2_b200 as h2
    m = pasta.P_MOD
    omega, delta = pasta.omega_for_k("fp", circ.K), scalar_delta(m)
    asm = h2.Assembly(circ.N, 12)
    ref = oracle_assembly(circ.N, 12)
    for cp in plonk_api_copies():
        asm.copy(*cp)
        oracle_copy(ref, *cp)
    mapping = asm.mapping
    assert mapping.shape == (12, circ.N, 2) and mapping.dtype == np.uint32
    assert [[tuple(int(x) for x in e) for e in col] for col in mapping] == ref[0]
    assert oracle_sigma(mapping, circ.N, omega, delta, m) == circ.permutation_columns(m, omega, delta)


@pytest.mark.parametrize("k", [5, 6, 7, 8, 9, 10])
def test_assembly_bench_circuit(k):
    import halo2_b200 as h2
    m = pasta.P_MOD
    n = 1 << k
    omega, delta = pasta.omega_for_k("fp", k), scalar_delta(m)
    assert omega == h2.EvaluationDomain("fp", BC.DEGREE, k, ZETA).omega
    asm = h2.Assembly(n, 3)
    for cp in bench_copies(k):
        asm.copy(*cp)
    _, sigma, _ = BC.columns(k, m, omega, delta, 7)
    assert oracle_sigma(asm.mapping, n, omega, delta, m) == sigma


def test_assembly_out_of_range_copies_raise():
    import halo2_b200 as h2
    asm = h2.Assembly(8, 3)
    asm.copy(0, 7, 2, 0)
    before = asm.mapping.copy()
    for bad in ((0, 8, 1, 0), (0, 0, 1, 8), (0, -1, 1, 0)):
        with pytest.raises(IndexError):
            asm.copy(*bad)
    for bad in ((3, 0, 1, 0), (0, 0, -1, 0)):
        with pytest.raises(ValueError):
            asm.copy(*bad)
    assert (asm.mapping == before).all()
    ref = oracle_assembly(8, 3)
    with pytest.raises(IndexError):
        oracle_copy(ref, 0, 8, 1, 0)


# ---- 2. the device bodies on the host emulation ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emul_build.build())


def emu_sigma(emu, field: str, mapping: np.ndarray, k: int, omega: int, delta: int, piece: int = KEYGEN_CHUNK):
    cols = mapping.shape[0]
    mp = np.ascontiguousarray(mapping, dtype=np.uint32)
    out = np.zeros((cols << k, 32), dtype=np.uint8)
    rc = emu.emu_permutation_sigma(cref.FIELD_ID[field], mp.ctypes.data_as(ctypes.c_void_p), cols, k, cref._p(cref.ints_to_bytes([omega])),
                                   cref._p(cref.ints_to_bytes([delta])), ctypes.c_uint64(piece), cref._p(out))
    return rc, [cref.bytes_to_ints(out[i << k:(i + 1) << k]) for i in range(cols)]


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_emul_tables(emu, field):
    m = pasta.FIELDS[field]
    emu.emu_keygen_tables.restype = ctypes.c_uint64
    for k in range(0, 13):
        omega, delta = pasta.omega_for_k(field, k), scalar_delta(m)
        h = emu.emu_keygen_split(k)
        assert h == (k + 1) // 2 and h + (k - h) == k and (k % 2 == 0 or h == k - h + 1)
        for cols in (1, 3, 12):
            out = np.zeros(((1 << h) + (1 << (k - h)) + cols, 32), dtype=np.uint8)
            got = emu.emu_keygen_tables(cref.FIELD_ID[field], cref._p(cref.ints_to_bytes([omega])), cref._p(cref.ints_to_bytes([delta])), k, cols,
                                        cref._p(out))
            assert got == out.shape[0]
            want = ([pow(omega, t, m) for t in range(1 << h)] + [pow(omega, t << h, m) for t in range(1 << (k - h))]
                    + [pow(delta, c, m) for c in range(cols)])
            assert cref.bytes_to_ints(out) == want


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_emul_sigma_matches_oracle(emu, field):
    m = pasta.FIELDS[field]
    rng = np.random.default_rng(19)
    delta = scalar_delta(m)
    for k in range(1, 13):
        n = 1 << k
        omega = pasta.omega_for_k(field, k)
        for cols in (1, 3, 12):
            mp = random_mapping(rng, cols, n)
            rc, got = emu_sigma(emu, field, mp, k, omega, delta)
            assert rc == 0
            assert got == oracle_sigma(mp, n, omega, delta, m), (k, cols)
        # the identity mapping: sigma_i[j] = delta^i omega^j
        ident = np.stack(np.meshgrid(np.arange(3), np.arange(n), indexing="ij"), axis=-1).astype(np.uint32)
        rc, got = emu_sigma(emu, field, ident, k, omega, delta)
        assert rc == 0 and got == [[pow(delta, i, m) * pow(omega, j, m) % m for j in range(n)] for i in range(3)]
    # several launches per column (the device's pieces of 2^22 rows, here of 5), and a delta / omega that are not the domain's
    k, n = 6, 64
    w, d = pasta.gen_scalars(field, 3, 2)
    mp = random_mapping(rng, 3, n)
    rc, got = emu_sigma(emu, field, mp, k, w, d, piece=5)
    assert rc == 0 and got == oracle_sigma(mp, n, w, d, m)


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_emul_sigma_rejects_out_of_range_entries(emu, field):
    m = pasta.FIELDS[field]
    k, n, cols = 4, 16, 3
    omega = pasta.omega_for_k(field, k)
    rng = np.random.default_rng(5)
    for where, bad in (((0, 0), (cols, 0)), ((2, 15), (0, n)), ((1, 7), (0xFFFFFFFF, 0xFFFFFFFF))):
        mp = random_mapping(rng, cols, n)
        mp[where] = bad
        rc, _ = emu_sigma(emu, field, mp, k, omega, scalar_delta(m))
        assert rc == 1
    rc, _ = emu_sigma(emu, field, random_mapping(rng, cols, n), k, omega, scalar_delta(m))
    assert rc == 0


# ---- 3. keygen.py over an ABI stand-in ---------------------------------------------------------------------------------
def test_keygen_pk_reproduces_the_test_provers_key():
    """keygen_pk's resident key at k = 5 holds exactly the values create_proof_engine's own keygen part computes, and a proof
    made with it is the proof made with the host-built sigma."""
    import halo2_b200 as h2
    from tests import multiopen_cases as MC
    from tests import plonk_prover as PP
    from tests import plonk_verifier as PV
    from tests import prover_replay as R
    k = 5
    c, m, gens, fixed, sigma, adv, copies = _bench_setup(k)
    n = 1 << k
    delta = scalar_delta(m)
    with fake_engine.installed() as fake:
        prm = h2.Params("vesta", k, *gens[:3], u=gens[3])
        D = h2.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
        asm = h2.Assembly(n, 3)
        for cp in copies:
            asm.copy(*cp)
        fc, pc = h2.keygen_vk(prm, D, fixed, asm, delta)
        assert fake.calls.count("h2_poly_permutation_sigma") == 1 and fake.calls.count("h2_msm_registered_polys_affine") == 1
        assert not fake.polys
        A = cref.bytes_to_affine
        cl = lambda v: pasta.to_affine(c, pasta.best_multiexp(c, list(v) + [1], [A(x) for x in gens[1]] + [A(gens[2][0])]))
        assert [A(x) for x in fc] == [cl(f) for f in fixed] and [A(x) for x in pc] == [cl(s) for s in sigma]
        vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, c.p, m, D.omega, [A(x) for x in fc], [A(x) for x in pc]))
        fake.calls.clear()
        pk = h2.keygen_pk(prm, D, fixed, asm, delta, BC.BLINDING_FACTORS)
        assert fake.calls.count("h2_poly_permutation_sigma") == 1
        assert fake.calls.count("h2_poly_lagrange_to_coeff") == fake.calls.count("h2_poly_coeff_to_extended") == 4 + 3 + 3
        adv_bytes = [cref.ints_to_bytes(col) for col in adv]
        ref_pk = {}
        T = R.Blake2bTranscript(m)
        PP.create_proof_engine(h2, prm, vk, fixed, sigma, [adv_bytes], [[]], MC.SeededRng("fp", 5, True), T, ZETA, delta, pk=ref_pk)
        want = bytes(T.proof)
        mine = prover_pk_dict(pk)
        for key in ("fixed_l", "fixed_p", "fixed_c", "sigma_l", "sigma_p", "sigma_c", "l"):
            assert len(mine[key]) == len(ref_pk[key])
            for a, b in zip(mine[key], ref_pk[key]):
                assert a.len == b.len and (a.download() == b.download()).all(), key
        T = R.Blake2bTranscript(m)
        PP.create_proof_engine(h2, prm, vk, None, None, [adv_bytes], [[]], MC.SeededRng("fp", 5, True), T, ZETA, delta, pk=mine)
        assert bytes(T.proof) == want
        PP.close_proving_key(ref_pk)
        pk.close()
        assert not fake.polys
        prm.close()


def test_keygen_accepts_assigned_fixed_columns():
    """Fixed columns given as (numerator, denominator) pairs commit like their quotients."""
    import halo2_b200 as h2
    k = 3
    n = 1 << k
    m = pasta.P_MOD
    pts = cref.gen_points("vesta", 7, n + 2)
    with fake_engine.installed() as fake:
        prm = h2.Params("vesta", k, pts[:n], pts[:n], pts[n:n + 1], u=pts[n + 1:])
        D = h2.EvaluationDomain("fp", 3, k, ZETA)
        num = pasta.gen_scalars("fp", 1, n)
        den = [1, 0, 5, 1, m - 1, 3, 1, 9]
        quot = oracle_batch_invert_assigned([num], [den], m)[0]
        asm = h2.Assembly(n, 2)
        asm.copy(0, 1, 1, 6)
        got = h2.keygen_vk(prm, D, [(num, den), quot], asm, scalar_delta(m))
        assert (got[0][0] == got[0][1]).all() and got[1].shape == (2, 64)
        pk = h2.keygen_pk(prm, D, [(num, den)], asm, scalar_delta(m), 2)
        assert cref.bytes_to_ints(pk.fixed_values[0].download()) == quot
        assert [cref.bytes_to_ints(p.download()) for p in pk.permutation.permutations] == oracle_sigma(asm.mapping, n, D.omega, scalar_delta(m), m)
        l_vals = []
        for p in (pk.l0, pk.l_blind, pk.l_last):                   # back to Lagrange values: extended_to_coeff, then the forward NTT
            co = D.extended_to_coeff_resident(p)
            vals = cref.best_fft("fp", np.ascontiguousarray(co.download()[:n]), D.omega, k)
            l_vals.append(cref.bytes_to_ints(vals))
            co.close()
        assert l_vals == [[1] + [0] * 7, [0] * 6 + [1, 1], [0] * 5 + [1, 0, 0]]
        pk.close()
        prm.close()
        assert not fake.polys


# ---- 4. batch_invert_assigned ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("field", ["fp", "fq"])
def test_batch_invert_assigned_resident(field):
    import halo2_b200 as h2
    m = pasta.FIELDS[field]
    n = 16
    rnd = random.Random(4)
    nums = [pasta.gen_scalars(field, 10 + i, n) for i in range(3)]
    dens = [[1] * n,                                                          # every value trivial
            [0, 1, 2, 0] + pasta.gen_scalars(field, 20, n - 4),             # zero, trivial and rational
            [rnd.choice([0, 1, rnd.randrange(m)]) for _ in range(n)]]
    nums[2][3] = 0
    want = oracle_batch_invert_assigned(nums, dens, m)
    with fake_engine.installed() as fake:
        rn = [h2.ResidentPoly(field, n, cref.ints_to_bytes(v)) for v in nums]
        rd = [h2.ResidentPoly(field, n, cref.ints_to_bytes(v)) for v in dens]
        out = h2.batch_invert_assigned_resident(rn, rd)
        assert [cref.bytes_to_ints(p.download()) for p in out] == want
        assert [cref.bytes_to_ints(p.download()) for p in rd] == [[x % m for x in d] for d in dens]   # the inputs are left alone
        assert fake.calls.count("h2_poly_batch_invert") == 3 and fake.calls.count("h2_poly_eval_ast") == 3
        for p in rn + rd + out:
            p.close()
        assert not fake.polys
