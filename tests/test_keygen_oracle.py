"""CPU checks of key generation (halo2_b200/keygen.py, csrc/keygen.cuh) against a restatement of the reference
(plonk/permutation/keygen.rs:24-211, plonk/keygen.rs:240-336, poly.rs:135-180):

- the mirror's Assembly, fed the copy sequences of the plonk_api and benchmark circuits, gives the mappings whose sigma
  polynomials the test circuits pin;
- the device bodies of the sigma kernel and its power tables, on the host emulation, equal the reference's serial
  omega-power loop and deltaomega gather;
- keygen_pk / keygen_vk / batch_invert_assigned_resident run their calls, in their order, over an ABI stand-in (the
  sigma kernel on the emulation), and reproduce the test prover's proving-key values."""
import contextlib
import ctypes
import random

import numpy as np
import pytest

from oracle import cref, pasta
from tests import bench_circuit as BC
from tests import fake_engine
from tests import plonk_api_circuit as circ
from tests.kernel_emul import build as emul_build
from tests.test_oracle_golden import FP_ZETA_INDEX

KEYGEN_CHUNK = 1 << 22                                             # rows per launch in capi_poly.cu (H2_KEYGEN_CHUNK)
ZETA = pasta.zeta_candidates("fp")[FP_ZETA_INDEX]


# ---- the reference, restated -------------------------------------------------------------------------------------------
def oracle_assembly(n: int, num_columns: int):
    """Assembly::new (permutation/keygen.rs:25-43): (mapping, aux, sizes) as lists of lists of (column, row) tuples."""
    mapping = [[(i, j) for j in range(n)] for i in range(num_columns)]
    aux = [[(i, j) for j in range(n)] for i in range(num_columns)]
    sizes = [[1] * n for _ in range(num_columns)]
    return mapping, aux, sizes


def oracle_copy(asm, left_column: int, left_row: int, right_column: int, right_row: int) -> None:
    """Assembly::copy (permutation/keygen.rs:45-100); IndexError for Error::BoundsFailure."""
    mapping, aux, sizes = asm
    if left_row >= len(mapping[left_column]) or right_row >= len(mapping[right_column]):
        raise IndexError("BoundsFailure")
    left_cycle = aux[left_column][left_row]
    right_cycle = aux[right_column][right_row]
    if left_cycle == right_cycle:
        return
    if sizes[left_cycle[0]][left_cycle[1]] < sizes[right_cycle[0]][right_cycle[1]]:
        left_cycle, right_cycle = right_cycle, left_cycle
    sizes[left_cycle[0]][left_cycle[1]] += sizes[right_cycle[0]][right_cycle[1]]
    i = right_cycle
    while True:
        aux[i[0]][i[1]] = left_cycle
        i = mapping[i[0]][i[1]]
        if i == right_cycle:
            break
    tmp = mapping[left_column][left_row]
    mapping[left_column][left_row] = mapping[right_column][right_row]
    mapping[right_column][right_row] = tmp


def oracle_sigma(mapping, n: int, omega: int, delta: int, m: int):
    """build_vk / build_pk's permutation polynomials (permutation/keygen.rs:108-143): the serial omega-power loop, the
    deltaomega table, the gather.  `mapping[i][j]` = (column, row)."""
    omega_powers = []
    cur = 1
    for _ in range(n):
        omega_powers.append(cur)
        cur = cur * omega % m
    deltaomega = []
    cur = 1
    for _ in range(len(mapping)):
        deltaomega.append([o * cur % m for o in omega_powers])
        cur = cur * delta % m
    return [[deltaomega[int(c)][int(r)] for c, r in mapping[i]] for i in range(len(mapping))]


def oracle_batch_invert_assigned(numerators, denominators, m: int):
    """batch_invert_assigned (poly.rs:135-180): numerator * denominator^-1, with BatchInvert leaving a zero denominator 0."""
    return [[a * (pow(d, -1, m) if d % m else 0) % m for a, d in zip(nums, dens)] for nums, dens in zip(numerators, denominators)]


def plonk_api_copies():
    """The plonk_api circuit's copy constraints in the order synthesis makes them (tests/plonk_api.rs:399-400, each twice by
    StandardCs::copy, :216-217): columns a = 0, b = 1, c = 2 of the permutation."""
    for it in range(10):
        rm, ra = 1 + 2 * it, 2 + 2 * it
        yield from [(0, rm, 0, ra)] * 2
        yield from [(1, ra, 2, rm)] * 2


def bench_copies(k: int):
    """The benchmark circuit's (benches/plonk.rs:226-241): copy(a0, a1) and copy(b1, c0) per multiply / add pair."""
    for it in range((1 << (k - 1)) - 3):
        rm, ra = 2 * it, 2 * it + 1
        yield 0, rm, 0, ra
        yield 1, ra, 2, rm


def delta_of(m: int) -> int:
    return pow(pasta.MULT_GEN, 1 << pasta.S_2ADICITY, m)          # F::DELTA


def prover_pk_dict(pk):
    """The proving key in the shape tests/plonk_prover.create_proof_engine(pk=...) keeps it."""
    P = pk.permutation
    return {"fixed_l": pk.fixed_values, "fixed_p": pk.fixed_polys, "fixed_c": pk.fixed_cosets, "sigma_l": P.permutations,
            "sigma_p": P.polys, "sigma_c": P.cosets, "l": [pk.l0, pk.l_blind, pk.l_last]}


# ---- 1. the mirror's Assembly ------------------------------------------------------------------------------------------
def test_assembly_plonk_api_circuit():
    import halo2_b200 as h2
    m = pasta.P_MOD
    omega, delta = pasta.omega_for_k("fp", circ.K), delta_of(m)
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
    omega, delta = pasta.omega_for_k("fp", k), delta_of(m)
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


def random_mapping(rng, cols: int, n: int) -> np.ndarray:
    """Random in-range (column, row) entries, with rows 0 and n - 1 and every column present."""
    mp = np.empty((cols, n, 2), dtype=np.uint32)
    mp[..., 0] = rng.integers(0, cols, size=(cols, n))
    mp[..., 1] = rng.integers(0, n, size=(cols, n))
    mp[0, 0] = (cols - 1, n - 1)
    mp[cols - 1, n - 1] = (0, 0)
    mp[:, 0, 0] = np.arange(cols)
    return mp


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
        omega, delta = pasta.omega_for_k(field, k), delta_of(m)
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
    delta = delta_of(m)
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
        rc, _ = emu_sigma(emu, field, mp, k, omega, delta_of(m))
        assert rc == 1
    rc, _ = emu_sigma(emu, field, random_mapping(rng, cols, n), k, omega, delta_of(m))
    assert rc == 0


# ---- 3. keygen.py over an ABI stand-in ---------------------------------------------------------------------------------
class KeygenFakeLib(fake_engine.FakeLib):
    """tests/fake_engine.FakeLib plus h2_poly_permutation_sigma, whose kernel bodies run on the host emulation with the
    library's argument checks."""

    def h2_poly_permutation_sigma(self, dst, cols, k, mapping, omega, delta, repr_):
        self._log("h2_poly_permutation_sigma")
        cols, k = fake_engine._v(cols), fake_engine._v(k)
        if k > 30:
            return self._fail("h2_poly_permutation_sigma: k > 30")
        if cols == 0:
            return 0
        hs = [int(dst[i]) for i in range(cols)]
        unknown = [i for i, h in enumerate(hs) if h not in self.polys]
        if unknown:
            return self._fail(f"h2_poly_permutation_sigma: dst[{unknown[0]}]: unknown polynomial handle")
        c = fake_engine.clash(fake_engine.args("dst", hs, True))
        if c:
            return self._fail(f"h2_poly_permutation_sigma: {c}")
        field = self.polys[hs[0]][0]
        n = 1 << k
        if any(self.polys[h][0] != field or self.polys[h][1].shape[0] < n for h in hs):
            return self._fail("h2_poly_permutation_sigma: a polynomial of another field or shorter than 2^k")
        mp = np.frombuffer(ctypes.string_at(fake_engine._v(mapping), 8 * cols * n), dtype=np.uint32).copy()
        out = np.zeros((cols * n, 32), dtype=np.uint8)
        rc = self.emu.emu_permutation_sigma(cref.FIELD_ID[field], mp.ctypes.data_as(ctypes.c_void_p), cols, k,
                                            cref._p(fake_engine._rd(omega, 32)), cref._p(fake_engine._rd(delta, 32)), ctypes.c_uint64(KEYGEN_CHUNK),
                                            cref._p(out))
        if rc:
            return self._fail("h2_poly_permutation_sigma: a mapping entry is outside the permutation's columns or the domain's rows")
        for i, h in enumerate(hs):
            self.polys[h][1][:n] = out[i * n:(i + 1) * n]
        return 0


@contextlib.contextmanager
def installed():
    from halo2_b200 import lib as L
    saved = (L._lib, L._inited_device)
    fake = KeygenFakeLib()
    L._lib, L._inited_device = fake, 0
    try:
        yield fake
    finally:
        L._lib, L._inited_device = saved


def _bench_setup(k: int):
    c = pasta.VESTA
    m = pasta.P_MOD
    n = 1 << k
    pts = cref.gen_points("vesta", 99, n + 2)
    gens = (pts[:n], cref.params_lagrange("vesta", pts[:n], k, pasta.inv(pasta.omega_for_k("fp", k), m), pow(pasta.inv(2, m), k, m)),
            pts[n:n + 1], pts[n + 1:n + 2])
    omega = pasta.omega_for_k("fp", k)
    fixed, sigma, adv = BC.columns(k, m, omega, delta_of(m), circ.A_SMALL * ZETA % m)
    asm_copies = list(bench_copies(k))
    return c, m, gens, fixed, sigma, adv, asm_copies


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
    delta = delta_of(m)
    with installed() as fake:
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
    with installed() as fake:
        prm = h2.Params("vesta", k, pts[:n], pts[:n], pts[n:n + 1], u=pts[n + 1:])
        D = h2.EvaluationDomain("fp", 3, k, ZETA)
        num = pasta.gen_scalars("fp", 1, n)
        den = [1, 0, 5, 1, m - 1, 3, 1, 9]
        quot = oracle_batch_invert_assigned([num], [den], m)[0]
        asm = h2.Assembly(n, 2)
        asm.copy(0, 1, 1, 6)
        got = h2.keygen_vk(prm, D, [(num, den), quot], asm, delta_of(m))
        assert (got[0][0] == got[0][1]).all() and got[1].shape == (2, 64)
        pk = h2.keygen_pk(prm, D, [(num, den)], asm, delta_of(m), 2)
        assert cref.bytes_to_ints(pk.fixed_values[0].download()) == quot
        assert [cref.bytes_to_ints(p.download()) for p in pk.permutation.permutations] == oracle_sigma(asm.mapping, n, D.omega, delta_of(m), m)
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
    with installed() as fake:
        rn = [h2.ResidentPoly(field, n, cref.ints_to_bytes(v)) for v in nums]
        rd = [h2.ResidentPoly(field, n, cref.ints_to_bytes(v)) for v in dens]
        out = h2.batch_invert_assigned_resident(rn, rd)
        assert [cref.bytes_to_ints(p.download()) for p in out] == want
        assert [cref.bytes_to_ints(p.download()) for p in rd] == [[x % m for x in d] for d in dens]   # the inputs are left alone
        assert fake.calls.count("h2_poly_batch_invert") == 3 and fake.calls.count("h2_poly_eval_ast") == 3
        for p in rn + rd + out:
            p.close()
        assert not fake.polys
