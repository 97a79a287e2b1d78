"""GPU checks of the column-batched transforms (h2_poly_lagrange_to_coeff_batch / h2_poly_coeff_to_extended_batch),
h2_poly_set_rows, and instance_commit / advice_commit against a composition of per-column calls."""
import ctypes

import numpy as np
import pytest

import halo2_b200
from halo2_b200 import lib as L
from oracle import cref, pasta
from tests import columns_cases as CC

pytestmark = pytest.mark.gpu

_SCRATCH = 1 << 28   # ntt.cuh: H2_NTT_BATCH_SCRATCH


def _domain(field, k, ext_k):
    # a domain with extended_k = ext_k: quotient degree 2^(ext_k - k)
    return halo2_b200.EvaluationDomain(field, (1 << (ext_k - k)) + 1, k, pasta.zeta_candidates(field)[0])


def _group(log_n, count):
    if log_n <= 10:
        return count
    return max(1, min(count, _SCRATCH // (32 << log_n), 65535))


def _cols(field, seed, count, n):
    return [halo2_b200.ResidentPoly(field, n, cref.gen_scalars(field, seed + c, n)) for c in range(count)]


def _close(polys):
    for p in polys:
        p.close()


def _check_batch(D, count, seed, in_place=False):
    """Both batched transforms of `count` columns against the one-column calls, byte for byte, and their launch counts."""
    field, n, N = D.field, D.n, D.extended_len()
    src = _cols(field, seed, count, n)
    ref = [D.lagrange_to_coeff_resident(s, out=halo2_b200.ResidentPoly(field, n)) for s in src]
    before = L.launch_count()
    one = D.lagrange_to_coeff_resident(src[0], out=halo2_b200.ResidentPoly(field, n))
    one_launches = L.launch_count() - before
    ref_ext = [D.coeff_to_extended_resident(p) for p in ref]
    before = L.launch_count()
    one_ext = D.coeff_to_extended_resident(ref[0])
    one_ext_launches = L.launch_count() - before
    if in_place:
        work = _cols(field, seed, count, n)
        before = L.launch_count()
        co = D.lagrange_to_coeff_batch_resident(work)
    else:
        before = L.launch_count()
        co = D.lagrange_to_coeff_batch_resident(src, out=[halo2_b200.ResidentPoly(field, n) for _ in src])
    assert L.launch_count() - before == one_launches * -(-count // _group(D.k, count)), (D.k, count)
    before = L.launch_count()
    ext = D.coeff_to_extended_batch_resident(co)
    assert L.launch_count() - before == one_ext_launches * -(-count // _group(D.extended_k, count)), (D.extended_k, count)
    for c in range(count):
        assert np.array_equal(co[c].download(n), ref[c].download(n)), (field, D.k, count, c)
        assert np.array_equal(ext[c].download(N), ref_ext[c].download(N)), (field, D.k, D.extended_k, count, c)
    _close(src + ref + ref_ext + co + ext + [one, one_ext])


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_batched_transforms_equal_one_column_calls(field):
    for k in range(1, 21):
        D = _domain(field, k, k + (2 if k < 17 else 1))
        for count in (1, 3, 17):
            _check_batch(D, count, 1000 * k + count)


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_batched_transforms_in_place_shared_and_on_a_lane(field):
    for k in (4, 10, 11, 14, 18):
        _check_batch(_domain(field, k, k + 2), 3, 7 * k, in_place=True)
    # shared sources, one of them listed for two columns
    D = _domain(field, 12, 14)
    src = _cols(field, 5, 2, D.n)
    halo2_b200.share_resident(src)
    cols = [src[0], src[1], src[0]]
    co = D.lagrange_to_coeff_batch_resident(cols, out=[halo2_b200.ResidentPoly(field, D.n) for _ in cols])
    for p, s in zip(co, cols):
        one = D.lagrange_to_coeff_resident(s, out=halo2_b200.ResidentPoly(field, D.n))
        assert np.array_equal(p.download(), one.download())
        one.close()
    _close(co)
    with L.Lane():
        for k in (9, 14):
            _check_batch(_domain(field, k, k + 2), 5, 11 * k)
        _check_batch(_domain(field, 12, 14), 3, 99, in_place=True)
        # a shared source from the primary context, read on the lane
        co = D.lagrange_to_coeff_batch_resident(src, out=[halo2_b200.ResidentPoly(field, D.n) for _ in src])
        ref = [D.lagrange_to_coeff_resident(s, out=halo2_b200.ResidentPoly(field, D.n)) for s in src]
        assert all(np.array_equal(a.download(), b.download()) for a, b in zip(co, ref))
        _close(co + ref)
    _close(src)


def test_bulk_copy_variant_batches_the_same_way():
    """The opt-in bulk-copy (TMA) pass kernel takes the columns in grid.y too: the same bytes as the one-column calls."""
    lib = L.init()
    L.check(lib.h2_test_set_ntt_tma(1))
    try:
        for field in ("fp", "fq"):
            for k in (11, 14, 17):
                _check_batch(_domain(field, k, k + 2), 5, 13 * k)
    finally:
        L.check(lib.h2_test_set_ntt_tma(0))


def _call(name, dst, src, k, ext_k=None):
    field = "fp"
    D = _domain(field, k, ext_k or k + 1)
    hs = lambda ps: (ctypes.c_uint64 * len(ps))(*[p if isinstance(p, int) else p._h.value for p in ps])   # noqa: E731
    lib = L.init()
    if name == "l2c":
        return lib.h2_poly_lagrange_to_coeff_batch(hs(dst), hs(src), ctypes.c_size_t(len(dst)), ctypes.c_uint32(k), L.ptr(L.fe_bytes(D.omega_inv)),
                                                   L.ptr(L.fe_bytes(D.ifft_divisor)), L.REPR_CANONICAL)
    return lib.h2_poly_coeff_to_extended_batch(hs(dst), hs(src), ctypes.c_size_t(len(dst)), ctypes.c_uint32(k), ctypes.c_uint32(D.extended_k),
                                               L.ptr(L.fe_bytes(D.g_coset)), L.ptr(L.fe_bytes(D.extended_omega)), L.REPR_CANONICAL)


@pytest.mark.parametrize("on_lane", [False, True])
def test_argument_errors_name_the_column_launch_nothing_and_change_nothing(on_lane):
    lane = L.Lane().bind() if on_lane else None
    try:
        k, n = 8, 256
        a = _cols("fp", 1, 4, n)
        d = _cols("fp", 9, 4, 4 * n)
        short = halo2_b200.ResidentPoly("fp", n // 2)
        other = halo2_b200.ResidentPoly("fq", n)
        shared = _cols("fp", 20, 1, n)
        halo2_b200.share_resident(shared)
        snap = [p.download() for p in a + d]
        cases = [
            ("l2c", [d[0], d[1], d[0]], a[:3], k, None, "dst\\[2\\] is also dst\\[0\\]"),
            ("l2c", [a[1], d[1]], [a[0], a[1]], k, None, "dst\\[0\\] is also src\\[1\\]"),
            ("l2c", [d[0], d[1]], [a[0], short], k, None, "src\\[1\\]: a polynomial holds fewer than 2\\^k"),
            ("c2e", [d[0], short], [a[0], a[1]], k, k + 2, "dst\\[1\\]: a polynomial holds fewer than 2\\^ext_k"),
            ("l2c", [d[0], 987654321], [a[0], a[1]], k, None, "dst\\[1\\]: unknown polynomial handle"),
            ("l2c", [d[0], d[1]], [a[0], 987654321], k, None, "src\\[1\\]: unknown polynomial handle"),
            ("l2c", [d[0], shared[0]], [a[0], a[1]], k, None, "dst\\[1\\]: the polynomial is shared"),
            ("l2c", [d[0], d[1]], [a[0], other], k, None, "src\\[1\\]: the polynomials live in different fields"),
            ("c2e", [d[0], d[1]], [a[0], d[1]], k, k + 2, "dst\\[1\\] == src\\[1\\]: in place needs equal input and output sizes"),
        ]
        for name, dst, src, kk, ext_k, msg in cases:
            before = L.launch_count()
            with pytest.raises(L.H2Error, match=msg):
                L.check(_call(name, dst, src, kk, ext_k))
            assert L.launch_count() == before, msg
        assert all(np.array_equal(p.download(), s) for p, s in zip(a + d, snap))
        before = L.launch_count()
        L.check(_call("l2c", [], [], k))                       # count == 0: nothing
        assert L.launch_count() == before
        # set_rows: a repeated polynomial or rows past the end fail before the upload and change nothing
        vals = np.stack([cref.gen_scalars("fp", 3, 6)] * 2)
        for polys, start, msg in (([a[0], a[0]], 10, "polys\\[1\\] is also polys\\[0\\]"),
                                  ([a[0], short], n // 2 - 3, "polys\\[1\\]: a polynomial holds fewer than start \\+ rows elements"),
                                  ([a[0], shared[0]], 0, "polys\\[1\\]: the polynomial is shared")):
            before = L.launch_count()
            with pytest.raises(L.H2Error, match=msg):
                halo2_b200.set_rows_resident(polys, start, vals)
            assert L.launch_count() == before
        assert all(np.array_equal(p.download(), s) for p, s in zip(a + d, snap))
        _close(a + d + [short, other] + shared)
    finally:
        if lane is not None:
            lane.close()


def test_set_rows_equals_per_column_copies():
    n, start, rows = 1 << 11, (1 << 11) - 6, 6
    a, b = _cols("fq", 3, 7, n), _cols("fq", 3, 7, n)
    vals = np.stack([cref.gen_scalars("fq", 40 + c, rows) for c in range(7)])
    before = L.launch_count()
    halo2_b200.set_rows_resident(a, start, vals)
    assert L.launch_count() - before == 1
    for p, v in zip(b, vals):
        t = halo2_b200.ResidentPoly("fq", rows, v)
        p.copy_from(t, rows, dst_off=start)
        t.close()
    assert all(np.array_equal(x.download(), y.download()) for x, y in zip(a, b))
    _close(a + b)


def _params(curve, k):
    return halo2_b200.Params.new(curve, k)


def test_phases_of_the_plonk_api_circuit():
    from tests import plonk_verifier as PV
    from tests import plonk_api_circuit as circ
    vk = PV.PinnedKey(circ.CASE["key_text"])
    prm = _params("vesta", vk.k)
    advice, instances = [circ.witness(), circ.witness()], [[[2]], [[2]]]
    D = halo2_b200.EvaluationDomain("fp", vk.degree(), vk.k, circ.ZETA)
    bf = vk.blinding_factors()
    CC.assert_same(CC.composition_phases(halo2_b200, prm, D, bf, advice, instances, 777), CC.batched_phases(halo2_b200, prm, D, bf, advice, instances, 777))
    prm.close()


def test_phases_of_a_golden_proof_shape():
    """A k = 11 circuit of the reference's stored proofs (10 advice columns, extended_k = 14), two proofs per call."""
    from tests import plonk_verifier as PV
    case = next(c for c in PV.load_golden_proofs() if PV.PinnedKey(c["key_text"]).k == 11 and PV.PinnedKey(c["key_text"]).num_advice_columns == 10)
    vk = PV.PinnedKey(case["key_text"])
    assert vk.extended_k == 14
    field = {pasta.P_MOD: "fp", pasta.Q_MOD: "fq"}[vk.scalar_modulus]
    curve = {"fp": "vesta", "fq": "pallas"}[field]
    prm = _params(curve, 11)
    zeta = pasta.zeta_candidates(field)[0]
    advice = CC.random_columns(field, 5, 2, 10, 1 << 11)
    instances = [[[3, 4, 5]] * vk.num_instance_columns] * 2
    D = halo2_b200.EvaluationDomain(field, vk.degree(), 11, zeta)
    bf = vk.blinding_factors()
    CC.assert_same(CC.composition_phases(halo2_b200, prm, D, bf, advice, instances, 91), CC.batched_phases(halo2_b200, prm, D, bf, advice, instances, 91))
    prm.close()


def test_phases_of_the_benchmark_circuit_shape():
    """The benchmark circuit's shape (benches/plonk.rs) at k = 14: 5 advice columns, one instance column, two proofs per call."""
    from tests import bench_circuit as BC
    zeta = pasta.zeta_candidates("fp")[0]
    D = halo2_b200.EvaluationDomain("fp", BC.DEGREE, 14, zeta)
    prm = _params("vesta", 14)
    advice = CC.random_columns("fp", 9, 2, 5, 1 << 14)
    instances = [[list(range(1, 40))], [[7] * 100]]
    bf = BC.BLINDING_FACTORS
    CC.assert_same(CC.composition_phases(halo2_b200, prm, D, bf, advice, instances, 5), CC.batched_phases(halo2_b200, prm, D, bf, advice, instances, 5))
    prm.close()
