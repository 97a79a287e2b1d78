"""GPU checks of h2_poly_vanishing_quotient and halo2_b200.vanishing: the fused call against the existing path
(divide_by_vanishing_poly + extended_to_coeff + one copy per piece), a proof composed with the module against
create_proof_engine, the argument checks, cleanup on failure, and a run on a lane over a shared key."""
import ctypes

import numpy as np
import pytest

import halo2_b200
from halo2_b200 import lib as L
from halo2_b200 import vanishing as V
from oracle import cref, pasta
from tests import arguments_cases as AC
from tests import multiopen_cases as MC
from tests import plonk_api_circuit as circ
from tests import plonk_prover as PP
from tests import vanishing_cases as VC

pytestmark = pytest.mark.gpu

WHO = "h2_poly_vanishing_quotient"


def _close(polys):
    for p in polys:
        p.close()


def _old_pieces(D, h_ext):
    """The existing path: divide_by_vanishing_poly in place on a copy, extended_to_coeff, one copy per piece."""
    N, n, d = D.extended_len(), D.n, D.quotient_poly_degree
    tmp = halo2_b200.ResidentPoly(D.field, N).copy_from(h_ext, N)
    D.divide_by_vanishing_poly_resident(tmp)
    h = D.extended_to_coeff_resident(tmp)
    pieces = [halo2_b200.ResidentPoly(D.field, n).copy_from(h, n, src_off=i * n) for i in range(d)]
    _close([tmp, h])
    return pieces


def _same(a, b, n):
    return all(np.array_equal(x.download(n), y.download(n)) for x, y in zip(a, b)) and len(a) == len(b)


def _check_parity(D, seed):
    h_ext = halo2_b200.ResidentPoly(D.field, D.extended_len(), cref.gen_scalars(D.field, seed, D.extended_len()))
    before = h_ext.download()
    want = _old_pieces(D, h_ext)
    got = V.vanishing_quotient_resident(D, h_ext)
    assert _same(got, want, D.n), (D.field, D.k, D.extended_k)
    assert np.array_equal(h_ext.download(), before)                       # the source is only read
    _close(got + want + [h_ext])


def _zeta(field):
    return pasta.zeta_candidates(field)[0]


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("degree", [3, 5])
def test_pieces_equal_the_existing_path(field, degree):
    for k in range(1, 21):
        _check_parity(halo2_b200.EvaluationDomain(field, degree, k, _zeta(field)), 500 * k + degree)


def _golden_k11():
    from tests import plonk_verifier as PV
    case = next(c for c in PV.load_golden_proofs() if PV.PinnedKey(c["key_text"]).k == 11 and PV.PinnedKey(c["key_text"]).extended_k == 14)
    return PV.PinnedKey(case["key_text"])


def test_pieces_equal_the_existing_path_at_the_golden_keys_degree():
    vk = _golden_k11()
    field = {pasta.P_MOD: "fp", pasta.Q_MOD: "fq"}[vk.scalar_modulus]
    D = halo2_b200.EvaluationDomain(field, vk.degree(), 11, _zeta(field))
    assert D.extended_k == 14 and 6 <= vk.degree() <= 9
    _check_parity(D, 11)


def test_the_bulk_copy_setting_changes_nothing():
    """The opt-in bulk-copy pass kernel does not take the fused passes: with it on, the call gives the same bytes."""
    lib = L.init()
    L.check(lib.h2_test_set_ntt_tma(1))
    try:
        for k in (9, 14):
            _check_parity(halo2_b200.EvaluationDomain("fp", 5, k, _zeta("fp")), k)
    finally:
        L.check(lib.h2_test_set_ntt_tma(0))


def _plonk_api():
    vk = circ.plonk_api_key()
    return vk, circ.fixed_columns(circ.M, circ.ZETA), circ.permutation_columns(circ.M, vk.omega, circ.DELTA)


def _assert_same(want, got):
    assert len(want["points"]) == len(got["points"]) and all(np.array_equal(a, b) for a, b in zip(want["points"], got["points"]))
    assert want["scalars"] == got["scalars"]
    assert len(want["queries"]) == len(got["queries"]) == 2
    for (wx, wa, wb), (gx, ga, gb) in zip(want["queries"], got["queries"]):
        assert wx == gx and wb == gb and np.array_equal(wa, ga)
    assert want["proof"] == got["proof"]


def _engine_and_package(prm, D, vk, fixed, sigma, advice, instances, seed):
    """VC.record of create_proof_engine and of create_proof_package (over a key from arguments_cases.proving_key) on the same
    inputs and seeded rng."""
    engine_pk, pk = {}, AC.proving_key(halo2_b200, D, fixed, sigma, vk.blinding_factors())
    try:
        want = VC.record(halo2_b200, circ.M, lambda eng, t: PP.create_proof_engine(eng, prm, vk, fixed, sigma, advice, instances,
                                                                                  MC.SeededRng("fp", seed, True), t, circ.ZETA, circ.DELTA, pk=engine_pk))
        got = VC.record(halo2_b200, circ.M, lambda eng, t: AC.create_proof_package(eng, prm, D, pk, vk, advice, instances,
                                                                                  MC.SeededRng("fp", seed, True), t, circ.DELTA))
    finally:
        PP.close_proving_key(engine_pk)
        pk.close()
    return want, got


def test_the_module_equals_create_proof_engine_on_the_plonk_api_circuit():
    """Under the golden key and one seeded rng, a proof whose vanishing argument comes from the module (create_proof_package)
    and create_proof_engine's: the random commitment, the h piece commitments (every point written), random_eval (every scalar
    written), h_poly / h_blind and random_poly / random_blind (the last two queries) and the proof bytes, which the engine's
    verifier and the restated reference verifier accept."""
    from tests import plonk_verifier as PV
    vk, fixed, sigma = _plonk_api()
    prm = halo2_b200.Params.new("vesta", 5)
    try:
        inst = [[[2]], [[2]]]
        D = halo2_b200.EvaluationDomain("fp", vk.degree(), vk.k, circ.ZETA)
        want, got = _engine_and_package(prm, D, vk, fixed, sigma, [circ.witness(), circ.witness()], inst, 777)
        _assert_same(want, got)
        assert len(got["proof"]) == 4160
        gens = (prm.g, prm.g_lagrange, prm.w, prm.u)
        earm = PV.EngineArm(halo2_b200, "vesta", 5, *gens)
        try:
            assert PV.verify_proof(earm, vk, got["proof"], inst, circ.DELTA)
        finally:
            earm.close()
        assert PV.verify_proof(PV.OracleArm("vesta", 5, *gens), vk, got["proof"], inst, circ.DELTA)
    finally:
        prm.close()


def test_the_module_equals_create_proof_engine_on_the_benchmark_circuit_k14():
    """The benchmark circuit (benches/plonk.rs, degree 5: four pieces of a 4n extended domain) at k = 14, key built as
    tests/test_gpu_zz_real_proof.py builds it; create_proof_engine keeps its own resident key, the package proves over
    arguments_cases.proving_key's."""
    from tests import bench_circuit as BC
    from tests import plonk_verifier as PV
    k, m = 14, circ.M
    n = 1 << k
    pts = cref.gen_points("vesta", 77, n + 2)
    g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    prm = halo2_b200.Params("vesta", k, g, halo2_b200.lagrange_generators("vesta", k, g), w, u=u)
    try:
        D = halo2_b200.EvaluationDomain("fp", BC.DEGREE, k, circ.ZETA)
        assert D.quotient_poly_degree == 4 and D.extended_k == k + 2
        fixed, sigma, adv = BC.columns(k, m, D.omega, circ.DELTA, circ.A_SMALL * circ.ZETA % m)
        fb, sb, ab = ([cref.ints_to_bytes(c_) for c_ in cols] for cols in (fixed, sigma, adv))
        xy = lambda col: cref.bytes_to_affine(halo2_b200.batch_normalize(prm.commit_lagrange(col, halo2_b200.Blind(1)).reshape(1, 96), "vesta")[0])  # noqa: E731
        vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, pasta.Q_MOD, m, D.omega, [xy(c_) for c_ in fb], [xy(c_) for c_ in sb]))
        want, got = _engine_and_package(prm, D, vk, fb, sb, [ab], [[]], 5)
        _assert_same(want, got)
        arm = PV.EngineArm(halo2_b200, "vesta", k, params=prm)
        assert PV.verify_proof(arm, vk, got["proof"], [[]], circ.DELTA)
    finally:
        prm.close()


def _call(pieces, src, k, ext_k, t=None, t_len=None, count=None, nulls=()):
    """One h2_poly_vanishing_quotient call; the scalars and t_evals are those of the fp domain k = 6, extended_k = 8."""
    D = halo2_b200.EvaluationDomain("fp", 5, 6, _zeta("fp"))
    if t is None:
        t = np.ascontiguousarray(np.stack([L.fe_bytes(v) for v in D.t_evaluations]))
    keep = {"ext_omega_inv": L.fe_bytes(D.extended_omega_inv), "ext_divisor": L.fe_bytes(D.extended_ifft_divisor), "zeta": L.fe_bytes(D.g_coset),
            "t_evals": t}
    scal = {name: None if name in nulls else L.ptr(arr) for name, arr in keep.items()}
    hs = (ctypes.c_uint64 * max(len(pieces), 1))(*[p if isinstance(p, int) else p._h.value for p in pieces])
    return L.init().h2_poly_vanishing_quotient(None if "pieces" in nulls else hs, ctypes.c_size_t(len(pieces) if count is None else count),
                                               ctypes.c_uint64(src if isinstance(src, int) else src._h.value), ctypes.c_uint32(k),
                                               ctypes.c_uint32(ext_k), scal["ext_omega_inv"], scal["ext_divisor"], scal["zeta"], scal["t_evals"],
                                               ctypes.c_uint32(t.shape[0] if t_len is None else t_len), L.REPR_CANONICAL)


@pytest.mark.parametrize("on_lane", [False, True])
def test_argument_errors_name_the_argument_launch_nothing_and_change_nothing(on_lane):
    lane = L.Lane().bind() if on_lane else None
    try:
        k, ext_k, n, N = 6, 8, 64, 256
        src = halo2_b200.ResidentPoly("fp", N, cref.gen_scalars("fp", 1, N))
        pieces = [halo2_b200.ResidentPoly("fp", n, cref.gen_scalars("fp", 10 + i, n)) for i in range(4)]
        short = halo2_b200.ResidentPoly("fp", n - 1)
        short_src = halo2_b200.ResidentPoly("fp", N - 1)
        other = halo2_b200.ResidentPoly("fq", n)
        shared = halo2_b200.ResidentPoly("fp", n).share()
        snap = [p.download() for p in pieces + [src]]
        p0, p1, p2, p3 = pieces
        cases = [
            (dict(pieces=[p0, 987654321], src=src), "pieces[1]: unknown polynomial handle"),
            (dict(pieces=[p0, p1], src=987654321), "unknown polynomial handle"),
            (dict(pieces=[p0, other], src=src), "pieces[1]: the polynomials live in different fields"),
            (dict(pieces=[p0, p1, shared], src=src), "pieces[2]: the polynomial is shared (read-only)"),
            (dict(pieces=[p0, p1, short], src=src), "pieces[2]: a polynomial holds fewer than 2^k elements"),
            (dict(pieces=[p0, p1, p0], src=src), "pieces[2] is also pieces[0]"),
            (dict(pieces=[p0, src], src=src), "pieces[1] is also src"),
            (dict(pieces=[p0, p1], src=short_src), "a polynomial holds fewer than 2^ext_k elements"),
            (dict(pieces=[], src=src, count=0), "count must be at least 1 and count * 2^k at most 2^ext_k"),
            (dict(pieces=[p0, p1, p2, p3, p0], src=src), "count must be at least 1 and count * 2^k at most 2^ext_k"),
            (dict(pieces=[p0], src=src, k=9), "ext_k < k"),
            (dict(pieces=[p0], src=src, ext_k=31), "ext_k > 30"),
            (dict(pieces=[p0], src=src, t_len=3), "t_len must be a power of two <= 2^ext_k"),
            (dict(pieces=[p0], src=src, t_len=0), "t_len must be a power of two <= 2^ext_k"),
            (dict(pieces=[p0], src=src, t_len=512, t=np.zeros((512, 32), np.uint8)), "t_len must be a power of two <= 2^ext_k"),
            (dict(pieces=[p0], src=src, nulls=("pieces",)), "null handle array"),
        ] + [(dict(pieces=[p0], src=src, nulls=(name,)), f"null {name}") for name in ("ext_omega_inv", "ext_divisor", "zeta", "t_evals")]
        for kw, msg in cases:
            kw = {"k": k, "ext_k": ext_k, **kw}
            before = L.launch_count()
            rc = _call(**kw)
            assert rc != 0 and L.load().h2_last_error().decode() == f"{WHO}: {msg}", (msg, L.load().h2_last_error())
            assert L.launch_count() == before, msg
        assert all(np.array_equal(p.download(), s) for p, s in zip(pieces + [src], snap))
        L.check(_call(pieces, src, k, ext_k))                                # and the same arguments, corrected, work
        _close(pieces + [src, short, short_src, other, shared])
    finally:
        if lane is not None:
            lane.close()


class _Counting(halo2_b200.ResidentPoly):
    live = set()

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        _Counting.live.add(self._h.value)

    def close(self):
        _Counting.live.discard(self._h.value)
        super().close()


class _Rng:
    def __init__(self, fail_at=None):
        self.inner, self.fail_at, self.i = MC.SeededRng("fp", 3, True), fail_at, 0

    def scalar(self):
        self.i += 1
        if self.i == self.fail_at:
            raise RuntimeError("rng failed")
        return self.inner.scalar()

    def poly(self, n):
        return self.inner.poly(n)


def test_a_failing_construct_leaves_nothing_allocated(monkeypatch):
    """construct fails in the evaluation, in the quotient call and in the blinds after it: every polynomial the module opened
    is closed again, and the extended temporary never outlives the call."""
    monkeypatch.setattr(V, "ResidentPoly", _Counting)
    k = 8
    D = halo2_b200.EvaluationDomain("fp", 5, k, _zeta("fp"))
    prm = halo2_b200.Params.new("vesta", k)
    cols = [halo2_b200.ResidentPoly("fp", D.extended_len(), cref.gen_scalars("fp", 20 + i, D.extended_len())) for i in range(2)]
    try:
        ev = halo2_b200.Evaluator(D, "extended")
        a, b = (ev.register_poly(c) for c in cols)
        committed, _ = V.vanishing_commit(prm, D, _Rng())
        opened = set(_Counting.live)
        bad = halo2_b200.EvaluationDomain("fp", 5, k, _zeta("fp"))
        bad.extended_k -= 1                                               # the evaluation's output is one coset too short
        with pytest.raises(L.H2Error):
            committed.construct(prm, bad, ev, [a * b], 5, _Rng())
        assert _Counting.live == opened
        bad = halo2_b200.EvaluationDomain("fp", 5, k, _zeta("fp"))
        bad.t_evaluations = bad.t_evaluations[:3]                         # not a power of two: the quotient call fails
        with pytest.raises(L.H2Error, match=f"{WHO}: t_len must be a power of two"):
            committed.construct(prm, bad, ev, [a * b], 5, _Rng())
        assert _Counting.live == opened
        with pytest.raises(RuntimeError, match="rng failed"):
            committed.construct(prm, D, ev, [a * b], 5, _Rng(fail_at=2))
        assert _Counting.live == opened
        constructed, cm = committed.construct(prm, D, ev, [a * b, a + b], 5, _Rng())
        assert len(_Counting.live) == len(opened) + 4 and cm.shape == (4, 64)
        evaluated, _ = constructed.evaluate(D, 12345)
        evaluated.close()
        constructed.close()
        assert not _Counting.live
    finally:
        _close(cols)
        prm.close()


def test_on_a_lane_against_a_shared_key():
    """h(X) of a shared proving key's extended cosets, evaluated and constructed on a lane: the same pieces and commitments as
    the existing path on the primary context, and a shared source works too."""
    k = 12
    D = halo2_b200.EvaluationDomain("fp", 5, k, _zeta("fp"))
    prm = halo2_b200.Params.new("vesta", k)
    key = [D.coeff_to_extended_resident(halo2_b200.ResidentPoly("fp", D.n, cref.gen_scalars("fp", 40 + i, D.n))) for i in range(3)]
    halo2_b200.share_resident(key)
    ev = halo2_b200.Evaluator(D, "extended")
    a, b, c = (ev.register_poly(p) for p in key)
    exprs = [a * b - c, a.with_rotation(1) * c, b + c * 7]
    y = 987654321
    h_ext = ev.evaluate(halo2_b200.Ast.distribute_powers(exprs, y))
    want = _old_pieces(D, h_ext)
    rng = MC.SeededRng("fp", 8, True)
    blinds = [rng.scalar() for _ in want]
    want_cm = prm.commit_resident_affine(want, [halo2_b200.Blind(x) for x in blinds])
    shared_src = halo2_b200.ResidentPoly("fp", D.extended_len()).copy_from(h_ext, D.extended_len()).share()
    want_bytes = [p.download() for p in want]          # the primary context's polynomials are not readable on a lane
    try:
        with L.Lane():
            ev_lane = halo2_b200.Evaluator(D, "extended")
            la, lb, lc = (ev_lane.register_poly(p) for p in key)
            committed, _ = V.vanishing_commit(prm, D, MC.SeededRng("fp", 1, True))
            constructed, cm = committed.construct(prm, D, ev_lane, [la * lb - lc, la.with_rotation(1) * lc, lb + lc * 7], y,
                                                  MC.SeededRng("fp", 8, True))
            assert all(np.array_equal(p.download(), w) for p, w in zip(constructed.h_pieces, want_bytes))
            assert np.array_equal(cm, want_cm)
            from_shared = V.vanishing_quotient_resident(D, shared_src)
            assert all(np.array_equal(p.download(), w) for p, w in zip(from_shared, want_bytes))
            _close(from_shared)
            constructed.close()
    finally:
        _close(want + [h_ext, shared_src] + key)
        prm.close()
