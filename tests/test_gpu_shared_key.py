"""GPU tests of shared polynomials (h2_poly_share, ResidentPoly.share, ProvingKey.share): one read-only proving key that
every prover lane and the primary context read.

- every entry point that reads a polynomial gives, with a shared handle on another lane and on the primary context, the
  bytes it gives with a private copy there (an IPA opening from h2_ipa_begin_poly included);
- every entry point that writes a polynomial refuses a shared handle, names itself and says "shared", on the owner lane,
  another lane and the primary context, and the polynomial is unchanged;
- sharing is all or nothing, re-sharing is a no-op and another lane's handle cannot be shared;
- a shared polynomial outlives the lane that shared it, is freed from any lane (then unknown everywhere), its free waits
  for reads another lane queued, and h2_shutdown frees it;
- at k = 14 the benchmark circuit's key, built once and shared, proves on 4 lanes at once byte for byte like a private key,
  the proofs verify, and the key is unchanged -- also when the lane that built it is gone."""
import ctypes
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests import bench_circuit as BC  # noqa: E402
from tests import plonk_api_circuit as circ  # noqa: E402
from tests.abi_cases import _bind, _create, _destroy, _err, _lib, _run_parallel  # noqa: E402
from tests.bench_circuit import bench_copies  # noqa: E402
from tests.plonk_api_circuit import ZETA  # noqa: E402
from tests.plonk_prover import prover_pk_bytes, prover_pk_dict  # noqa: E402
from tests.plonk_verifier import scalar_delta  # noqa: E402

SEED = 0x5348415245
K, N = 10, 1 << 10
M = pasta.P_MOD
DEGREE = 5                                                          # extended cosets of 4 n, like the benchmark circuit


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


@pytest.fixture(scope="module")
def prm(eng):
    pts = cref.gen_points("vesta", SEED, N + 2)
    p = eng.Params("vesta", K, pts[:N], eng.lagrange_generators("vesta", K, pts[:N]), pts[N:N + 1], u=pts[N + 1:])
    yield p
    p.close()


def _dom(eng):
    return eng.EvaluationDomain("fp", DEGREE, K, ZETA)


def _fe(x):
    from halo2_b200 import lib as L
    return L.ptr(L.fe_bytes(int(x) % M))


def _h(p) -> ctypes.c_uint64:
    return ctypes.c_uint64(p if isinstance(p, int) else p._h.value)


def _known(h) -> bool:
    """The calling thread's context can read handle h."""
    return _lib().h2_poly_download(_h(h), None, ctypes.c_size_t(0), 0) == 0


def _build_set(eng):
    """On the calling context: Lagrange values, their coefficients and extended coset, and a lookup input / table pair."""
    dom = _dom(eng)
    lag = eng.ResidentPoly("fp", N, cref.gen_scalars("fp", SEED + 1, N))
    coeff = dom.lagrange_to_coeff_resident(lag, out=eng.ResidentPoly("fp", N))
    ext = dom.coeff_to_extended_resident(coeff)
    table = cref.gen_scalars("fp", SEED + 2, N)
    inputs = table[np.random.default_rng(SEED).integers(0, N - 7, N)]
    return {"lag": lag, "coeff": coeff, "ext": ext, "table": eng.ResidentPoly("fp", N, table), "input": eng.ResidentPoly("fp", N, inputs)}


def _reads(eng, prm, P):
    """Every entry point that reads a polynomial, over the polynomials of P; what each computed, as bytes."""
    lib = _lib()
    dom = _dom(eng)
    live, out = [], {}

    def rp(length=N, vals=None):
        p = eng.ResidentPoly("fp", length, vals)
        live.append(p)
        return p
    x = int.from_bytes(hashlib.sha256(b"x").digest(), "little") % M
    try:
        out["download"] = b"".join(P[k].download().tobytes() for k in sorted(P))
        out["copy"] = rp().copy_from(P["lag"], N - 3, src_off=3, dst_off=1).download().tobytes()
        out["l2c"] = dom.lagrange_to_coeff_resident(P["lag"], out=rp()).download().tobytes()
        out["c2e"] = dom.coeff_to_extended_resident(P["coeff"], out=rp(dom.extended_len())).download().tobytes()
        out["e2c"] = dom.extended_to_coeff_resident(P["ext"], out=rp(N * dom.quotient_poly_degree)).download().tobytes()
        out["prod"] = eng.running_product_resident(P["lag"], init=7, dst=rp()).download().tobytes()
        out["kate"] = eng.kate_division_resident([P["coeff"]], [x], dst=[rp()])[0].download().tobytes()
        d = rp(vals=cref.gen_scalars("fp", SEED + 3, N))
        assert lib.h2_poly_scale_add(d._h, _fe(3), P["lag"]._h, _fe(5), ctypes.c_size_t(N), 0) == 0, _err()
        out["scale_add"] = d.download().tobytes()
        ev = eng.Evaluator(dom, "extended")
        A, B = ev.register_poly(P["ext"]), ev.register_poly(rp(dom.extended_len(), P["ext"].download()))
        out["ast"] = ev.evaluate(A * A + A.with_rotation(1) * eng.Ast.constant_term(11) - B, out=rp(dom.extended_len())).download().tobytes()
        ev.close()
        out["eval"] = repr(eng.eval_polynomial_resident([P["coeff"], P["lag"]], [x, x + 1]))
        out["inner"] = repr(eng.inner_product_resident([P["coeff"]], [P["lag"]]))
        pa, ps = eng.permute_expression_pair_resident(P["input"], P["table"], N - 7, rp(), rp())
        out["lookup"] = pa.download(N - 7).tobytes() + ps.download(N - 7).tobytes()
        # Jacobian results: only the group element is defined, so compare affine encodings
        out["commit"] = b"".join(cref.jac_to_affine("vesta", x).tobytes()
                                 for x in prm.commit_resident([P["coeff"], P["lag"]], [eng.Blind(9), eng.Blind(10)]))
        out["commit_affine"] = prm.commit_resident_affine([P["lag"]], [eng.Blind(9)], lagrange=True).tobytes()
        lr = [int.from_bytes(hashlib.sha256(b"lr%d" % j).digest(), "little") % M for j in range(2 * K)]

        def challenge(j, l_xy, r_xy):
            return int.from_bytes(hashlib.sha256(l_xy.tobytes() + r_xy.tobytes()).digest(), "little") % M or 1
        ls, rs, c = prm.ipa_rounds_transcript(P["coeff"], x, 12345, challenge, lr[:K], lr[K:])
        out["ipa"] = ls.tobytes() + rs.tobytes() + repr(c).encode()
    finally:
        for p in live:
            p.close()
    return out


# ---- 1. reads -----------------------------------------------------------------------------------------------------------
def test_reads_everywhere(eng, prm):
    a, b = _create(), _create()
    S = None
    try:
        assert _bind(a) == 0
        S = _build_set(eng)
        want_values = {k: p.download().tobytes() for k, p in S.items()}
        eng.share_resident(list(S.values()))
        assert all(p.shared for p in S.values())
        for lane in (b, 0):
            assert _bind(lane) == 0
            assert {k: p.download().tobytes() for k, p in S.items()} == want_values
            P = {k: eng.ResidentPoly("fp", p.len, p.download()) for k, p in S.items()}    # private copies on this context
            try:
                assert _reads(eng, prm, S) == _reads(eng, prm, P), lane
            finally:
                for p in P.values():
                    p.close()
    finally:
        _bind(0)
        if S:
            for p in S.values():
                p.close()
        _destroy(a)
        _destroy(b)


# ---- 2. writes ----------------------------------------------------------------------------------------------------------
def _write_calls(eng, S, P):
    """(entry point, call) for every entry point that writes a polynomial, each with a shared output from S and private
    inputs from P."""
    lib = _lib()
    dom = _dom(eng)
    vals = np.zeros((N, 32), dtype=np.uint8)
    t = np.ascontiguousarray(np.stack([eng.lib.fe_bytes(v) for v in dom.t_evaluations]))
    u = np.ascontiguousarray(np.stack([eng.lib.fe_bytes(j + 2) for j in range(K)]))
    pts = np.ascontiguousarray(np.stack([eng.lib.fe_bytes(5)]))
    ident = np.stack(np.meshgrid(np.arange(1), np.arange(N), indexing="ij"), axis=-1).astype(np.uint32)
    copies = np.array([[0, 1, 0, 2]], dtype=np.uint32)
    arr = lambda *ps: (ctypes.c_uint64 * len(ps))(*[p._h.value for p in ps])
    code = np.array([[0, 0, 0, 0]], dtype=np.uint32)                    # POLY 0
    s_lag, s_coeff, s_ext = S["lag"], S["coeff"], S["ext"]
    return [
        ("h2_poly_upload", lambda: lib.h2_poly_upload(s_lag._h, eng.lib.ptr(vals), ctypes.c_size_t(N), 0)),
        ("h2_poly_add_at", lambda: lib.h2_poly_add_at(s_lag._h, ctypes.c_size_t(0), _fe(1), 0)),
        ("h2_poly_batch_invert", lambda: lib.h2_poly_batch_invert(s_lag._h, ctypes.c_size_t(N))),
        ("h2_poly_divide_by_vanishing", lambda: lib.h2_poly_divide_by_vanishing(s_ext._h, ctypes.c_uint32(dom.extended_k), eng.lib.ptr(t),
                                                                                 ctypes.c_uint32(t.shape[0]), 0)),
        ("h2_poly_compute_s", lambda: lib.h2_poly_compute_s(s_lag._h, eng.lib.ptr(u), ctypes.c_uint32(K), _fe(1), 0, 0)),
        ("h2_poly_copy", lambda: lib.h2_poly_copy(s_lag._h, ctypes.c_size_t(0), P["lag"]._h, ctypes.c_size_t(0), ctypes.c_size_t(4))),
        ("h2_poly_lagrange_to_coeff", lambda: lib.h2_poly_lagrange_to_coeff(s_coeff._h, P["lag"]._h, ctypes.c_uint32(K), _fe(dom.omega_inv),
                                                                             _fe(dom.ifft_divisor), 0)),
        ("h2_poly_lagrange_to_coeff", lambda: lib.h2_poly_lagrange_to_coeff(s_lag._h, s_lag._h, ctypes.c_uint32(K), _fe(dom.omega_inv),
                                                                             _fe(dom.ifft_divisor), 0)),      # in place
        ("h2_poly_coeff_to_extended", lambda: lib.h2_poly_coeff_to_extended(s_ext._h, P["coeff"]._h, ctypes.c_uint32(K), ctypes.c_uint32(dom.extended_k),
                                                                             _fe(dom.g_coset), _fe(dom.extended_omega), 0)),
        ("h2_poly_extended_to_coeff", lambda: lib.h2_poly_extended_to_coeff(s_ext._h, P["ext"]._h, ctypes.c_uint32(dom.extended_k),
                                                                             _fe(dom.extended_omega_inv), _fe(dom.extended_ifft_divisor), _fe(dom.g_coset),
                                                                             ctypes.c_size_t(N), 0)),
        ("h2_poly_running_product", lambda: lib.h2_poly_running_product(s_lag._h, P["lag"]._h, ctypes.c_size_t(N), _fe(1), 0)),
        ("h2_poly_kate_division", lambda: lib.h2_poly_kate_division(arr(s_lag), arr(P["coeff"]), ctypes.c_size_t(1), ctypes.c_size_t(N),
                                                                     eng.lib.ptr(pts), 0)),
        ("h2_poly_scale_add", lambda: lib.h2_poly_scale_add(s_lag._h, _fe(2), P["lag"]._h, _fe(3), ctypes.c_size_t(N), 0)),
        ("h2_poly_eval_ast", lambda: lib.h2_poly_eval_ast(s_lag._h, arr(P["lag"]), ctypes.c_size_t(1), ctypes.c_uint32(K),
                                                           code.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(1), None, ctypes.c_size_t(0),
                                                           None, None, 0)),
        ("h2_poly_lookup_permute", lambda: lib.h2_poly_lookup_permute(P["input"]._h, P["table"]._h, ctypes.c_size_t(N - 7), s_lag._h, P["coeff"]._h)),
        ("h2_poly_lookup_permute", lambda: lib.h2_poly_lookup_permute(P["input"]._h, P["table"]._h, ctypes.c_size_t(N - 7), P["coeff"]._h, s_lag._h)),
        ("h2_poly_permutation_sigma", lambda: lib.h2_poly_permutation_sigma(arr(s_lag), ctypes.c_size_t(1), ctypes.c_uint32(K),
                                                                             ident.ctypes.data_as(ctypes.c_void_p), _fe(dom.omega), _fe(scalar_delta(M)), 0)),
        ("h2_poly_permutation_sigma_copies", lambda: lib.h2_poly_permutation_sigma_copies(arr(s_lag), ctypes.c_size_t(1), ctypes.c_uint32(K),
                                                                                           copies.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(1),
                                                                                           _fe(dom.omega), _fe(scalar_delta(M)), 0)),
    ]


def test_writes_refused(eng):
    a, b = _create(), _create()
    S = None
    try:
        assert _bind(a) == 0
        S = _build_set(eng)
        want = {k: p.download().tobytes() for k, p in S.items()}
        eng.share_resident(list(S.values()))
        for lane in (a, b, 0):
            assert _bind(lane) == 0
            P = _build_set(eng)
            try:
                calls = _write_calls(eng, S, P)
                assert len(calls) == 18
                for name, call in calls:
                    assert call() != 0, (lane, name)
                    assert "shared" in _err() and _err().startswith(name), (lane, name, _err())
                assert {k: p.download().tobytes() for k, p in S.items()} == want, lane
            finally:
                for p in P.values():
                    p.close()
    finally:
        _bind(0)
        if S:
            for p in S.values():
                p.close()
        _destroy(a)
        _destroy(b)


# ---- 3. sharing rules ---------------------------------------------------------------------------------------------------
def test_sharing_rules(eng):
    lib = _lib()
    a, b = _create(), _create()
    try:
        assert _bind(b) == 0
        foreign = eng.ResidentPoly("fp", 8)
        assert _bind(a) == 0
        p, q = eng.ResidentPoly("fp", 8, cref.gen_scalars("fp", SEED + 4, 8)), eng.ResidentPoly("fp", 8)
        assert lib.h2_poly_share(None, ctypes.c_size_t(0)) == 0, _err()
        # all or nothing: an unknown handle, or another lane's, fails the call and p stays private
        for bad in (0xDEADBEEF, foreign._h.value):
            hs = (ctypes.c_uint64 * 2)(p._h.value, bad)
            assert lib.h2_poly_share(hs, ctypes.c_size_t(2)) != 0 and "unknown" in _err()
        with pytest.raises(eng.H2Error, match="unknown"):
            eng.share_resident([p, foreign])
        assert not p.shared
        assert _bind(b) == 0
        assert not _known(p)
        assert _bind(a) == 0
        assert p.add_at(0, 1) is None                                   # still writable on its own lane
        # sharing, then again (a no-op), and listed twice with a private one
        p.share()
        assert p.shared
        hs = (ctypes.c_uint64 * 3)(p._h.value, q._h.value, p._h.value)
        assert lib.h2_poly_share(hs, ctypes.c_size_t(3)) == 0, _err()
        assert lib.h2_poly_share(hs, ctypes.c_size_t(3)) == 0, _err()
        for lane in (b, 0):
            assert _bind(lane) == 0
            assert _known(p) and _known(q)
            assert not _known(foreign) or lane == b
        assert _bind(b) == 0
        foreign.close()
        assert _bind(a) == 0
        p.close()
        q.close()
    finally:
        _bind(0)
        _destroy(a)
        _destroy(b)


def test_share_before_init_fails(eng):
    lib = _lib()
    from halo2_b200 import lib as L
    dev = L._inited_device
    assert lib.h2_shutdown() == 0
    try:
        hs = (ctypes.c_uint64 * 1)(1)
        assert lib.h2_poly_share(hs, ctypes.c_size_t(1)) != 0 and "h2_init" in _err()
    finally:
        assert lib.h2_init(dev) == 0


# ---- 4. lifetime --------------------------------------------------------------------------------------------------------
def test_outlives_its_lane_and_frees_from_another(eng):
    lib = _lib()
    a, b = _create(), _create()
    try:
        assert _bind(a) == 0
        vals = cref.gen_scalars("fp", SEED + 5, 64)
        p = eng.ResidentPoly("fp", 64, vals).share()
        priv = eng.ResidentPoly("fp", 64, vals)
        h = p._h.value
        assert _bind(0) == 0
        assert _destroy(a) == 0, _err()                                  # frees the lane's own polynomials only
        a = None
        assert (p.download() == vals).all()
        assert _bind(b) == 0
        assert (p.download() == vals).all()
        assert not _known(priv)
        priv._h.value = 0
        assert lib.h2_poly_free(ctypes.c_uint64(h)) == 0, _err()         # freed from lane B
        for lane in (b, 0):
            assert _bind(lane) == 0
            assert not _known(h) and "unknown" in _err()
        assert lib.h2_poly_free(ctypes.c_uint64(h)) != 0 and "unknown" in _err()
        p._h.value = 0
    finally:
        _bind(0)
        if a:
            _destroy(a)
        _destroy(b)


def test_free_waits_for_queued_reads(eng):
    """Lane B queues an Ast over shared inputs into its own output and does not synchronise; lane A frees the inputs; B's
    result is still the one computed before, and the inputs are unknown afterwards.  The free ends in cudaFree, which also
    waits for the device, so this checks the outcome, not that the free's own device synchronisation is the step that
    waited; no call is reading the inputs at the moment of the free, so the wait for users is not exercised here."""
    lib = _lib()
    dom = eng.EvaluationDomain("fp", DEGREE, 18, ZETA)                # 2^20 extended values per operand
    a, b = _create(), _create()
    try:
        assert _bind(a) == 0
        ins = []
        for i in range(3):
            co = eng.ResidentPoly("fp", dom.n, cref.gen_scalars("fp", SEED + 10 + i, dom.n))
            ins.append(dom.coeff_to_extended_resident(co))
            co.close()
        eng.share_resident(ins)
        assert _bind(b) == 0
        ev = eng.Evaluator(dom, "extended")
        X, Y, Z = (ev.register_poly(p) for p in ins)
        ast = (X * Y + Z.with_rotation(1)) * (X + Z) * (Y * Y + X.with_rotation(1))
        want = ev.evaluate(ast).download()                               # synchronous
        out = eng.ResidentPoly("fp", dom.extended_len())
        ev.evaluate(ast, out=out)                                        # queued, not synchronised
        assert _bind(a) == 0
        handles = [p._h.value for p in ins]
        for p in ins:
            p.close()
        assert _bind(b) == 0
        assert (out.download() == want).all()
        assert not any(_known(h) for h in handles)
        out.close()
    finally:
        _bind(0)
        _destroy(a)
        _destroy(b)


def test_shutdown_frees_shared(eng):
    lib = _lib()
    from halo2_b200 import lib as L
    dev = L._inited_device
    a = _create()
    assert _bind(a) == 0
    p = eng.ResidentPoly("fp", 16, cref.gen_scalars("fp", SEED + 6, 16)).share()
    assert _bind(0) == 0
    q = eng.ResidentPoly("fp", 16).share()
    old = [p._h.value, q._h.value]
    assert lib.h2_shutdown() == 0
    assert lib.h2_init(dev) == 0
    for h in old:
        assert not _known(h) and "unknown" in _err()
        assert lib.h2_poly_free(ctypes.c_uint64(h)) != 0 and "unknown" in _err()
    fresh = eng.ResidentPoly("fp", 16)
    assert fresh._h.value not in old
    fresh.close()
    p._h.value = q._h.value = 0


# ---- 5. end to end ------------------------------------------------------------------------------------------------------
def test_shared_key_proves_on_four_lanes_k14(eng):
    from tests import multiopen_cases as MC
    from tests import plonk_prover as PP
    from tests import plonk_verifier as PV
    from tests import prover_replay as R
    k = 14
    n = 1 << k
    delta = scalar_delta(M)
    pts = cref.gen_points("vesta", 99, n + 2)
    g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    prm14 = eng.Params("vesta", k, g, eng.lagrange_generators("vesta", k, g), w, u=u)
    D = eng.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
    fixed, _, adv = BC.columns(k, M, D.omega, delta, circ.A_SMALL * ZETA % M)
    ab = [cref.ints_to_bytes(c_) for c_ in adv]
    cc = eng.CopyConstraints(n, 3)
    cc.extend(np.array(list(bench_copies(k)), dtype=np.uint32))
    seeds = [[20 + 2 * i, 21 + 2 * i] for i in range(4)]
    keys = []

    def prove(pk, seed):
        T = R.Blake2bTranscript(M)
        PP.create_proof_engine(eng, prm14, vk, None, None, [ab], [[]], MC.SeededRng("fp", seed, True), T, ZETA, delta, pk=prover_pk_dict(pk))
        return bytes(T.proof)

    def on_lanes(pk):
        def lane(i):
            def go():
                with eng.Lane():
                    return [prove(pk, s) for s in seeds[i]]
            return go
        return _run_parallel([lane(i) for i in range(4)])
    try:
        fc, pc = eng.keygen_vk(prm14, D, fixed, cc, delta)
        A = cref.bytes_to_affine
        vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, pasta.Q_MOD, M, D.omega, [A(x) for x in fc], [A(x) for x in pc]))
        private = eng.keygen_pk(prm14, D, fixed, cc, delta, BC.BLINDING_FACTORS)
        keys.append(private)
        want = [[prove(private, s) for s in ss] for ss in seeds]          # serially, private key, primary context
        assert len({p for ps in want for p in ps}) == 8
        key_bytes = prover_pk_bytes(private)
        # the key built on the primary context and shared
        pk = eng.keygen_pk(prm14, D, fixed, cc, delta, BC.BLINDING_FACTORS)
        keys.append(pk)
        assert pk.share() is pk and all(p.shared for p in pk._all())
        assert on_lanes(pk) == want
        assert prover_pk_bytes(pk) == key_bytes
        arm = PV.EngineArm(eng, "vesta", k, params=prm14)
        try:
            assert all(PV.verify_proof(arm, vk, p, [[]], delta) for ps in want for p in ps)
            bad = bytearray(want[1][0])
            bad[len(bad) // 2] ^= 4
            assert not PV.verify_proof(arm, vk, bytes(bad), [[]], delta)
        finally:
            arm.close()
        # the key built on a lane, shared there, and the lane destroyed before the proofs start
        lane = _create()
        assert _bind(lane) == 0
        try:
            pk2 = eng.keygen_pk(prm14, D, fixed, cc, delta, BC.BLINDING_FACTORS).share()
            keys.append(pk2)
        finally:
            assert _bind(0) == 0
            assert _destroy(lane) == 0, _err()
        assert on_lanes(pk2) == want
        assert prover_pk_bytes(pk2) == key_bytes
    finally:
        for key in keys:
            key.close()
        prm14.close()
