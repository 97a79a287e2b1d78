"""GPU tests of prover lanes (h2_lane_create / h2_lane_bind / h2_lane_destroy, halo2_b200.Lane): extra contexts on the
primary device that let independent provers on different host threads run at once.  Covers every rule of the ABI
(include/halo2_b200.h, "lanes"): the lifecycle and its errors, ownership of polynomials and IPA sessions, shared base sets,
per-lane settings, and that work run concurrently on several lanes gives exactly what the same work gives serially on the
primary context.  Concurrency here is ordinary parallel work whose results are checked; nothing tries to provoke a race."""
import ctypes
import hashlib
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests import prover_replay as R  # noqa: E402
from tests.abi_cases import _bind, _create, _destroy, _err, _lib, _run_parallel  # noqa: E402

SEED = 0x4C414E4553
MAX_LANES = 16          # include/halo2_b200.h


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


def _device() -> int:
    from halo2_b200 import lib as L
    return L._inited_device


def _plan():
    out = (ctypes.c_uint32 * 8)()
    assert _lib().h2_test_last_msm_plan(out) == 0, _err()
    return list(out)


def _affine(curve, xyz):
    return cref.bytes_to_affine(cref.jac_to_affine(curve, xyz))


def _in_thread(fn):
    """Runs fn() on a new host thread; returns its result or raises its exception."""
    box = {}

    def run():
        try:
            box["r"] = fn()
        except BaseException as e:  # noqa: BLE001
            box["e"] = e
    t = threading.Thread(target=run)
    t.start()
    t.join()
    if "e" in box:
        raise box["e"]
    return box.get("r")


# ---- lifecycle and errors ---------------------------------------------------------------------------------------------
def test_lifecycle_errors(eng):
    lib = _lib()
    dev = _device()
    # before h2_init
    assert lib.h2_shutdown() == 0
    h = ctypes.c_uint64(0)
    assert lib.h2_lane_create(ctypes.byref(h)) != 0 and "h2_init" in _err()
    assert lib.h2_init(dev) == 0
    # the maximum lane count
    lanes = [_create() for _ in range(MAX_LANES)]
    assert len(set(lanes)) == MAX_LANES and 0 not in lanes
    assert lib.h2_lane_create(ctypes.byref(h)) != 0 and "lanes" in _err()
    for x in lanes:
        assert _destroy(x) == 0, _err()
    # binding or destroying an unknown lane; a destroyed lane is unknown
    assert _bind(lanes[0]) != 0 and "unknown" in _err()
    assert _bind(0xDEADBEEF) != 0 and "unknown" in _err()
    assert _destroy(lanes[0]) != 0 and "unknown" in _err()
    assert _bind(0) == 0
    # destroying a lane another thread is bound to
    a = _create()
    bound, release = threading.Event(), threading.Event()

    def holder():
        assert _bind(a) == 0
        bound.set()
        release.wait(60)
        assert _bind(0) == 0
    t = threading.Thread(target=holder)
    t.start()
    assert bound.wait(60)
    assert _destroy(a) != 0 and "another thread" in _err()
    release.set()
    t.join()
    assert _destroy(a) == 0, _err()
    # the calling thread may destroy the lane it is bound to, and is back on the primary context afterwards
    b = _create()
    assert _bind(b) == 0
    p = eng.ResidentPoly("fp", 8, cref.gen_scalars("fp", SEED, 8))
    assert _destroy(b) == 0, _err()
    assert lib.h2_poly_download(p._h, None, ctypes.c_size_t(0), 0) != 0 and "unknown" in _err()   # freed with its lane
    p._h.value = 0
    q = eng.ResidentPoly("fp", 8)            # the primary works
    q.close()


def test_stale_handles_after_shutdown(eng):
    lib = _lib()
    dev = _device()
    a, b = _create(), _create()
    ready, go, done = threading.Event(), threading.Event(), {}

    def bound_thread():                      # bound to b across the shutdown: its calls fail until it binds again
        assert _bind(b) == 0
        ready.set()
        go.wait(60)
        h = ctypes.c_uint64(0)
        done["stale_rc"] = lib.h2_poly_alloc(0, ctypes.c_size_t(4), ctypes.byref(h))
        done["stale_err"] = _err()
        done["rebind"] = _bind(0)
        done["fresh_rc"] = lib.h2_poly_alloc(0, ctypes.c_size_t(4), ctypes.byref(h))
        lib.h2_poly_free(h)
    t = threading.Thread(target=bound_thread)
    t.start()
    assert ready.wait(60)
    assert _bind(a) == 0
    pa = eng.ResidentPoly("fp", 16, cref.gen_scalars("fp", SEED + 1, 16))
    old_poly = pa._h.value
    assert lib.h2_shutdown() == 0
    assert lib.h2_init(dev) == 0
    go.set()
    t.join()
    assert done["stale_rc"] != 0 and "h2_shutdown" in done["stale_err"]
    assert done["rebind"] == 0 and done["fresh_rc"] == 0
    # this thread was bound to a, which h2_shutdown destroyed: it is on the primary context again
    for h in (a, b):
        assert _bind(h) != 0 and "unknown" in _err()
        assert _destroy(h) != 0 and "unknown" in _err()
    fresh = [_create() for _ in range(2)]
    assert not set(fresh) & {a, b}
    assert _bind(fresh[0]) == 0
    assert lib.h2_poly_free(ctypes.c_uint64(old_poly)) != 0 and "unknown" in _err()
    assert _bind(0) == 0
    for h in fresh:
        assert _destroy(h) == 0, _err()
    pa._h.value = 0


# ---- ownership --------------------------------------------------------------------------------------------------------
def test_ownership_and_shared_bases(eng):
    lib = _lib()
    k, n = 6, 64
    pts = cref.gen_points("vesta", SEED + 2, n + 2)
    prm = eng.Params("vesta", k, pts[:n], pts[:n], pts[n:n + 1], u=pts[n + 1:])     # registered on the primary
    vals = cref.gen_scalars("fp", SEED + 3, n)
    want_commit = prm.commit_many_affine([vals], [eng.Blind(7)])
    a, b = _create(), _create()
    try:
        # lane A: a polynomial and an open IPA session over the primary's base set
        assert _bind(a) == 0
        pa = eng.ResidentPoly("fp", n, vals)
        sess = ctypes.c_uint64(0)
        x3 = eng.lib.fe_bytes(12345)
        assert lib.h2_ipa_begin_poly(prm._h_g, ctypes.c_uint32(k), pa._h, eng.lib.ptr(x3), 0, ctypes.byref(sess)) == 0, _err()
        got_a = prm.commit_resident_affine([pa], [eng.Blind(7)])
        # lane B and the primary do not know A's handles
        out = np.zeros((n, 32), dtype=np.uint8)
        lr = np.zeros((2, 64), dtype=np.uint8)
        zb = eng.lib.fe_bytes(3)
        for lane in (b, 0):
            assert _bind(lane) == 0
            assert lib.h2_poly_download(pa._h, eng.lib.ptr(out), ctypes.c_size_t(n), 0) != 0 and "unknown" in _err()
            assert lib.h2_poly_free(pa._h) != 0 and "unknown" in _err()
            assert lib.h2_ipa_round_affine(sess, eng.lib.ptr(zb), eng.lib.ptr(zb), eng.lib.ptr(zb), 0, eng.lib.ptr(lr)) != 0
            assert "unknown" in _err()
            assert lib.h2_ipa_finish(sess, 0, None) != 0 and "unknown" in _err()
        # the shared base set from lane B (and from the primary, above)
        assert _bind(b) == 0
        pb = eng.ResidentPoly("fp", n, vals)
        got_b = prm.commit_resident_affine([pb], [eng.Blind(7)])
        pb.close()
        assert (got_a == want_commit).all() and (got_b == want_commit).all()
        # releasing the set while A's session is open fails, from any lane
        assert lib.h2_bases_release(prm._h_g) != 0 and "IPA session" in _err()
        assert _bind(0) == 0
        assert lib.h2_bases_release(prm._h_g) != 0 and "IPA session" in _err()
        # lane A's objects are intact
        assert _bind(a) == 0
        assert (pa.download() == vals).all()
        assert lib.h2_ipa_round_affine(sess, eng.lib.ptr(zb), eng.lib.ptr(zb), eng.lib.ptr(zb), 0, eng.lib.ptr(lr)) == 0, _err()
        assert lib.h2_ipa_finish(sess, 0, None) == 0, _err()
        pa.close()
        assert _bind(0) == 0
        assert lib.h2_bases_release(prm._h_g) == 0, _err()   # after h2_ipa_finish
        prm._h_g.value = 0
    finally:
        _bind(0)
        prm.close()
        _destroy(a)
        _destroy(b)


def test_lane_destroy_ends_its_sessions(eng):
    """A lane destroyed with an IPA session open gives the base set back: it can be released afterwards."""
    lib = _lib()
    k, n = 5, 32
    pts = cref.gen_points("vesta", SEED + 4, n + 2)
    prm = eng.Params("vesta", k, pts[:n], pts[:n], pts[n:n + 1], u=pts[n + 1:])
    with eng.Lane():
        sess = ctypes.c_uint64(0)
        pp = cref.gen_scalars("fp", SEED + 5, n)
        assert lib.h2_ipa_begin(prm._h_g, ctypes.c_uint32(k), eng.lib.ptr(pp), eng.lib.ptr(eng.lib.fe_bytes(9)), 0, ctypes.byref(sess)) == 0
        assert lib.h2_bases_release(prm._h_g) != 0
    assert lib.h2_bases_release(prm._h_g) == 0, _err()
    prm._h_g.value = 0
    prm.close()


# ---- settings ---------------------------------------------------------------------------------------------------------
def test_settings_are_per_lane(eng):
    lib = _lib()
    k, n = 10, 1024
    pts = cref.gen_points("vesta", SEED + 6, n + 1)
    prm = eng.Params("vesta", k, pts[:n], pts[:n], pts[n:n + 1])
    sc = cref.gen_scalars("fp", SEED + 7, 3000)
    mp = cref.gen_points("vesta", SEED + 8, 3000)
    want = _affine("vesta", eng.best_multiexp(sc, mp, "vesta"))
    c0 = _plan()[1]
    c_over = 7 if c0 != 7 else 9
    a, b = _create(), _create()
    try:
        assert _bind(a) == 0
        assert lib.h2_set_window_bits(ctypes.c_uint32(c_over)) == 0
        assert lib.h2_test_set_fast_fixed(0) == 0
        assert _affine("vesta", eng.best_multiexp(sc, mp, "vesta")) == want
        assert _plan()[1] == c_over
        prm.commit_many_affine([sc[:n]], [eng.Blind(1)])
        assert _plan()[0] == 1 and _plan()[6] == 0                     # window table, full pass
        for lane in (b, 0):                                            # neither B nor the primary sees A's settings
            assert _bind(lane) == 0
            assert _affine("vesta", eng.best_multiexp(sc, mp, "vesta")) == want
            assert _plan()[1] == c0
            prm.commit_many_affine([sc[:n]], [eng.Blind(1)])
            assert _plan()[0] == 1 and _plan()[6] == 1                 # the fast pass
        # a new lane starts with the defaults, not with copies of the primary's settings
        assert _bind(0) == 0
        assert lib.h2_set_window_bits(ctypes.c_uint32(c_over)) == 0
        c = _create()
        assert _bind(c) == 0
        eng.best_multiexp(sc, mp, "vesta")
        assert _plan()[1] == c0
        assert _bind(0) == 0
        assert _destroy(c) == 0
    finally:
        _bind(0)
        lib.h2_set_window_bits(ctypes.c_uint32(0))
        _destroy(a)
        _destroy(b)
        prm.close()


# ---- concurrent parity ------------------------------------------------------------------------------------------------
K = 12
MSM_N = (1 << 18) + 77
ZETA = pow(5, (R.P_MOD - 1) // 3, R.P_MOD)


@pytest.fixture(scope="module")
def shared(eng):
    n = 1 << K
    pts = cref.gen_points("vesta", SEED + 10, n + 2)
    prm = eng.Params("vesta", K, pts[:n], pts[:n], pts[n:n + 1], u=pts[n + 1:])
    d = {"prm": prm, "msm_points": cref.gen_points("vesta", SEED + 11, MSM_N), "enc": eng.compress_points(pts[:300], "vesta")}
    yield d
    prm.close()


def _workload(eng, sh, seed):
    """One seeded pass over every kind of call a prover makes; returns what each call computed, as bytes (group elements
    as affine encodings)."""
    m, n = R.P_MOD, 1 << K
    prm = sh["prm"]
    out = {}
    live = []

    def rp(values=None, length=n):
        p = eng.ResidentPoly("fp", length, values)
        live.append(p)
        return p
    try:
        out["msm"] = repr(_affine("vesta", eng.best_multiexp(cref.gen_scalars("fp", seed, MSM_N), sh["msm_points"], "vesta")))
        cols = [cref.gen_scalars("fp", seed + 1 + i, n) for i in range(4)]
        out["commit"] = prm.commit_many_affine(cols, [eng.Blind(seed + i) for i in range(4)]).tobytes()
        out["commit_l"] = prm.commit_many_affine(cols[:2], [eng.Blind(1), eng.Blind(2)], lagrange=True).tobytes()
        dom = eng.EvaluationDomain("fp", R.DEGREE_J, K, ZETA)
        lag = rp(cols[0])
        coeff = dom.lagrange_to_coeff_resident(lag, out=rp())
        ext = dom.coeff_to_extended_resident(coeff, out=rp(length=dom.extended_len()))
        back = dom.extended_to_coeff_resident(ext, out=rp(length=n * dom.quotient_poly_degree))
        out["l2c"], out["c2e"], out["e2c"] = coeff.download().tobytes(), ext.download().tobytes(), back.download().tobytes()
        ev = eng.Evaluator(dom, "extended")
        ext2 = dom.coeff_to_extended_resident(dom.lagrange_to_coeff_resident(rp(cols[1]), out=rp()), out=rp(length=dom.extended_len()))
        A, B = ev.register_poly(ext), ev.register_poly(ext2)
        ast_out = ev.evaluate(A * B + B.with_rotation(1) * eng.Ast.constant_term(seed) - A, out=rp(length=dom.extended_len()))
        out["ast"] = ast_out.download().tobytes()
        ev.close()
        inv = eng.batch_invert_resident(rp(cols[2]))
        out["inv"] = inv.download().tobytes()
        out["prod"] = eng.running_product_resident(inv, init=seed, dst=rp()).download().tobytes()
        rnd = np.random.default_rng(seed)
        table = cref.gen_scalars("fp", seed + 20, n)
        usable = n - 7
        inputs = table[rnd.integers(0, usable, n)]
        pa, ps = eng.permute_expression_pair_resident(rp(inputs), rp(table), usable, rp(), rp())
        out["lookup"] = pa.download(usable).tobytes() + ps.download(usable).tobytes()
        x = int.from_bytes(hashlib.sha256(b"x%d" % seed).digest(), "little") % m
        out["eval"] = repr(eng.eval_polynomial_resident([coeff], [x]))
        out["kate"] = eng.kate_division_resident([coeff], [x], dst=[rp()])[0].download().tobytes()
        lr = [int.from_bytes(hashlib.sha256(b"lr%d-%d" % (seed, j)).digest(), "little") % m for j in range(2 * K)]

        def challenge(j, l_xy, r_xy):
            return int.from_bytes(hashlib.sha256(l_xy.tobytes() + r_xy.tobytes()).digest(), "little") % m or 1
        ls, rs, c = prm.ipa_rounds_transcript(coeff, x, seed + 3, challenge, lr[:K], lr[K:])
        out["ipa"] = ls.tobytes() + rs.tobytes() + repr(c).encode()
        msm = eng.MSM(prm)
        msm.add_compute_s(lr[:K], seed + 5)
        msm.add_to_w_scalar(seed + 6)
        msm.append_term(seed + 7, sh["msm_points"][0])
        out["verifier_msm"] = repr(_affine("vesta", msm.evaluate())) + repr(msm.eval())
        msm.close()
        out["decompress"] = eng.decompress_points(sh["enc"], "vesta").tobytes()
    finally:
        for p in live:
            p.close()
    return out


def test_concurrent_parity(eng, shared):
    seeds = [SEED + 100 * i for i in range(4)]
    want = [_workload(eng, shared, s) for s in seeds]            # serially, on the primary context
    assert want[0] != want[1]

    def on_lane(i):
        def go():
            got = []
            with eng.Lane():
                for _ in range(3):
                    got.append(_workload(eng, shared, seeds[i]))
            return got
        return go
    for i, got in enumerate(_run_parallel([on_lane(i) for i in range(4)])):
        for it in got:
            for key in want[i]:
                assert it[key] == want[i][key], (i, key)


def test_concurrent_replay(eng):
    k = 14
    n = 1 << k
    pts = cref.gen_points("vesta", SEED + 30, n + 2)
    g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    gl = eng.lagrange_generators("vesta", k, g)
    omega = pasta.omega_for_k("fp", k)
    inputs = [R.replay_inputs(cref, k, SEED + 40 + i) for i in range(4)]
    want = []
    arm = R.GpuArm(eng, k, g, gl, w, u)                          # serially, on the primary context
    try:
        for inp in inputs:
            want.append(R.run(arm, inp, k, omega))
            arm.free()
    finally:
        arm.close()
    assert len(set(want)) == 4

    def on_lane(i):
        def go():
            with eng.Lane():
                a = R.GpuArm(eng, k, g, gl, w, u)
                try:
                    return R.run(a, inputs[i], k, omega)
                finally:
                    a.close()
        return go
    got = _run_parallel([on_lane(i) for i in range(4)])
    assert got == want
    gv = R.GpuVerifierArm(eng, k, g, gl, w, u)
    try:
        for proof in got:
            assert R.verify(gv, proof, k, omega)
    finally:
        if gv._own:
            gv.params.close()


# ---- multi-GPU ----------------------------------------------------------------------------------------------------------
def test_multi_gpu_rejected_on_lane(eng):
    lib = _lib()
    sc = cref.gen_scalars("fp", SEED + 50, 64)
    pts = cref.gen_points("vesta", SEED + 51, 64)
    out = np.zeros(96, dtype=np.uint8)
    with eng.Lane():
        assert lib.h2_msm_multi_gpu(1, eng.lib.ptr(sc), eng.lib.ptr(pts), ctypes.c_size_t(64), 0, eng.lib.ptr(out)) != 0
        assert "lane" in _err()
        assert lib.h2_multi_init(1) != 0 and "lane" in _err()


def test_multi_bases_stale_after_shutdown(eng):
    lib = _lib()
    if lib.h2_device_count() < 2:
        pytest.skip("needs 2 devices")
    dev = _device()
    pts = cref.gen_points("vesta", SEED + 52, 100)
    h = ctypes.c_uint64(0)
    assert lib.h2_multi_init(2) == 0, _err()
    assert lib.h2_multi_bases_register(1, eng.lib.ptr(pts), ctypes.c_size_t(100), 0, ctypes.byref(h)) == 0, _err()
    assert lib.h2_shutdown() == 0
    assert lib.h2_init(dev) == 0
    assert lib.h2_multi_init(2) == 0, _err()
    sc = cref.gen_scalars("fp", SEED + 53, 100)
    out = np.zeros(96, dtype=np.uint8)
    assert lib.h2_msm_multi_registered(h, eng.lib.ptr(sc), ctypes.c_size_t(100), 0, eng.lib.ptr(out)) != 0 and "unknown" in _err()
    assert lib.h2_multi_bases_release(h) != 0 and "unknown" in _err()
