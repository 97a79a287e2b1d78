"""GPU tests added in round 2: the single-process multi-GPU entry points (run on however many devices the box has --
one device exercises the whole code path with G = 1), staged transfers from pageable memory, the concurrent-caller pattern
of BatchVerifier, and the round-1 advisor findings."""
import ctypes
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402

SEED = 0x48414C4F32


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


def _affine(curve, xyz):
    return cref.bytes_to_affine(cref.jac_to_affine(curve, xyz))


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_msm_multi_gpu_single_process(eng, curve):
    """h2_msm_multi_gpu / h2_msm_multi_registered vs the oracle, for every device count the box offers, incl. n < G,
    n = 0 and ragged shards.  SURVEY.md section 8(e): the result is the same group element whatever G is."""
    from halo2_b200 import lib as L, parallel
    ndev = L.load().h2_device_count()
    c = pasta.CURVES[curve]
    n = 3001
    kb = cref.gen_scalars(c.scalar, SEED + 31, n)
    pb = cref.gen_points(curve, SEED + 32, n)
    want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
    for g in sorted({1, min(2, ndev), ndev}):
        assert parallel.multi_init(g) == g
        assert _affine(curve, parallel.best_multiexp_multi_gpu(kb, pb, curve)) == want
        for m in (0, 1, g - 1 if g > 1 else 2, 2 * g + 1):
            w = cref.bytes_to_affine(cref.best_multiexp(curve, kb[:m], pb[:m])) if m else None
            assert _affine(curve, parallel.best_multiexp_multi_gpu(kb[:m], pb[:m], curve)) == w
        mb = parallel.MultiGpuBases(pb, curve)
        assert _affine(curve, mb.msm(kb)) == want
        k2 = cref.gen_scalars(c.scalar, SEED + 33, n)
        assert _affine(curve, mb.msm(k2)) == cref.bytes_to_affine(cref.best_multiexp(curve, k2, pb))
        mb.close()
    # a larger problem takes the chunked, threaded upload path on every device
    n = 1 << 17
    kb = cref.gen_scalars(c.scalar, SEED + 34, n)
    pb = cref.gen_points(curve, SEED + 35, n)
    assert _affine(curve, parallel.best_multiexp_multi_gpu(kb, pb, curve)) == _affine(curve, eng.best_multiexp(kb, pb, curve))
    assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))


def test_staged_and_plain_transfers_agree(eng):
    """Pageable numpy buffers go through the pinned staging ring (MSM inputs on an uploader thread, NTT in and out);
    results must equal the plain cudaMemcpyAsync path and the oracle."""
    from halo2_b200 import lib as L
    lib = L.init()
    c = pasta.PALLAS
    n = (1 << 18) + 77                       # > 4 MiB of bases: uploader thread; 3 chunks
    kb = cref.gen_scalars(c.scalar, SEED + 41, n)
    pb = cref.gen_points("pallas", SEED + 42, n)
    outs = []
    for on in (1, 0, 1):
        L.check(lib.h2_test_set_staging(on))
        outs.append(_affine("pallas", eng.best_multiexp(kb, pb, "pallas")))
    L.check(lib.h2_test_set_staging(1))
    assert outs[0] == outs[1] == outs[2] == cref.bytes_to_affine(cref.best_multiexp("pallas", kb, pb))
    log_n = 19                               # 16 MiB each way: two ring slots in flight
    a = cref.gen_scalars("fq", SEED + 43, 1 << log_n)
    w = pasta.omega_for_k("fq", log_n)
    want = cref.best_fft("fq", a, w, log_n)
    for on in (1, 0):
        L.check(lib.h2_test_set_staging(on))
        got = a.copy()
        eng.best_fft(got, w, log_n, "fq")
        assert (got == want).all()
    L.check(lib.h2_test_set_staging(1))


def test_concurrent_callers(eng):
    """BatchVerifier::finalize calls the MSM from many rayon workers at once (plonk/verifier/batch.rs:97-110 ->
    verifier.rs:100): exported functions must be thread-safe.  8 host threads x mixed calls, each result vs the oracle."""
    c = pasta.VESTA
    k = 8
    n = 1 << k
    bases = cref.gen_points("vesta", SEED + 51, n + 2)
    prm = eng.Params("vesta", k, bases[:n], bases[:n], bases[n:n + 1], u=bases[n + 1:])
    polys = [cref.gen_scalars(c.scalar, SEED + 60 + i, n) for i in range(8)]
    want_commit = [cref.bytes_to_affine(cref.best_multiexp("vesta", np.concatenate([p, cref.ints_to_bytes([i + 1])]), bases[:n + 1]))
                   for i, p in enumerate(polys)]
    pts = cref.gen_points("vesta", SEED + 52, 777)
    ks = [cref.gen_scalars(c.scalar, SEED + 70 + i, 777) for i in range(8)]
    want_msm = [cref.bytes_to_affine(cref.best_multiexp("vesta", kk, pts)) for kk in ks]
    w = pasta.omega_for_k("fp", 10)
    ntt_in = [cref.gen_scalars("fp", SEED + 80 + i, 1 << 10) for i in range(8)]
    want_ntt = [cref.best_fft("fp", a, w, 10) for a in ntt_in]
    errs = []

    def worker(i):
        try:
            for rep in range(6):
                assert _affine("vesta", prm.commit_lagrange(polys[i], eng.Blind(i + 1))) == want_commit[i]
                assert _affine("vesta", eng.best_multiexp(ks[i], pts, "vesta")) == want_msm[i]
                a = ntt_in[i].copy()
                eng.best_fft(a, w, 10, "fp")
                assert (a == want_ntt[i]).all()
        except Exception as e:  # noqa: BLE001
            errs.append((i, repr(e)))

    th = [threading.Thread(target=worker, args=(i,)) for i in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    prm.close()


def test_advisor_findings_round1(eng):
    """ADVICE.md round 1: (a) n == 0 batched commits return `batch` identities; (b) a fresh ResidentPoly is zero-filled
    and kate_division writes the zero the reference pushes behind the quotient; (c) kate_division rejects a quotient that
    aliases ANY dividend of the batch or appears twice; (d) an IPA-capable base set (g ++ [w, u]) commits."""
    from halo2_b200 import lib as L
    lib = L.init()
    c = pasta.VESTA
    k = 5
    n = 1 << k
    bases = cref.gen_points("vesta", SEED + 91, n + 2)
    prm = eng.Params("vesta", k, bases[:n], bases[:n], bases[n:n + 1], u=bases[n + 1:])
    # (a) three empty scalar vectors, no blinds, against the resident table
    out = np.full((3, 96), 0xAB, dtype=np.uint8)
    L.check(lib.h2_msm_registered_batch(prm._h_g, None, ctypes.c_size_t(0), None, ctypes.c_size_t(3), L.REPR_CANONICAL, L.ptr(out)))
    assert all(_affine("vesta", o) is None for o in out)
    # (b)
    p = eng.ResidentPoly("fp", n)
    assert (p.download() == 0).all()
    a = pasta.gen_scalars("fp", SEED + 92, n)
    src = eng.ResidentPoly("fp", n)
    src.upload(cref.ints_to_bytes(a))
    dst = eng.ResidentPoly("fp", n)
    dst.upload(cref.ints_to_bytes([7] * n))                        # stale contents
    eng.kate_division_resident([src], [12345], dst=[dst])
    got = cref.bytes_to_ints(dst.download())
    assert got[:n - 1] == pasta.kate_division("fp", a, 12345) and got[n - 1] == 0
    # committing n coefficients of the quotient therefore equals the reference's kate_division + push(ZERO) + commit
    want = pasta.to_affine(c, pasta.best_multiexp(c, got[:n - 1] + [0, 9], [cref.bytes_to_affine(x) for x in bases[:n + 1]]))
    assert _affine("vesta", prm.commit_resident([dst], [eng.Blind(9)])[0]) == want
    # (c)
    other = eng.ResidentPoly("fp", n)
    other.upload(cref.ints_to_bytes(a))
    with pytest.raises(eng.H2Error):
        eng.kate_division_resident([src, dst], [3, 4], dst=[dst, other])      # dst[0] is src[1]
    with pytest.raises(eng.H2Error):
        eng.kate_division_resident([src, other], [3, 4], dst=[dst, dst])      # duplicate quotient handle
    # (d) commit over a set that also holds u (n + 2 bases): the blind rides on bases[n]
    poly = cref.gen_scalars(c.scalar, SEED + 93, n)
    assert _affine("vesta", prm.commit(poly, eng.Blind(3))) == cref.bytes_to_affine(
        cref.best_multiexp("vesta", np.concatenate([poly, cref.ints_to_bytes([3])]), bases[:n + 1]))
    for q in (p, src, dst, other):
        q.close()
    prm.close()


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_ntt_tma_pass_kernel(eng, field):
    """The bulk-copy (TMA) form of the NTT passes (cp.async.bulk + mbarrier, persistent CTAs, dense shared-memory tiles; opt-in
    via h2_test_set_ntt_tma) against the oracle: plain transforms with a true root and a random omega, ifft, coeff_to_extended
    (zero padding + zeta scaling inside the first step), extended_to_coeff (un-scaling + truncation in the last step)."""
    from halo2_b200 import lib as L
    lib = L.init()
    L.check(lib.h2_test_set_ntt_tma(1))
    try:
        for log_n in (11, 13, 16, 18):
            a = cref.gen_scalars(field, 300 + log_n, 1 << log_n)
            for w in (pasta.omega_for_k(field, log_n), pasta.gen_scalars(field, 79, 1)[0]):
                got = a.copy()
                eng.best_fft(got, w, log_n, field)
                assert (got == cref.best_fft(field, a, w, log_n)).all(), (field, log_n)
        for (j, k) in ((4, 10), (5, 12), (5, 14)):
            d = pasta.EvaluationDomain(field, j, k)
            dom = eng.EvaluationDomain(field, j, k, d.g_coset)
            a = cref.gen_scalars(field, 7, 1 << k)
            co = cref.ifft(field, a, d.omega_inv, k, d.ifft_divisor)
            assert (dom.lagrange_to_coeff(a) == co).all()
            ext = cref.coeff_to_extended(field, co, k, d.extended_k, d.g_coset, d.extended_omega)
            assert (dom.coeff_to_extended(co) == ext).all()
            back = cref.extended_to_coeff(field, ext, d.extended_k, d.extended_omega_inv, d.extended_ifft_divisor, d.g_coset, (1 << k) * (j - 1))
            assert (dom.extended_to_coeff(ext) == back).all()
    finally:
        L.check(lib.h2_test_set_ntt_tma(0))


@pytest.mark.parametrize("curve", ["pallas", "vesta"])
def test_batched_affine_accumulation(eng, curve):
    """Large one-shot MSMs pair up their buckets' points in affine coordinates first (msm.cuh K4a: halving rounds with a
    shared inversion, then the XYZZ chain).  Every round count and batch size gives the oracle's point -- on random inputs
    and on inputs whose buckets are full of P + P, P + (-P) and identity operands (repeated / negated / missing bases under
    repeated scalars), where the batch runs on substitute denominators."""
    from halo2_b200 import lib as L
    lib = L.init()
    c = pasta.CURVES[curve]
    n = (1 << 17) + 5                          # 2 x 8 x n > 2^20 references: the throughput path
    kb = cref.gen_scalars(c.scalar, SEED + 91, n)
    pb = cref.gen_points(curve, SEED + 92, n)
    want = cref.bytes_to_affine(cref.best_multiexp(curve, kb, pb))
    # degenerate variant: every (scalar, base) pair appears twice -- the copies meet in the same buckets (a few thousand of
    # them side by side: P + P) -- a third of the copies negated (P + (-P)), every 50th base the identity.  Two copies keep
    # the bins of the single-pass sort from overflowing, so the batched rounds really run (checked through the sort flag).
    kd, pd = kb.copy(), pb.copy()
    half = n // 2
    kd[half:2 * half], pd[half:2 * half] = kb[:half], pb[:half]
    negm = np.zeros(n, dtype=bool)
    negm[half:2 * half] = (np.arange(half) % 3) == 2
    ys = cref.bytes_to_ints(np.ascontiguousarray(pd[negm, 32:]))
    pd[negm, 32:] = cref.ints_to_bytes([(c.p - y) % c.p for y in ys])
    pd[(np.arange(n) % 50) == 7] = 0
    want_d = cref.bytes_to_affine(cref.best_multiexp(curve, kd, pd))
    try:
        for rounds, target in ((3, 64), (0, 0), (1, 64), (2, 8), (3, 200), (3, 1)):
            L.check(lib.h2_test_set_batched_affine(rounds, target))
            assert _affine(curve, eng.best_multiexp(kb, pb, curve)) == want, (rounds, target)
            assert _affine(curve, eng.best_multiexp(kd, pd, curve)) == want_d, ("degenerate", rounds, target)
            fl = ctypes.c_uint32(0)
            L.check(lib.h2_test_last_msm_flags(ctypes.byref(fl)))
            assert fl.value & 2 == 0, "the exact sort ran: the batched-affine rounds were skipped"
    finally:
        L.check(lib.h2_test_set_batched_affine(0, 32))


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_lookup_permuted_columns(eng, field):
    """permute_expression_pair (plonk/lookup/prover.rs:563-647) on resident columns against the oracle's line-for-line
    restatement: every size class of the sort (one shared-memory block, several blocks + global stages, non powers of two),
    tables with few / many distinct values, small integers (the high limbs tie) and full-width values, rows past usable_rows
    untouched, and the failure when an input value is missing from the table."""
    import random
    import halo2_b200 as h2
    m = pasta.FIELDS[field]
    rnd = random.Random(5)
    for n, u, distinct, small in ((8, 5, 3, True), (64, 64, 1, False), (1024, 1019, 40, True), (1 << 12, (1 << 12) - 6, 4000, False),
                                  (1 << 14, (1 << 14) - 6, 1 << 10, True), (3000, 2500, 2500, False)):
        pool = [rnd.randrange(1 << 12) if small else rnd.randrange(m) for _ in range(distinct)]
        tab = (pool + [rnd.choice(pool) for _ in range(u)])[:u] if distinct <= u else pool[:u]
        rnd.shuffle(tab)
        inp = [rnd.choice(tab) for _ in range(u)]
        tail = [rnd.randrange(m) for _ in range(n - u)]
        a = h2.ResidentPoly(field, n, cref.ints_to_bytes(inp + tail))
        t = h2.ResidentPoly(field, n, cref.ints_to_bytes(tab + tail))
        marker = [123456789 + i for i in range(n)]
        oa = h2.ResidentPoly(field, n, cref.ints_to_bytes(marker))
        ot = h2.ResidentPoly(field, n, cref.ints_to_bytes(marker))
        h2.permute_expression_pair_resident(a, t, u, oa, ot)
        want_a, want_s = pasta.permute_expression_pair(field, inp, tab, u)
        got_a, got_s = cref.bytes_to_ints(oa.download()), cref.bytes_to_ints(ot.download())
        assert got_a[:u] == want_a and got_s[:u] == want_s, (n, u, distinct)
        assert got_a[u:] == marker[u:] and got_s[u:] == marker[u:]             # the blinding rows are the caller's
        # an input value that the table does not hold: Error::ConstraintSystemFailure
        bad = list(inp)
        bad[u // 2] = (max(tab) + 1) % m if small else (tab[0] + 1) % m
        if bad[u // 2] not in set(tab):
            b = h2.ResidentPoly(field, n, cref.ints_to_bytes(bad + tail))
            with pytest.raises(h2.H2Error):
                h2.permute_expression_pair_resident(b, t, u, oa, ot)
            b.close()
        for p in (a, t, oa, ot):
            p.close()


def test_fast_fixed_base_pass_and_its_fallback(eng):
    """Fixed-base passes run without their fallback kernels first and re-run in full when a device flag comes back set
    (h2_test_set_fast_fixed): ordinary polynomials take the fast pass, constant / 0-1 / all-equal columns overflow the sort bins
    and take the re-run -- same points either way, through every entry point that issues such a pass (single and batched commits,
    commits of resident polynomials with batch_normalize, the IPA round loop), eager, captured and replayed.  After each pass,
    h2_test_last_msm_plan reports (fast, re-run): with fast passes on, a pass either ran fast and stood (1, 0) or re-ran in full
    (0, 1); with them off, every pass runs in full once (0, 0)."""
    import halo2_b200 as h2
    from halo2_b200 import lib as L
    lib = L.init()

    def fast_rerun():
        out = (ctypes.c_uint32 * 8)()
        L.check(lib.h2_test_last_msm_plan(out))
        return out[6], out[7]

    def check_plan(on, want=None):
        got = fast_rerun()
        if not on:
            assert got == (0, 0), got
        elif want is not None:
            assert got == want, got
        else:
            assert got in ((1, 0), (0, 1)), got
    # a single commit: the random column stands, the all-ones, 0/1 and all-(r - 1) columns re-run; the all-zero column's scalars
    # may add no references at all
    single_want = [(1, 0), None, (0, 1), (0, 1), (0, 1), None]
    curve, c, k = "vesta", pasta.VESTA, 9
    n = 1 << k
    g = cref.gen_points(curve, SEED + 700, n + 2)
    polys = [cref.gen_scalars(c.scalar, SEED + 701, n), cref.ints_to_bytes([0] * n), cref.ints_to_bytes([1] * n),
             cref.ints_to_bytes([i & 1 for i in range(n)]), cref.ints_to_bytes([c.r - 1] * n), cref.gen_scalars(c.scalar, SEED + 702, n)]
    blind = h2.Blind(11)
    wants = [cref.bytes_to_affine(cref.best_multiexp(curve, np.concatenate([p, cref.ints_to_bytes([11])]), g[:n + 1])) for p in polys]
    ch = pasta.gen_scalars(c.scalar, SEED + 703, k)
    lr = pasta.gen_scalars(c.scalar, SEED + 704, k)
    ipa_want = {}
    for name, pp in (("random", polys[0]), ("constant", polys[4])):
        ipa_want[name] = cref.ipa_rounds(curve, g, k, pp, 3, 5, cref.ints_to_bytes(ch), cref.ints_to_bytes(lr), cref.ints_to_bytes(lr))
    try:
        for on in (1, 0, 1):
            L.check(lib.h2_test_set_fast_fixed(on))
            params = h2.Params(curve, k, g[:n], g[:n], g[n:n + 1], u=g[n + 1:n + 2])
            for rep in range(3):
                for p, want, plan in zip(polys, wants, single_want):
                    assert _affine(curve, params.commit(p, blind)) == want, (on, rep)
                    check_plan(on, plan)
            assert [_affine(curve, m) for m in params.commit_many(polys, [blind] * len(polys))] == wants, on
            check_plan(on, (0, 1))
            res = [h2.ResidentPoly(c.scalar, n, p) for p in polys]
            for rep in range(3):
                aff = params.commit_resident_affine(res, [blind] * len(res))
                assert [cref.bytes_to_affine(a) for a in aff] == wants, (on, rep)
                check_plan(on, (0, 1))

            def challenge(j, a, b):   # right after round j's pass; whether a round of a constant p' re-runs depends on the challenges
                check_plan(on)
                return ch[j]
            for name, pp in (("random", polys[0]), ("constant", polys[4])):
                wl, wr, wc = ipa_want[name]
                for rep in range(2):
                    gl_, gr_, gc_ = params.ipa_rounds(pp, 3, 5, challenge, lr, lr)
                    assert gc_ == wc, (on, name)
                    for j in range(k):
                        assert (cref.jac_to_affine(curve, gl_[j]) == wl[j]).all() and (cref.jac_to_affine(curve, gr_[j]) == wr[j]).all(), (on, name, j)
            for r_ in res:
                r_.close()
            params.close()
    finally:
        L.check(lib.h2_test_set_fast_fixed(1))
