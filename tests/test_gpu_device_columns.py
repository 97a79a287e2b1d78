"""GPU tests of the device-memory column transfers (h2_poly_upload_dev / h2_poly_download_dev, K25 columns_io.cuh, and
ResidentPoly.from_tensor / upload_tensor / to_tensor, upload_tensors_resident / download_tensors_resident):

- the resident bytes equal h2_poly_upload's of the same elements and the exported bytes h2_poly_download's, k = 0 ... 20,
  both fields, both reprs, 1, 3 and 17 columns of different lengths per call, random 256-bit inputs (most of them >= p);
- the stream contract with no host synchronisation between the calls, on the primary context and on a lane;
- instance_commit / advice_commit / keygen fed CUDA tensors give the host columns' commitments and keys, and proofs composed
  from the phase calls (tests/plonk_prover.create_proof_engine) the host columns' bytes, which the verifier accepts;
- every refusal happens before anything is launched and leaves the destination alone;
- a lane exports a shared key's polynomial."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests import arguments_cases as AC  # noqa: E402
from tests import multiopen_cases as MC  # noqa: E402
from tests import plonk_api_circuit as circ  # noqa: E402
from tests import plonk_prover as PP  # noqa: E402
from tests import plonk_verifier as PV  # noqa: E402
from tests import prover_replay as R  # noqa: E402

REPRS = {"canonical": 0, "montgomery": 1}


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(params=["primary", "lane"])
def ctx(request, eng):
    if request.param == "lane":
        with eng.Lane():
            yield eng
    else:
        yield eng


def _L():
    from halo2_b200 import lib as L
    return L


def _raw(p, n=None):
    """The resident bytes themselves (Montgomery form) through the host path."""
    L = _L()
    n = p.len if n is None else n
    out = np.zeros((n, 32), dtype=np.uint8)
    L.check(L.load().h2_poly_download(p._h, L.ptr(out), ctypes.c_size_t(n), L.REPR_MONTGOMERY))
    return out


def _host_upload(eng, field, n, a, repr_):
    L = _L()
    p = eng.ResidentPoly(field, n)
    if a.shape[0]:
        L.check(L.load().h2_poly_upload(p._h, L.ptr(a), ctypes.c_size_t(a.shape[0]), REPRS[repr_]))
    return p


def _host_download(p, n, repr_):
    L = _L()
    out = np.zeros((n, 32), dtype=np.uint8)
    L.check(L.load().h2_poly_download(p._h, L.ptr(out), ctypes.c_size_t(n), REPRS[repr_]))
    return out


def _random(rng, n, specials=True):
    a = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    if specials and n:
        a[0] = 0xFF                                                   # all-ones
        a[n // 2] = np.frombuffer(pasta.P_MOD.to_bytes(32, "little"), dtype=np.uint8)
    return a


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("repr_", ["canonical", "montgomery"])
def test_equals_the_host_path(eng, torch, field, repr_):
    rng = np.random.default_rng(0xC0 + 2 * REPRS[repr_] + (field == "fq"))
    for k in range(21):
        n = 1 << k
        for count in (1, 3, 17):
            lens = [n if i % 3 == 0 else max(0, n - 1 - 7 * i) if i % 3 == 1 else n >> 1 for i in range(count)]
            host = [_random(rng, ln) for ln in lens]
            tens = [torch.from_numpy(a).cuda() for a in host]
            dev = [eng.ResidentPoly(field, n) for _ in lens]
            ref = [_host_upload(eng, field, n, a, repr_) for a in host]
            try:
                eng.upload_tensors_resident(dev, tens, repr=repr_)
                for d, r, ln in zip(dev, ref, lens):
                    assert np.array_equal(_raw(d), _raw(r)), (k, count, ln)
                got = eng.download_tensors_resident(ref, lens, repr=repr_)
                for t, r, ln in zip(got, ref, lens):
                    assert t.shape == (ln, 32) and np.array_equal(t.cpu().numpy(), _host_download(r, ln, repr_)), (k, count, ln)
                if count == 1:
                    one = eng.ResidentPoly.from_tensor(field, tens[0], length=n, repr=repr_)
                    try:
                        assert np.array_equal(_raw(one), _raw(ref[0]))
                        assert np.array_equal(one.to_tensor(repr=repr_).cpu().numpy(), _host_download(ref[0], n, repr_))
                    finally:
                        one.close()
            finally:
                for p in dev + ref:
                    p.close()


def _fft_input(torch, n, stream, seed):
    """Canonical elements < 2^254 < p, written by torch kernels on `stream`."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.cuda.stream(stream):
        t = torch.randint(0, 256, (n, 32), dtype=torch.uint8, device="cuda", generator=g)
        for _ in range(20):                                           # enough queued work that a missing wait would show
            t = (t.to(torch.int32) * 1 + 0).to(torch.uint8)
        t[:, 31] &= 0x3F
    return t


def test_stream_order_upload(ctx, torch):
    """A torch kernel writes the tensor on a side stream, upload_tensor runs on that stream, a resident transform follows on
    the context's stream: the transform sees the tensor."""
    L = _L()
    log_n, field = 18, "fp"
    n = 1 << log_n
    omega = pasta.omega_for_k(field, log_n)
    side = torch.cuda.Stream()
    t = _fft_input(torch, n, side, 11)
    a = ctx.ResidentPoly(field, n)
    out = ctx.ResidentPoly(field, n)
    try:
        a.upload_tensor(t, stream=side)
        L.check(L.load().h2_poly_lagrange_to_coeff(out._h, a._h, ctypes.c_uint32(log_n), L.ptr(L.fe_bytes(omega)), L.ptr(L.fe_bytes(1)),
                                                   L.REPR_CANONICAL))
        got = out.download()
        torch.cuda.synchronize()
        assert np.array_equal(got, cref.best_fft(field, t.cpu().numpy(), omega, log_n))
    finally:
        a.close()
        out.close()


def test_stream_order_download(ctx, torch):
    """to_tensor after a resident transform, then a torch op on the caller's stream: the op sees the exported values."""
    L = _L()
    log_n, field = 18, "fq"
    n = 1 << log_n
    omega = pasta.omega_for_k(field, log_n)
    vals = cref.gen_scalars(field, 12, n)
    a = ctx.ResidentPoly(field, n, vals)
    side = torch.cuda.Stream()
    try:
        L.check(L.load().h2_poly_lagrange_to_coeff(a._h, a._h, ctypes.c_uint32(log_n), L.ptr(L.fe_bytes(omega)), L.ptr(L.fe_bytes(1)),
                                                   L.REPR_CANONICAL))
        t = a.to_tensor(stream=side)
        with torch.cuda.stream(side):
            doubled = torch.cat([t, t])                               # a torch op behind the export on the same stream
        side.synchronize()
        want = cref.best_fft(field, vals, omega, log_n)
        assert np.array_equal(doubled.cpu().numpy(), np.concatenate([want, want]))
    finally:
        a.close()


def test_refused_before_launch(eng, torch):
    L = _L()
    lib = L.load()
    fp = eng.ResidentPoly("fp", 64)
    fq = eng.ResidentPoly("fq", 64)
    shared = eng.ResidentPoly("fp", 64, cref.gen_scalars("fp", 3, 64)).share()
    buf = torch.zeros(64 * 32 + 64, dtype=torch.uint8, device="cuda")
    host = np.zeros((64, 32), dtype=np.uint8)
    try:
        before_fp, before_fq = _raw(fp), _raw(fq)
        torch.cuda.synchronize()
        count = L.launch_count()
        s = torch.cuda.current_stream().cuda_stream
        base = buf.data_ptr()
        cases = [
            ("h2_poly_upload_dev", [fp], [host.ctypes.data], [4], "d_src\\[0\\]: not device memory \\(host columns go through h2_poly_upload\\)"),
            ("h2_poly_download_dev", [fp], [host.ctypes.data], [4], "d_dst\\[0\\]: not device memory \\(host columns go through h2_poly_download\\)"),
            ("h2_poly_upload_dev", [fp], [base + 8], [4], "d_src\\[0\\]: not 16-byte aligned"),
            ("h2_poly_download_dev", [fp], [base + 8], [4], "d_dst\\[0\\]: not 16-byte aligned"),
            ("h2_poly_upload_dev", [fp], [base], [65], "polys\\[0\\]: a polynomial holds fewer than lens\\[0\\] elements"),
            ("h2_poly_upload_dev", [fq, fq], [base, base], [1, 1], "polys\\[1\\] is also polys\\[0\\]"),
            ("h2_poly_upload_dev", [shared], [base], [1], "polys\\[0\\]: the polynomial is shared"),
            ("h2_poly_upload_dev", [fp, fq], [base, base], [1, 1], "polys\\[1\\]: the polynomials live in different fields"),
            ("h2_poly_download_dev", [fp, fq], [base, base], [1, 1], "polys\\[1\\]: the polynomials live in different fields"),
            ("h2_poly_download_dev", [fp, fp], [base, base + 32 * 3], [4, 4], "d_dst\\[1\\]: overlaps d_dst\\[0\\]"),
            ("h2_poly_download_dev", [fp, fp, fp], [base + 32 * 40, base, base + 32 * 10], [8, 30, 4], "d_dst\\[2\\]: overlaps d_dst\\[1\\]"),
        ]
        for name, ps, ptrs, lens, msg in cases:
            with pytest.raises(L.H2Error, match=msg):
                eng.poly._dev_io(name, ps, ptrs, lens, 0, s)
        with pytest.raises(L.H2Error, match="unknown repr"):
            eng.poly._dev_io("h2_poly_upload_dev", [fp], [base], [1], 7, s)
        assert lib.h2_poly_upload_dev(None, ctypes.c_size_t(0), None, None, 0, None) == 0
        torch.cuda.synchronize()
        assert L.launch_count() == count
        assert np.array_equal(_raw(fp), before_fp) and np.array_equal(_raw(fq), before_fq) and not buf.any()
        # a misaligned view of a tensor, through the tensor API
        with pytest.raises(L.H2Error, match="not 16-byte aligned"):
            fp.upload_tensor(buf[8:8 + 32 * 4].view(4, 32))
        assert L.launch_count() == count
    finally:
        for p in (fp, fq, shared):
            p.close()


def test_lane_exports_a_shared_polynomial(eng, torch):
    vals = cref.gen_scalars("fp", 21, 4096)
    key = eng.ResidentPoly("fp", 4096, vals).share()
    try:
        with eng.Lane():
            t = key.to_tensor()
            torch.cuda.current_stream().synchronize()
            assert np.array_equal(t.cpu().numpy(), vals)
    finally:
        key.close()


# ---- the phases fed CUDA tensors ----

def _cuda(torch, cols):
    return [torch.from_numpy(np.ascontiguousarray(c)).cuda() for c in cols]


def _proof(eng, prm, pk, vk, advice, inst, seed):
    T = R.Blake2bTranscript(circ.M)
    PP.create_proof_engine(eng, prm, vk, None, None, advice, inst, MC.SeededRng("fp", seed, True), T, circ.ZETA, circ.DELTA, pk=pk)
    return bytes(T.proof)


def _same_proof(eng, torch, prm, pk, vk, advice, inst, seed, k):
    want = _proof(eng, prm, pk, vk, advice, inst, seed)
    adv_t = [_cuda(torch, per) for per in advice]
    inst_t = [_cuda(torch, [cref.ints_to_bytes([v % circ.M for v in col]) for col in per]) for per in inst]
    got = _proof(eng, prm, pk, vk, adv_t, inst_t, seed)
    assert got == want
    assert PV.verify_proof(PV.EngineArm(eng, "vesta", k, params=prm), vk, got, inst, circ.DELTA)


def test_proof_plonk_api_circuit(eng, torch):
    vk = PV.PinnedKey(circ.CASE["key_text"])
    fixed, sigma = circ.fixed_columns(circ.M, circ.ZETA), circ.permutation_columns(circ.M, vk.omega, circ.DELTA)
    prm = eng.Params.new("vesta", 5)
    D = eng.EvaluationDomain("fp", vk.degree(), vk.k, circ.ZETA)
    pk = PP.proving_key(eng, D, fixed, sigma, vk.blinding_factors())
    try:
        adv = [[cref.ints_to_bytes([v % circ.M for v in col]) for col in circ.witness()] for _ in range(2)]
        _same_proof(eng, torch, prm, pk, vk, adv, [[[2]], [[2]]], 777, 5)
    finally:
        pk.close()
        prm.close()


def test_proof_benchmark_circuit_k14(eng, torch):
    from tests import bench_circuit as BC
    k, m = 14, circ.M
    prm = eng.Params.new("vesta", k)
    D = eng.EvaluationDomain("fp", BC.DEGREE, k, circ.ZETA)
    fixed, sigma, adv = BC.columns(k, m, D.omega, circ.DELTA, circ.A_SMALL * circ.ZETA % m)
    fb, sb, ab = ([cref.ints_to_bytes(c_) for c_ in cols] for cols in (fixed, sigma, adv))
    commit = lambda v: cref.bytes_to_affine(eng.batch_normalize(prm.commit_lagrange(v, eng.Blind(1)).reshape(1, 96), "vesta")[0])  # noqa: E731
    vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, pasta.Q_MOD, m, D.omega, [commit(c) for c in fb], [commit(c) for c in sb]))
    pk = PP.proving_key(eng, D, fb, sb, vk.blinding_factors())
    try:
        _same_proof(eng, torch, prm, pk, vk, [ab], [[]], 5, k)
    finally:
        pk.close()
        prm.close()


@pytest.mark.parametrize("k", [8, 16])
def test_proof_nonlinear_circuit(eng, torch, k):
    prm = eng.Params.new("vesta", k)
    commit = lambda c: cref.bytes_to_affine(eng.batch_normalize(prm.commit_lagrange(cref.ints_to_bytes(c), eng.Blind(1)).reshape(1, 96), "vesta")[0])  # noqa: E731
    vk, D, fixed, sigma, advice, inst = AC.nonlinear_case(eng, k, commit, circ.ZETA, circ.DELTA)
    pk = PP.proving_key(eng, D, fixed, sigma, vk.blinding_factors())
    try:
        adv = [cref.ints_to_bytes(c) for c in advice]
        _same_proof(eng, torch, prm, pk, vk, [adv, adv], [inst, inst], 40 + k, k)
    finally:
        pk.close()
        prm.close()


def test_phase_commitments(eng, torch):
    """instance_commit (short columns zero-padded, InstanceTooLarge from the shape), advice_commit and keygen_vk / keygen_pk
    with CUDA tensors equal the host columns' results."""
    from tests import bench_circuit as BC
    k, m = 10, circ.M
    prm = BC._bench_params(eng, k)
    D = eng.EvaluationDomain("fp", BC.DEGREE, k, circ.ZETA)
    fixed, _, adv = BC.columns(k, m, D.omega, circ.DELTA, circ.A_SMALL * circ.ZETA % m)
    fb, ab = [cref.ints_to_bytes(c) for c in fixed], [cref.ints_to_bytes(c) for c in adv]
    bf = 5
    inst = [[cref.gen_scalars("fp", 60, 7), cref.gen_scalars("fp", 61, D.n - bf - 1)], [cref.gen_scalars("fp", 62, 0)]]
    out = []
    try:
        want = eng.instance_commit(prm, D, inst, bf)
        got = eng.instance_commit(prm, D, [_cuda(torch, per) for per in inst], bf)
        out += want + got
        for w, g in zip(want, got):
            assert np.array_equal(w.commitments, g.commitments)
            for a, b in zip(w.values + w.cosets, g.values + g.cosets):
                assert np.array_equal(_raw(a), _raw(b))
        count = eng.launch_count()
        with pytest.raises(eng.InstanceTooLarge):
            eng.instance_commit(prm, D, [[torch.zeros((D.n - bf, 32), dtype=torch.uint8, device="cuda")]], bf)
        assert eng.launch_count() == count
        want = eng.advice_commit(prm, D, [ab, ab[:2]], MC.SeededRng("fp", 9, True), bf)
        got = eng.advice_commit(prm, D, [_cuda(torch, ab), _cuda(torch, ab[:2])], MC.SeededRng("fp", 9, True), bf)
        out += want + got
        for w, g in zip(want, got):
            assert np.array_equal(w.commitments, g.commitments) and w.blinds == g.blinds
            for a, b in zip(w.values + w.cosets, g.values + g.cosets):
                assert np.array_equal(_raw(a), _raw(b))
        asm = BC._bench_assembly(eng, k)
        fc, pc = eng.keygen_vk(prm, D, fb, asm, circ.DELTA)
        fc_t, pc_t = eng.keygen_vk(prm, D, _cuda(torch, fb), asm, circ.DELTA)
        assert np.array_equal(fc, fc_t) and np.array_equal(pc, pc_t)
        pk = eng.keygen_pk(prm, D, fb, asm, circ.DELTA, BC.BLINDING_FACTORS)
        pk_t = eng.keygen_pk(prm, D, _cuda(torch, fb), asm, circ.DELTA, BC.BLINDING_FACTORS)
        try:
            for a, b in zip(pk.fixed_values + pk.fixed_polys + pk.fixed_cosets, pk_t.fixed_values + pk_t.fixed_polys + pk_t.fixed_cosets):
                assert np.array_equal(_raw(a), _raw(b))
        finally:
            pk.close()
            pk_t.close()
    finally:
        for s in out:
            for p in s.values + s.polys + s.cosets:
                p.close()
        prm.close()
