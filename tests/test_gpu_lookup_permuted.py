"""GPU tests of the lookup argument's permuted columns in one call (h2_poly_lookup_permuted; halo2_b200.lookup_permute_resident /
lookup_commit_permuted):

- the outputs equal the oracle's permute_expression_pair (oracle/cref.py) plus the blinding rows, k = 4 .. 20, 1 / 3 / 16
  lookups per call, uniform inputs and inputs with 90 % of the rows on one value;
- at k = 14 .. 20 they are byte-identical to the per-lookup composition (h2_poly_lookup_permute and the rows uploaded);
- the plonk_api proof's permuted commitments, and its lookup z columns through lookup_commit_product, match the proof bytes;
- every validation error, on the primary context and on a lane, fails with a message and leaves the outputs at their markers;
- two lanes running the call concurrently give the serial bytes, with inputs shared between them."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import cref, pasta  # noqa: E402
from tests.abi_cases import _err, _run_parallel  # noqa: E402
from tests.lookup_permuted_cases import columns, composition  # noqa: E402

SEED = 0x4C4B5032


@pytest.fixture(scope="module")
def eng():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    return halo2_b200


def _close(*groups):
    for g in groups:
        for p in g:
            p.close()


CASES = [(k, (1, 3, 16)[k % 3]) for k in range(4, 21)] + [(20, 16), (14, 1), (11, 3)]


@pytest.mark.parametrize("k,count", CASES)
def test_outputs_equal_the_reference(eng, k, count):
    field = "fp" if k % 2 else "fq"
    m = pasta.FIELDS[field]
    n, bf = 1 << k, 5 if k > 4 else 2
    u, rows = n - bf - 1, bf + 1
    D = eng.EvaluationDomain(field, 3, k, pasta.zeta_candidates(field)[0])
    cols = [columns(field, n, u, SEED + 7 * k + b, hot=b % 2 == 1) for b in range(count)]
    pairs = [(eng.ResidentPoly(field, n, a), eng.ResidentPoly(field, n, t)) for a, t in cols]
    blinding = pasta.gen_scalars(field, SEED + k, count * 2 * rows)
    out = eng.lookup_permute_resident(D, pairs, bf, blinding)
    try:
        for b, ((a, t), (pi, pt)) in enumerate(zip(cols, out)):
            want = cref.permute_expression_pair(a, t, u)
            assert want is not None
            got_a, got_t = pi.download(), pt.download()
            assert (got_a[:u] == want[0][:u]).all() and (got_t[:u] == want[1][:u]).all(), (k, b)
            blind = cref.ints_to_bytes([x % m for x in blinding[2 * rows * b:2 * rows * (b + 1)]])
            assert (got_a[u:] == blind[:rows]).all() and (got_t[u:] == blind[rows:]).all(), (k, b)
    finally:
        _close([p for pr in pairs for p in pr], [p for pr in out for p in pr])


@pytest.mark.parametrize("k", [14, 16, 18, 20])
def test_byte_identical_to_the_composition(eng, k):
    field, n, bf, count = "fp", 1 << k, 5, 4
    u = n - bf - 1
    D = eng.EvaluationDomain(field, 3, k, pasta.zeta_candidates(field)[0])
    pairs = [tuple(eng.ResidentPoly(field, n, c) for c in columns(field, n, u, SEED + 100 * k + b, hot=b >= 2)) for b in range(count)]
    blinding = pasta.gen_scalars(field, SEED + 3 * k, count * 2 * (bf + 1))
    new = eng.lookup_permute_resident(D, pairs, bf, blinding)
    old = composition(eng, D, pairs, bf, blinding)
    try:
        for x, y in zip(new, old):
            assert (x[0].download() == y[0].download()).all() and (x[1].download() == y[1].download()).all()
    finally:
        _close([p for pr in pairs + new + old for p in pr])


def test_plonk_api_proof(eng):
    """The plonk_api circuit (k = 5, two proofs, lookups), proved by create_proof_engine with the oracle prover's bytes:
    lookup_commit_permuted, fed the recorded theta and draws, gives the permuted commitments at their offsets in the oracle's
    proof, and lookup_commit_product, given its result as it is and the recorded beta, gamma and draws, gives the lookup
    product commitments."""
    from tests import bench_circuit as BC
    from tests import multiopen_cases as MC
    from tests import plonk_api_circuit as circ
    from tests import prover_replay as R
    vk = circ.plonk_api_key()
    bf, L = vk.blinding_factors(), len(vk.lookups)
    prm = BC._bench_params(eng, 5)
    try:
        proof, seen = circ.plonk_api_proof(eng, prm)
        assert proof == circ.plonk_api_oracle_proof(prm.g, prm.w, prm.u)
        D, ev, lookups = circ.plonk_api_lookups(eng, seen)
        perm, cm = eng.lookup_commit_permuted(prm, D, ev, lookups, seen["theta"], bf, MC.ReplayRng(seen["draws"][seen["draws_at_theta"]:]))
        at = seen["points_at_theta"]
        assert len(cm) == 2 * 2 * L and proof[32 * at:32 * (at + len(cm))] == R._encode(cm, circ.M)
        nsets = -(-len(vk.permutation_columns) // (vk.degree() - 2))
        first = at + len(cm) + 2 * nsets                            # the lookup products follow the permutation products
        beta, gamma = seen["challenges"][1], seen["challenges"][2]
        z, zcm = eng.lookup_commit_product(prm, D, perm, beta, gamma, bf, MC.ReplayRng(seen["draws"][seen["point_draws"][first - 1]:]))
        assert len(zcm) == 2 * L and proof[32 * first:32 * (first + len(zcm))] == R._encode(zcm, circ.M)
        _close([p for per in perm for q in per for p in q[:8]], ev.polys, [q[0] for per in z for q in per])
    finally:
        prm.close()


# ---- validation ---------------------------------------------------------------------------------------------------------
def _error_cases(eng):
    from halo2_b200 import lib as L
    lib = L.load()
    k, n, field, bf = 4, 16, "fp", 2
    u = n - bf - 1
    mk = lambda seed, ln=n, f=field: eng.ResidentPoly(f, ln, cref.gen_scalars(f, SEED + seed, ln))
    cols = [columns(field, n, u, SEED + 40 + b, hot=False) for b in range(2)]
    ins = [eng.ResidentPoly(field, n, c) for pair in cols for c in pair]      # input 0, table 0, input 1, table 1
    outs = [mk(1), mk(2), mk(3), mk(4)]
    fq, short, sh = mk(9, f="fq"), mk(10, n - 1), mk(11).share()
    gone = mk(12)
    gone_h = gone._h.value
    gone.close()
    H = lambda ps: (ctypes.c_uint64 * len(ps))(*[p if isinstance(p, int) else p._h.value for p in ps])
    blind = cref.gen_scalars(field, SEED + 13, 2 * 2 * (bf + 1))
    before = [q.download() for q in outs]
    missing = ins[2].download()
    missing[u // 2] = cref.ints_to_bytes([pasta.FIELDS[field] - 3])[0]       # a value no table holds: lookup 1 misses
    miss = eng.ResidentPoly(field, n, missing)

    def call(o=None, i=None, kk=k, b=bf, count=2):
        o, i = o or outs, i or ins
        return lib.h2_poly_lookup_permuted(H(o[0::2]), H(o[1::2]), ctypes.c_size_t(count), H(i[0::2]), H(i[1::2]), ctypes.c_uint32(kk),
                                           L.ptr(blind), ctypes.c_uint32(b), 0)

    def untouched():
        assert all((q.download() == b).all() for q, b in zip(outs, before))

    try:
        cases = [
            (lambda: call(o=[outs[0], 0xDEADBEEF, outs[2], outs[3]]), "out_tables[0]: unknown polynomial handle"),
            (lambda: call(o=[outs[0], outs[1], gone_h, outs[3]]), "out_inputs[1]: unknown polynomial handle"),
            (lambda: call(i=[ins[0], ins[1], 0xDEADBEEF, ins[3]]), "inputs[1]: unknown polynomial handle"),
            (lambda: call(i=[ins[0], fq, ins[2], ins[3]]), "tables[0]: the polynomials live in different fields"),
            (lambda: call(o=[outs[0], outs[1], fq, outs[3]]), "out_inputs[1]: the polynomials live in different fields"),
            (lambda: call(i=[ins[0], ins[1], short, ins[3]]), "inputs[1]: a polynomial holds fewer than 2^k elements"),
            (lambda: call(o=[outs[0], short, outs[2], outs[3]]), "out_tables[0]: a polynomial holds fewer than 2^k elements"),
            (lambda: call(o=[outs[0], outs[1], sh, outs[3]]), "out_inputs[1]: the polynomial is shared (read-only)"),
            (lambda: call(o=[outs[0], outs[1], outs[0], outs[3]]), "out_inputs[1] is also out_inputs[0]"),
            (lambda: call(o=[outs[0], ins[3], outs[2], outs[3]]), "out_tables[0] is also tables[1]"),
            (lambda: call(b=n - 1), "blinding_factors + 1 >= n"), (lambda: call(kk=31), "k > 30"),
            (lambda: call(count=65536), "more than 65535"),
            (lambda: call(i=[ins[0], ins[1], miss, ins[3]]), "lookup 1: an input value does not occur"),
            (lambda: call(i=[miss, ins[3], miss, ins[3]]), "lookup 0: an input value does not occur"),
        ]
        for j, (fn, msg) in enumerate(cases):
            assert fn() != 0 and msg in _err(), (j, _err())
            untouched()
        assert call(count=0) == 0
        untouched()
        assert call(i=[ins[0], ins[1], ins[0], ins[1]]) == 0               # inputs may repeat
        assert not all((q.download() == b).all() for q, b in zip(outs, before))
    finally:
        _close(ins, outs, [fq, short, sh, miss])


def test_errors_name_the_argument_on_the_primary_context(eng):
    _error_cases(eng)


def test_errors_name_the_argument_on_a_lane(eng):
    def go():
        with eng.Lane():
            _error_cases(eng)
    _run_parallel([go])


def test_two_lanes_concurrently_with_shared_inputs(eng):
    k, field, bf, count = 16, "fq", 5, 3
    n = 1 << k
    u = n - bf - 1
    D = eng.EvaluationDomain(field, 3, k, pasta.zeta_candidates(field)[0])
    cols = [columns(field, n, u, SEED + 300 + b, hot=b == 1) for b in range(count)]
    shared = [eng.ResidentPoly(field, n, c).share() for pair in cols for c in pair]
    pairs = list(zip(shared[0::2], shared[1::2]))
    blinding = pasta.gen_scalars(field, SEED + 301, count * 2 * (bf + 1))
    serial = eng.lookup_permute_resident(D, pairs, bf, blinding)
    want = [(a.download(), t.download()) for a, t in serial]

    def go():
        with eng.Lane():
            got = []
            for _ in range(3):
                out = eng.lookup_permute_resident(D, pairs, bf, blinding)
                got.append([(a.download(), t.download()) for a, t in out])
                _close([p for pr in out for p in pr])
            return got
    try:
        for got in _run_parallel([go, go]):
            for run in got:
                assert all((a == wa).all() and (t == wt).all() for (a, t), (wa, wt) in zip(run, want))
    finally:
        _close([p for pr in serial for p in pr], shared)
