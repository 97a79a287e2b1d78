"""GPU checks of halo2_b200.arguments: proofs composed from the phase calls (tests/plonk_prover.create_proof_engine) of the
circuit with a selector-gated two-row lookup at k = 8 ... 18, the same proofs on a lane over a shared proving key, and cleanup
when construct or evaluate fails.  tests/test_gpu_zz_real_proof.py checks the composition's bytes against the references."""
import pytest

import halo2_b200
from halo2_b200 import arguments as A
from halo2_b200 import lib as L
from halo2_b200 import poly as P
from oracle import cref
from tests import arguments_cases as AC
from tests import multiopen_cases as MC
from tests import plonk_api_circuit as circ
from tests import plonk_prover as PP
from tests import plonk_verifier as PV
from tests import prover_replay as R

pytestmark = pytest.mark.gpu


def _proof(prm, vk, pk, advice, inst, seed, hook=None):
    T = R.Blake2bTranscript(circ.M)
    PP.create_proof_engine(halo2_b200, prm, vk, None, None, advice, inst, MC.SeededRng("fp", seed, True), T, circ.ZETA, circ.DELTA, pk=pk,
                           on_construct=hook)
    return bytes(T.proof)


def _commit(prm, values):
    """commit_lagrange with Blind::default(), affine (x, y) ints."""
    vals = values if hasattr(values, "dtype") else cref.ints_to_bytes(values)
    return cref.bytes_to_affine(halo2_b200.batch_normalize(prm.commit_lagrange(vals, halo2_b200.Blind(1)).reshape(1, 96), "vesta")[0])


def _nonlinear(k):
    prm = halo2_b200.Params.new("vesta", k)
    vk, D, fixed, sigma, advice, inst = AC.nonlinear_case(halo2_b200, k, lambda c: _commit(prm, c), circ.ZETA, circ.DELTA)
    adv = [cref.ints_to_bytes(c) for c in advice]
    return prm, vk, D, PP.proving_key(halo2_b200, D, fixed, sigma, vk.blinding_factors()), adv, inst


@pytest.mark.parametrize("k", [8, 12, 16, 18])
def test_nonlinear_lookup_circuit(k):
    """Two proofs, three permutation sets.  The engine's verifier accepts the proof at every k and the restated reference
    verifier at k = 8 (its multiexps are Python integers); a flipped byte and a wrong instance are rejected.  The circuit
    exercises the difference: the coset compression and the extended Lagrange column differ for every lookup."""
    prm, vk, D, pk, adv, inst = _nonlinear(k)
    try:
        assert len(vk.permutation_columns) == 10 and vk.degree() - 2 == 4
        seen, hook = AC.coset_compression_differs(halo2_b200, D)
        proof = _proof(prm, vk, pk, [adv, adv], [inst, inst], 40 + k, hook=hook)
        assert seen == [True] * 4
        arms = [PV.EngineArm(halo2_b200, "vesta", k, params=prm)]
        if k == 8:
            arms.append(PV.OracleArm("vesta", k, prm.g, prm.g_lagrange, prm.w, prm.u))
        bad = bytearray(proof)
        bad[len(proof) // 3] ^= 1
        for arm in arms:
            assert PV.verify_proof(arm, vk, proof, [inst, inst], circ.DELTA), arm.name
            assert not PV.verify_proof(arm, vk, bytes(bad), [inst, inst], circ.DELTA), arm.name
            assert not PV.verify_proof(arm, vk, proof, [inst, [[inst[0][0] + 1]]], circ.DELTA), arm.name
    finally:
        pk.close()
        prm.close()


def test_on_a_lane_with_a_shared_key():
    """The same proofs on a lane over pk.share() equal the primary context's, byte for byte."""
    prm, vk, D, pk, adv, inst = _nonlinear(12)
    try:
        pk.share()
        want = _proof(prm, vk, pk, [adv, adv], [inst, inst], 3)
        with L.Lane():
            got = _proof(prm, vk, pk, [adv, adv], [inst, inst], 3)
        assert got == want
        assert PV.verify_proof(PV.EngineArm(halo2_b200, "vesta", 12, params=prm), vk, got, [inst, inst], circ.DELTA)
    finally:
        pk.close()
        prm.close()


class _Counting(halo2_b200.ResidentPoly):
    live = set()

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        _Counting.live.add(self._h.value)

    def close(self):
        _Counting.live.discard(self._h.value)
        super().close()


def test_failing_construct_and_evaluate_leave_nothing_allocated(monkeypatch):
    """The lookups' construct fails in its batched transform (polynomials of the primary context used on a lane) after it
    allocated the product cosets, and evaluate fails in its h2_poly_eval: no polynomial they made stays allocated.  A
    refused permutation construct allocates nothing."""
    monkeypatch.setattr(P, "ResidentPoly", _Counting)
    k = 6
    D = halo2_b200.EvaluationDomain("fp", 6, k, circ.ZETA)
    n, N = D.n, D.extended_len()
    rp = lambda length, s: halo2_b200.ResidentPoly("fp", length, cref.gen_scalars("fp", s, length))   # noqa: E731
    permuted = [halo2_b200.Permuted(*[rp(n, 10 * i + j) for j in range(6)], rp(N, 10 * i + 6), rp(N, 10 * i + 7), 3, 4) for i in range(2)]
    look = A.LookupCommitted(permuted, [(rp(n, 100 + i), 5) for i in range(2)])
    ev = halo2_b200.Evaluator(D, "extended")
    leaves = [ev.register_poly(rp(N, 200 + i)) for i in range(5)]
    l0, lb, ll, a, b = leaves
    exprs = [([a * b], [b]), ([a + b], [a])]
    try:
        with L.Lane():
            lane_ev = halo2_b200.Evaluator(D, "extended")
            before = set(_Counting.live)
            with pytest.raises(L.H2Error):
                look.construct(lane_ev, exprs, 2, 3, 4, l0, lb, ll)
            assert _Counting.live == before
            with pytest.raises(L.H2Error):
                A.LookupConstructed(look, []).evaluate(D, 12345)
            assert _Counting.live == before
        constructed, es = look.construct(ev, exprs, 2, 3, 4, l0, lb, ll)
        assert len(es) == 10 and len(_Counting.live) == 2
        evaluated, evals = constructed.evaluate(D, 12345)
        want = halo2_b200.eval_polynomial_resident([look.products[0][0]], [12345], n=n)[0]
        assert evals[0] == want and len(evals) == 10
        from halo2_b200.keygen import PermutationProvingKey
        sig = [rp(n, 300 + i) for i in range(10)]
        pk = halo2_b200.ProvingKey([], [], [], PermutationProvingKey([], sig, [rp(N, 400 + i) for i in range(10)]), None, None, None)
        perm = A.PermutationCommitted([(rp(n, 500 + i), rp(N, 600 + i), 7) for i in range(2)])
        count = L.launch_count()
        with pytest.raises(L.H2Error, match="make 3 sets, got 2"):
            perm.construct(ev, pk, leaves * 2, l0, lb, ll, 2, 3, 5, 4, 5)
        assert L.launch_count() == count
        evaluated.close()
        assert not _Counting.live
        perm.close()
        pk.close()
    finally:
        for p in ev.polys:
            p.close()
        look.close()
