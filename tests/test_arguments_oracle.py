"""The permutation and lookup arguments' construct / evaluate / open and the column evaluations (halo2_b200.arguments) over
the ABI stand-in, without a GPU:

- a circuit with a selector-gated, two-row lookup (tests/arguments_cases.py) at k = 4 ... 6, two proofs and three
  permutation sets: tests/plonk_prover.create_proof_engine's proofs are accepted, a flipped byte or a wrong instance is
  rejected, and its compressed input and table differ between the coset compression and the extended Lagrange column;
- every argument error raises before any launch, and every object frees what it allocated on every path."""
import numpy as np
import pytest

import halo2_b200
from halo2_b200 import arguments as A
from halo2_b200 import lib as L
from tests import arguments_cases as AC
from tests import fake_engine
from tests import multiopen_cases as MC
from tests import plonk_api_circuit as circ
from tests import plonk_prover as PP
from tests import plonk_verifier as PV
from tests import prover_replay as R


def _gens(prm_gens):
    return tuple(np.asarray(g) for g in prm_gens)


def _nonlinear_proof(k, seed=11, instance=None, hook=None):
    prm, commit, gens = AC.params_for(halo2_b200, k)
    vk, D, fixed, sigma, advice, inst = AC.nonlinear_case(halo2_b200, k, commit, circ.ZETA, circ.DELTA)
    insts = [inst, inst] if instance is None else instance
    try:
        T = R.Blake2bTranscript(circ.M)
        PP.create_proof_engine(halo2_b200, prm, vk, fixed, sigma, [advice, advice], insts, MC.SeededRng("fp", seed, True), T, circ.ZETA, circ.DELTA,
                               on_construct=hook(D) if hook else None)
    finally:
        prm.close()
    return vk, bytes(T.proof), inst, gens


@pytest.mark.parametrize("k", [4, 5, 6])
def test_nonlinear_lookup_circuit_verifies(k):
    with fake_engine.installed() as fake:
        seen = []

        def hook(D):
            s, h = AC.coset_compression_differs(halo2_b200, D)
            seen.append(s)
            return h
        vk, proof, inst, gens = _nonlinear_proof(k, hook=hook)
        assert not fake.polys
    assert len(vk.permutation_columns) == 10 and vk.degree() - 2 == 4          # three sets
    assert seen[0] == [True] * 4                                   # input and table of both proofs
    arm = PV.OracleArm("vesta", k, *_gens(gens))
    assert PV.verify_proof(arm, vk, proof, [inst, inst], circ.DELTA)
    bad = bytearray(proof)
    bad[len(proof) // 2] ^= 1
    assert not PV.verify_proof(arm, vk, bytes(bad), [inst, inst], circ.DELTA)
    wrong = [[[inst[0][0] + 1]], inst]
    assert not PV.verify_proof(arm, vk, proof, wrong, circ.DELTA)


def test_nonlinear_lookup_circuit_with_the_wrong_public_input_is_rejected():
    """A proof made for another public input than the copy constraint ties to the witness fails verification."""
    with fake_engine.installed():
        vk, proof, inst, gens = _nonlinear_proof(4, instance=[[[5]], [[5]]])
    assert not PV.verify_proof(PV.OracleArm("vesta", 4, *_gens(gens)), vk, proof, [[[5]], [[5]]], circ.DELTA)


# ---- argument errors ---------------------------------------------------------------------------------------------------
def _setup(fake, k=4, sets=3, lookups=2):
    D = halo2_b200.EvaluationDomain("fp", 6, k, circ.ZETA)
    n, N = D.n, D.extended_len()
    rp = lambda length: halo2_b200.ResidentPoly("fp", length)     # noqa: E731
    from halo2_b200.keygen import PermutationProvingKey
    sig = [rp(n) for _ in range(4 * sets - 2)]
    pk = halo2_b200.ProvingKey([], [], [], PermutationProvingKey([], sig, [rp(N) for _ in sig]), None, None, None)
    perm = A.PermutationCommitted([(rp(n), rp(N), 7 + i) for i in range(sets)])
    permuted = [halo2_b200.Permuted(*[rp(n) for _ in range(6)], rp(N), rp(N), 3, 4) for _ in range(lookups)]
    look = A.LookupCommitted(permuted, [(rp(n), 5) for _ in range(lookups)])
    ev = halo2_b200.Evaluator(D, "extended")
    ls = [ev.register_poly(rp(N)) for _ in range(3)]
    cols = [ev.register_poly(rp(N)) for _ in sig]
    return D, pk, perm, look, ev, ls, cols


def _expect(fake, msg, fn):
    calls, polys = len(fake.calls), set(fake.polys)
    with pytest.raises(L.H2Error, match=msg):
        fn()
    assert len(fake.calls) == calls and set(fake.polys) == polys, msg


def test_argument_errors_raise_before_any_launch():
    with fake_engine.installed() as fake:
        D, pk, perm, look, ev, (l0, lb, ll), cols = _setup(fake)
        registered = len(ev.polys)
        c = lambda committed, **kw: committed.construct(ev, pk, kw.get("cols", cols), l0, lb, ll, 2, 3, 5, kw.get("chunk", 4), 5)  # noqa: E731
        _expect(fake, "10 permutation polynomials in chunks of 4 make 3 sets, got 2", lambda: c(A.PermutationCommitted(perm.sets[:2])))
        _expect(fake, "make 5 sets, got 3", lambda: c(perm, chunk=2))
        _expect(fake, "expected one column leaf per permutation polynomial", lambda: c(perm, cols=cols[:-1]))
        _expect(fake, "chunk_len must be at least 1", lambda: c(perm, chunk=0))
        short = [(halo2_b200.ResidentPoly("fp", D.n - 1), s[1], s[2]) if i == 1 else s for i, s in enumerate(perm.sets)]
        _expect(fake, r"permutation_product_poly\[1\]: a polynomial holds fewer than 16 elements", lambda: c(A.PermutationCommitted(short)))
        closed = halo2_b200.ResidentPoly("fp", D.extended_len())
        closed.close()
        bad = [(s[0], closed, s[2]) if i == 2 else s for i, s in enumerate(perm.sets)]
        _expect(fake, r"permutation_product_coset\[2\]: not an open resident polynomial", lambda: c(A.PermutationCommitted(bad)))
        other = [(halo2_b200.ResidentPoly("fq", D.n), s[1], s[2]) if i == 0 else s for i, s in enumerate(perm.sets)]
        _expect(fake, r"permutation_product_poly\[0\]: the polynomial lives in another field", lambda: c(A.PermutationCommitted(other)))
        _expect(fake, r"permutation_product_poly\[0\]", lambda: A.PermutationConstructed(A.PermutationCommitted(other), 5).evaluate(D, 9))
        assert len(ev.polys) == registered                         # a refused construct registers nothing
        a, b = cols[0], cols[1]
        exprs = [([a * b], [b]), ([a], [b + a])]
        lc = lambda committed, ex=exprs: committed.construct(ev, ex, 2, 3, 4, l0, lb, ll)   # noqa: E731
        _expect(fake, "2 permuted lookups but 1 product columns", lambda: lc(A.LookupCommitted(look.permuted, look.products[:1])))
        _expect(fake, "2 committed lookups but 1 lookup expressions", lambda: lc(look, exprs[:1]))
        _expect(fake, r"lookups\[1\]: 1 input expressions and 2 table expressions", lambda: lc(look, [exprs[0], ([a], [a, b])]))
        prods = [look.products[0], (closed, 5)]
        _expect(fake, r"products\[1\]: not an open resident polynomial", lambda: lc(A.LookupCommitted(look.permuted, prods)))
        short_coset = look.permuted[1]._replace(permuted_table_coset=halo2_b200.ResidentPoly("fp", D.extended_len() // 2))
        _expect(fake, r"permuted_table_coset\[1\]: a polynomial holds fewer than 128 elements",
                lambda: lc(A.LookupCommitted([look.permuted[0], short_coset], look.products)))
        _expect(fake, r"products\[1\]", lambda: A.LookupConstructed(A.LookupCommitted(look.permuted, prods), []).evaluate(D, 9))
        assert len(ev.polys) == registered
        fx = look.products[0][0]
        _expect(fake, "1 proofs' instance columns but 2 proofs' advice columns", lambda: A.evaluate_columns(D, 9, [[]], [[fx], [fx]], [], [], [(0, 0)], []))
        _expect(fake, r"advice_queries\[1\]: column 1 of 1", lambda: A.evaluate_columns(D, 9, [[]], [[fx]], [], [], [(0, 0), (1, 1)], []))
        _expect(fake, r"fixed polys\[0\]: not an open resident polynomial", lambda: A.evaluate_columns(D, 9, [[]], [[fx]], [closed], [], [], [(0, 0)]))
        _expect(fake, "one advice blind per advice column", lambda: A.open_columns(D, 9, [[]], [[fx]], [[]], [], [], [(0, 0)], []))


def test_objects_free_what_they_allocated_on_every_path(monkeypatch):
    """construct of the lookups makes the product cosets and frees them when the batched transform fails; each object's
    close frees its polynomials and those of what it was made from; evaluations allocate nothing."""
    with fake_engine.installed() as fake:
        D, pk, perm, look, ev, (l0, lb, ll), cols = _setup(fake)
        a, b = cols[0], cols[1]
        exprs = [([a * b], [b]), ([a], [b + a])]
        held = set(fake.polys)

        def failing(*args):
            fake.err = b"h2_poly_coeff_to_extended_batch: injected"
            return 1
        monkeypatch.setattr(fake, "h2_poly_coeff_to_extended_batch", failing)
        with pytest.raises(L.H2Error, match="injected"):
            look.construct(ev, exprs, 2, 3, 4, l0, lb, ll)
        assert set(fake.polys) == held
        monkeypatch.undo()
        constructed, es = look.construct(ev, exprs, 2, 3, 4, l0, lb, ll)
        assert len(es) == 10 and len(constructed.product_cosets) == 2
        assert fake.calls.count("h2_poly_coeff_to_extended_batch") == 1       # one batched transform for both lookups
        assert len(set(fake.polys) - held) == 2
        evaluated, evals = constructed.evaluate(D, 12345)
        assert len(evals) == 10 and fake.calls[-1] == "h2_poly_eval" and len(set(fake.polys) - held) == 2
        assert [q.point for q in evaluated.open(12345)][:3] == [12345] * 3
        pc, pes = perm.construct(ev, pk, cols, l0, lb, ll, 2, 3, 5, 4, 5)
        assert len(pes) == 2 + 2 + 3
        pe, pevals = pc.evaluate(D, 12345)
        assert len(pevals) == 3 * 2 + 2 and fake.calls[-1] == "h2_poly_eval"
        assert len(pe.open(12345)) == 3 * 2 + 2
        assert len(A.permutation_key_evaluate(pk, D, 7)) == 10 and len(A.permutation_key_open(pk, 7)) == 10
        own = [p._h.value for s in perm.sets for p in s[:2]] + [q._h.value for p in look.permuted for q in p[:8]] + [z._h.value for z, _ in look.products]
        evaluated.close()
        pe.close()
        assert not set(own + [c._h.value for c in constructed.product_cosets]) & set(fake.polys)
        evaluated.close()                                          # closing twice is harmless
