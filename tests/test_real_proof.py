"""CPU check that ties the PROVER side of the path to the reference's verification equation (no GPU): a real proof of the
reference's own test circuit (halo2_proofs/tests/plonk_api.rs:21-420: the "Combined add-mult" and "Public input" gates, a
lookup, a twelve-column permutation; k = 5) is produced by the oracle's restatements -- lagrange_to_coeff / coeff_to_extended /
extended_to_coeff (best_fft at G = scalar), divide_by_vanishing_poly, permute_expression_pair, eval_polynomial, kate_division,
commit / commit_lagrange, the multi-point opening, the opening argument; tests/plonk_prover.py restates plonk::create_proof
around them -- under the reference's GOLDEN verifying key, and is accepted by the verifier that the reference's sixteen golden
proofs pin (tests/plonk_verifier.py).  It has the golden proof's length, byte for byte the same layout."""
import pytest

from oracle import cref, pasta
from tests import fake_engine
from tests import multiopen_cases as MC
from tests import plonk_api_circuit as circ
from tests import plonk_prover as PP
from tests import plonk_verifier as PV
from tests import prover_replay as R
from tests.plonk_api_circuit import CASE, DELTA, M, ZETA, prove, witness

# the entry points of the prover phases and of key generation, and how often create_proof_engine calls each on the plonk_api
# circuit (two proofs, one lookup each): the transforms batch the instance columns, the advice columns and each proof's lookup
# products; key generation is not part of a proof
PHASE_CALLS = {"h2_poly_lagrange_to_coeff_batch": 2, "h2_poly_coeff_to_extended_batch": 2 + 2, "h2_poly_set_rows": 1,
               "h2_poly_lookup_permuted": 1, "h2_poly_permutation_product": 1, "h2_poly_lookup_product": 1, "h2_poly_vanishing_quotient": 1,
               "h2_poly_permutation_sigma": 0, "h2_poly_permutation_sigma_copies": 0}
# the finer calls a per-column composition of the same proof would make instead
FINER_CALLS = {"h2_poly_lookup_permute", "h2_poly_batch_invert", "h2_poly_running_product", "h2_poly_divide_by_vanishing",
               "h2_poly_extended_to_coeff"}


@pytest.fixture(scope="module")
def setup():
    c = pasta.VESTA
    P = pasta.Params.new(c, 5)                                     # Params::<EqAffine>::new(5)
    vk = PV.PinnedKey(CASE["key_text"])
    fixed = circ.fixed_columns(M, ZETA)                            # the circuit's fixed columns and permutation polynomials:
    sigma = circ.permutation_columns(M, vk.omega, DELTA)           # their commitments ARE the golden key's (tests/test_oracle_golden.py)
    gens = (cref.affines_to_bytes(P.g), cref.affines_to_bytes(P.g_lagrange), cref.affines_to_bytes([P.w]), cref.affines_to_bytes([P.u]))
    return c, P, vk, fixed, sigma, gens


def test_real_proof_of_the_reference_circuit_verifies(setup):
    c, P, vk, fixed, sigma, gens = setup
    arm = PV.OracleArm("vesta", 5, *gens)
    inst = [[[2]], [[2]]]
    proof = prove(setup, [witness(), witness()], inst, 777)
    assert len(proof) == len(CASE["proof"]) == 4160                # the same layout as tests/plonk_api_proof.bin
    assert PV.verify_proof(arm, vk, proof, inst, DELTA)
    assert proof != CASE["proof"]                                  # other randomness than the reference's OsRng run, of course
    # other randomness, another valid proof; the strategies of the reference's test accept it too
    proof2 = prove(setup, [witness(), witness()], inst, 778)
    assert proof2 != proof and PV.verify_proof(arm, vk, proof2, inst, DELTA)
    assert PV.verify_proof(arm, vk, proof2, inst, DELTA, process=arm.accumulate)
    # through the engine's host mirror (ABI stand-in): the same verdicts
    import halo2_b200
    with fake_engine.installed():
        earm = PV.EngineArm(halo2_b200, "vesta", 5, *gens)
        assert PV.verify_proof(earm, vk, proof, inst, DELTA)
        flipped = bytearray(proof)
        flipped[700] ^= 2
        assert not PV.verify_proof(earm, vk, bytes(flipped), inst, DELTA)
        earm.close()
    # the proof is bound to its public input and to every byte
    assert not PV.verify_proof(arm, vk, proof, [[[2]], [[3]]], DELTA)
    for off in (3, 1500, 4100):
        bad = bytearray(proof)
        bad[off] ^= 1
        assert not PV.verify_proof(arm, vk, bytes(bad), inst, DELTA)


def test_single_instance_and_unsatisfied_witness(setup):
    c, P, vk, fixed, sigma, gens = setup
    arm = PV.OracleArm("vesta", 5, *gens)
    one = prove(setup, [witness()], [[[2]]], 900)
    assert len(one) < 4160 and PV.verify_proof(arm, vk, one, [[[2]]], DELTA)
    # a witness that violates the multiplication gate in one row: the quotient is no polynomial, the prover still runs (like the
    # reference's, which checks nothing), and the verifier rejects
    bad = prove(setup, [witness(break_row=5)], [[[2]]], 901)
    assert not PV.verify_proof(arm, vk, bad, [[[2]]], DELTA)
    # a public input the witness does not match (the "Public input" gate, sp * (a - p))
    wrong = prove(setup, [witness()], [[[3]]], 902)
    assert not PV.verify_proof(arm, vk, wrong, [[[3]]], DELTA)


def test_real_proof_through_the_engine_api(setup):
    """The same prover composed from the engine's phase calls (tests/plonk_prover.create_proof_engine: instance_commit /
    advice_commit, the lookups' permuted and product columns, the permutation products, the vanishing argument, the arguments'
    construct / evaluate / open, halo2_b200.multiopen / opening) over the ABI stand-in -- transforms and group operations
    through the oracle, the device bodies on the host emulation: with the same seeded randomness it writes THE SAME 4 160 BYTES
    as the oracle's prover, through one call of each phase entry point and none of the finer calls, frees every resident
    polynomial it allocated, and the golden-proof-pinned verifier accepts the bytes."""
    import halo2_b200
    c, P, vk, fixed, sigma, gens = setup
    inst = [[[2]], [[2]]]
    want = prove(setup, [witness(), witness()], inst, 777)
    with fake_engine.installed() as fake:
        prm = halo2_b200.Params("vesta", 5, gens[0], gens[1], gens[2], u=gens[3])
        T = R.Blake2bTranscript(M)
        PP.create_proof_engine(halo2_b200, prm, vk, fixed, sigma, [witness(), witness()], inst, MC.SeededRng("fp", 777, True), T, ZETA, DELTA)
        got = bytes(T.proof)
        assert len(got) == 4160 and got == want
        assert {name: fake.calls.count(name) for name in PHASE_CALLS} == PHASE_CALLS
        assert not FINER_CALLS & set(fake.calls)
        assert not fake.polys                                      # every resident polynomial the prover allocated is released
        earm = PV.EngineArm(halo2_b200, "vesta", 5, *gens)
        assert PV.verify_proof(earm, vk, got, inst, DELTA)
        earm.close()
        prm.close()


@pytest.mark.parametrize("k", [4, 6])
def test_benchmark_circuit_real_proof(k):
    """The circuit of the reference's prover benchmark (benches/plonk.rs: StandardPlonk, every usable row filled; rebuilt in
    tests/bench_circuit.py) with a key generated here (commit_lagrange of its fixed and permutation columns, Blind::default(),
    plonk/keygen.rs:233-236): the oracle's prover and the engine's phase composition (over the ABI stand-in, the proving key's
    resident polynomials kept between two proofs in a dict, as `bench.py` keeps them) write the same proof, and both verifiers
    accept it.  This is the workload `bench.py`'s `extra.create_proof_k14_real` times on the GPU at k = 14."""
    import halo2_b200
    from tests import bench_circuit as BC
    c = pasta.VESTA
    n = 1 << k
    pts = cref.gen_points("vesta", 99, n + 2)
    A = cref.bytes_to_affine
    P = pasta.Params.from_generators(c, k, [A(x) for x in pts[:n]], A(pts[n]), A(pts[n + 1]))
    D = pasta.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
    fixed, sigma, adv = BC.columns(k, M, D.omega, DELTA, circ.A_SMALL * ZETA % M)
    cl = lambda v: pasta.to_affine(c, pasta.best_multiexp(c, list(v) + [1], P.g_lagrange + [P.w]))
    vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, c.p, M, D.omega, [cl(f) for f in fixed], [cl(s_) for s_ in sigma]))
    assert (vk.degree(), vk.blinding_factors(), vk.extended_k) == (5, BC.BLINDING_FACTORS, k + 2)
    W = R._WriteT(M)
    PP.create_proof(c, P.g, P.g_lagrange, P.w, P.u, vk, fixed, sigma, [adv], [[]], MC.SeededRng("fp", 5, False), W, ZETA, DELTA)
    want = bytes(W.T.proof)
    # 3 advice + 1 permutation product + random + 4 h pieces + f + s + 2k rounds; 3 + 4 + 1 + 3 + 2 evaluations + the q's + c, f
    gens = (cref.affines_to_bytes(P.g), cref.affines_to_bytes(P.g_lagrange), cref.affines_to_bytes([P.w]), cref.affines_to_bytes([P.u]))
    assert PV.verify_proof(PV.OracleArm("vesta", k, *gens), vk, want, [[]], DELTA)
    with fake_engine.installed() as fake:
        prm = halo2_b200.Params("vesta", k, gens[0], gens[1], gens[2], u=gens[3])
        pk = {}
        adv_bytes = [cref.ints_to_bytes(col) for col in adv]
        for seed, expect in ((5, want), (6, None)):
            T = R.Blake2bTranscript(M)
            PP.create_proof_engine(halo2_b200, prm, vk, fixed, sigma, [adv_bytes], [[]], MC.SeededRng("fp", seed, True), T, ZETA, DELTA, pk=pk)
            got = bytes(T.proof)
            assert expect is None or got == expect
            assert not FINER_CALLS & set(fake.calls)
            earm = PV.EngineArm(halo2_b200, "vesta", k, params=prm)
            assert PV.verify_proof(earm, vk, got, [[]], DELTA)
            earm.close()
        assert all(p._h.value for p in pk["key"].fixed_cosets)         # the key's polynomials stayed resident between the proofs
        # the timed CPU arm of bench.py's extra.create_proof_k14_real: the same prover on the C restatement, the same bytes
        cp = PP.CrefProver(cref, "vesta", "fp", *gens, threads=4)
        T = R.Blake2bTranscript(M)
        cp.create_proof(vk, fixed, sigma, [adv_bytes], [[]], MC.SeededRng("fp", 5, True), T, ZETA, DELTA)
        assert bytes(T.proof) == want and cp.hot_s > 0 and set(cp.by_kind) >= {"commit", "commit_lagrange", "ipa", "kate_division"}
        PP.close_proving_key(pk)
        assert not fake.polys
        prm.close()


def test_cref_prover_matches_the_oracle_on_the_reference_circuit(setup):
    """PP.CrefProver (the C restatement's hot calls under the same control flow: the timed CPU arm for real proofs) on the
    plonk_api circuit -- lookup, instance column, six permutation sets, two instances: the oracle prover's 4 160 bytes."""
    c, P, vk, fixed, sigma, gens = setup
    inst = [[[2]], [[2]]]
    want = prove(setup, [witness(), witness()], inst, 777)
    cp = PP.CrefProver(cref, "vesta", "fp", *gens, threads=4)
    T = R.Blake2bTranscript(M)
    cp.create_proof(vk, fixed, sigma, [witness(), witness()], inst, MC.SeededRng("fp", 777, True), T, ZETA, DELTA)
    assert bytes(T.proof) == want
