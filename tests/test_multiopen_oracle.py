"""CPU checks of the multi-point opening argument (no GPU): the oracle's restatement of poly/multiopen against the
reference's own tests -- `test_roundtrip` (poly/multiopen.rs:278-373), `test_identical_queries` (:375-481), the
`test_intermediate_sets` property (:556-627) -- a PLONK-shaped query list with rotations, lagrange_interpolate
(arithmetic.rs:376-432), and the engine's host mirror (halo2_b200.multiopen / opening) over tests/fake_engine.py: the same
proof bytes as the oracle, accepted by both verifiers."""
import numpy as np
import pytest

from oracle import cref, pasta
from tests import fake_engine
from tests import multiopen_cases as MC

SEED = MC.SEED


def _gens(curve, k, real):
    c = pasta.CURVES[curve]
    n = 1 << k
    if real:                                                       # Params::new(K): hash_to_curve generators
        g, w, u = pasta.params_generators(c, k)
        return cref.affines_to_bytes(g), cref.affines_to_bytes([w]), cref.affines_to_bytes([u])
    pts = cref.gen_points(curve, SEED + 1, n + 2)
    return pts[:n], pts[n:n + 1], pts[n + 1:n + 2]


@pytest.fixture()
def eng():
    import halo2_b200
    with fake_engine.installed() as fake:
        halo2_b200._fake = fake
        yield halo2_b200
        del halo2_b200._fake


def test_roundtrip_and_identical_queries_oracle():
    g, w, u = _gens("vesta", 4, real=True)                          # Params::<EqAffine>::new(4)
    MC.roundtrip(MC.OracleSide("vesta", 4, g, w, u), "fp")


def test_roundtrip_host_mirror_matches_oracle(eng):
    g, w, u = _gens("vesta", 3, real=False)
    want = MC.roundtrip(MC.OracleSide("vesta", 3, g, w, u), "fp")
    side = MC.EngineSide(eng, "vesta", 3, g, w, u)
    got = MC.roundtrip(side, "fp")
    assert got == want
    # a repeated (polynomial, point) query: the reference's prover returns io::Error InvalidInput (prover.rs:41-46)
    p = eng.ResidentPoly("fp", 8, cref.ints_to_bytes(list(range(8))))
    from tests import prover_replay as R
    with pytest.raises(ValueError):
        eng.multiopen.create_proof(side.params, MC.SeededRng("fp", 1, True), R.Blake2bTranscript(),
                                   [eng.multiopen.ProverQuery(5, p, eng.Blind(1)), eng.multiopen.ProverQuery(5, p, eng.Blind(1))])
    side.close()


@pytest.mark.parametrize("curve,k", [("vesta", 3), ("pallas", 2)])
def test_plonk_shaped_queries(eng, curve, k):
    """Rotations: point sets {x, xw} (two columns, queried in different orders), {x}, {x, xw, xw^-1} -- lagrange_interpolate
    through two and three points, successive kate divisions, the x_2 fold over three sets."""
    c = pasta.CURVES[curve]
    g, w, u = _gens(curve, k, real=False)
    polys, blinds, plan = MC.plonk_shaped(c.scalar, k, SEED + 40)
    osd = MC.OracleSide(curve, k, g, w, u)
    esd = MC.EngineSide(eng, curve, k, g, w, u)
    proof = osd.prove(polys, blinds, plan, SEED + 50)
    assert esd.prove(polys, blinds, plan, SEED + 50) == proof
    # 3 sets -> f commitment, 3 evaluations, the opening
    assert len(proof) == 32 * (1 + 3 + 1 + 2 * k + 2)
    oc = [osd.commit(p, b) for p, b in zip(polys, blinds)]
    ec = [esd.commit(p, b) for p, b in zip(polys, blinds)]
    assert [cref.bytes_to_affine(x) for x in ec] == oc
    good = MC.evals_for(c.scalar, polys, plan)
    assert osd.verify(proof, oc, good) and esd.verify(proof, ec, good)
    for j in (0, 3, 5, 7):                                          # one wrong evaluation, in each kind of set
        bad = list(good)
        bad[j] = (bad[j][0], bad[j][1], (bad[j][2] + 1) % c.r)
        assert not osd.verify(proof, oc, bad) and not esd.verify(proof, ec, bad), j
    swapped = [ec[1], ec[0]] + ec[2:]                               # the right evaluations against the wrong commitments
    assert not esd.verify(proof, swapped, good)
    flip = bytearray(proof)
    flip[32 * 2 + 1] ^= 4                                           # one of the q evaluations
    assert not esd.verify(bytes(flip), ec, good) and not osd.verify(bytes(flip), oc, good)
    # the verifier accepts an MSM of commitments in place of a commitment (CommitmentReference::MSM, verifier.rs:62-66):
    # column 1 = 2 * column 1' + 3 * column 0 as an MSM over the two commitments
    r = c.r
    half = [(p1 - 3 * p0) * pow(2, -1, r) % r for p0, p1 in zip(polys[0], polys[1])]
    half_blind = (blinds[1] - 3 * blinds[0]) * pow(2, -1, r) % r
    hc = esd.commit(half, half_blind)
    m_e = eng.MSM(esd.params)
    m_e.append_term(2, hc)
    m_e.append_term(3, ec[0])
    assert esd.verify(proof, [ec[0], m_e] + ec[2:], good)
    m_o = pasta.MSM(osd.c, osd.g, osd.w, osd.u)
    m_o.append_term(2, cref.bytes_to_affine(hc))
    m_o.append_term(3, oc[0])
    assert osd.verify(proof, [oc[0], m_o] + oc[2:], good)
    esd.close()


def test_intermediate_sets_property():
    """multiopen.rs:556-627 (`test_intermediate_sets`): the set indices and point indices depend on WHICH queries share points,
    not on the points' values; and point_sets lists every set's points in point-index order."""
    from halo2_b200.multiopen import VerifierQuery, construct_intermediate_sets
    rng = np.random.default_rng(SEED)
    for trial in range(40):
        num_points, num_cols, num_queries = 8, 8, 16
        pairs = set()
        while len(pairs) < num_queries:
            pairs.add((int(rng.integers(num_cols)), int(rng.integers(num_points))))
        pairs = list(pairs)
        rng.shuffle(pairs)
        cols = [object() for _ in range(num_cols)]
        outs = []
        for rep in range(2):
            pts = cref.bytes_to_ints(cref.gen_scalars("fp", SEED + 100 * trial + rep, num_points))
            ev = cref.bytes_to_ints(cref.gen_scalars("fp", SEED + 100 * trial + rep + 50, num_queries))
            mine = construct_intermediate_sets([VerifierQuery(cols[cm], pts[pi], e) for (cm, pi), e in zip(pairs, ev)])
            theirs = pasta.construct_intermediate_sets([pasta.VerifierQuery(cols[cm], pts[pi], e) for (cm, pi), e in zip(pairs, ev)], prover=False)
            assert mine is not None and theirs is not None
            data, point_sets = mine
            assert [(d.set_index, d.point_indices, d.evals) for d in data] == [(t["set_index"], t["point_indices"], t["evals"]) for t in theirs[0]]
            assert point_sets == theirs[1]
            for d in data:                                          # every commitment's evals sit in its set's point order
                first_seen = {}
                for (cm, pi), e in zip(pairs, ev):
                    if cols[cm] is d.commitment:
                        first_seen[pts[pi]] = e
                assert [first_seen[p] for p in point_sets[d.set_index]] == d.evals
            outs.append([(d.set_index, d.point_indices) for d in data])
        assert outs[0] == outs[1]
    # a repeated (commitment, point) pair
    cm = object()
    assert construct_intermediate_sets([VerifierQuery(cm, 5, 1), VerifierQuery(cm, 5, 2)]) is None
    assert pasta.construct_intermediate_sets([pasta.VerifierQuery(cm, 5, 1), pasta.VerifierQuery(cm, 5, 2)], prover=False) is None


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_lagrange_interpolate(field):
    """arithmetic.rs:376-432 and its test (:460-478): the interpolant passes through the points; both restatements agree."""
    from halo2_b200.multiopen import lagrange_interpolate
    m = pasta.FIELDS[field]
    for npts in (1, 2, 3, 5, 9):
        pts = cref.bytes_to_ints(cref.gen_scalars(field, SEED + npts, npts))
        ev = cref.bytes_to_ints(cref.gen_scalars(field, SEED + npts + 20, npts))
        co = pasta.lagrange_interpolate(m, pts, ev)
        assert len(co) == npts and [pasta.eval_polynomial_mod(m, co, p) for p in pts] == ev
        assert lagrange_interpolate(pts, ev, m) == co


@pytest.mark.parametrize("field", ["fq", "fp"])
def test_l_i(field):
    """poly/domain.rs:541-569 (`test_l_i`, pallas::Scalar, k = 3): l_i_range(x, x^n, -7..=7) against the Lagrange basis polynomials
    built by lagrange_interpolate over the domain -- on the oracle's EvaluationDomain and on the host mirror's (host arithmetic:
    the mirror's constructor and these two methods touch no device); rotate_omega alongside (domain.rs:408-418)."""
    import halo2_b200
    m = pasta.FIELDS[field]
    for D in (pasta.EvaluationDomain(field, 1 + 1, 3), halo2_b200.EvaluationDomain(field, 1 + 1, 3, pasta.zeta_candidates(field)[0])):
        points = [pow(D.omega, i, m) for i in range(8)]
        basis = [pasta.lagrange_interpolate(m, points, [1 if j == i else 0 for j in range(8)]) for i in range(8)]
        x = cref.bytes_to_ints(cref.gen_scalars(field, SEED + 77, 1))[0]
        xn = pow(x, 8, m)
        ev = D.l_i_range(x, xn, range(-7, 8))
        assert len(ev) == 15
        for i in range(8):
            assert pasta.eval_polynomial_mod(m, basis[i], x) == ev[7 + i]
            assert pasta.eval_polynomial_mod(m, basis[(8 - i) % 8], x) == ev[7 - i]
        assert D.rotate_omega(x, 3) == x * pow(D.omega, 3, m) % m and D.rotate_omega(x, -2) * pow(D.omega, 2, m) % m == x
        assert D.rotate_omega(D.rotate_omega(x, 5), -5) == x
