"""CPU checks of the column-batched transforms and of instance_commit / advice_commit: the batched NTT pass bodies on the
host emulation against the oracle's transforms, h2_poly_set_rows on the ABI stand-in (tests/fake_engine.py) against
per-column copies, and the two phases over the stand-in against
create_proof_engine's per-column composition on the plonk_api circuit."""
import ctypes

import numpy as np
import pytest

from oracle import cref, pasta
from tests import columns_cases as CC
from tests import fake_engine
from tests import plonk_api_circuit as circ
from tests.kernel_emul import build as emul_build


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emul_build.build())


def _batch(emu, field, mode, cols, in_log, log_n, omega, zeta=None, div=None, group=0, in_place=False, nthr=64):
    count = len(cols)
    stack = np.ascontiguousarray(np.stack(cols))
    out = np.zeros((count, 1 << log_n, 32), dtype=np.uint8)
    launches = emu.emu_ntt_batch(cref.FIELD_ID[field], mode, cref._p(stack), ctypes.c_uint64(count), in_log, log_n, cref._p(cref._fe(omega)),
                                 cref._p(cref._fe(zeta)) if zeta is not None else None, cref._p(cref._fe(div)) if div is not None else None,
                                 cref._p(out), ctypes.c_uint64(group), int(in_place), nthr)
    return out, launches


def _one_column_launches(log_n):
    return 1 if log_n <= 10 else -(-log_n // 7)      # ntt_plan: one pass up to 2^10, else passes of at most 7 stages


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_batched_bodies_equal_the_oracle(emu, field):
    """Columns of one size in one run: each equals the oracle's lagrange_to_coeff / coeff_to_extended, for 2^0 to 2^12, and
    a run issues the launches of one column."""
    m = pasta.FIELDS[field]
    zeta = pasta.zeta_candidates(field)[0]
    for k in range(0, 13):
        count = 3 if k < 11 else 2
        cols = [cref.gen_scalars(field, 1000 * k + c, 1 << k) for c in range(count)]
        w_inv, div = pasta.inv(pasta.omega_for_k(field, k), m), pasta.inv((1 << k) % m, m)
        got, launches = _batch(emu, field, 1, cols, k, k, w_inv, div=div, nthr=(7 if k < 6 else 64))
        for c in range(count):
            assert (got[c] == cref.ifft(field, cols[c], w_inv, k, div)).all(), (field, k, c)
        assert launches == _one_column_launches(k)
        ext_k = k + (2 if k <= 10 else 1)
        ew = pasta.omega_for_k(field, ext_k)
        got, launches = _batch(emu, field, 2, cols, k, ext_k, ew, zeta=zeta)
        for c in range(count):
            assert (got[c] == cref.coeff_to_extended(field, cols[c], k, ext_k, zeta, ew)).all(), (field, k, ext_k, c)
        assert launches == _one_column_launches(ext_k)


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_batched_bodies_in_place_and_in_groups(emu, field):
    """dst == src for every column, and a batch split into groups (the scratch cap) with a short last group: the same bytes."""
    m = pasta.FIELDS[field]
    for k in (4, 10, 11, 13):
        cols = [cref.gen_scalars(field, 77 + c, 1 << k) for c in range(5)]
        w_inv, div = pasta.inv(pasta.omega_for_k(field, k), m), pasta.inv((1 << k) % m, m)
        want = [cref.ifft(field, a, w_inv, k, div) for a in cols]
        got, _ = _batch(emu, field, 1, cols, k, k, w_inv, div=div, in_place=True)
        assert all((got[c] == want[c]).all() for c in range(5)), k
        got, launches = _batch(emu, field, 1, cols, k, k, w_inv, div=div, group=2)
        assert all((got[c] == want[c]).all() for c in range(5)), k
        assert launches == 3 * _one_column_launches(k)


def _gens():
    P = pasta.Params.new(pasta.VESTA, 5)
    return cref.affines_to_bytes(P.g), cref.affines_to_bytes(P.g_lagrange), cref.affines_to_bytes([P.w]), cref.affines_to_bytes([P.u])


def test_set_rows_equals_per_column_copies():
    import halo2_b200
    with fake_engine.installed() as fake:
        n, start, rows = 32, 26, 6
        cols = [cref.gen_scalars("fp", 5 + c, n) for c in range(4)]
        vals = [cref.gen_scalars("fp", 50 + c, rows) for c in range(4)]
        a = [halo2_b200.ResidentPoly("fp", n, c) for c in cols]
        b = [halo2_b200.ResidentPoly("fp", n, c) for c in cols]
        halo2_b200.set_rows_resident(a, start, np.stack(vals))
        assert fake.calls.count("h2_poly_set_rows") == 1
        for p, v in zip(b, vals):
            p.copy_from(halo2_b200.ResidentPoly("fp", rows, v), rows, dst_off=start)
        for x, y in zip(a, b):
            assert (x.download() == y.download()).all()
        with pytest.raises(halo2_b200.H2Error, match=r"h2_poly_set_rows: polys\[1\] is also polys\[0\]"):
            halo2_b200.set_rows_resident([a[0], a[0]], start, np.stack(vals[:2]))


def test_phases_of_the_plonk_api_circuit():
    """instance_commit and advice_commit over the stand-in equal create_proof_engine's instance and advice phases on the
    plonk_api circuit (k = 5, 5 advice columns, two proofs) under the same rng: the commitments in transcript order and the
    bytes of every column's values, polynomial and coset.  advice_commit makes one set_rows call, and the two phases one
    batched call per transform each."""
    import halo2_b200
    vk = circ.plonk_api_key()
    with fake_engine.installed() as fake:
        g, gl, w, u = _gens()
        prm = halo2_b200.Params("vesta", 5, g, gl, w, u=u)
        advice, instances = [circ.witness(), circ.witness()], [[[2]], [[2]]]
        want = CC.engine_phases(halo2_b200, prm, vk, advice, instances, 777, circ.ZETA)
        fake.calls.clear()
        got = CC.batched_phases(halo2_b200, prm, vk, advice, instances, 777, circ.ZETA)
        for name in ("h2_poly_set_rows", "h2_poly_lagrange_to_coeff_batch", "h2_poly_coeff_to_extended_batch"):
            assert fake.calls.count(name) == (1 if name == "h2_poly_set_rows" else 2), name
        assert fake.calls.count("h2_msm_registered_polys_affine") == 2
        assert len(want["written"]) == 10 and len(want["common"]) == 2
        CC.assert_same(want, got)
        prm.close()


def test_instance_too_large():
    import halo2_b200
    vk = circ.plonk_api_key()
    with fake_engine.installed():
        g, gl, w, u = _gens()
        prm = halo2_b200.Params("vesta", 5, g, gl, w, u=u)
        D = halo2_b200.EvaluationDomain("fp", vk.degree(), vk.k, circ.ZETA)
        bf = vk.blinding_factors()
        ok = halo2_b200.instance_commit(prm, D, [[[1] * (D.n - bf - 1)]], bf)
        for p in ok[0].values + ok[0].polys + ok[0].cosets:
            p.close()
        with pytest.raises(halo2_b200.InstanceTooLarge):
            halo2_b200.instance_commit(prm, D, [[[1]], [[1] * (D.n - bf)]], bf)
        prm.close()
