"""CPU checks of shared proving keys on the host side (halo2_b200.ProvingKey.share, ResidentPoly.share / shared / close) over
an ABI stand-in: the key goes to h2_poly_share in one call that holds every one of its polynomials, a failed share leaves
nothing marked shared, and the entry point is declared in the header and exported by lib.SYMBOLS."""

import numpy as np
import pytest

from oracle import pasta
from tests import bench_circuit as BC
from tests import fake_engine
from tests.abi_cases import _header_symbols
from tests.plonk_api_circuit import ZETA
from tests.plonk_verifier import scalar_delta


@pytest.fixture
def fake():
    with fake_engine.installed() as f:
        yield f


def _small_key(h2, k=4):
    m = pasta.P_MOD
    n = 1 << k
    _, _, gens, fixed, _, _, copies = BC._bench_setup(k)
    prm = h2.Params("vesta", k, *gens[:3], u=gens[3])
    D = h2.EvaluationDomain("fp", BC.DEGREE, k, ZETA)
    asm = h2.Assembly(n, 3)
    for cp in copies:
        asm.copy(*cp)
    return prm, h2.keygen_pk(prm, D, fixed, asm, scalar_delta(m), BC.BLINDING_FACTORS)


def test_proving_key_share_is_one_call_with_every_polynomial(fake):
    import halo2_b200 as h2
    prm, pk = _small_key(h2)
    polys = pk._all()
    assert len(polys) == 3 * 4 + 3 * 3 + 3                          # fixed and sigma columns in three forms, l_0 / l_blind / l_last
    assert not any(p.shared for p in polys)
    fake.calls.clear()
    assert pk.share() is pk
    assert fake.share_calls == [[p._h.value for p in polys]]
    assert all(p.shared for p in polys)
    assert fake.shared == {p._h.value for p in polys}
    handles = [p._h.value for p in polys]
    pk.close()
    assert fake.freed[-len(handles):] == handles and not fake.shared
    assert all(p._h.value == 0 for p in polys)
    prm.close()
    assert not fake.polys


def test_resident_poly_share_and_close(fake):
    import halo2_b200 as h2
    p = h2.ResidentPoly("fp", 8, np.zeros((8, 32), dtype=np.uint8))
    q = h2.ResidentPoly("fp", 8)
    assert not p.shared and not q.shared
    h = p._h.value
    assert p.share() is p
    assert p.shared and not q.shared
    assert fake.share_calls == [[h]]
    p.close()
    assert fake.freed == [h] and h not in fake.polys and p._h.value == 0
    q.close()
    assert not fake.polys


def test_failed_share_marks_nothing(fake):
    import halo2_b200 as h2
    p = h2.ResidentPoly("fp", 8)
    gone = h2.ResidentPoly("fp", 8)
    gone_h = gone._h.value
    gone.close()
    gone._h.value = gone_h                                          # a handle the library no longer knows
    with pytest.raises(h2.H2Error, match="unknown"):
        h2.share_resident([p, gone])
    assert not p.shared and not gone.shared and not fake.shared
    gone._h.value = 0
    p.close()


def test_header_declares_h2_poly_share():
    from halo2_b200 import lib as L
    assert "h2_poly_share" in _header_symbols()
    assert "h2_poly_share" in L.SYMBOLS
    assert sorted(L.SYMBOLS) == _header_symbols()
