"""CPU checks of shared proving keys on the host side (halo2_b200.ProvingKey.share, ResidentPoly.share / shared / close) over
an ABI stand-in: the key goes to h2_poly_share in one call that holds every one of its polynomials, a failed share leaves
nothing marked shared, and the entry point is declared in the header and exported by lib.SYMBOLS."""

import numpy as np
import pytest

from tests import bench_circuit as BC
from tests import fake_engine
from tests import test_keygen_oracle as KO
from tests.test_abi import _header_symbols


class SharingFakeLib(KO.KeygenFakeLib):
    """The keygen stand-in plus h2_poly_share with the library's all-or-nothing rule (the calling context's or already
    shared handles only), recording each call's handles."""

    def __init__(self):
        super().__init__()
        self.shared, self.share_calls, self.freed = set(), [], []

    def h2_poly_share(self, polys, n):
        n = fake_engine._v(n)
        hs = [int(x) for x in polys[:n]]
        self.share_calls.append(hs)
        if any(h not in self.polys for h in hs):
            return self._fail("h2_poly_share: unknown polynomial handle")
        self.shared.update(hs)
        return 0

    def h2_poly_free(self, h):
        self.freed.append(fake_engine._v(h))
        self.shared.discard(fake_engine._v(h))
        return super().h2_poly_free(h)


def _installed(monkeypatch):
    from halo2_b200 import lib as L
    fake = SharingFakeLib()
    monkeypatch.setattr(L, "_lib", fake)
    monkeypatch.setattr(L, "_inited_device", 0)
    return fake


def _small_key(h2, k=4):
    m = KO.pasta.P_MOD
    n = 1 << k
    _, _, gens, fixed, _, _, copies = KO._bench_setup(k)
    prm = h2.Params("vesta", k, *gens[:3], u=gens[3])
    D = h2.EvaluationDomain("fp", BC.DEGREE, k, KO.ZETA)
    asm = h2.Assembly(n, 3)
    for cp in copies:
        asm.copy(*cp)
    return prm, h2.keygen_pk(prm, D, fixed, asm, KO.delta_of(m), BC.BLINDING_FACTORS)


def test_proving_key_share_is_one_call_with_every_polynomial(monkeypatch):
    import halo2_b200 as h2
    fake = _installed(monkeypatch)
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


def test_resident_poly_share_and_close(monkeypatch):
    import halo2_b200 as h2
    fake = _installed(monkeypatch)
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


def test_failed_share_marks_nothing(monkeypatch):
    import halo2_b200 as h2
    fake = _installed(monkeypatch)
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
