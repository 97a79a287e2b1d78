"""The instance and advice phases of plonk::create_proof two ways, for the column tests: create_proof_engine's per-column
composition (run up to its first challenge) and halo2_b200.instance_commit / advice_commit.  Both return the same record:
the points in transcript order and the bytes of every column's values, coefficient form and coset."""
from __future__ import annotations

import contextlib
import ctypes

import numpy as np

from oracle import cref, pasta
from tests import fake_engine
from tests import multiopen_cases as MC
from tests import plonk_prover as PP
from tests import prover_replay as R


class _Stop(Exception):
    pass


class ShapeKey:
    """What create_proof_engine reads from a key before its first challenge, for a circuit shape without a pinned key."""

    def __init__(self, field: str, k: int, degree: int, blinding_factors: int, zeta: int):
        self.scalar_modulus, self.k, self._deg, self._bf = pasta.FIELDS[field], k, degree, blinding_factors
        d = pasta.EvaluationDomain(field, degree, k, zeta)
        self.extended_k, self.omega = d.extended_k, d.omega

    def blinding_factors(self) -> int:
        return self._bf

    def degree(self) -> int:
        return self._deg

    def transcript_repr(self) -> int:
        return 0


def _skip_key():
    """A proving-key dict that makes create_proof_engine skip its keygen part (the phases here do not read it)."""
    return {"fixed_l": [], "fixed_p": [], "fixed_c": [], "sigma_l": [], "sigma_p": [], "sigma_c": [], "l": [None, None, None]}


def engine_phases(h2, prm, vk, advice, instances, seed: int, zeta: int) -> dict:
    """create_proof_engine through its instance and advice phases, under SeededRng(seed)."""
    field = {pasta.P_MOD: "fp", pasta.Q_MOD: "fq"}[vk.scalar_modulus]
    rec = {"common": [], "written": [], "values": [], "polys": [], "cosets": []}

    class D(h2.EvaluationDomain):
        def lagrange_to_coeff_resident(self, a, out=None):
            rec["values"].append(a.download(self.n))
            r = super().lagrange_to_coeff_resident(a, out)
            rec["polys"].append(r.download(self.n))
            return r

        def coeff_to_extended_resident(self, a, out=None):
            r = super().coeff_to_extended_resident(a, out)
            rec["cosets"].append(r.download(self.extended_len()))
            return r

    class Eng:
        EvaluationDomain = D

        def __getattr__(self, name):
            return getattr(h2, name)

    class T(R.Blake2bTranscript):
        def common_point(self, xy):
            rec["common"].append(np.array(xy, dtype=np.uint8).reshape(64))
            super().common_point(xy)

        def write_point(self, xy):
            rec["written"].append(np.array(xy, dtype=np.uint8).reshape(64))
            super().write_point(xy)

        def squeeze_challenge(self):
            raise _Stop()

    try:
        PP.create_proof_engine(Eng(), prm, vk, [], [], advice, instances, MC.SeededRng(field, seed, True), T(vk.scalar_modulus), zeta, 0,
                               pk=_skip_key())
    except _Stop:
        pass
    return rec


def batched_phases(h2, prm, vk, advice, instances, seed: int, zeta: int) -> dict:
    """instance_commit and advice_commit on the same inputs under SeededRng(seed); closes what they made."""
    field = {pasta.P_MOD: "fp", pasta.Q_MOD: "fq"}[vk.scalar_modulus]
    D = h2.EvaluationDomain(field, vk.degree(), vk.k, zeta)
    bf = vk.blinding_factors()
    inst = h2.instance_commit(prm, D, instances, bf)
    adv = h2.advice_commit(prm, D, advice, MC.SeededRng(field, seed, True), bf)
    rec = {"common": [c for s in inst for c in s.commitments], "written": [c for s in adv for c in s.commitments],
           "values": [], "polys": [], "cosets": []}
    for s in list(inst) + list(adv):
        rec["values"] += [p.download(D.n) for p in s.values]
        rec["polys"] += [p.download(D.n) for p in s.polys]
        rec["cosets"] += [p.download(D.extended_len()) for p in s.cosets]
        for p in s.values + s.polys + s.cosets:
            p.close()
    return rec


def assert_same(want: dict, got: dict) -> None:
    for key in ("common", "written", "values", "polys", "cosets"):
        assert len(want[key]) == len(got[key]), key
        for i, (a, b) in enumerate(zip(want[key], got[key])):
            assert np.array_equal(np.asarray(a, dtype=np.uint8), np.asarray(b, dtype=np.uint8)), (key, i)


def random_columns(field: str, seed: int, proofs: int, columns: int, n: int):
    return [[cref.gen_scalars(field, seed + 100 * p + c, n) for c in range(columns)] for p in range(proofs)]


class ColumnsFake(fake_engine.FakeLib):
    """The ABI stand-in with the column-batched transforms (the batched pass bodies on the host emulation,
    emul_ntt_batch.cpp) and h2_poly_set_rows, with the library's checks that the host mirror can reach."""

    def _transform_batch(self, who, mode, dst, src, count, in_log, log_n, omega, zeta, divisor):
        self._log(who)
        count = fake_engine._v(count)
        if count == 0:
            return 0
        d, s = [int(dst[i]) for i in range(count)], [int(src[i]) for i in range(count)]
        c = fake_engine.clash(fake_engine.args("dst", d, True) + fake_engine.args("src", s, False), in_place=("dst", "src"))
        if c:
            return self._fail(f"{who}: {c}")
        f = self.polys[s[0]][0]
        in_log, log_n = fake_engine._v(in_log), fake_engine._v(log_n)
        rd = fake_engine._rd
        stack = np.ascontiguousarray(np.stack([self.polys[h][1][:1 << in_log] for h in s]))
        out = np.zeros((count, 1 << log_n, 32), dtype=np.uint8)
        self.emu.emu_ntt_batch(cref.FIELD_ID[f], mode, cref._p(stack), ctypes.c_uint64(count), in_log, log_n, cref._p(rd(omega, 32)),
                               cref._p(rd(zeta, 32)) if zeta is not None else None, cref._p(rd(divisor, 32)) if divisor is not None else None,
                               cref._p(out), ctypes.c_uint64(0), 0, 64)
        for i, h in enumerate(d):
            self.polys[h][1][:1 << log_n] = out[i]
        return 0

    def h2_poly_lagrange_to_coeff_batch(self, dst, src, count, k, omega_inv, divisor, repr_):
        return self._transform_batch("h2_poly_lagrange_to_coeff_batch", 1, dst, src, count, k, k, omega_inv, None, divisor)

    def h2_poly_coeff_to_extended_batch(self, dst, src, count, k, ext_k, zeta, ext_omega, repr_):
        return self._transform_batch("h2_poly_coeff_to_extended_batch", 2, dst, src, count, k, ext_k, ext_omega, zeta, None)

    def h2_poly_set_rows(self, polys, count, start, rows, values, repr_):
        self._log("h2_poly_set_rows")
        count, start, rows = fake_engine._v(count), fake_engine._v(start), fake_engine._v(rows)
        if count == 0 or rows == 0:
            return 0
        hs = [int(polys[i]) for i in range(count)]
        short = [i for i, h in enumerate(hs) if start + rows > self.polys[h][1].shape[0]]
        if short:
            return self._fail(f"h2_poly_set_rows: polys[{short[0]}]: a polynomial holds fewer than start + rows elements")
        c = fake_engine.clash(fake_engine.args("polys", hs, True))
        if c:
            return self._fail(f"h2_poly_set_rows: {c}")
        vals = fake_engine._rd(values, 32 * count * rows).reshape(count, rows, 32)
        for i, h in enumerate(hs):
            self.polys[h][1][start:start + rows] = vals[i]
        return 0


@contextlib.contextmanager
def installed():
    """halo2_b200.lib bound to a ColumnsFake for the duration of the block (and back to whatever it was afterwards)."""
    from halo2_b200 import lib as L
    saved = (L._lib, L._inited_device)
    fake = ColumnsFake()
    L._lib, L._inited_device = fake, 0
    try:
        yield fake
    finally:
        L._lib, L._inited_device = saved
