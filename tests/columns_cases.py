"""The instance and advice phases of plonk::create_proof two ways, for the column tests: a composition of per-column calls
and halo2_b200.instance_commit / advice_commit.  Both return the same record: the points in transcript order and the bytes
of every column's values, coefficient form and coset."""
from __future__ import annotations

import numpy as np

from oracle import cref
from tests import multiopen_cases as MC


def composition_phases(h2, prm, D, bf: int, advice, instances, seed: int) -> dict:
    """The instance and advice phases one column at a time under SeededRng(seed): each column uploaded (an advice column's
    last n - usable rows overwritten with the rng's draws, prover.rs:276-282), the columns of a proof committed in one pass
    (instances with Blind::default(), advice with one drawn blind per column), then lagrange_to_coeff and coeff_to_extended
    per column.  Closes what it made."""
    rng = MC.SeededRng(D.field, seed, True)
    n, usable = D.n, D.n - (bf + 1)
    rec = {"common": [], "written": [], "values": [], "polys": [], "cosets": []}
    live = []

    def resident(vals, length=n):
        p = h2.ResidentPoly(D.field, length, None if vals is None else vals if hasattr(vals, "dtype") else cref.ints_to_bytes([v % D.m for v in vals]))
        live.append(p)
        return p

    def transform(vals):
        polys = [D.lagrange_to_coeff_resident(v, out=resident(None)) for v in vals]
        cosets = [D.coeff_to_extended_resident(p, out=resident(None, D.extended_len())) for p in polys]
        rec["values"] += [v.download(n) for v in vals]
        rec["polys"] += [p.download(n) for p in polys]
        rec["cosets"] += [c.download(D.extended_len()) for c in cosets]

    def commit(vals, blinds):
        return list(prm.commit_resident_affine(vals, [h2.Blind(b) for b in blinds], lagrange=True)) if vals else []

    try:
        for inst in instances:
            vals = [resident(list(col) + [0] * (n - len(col))) for col in inst]
            rec["common"] += commit(vals, [1] * len(vals))
            transform(vals)
        for cols in advice:
            vals = []
            for col in cols:
                v = resident(col)
                v.copy_from(resident([rng.scalar() for _ in range(n - usable)], n - usable), n - usable, dst_off=usable)
                vals.append(v)
            rec["written"] += commit(vals, [rng.scalar() for _ in vals])
            transform(vals)
    finally:
        for p in live:
            p.close()
    return rec


def batched_phases(h2, prm, D, bf: int, advice, instances, seed: int) -> dict:
    """instance_commit and advice_commit on the same inputs under SeededRng(seed); closes what they made."""
    inst = h2.instance_commit(prm, D, instances, bf)
    adv = h2.advice_commit(prm, D, advice, MC.SeededRng(D.field, seed, True), bf)
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
