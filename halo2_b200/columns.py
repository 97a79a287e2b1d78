"""The prover's instance and advice columns over the C ABI: the instance part of plonk::create_proof
(/root/reference/halo2_proofs/src/plonk/prover.rs:79-124) and the advice part (:269-335), every column of every proof at once:
one commitment pass, then one column-batched lagrange_to_coeff and one coeff_to_extended (csrc/ntt.cuh), so each NTT pass
is one launch for all the columns instead of one per column.

The library has no transcript: the functions return the commitments, and the caller writes them in proof order, as the
reference does (`common_point` for instances, `write_point` for advice).
"""
from __future__ import annotations

from typing import List, NamedTuple, Sequence

import numpy as np

from . import lib as _l
from .poly import (Blind, EvaluationDomain, Params, ResidentPoly, _split, _tensor_rows, freed_on_failure, is_device_tensor, set_rows_resident,
                   upload_tensors_resident)


class InstanceTooLarge(_l.H2Error):
    """Error::InstanceTooLarge (plonk/prover.rs:84-86): an instance column longer than n - (blinding_factors + 1)."""


class InstanceSingle(NamedTuple):
    """plonk::prover's InstanceSingle (:79-124) on the device, for one proof."""
    commitments: np.ndarray                # (columns, 64) affine, commit_lagrange with Blind::default()
    values: List[ResidentPoly]             # Lagrange basis, zero-padded to n
    polys: List[ResidentPoly]              # coefficient form
    cosets: List[ResidentPoly]             # extended domain


class AdviceSingle(NamedTuple):
    """plonk::prover's AdviceSingle (:269-335) on the device, for one proof."""
    commitments: np.ndarray                # (columns, 64) affine
    blinds: List[int]
    values: List[ResidentPoly]             # Lagrange basis, blinding rows included
    polys: List[ResidentPoly]              # coefficient form
    cosets: List[ResidentPoly]             # extended domain


def _transforms(domain: EvaluationDomain, values: List[ResidentPoly], fresh):
    """lagrange_to_coeff then coeff_to_extended of every column, one call each, into new polynomials from `fresh`."""
    polys = [fresh.keep(ResidentPoly(domain.field, domain.n)) for _ in values]
    domain.lagrange_to_coeff_batch_resident(values, out=polys)
    cosets = [fresh.keep(ResidentPoly(domain.field, domain.extended_len())) for _ in values]
    domain.coeff_to_extended_batch_resident(polys, out=cosets)
    return polys, cosets


def instance_commit(params: Params, domain: EvaluationDomain, instances: Sequence[Sequence], blinding_factors: int) -> List[InstanceSingle]:
    """The instance columns of every proof (plonk/prover.rs:79-124): `instances[p]` is proof p's list of columns (ints,
    (len, 32) uint8 arrays, or CUDA tensors as ResidentPoly.from_tensor takes them).  Each column is zero-padded to n and
    committed with Blind::default(); raises InstanceTooLarge when a column is longer than n - (blinding_factors + 1).  The
    tensor columns go up in one h2_poly_upload_dev on torch's current stream.  Returns one InstanceSingle per proof."""
    n, m = domain.n, domain.m
    cols = [col if is_device_tensor(col) else _l.fe_array(col, m) for per in instances for col in per]
    rows = [_tensor_rows(c, "an instance column") if is_device_tensor(c) else c.shape[0] for c in cols]
    if any(r > n - (blinding_factors + 1) for r in rows):
        raise InstanceTooLarge("instance column longer than n - (blinding_factors + 1) (Error::InstanceTooLarge)")
    with freed_on_failure() as fresh:
        values = [fresh.keep(ResidentPoly(domain.field, n, c if r and not is_device_tensor(c) else None))   # allocated zero-filled: the padding
                  for c, r in zip(cols, rows)]
        dev = [(p, c) for p, c, r in zip(values, cols, rows) if r and is_device_tensor(c)]
        upload_tensors_resident([p for p, _ in dev], [c for _, c in dev])
        cm = params.commit_resident_affine(values, [Blind() for _ in values], lagrange=True)
        polys, cosets = _transforms(domain, values, fresh) if values else ([], [])
    sizes = [len(per) for per in instances]
    return [InstanceSingle(c, v, p, e) for c, v, p, e in zip(_split(cm, sizes), _split(values, sizes), _split(polys, sizes), _split(cosets, sizes))]


def advice_commit(params: Params, domain: EvaluationDomain, advice: Sequence[Sequence], rng, blinding_factors: int) -> List[AdviceSingle]:
    """The advice columns of every proof (plonk/prover.rs:269-335): `advice[p]` is proof p's list of n-row Lagrange columns,
    host arrays (ints or (n, 32) uint8), CUDA tensors (as ResidentPoly.from_tensor takes them; all of them go up in one
    h2_poly_upload_dev on torch's current stream) or ResidentPolys, which receive their blinding rows in place.  `rng`
    (scalar() -> int) is drawn in the reference's order: per proof, per column, the blinding_factors + 1 unusable rows in row
    order, then one blind per column (:276-282, :294-304).  One h2_poly_set_rows writes every column's blinding rows, one
    commitment pass commits them, and the transforms run one batched call each.  Returns one AdviceSingle per proof."""
    n, m = domain.n, domain.m
    rows = blinding_factors + 1
    usable = n - rows
    blinding, blinds = [], []
    for per in advice:
        for _ in per:
            blinding.append([rng.scalar() for _ in range(rows)])
        blinds.append([rng.scalar() for _ in per])
    with freed_on_failure() as fresh:
        values, dev = [], []
        for per in advice:
            for col in per:
                if isinstance(col, ResidentPoly):
                    if col.len < n:
                        raise _l.H2Error("an advice column holds fewer than n rows")
                    values.append(col)
                    continue
                if is_device_tensor(col):
                    if _tensor_rows(col, "an advice column") != n:
                        raise _l.H2Error("an advice column does not have n rows")
                    values.append(fresh.keep(ResidentPoly(domain.field, n)))
                    dev.append((values[-1], col))
                    continue
                arr = _l.fe_array(col, m)
                if arr.shape[0] != n:
                    raise _l.H2Error("an advice column does not have n rows")
                values.append(fresh.keep(ResidentPoly(domain.field, n, arr)))
        upload_tensors_resident([p for p, _ in dev], [c for _, c in dev])   # before the blinding rows overwrite their tail
        set_rows_resident(values, usable, blinding)
        cm = params.commit_resident_affine(values, [Blind(b) for per in blinds for b in per], lagrange=True)
        polys, cosets = _transforms(domain, values, fresh) if values else ([], [])
    sizes = [len(per) for per in advice]
    return [AdviceSingle(c, b, v, p, e)
            for c, b, v, p, e in zip(_split(cm, sizes), blinds, _split(values, sizes), _split(polys, sizes), _split(cosets, sizes))]
