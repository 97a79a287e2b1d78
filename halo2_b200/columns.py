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
from .poly import EvaluationDomain, Params, ResidentPoly, _tensor_rows, is_device_tensor, set_rows_resident, upload_tensors_resident
from .products import _commit


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


def _column_bytes(col, m: int) -> np.ndarray:
    if isinstance(col, np.ndarray):
        return _l.as_u8(col, 32)
    return np.frombuffer(b"".join((int(v) % m).to_bytes(32, "little") for v in col), dtype=np.uint8).reshape(-1, 32)


def _transforms(domain: EvaluationDomain, values: List[ResidentPoly], live: List[ResidentPoly]):
    """lagrange_to_coeff then coeff_to_extended of every column, one call each; new polynomials go to `live`."""
    polys = [ResidentPoly(domain.field, domain.n) for _ in values]
    live += polys
    domain.lagrange_to_coeff_batch_resident(values, out=polys)
    cosets = [ResidentPoly(domain.field, domain.extended_len()) for _ in values]
    live += cosets
    domain.coeff_to_extended_batch_resident(polys, out=cosets)
    return polys, cosets


def _split(flat: list, sizes: Sequence[int]) -> List[list]:
    out, at = [], 0
    for s in sizes:
        out.append(flat[at:at + s])
        at += s
    return out


def instance_commit(params: Params, domain: EvaluationDomain, instances: Sequence[Sequence], blinding_factors: int) -> List[InstanceSingle]:
    """The instance columns of every proof (plonk/prover.rs:79-124): `instances[p]` is proof p's list of columns (ints,
    (len, 32) uint8 arrays, or CUDA tensors as ResidentPoly.from_tensor takes them).  Each column is zero-padded to n and
    committed with Blind::default(); raises InstanceTooLarge when a column is longer than n - (blinding_factors + 1).  The
    tensor columns go up in one h2_poly_upload_dev on torch's current stream.  Returns one InstanceSingle per proof."""
    n, m = domain.n, domain.m
    cols = [col if is_device_tensor(col) else _column_bytes(col, m) for per in instances for col in per]
    rows = [_tensor_rows(c, "an instance column") if is_device_tensor(c) else c.shape[0] for c in cols]
    if any(r > n - (blinding_factors + 1) for r in rows):
        raise InstanceTooLarge("instance column longer than n - (blinding_factors + 1) (Error::InstanceTooLarge)")
    live: List[ResidentPoly] = []
    try:
        for c, r in zip(cols, rows):
            host = r and not is_device_tensor(c)
            live.append(ResidentPoly(domain.field, n, c if host else None))   # allocated zero-filled: the padding
        values = list(live)
        dev = [(p, c) for p, c, r in zip(values, cols, rows) if r and is_device_tensor(c)]
        upload_tensors_resident([p for p, _ in dev], [c for _, c in dev])
        cm = _commit(params, values, [1] * len(values))
        polys, cosets = _transforms(domain, values, live) if values else ([], [])
    except BaseException:
        for p in live:
            p.close()
        raise
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
    live: List[ResidentPoly] = []
    try:
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
                    live.append(ResidentPoly(domain.field, n))
                    values.append(live[-1])
                    dev.append((live[-1], col))
                    continue
                arr = _column_bytes(col, m)
                if arr.shape[0] != n:
                    raise _l.H2Error("an advice column does not have n rows")
                live.append(ResidentPoly(domain.field, n, arr))
                values.append(live[-1])
        upload_tensors_resident([p for p, _ in dev], [c for _, c in dev])   # before the blinding rows overwrite their tail
        flat_blinds = [b for per in blinds for b in per]
        set_rows_resident(values, usable, blinding)
        cm = _commit(params, values, flat_blinds)
        polys, cosets = _transforms(domain, values, live) if values else ([], [])
    except BaseException:
        for p in live:
            p.close()
        raise
    sizes = [len(per) for per in advice]
    return [AdviceSingle(c, b, v, p, e)
            for c, b, v, p, e in zip(_split(cm, sizes), blinds, _split(values, sizes), _split(polys, sizes), _split(cosets, sizes))]
