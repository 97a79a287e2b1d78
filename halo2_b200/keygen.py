"""Host-side mirror of key generation over the C ABI: plonk::keygen_vk / keygen_pk
(/root/reference/halo2_proofs/src/plonk/keygen.rs:188-336), the permutation argument's Assembly and build_vk / build_pk
(plonk/permutation/keygen.rs:16-211) and batch_invert_assigned (poly.rs:135-180).

The copy-constraint bookkeeping is either the reference's sequential algorithm on the host (`Assembly.copy`, whose mapping
h2_poly_permutation_sigma turns into sigma) or, with `CopyConstraints`, the list of copies itself, which
h2_poly_permutation_sigma_copies turns into the same sigma on the device (csrc/assembly.cuh, then csrc/keygen.cuh).
Everything of size n per column runs on the device and stays there: the transforms and commitments are the engine's
resident ones.  Circuit synthesis and selector
compression are the caller's: keygen_vk / keygen_pk take the final fixed columns.
"""
from __future__ import annotations

import ctypes
from typing import List, Sequence, Union

import numpy as np

from . import lib as _l
from .evaluator import AstLeaf, compile_ast
from .poly import (FIELDS, Blind, EvaluationDomain, Params, ResidentPoly, _handles, _tensor_rows, batch_invert_resident, freed_on_failure, is_device_tensor,
                   share_resident)


class Assembly:
    """plonk/permutation/keygen.rs:16-100 for `num_columns` permutation columns of `n` rows.  A cell (column, row) is kept as
    the integer column * n + row, so `mapping`, `aux` and `sizes` are flat numpy arrays; `mapping` (the property) gives the
    reference's Vec<Vec<(usize, usize)>> as a (num_columns, n, 2) uint32 array of (column, row) pairs."""

    def __init__(self, n: int, num_columns: int):
        self.n, self.num_columns = int(n), int(num_columns)
        assert self.n > 0 and self.n & (self.n - 1) == 0, "n = params.n is a power of two"
        self._log_n = self.n.bit_length() - 1
        cells = np.arange(self.n * self.num_columns, dtype=np.int64)
        # every cell starts in a 1-cycle: mapping and aux are identical (:25-43)
        self._mapping = cells.copy()
        self._aux = cells
        self._sizes = np.ones(self.n * self.num_columns, dtype=np.int64)

    def copy(self, left_column: int, left_row: int, right_column: int, right_row: int) -> None:
        """Assembly::copy (:45-100).  Columns are indices into the permutation's column list; a column outside it raises
        ValueError (Error::ColumnNotInPermutation), a row outside [0, n) IndexError (Error::BoundsFailure)."""
        n = self.n
        for c in (left_column, right_column):
            if not 0 <= c < self.num_columns:
                raise ValueError(f"column {c} is not in the permutation ({self.num_columns} columns)")
        if not (0 <= left_row < n and 0 <= right_row < n):
            raise IndexError(f"row out of bounds: {left_row}, {right_row} (n = {n})")
        mapping, aux, sizes = self._mapping, self._aux, self._sizes
        left, right = left_column * n + left_row, right_column * n + right_row
        left_cycle, right_cycle = int(aux[left]), int(aux[right])
        if left_cycle == right_cycle:                          # same cycle: nothing to do
            return
        if sizes[left_cycle] < sizes[right_cycle]:
            left_cycle, right_cycle = right_cycle, left_cycle
        sizes[left_cycle] += sizes[right_cycle]                # merge the right cycle into the left one
        i = right_cycle
        while True:
            aux[i] = left_cycle
            i = int(mapping[i])
            if i == right_cycle:
                break
        mapping[left], mapping[right] = mapping[right], mapping[left]

    @property
    def mapping(self) -> np.ndarray:
        out = np.empty((self.num_columns, self.n, 2), dtype=np.uint32)
        out[..., 0] = (self._mapping >> self._log_n).reshape(self.num_columns, self.n)
        out[..., 1] = (self._mapping & (self.n - 1)).reshape(self.num_columns, self.n)
        return out


class CopyConstraints:
    """The permutation argument's copy constraints as a list, in the order synthesis makes them: what `Assembly` consumes,
    without replaying its cycle bookkeeping on the host.  build_permutation_polys / keygen_vk / keygen_pk take it in place
    of an Assembly and get the same key: the cycles are computed on the device from the list (csrc/assembly.cuh).
    `copies` gives the list as an (m, 4) uint32 array of (left column, left row, right column, right row)."""

    def __init__(self, n: int, num_columns: int):
        self.n, self.num_columns = int(n), int(num_columns)
        assert self.n > 0 and self.n & (self.n - 1) == 0, "n = params.n is a power of two"
        self._arrays: List[np.ndarray] = []
        self._pending: List[tuple] = []

    def copy(self, left_column: int, left_row: int, right_column: int, right_row: int) -> None:
        """Assembly.copy's checks, then the copy is recorded: a column outside the permutation raises ValueError
        (Error::ColumnNotInPermutation), a row outside [0, n) IndexError (Error::BoundsFailure)."""
        for c in (left_column, right_column):
            if not 0 <= c < self.num_columns:
                raise ValueError(f"column {c} is not in the permutation ({self.num_columns} columns)")
        if not (0 <= left_row < self.n and 0 <= right_row < self.n):
            raise IndexError(f"row out of bounds: {left_row}, {right_row} (n = {self.n})")
        self._pending.append((int(left_column), int(left_row), int(right_column), int(right_row)))

    def extend(self, copies) -> None:
        """Records an (m, 4) integer array of copies, checked as a whole: when a row of it fails copy()'s checks, the first
        such row raises copy()'s exception (naming its index) and nothing of the array is recorded."""
        a = np.asarray(copies)
        if a.size == 0:
            return
        if a.ndim != 2 or a.shape[1] != 4 or a.dtype.kind not in "iu":
            raise TypeError("copies must be an (m, 4) integer array of (left column, left row, right column, right row)")
        bad_col = ((a[:, [0, 2]] < 0) | (a[:, [0, 2]] >= self.num_columns)).any(axis=1)
        bad_row = ((a[:, [1, 3]] < 0) | (a[:, [1, 3]] >= self.n)).any(axis=1)
        bad = np.flatnonzero(bad_col | bad_row)
        if bad.size:
            i = int(bad[0])
            if bad_col[i]:
                raise ValueError(f"copy {i}: a column of {a[i].tolist()} is not in the permutation ({self.num_columns} columns)")
            raise IndexError(f"copy {i}: a row of {a[i].tolist()} is out of bounds (n = {self.n})")
        self._flush()
        self._arrays.append(a.astype(np.uint32))

    def _flush(self) -> None:
        if self._pending:
            self._arrays.append(np.array(self._pending, dtype=np.uint32).reshape(-1, 4))
            self._pending = []

    def __len__(self) -> int:
        return sum(a.shape[0] for a in self._arrays) + len(self._pending)

    @property
    def copies(self) -> np.ndarray:
        self._flush()
        if len(self._arrays) != 1:
            self._arrays = [np.concatenate(self._arrays) if self._arrays else np.zeros((0, 4), dtype=np.uint32)]
        return self._arrays[0]


def build_permutation_polys(domain: EvaluationDomain, assembly: Union[Assembly, CopyConstraints], delta: int) -> List[ResidentPoly]:
    """The permutation polynomials of build_vk / build_pk (permutation/keygen.rs:108-143, :161-198) in the Lagrange basis,
    resident: sigma_i[j] = delta^c * omega^r for (c, r) = mapping[i][j].  `delta` is F::DELTA.  From an Assembly the
    mapping goes up; from CopyConstraints the copy list goes up and the mapping is computed on the device."""
    if assembly.n != domain.n:
        raise _l.H2Error(f"the assembly has {assembly.n} rows, the domain {domain.n}")
    cols = assembly.num_columns
    if not cols:
        return []
    omega, dl = _l.ptr(_l.fe_bytes(domain.omega)), _l.ptr(_l.fe_bytes(int(delta) % domain.m))
    with freed_on_failure() as fresh:
        polys = [fresh.keep(ResidentPoly(domain.field, domain.n)) for _ in range(cols)]
        if isinstance(assembly, CopyConstraints):
            copies = np.ascontiguousarray(assembly.copies, dtype=np.uint32)
            _l.check(_l.init().h2_poly_permutation_sigma_copies(_handles(polys), ctypes.c_size_t(cols), ctypes.c_uint32(domain.k),
                                                                copies.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(copies.shape[0]),
                                                                omega, dl, _l.REPR_CANONICAL))
        else:
            mapping = np.ascontiguousarray(assembly.mapping)
            _l.check(_l.init().h2_poly_permutation_sigma(_handles(polys), ctypes.c_size_t(cols), ctypes.c_uint32(domain.k),
                                                         mapping.ctypes.data_as(ctypes.c_void_p), omega, dl, _l.REPR_CANONICAL))
    return polys


def batch_invert_assigned_resident(numerators: Sequence[ResidentPoly], denominators: Sequence[ResidentPoly]) -> List[ResidentPoly]:
    """batch_invert_assigned (poly.rs:135-180) on resident columns of Assigned values split into numerators and
    denominators (a trivial denominator is 1): out[i][j] = numerators[i][j] / denominators[i][j], and 0 where the denominator
    is 0, as ff::BatchInvert leaves zeros alone.  Returns new polynomials; the inputs are not changed."""
    assert len(numerators) == len(denominators)
    lib = _l.init()
    with freed_on_failure() as out:
        for num, den in zip(numerators, denominators):
            n = num.len
            assert n & (n - 1) == 0 and den.len >= n and den.field == num.field, "columns of 2^k elements in one field"
            code, consts = compile_ast(AstLeaf(0) * AstLeaf(1), FIELDS[num.field], 1)
            inv = ResidentPoly(num.field, n)
            res = out.keep(ResidentPoly(num.field, n))
            try:
                inv.copy_from(den, n)
                batch_invert_resident(inv, n)
                one = _l.ptr(_l.fe_bytes(1))
                _l.check(lib.h2_poly_eval_ast(res._h, _handles([num, inv]), ctypes.c_size_t(2), ctypes.c_uint32(n.bit_length() - 1),
                                              code.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(code.shape[0]), None, ctypes.c_size_t(len(consts)),
                                              one, one, _l.REPR_CANONICAL))
            finally:
                inv.close()
    return list(out)


def _lagrange_column(domain: EvaluationDomain, values) -> ResidentPoly:
    """n values (ints, an (n, 32) uint8 array, or a CUDA tensor as ResidentPoly.from_tensor takes it) as a resident column."""
    if is_device_tensor(values):
        assert _tensor_rows(values, "a fixed column") == domain.n, "a fixed column must have n values"
        return ResidentPoly.from_tensor(domain.field, values)
    vals = _l.fe_array(values, domain.m)
    assert vals.shape[0] == domain.n, "a fixed column must have n values"
    return ResidentPoly(domain.field, domain.n, vals)


def _fixed_values(domain: EvaluationDomain, fixed) -> List[ResidentPoly]:
    """The fixed columns as resident Lagrange values.  A column is its values (ints, an (n, 32) uint8 array or a CUDA
    tensor) or a (numerators, denominators) pair of such, which goes through batch_invert_assigned_resident."""
    with freed_on_failure() as out:
        for col in fixed:
            if isinstance(col, tuple):
                num, den = (ResidentPoly.from_tensor(domain.field, v, length=domain.n) if is_device_tensor(v) else
                            ResidentPoly(domain.field, domain.n, _l.fe_array(v, domain.m)) for v in col)
                try:
                    out.extend(batch_invert_assigned_resident([num], [den]))
                finally:
                    num.close()
                    den.close()
            else:
                out.append(_lagrange_column(domain, col))
    return list(out)


def keygen_vk(params: Params, domain: EvaluationDomain, fixed, assembly: Union[Assembly, CopyConstraints], delta: int):
    """keygen_vk's commitments (keygen.rs:188-236, permutation/keygen.rs:102-153): commit_lagrange of every fixed column and
    every permutation polynomial with Blind::default(), in one pass over the resident generators.  Returns
    (fixed_commitments, permutation_commitments) as affine (m, 64) uint8 arrays in the reference's order."""
    assert params.n == domain.n
    polys = _fixed_values(domain, fixed)
    nf = len(polys)
    try:
        polys += build_permutation_polys(domain, assembly, delta)
        cm = params.commit_resident_affine(polys, [Blind() for _ in polys], lagrange=True)
        return cm[:nf], cm[nf:]
    finally:
        for p in polys:
            p.close()


class PermutationProvingKey:
    """permutation::ProvingKey (permutation.rs): the sigma polynomials' Lagrange values, coefficients and extended cosets."""

    def __init__(self, permutations: List[ResidentPoly], polys: List[ResidentPoly], cosets: List[ResidentPoly]):
        self.permutations, self.polys, self.cosets = permutations, polys, cosets


class ProvingKey:
    """plonk::ProvingKey (plonk.rs) without the verifying key: every polynomial resident.  `fixed_values` / `fixed_polys` /
    `fixed_cosets`, `permutation.{permutations, polys, cosets}`, and the extended cosets `l0`, `l_blind`, `l_last`.  The key
    belongs to the lane (or the primary context) that built it until share() makes it readable from every lane; close()
    frees it."""

    def __init__(self, fixed_values, fixed_polys, fixed_cosets, permutation: PermutationProvingKey, l0, l_blind, l_last):
        self.fixed_values, self.fixed_polys, self.fixed_cosets = fixed_values, fixed_polys, fixed_cosets
        self.permutation = permutation
        self.l0, self.l_blind, self.l_last = l0, l_blind, l_last

    def _all(self) -> List[ResidentPoly]:
        P = self.permutation
        return (list(self.fixed_values) + list(self.fixed_polys) + list(self.fixed_cosets) + list(P.permutations) + list(P.polys)
                + list(P.cosets) + [p for p in (self.l0, self.l_blind, self.l_last) if p is not None])

    def share(self) -> "ProvingKey":
        """Shares every polynomial of the key in one h2_poly_share call: one resident copy that provers on every lane read.
        Call it on the lane that built the key; the key is read-only afterwards.  Returns the key."""
        share_resident(self._all())
        return self

    def close(self) -> None:
        for p in self._all():
            p.close()


def keygen_pk(params: Params, domain: EvaluationDomain, fixed, assembly: Union[Assembly, CopyConstraints], delta: int,
              blinding_factors: int) -> ProvingKey:
    """keygen_pk (keygen.rs:240-336, permutation/keygen.rs:155-211) on the device: the fixed and permutation columns in all
    three forms, and l_0 / l_blind / l_last (1 on row 0 / on the last `blinding_factors` rows / on row n - blinding_factors - 1,
    :306-325) as extended cosets.  The indicator columns start from a zero allocation and get their ones by add_at."""
    assert params.n == domain.n
    n = domain.n
    assert 0 <= blinding_factors < n - 1
    with freed_on_failure() as fresh:
        def coeff(lag):
            return domain.lagrange_to_coeff_resident(lag, out=fresh.keep(ResidentPoly(domain.field, n)))

        def ext(co):
            return fresh.keep(domain.coeff_to_extended_resident(co))

        fixed_values = [fresh.keep(p) for p in _fixed_values(domain, fixed)]
        fixed_polys = [coeff(v) for v in fixed_values]
        fixed_cosets = [ext(p) for p in fixed_polys]
        perms = [fresh.keep(p) for p in build_permutation_polys(domain, assembly, delta)]
        perm_polys = [coeff(v) for v in perms]
        perm = PermutationProvingKey(perms, perm_polys, [ext(p) for p in perm_polys])
        ls = []
        for rows in ([0], range(n - blinding_factors, n), [n - blinding_factors - 1]):
            lag = ResidentPoly(domain.field, n)                    # zero-filled by the allocation
            try:
                for r in rows:
                    lag.add_at(r, 1)
                domain.lagrange_to_coeff_resident(lag)              # in place
                ls.append(ext(lag))
            finally:
                lag.close()
    return ProvingKey(fixed_values, fixed_polys, fixed_cosets, perm, *ls)
