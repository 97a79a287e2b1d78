"""The prover's product columns over the C ABI: permutation::Argument::commit
(/root/reference/halo2_proofs/src/plonk/permutation/prover.rs:47-195) and lookup::Permuted::commit_product
(plonk/lookup/prover.rs:253-390), every column of every proof in one device call (csrc/grandproduct.cuh), and the lookup
argument's permuted columns before them, lookup::Argument::commit_permuted (:76-243), likewise in one call (csrc/lookup.cuh).

The library has no transcript: the commit functions return the commitments in the order the reference writes them, and the
caller writes them to its own transcript.
"""
from __future__ import annotations

import ctypes
from typing import List, NamedTuple, Sequence, Tuple

from . import lib as _l
from .evaluator import Ast
from .poly import Blind, EvaluationDomain, Params, ResidentPoly, _handles, _split, freed_on_failure


def permutation_product_resident(domain: EvaluationDomain, columns: Sequence[Sequence[ResidentPoly]], sigmas: Sequence[ResidentPoly], beta: int,
                                 gamma: int, delta: int, chunk_len: int, blinding_factors: int, blinding: Sequence[int]) -> List[List[ResidentPoly]]:
    """The permutation argument's product columns z (Lagrange basis, resident) of every proof: `columns[p]` are proof p's
    resident Lagrange columns in the argument's column order, `sigmas` the key's permutation polynomials, `delta` = F::DELTA.
    `blinding` holds the blinding rows, proofs x sets x blinding_factors values in the rng's order.  Returns, per proof, its
    sets' z columns (h2_poly_permutation_product)."""
    m, n, proofs, cols = domain.m, domain.n, len(columns), len(sigmas)
    if any(len(c) != cols for c in columns):
        raise _l.H2Error("every proof needs one column per permutation polynomial")
    if chunk_len < 1:
        raise _l.H2Error("chunk_len must be at least 1")
    sets = -(-cols // chunk_len)
    if len(blinding) != proofs * sets * blinding_factors:
        raise _l.H2Error(f"expected {proofs * sets * blinding_factors} blinding values, got {len(blinding)}")
    bl = _l.fe_array(blinding, m) if blinding else None                       # no blinding rows: a null pointer
    with freed_on_failure() as fresh:
        z = [fresh.keep(ResidentPoly(domain.field, n)) for _ in range(proofs * sets)]
        _l.check(_l.init().h2_poly_permutation_product(
            _handles(z), ctypes.c_size_t(proofs), _handles([c for per in columns for c in per]), _handles(sigmas), ctypes.c_size_t(cols),
            ctypes.c_uint32(chunk_len), ctypes.c_uint32(domain.k), _l.ptr(_l.fe_bytes(beta % m)), _l.ptr(_l.fe_bytes(gamma % m)),
            _l.ptr(_l.fe_bytes(domain.omega)), _l.ptr(_l.fe_bytes(delta % m)), _l.ptr(bl), ctypes.c_uint32(blinding_factors),
            _l.REPR_CANONICAL))
    return [z[p * sets:(p + 1) * sets] for p in range(proofs)]


def lookup_product_resident(domain: EvaluationDomain, lookups: Sequence[Sequence[Tuple[ResidentPoly, ResidentPoly, ResidentPoly, ResidentPoly]]],
                            beta: int, gamma: int, blinding_factors: int, blinding: Sequence[int]) -> List[List[ResidentPoly]]:
    """The lookup argument's product columns z (Lagrange basis, resident): `lookups[p]` is proof p's list of (compressed input,
    compressed table, permuted input, permuted table) columns; `blinding` holds blinding_factors values per lookup, in order.
    Returns, per proof, its lookups' z columns (h2_poly_lookup_product)."""
    m, n = domain.m, domain.n
    flat = [lk for per in lookups for lk in per]
    if len(blinding) != len(flat) * blinding_factors:
        raise _l.H2Error(f"expected {len(flat) * blinding_factors} blinding values, got {len(blinding)}")
    bl = _l.fe_array(blinding, m) if blinding else None
    with freed_on_failure() as fresh:
        z = [fresh.keep(ResidentPoly(domain.field, n)) for _ in flat]
        parts = [_handles([lk[j] for lk in flat]) for j in range(4)]
        _l.check(_l.init().h2_poly_lookup_product(_handles(z), ctypes.c_size_t(len(flat)), *parts, ctypes.c_uint32(domain.k),
                                                   _l.ptr(_l.fe_bytes(beta % m)), _l.ptr(_l.fe_bytes(gamma % m)), _l.ptr(bl),
                                                   ctypes.c_uint32(blinding_factors), _l.REPR_CANONICAL))
    return _split(z, [len(per) for per in lookups])


def permutation_commit(params: Params, domain: EvaluationDomain, pk, columns: Sequence[Sequence[ResidentPoly]], beta: int, gamma: int, delta: int,
                       chunk_len: int, blinding_factors: int, rng):
    """permutation::Argument::commit (permutation/prover.rs:47-195) for every proof at once.  `pk` is a ProvingKey (its
    permutation.permutations are the sigma columns), `columns[p]` proof p's columns in the argument's column order, `rng`
    an object with scalar() -> int, drawn in the reference's order: per proof, per set, blinding_factors values, then the
    set's blind (:155-171).  One product call, one commitment pass (commit_lagrange), then lagrange_to_coeff and
    coeff_to_extended per set.  Returns (sets, commitments): sets[p] = [(poly, coset, blind) per set], and the (proofs x sets,
    64) affine commitments in the order the reference writes them to the transcript."""
    sigmas = pk.permutation.permutations
    proofs, sets = len(columns), -(-len(sigmas) // max(int(chunk_len), 1))
    blinding, blinds = [], []
    for _ in range(proofs * sets):
        blinding += [rng.scalar() for _ in range(blinding_factors)]
        blinds.append(rng.scalar())
    z = [p for per in permutation_product_resident(domain, columns, sigmas, beta, gamma, delta, chunk_len, blinding_factors, blinding) for p in per]
    with freed_on_failure() as fresh:
        fresh.extend(z)
        cm = params.commit_resident_affine(z, [Blind(b) for b in blinds], lagrange=True)
        cosets = []
        for p in z:
            domain.lagrange_to_coeff_resident(p)                                  # in place: z becomes permutation_product_poly
            cosets.append(fresh.keep(domain.coeff_to_extended_resident(p)))
    return [list(zip(z, cosets, blinds))[p * sets:(p + 1) * sets] for p in range(proofs)], cm


def lookup_commit_product(params: Params, domain: EvaluationDomain, lookups, beta: int, gamma: int, blinding_factors: int, rng):
    """lookup::Permuted::commit_product (lookup/prover.rs:253-390) for every lookup of every proof at once.  `lookups[p]` is
    proof p's list of (compressed input, compressed table, permuted input, permuted table) Lagrange columns; `rng` is drawn
    per lookup: blinding_factors values, then product_blind (:317-321, :334).  Returns (products, commitments):
    products[p] = [(z poly in coefficient form, blind) per lookup], and the affine commitments in write order."""
    count = sum(len(per) for per in lookups)
    blinding, blinds = [], []
    for _ in range(count):
        blinding += [rng.scalar() for _ in range(blinding_factors)]
        blinds.append(rng.scalar())
    z = lookup_product_resident(domain, lookups, beta, gamma, blinding_factors, blinding)
    flat = [p for per in z for p in per]
    with freed_on_failure() as fresh:
        fresh.extend(flat)
        cm = params.commit_resident_affine(flat, [Blind(b) for b in blinds], lagrange=True)
        for p in flat:
            domain.lagrange_to_coeff_resident(p)
    return [list(zip(per, bl)) for per, bl in zip(z, _split(blinds, [len(per) for per in z]))], cm


def lookup_permute_resident(domain: EvaluationDomain, pairs: Sequence[Tuple[ResidentPoly, ResidentPoly]], blinding_factors: int,
                            blinding: Sequence[int]) -> List[Tuple[ResidentPoly, ResidentPoly]]:
    """The lookup argument's permuted columns (Lagrange basis, resident) of every (compressed input, compressed table) pair:
    permute_expression_pair (lookup/prover.rs:563-647) over the usable rows, then the blinding rows (:622-627).  `blinding`
    holds, per pair, blinding_factors + 1 input rows then as many table rows.  Returns one (permuted input, permuted table)
    per pair (h2_poly_lookup_permuted); fails, naming the lowest pair, when an input value is missing from its table."""
    m, n, rows = domain.m, domain.n, blinding_factors + 1
    if len(blinding) != len(pairs) * 2 * rows:
        raise _l.H2Error(f"expected {len(pairs) * 2 * rows} blinding values, got {len(blinding)}")
    bl = _l.fe_array(blinding, m) if blinding else None
    with freed_on_failure() as fresh:
        out = [fresh.keep(ResidentPoly(domain.field, n)) for _ in range(2 * len(pairs))]
        _l.check(_l.init().h2_poly_lookup_permuted(_handles(out[0::2]), _handles(out[1::2]), ctypes.c_size_t(len(pairs)),
                                                    _handles([p[0] for p in pairs]), _handles([p[1] for p in pairs]), ctypes.c_uint32(domain.k),
                                                    _l.ptr(bl), ctypes.c_uint32(blinding_factors), _l.REPR_CANONICAL))
    return list(zip(out[0::2], out[1::2]))


class Permuted(NamedTuple):
    """lookup::Permuted (lookup/prover.rs:51-62) on the device.  Its first four items are what lookup_commit_product takes."""
    compressed_input: ResidentPoly         # Lagrange basis
    compressed_table: ResidentPoly
    permuted_input: ResidentPoly           # Lagrange basis, blinding rows included
    permuted_table: ResidentPoly
    permuted_input_poly: ResidentPoly      # coefficient form
    permuted_table_poly: ResidentPoly
    permuted_input_coset: ResidentPoly     # extended domain
    permuted_table_coset: ResidentPoly
    permuted_input_blind: int
    permuted_table_blind: int


def lookup_commit_permuted(params: Params, domain: EvaluationDomain, evaluator, lookups, theta: int, blinding_factors: int, rng):
    """lookup::Argument::commit_permuted (lookup/prover.rs:76-243) for every lookup of every proof at once.  `evaluator` is a
    Lagrange-basis Evaluator and `lookups[p]` proof p's list of (input expressions, table expressions), each a list of Ast over
    it.  Each list is compressed by the fold acc * theta + e from ConstantTerm(0) (:167-176), one Ast program per column; then
    one permute call, one commitment pass of all columns, and lagrange_to_coeff / coeff_to_extended per column.  `rng` is drawn
    per proof, per lookup: blinding_factors + 1 input rows, as many table rows, the input blind, the table blind (:622-624,
    :203-216).  Returns (permuted, commitments): permuted[p] = [Permuted per lookup], which lookup_commit_product takes as it
    is, and the affine commitments in the order the reference writes them (per proof, per lookup, input then table)."""
    rows = blinding_factors + 1
    blinding, blinds = [], []
    for per in lookups:
        for _ in per:
            blinding += [rng.scalar() for _ in range(2 * rows)]
            blinds += [rng.scalar(), rng.scalar()]

    def compress(exprs):
        acc = Ast.constant_term(0)
        for e in exprs:
            acc = acc * theta + e
        return evaluator.evaluate(acc)

    with freed_on_failure() as fresh:
        compressed = [fresh.keep(compress(e)) for per in lookups for inp, tab in per for e in (inp, tab)]
        permuted = [fresh.keep(q) for pair in lookup_permute_resident(domain, list(zip(compressed[0::2], compressed[1::2])), blinding_factors, blinding)
                    for q in pair]
        cm = params.commit_resident_affine(permuted, [Blind(b) for b in blinds], lagrange=True)
        extra = []
        for q in permuted:
            co = domain.lagrange_to_coeff_resident(q, out=fresh.keep(ResidentPoly(domain.field, domain.n)))
            extra += [co, fresh.keep(domain.coeff_to_extended_resident(co))]
    flat = [Permuted(compressed[i], compressed[i + 1], permuted[i], permuted[i + 1], extra[2 * i], extra[2 * i + 2], extra[2 * i + 1],
                     extra[2 * i + 3], blinds[i], blinds[i + 1]) for i in range(0, len(permuted), 2)]
    return _split(flat, [len(per) for per in lookups]), cm
