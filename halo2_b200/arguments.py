"""The second half of the permutation and lookup arguments over the C ABI: permutation::prover::Committed::construct,
Constructed::evaluate, Evaluated::open and the proving key's evaluate / open (halo2_proofs/src/plonk/permutation/prover.rs:197-420),
lookup::prover::Committed::construct, Constructed::evaluate and Evaluated::open (plonk/lookup/prover.rs:401-540), and the
column evaluations and queries of plonk::create_proof (plonk/prover.rs:598-656, :677-722).

With these and the earlier phases (columns, products, vanishing) a whole proof composes from library calls; the caller
supplies the gates' h(X) expressions and the circuit's query lists.  No new kernel is involved: the constraints are Ast
programs for the extended-domain Evaluator (csrc/asteval.cuh), the lookup products reach the coset in one batched transform,
and each evaluate is one h2_poly_eval call.

A lookup's input and table expressions are compressed on the extended coset, as an Ast over the caller's coset leaves
(lookup/prover.rs:172-176), not by extending the compressed Lagrange column: the two agree only when every expression is
linear in the columns, and the verifier recomputes the expression from the column evaluations at x.

The library has no transcript: every evaluate returns the scalars the caller writes, in the order the reference writes them,
and every open returns the queries in the reference's order.  Each object keeps what it was built from and close() frees all
of its resident polynomials; a call that fails frees what it allocated.
"""
from __future__ import annotations

from typing import List, NamedTuple, Sequence, Tuple

from . import lib as _l
from .evaluator import Ast, AstLeaf
from .multiopen import ProverQuery
from .poly import Blind, EvaluationDomain, ResidentPoly, _split, eval_polynomial_resident, freed_on_failure
from .products import Permuted


def _check(label: str, polys: Sequence[ResidentPoly], field: str, length: int) -> None:
    """Raises H2Error, naming the argument and index, for a closed polynomial, one of another field or one shorter than `length`."""
    for i, p in enumerate(polys):
        if not isinstance(p, ResidentPoly) or not p._h.value:
            raise _l.H2Error(f"{label}[{i}]: not an open resident polynomial")
        if p.field != field:
            raise _l.H2Error(f"{label}[{i}]: the polynomial lives in another field than the domain")
        if p.len < length:
            raise _l.H2Error(f"{label}[{i}]: a polynomial holds fewer than {length} elements")


def _leaf(evaluator, poly: ResidentPoly) -> AstLeaf:
    """The evaluator's leaf of `poly`, registered once however many proofs use it."""
    for i, p in enumerate(evaluator.polys):
        if p is poly:
            return AstLeaf(i)
    return evaluator.register_poly(poly)


def _evaluate(pairs, n: int) -> List[int]:
    """eval_polynomial of every (poly, point) pair in one h2_poly_eval call."""
    if not pairs:
        return []
    return eval_polynomial_resident([p for p, _ in pairs], [x for _, x in pairs], n=n)


# ---- the permutation argument ------------------------------------------------------------------------------------------
class PermutationCommitted(NamedTuple):
    """permutation::prover::Committed (permutation/prover.rs:27-35) of one proof: per set (permutation_product_poly in
    coefficient form, permutation_product_coset on the extended domain, permutation_product_blind), which is one proof's entry
    of what permutation_commit returns."""
    sets: List[Tuple[ResidentPoly, ResidentPoly, int]]

    def construct(self, evaluator, pk, columns: Sequence[Ast], l0: AstLeaf, l_blind: AstLeaf, l_last: AstLeaf, beta: int, gamma: int,
                  delta: int, chunk_len: int, blinding_factors: int) -> Tuple["PermutationConstructed", List[Ast]]:
        """Committed::construct (:197-312).  `evaluator` is the caller's extended-domain Evaluator, `pk` a ProvingKey (its
        permutation.cosets are the sigma cosets), `columns` the cosets' leaves of the argument's columns in its order, `delta`
        = F::DELTA and chunk_len = cs_degree - 2.  Registers every set's coset and the sigma cosets with `evaluator` and
        returns (PermutationConstructed, the expressions in the reference's order): (1 - z_0) l_0, (z_l^2 - z_l) l_last, the
        chaining terms, then one (left - right) (1 - (l_last + l_blind)) per set."""
        d = evaluator.domain
        sigma_cosets = list(pk.permutation.cosets)
        if chunk_len < 1:
            raise _l.H2Error("chunk_len must be at least 1")
        if len(columns) != len(sigma_cosets):
            raise _l.H2Error(f"expected one column leaf per permutation polynomial ({len(sigma_cosets)}), got {len(columns)}")
        sets = -(-len(sigma_cosets) // chunk_len)
        if len(self.sets) != sets:
            raise _l.H2Error(f"{len(sigma_cosets)} permutation polynomials in chunks of {chunk_len} make {sets} sets, got {len(self.sets)}")
        _check("permutation_product_poly", [s[0] for s in self.sets], d.field, d.n)
        _check("permutation_product_coset", [s[1] for s in self.sets], d.field, d.extended_len())
        _check("pk.permutation.cosets", sigma_cosets, d.field, d.extended_len())
        m = d.m
        one, beta_c, gamma_c = Ast.constant_term(1), Ast.constant_term(beta), Ast.constant_term(gamma)
        last_rotation = -(blinding_factors + 1)
        z = [_leaf(evaluator, s[1]) for s in self.sets]
        sigmas = [_leaf(evaluator, p) for p in sigma_cosets]
        exprs: List[Ast] = []
        if z:
            exprs.append((one - z[0]) * l0)                                              # :233-239
            exprs.append((z[-1] * z[-1] - z[-1]) * l_last)                               # :241-248
            for a in range(1, len(z)):                                                   # :250-266
                exprs.append((z[a] - z[a - 1].with_rotation(last_rotation)) * l0)
        active = one - (l_last + l_blind)
        for a, zl in enumerate(z):                                                       # :267-309
            cols = columns[a * chunk_len:(a + 1) * chunk_len]
            left = zl.with_rotation(1)
            for col, sigma in zip(cols, sigmas[a * chunk_len:(a + 1) * chunk_len]):
                left = left * (col + beta_c * sigma + gamma_c)
            right = zl
            current_delta = beta * pow(delta, a * chunk_len, m) % m
            for col in cols:
                right = right * (col + Ast.linear_term(current_delta) + gamma_c)
                current_delta = current_delta * delta % m
            exprs.append((left - right) * active)
        return PermutationConstructed(self, blinding_factors), exprs

    def close(self) -> None:
        for s in self.sets:
            s[0].close()
            s[1].close()


class PermutationConstructed(NamedTuple):
    """permutation::prover::Constructed (:37-44): the committed sets and the blinding factors that place the last rotation."""
    committed: PermutationCommitted
    blinding_factors: int

    def evaluate(self, domain: EvaluationDomain, x: int) -> Tuple["PermutationEvaluated", List[int]]:
        """Constructed::evaluate (:341-386): per set z(x) and z(x omega), and z(x omega^last) for every set but the last, in one
        h2_poly_eval call.  Returns (PermutationEvaluated, the scalars in the order the caller writes them)."""
        sets = self.committed.sets
        _check("permutation_product_poly", [s[0] for s in sets], domain.field, domain.n)
        x_next, x_last = domain.rotate_omega(x, 1), domain.rotate_omega(x, -(self.blinding_factors + 1))
        pairs = []
        for a, (poly, _, _) in enumerate(sets):
            pairs += [(poly, x), (poly, x_next)]
            if a + 1 < len(sets):
                pairs.append((poly, x_last))
        return PermutationEvaluated(self, domain), _evaluate(pairs, domain.n)

    def close(self) -> None:
        self.committed.close()


class PermutationEvaluated(NamedTuple):
    """permutation::prover::Evaluated (:46-48)."""
    constructed: PermutationConstructed
    domain: EvaluationDomain

    def open(self, x: int) -> List[ProverQuery]:
        """Evaluated::open (:388-420): every set at x and x omega, then every set but the last at x omega^last, from the
        second-to-last set down to the first."""
        sets = self.constructed.committed.sets
        x_next = self.domain.rotate_omega(x, 1)
        x_last = self.domain.rotate_omega(x, -(self.constructed.blinding_factors + 1))
        out = []
        for poly, _, blind in sets:
            out += [ProverQuery(x, poly, Blind(blind)), ProverQuery(x_next, poly, Blind(blind))]
        for poly, _, blind in list(reversed(sets))[1:]:
            out.append(ProverQuery(x_last, poly, Blind(blind)))
        return out

    def close(self) -> None:
        self.constructed.close()


def permutation_key_evaluate(pk, domain: EvaluationDomain, x: int) -> List[int]:
    """permutation::ProvingKey::evaluate (:329-339): every sigma polynomial at x, in one h2_poly_eval call."""
    polys = list(pk.permutation.polys)
    _check("pk.permutation.polys", polys, domain.field, domain.n)
    return _evaluate([(p, x) for p in polys], domain.n)


def permutation_key_open(pk, x: int) -> List[ProverQuery]:
    """permutation::ProvingKey::open (:315-327): every sigma polynomial at x with Blind::default()."""
    return [ProverQuery(x, p, Blind()) for p in pk.permutation.polys]


# ---- the lookup argument -----------------------------------------------------------------------------------------------
def _compress(expressions: Sequence[Ast], theta: int) -> Ast:
    """The coset compression of lookup/prover.rs:172-176: acc * ConstantTerm(theta) + e from ConstantTerm(0)."""
    acc = Ast.constant_term(0)
    for e in expressions:
        acc = acc * Ast.constant_term(theta) + e
    return acc


class LookupCommitted(NamedTuple):
    """lookup::prover::Committed (lookup/prover.rs:64-69) of every lookup of one proof: `permuted` is the proof's entry of
    lookup_commit_permuted, `products` its entry of lookup_commit_product ((product_poly in coefficient form,
    product_blind) per lookup)."""
    permuted: List[Permuted]
    products: List[Tuple[ResidentPoly, int]]

    def construct(self, evaluator, lookups: Sequence[Tuple[Sequence[Ast], Sequence[Ast]]], theta: int, beta: int, gamma: int,
                  l0: AstLeaf, l_blind: AstLeaf, l_last: AstLeaf) -> Tuple["LookupConstructed", List[Ast]]:
        """Committed::construct (:401-478) of every lookup.  `lookups[i]` are lookup i's (input expressions, table expressions)
        as Ast over `evaluator`'s leaves (the extended domain's).  Each list is compressed on the coset; no transform is made
        for the compressed columns.  Every product z reaches the coset in one h2_poly_coeff_to_extended_batch call, and the
        product and permuted cosets are registered with `evaluator`.  Returns (LookupConstructed, five expressions per
        lookup in the reference's order)."""
        d = evaluator.domain
        if len(self.permuted) != len(self.products):
            raise _l.H2Error(f"{len(self.permuted)} permuted lookups but {len(self.products)} product columns")
        if len(lookups) != len(self.permuted):
            raise _l.H2Error(f"{len(self.permuted)} committed lookups but {len(lookups)} lookup expressions")
        for i, (inp, tab) in enumerate(lookups):
            if len(inp) != len(tab) or not inp:
                raise _l.H2Error(f"lookups[{i}]: {len(inp)} input expressions and {len(tab)} table expressions")
        n, big = d.n, d.extended_len()
        _check("products", [z for z, _ in self.products], d.field, n)
        _check("permuted_input_poly", [p.permuted_input_poly for p in self.permuted], d.field, n)
        _check("permuted_table_poly", [p.permuted_table_poly for p in self.permuted], d.field, n)
        _check("permuted_input_coset", [p.permuted_input_coset for p in self.permuted], d.field, big)
        _check("permuted_table_coset", [p.permuted_table_coset for p in self.permuted], d.field, big)
        cosets = d.coeff_to_extended_batch_resident([z for z, _ in self.products]) if self.products else []
        with freed_on_failure() as fresh:
            fresh.extend(cosets)
            one, beta_c, gamma_c = Ast.constant_term(1), Ast.constant_term(beta), Ast.constant_term(gamma)
            active = one - (l_last + l_blind)
            exprs: List[Ast] = []
            for (inp, tab), p, coset in zip(lookups, self.permuted, cosets):
                z, a, s = _leaf(evaluator, coset), _leaf(evaluator, p.permuted_input_coset), _leaf(evaluator, p.permuted_table_coset)
                left = z.with_rotation(1) * (a + beta_c) * (s + gamma_c)
                right = z * (_compress(inp, theta) + beta_c) * (_compress(tab, theta) + gamma_c)
                exprs += [(one - z) * l0,                                               # :418-419
                          (z * z - z) * l_last,                                         # :421-425
                          (left - right) * active,                                      # :426-447
                          (a - s) * l0,                                                 # :448-456
                          (a - s) * (a - a.with_rotation(-1)) * active]                 # :457-469
        return LookupConstructed(self, cosets), exprs

    def close(self) -> None:
        for q in [q for p in self.permuted for q in p[:8]] + [z for z, _ in self.products]:
            q.close()


class LookupConstructed(NamedTuple):
    """lookup::prover::Constructed (:71-78) of every lookup of one proof, with the product cosets construct made."""
    committed: LookupCommitted
    product_cosets: List[ResidentPoly]

    def evaluate(self, domain: EvaluationDomain, x: int) -> Tuple["LookupEvaluated", List[int]]:
        """Constructed::evaluate (:482-510): per lookup z(x), z(x omega), A'(x), A'(x omega^-1) and S'(x), in one h2_poly_eval
        call.  Returns (LookupEvaluated, the scalars in the order the caller writes them)."""
        c = self.committed
        _check("products", [z for z, _ in c.products], domain.field, domain.n)
        _check("permuted_input_poly", [p.permuted_input_poly for p in c.permuted], domain.field, domain.n)
        _check("permuted_table_poly", [p.permuted_table_poly for p in c.permuted], domain.field, domain.n)
        x_prev, x_next = domain.rotate_omega(x, -1), domain.rotate_omega(x, 1)
        pairs = []
        for p, (z, _) in zip(c.permuted, c.products):
            pairs += [(z, x), (z, x_next), (p.permuted_input_poly, x), (p.permuted_input_poly, x_prev), (p.permuted_table_poly, x)]
        return LookupEvaluated(self, domain), _evaluate(pairs, domain.n)

    def close(self) -> None:
        for p in self.product_cosets:
            p.close()
        self.committed.close()


class LookupEvaluated(NamedTuple):
    """lookup::prover::Evaluated (:80-82)."""
    constructed: LookupConstructed
    domain: EvaluationDomain

    def open(self, x: int) -> List[ProverQuery]:
        """Evaluated::open (:513-540), per lookup: z at x, A' at x, S' at x, A' at x omega^-1, z at x omega."""
        c = self.constructed.committed
        x_prev, x_next = self.domain.rotate_omega(x, -1), self.domain.rotate_omega(x, 1)
        out = []
        for p, (z, zb) in zip(c.permuted, c.products):
            bi, bt, bz = Blind(p.permuted_input_blind), Blind(p.permuted_table_blind), Blind(zb)
            out += [ProverQuery(x, z, bz), ProverQuery(x, p.permuted_input_poly, bi), ProverQuery(x, p.permuted_table_poly, bt),
                    ProverQuery(x_prev, p.permuted_input_poly, bi), ProverQuery(x_next, z, bz)]
        return out

    def close(self) -> None:
        self.constructed.close()


# ---- the columns' evaluations and queries ------------------------------------------------------------------------------
def _column_pairs(domain: EvaluationDomain, x: int, instance_polys, advice_polys, fixed_polys, instance_queries, advice_queries,
                  fixed_queries):
    """The (poly, point) pairs of every query in the reference's order -- per proof the instance queries, per proof the advice
    queries, then the fixed queries -- after checking every argument."""
    if len(instance_polys) != len(advice_polys):
        raise _l.H2Error(f"{len(instance_polys)} proofs' instance columns but {len(advice_polys)} proofs' advice columns")
    groups = [("instance", per, instance_queries) for per in instance_polys] + [("advice", per, advice_queries) for per in advice_polys]
    groups.append(("fixed", fixed_polys, fixed_queries))
    for kind, polys, queries in groups:
        _check(f"{kind} polys", polys, domain.field, domain.n)
        for i, (col, _) in enumerate(queries):
            if not 0 <= col < len(polys):
                raise _l.H2Error(f"{kind}_queries[{i}]: column {col} of {len(polys)}")
    return [[(polys[col], domain.rotate_omega(x, rot)) for col, rot in queries] for _, polys, queries in groups]


def evaluate_columns(domain: EvaluationDomain, x: int, instance_polys, advice_polys, fixed_polys, instance_queries, advice_queries,
                     fixed_queries) -> Tuple[List[List[int]], List[List[int]], List[int]]:
    """The instance, advice and fixed evaluations of plonk::create_proof (plonk/prover.rs:598-656) in one h2_poly_eval call.
    `instance_polys[p]` / `advice_polys[p]` are proof p's coefficient-form columns, `fixed_polys` the key's, and each query list
    holds the circuit's (column index, rotation) pairs.  Returns (instance evals per proof, advice evals per proof, fixed
    evals): the caller writes every proof's instance evals, then every proof's advice evals, then the fixed evals."""
    groups = _column_pairs(domain, x, instance_polys, advice_polys, fixed_polys, instance_queries, advice_queries, fixed_queries)
    out = _split(_evaluate([pair for g in groups for pair in g], domain.n), [len(g) for g in groups])
    proofs = len(instance_polys)
    return out[:proofs], out[proofs:2 * proofs], out[-1]


def open_columns(domain: EvaluationDomain, x: int, instance_polys, advice_polys, advice_blinds, fixed_polys, instance_queries,
                 advice_queries, fixed_queries) -> Tuple[List[List[ProverQuery]], List[List[ProverQuery]], List[ProverQuery]]:
    """The columns' queries of plonk::create_proof (plonk/prover.rs:677-722): per proof the instance queries (Blind::default())
    and the advice queries (`advice_blinds[p][column]`), and the fixed queries (Blind::default()).  The reference opens, per
    proof, its instance, advice, permutation and lookup queries, and after every proof the fixed queries, the key's
    permutation queries and the vanishing argument's."""
    if len(advice_blinds) != len(advice_polys) or any(len(b) != len(p) for b, p in zip(advice_blinds, advice_polys)):
        raise _l.H2Error("expected one advice blind per advice column of every proof")
    groups = _column_pairs(domain, x, instance_polys, advice_polys, fixed_polys, instance_queries, advice_queries, fixed_queries)
    proofs = len(instance_polys)
    inst = [[ProverQuery(pt, poly, Blind()) for poly, pt in g] for g in groups[:proofs]]
    adv = [[ProverQuery(pt, poly, Blind(advice_blinds[p][col])) for (poly, pt), (col, _) in zip(g, advice_queries)]
           for p, g in enumerate(groups[proofs:2 * proofs])]
    return inst, adv, [ProverQuery(pt, poly, Blind()) for poly, pt in groups[-1]]
