"""Host-side mirror of poly::Evaluator / poly::Ast (/root/reference/halo2_proofs/src/poly/evaluator.rs:85-437) over the C ABI:
the expression tree the prover builds for h(X) (plonk/prover.rs, plonk/vanishing) is flattened into a postfix program and run by
ONE kernel over device-resident polynomials (csrc/asteval.cuh) -- SURVEY.md section 8(f) row 3.

Same surface as the reference: `Evaluator.register_poly` returns a leaf, leaves take `.with_rotation(r)`, expressions combine
with + - * (Ast * Ast, Ast * scalar) and unary minus, `Ast.distribute_powers(terms, base)`, `Ast.linear_term(s)`,
`Ast.constant_term(s)`; `Evaluator.evaluate(ast)` returns the result polynomial (resident).
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence

import numpy as np

from . import lib as _l
from .poly import EvaluationDomain, ResidentPoly, freed_on_failure

OP_POLY, OP_CONST, OP_LINEAR, OP_ADD, OP_MUL, OP_SCALE, OP_NEG = range(7)


class Ast:
    """poly/evaluator.rs:237-331.  Nodes: ("poly", index, rotation) | ("add", a, b) | ("mul", a, b) | ("scale", a, s) |
    ("dp", terms, base) | ("lin", s) | ("const", s)."""

    def __init__(self, kind: str, *args):
        self.kind, self.args = kind, args

    # evaluator.rs:272-276
    @staticmethod
    def distribute_powers(terms: Sequence["Ast"], base: int) -> "Ast":
        return Ast("dp", list(terms), int(base))

    @staticmethod
    def linear_term(scalar: int) -> "Ast":
        return Ast("lin", int(scalar))

    @staticmethod
    def constant_term(scalar: int) -> "Ast":
        return Ast("const", int(scalar))

    def __add__(self, other: "Ast") -> "Ast":          # :294-300
        return Ast("add", self, other)

    def __neg__(self) -> "Ast":                        # :286-292: Scale(-1)
        return Ast("scale", self, -1)

    def __sub__(self, other: "Ast") -> "Ast":          # :310-316: self + (-other)
        return self + (-other)

    def __mul__(self, other) -> "Ast":                 # :326-331 (Ast * F), :384-397 (Ast * Ast: extended basis only)
        if isinstance(other, Ast):
            return Ast("mul", self, other)
        return Ast("scale", self, int(other))


class AstLeaf(Ast):
    """poly/evaluator.rs:37-79."""

    def __init__(self, index: int, rotation: int = 0):
        super().__init__("poly", index, rotation)
        self.index, self.rotation = index, rotation

    def with_rotation(self, rotation: int) -> "AstLeaf":
        return AstLeaf(self.index, int(rotation))


def compile_ast(ast: Ast, modulus: int, rotation_stride: int):
    """Flattens an Ast into (code (n, 4) uint32, constants list): the postfix program of csrc/asteval.cuh."""
    code: List[List[int]] = []
    consts: List[int] = []
    index = {}

    def const(v: int) -> int:
        v %= modulus
        if v not in index:
            index[v] = len(consts)
            consts.append(v)
        return index[v]

    def walk(node: Ast) -> None:
        k, a = node.kind, node.args
        if k == "poly":
            code.append([OP_POLY, a[0], (a[1] * rotation_stride) & 0xFFFFFFFF, 0])
        elif k == "add":
            walk(a[0]); walk(a[1]); code.append([OP_ADD, 0, 0, 0])
        elif k == "mul":
            walk(a[0]); walk(a[1]); code.append([OP_MUL, 0, 0, 0])
        elif k == "scale":
            walk(a[0]); code.append([OP_SCALE, const(a[1]), 0, 0])
        elif k == "dp":        # fold from the zero constant: acc = acc * base + term  (evaluator.rs:182-193)
            code.append([OP_CONST, const(0), 0, 0])
            for term in a[0]:
                code.append([OP_SCALE, const(a[1]), 0, 0])
                walk(term)
                code.append([OP_ADD, 0, 0, 0])
        elif k == "lin":
            code.append([OP_LINEAR, const(a[0]), 0, 0])
        elif k == "const":
            code.append([OP_CONST, const(a[0]), 0, 0])
        else:
            raise ValueError(f"unknown Ast node {k}")

    walk(ast)
    return np.ascontiguousarray(np.array(code, dtype=np.uint32).reshape(-1, 4)), consts


class Evaluator:
    """poly/evaluator.rs:85-228 for one basis of one EvaluationDomain: basis = "lagrange" (2^k values, rotation = 1 position)
    or "extended" (2^extended_k values, rotation = 2^(extended_k - k) positions, poly/domain.rs:286-295)."""

    def __init__(self, domain: EvaluationDomain, basis: str = "extended"):
        assert basis in ("lagrange", "extended")
        self.domain, self.basis = domain, basis
        self.log_n = domain.k if basis == "lagrange" else domain.extended_k
        self.stride = 1 if basis == "lagrange" else 1 << (domain.extended_k - domain.k)
        self.polys: List[ResidentPoly] = []
        self._owned: List[ResidentPoly] = []

    def register_poly(self, poly) -> AstLeaf:
        """evaluator.rs:105-113.  `poly`: a ResidentPoly (kept by reference) or host values (uploaded)."""
        if not isinstance(poly, ResidentPoly):
            arr = _l.as_u8(poly, 32)
            assert arr.shape[0] == 1 << self.log_n
            poly = ResidentPoly(self.domain.field, arr.shape[0], arr)
            self._owned.append(poly)
        assert poly.len >= 1 << self.log_n and poly.field == self.domain.field
        self.polys.append(poly)
        return AstLeaf(len(self.polys) - 1)

    def evaluate(self, ast: Ast, out: Optional[ResidentPoly] = None) -> ResidentPoly:
        """evaluator.rs:129-228."""
        d = self.domain
        code, consts = compile_ast(ast, d.m, self.stride)
        cs = _l.fe_array(consts, d.m)
        omega = d.omega if self.basis == "lagrange" else d.extended_omega
        lin = 1 if self.basis == "lagrange" else d.g_coset
        hs = (ctypes.c_uint64 * max(len(self.polys), 1))(*[p._h.value for p in self.polys])
        with freed_on_failure() as fresh:
            out = fresh.keep(ResidentPoly(d.field, 1 << self.log_n)) if out is None else out
            _l.check(_l.init().h2_poly_eval_ast(out._h, hs, ctypes.c_size_t(len(self.polys)), ctypes.c_uint32(self.log_n),
                                                code.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(code.shape[0]), _l.ptr(cs),
                                                ctypes.c_size_t(len(consts)), _l.ptr(_l.fe_bytes(omega)), _l.ptr(_l.fe_bytes(lin)), _l.REPR_CANONICAL))
        return out

    def close(self) -> None:
        for p in self._owned:
            p.close()
        self._owned = []
