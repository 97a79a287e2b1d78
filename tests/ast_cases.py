"""Ast cases shared by the evaluator tests (poly/evaluator.rs:129-228): the package's Ast in the oracle's nested-tuple form,
and an h(X)-shaped expression that reaches every node kind."""
from __future__ import annotations


def _ast_tuple(node):
    """halo2_b200.evaluator.Ast -> the oracle's nested-tuple form."""
    k, a = node.kind, node.args
    if k == "poly":
        return ("poly", a[0], a[1])
    if k in ("add", "mul"):
        return (k, _ast_tuple(a[0]), _ast_tuple(a[1]))
    if k == "scale":
        return ("scale", _ast_tuple(a[0]), a[1])
    if k == "dp":
        return ("dp", [_ast_tuple(t) for t in a[0]], a[1])
    return (k, a[0])


def _quotient_like_ast(ev_leaves, y, theta):
    """An h(X)-shaped expression: gates folded by powers of y (DistributePowers), products of rotated columns, a scaled
    selector, the identity term of the permutation argument (LinearTerm) and a constant."""
    from halo2_b200.evaluator import Ast
    a, b, c, q = ev_leaves
    gate0 = (a * b - c) * q
    gate1 = (a.with_rotation(1) - a) * (b.with_rotation(-1) + Ast.constant_term(7)) * 3
    perm = (c + Ast.linear_term(theta) + Ast.constant_term(11)) * (a.with_rotation(-2) + b * theta)
    return Ast.distribute_powers([gate0, gate1, -perm, q.with_rotation(3)], y) + Ast.constant_term(0) * 5
