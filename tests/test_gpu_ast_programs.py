"""The expression evaluator (h2_poly_eval_ast, csrc/asteval.cuh) on the programs the prover really runs and on programs no
mirror emits, against references that do not share its code path.

Every proof goes through this kernel several times: the lookups' compressed columns, the permutation and lookup products'
numerators and denominators (Lagrange basis), and the whole of h(X) over the extended coset.  Three references:
  - a big-integer walk of the Ast tree, one row at a time (`_walk`): it does not go through compile_ast;
  - a big-integer interpreter of the postfix code (`_interpret`), for programs written by hand;
  - the C oracle's interpreter of the same postfix code (cref.ast_eval) and pasta.ast_evaluate, the oracle's tree walk.

The cases:
  - the golden programs: for every pinned key of tests/golden/golden_proofs.json.gz, the Lagrange-basis programs and h(X) of
    two proofs, built by tests/plonk_prover.py's builders and the product programs below, over seeded columns with rows of
    0, 1 and m - 1;
  - generated trees over every node kind and the rotations where wrapping goes wrong, at 1 to 1024 rows;
  - raw programs: NEG, the operand-stack and program-length limits, LinearTerm at n = 1 and 2, shifts of INT32_MIN and
    INT32_MAX, hundreds of leaf handles, thousands of constants, operands longer than 2^log_n;
  - the rest of the quotient pipeline (divide_by_vanishing_poly, extended_to_coeff) on h(X) of one key per degree.
Each case runs on the device (marked gpu) and through the host emulation of the kernel body (emu_ast_eval), where the golden
programs use a smaller domain: a program depends on the domain only through its rotation stride."""
import ctypes
import random
import types

import numpy as np
import pytest

from oracle import cref, pasta
from tests import plonk_prover as PP
from tests import plonk_verifier as PV

SEED = 0x41535450
FIELDS = ("fp", "fq")
STACK = 24                                   # H2_AST_STACK
MAX_CODE = 1 << 20                           # the longest program h2_poly_eval_ast takes
OP_POLY, OP_CONST, OP_LINEAR, OP_ADD, OP_MUL, OP_SCALE, OP_NEG = range(7)
CASES = PV.load_golden_proofs()
# per key: (instructions, depth) of compile_ast(distribute_powers(gates, y)), the gate part of h(X)
GATE_PART = {"plonk_api": (35, 5), "ecc_chip": (2683, 7), "ecc_chip_4_5b": (2683, 7), "merkle_chip": (645, 9),
             "merkle_with_private_init_chip_4_5b": (665, 9), "sinsemilla_chip": (3059, 9), "sinsemilla_with_private_init_chip_4_5b": (3059, 9)}
# one key per degree 6 to 9 (quotients of 5n to 8n coefficients at k = 11) for the quotient pipeline
PIPELINE = {"lookup_range_check": 6, "merkle_chip": 7, "lookup_range_check_4_5b": 8, "sinsemilla_chip": 9}


def _ast():
    from halo2_b200.evaluator import Ast, AstLeaf, compile_ast
    return Ast, AstLeaf, compile_ast


# ------------------------------------------------------------------------------------------ references
def _walk(node, row: int, n: int, stride: int, m: int, col, lin: int) -> int:
    """One row of an Ast, walked as a tree over Python integers.  `col(index, row)`: a leaf's value; `lin`: the basis'
    LinearTerm factor at this row (omega^row, or zeta * extended_omega^row)."""
    k, a = node.kind, node.args
    if k == "poly":
        return col(a[0], (row + a[1] * stride) % n)
    if k == "add":
        return (_walk(a[0], row, n, stride, m, col, lin) + _walk(a[1], row, n, stride, m, col, lin)) % m
    if k == "mul":
        return _walk(a[0], row, n, stride, m, col, lin) * _walk(a[1], row, n, stride, m, col, lin) % m
    if k == "scale":
        return _walk(a[0], row, n, stride, m, col, lin) * a[1] % m
    if k == "dp":
        acc = 0
        for t in a[0]:
            acc = (acc * a[1] + _walk(t, row, n, stride, m, col, lin)) % m
        return acc
    if k == "lin":
        return a[0] * lin % m
    if k == "const":
        return a[0] % m
    raise ValueError(k)


def _interpret(code, consts, col, row: int, n: int, m: int, lin: int) -> int:
    """One row of a postfix program over Python integers: shifts are signed 32-bit and wrap at n."""
    st = []
    for op, arg, shift, _ in code.tolist():
        if op == OP_POLY:
            st.append(col(arg, (row + (shift - (1 << 32) if shift >= 1 << 31 else shift)) % n))
        elif op == OP_CONST:
            st.append(consts[arg] % m)
        elif op == OP_LINEAR:
            st.append(consts[arg] * lin % m)
        elif op == OP_ADD:
            b = st.pop()
            st[-1] = (st[-1] + b) % m
        elif op == OP_MUL:
            b = st.pop()
            st[-1] = st[-1] * b % m
        elif op == OP_SCALE:
            st[-1] = st[-1] * consts[arg] % m
        else:
            st[-1] = -st[-1] % m
    assert len(st) == 1
    return st[0]


def _depth(code) -> int:
    d = top = 0
    for op in code[:, 0].tolist():
        d += 1 if op in (OP_POLY, OP_CONST, OP_LINEAR) else -1 if op in (OP_ADD, OP_MUL) else 0
        top = max(top, d)
    return top


# ------------------------------------------------------------------------------------------ the two evaluators
def _device_eval(field, cols, log_n, code, consts, omega, lin, which=None):
    """h2_poly_eval_ast over freshly uploaded columns (count, 2^log_n, 32); the canonical result.  Leaf handle i is column
    which[i] (default: i), so one resident polynomial may stand behind several handles."""
    import halo2_b200 as eng
    from halo2_b200 import lib as L
    lib = L.init()
    n = 1 << log_n
    polys = [eng.ResidentPoly(field, n, c) for c in cols]
    out = eng.ResidentPoly(field, n)
    try:
        handles = [polys[w]._h.value for w in (range(len(cols)) if which is None else which)]
        L.check(_call(lib, L, out, handles, log_n, code, consts, omega, lin))
        return out.download()
    finally:
        for p in polys + [out]:
            p.close()


def _call(lib, L, out, handles, log_n, code, consts, omega, lin):
    hs = (ctypes.c_uint64 * max(len(handles), 1))(*handles)
    cs = cref.ints_to_bytes(consts) if len(consts) else None
    return lib.h2_poly_eval_ast(out._h, hs, ctypes.c_size_t(len(handles)), ctypes.c_uint32(log_n), code.ctypes.data_as(ctypes.c_void_p),
                                ctypes.c_size_t(code.shape[0]), L.ptr(cs), ctypes.c_size_t(len(consts)),
                                L.ptr(L.fe_bytes(omega)), L.ptr(L.fe_bytes(lin)), L.REPR_CANONICAL)


_EMU = []


def _emu():
    if not _EMU:
        from tests.kernel_emul import build as emul_build
        _EMU.append(ctypes.CDLL(emul_build.build()))
    return _EMU[0]


def _emu_eval(field, cols, log_n, code, consts, omega, lin, which=None):
    """The kernel body run serially on the host (tests/kernel_emul/emul_asteval.cpp); `which` as for _device_eval."""
    emu = _emu()
    n = 1 << log_n
    cols = cols if which is None else cols[list(which)]
    pb = np.ascontiguousarray(cols if len(cols) else np.zeros((1, n, 32), dtype=np.uint8))
    cs = cref.ints_to_bytes(consts) if len(consts) else np.zeros((1, 32), dtype=np.uint8)
    out = np.zeros((n, 32), dtype=np.uint8)
    assert emu.emu_ast_eval(cref.FIELD_ID[field], cref._p(pb), len(cols), log_n, code.ctypes.data_as(ctypes.c_void_p), code.shape[0], cref._p(cs),
                            len(consts), cref._p(cref._fe(omega)), cref._p(cref._fe(lin)), cref._p(out)) == 0
    return out


# ------------------------------------------------------------------------------------------ inputs
def _columns(field, count, n, seed):
    """(count, n, 32) seeded canonical values; row 1 is 0, row 2 is 1 and row 3 is m - 1 in every column (when n > 3), and
    three more rows of each column hold one of the three."""
    m = pasta.FIELDS[field]
    cols = cref.gen_scalars(field, seed, max(count, 1) * n).reshape(max(count, 1), n, 32)[:count].copy()
    special = [cref.ints_to_bytes([v])[0] for v in (0, 1, m - 1)]
    rnd = random.Random(seed)
    for c in range(count):
        for r, v in zip((1, 2, 3), special):
            if r < n:
                cols[c, r] = v
        for _ in range(3):
            cols[c, rnd.randrange(n)] = special[rnd.randrange(3)]
    return cols


def _col_reader(cols):
    cache = {}

    def col(i, r):
        if (i, r) not in cache:
            cache[(i, r)] = int.from_bytes(cols[i, r].tobytes(), "little")
        return cache[(i, r)]
    return col


def _rows(n, shifts, count, seed):
    """Rows 0 to 3 and n - 1, both sides of every shift's wrap, then seeded rows up to `count`; every row when n <= count."""
    if n <= count:
        return list(range(n))
    rows = {0, 1, 2, 3, n - 1}
    for s in shifts:
        s %= n
        if s:
            rows |= {n - s - 1, n - s}                    # the last row that reads forward, the first that wraps
    rnd = random.Random(seed)
    while len(rows) < count:
        rows.add(rnd.randrange(n))
    return sorted(rows)


def _lin_factor(m, omega, lin_base, row):
    return lin_base * pow(omega, row, m) % m


def _shifts(code):
    return {s - (1 << 32) if s >= 1 << 31 else s for op, _, s, _ in code.tolist() if op == OP_POLY}


# ------------------------------------------------------------------------------------------ the golden programs
class _Leaves:
    def __init__(self):
        self.count = 0

    def new(self, k):
        _, AstLeaf, _ = _ast()
        self.count += k
        return [AstLeaf(self.count - k + i) for i in range(k)]


# The product columns' programs (Lagrange basis) of the reference's loops; the batched product calls run them in one kernel.
def permutation_denominator(eng, cols, sigmas, beta: int, gamma: int):
    """permutation/prover.rs commit, before batch_invert: prod_j (beta * sigma_j + gamma + column_j) over one chunk of columns."""
    den = None
    for col, sl in zip(cols, sigmas):
        term = sl * beta + eng.Ast.constant_term(gamma) + col
        den = term if den is None else den * term
    return den


def permutation_numerator(eng, inv_den, cols, first: int, beta: int, gamma: int, delta: int, m: int):
    """permutation/prover.rs commit, after batch_invert: 1 / den * prod_j (beta * delta^(first + j) * omega^row + gamma + column_j); `first` is the
    chunk's first global column index."""
    num = inv_den
    for j, col in enumerate(cols):
        num = num * (eng.Ast.linear_term(pow(delta, first + j, m) * beta % m) + eng.Ast.constant_term(gamma) + col)
    return num


def lookup_product_denominator(eng, permuted_input, permuted_table, beta: int, gamma: int):
    """lookup/prover.rs commit_product, before batch_invert: (A' + beta) (S' + gamma)."""
    return (permuted_input + eng.Ast.constant_term(beta)) * (permuted_table + eng.Ast.constant_term(gamma))


def lookup_product_numerator(eng, inv_den, input_, table, beta: int, gamma: int):
    """lookup/prover.rs commit_product, after batch_invert: 1 / den * (A + beta) (S + gamma), A and S the compressed columns."""
    return inv_den * (input_ + eng.Ast.constant_term(beta)) * (table + eng.Ast.constant_term(gamma))


def golden_programs(vk: PV.PinnedKey, m: int, num_proofs: int, seed: int):
    """The prover's programs of `num_proofs` proofs under `vk`, built by the builders above and tests/plonk_prover.py's with seeded
    challenges in the field of modulus m: ([(name, Lagrange-basis Ast)], Lagrange leaf count, h(X), extended leaf count,
    the gate part of h(X))."""
    Ast, _, _ = _ast()
    E = types.SimpleNamespace(Ast=Ast)
    rnd = random.Random(seed)
    theta, beta, gamma, y = (rnd.randrange(m) for _ in range(4))
    delta = PV.scalar_delta(m)
    chunk_len = vk.degree() - 2
    n_sets = -(-len(vk.permutation_columns) // chunk_len)
    lag = _Leaves()
    FL, SL = lag.new(vk.num_fixed_columns), lag.new(len(vk.permutation_columns))
    AL = [lag.new(vk.num_advice_columns) for _ in range(num_proofs)]
    IL = [lag.new(vk.num_instance_columns) for _ in range(num_proofs)]
    progs = []
    for pr in range(num_proofs):
        for li, (inp, tab) in enumerate(vk.lookups):
            progs += [(f"lookup {li} input", PP.lookup_compression(E, inp, theta, FL, AL[pr], IL[pr])),
                      (f"lookup {li} table", PP.lookup_compression(E, tab, theta, FL, AL[pr], IL[pr]))]
        leaf = lambda col: {"Advice": AL[pr], "Fixed": FL, "Instance": IL[pr]}[col[0]][col[1]]
        for first in range(0, len(vk.permutation_columns), chunk_len):
            cols = [leaf(c) for c in vk.permutation_columns[first:first + chunk_len]]
            progs += [(f"permutation {first} den", permutation_denominator(E, cols, SL[first:first + chunk_len], beta, gamma)),
                      (f"permutation {first} num", permutation_numerator(E, lag.new(1)[0], cols, first, beta, gamma, delta, m))]
        for li in range(len(vk.lookups)):
            PI, PT, CI, CT = lag.new(4)
            progs += [(f"lookup {li} product den", lookup_product_denominator(E, PI, PT, beta, gamma)),
                      (f"lookup {li} product num", lookup_product_numerator(E, lag.new(1)[0], CI, CT, beta, gamma))]
    ext = _Leaves()
    FC, SC, LG = ext.new(vk.num_fixed_columns), ext.new(len(vk.permutation_columns)), ext.new(3)
    exprs, gates = [], None
    for pr in range(num_proofs):
        AC, IC, ZC = ext.new(vk.num_advice_columns), ext.new(vk.num_instance_columns), ext.new(n_sets if vk.permutation_columns else 0)
        LK = [tuple(ext.new(5)) for _ in vk.lookups]
        exprs += PP.vanishing_expressions(E, vk, beta, gamma, delta, FC, SC, LG, AC, IC, ZC, LK)
        gates = gates or Ast.distribute_powers(exprs[:len(vk.gates)], y)
    return progs, lag.count, Ast.distribute_powers(exprs, y), ext.count, gates


def _check_golden(evaluate, case, field, k, min_rows):
    """Every program of the key in `case`, with two proofs, run at 2^k rows (Lagrange) and at the key's extended size relative
    to k, in `field`: the whole output against cref.ast_eval of the same code, `min_rows` or more rows against the tree walk,
    the depth within the operand stack.  Returns the extended domain and h(X)'s values, for the quotient pipeline."""
    _, _, compile_ast = _ast()
    vk = PV.PinnedKey(case["key_text"])
    m = pasta.FIELDS[field]
    D = pasta.EvaluationDomain(field, vk.degree(), k, pasta.zeta_candidates(field)[0])
    assert D.extended_k - k == vk.extended_k - vk.k
    progs, n_lag, h, n_ext, gates = golden_programs(vk, m, 2, SEED + k)
    gcode, gconsts = compile_ast(gates, m, 1)
    print(f"\n{case['name']} ({field}, k = {k}): gate part {gcode.shape[0]} instructions / {len(gconsts)} constants / depth {_depth(gcode)}")
    if case["name"] in GATE_PART:
        assert (gcode.shape[0], _depth(gcode)) == GATE_PART[case["name"]]
    widest = 0
    for basis, log_n, ast, count in [("lagrange", k, a, n_lag) for _, a in progs] + [("extended", D.extended_k, h, n_ext)]:
        n, stride = 1 << log_n, 1 << (log_n - k)
        omega, lin_base = (D.omega, 1) if basis == "lagrange" else (D.extended_omega, D.g_coset)
        code, consts = compile_ast(ast, m, stride)
        depth = _depth(code)
        widest = max(widest, depth)
        assert depth <= STACK, (case["name"], basis, depth)
        cols = _columns(field, count, n, SEED + 7 * log_n + count)
        got = evaluate(field, cols, log_n, code, consts, omega, lin_base)
        assert (got == cref.ast_eval(field, cols, log_n, code, consts, omega, lin_base)).all(), (case["name"], basis)
        col = _col_reader(cols)
        for row in _rows(n, _shifts(code), min_rows, SEED + log_n):
            want = _walk(ast, row, n, stride, m, col, _lin_factor(m, omega, lin_base, row))
            assert int.from_bytes(got[row].tobytes(), "little") == want, (case["name"], basis, row)
        if basis == "extended":
            print(f"  h(X): {code.shape[0]} instructions / {len(consts)} constants / {count} leaves / depth {depth}; deepest program {widest}")
            return D, got
    raise AssertionError("unreachable")


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_programs_emulated(case, field):
    """The golden programs through the host emulation of the kernel body at k = 3 (8 rows, the key's own rotation stride):
    every row against the tree walk."""
    _check_golden(_emu_eval, case, field, 3, 64)


@pytest.mark.gpu
@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_programs_device(case, field):
    """The golden programs on the device at the key's own k and extended_k; for one key per degree, in the key's own field,
    h(X) then goes through divide_by_vanishing_poly and extended_to_coeff on the device against the oracle's steps."""
    import halo2_b200 as eng
    vk = PV.PinnedKey(case["key_text"])
    D, h = _check_golden(_device_eval, case, field, vk.k, 64)
    if case["name"] not in PIPELINE or pasta.FIELDS[field] != vk.scalar_modulus:
        return
    assert vk.degree() == PIPELINE[case["name"]]
    d = eng.EvaluationDomain(field, vk.degree(), vk.k, D.g_coset)
    res = eng.ResidentPoly(field, D.extended_len(), h)
    d.divide_by_vanishing_poly_resident(res)
    div = D.divide_by_vanishing_poly(cref.bytes_to_ints(h))
    assert cref.bytes_to_ints(res.download()) == div
    got = d.extended_to_coeff_resident(res)
    want = cref.extended_to_coeff(field, cref.ints_to_bytes(div), D.extended_k, D.extended_omega_inv, D.extended_ifft_divisor, D.g_coset,
                                  D.n * (vk.degree() - 1))
    assert got.len == D.n * (vk.degree() - 1) and (got.download() == want).all()
    got.close()
    res.close()


# ------------------------------------------------------------------------------------------ generated trees
def _gen_tree(rnd, m, n_leaves, n, height):
    """A random Ast over every node kind: leaves with the rotations where wrapping goes wrong, constants and LinearTerms of
    0, 1 and m - 1, scales by 0, 1 and m - 1, DistributePowers of 0, 1 and several terms."""
    Ast, AstLeaf, _ = _ast()
    special = lambda: rnd.choice([0, 1, m - 1, rnd.randrange(m)])
    kinds = ["poly", "const", "lin"] + (["add", "mul", "scale", "dp"] * 2 if height > 0 else [])
    kind = rnd.choice(kinds)
    if kind == "poly":
        rot = rnd.choice([0, 1, -1, 2, -2, n - 1, -(n - 1), n, -n, n + 1, -(n + 1), 3 * n + 5, rnd.randrange(-(1 << 24), 1 << 24)])
        return AstLeaf(rnd.randrange(n_leaves)).with_rotation(rot)
    if kind == "const":
        return Ast.constant_term(special())
    if kind == "lin":
        return Ast.linear_term(special())
    sub = lambda: _gen_tree(rnd, m, n_leaves, n, height - 1)
    if kind == "scale":
        return sub() * special()
    if kind == "dp":
        return Ast.distribute_powers([sub() for _ in range(rnd.choice([0, 1, rnd.randint(2, 5)]))], special())
    return sub() + sub() if kind == "add" else sub() * sub()


def _domain(field, basis, log_n):
    """A domain whose `basis` has 2^log_n values: Lagrange at k = log_n; extended at k = log_n - 1 (stride 2), or k = 0 with
    stride 1 when log_n = 0."""
    zeta = pasta.zeta_candidates(field)[0]
    if basis == "lagrange" or log_n == 0:
        return pasta.EvaluationDomain(field, 2, log_n, zeta)
    return pasta.EvaluationDomain(field, 3, log_n - 1, zeta)


def _check_generated(evaluate, field, basis, log_n, trees):
    _, _, compile_ast = _ast()
    d = _domain(field, basis, log_n)
    m, n = d.m, 1 << log_n
    stride = 1 if basis == "lagrange" else 1 << (d.extended_k - d.k)
    omega, lin_base = (d.omega, 1) if basis == "lagrange" else (d.extended_omega, d.g_coset)
    rnd = random.Random(SEED + 31 * log_n + (basis == "extended") + 2 * (field == "fq"))
    cols = _columns(field, 6, n, SEED + 100 + log_n)
    ints = [cref.bytes_to_ints(c) for c in cols]
    done = 0
    while done < trees:
        ast = _gen_tree(rnd, m, 6, d.n, rnd.randint(1, 6))
        code, consts = compile_ast(ast, m, stride)
        if _depth(code) > STACK:
            continue
        got = cref.bytes_to_ints(evaluate(field, cols, log_n, code, consts, omega, lin_base))
        assert got == pasta.ast_evaluate(d, basis, _tuple(ast), ints), (basis, log_n, done)
        assert got == cref.bytes_to_ints(cref.ast_eval(field, cols, log_n, code, consts, omega, lin_base)), (basis, log_n, done)
        done += 1


def _tuple(node):
    """halo2_b200.evaluator.Ast -> the nested tuples of pasta.ast_evaluate."""
    k, a = node.kind, node.args
    if k in ("add", "mul"):
        return (k, _tuple(a[0]), _tuple(a[1]))
    if k == "scale":
        return ("scale", _tuple(a[0]), a[1])
    if k == "dp":
        return ("dp", [_tuple(t) for t in a[0]], a[1])
    return (k,) + tuple(a)


GENERATED = [(b, log_n) for b in ("lagrange", "extended") for log_n in (0, 1, 2, 3, 6, 10)]


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("basis,log_n", GENERATED)
def test_generated_programs_emulated(field, basis, log_n):
    _check_generated(_emu_eval, field, basis, log_n, 40 if log_n <= 6 else 8)


@pytest.mark.gpu
@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("basis,log_n", GENERATED)
def test_generated_programs_device(field, basis, log_n):
    _check_generated(_device_eval, field, basis, log_n, 40 if log_n <= 6 else 16)


# ------------------------------------------------------------------------------------------ raw programs
def _prog(rows):
    return np.ascontiguousarray(np.array(rows, dtype=np.int64).astype(np.uint32).reshape(-1, 4))


def _stack_program(depth, n_polys):
    """Pushes `depth` operands (leaves, a constant, a LinearTerm), negates the top, then folds them with alternating MUL
    and ADD: an operand stack exactly `depth` deep."""
    rows = []
    for i in range(depth):
        rows.append([OP_POLY, i % n_polys, i - depth // 2, 0] if i % 3 else [(OP_CONST, OP_LINEAR)[i % 2], i % 2, 0, 0])
    rows.append([OP_NEG, 0, 0, 0])
    rows += [[OP_MUL if i % 2 else OP_ADD, 0, 0, 0] for i in range(depth - 1)]
    return _prog(rows)


def raw_programs(m, n):
    """(name, code, consts, n_polys) of programs the Python and Rust flatteners never emit; every one is within the limits."""
    rnd = random.Random(SEED + n)
    c = lambda k: [rnd.randrange(m) for _ in range(k)]
    many = c(5000)
    progs = [
        ("neg of a leaf", _prog([[OP_POLY, 0, 0, 0], [OP_NEG, 0, 0, 0]]), [], 2),
        ("neg of zero", _prog([[OP_CONST, 0, 0, 0], [OP_NEG, 0, 0, 0]]), [0], 1),
        ("neg of m - 1 and twice", _prog([[OP_CONST, 0, 0, 0], [OP_NEG, 0, 0, 0], [OP_POLY, 1, 1, 0], [OP_NEG, 0, 0, 0], [OP_NEG, 0, 0, 0],
                                          [OP_MUL, 0, 0, 0], [OP_NEG, 0, 0, 0]]), [m - 1], 2),
        ("neg under a scale", _prog([[OP_POLY, 0, 0, 0], [OP_POLY, 1, -1, 0], [OP_NEG, 0, 0, 0], [OP_SCALE, 0, 0, 0], [OP_ADD, 0, 0, 0]]), c(1), 2),
        ("depth 24", _stack_program(STACK, 3), c(2), 3),
        ("shifts of INT32_MIN and INT32_MAX", _prog([[OP_POLY, 0, -(1 << 31), 0], [OP_POLY, 1, (1 << 31) - 1, 0], [OP_MUL, 0, 0, 0],
                                                     [OP_POLY, 0, (1 << 31) - 1, 0], [OP_ADD, 0, 0, 0], [OP_POLY, 1, -(1 << 31) + 1, 0],
                                                     [OP_ADD, 0, 0, 0]]), [], 2),
        ("LinearTerm", _prog([[OP_LINEAR, 0, 0, 0], [OP_LINEAR, 1, 0, 0], [OP_MUL, 0, 0, 0], [OP_POLY, 0, 1, 0], [OP_LINEAR, 2, 0, 0],
                              [OP_ADD, 0, 0, 0], [OP_ADD, 0, 0, 0]]), [1, m - 1, rnd.randrange(m)], 1),
    ]
    # 300 leaf handles (the caller repeats operands: handle i is column i % 7), each scaled while the running sum sits below it
    rows = [[OP_POLY, 0, 0, 0]]
    for i in range(1, 300):
        rows += [[OP_POLY, i, rnd.randrange(-3, 4), 0], [OP_SCALE, i % 3, 0, 0], [OP_MUL if i % 4 == 0 else OP_ADD, 0, 0, 0]]
    progs.append(("300 leaf handles", _prog(rows), c(3), 300))
    # 5000 constants, each used once by CONST, SCALE or LINEAR, the last index included
    rows = [[OP_CONST, 0, 0, 0]]
    for i in range(1, len(many)):
        rows += [[OP_LINEAR, i, 0, 0], [OP_ADD, 0, 0, 0]] if i % 3 == 0 else [[OP_CONST, i, 0, 0], [OP_MUL, 0, 0, 0]] if i % 3 == 1 else \
            [[OP_SCALE, i, 0, 0]]
    progs.append(("5000 constants", _prog(rows + [[OP_POLY, 0, n, 0], [OP_ADD, 0, 0, 0]]), many, 1))
    return progs


def _longest_program():
    """2^20 instructions: a leaf, (2^20 - 2) / 2 pairs of CONST / ADD, a NEG."""
    rows = np.zeros((MAX_CODE, 4), dtype=np.uint32)
    rows[0] = [OP_POLY, 0, 1, 0]
    rows[1:-1:2, 0] = OP_CONST
    rows[1:-1:2, 1] = np.arange((MAX_CODE - 2) // 2) % 3
    rows[2:-1:2, 0] = OP_ADD
    rows[-1, 0] = OP_NEG
    return rows


def _check_raw(evaluate, field, log_n):
    m = pasta.FIELDS[field]
    n = 1 << log_n
    d = pasta.EvaluationDomain(field, 3, log_n, pasta.zeta_candidates(field)[0])
    omega, lin_base = d.omega, d.g_coset                 # a LinearTerm in the coset's form: zeta * omega^row
    cols = _columns(field, 7, n, SEED + 500 + log_n)
    for name, code, consts, n_polys in raw_programs(m, n):
        assert _depth(code) <= STACK and code.shape[0] <= MAX_CODE
        which = [i % len(cols) for i in range(n_polys)]       # 300 handles name 7 columns
        operands = np.ascontiguousarray(cols[which])
        got = evaluate(field, cols, log_n, code, consts, omega, lin_base, which)
        assert (got == cref.ast_eval(field, operands, log_n, code, consts, omega, lin_base)).all(), (name, log_n)
        col = _col_reader(operands)
        for row in range(n) if n <= 64 else _rows(n, _shifts(code), 64, SEED):
            want = _interpret(code, consts, col, row, n, m, _lin_factor(m, omega, lin_base, row))
            assert int.from_bytes(got[row].tobytes(), "little") == want, (name, log_n, row)
    assert _depth(_stack_program(STACK, 3)) == STACK


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("log_n", [0, 1, 2, 5, 11])
def test_raw_programs_emulated(field, log_n):
    _check_raw(_emu_eval, field, log_n)


@pytest.mark.gpu
@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("log_n", [0, 1, 2, 5, 11])
def test_raw_programs_device(field, log_n):
    _check_raw(_device_eval, field, log_n)


@pytest.mark.parametrize("field", FIELDS)
def test_longest_program_emulated(field):
    """2^20 instructions at two rows against the postfix interpreter."""
    m = pasta.FIELDS[field]
    code, consts = _longest_program(), [1, m - 1, 5]
    cols = _columns(field, 1, 2, SEED + 600)
    got = _emu_eval(field, cols, 1, code, consts, 1, 1)
    col = _col_reader(cols)
    assert [int.from_bytes(got[r].tobytes(), "little") for r in range(2)] == [_interpret(code, consts, col, r, 2, m, 1) for r in range(2)]


@pytest.mark.gpu
@pytest.mark.parametrize("field", FIELDS)
def test_program_limits_device(field):
    """The host's limits: a program of exactly 2^20 instructions and one exactly 24 operands deep are evaluated; one more
    instruction, or one operand deeper, is refused before anything is launched and the output keeps its values.  Operands
    longer than 2^log_n hold a marker past 2^log_n: rotations wrap at 2^log_n, never into the tail, and the output's tail
    is not written."""
    import halo2_b200 as eng
    from halo2_b200 import lib as L
    lib = L.init()
    m = pasta.FIELDS[field]
    log_n, n = 1, 2
    cols = _columns(field, 3, n, SEED + 600)
    polys = [eng.ResidentPoly(field, n, c) for c in cols]
    out = eng.ResidentPoly(field, n, cref.ints_to_bytes([7, 8]))
    hs = [p._h.value for p in polys]
    col = _col_reader(cols)
    code, consts = _longest_program(), [1, m - 1, 5]
    L.check(_call(lib, L, out, hs, log_n, code, consts, 1, 1))
    assert cref.bytes_to_ints(out.download()) == [_interpret(code, consts, col, r, n, m, 1) for r in range(n)]
    deep = _stack_program(STACK, 3)
    L.check(_call(lib, L, out, hs, log_n, deep, [3, 4], m - 1, 1))
    assert cref.bytes_to_ints(out.download()) == [_interpret(deep, [3, 4], col, r, n, m, (m - 1) if r else 1) for r in range(n)]
    before = out.download()
    too_long = np.concatenate([code, np.array([[OP_NEG, 0, 0, 0]], dtype=np.uint32)])
    for bad in (too_long, _stack_program(STACK + 1, 3)):
        launches = eng.launch_count()                 # a download may launch a conversion kernel: count around the call alone
        assert _call(lib, L, out, hs, log_n, bad, [3, 4] if bad.shape[0] < 100 else consts, m - 1, 1) != 0
        assert eng.launch_count() == launches
        assert (out.download() == before).all()
    for p in polys + [out]:
        p.close()
    # operands of 2^log_n + 37 elements with a marker in the tail, the output likewise
    log_n, n, tail = 5, 32, 37
    cols = _columns(field, 3, n, SEED + 601)
    marker = cref.ints_to_bytes([m - 2] * tail)
    polys = [eng.ResidentPoly(field, n + tail, np.concatenate([c, marker])) for c in cols]
    out = eng.ResidentPoly(field, n + tail, np.concatenate([np.zeros((n, 32), dtype=np.uint8), marker]))
    code = _prog([[OP_POLY, 0, n - 1, 0], [OP_POLY, 1, n + 3, 0], [OP_MUL, 0, 0, 0], [OP_POLY, 2, -1, 0], [OP_ADD, 0, 0, 0],
                  [OP_POLY, 0, (1 << 31) - 1, 0], [OP_MUL, 0, 0, 0]])
    L.check(_call(lib, L, out, [p._h.value for p in polys], log_n, code, [], 1, 1))
    got = out.download()
    col = _col_reader(cols)
    assert cref.bytes_to_ints(got[:n]) == [_interpret(code, [], col, r, n, m, 1) for r in range(n)]
    assert (got[n:] == marker).all()
    for p in polys + [out]:
        p.close()
