"""The circuit of the reference's prover benchmark (halo2_proofs/benches/plonk.rs:16-246: StandardPlonk with three advice columns
a, b, c under one permutation, four fixed columns sm, sa, sb, sc, one gate a*sa + b*sb + a*b*sm - c*sc, minimum degree 5; for a
given k it fills 2^k - 6 rows -- every usable row -- with (2^(k-1) - 3) multiply / add pairs and two copy constraints per pair),
rebuilt from its source as columns, permutation polynomials, a witness and a PINNED KEY TEXT in the format of
`format!("{:#?}", vk.pinned())`, so that tests/plonk_prover.py and tests/plonk_verifier.py can prove and verify it.  Test
infrastructure; the columns and the key text are pure integer bookkeeping (the commitments in the key text are supplied by the
caller's keygen).  Below them: the circuit's copy constraints, and its seeded generators and columns as the tests set them up."""
from __future__ import annotations

from oracle import cref, pasta
from tests import plonk_api_circuit as circ

BLINDING_FACTORS = 5                                               # max(3, 1 query per advice column) + 2, plonk/circuit.rs:1435-1460
DEGREE = 5                                                         # set_minimum_degree(5), benches/plonk.rs:183


def columns(k: int, modulus: int, omega: int, delta: int, a_value: int):
    """(fixed [sm, sa, sb, sc], sigma [a, b, c], advice [a, b, c]) as Lagrange values.  Rows (SimpleFloorPlanner, one row per
    region): 2i = raw_multiply (a, a, a^2; sc = sm = 1), 2i + 1 = raw_add (a, a^2, a^2 + a; sa = sb = sc = 1); copy(a0, a1) and
    copy(b1, c0) per pair (benches/plonk.rs:226-241), merged as plonk/permutation/keygen.rs:44-100."""
    n = 1 << k
    m = modulus
    pairs = (1 << (k - 1)) - 3
    a2 = a_value * a_value % m
    fixed = [[0] * n for _ in range(4)]
    adv = [[0] * n for _ in range(3)]
    ncols = 3
    mapping = [[(i, j) for j in range(n)] for i in range(ncols)]
    aux = [[(i, j) for j in range(n)] for i in range(ncols)]
    sizes = [[1] * n for _ in range(ncols)]

    def copy(lc, lr, rc, rr):
        left, right = aux[lc][lr], aux[rc][rr]
        if left == right:
            return
        if sizes[left[0]][left[1]] < sizes[right[0]][right[1]]:
            left, right = right, left
        sizes[left[0]][left[1]] += sizes[right[0]][right[1]]
        i = right
        while True:
            aux[i[0]][i[1]] = left
            i = mapping[i[0]][i[1]]
            if i == right:
                break
        mapping[lc][lr], mapping[rc][rr] = mapping[rc][rr], mapping[lc][lr]

    for it in range(pairs):
        rm, ra = 2 * it, 2 * it + 1
        fixed[0][rm], fixed[3][rm] = 1, 1                          # sm, sc
        fixed[1][ra], fixed[2][ra], fixed[3][ra] = 1, 1, 1         # sa, sb, sc
        adv[0][rm], adv[1][rm], adv[2][rm] = a_value, a_value, a2
        adv[0][ra], adv[1][ra], adv[2][ra] = a_value, a2, (a2 + a_value) % m
        copy(0, rm, 0, ra)                                         # copy(a0, a1)
        copy(1, ra, 2, rm)                                         # copy(b1, c0)
    omega_powers = [1] * n
    for j in range(1, n):
        omega_powers[j] = omega_powers[j - 1] * omega % m
    deltas = [pow(delta, i, m) for i in range(ncols)]
    sigma = [[deltas[mapping[i][j][0]] * omega_powers[mapping[i][j][1]] % m for j in range(n)] for i in range(ncols)]
    return fixed, sigma, adv


def _hex(v: int) -> str:
    return "0x%064x" % v


def pinned_key_text(k: int, extended_k: int, base_modulus: int, scalar_modulus: int, omega: int, fixed_commitments, permutation_commitments) -> str:
    """The key in the shape of `{:#?}` of PinnedVerificationKey (src/plonk.rs:117-131, circuit.rs:971-994): what
    tests/plonk_verifier.PinnedKey parses and hashes.  Advice queries come from enable_equality (a, b, c at Rotation::cur()),
    fixed queries from the gate in the order sa, sb, sc, sm (benches/plonk.rs:185-208)."""
    def q(kind, qi, ci):
        return f"{kind} {{\nquery_index: {qi},\ncolumn_index: {ci},\nrotation: Rotation(\n0,\n),\n}},"
    prod = lambda x, y: f"Product(\n{x}\n{y}\n),"
    a, b, c = q("Advice", 0, 0), q("Advice", 1, 1), q("Advice", 2, 2)
    sa, sb, sc, sm = q("Fixed", 0, 1), q("Fixed", 1, 2), q("Fixed", 2, 3), q("Fixed", 3, 0)
    gate = f"Sum(\nSum(\nSum(\n{prod(a, sa)}\n{prod(b, sb)}\n),\n{prod(prod(a, b), sm)}\n),\nNegated(\n{prod(c, sc)}\n),\n),"
    col = lambda idx, kind: f"Column {{\nindex: {idx},\ncolumn_type: {kind},\n}},"
    query = lambda idx, kind: f"(\n{col(idx, kind)}\nRotation(\n0,\n),\n),"
    pts = lambda ps: "\n".join(f"({_hex(x)}, {_hex(y)})," for x, y in ps)
    return "\n".join([
        "PinnedVerificationKey {",
        f'base_modulus: "0x{base_modulus:064x}",', f'scalar_modulus: "0x{scalar_modulus:064x}",',
        "domain: PinnedEvaluationDomain {", f"k: {k},", f"extended_k: {extended_k},", f"omega: {_hex(omega)},", "},",
        "cs: PinnedConstraintSystem {", "num_fixed_columns: 4,", "num_advice_columns: 3,", "num_instance_columns: 0,", "num_selectors: 0,",
        "gates: [", gate, "],",
        "advice_queries: [", query(0, "Advice"), query(1, "Advice"), query(2, "Advice"), "],",
        "instance_queries: [],",
        "fixed_queries: [", query(1, "Fixed"), query(2, "Fixed"), query(3, "Fixed"), query(0, "Fixed"), "],",
        "permutation: Argument {", "columns: [", col(0, "Advice"), col(1, "Advice"), col(2, "Advice"), "],", "},",
        "lookups: [],", "constants: [],", "minimum_degree: Some(\n5,\n),", "},",
        "fixed_commitments: [", pts(fixed_commitments), "],",
        "permutation: VerifyingKey {", "commitments: [", pts(permutation_commitments), "],", "},",
        "}"])


def bench_copies(k: int):
    """The copy constraints (benches/plonk.rs:226-241): copy(a0, a1) and copy(b1, c0) per multiply / add pair."""
    for it in range((1 << (k - 1)) - 3):
        rm, ra = 2 * it, 2 * it + 1
        yield 0, rm, 0, ra
        yield 1, ra, 2, rm


def _bench_setup(k: int):
    """(curve, modulus, (g, g_lagrange, w, u) of seeded generators, fixed, sigma, advice, copies) at k."""
    c = pasta.VESTA
    m = pasta.P_MOD
    n = 1 << k
    pts = cref.gen_points("vesta", 99, n + 2)
    gens = (pts[:n], cref.params_lagrange("vesta", pts[:n], k, pasta.inv(pasta.omega_for_k("fp", k), m), pow(pasta.inv(2, m), k, m)),
            pts[n:n + 1], pts[n + 1:n + 2])
    omega = pasta.omega_for_k("fp", k)
    fixed, sigma, adv = columns(k, m, omega, circ.DELTA, circ.A_SMALL * circ.ZETA % m)
    asm_copies = list(bench_copies(k))
    return c, m, gens, fixed, sigma, adv, asm_copies


def _bench_params(eng, k: int):
    """eng.Params over the seeded generators of _bench_setup, g_lagrange derived on the device."""
    n = 1 << k
    pts = cref.gen_points("vesta", 99, n + 2)
    g, w, u = pts[:n], pts[n:n + 1], pts[n + 1:n + 2]
    return eng.Params("vesta", k, g, eng.lagrange_generators("vesta", k, g), w, u=u)


def _bench_assembly(eng, k: int):
    asm = eng.Assembly(1 << k, 3)
    for cp in bench_copies(k):
        asm.copy(*cp)
    return asm
