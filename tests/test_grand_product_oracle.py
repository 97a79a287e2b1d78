"""CPU checks of the product-column kernels (csrc/grandproduct.cuh) on the host emulation, with capi_poly.cu's launch
schedule, against the reference's loops restated with big integers:

- permutation::Argument::commit (plonk/permutation/prover.rs:98-168): every set of every proof, the last_z hand-over from
  set to set, each proof's chain from ONE;
- lookup::Permuted::commit_product (plonk/lookup/prover.rs:279-337).

Both fields, k = 1 ... 10, partial last sets and chunk_len = 1, several proofs per call, rows whose denominator is exactly
zero, bf = 0 and bf = n - 2.  The restatements are also what tests/test_gpu_grand_product_fused.py checks the device against."""
import ctypes

import numpy as np
import pytest

from oracle import cref, pasta
from tests.kernel_emul import build as emul_build

SEED = 0x4B3231


def delta_of(m: int) -> int:
    return pow(pasta.MULT_GEN, 1 << pasta.S_2ADICITY, m)          # F::DELTA


# ---- the reference, restated -------------------------------------------------------------------------------------------
def oracle_permutation_product(columns, sigmas, beta, gamma, omega, delta, chunk_len, bf, blinding, m):
    """permutation/prover.rs:81-168 for every proof: columns[p][c] and sigmas[c] are lists of n ints, blinding the
    proofs x sets x bf values in the rng's order.  Returns z[p][a] (lists of n ints)."""
    n = len(sigmas[0])
    out, at = [], 0
    for cols in columns:
        last_z, deltaomega, sets = 1, 1, []
        for c0 in range(0, len(sigmas), chunk_len):
            mv = [1] * n
            for v, s in zip(cols[c0:c0 + chunk_len], sigmas[c0:c0 + chunk_len]):           # :101-116
                mv = [x * ((beta * s_i + gamma + v_i) % m) % m for x, s_i, v_i in zip(mv, s, v)]
            mv = [pasta.inv(x, m) if x else 0 for x in mv]                                   # :120 batch_invert
            for v in cols[c0:c0 + chunk_len]:                                                # :124-143
                cur = deltaomega
                for i in range(n):
                    mv[i] = mv[i] * ((cur * beta + gamma + v[i]) % m) % m
                    cur = cur * omega % m
                deltaomega = deltaomega * delta % m
            z = [last_z]
            for row in range(1, n):                                                          # :150-156
                z.append(z[row - 1] * mv[row - 1] % m)
            z[n - bf:] = blinding[at:at + bf]                                                # :158-161
            at += bf
            last_z = z[n - (bf + 1)]                                                         # :163
            sets.append(z)
        out.append(sets)
    return out


def oracle_lookup_product(a, s, a_perm, s_perm, beta, gamma, bf, blinding, m):
    """lookup/prover.rs:279-321 for one lookup: compressed input / table a, s and permuted a', s' (lists of n ints)."""
    n = len(a)
    lp = [(beta + x) * (gamma + y) % m for x, y in zip(a_perm, s_perm)]                     # :281-291
    lp = [pasta.inv(x, m) if x else 0 for x in lp]                                           # :295
    lp = [p * ((x + beta) % m) % m * ((y + gamma) % m) % m for p, x, y in zip(lp, a, s)]    # :299-309
    z, state = [], 1
    for cur in [1] + lp:                                                                     # :311-318
        state = state * cur % m
        z.append(state)
    return z[:n - bf] + list(blinding)                                                       # :319-321


# ---- the emulated kernels ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emul_build.build())


def _fe(x):
    return cref._p(cref.ints_to_bytes([x]))


def _blind_ptr(blinding):
    return cref._p(cref.ints_to_bytes(blinding)) if blinding else None


def emu_permutation_product(emu, field, columns, sigmas, beta, gamma, omega, delta, chunk_len, k, bf, blinding):
    n, proofs, cols = 1 << k, len(columns), len(sigmas)
    sets = -(-cols // chunk_len)
    data = cref.ints_to_bytes([x for per in columns for c in per for x in c] + [x for s in sigmas for x in s])
    out = np.zeros((proofs * sets * n, 32), dtype=np.uint8)
    emu.emu_permutation_product(cref.FIELD_ID[field], cref._p(data), proofs, cols, chunk_len, k, _fe(beta), _fe(gamma), _fe(omega), _fe(delta),
                                _blind_ptr(blinding), bf, cref._p(out))
    z = cref.bytes_to_ints(out)
    return [[z[(p * sets + a) * n:(p * sets + a + 1) * n] for a in range(sets)] for p in range(proofs)]


def emu_lookup_product(emu, field, lookups, beta, gamma, k, bf, blinding):
    n = 1 << k
    data = cref.ints_to_bytes([x for lk in lookups for col in lk for x in col])
    out = np.zeros((len(lookups) * n, 32), dtype=np.uint8)
    emu.emu_lookup_product(cref.FIELD_ID[field], cref._p(data), len(lookups), k, _fe(beta), _fe(gamma), _blind_ptr(blinding), bf, cref._p(out))
    z = cref.bytes_to_ints(out)
    return [z[b * n:(b + 1) * n] for b in range(len(lookups))]


def permutation_case(field, k, proofs, cols, bf, seed, zero_rows=()):
    """Random columns, sigmas and challenges; for each (proof, column, row) in zero_rows the column value makes that row's
    denominator term v + beta sigma + gamma exactly zero."""
    m, n = pasta.FIELDS[field], 1 << k
    beta, gamma = pasta.gen_scalars(field, seed, 2)
    sigmas = [pasta.gen_scalars(field, seed + 1 + c, n) for c in range(cols)]
    columns = [[pasta.gen_scalars(field, seed + 100 + 37 * p + c, n) for c in range(cols)] for p in range(proofs)]
    for p, c, r in zero_rows:
        columns[p][c][r] = (-(beta * sigmas[c][r] + gamma)) % m
    return m, beta, gamma, sigmas, columns


PERM_SHAPES = [  # (k, proofs, cols, chunk_len, bf): 1 to 4 sets, partial last sets, chunk_len = 1, bf = 0 and bf = n - 2
    (1, 1, 1, 1, 0), (1, 2, 3, 2, 0), (2, 2, 3, 1, 2), (3, 1, 4, 3, 6), (4, 3, 7, 2, 5), (5, 2, 3, 3, 5), (6, 2, 10, 3, 0),
    (7, 3, 5, 2, 4), (8, 2, 4, 1, 254), (9, 1, 6, 2, 3), (10, 2, 5, 2, 5), (10, 1, 1, 1, 1022),
]


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("k,proofs,cols,chunk_len,bf", PERM_SHAPES)
def test_emul_permutation_product(emu, field, k, proofs, cols, chunk_len, bf):
    n = 1 << k
    seed = SEED + 1000 * k + 10 * cols + chunk_len
    zero_rows = [(proofs - 1, cols - 1, n // 2)] if n > 2 else []
    m, beta, gamma, sigmas, columns = permutation_case(field, k, proofs, cols, bf, seed, zero_rows)
    omega, delta = pasta.omega_for_k(field, k), delta_of(m)
    sets = -(-cols // chunk_len)
    blinding = pasta.gen_scalars(field, seed + 7, proofs * sets * bf) if bf else []
    want = oracle_permutation_product(columns, sigmas, beta, gamma, omega, delta, chunk_len, bf, blinding, m)
    got = emu_permutation_product(emu, field, columns, sigmas, beta, gamma, omega, delta, chunk_len, k, bf, blinding)
    assert got == want
    for p in range(proofs):
        assert got[p][0][0] == 1                                    # every proof's chain starts at ONE
    if zero_rows and n // 2 < n - bf - 1:                           # the zero denominator stays zero: the product vanishes after it
        last = got[proofs - 1]
        a = (cols - 1) // chunk_len
        assert last[a][n // 2 + 1] == 0


@pytest.mark.parametrize("field", ["fp", "fq"])
def test_emul_permutation_carries_across_sets(emu, field):
    """The last_z hand-over: with one proof and four sets, set a + 1 starts at set a's row n - bf - 1."""
    k, cols, chunk_len, bf = 6, 11, 3, 5
    n = 1 << k
    m, beta, gamma, sigmas, columns = permutation_case(field, k, 1, cols, bf, SEED + 77)
    omega, delta = pasta.omega_for_k(field, k), delta_of(m)
    blinding = pasta.gen_scalars(field, SEED + 78, 4 * bf)
    got = emu_permutation_product(emu, field, columns, sigmas, beta, gamma, omega, delta, chunk_len, k, bf, blinding)[0]
    assert len(got) == 4
    for a in range(3):
        assert got[a + 1][0] == got[a][n - bf - 1] and got[a + 1][0] not in (0, 1)
        assert got[a][n - bf:] == blinding[a * bf:(a + 1) * bf]


LOOKUP_SHAPES = [(1, 1, 0), (2, 3, 2), (3, 2, 1), (5, 4, 5), (6, 1, 62), (8, 3, 3), (10, 2, 5), (10, 1, 0)]


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("k,count,bf", LOOKUP_SHAPES)
def test_emul_lookup_product(emu, field, k, count, bf):
    m, n = pasta.FIELDS[field], 1 << k
    seed = SEED + 5000 + 100 * k + count
    beta, gamma = pasta.gen_scalars(field, seed, 2)
    lookups = [[pasta.gen_scalars(field, seed + 10 * b + j + 1, n) for j in range(4)] for b in range(count)]
    if n > 2:
        lookups[-1][2][n // 2] = (-beta) % m                          # a' = -beta: that row's denominator is exactly zero
        lookups[0][3][1] = (-gamma) % m                               # s' = -gamma
    blinding = pasta.gen_scalars(field, seed + 9, count * bf) if bf else []
    want = [oracle_lookup_product(*lk, beta, gamma, bf, blinding[b * bf:(b + 1) * bf], m) for b, lk in enumerate(lookups)]
    got = emu_lookup_product(emu, field, lookups, beta, gamma, k, bf, blinding)
    assert got == want
    assert all(z[0] == 1 for z in got)
