"""The reference's key generation restated for the keygen tests (plonk/permutation/keygen.rs:24-143): Assembly::new and
Assembly::copy on lists of (column, row) tuples, the permutation polynomials from a mapping, and random mappings to feed
them."""
from __future__ import annotations

import numpy as np


def oracle_assembly(n: int, num_columns: int):
    """Assembly::new (permutation/keygen.rs:25-43): (mapping, aux, sizes) as lists of lists of (column, row) tuples."""
    mapping = [[(i, j) for j in range(n)] for i in range(num_columns)]
    aux = [[(i, j) for j in range(n)] for i in range(num_columns)]
    sizes = [[1] * n for _ in range(num_columns)]
    return mapping, aux, sizes


def oracle_copy(asm, left_column: int, left_row: int, right_column: int, right_row: int) -> None:
    """Assembly::copy (permutation/keygen.rs:45-100); IndexError for Error::BoundsFailure."""
    mapping, aux, sizes = asm
    if left_row >= len(mapping[left_column]) or right_row >= len(mapping[right_column]):
        raise IndexError("BoundsFailure")
    left_cycle = aux[left_column][left_row]
    right_cycle = aux[right_column][right_row]
    if left_cycle == right_cycle:
        return
    if sizes[left_cycle[0]][left_cycle[1]] < sizes[right_cycle[0]][right_cycle[1]]:
        left_cycle, right_cycle = right_cycle, left_cycle
    sizes[left_cycle[0]][left_cycle[1]] += sizes[right_cycle[0]][right_cycle[1]]
    i = right_cycle
    while True:
        aux[i[0]][i[1]] = left_cycle
        i = mapping[i[0]][i[1]]
        if i == right_cycle:
            break
    tmp = mapping[left_column][left_row]
    mapping[left_column][left_row] = mapping[right_column][right_row]
    mapping[right_column][right_row] = tmp


def oracle_sigma(mapping, n: int, omega: int, delta: int, m: int):
    """build_vk / build_pk's permutation polynomials (permutation/keygen.rs:108-143): the serial omega-power loop, the
    deltaomega table, the gather.  `mapping[i][j]` = (column, row)."""
    omega_powers = []
    cur = 1
    for _ in range(n):
        omega_powers.append(cur)
        cur = cur * omega % m
    deltaomega = []
    cur = 1
    for _ in range(len(mapping)):
        deltaomega.append([o * cur % m for o in omega_powers])
        cur = cur * delta % m
    return [[deltaomega[int(c)][int(r)] for c, r in mapping[i]] for i in range(len(mapping))]


def random_mapping(rng, cols: int, n: int) -> np.ndarray:
    """Random in-range (column, row) entries, with rows 0 and n - 1 and every column present."""
    mp = np.empty((cols, n, 2), dtype=np.uint32)
    mp[..., 0] = rng.integers(0, cols, size=(cols, n))
    mp[..., 1] = rng.integers(0, n, size=(cols, n))
    mp[0, 0] = (cols - 1, n - 1)
    mp[cols - 1, n - 1] = (0, 0)
    mp[:, 0, 0] = np.arange(cols)
    return mp


def wide_keygen_vk(h2, prm, D, delta: int, fixed_cols: int = 40, perm_cols: int = 30, seed: int = 5):
    """keygen_vk over `prm` of more fixed and permutation columns together than one MSM pass takes (64 polynomials), and the
    same columns committed one at a time with commit_lagrange.  Returns (keygen_vk's (fixed, permutation) commitments, the
    one-at-a-time ones), each an (m, 64) affine array."""
    import random
    from oracle import cref, pasta
    n, m = D.n, D.m
    fixed = [pasta.gen_scalars(D.field, seed + i, n) for i in range(fixed_cols)]
    asm = h2.Assembly(n, perm_cols)
    rnd = random.Random(seed)
    for _ in range(2 * perm_cols):
        asm.copy(rnd.randrange(perm_cols), rnd.randrange(n), rnd.randrange(perm_cols), rnd.randrange(n))
    got = h2.keygen_vk(prm, D, fixed, asm, delta)
    one = lambda col: h2.batch_normalize(prm.commit_lagrange(cref.ints_to_bytes(col), h2.Blind()).reshape(1, 96), prm.curve)[0]  # noqa: E731
    sigma = oracle_sigma(asm.mapping, n, D.omega, delta, m)
    return got, (np.stack([one(c) for c in fixed]), np.stack([one(s) for s in sigma]))
