"""ctypes front-end for oracle/halo2_oracle.c (TEST INFRASTRUCTURE ONLY -- see pasta.py).

Everything is canonical little-endian bytes held in numpy uint8 arrays:
scalars (n, 32), affine points (n, 64) with identity = 64 zero bytes.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libhalo2_oracle.so")
_lib: Optional[ctypes.CDLL] = None

FIELD_ID = {"fp": 0, "fq": 1}
CURVE_ID = {"pallas": 0, "vesta": 1}


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "halo2_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _SO


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        build()                  # no-op unless the source is newer than the library
        _lib = ctypes.CDLL(_SO)
        for name in ("orc_best_multiexp", "orc_naive_msm", "orc_best_fft", "orc_ifft", "orc_coeff_to_extended",
                     "orc_extended_to_coeff", "orc_field_op", "orc_scalar_mul", "orc_point_add",
                     "orc_jac_to_affine", "orc_on_curve", "orc_gen_scalars", "orc_gen_points", "orc_ec_fft",
                     "orc_batch_normalize", "orc_params_lagrange", "orc_ipa_rounds", "orc_eval_polynomial", "orc_kate_division", "orc_ast_eval", "orc_compute_s",
                     "orc_permutation_product", "orc_lookup_product", "orc_divide_by_vanishing_poly"):
            getattr(_lib, name).restype = ctypes.c_int
    return _lib


def _p(a: Optional[np.ndarray]):
    if a is None:
        return None
    assert a.dtype == np.uint8 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ctypes.c_void_p)


def _fe(x) -> np.ndarray:
    if isinstance(x, (int,)):
        return np.frombuffer(int(x).to_bytes(32, "little"), dtype=np.uint8).copy()
    a = np.ascontiguousarray(x, dtype=np.uint8)
    assert a.size == 32
    return a


def default_threads() -> int:
    return os.cpu_count() or 1


def best_multiexp(curve: str, scalars: np.ndarray, bases: np.ndarray, threads: Optional[int] = None) -> np.ndarray:
    n = scalars.shape[0]
    if bases.shape[0] != n:  # arithmetic.rs:144 assert_eq!
        raise AssertionError("best_multiexp: coeffs.len() != bases.len()")
    out = np.zeros(64, dtype=np.uint8)
    lib().orc_best_multiexp(CURVE_ID[curve], _p(np.ascontiguousarray(scalars)), _p(np.ascontiguousarray(bases)),
                            ctypes.c_size_t(n), threads or default_threads(), _p(out))
    return out


def naive_msm(curve: str, scalars: np.ndarray, bases: np.ndarray) -> np.ndarray:
    out = np.zeros(64, dtype=np.uint8)
    lib().orc_naive_msm(CURVE_ID[curve], _p(np.ascontiguousarray(scalars)), _p(np.ascontiguousarray(bases)),
                        ctypes.c_size_t(scalars.shape[0]), _p(out))
    return out


def best_fft(field: str, a: np.ndarray, omega, log_n: int, threads: Optional[int] = None) -> np.ndarray:
    if a.shape[0] != 1 << log_n:  # arithmetic.rs:205
        raise AssertionError("best_fft: a.len() != 1 << log_n")
    a = np.ascontiguousarray(a).copy()
    lib().orc_best_fft(FIELD_ID[field], _p(a), _p(_fe(omega)), ctypes.c_uint32(log_n), threads or default_threads())
    return a


def ifft(field: str, a: np.ndarray, omega_inv, log_n: int, divisor, threads: Optional[int] = None) -> np.ndarray:
    assert a.shape[0] == 1 << log_n
    a = np.ascontiguousarray(a).copy()
    lib().orc_ifft(FIELD_ID[field], _p(a), _p(_fe(omega_inv)), ctypes.c_uint32(log_n), _p(_fe(divisor)),
                   threads or default_threads())
    return a


def coeff_to_extended(field: str, a: np.ndarray, k: int, ext_k: int, zeta, ext_omega,
                      threads: Optional[int] = None) -> np.ndarray:
    assert a.shape[0] == 1 << k
    out = np.zeros((1 << ext_k, 32), dtype=np.uint8)
    lib().orc_coeff_to_extended(FIELD_ID[field], _p(np.ascontiguousarray(a)), ctypes.c_uint32(k),
                                ctypes.c_uint32(ext_k), _p(_fe(zeta)), _p(_fe(ext_omega)), _p(out),
                                threads or default_threads())
    return out


def extended_to_coeff(field: str, a: np.ndarray, ext_k: int, ext_omega_inv, ext_divisor, zeta, out_len: int,
                      threads: Optional[int] = None) -> np.ndarray:
    assert a.shape[0] == 1 << ext_k
    out = np.zeros((out_len, 32), dtype=np.uint8)
    lib().orc_extended_to_coeff(FIELD_ID[field], _p(np.ascontiguousarray(a)), ctypes.c_uint32(ext_k),
                                _p(_fe(ext_omega_inv)), _p(_fe(ext_divisor)), _p(_fe(zeta)),
                                ctypes.c_size_t(out_len), _p(out), threads or default_threads())
    return out


def ec_fft(curve: str, points_xyz: np.ndarray, omega, log_n: int, scale=None, threads: Optional[int] = None) -> np.ndarray:
    """best_fft with G = curve point (arithmetic.rs:192-295; call site poly/commitment.rs:81-82) on (n, 96) canonical
    Jacobian points, then `*g *= scale` (:84-89) when scale is given.  Returns a new array."""
    if points_xyz.shape[0] != 1 << log_n:  # arithmetic.rs:205
        raise AssertionError("best_fft: a.len() != 1 << log_n")
    a = np.ascontiguousarray(points_xyz, dtype=np.uint8).copy()
    lib().orc_ec_fft(CURVE_ID[curve], _p(a), _p(_fe(omega)), ctypes.c_uint32(log_n), _p(_fe(scale)) if scale is not None else None,
                     threads or default_threads())
    return a


def batch_normalize(curve: str, points_xyz: np.ndarray) -> np.ndarray:
    """group::Curve::batch_normalize: (n, 96) canonical Jacobian -> (n, 64) affine, identity = zeros."""
    a = np.ascontiguousarray(points_xyz, dtype=np.uint8).reshape(-1, 96)
    out = np.zeros((a.shape[0], 64), dtype=np.uint8)
    lib().orc_batch_normalize(CURVE_ID[curve], _p(a), ctypes.c_size_t(a.shape[0]), _p(out))
    return out


def params_lagrange(curve: str, g_xy: np.ndarray, k: int, omega_inv, minv, threads: Optional[int] = None) -> np.ndarray:
    """poly/commitment.rs:74-101: g -> g_lagrange (EC-iFFT, * 2^-k, batch_normalize)."""
    g = np.ascontiguousarray(g_xy, dtype=np.uint8)
    assert g.shape == (1 << k, 64)
    out = np.zeros((1 << k, 64), dtype=np.uint8)
    lib().orc_params_lagrange(CURVE_ID[curve], _p(g), ctypes.c_uint32(k), _p(_fe(omega_inv)), _p(_fe(minv)),
                              threads or default_threads(), _p(out))
    return out


def affine_to_jacobian_bytes(xy: np.ndarray) -> np.ndarray:
    """(n, 64) affine -> (n, 96) Jacobian with z = 1 (identity: z = 0, y = 1 like pasta's Ep::identity)."""
    a = np.ascontiguousarray(xy, dtype=np.uint8).reshape(-1, 64)
    out = np.zeros((a.shape[0], 96), dtype=np.uint8)
    out[:, :64] = a
    ident = ~a.any(axis=1)
    out[~ident, 64] = 1
    out[ident, 32] = 1
    return out


def eval_polynomial(field: str, poly: np.ndarray, point) -> int:
    """arithmetic.rs:297-303 (serial Horner, as the reference runs it)."""
    p = np.ascontiguousarray(poly, dtype=np.uint8).reshape(-1, 32)
    out = np.zeros(32, dtype=np.uint8)
    lib().orc_eval_polynomial(FIELD_ID[field], _p(p), ctypes.c_size_t(p.shape[0]), _p(_fe(point)), _p(out))
    return int.from_bytes(out.tobytes(), "little")


def compute_s(field: str, u, init) -> np.ndarray:
    """poly/commitment/verifier.rs:156-171 (the serial doubling loop); u: the k round challenges as ints."""
    ub = ints_to_bytes(list(u))
    out = np.zeros((1 << len(u), 32), dtype=np.uint8)
    if lib().orc_compute_s(FIELD_ID[field], _p(ub), len(u), _p(_fe(int(init))), _p(out)) != 0:
        raise AssertionError("compute_s: !u.is_empty()")
    return out


def kate_division(field: str, a: np.ndarray, b) -> np.ndarray:
    """arithmetic.rs:322-341 (serial)."""
    p = np.ascontiguousarray(a, dtype=np.uint8).reshape(-1, 32)
    out = np.zeros((max(p.shape[0] - 1, 0), 32), dtype=np.uint8)
    lib().orc_kate_division(FIELD_ID[field], _p(p), ctypes.c_size_t(p.shape[0]), _p(_fe(b)), _p(out))
    return out


def permutation_product(field: str, columns: np.ndarray, sigmas: np.ndarray, chunk_len: int, beta, gamma, omega, delta, blinding: np.ndarray,
                        bf: int) -> np.ndarray:
    """plonk/permutation/prover.rs:81-168 for every proof: columns (proofs, cols, n, 32), sigmas (cols, n, 32), blinding
    (proofs x sets x bf, 32) in the rng's order.  Returns z (proofs, sets, n, 32)."""
    c = np.ascontiguousarray(columns, dtype=np.uint8)
    s = np.ascontiguousarray(sigmas, dtype=np.uint8)
    proofs, cols, n = c.shape[0], c.shape[1], c.shape[2]
    assert s.shape == (cols, n, 32) and n & (n - 1) == 0
    sets = -(-cols // chunk_len)
    bl = np.ascontiguousarray(blinding, dtype=np.uint8).reshape(-1, 32)
    assert bl.shape[0] == proofs * sets * bf
    out = np.zeros((proofs, sets, n, 32), dtype=np.uint8)
    rc = lib().orc_permutation_product(FIELD_ID[field], _p(c), _p(s), ctypes.c_size_t(proofs), ctypes.c_size_t(cols), ctypes.c_size_t(chunk_len),
                                       ctypes.c_uint32(n.bit_length() - 1), _p(_fe(beta)), _p(_fe(gamma)), _p(_fe(omega)), _p(_fe(delta)),
                                       _p(bl) if bf else None, ctypes.c_uint32(bf), _p(out))
    assert rc == 0
    return out


def lookup_product(field: str, a: np.ndarray, s: np.ndarray, a_perm: np.ndarray, s_perm: np.ndarray, beta, gamma, blinding: np.ndarray,
                   bf: int) -> np.ndarray:
    """plonk/lookup/prover.rs:279-321 for one lookup: (n, 32) compressed input / table and permuted columns, bf blinding values."""
    cols = [np.ascontiguousarray(x, dtype=np.uint8).reshape(-1, 32) for x in (a, s, a_perm, s_perm)]
    n = cols[0].shape[0]
    assert all(x.shape[0] == n for x in cols) and n & (n - 1) == 0
    bl = np.ascontiguousarray(blinding, dtype=np.uint8).reshape(-1, 32)
    assert bl.shape[0] == bf
    out = np.zeros((n, 32), dtype=np.uint8)
    rc = lib().orc_lookup_product(FIELD_ID[field], *(_p(x) for x in cols), ctypes.c_uint32(n.bit_length() - 1), _p(_fe(beta)), _p(_fe(gamma)),
                                  _p(bl) if bf else None, ctypes.c_uint32(bf), _p(out))
    assert rc == 0
    return out


def divide_by_vanishing_poly(field: str, a: np.ndarray, t_evaluations) -> np.ndarray:
    """poly/domain.rs:329-348: a[i] * t_evaluations[i % len(t_evaluations)].  Returns a new array."""
    out = np.ascontiguousarray(a, dtype=np.uint8).reshape(-1, 32).copy()
    t = ints_to_bytes(t_evaluations)
    assert lib().orc_divide_by_vanishing_poly(FIELD_ID[field], _p(out), ctypes.c_size_t(out.shape[0]), _p(t), ctypes.c_size_t(t.shape[0])) == 0
    return out


def permute_expression_pair(input_expression: np.ndarray, table_expression: np.ndarray, usable_rows: int):
    """plonk/lookup/prover.rs:563-647 over the usable rows (canonical bytes); None where the reference fails (:605-608)."""
    a = np.ascontiguousarray(input_expression, dtype=np.uint8).reshape(-1, 32)
    t = np.ascontiguousarray(table_expression, dtype=np.uint8).reshape(-1, 32)
    u = int(usable_rows)
    oa, ot = np.zeros((u, 32), dtype=np.uint8), np.zeros((u, 32), dtype=np.uint8)
    rc = lib().orc_permute_expression_pair(_p(a), _p(t), ctypes.c_size_t(u), _p(oa), _p(ot))
    return None if rc else (oa, ot)


def ast_eval(field: str, polys: np.ndarray, log_n: int, code: np.ndarray, consts, omega, lin_base, threads: Optional[int] = None) -> np.ndarray:
    """Evaluator::evaluate (poly/evaluator.rs:129-228) from the postfix form of the Ast (see orc_ast_eval); polys (n_polys, 2^log_n, 32)."""
    p = np.ascontiguousarray(polys, dtype=np.uint8).reshape(-1, 1 << log_n, 32)
    c = np.ascontiguousarray(code, dtype=np.uint32).reshape(-1, 4)
    cs = ints_to_bytes(consts) if len(consts) else np.zeros((1, 32), dtype=np.uint8)
    out = np.zeros((1 << log_n, 32), dtype=np.uint8)
    lib().orc_ast_eval(FIELD_ID[field], _p(p), ctypes.c_uint32(p.shape[0]), ctypes.c_uint32(log_n), c.ctypes.data_as(ctypes.c_void_p),
                       ctypes.c_uint32(c.shape[0]), _p(cs), ctypes.c_uint32(len(consts)), _p(_fe(omega)), _p(_fe(lin_base)),
                       threads or default_threads(), _p(out))
    return out


def field_op(field: str, op: str, a, b=None) -> int:
    ops = {"add": 0, "sub": 1, "mul": 2, "inv": 3, "pow5": 4, "neg": 5}
    out = np.zeros(32, dtype=np.uint8)
    lib().orc_field_op(FIELD_ID[field], ops[op], _p(_fe(a)), _p(_fe(b)) if b is not None else None, _p(out))
    return int.from_bytes(out.tobytes(), "little")


def scalar_mul(curve: str, scalar, base: np.ndarray) -> np.ndarray:
    out = np.zeros(64, dtype=np.uint8)
    lib().orc_scalar_mul(CURVE_ID[curve], _p(_fe(scalar)), _p(np.ascontiguousarray(base)), _p(out))
    return out


def point_add(curve: str, a: np.ndarray, b: np.ndarray) -> np.ndarray:
    out = np.zeros(64, dtype=np.uint8)
    lib().orc_point_add(CURVE_ID[curve], _p(np.ascontiguousarray(a)), _p(np.ascontiguousarray(b)), _p(out))
    return out


def jac_to_affine(curve: str, xyz: np.ndarray) -> np.ndarray:
    out = np.zeros(64, dtype=np.uint8)
    lib().orc_jac_to_affine(CURVE_ID[curve], _p(np.ascontiguousarray(xyz, dtype=np.uint8).reshape(-1)), _p(out))
    return out


def on_curve(curve: str, xy: np.ndarray) -> bool:
    return bool(lib().orc_on_curve(CURVE_ID[curve], _p(np.ascontiguousarray(xy))))


def gen_scalars(field: str, seed: int, n: int) -> np.ndarray:
    out = np.zeros((n, 32), dtype=np.uint8)
    lib().orc_gen_scalars(FIELD_ID[field], ctypes.c_uint64(seed), ctypes.c_size_t(n), _p(out))
    return out


def gen_points(curve: str, seed: int, n: int) -> np.ndarray:
    out = np.zeros((n, 64), dtype=np.uint8)
    lib().orc_gen_points(CURVE_ID[curve], ctypes.c_uint64(seed), ctypes.c_size_t(n), _p(out))
    return out


# conversions between python ints / pasta.py affine tuples and byte arrays ---------------
def ints_to_bytes(xs) -> np.ndarray:
    return np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in xs), dtype=np.uint8).reshape(-1, 32).copy()


def bytes_to_ints(a: np.ndarray):
    a = np.ascontiguousarray(a, dtype=np.uint8).reshape(-1, 32)
    return [int.from_bytes(row.tobytes(), "little") for row in a]


def affines_to_bytes(pts) -> np.ndarray:
    out = np.zeros((len(pts), 64), dtype=np.uint8)
    for i, pt in enumerate(pts):
        if pt is not None:
            out[i, :32] = np.frombuffer(int(pt[0]).to_bytes(32, "little"), dtype=np.uint8)
            out[i, 32:] = np.frombuffer(int(pt[1]).to_bytes(32, "little"), dtype=np.uint8)
    return out


def bytes_to_affine(a: np.ndarray):
    b = np.ascontiguousarray(a, dtype=np.uint8).reshape(64).tobytes()
    x = int.from_bytes(b[:32], "little")
    y = int.from_bytes(b[32:], "little")
    return None if (x == 0 and y == 0) else (x, y)


def ipa_rounds(curve: str, bases: np.ndarray, k: int, p_prime: np.ndarray, x3, z, challenges: np.ndarray, l_rand: np.ndarray,
               r_rand: np.ndarray, threads: Optional[int] = None):
    """poly/commitment/prover.rs:100-142 (see orc_ipa_rounds).  bases = g || w || u.  Returns (L (k,64), R (k,64), c int)."""
    out_l = np.zeros((k, 64), dtype=np.uint8)
    out_r = np.zeros((k, 64), dtype=np.uint8)
    out_c = np.zeros(32, dtype=np.uint8)
    lib().orc_ipa_rounds(CURVE_ID[curve], _p(np.ascontiguousarray(bases)), ctypes.c_uint32(k), _p(np.ascontiguousarray(p_prime)),
                         _p(_fe(x3)), _p(_fe(z)), _p(np.ascontiguousarray(challenges)), _p(np.ascontiguousarray(l_rand)),
                         _p(np.ascontiguousarray(r_rand)), threads or default_threads(), _p(out_l), _p(out_r), _p(out_c))
    return out_l, out_r, int.from_bytes(out_c.tobytes(), "little")


def ipa_rounds_transcript(curve: str, bases: np.ndarray, k: int, p_prime: np.ndarray, x3, z, challenge, l_rand: np.ndarray,
                          r_rand: np.ndarray, threads: Optional[int] = None):
    """The same loop driven by a transcript: `challenge(j, l_xy (64,) uint8, r_xy (64,) uint8) -> int u_j` is called once per
    round, where the reference writes L_j, R_j and squeezes u_j (prover.rs:124-128).  Returns (L, R, c)."""
    out_l = np.zeros((k, 64), dtype=np.uint8)
    out_r = np.zeros((k, 64), dtype=np.uint8)
    out_c = np.zeros(32, dtype=np.uint8)
    CB = ctypes.CFUNCTYPE(None, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint8),
                          ctypes.c_void_p)

    def _cb(j, l_ptr, r_ptr, u_ptr, _ctx):
        u = int(challenge(int(j), np.ctypeslib.as_array(l_ptr, (64,)).copy(), np.ctypeslib.as_array(r_ptr, (64,)).copy()))
        ctypes.memmove(u_ptr, u.to_bytes(32, "little"), 32)

    cb = CB(_cb)
    lib().orc_ipa_rounds_cb(CURVE_ID[curve], _p(np.ascontiguousarray(bases)), ctypes.c_uint32(k), _p(np.ascontiguousarray(p_prime)),
                            _p(_fe(x3)), _p(_fe(z)), cb, None, _p(np.ascontiguousarray(l_rand)), _p(np.ascontiguousarray(r_rand)),
                            threads or default_threads(), _p(out_l), _p(out_r), _p(out_c))
    return out_l, out_r, int.from_bytes(out_c.tobytes(), "little")
