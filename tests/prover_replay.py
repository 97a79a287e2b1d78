"""A proof-shaped replay of plonk::create_proof's hot path with a REAL transcript (test / bench infrastructure).

The Rust prover cannot run here (no toolchain), so this drives the same sequence of hot-path calls the prover makes for the
`benches/plonk.rs` circuit (3 advice columns, one permutation product, degree 5 => extended_k = k + 2; SURVEY.md Appendix C)
-- in order, with the real data dependencies -- through two interchangeable arms:
  * GpuArm: the engine's reference-facing API on device-resident polynomials (halo2_b200);
  * CpuArm: the C restatement of the reference algorithm (oracle/halo2_oracle.c), i.e. the timed CPU baseline.
Both arms feed ONE implementation of the reference's transcript, Blake2bWrite with Challenge255
(/root/reference/halo2_proofs/src/transcript.rs:160-219, :289-318): every commitment is written as the reference writes
it (prefix 1 || x || y into the hash, the 32-byte compressed point into the proof), every evaluation as a scalar (prefix 2),
and every challenge is squeezed from the running BLAKE2b state (prefix 0, 64-byte digest reduced as from_uniform_bytes).
The challenges flow back into the computation (theta/beta/gamma into the permutation product, y into h(X), x into the
evaluations, x_1..x_4 into the multiopen combination, xi / z / u_j into the inner product argument,
poly/commitment/prover.rs:36-145), so two arms produce the same proof bytes iff every commitment, evaluation and opening
round they compute is bit-identical.  What is replayed is the CALL SCHEDULE on synthetic columns: the circuit's own
gate expressions and witness are stand-ins of the same shape and size (stated wherever a number from this file is quoted).

Order of operations (file:line in halo2_proofs/src):
  1. advice columns: commit_lagrange x3 (batched) -> write_point x3; lagrange_to_coeff x3; coeff_to_extended x3   plonk/prover.rs:305-328
  2. theta, beta, gamma; permutation product z: commit_lagrange, lagrange_to_coeff, coeff_to_extended                plonk/permutation/prover.rs:172-178
  3. vanishing random polynomial: commit                                                                             plonk/vanishing/prover.rs:36-60
  4. y; h(X) = Ast over the cosets, divide_by_vanishing_poly, extended_to_coeff, 4 pieces committed (batched)        plonk/vanishing/prover.rs:81-108
  5. x; evaluations of every polynomial at x (and the rotations) -> write_scalar                                     plonk/prover.rs:601-675
  6. multiopen: x_1, x_2, q polynomials, kate_division per point set, commit f; x_3; q evals; x_4; final p           poly/multiopen/prover.rs:29-124
  7. the opening: s_poly, commit, xi, z, p' = s xi + p, p'[0] -= p'(x_3), k rounds (L_j, R_j, u_j), c, f             poly/commitment/prover.rs:36-145
"""
from __future__ import annotations

import hashlib
import time
from typing import List, Sequence

import numpy as np

P_MOD = 0x40000000000000000000000000000000224698FC094CF91B992D30ED00000001   # Fp: the scalar field of Vesta (EqAffine)
CURVE, FIELD = "vesta", "fp"
DEGREE_J = 5   # benches/plonk.rs:183 set_minimum_degree(5) => quotient degree 4, extended_k = k + 2


class Blake2bTranscript:
    """transcript.rs:160-219 (Blake2bWrite) with Challenge255 (:289-318)."""

    def __init__(self, modulus: int = P_MOD):
        self.state = hashlib.blake2b(digest_size=64, person=b"Halo2-Transcript")
        self.proof = bytearray()
        self.modulus = modulus                                # of the curve's scalar field (the challenge space)

    def write_point(self, xy: np.ndarray) -> None:            # :183-187 write_point, :205-216 common_point
        b = bytes(np.ascontiguousarray(xy, dtype=np.uint8).reshape(64))
        if b == bytes(64):
            raise ValueError("cannot write points at infinity to the transcript")
        self.state.update(b"\x01" + b[:32] + b[32:])
        enc = bytearray(b[:32])
        enc[31] |= (b[32] & 1) << 7                            # C::to_bytes: x with the LSB of y in the top bit
        self.proof += enc

    def common_point(self, xy) -> None:                       # :205-216: into the hash only
        b = bytes(np.ascontiguousarray(xy, dtype=np.uint8).reshape(64))
        if b == bytes(64):
            raise ValueError("cannot write points at infinity to the transcript")
        self.state.update(b"\x01" + b)

    def common_scalar(self, s: int) -> None:                  # :218-223
        self.state.update(b"\x02" + int(s).to_bytes(32, "little"))

    def write_scalar(self, s: int) -> None:                   # :188-192, :218-223
        b = int(s).to_bytes(32, "little")
        self.state.update(b"\x02" + b)
        self.proof += b

    def squeeze_challenge(self) -> int:                       # :198-203; Challenge255::new = from_uniform_bytes of the 64-byte digest
        self.state.update(b"\x00")
        return int.from_bytes(self.state.copy().digest(), "little") % self.modulus


class _WriteT:
    """Blake2bTranscript on affine tuples (what the oracle speaks)."""

    def __init__(self, modulus):
        from oracle import cref
        self.T, self._bytes = Blake2bTranscript(modulus), lambda pt: cref.affines_to_bytes([pt])[0]

    def write_point(self, pt):
        self.T.write_point(self._bytes(pt))

    def write_scalar(self, s):
        self.T.write_scalar(s)

    def common_point(self, pt):
        self.T.common_point(self._bytes(pt))

    def common_scalar(self, s):
        self.T.common_scalar(s)

    def squeeze_challenge(self):
        return self.T.squeeze_challenge()


def _encode(points, m) -> bytes:
    """The proof bytes of `points` written to a fresh transcript."""
    T = Blake2bTranscript(m)
    for p in points:
        T.write_point(p)
    return bytes(T.proof)


class Blake2bRead:
    """transcript.rs:66-158 (Blake2bRead) with Challenge255: the verifier's view of the same transcript.  `decompress`:
    32 proof bytes -> (64,) uint8 affine x||y, raising on an invalid encoding (C::from_bytes, :91-100) -- the engine's
    h2_points_decompress in the GPU arm, the oracle's in the CPU arm."""

    def __init__(self, proof: bytes, decompress, modulus: int = P_MOD):
        self.state = hashlib.blake2b(digest_size=64, person=b"Halo2-Transcript")
        self.proof, self.pos, self.decompress, self.modulus = bytes(proof), 0, decompress, modulus

    def _take(self) -> bytes:
        if self.pos + 32 > len(self.proof):
            raise EOFError("proof too short")                 # read_exact fails, :93 / :104
        self.pos += 32
        return self.proof[self.pos - 32:self.pos]

    def read_point(self) -> np.ndarray:                       # :91-100, then common_point :130-141
        xy = np.ascontiguousarray(self.decompress(self._take()), dtype=np.uint8).reshape(64)
        if not xy.any():
            raise ValueError("cannot write points at infinity to the transcript")
        self.state.update(b"\x01" + bytes(xy[:32]) + bytes(xy[32:]))
        return xy

    def common_point(self, xy) -> None:                       # :128-141
        xy = np.ascontiguousarray(xy, dtype=np.uint8).reshape(64)
        if not xy.any():
            raise ValueError("cannot write points at infinity to the transcript")
        self.state.update(b"\x01" + bytes(xy[:32]) + bytes(xy[32:]))

    def common_scalar(self, s: int) -> None:                  # :143-148
        self.state.update(b"\x02" + int(s).to_bytes(32, "little"))

    def read_scalar(self) -> int:                             # :102-114, then common_scalar :143-148
        b = self._take()
        v = int.from_bytes(b, "little")
        if v >= self.modulus:
            raise ValueError("invalid field element encoding in proof")
        self.state.update(b"\x02" + b)
        return v

    def squeeze_challenge(self) -> int:                       # :121-128
        self.state.update(b"\x00")
        return int.from_bytes(self.state.copy().digest(), "little") % self.modulus


def _schedule_ast(kind, leaves, ch):
    """The elementwise programs of the replay (built from halo2_b200.evaluator.Ast, the mirror of poly/evaluator.rs)."""
    from halo2_b200.evaluator import Ast
    if kind == "perm_z":            # stand-in for the grand product's dependence on beta, gamma: z = base * beta + gamma
        return leaves[0] * ch["beta"] + Ast.constant_term(ch["gamma"])
    if kind == "h":                 # h(X)-shaped: two gates and a permutation-style product, folded by powers of y
        a, b, c, z = leaves
        gate0 = a * b - c
        gate1 = (a.with_rotation(1) - a) * (b.with_rotation(-1) + Ast.constant_term(7))
        perm = (z.with_rotation(1) + Ast.linear_term(ch["beta"]) + Ast.constant_term(ch["gamma"])) * (c + b * ch["theta"]) - z * a
        return Ast.distribute_powers([gate0, gate1, perm], ch["y"])
    if kind == "lincomb":           # sum_i coeff_i * poly_i
        acc = None
        for leaf, cf in zip(leaves, ch["coeffs"]):
            t = leaf * cf
            acc = t if acc is None else acc + t
        return acc
    raise ValueError(kind)


class GpuArm:
    name = "gpu"

    def __init__(self, h2, k, g, g_lagrange, w, u):
        self.h2, self.k, self.n = h2, k, 1 << k
        zeta = pow(5, (P_MOD - 1) // 3, P_MOD)
        self.params = h2.Params(CURVE, k, g, g_lagrange, w, u=u)
        self.dom = h2.EvaluationDomain(FIELD, DEGREE_J, k, zeta)
        self.ev_n = h2.Evaluator(self.dom, "lagrange")
        self.ev_ext = h2.Evaluator(self.dom, "extended")
        self._live: List = []

    def poly(self, values, length=None):
        arr = np.ascontiguousarray(values, dtype=np.uint8).reshape(-1, 32)
        p = self.h2.ResidentPoly(FIELD, length or arr.shape[0], arr)
        self._live.append(p)
        return p

    def empty(self, length):
        p = self.h2.ResidentPoly(FIELD, length)
        self._live.append(p)
        return p

    def commit(self, polys, blinds, lagrange):
        return self.params.commit_resident_affine(polys, [self.h2.Blind(b) for b in blinds], lagrange=lagrange)

    def l2c(self, p):
        return self.dom.lagrange_to_coeff_resident(p, out=self.empty(self.n))

    def c2e(self, p):
        return self.dom.coeff_to_extended_resident(p, out=self.empty(self.dom.extended_len()))

    def e2c(self, p):
        return self.dom.extended_to_coeff_resident(p, out=self.empty(self.n * self.dom.quotient_poly_degree))

    def vanish(self, p):
        return self.dom.divide_by_vanishing_poly_resident(p)

    def ast(self, kind, polys, ch, extended):
        ev = self.ev_ext if extended else self.ev_n
        ev.polys = []
        leaves = [ev.register_poly(p) for p in polys]
        return ev.evaluate(_schedule_ast(kind, leaves, ch), out=self.empty(self.dom.extended_len() if extended else self.n))

    def evals(self, polys, points):
        return self.h2.eval_polynomial_resident(polys, points, n=self.n)

    def kate(self, p, point):
        return self.h2.kate_division_resident([p], [point], dst=[self.empty(self.n)], n=self.n)[0]

    def pieces(self, p, count):
        return [self.empty(self.n).copy_from(p, self.n, src_off=i * self.n) for i in range(count)]

    def add_at(self, p, idx, delta):
        p.add_at(idx, delta)

    def ipa(self, p_prime, x3, z, challenge, l_rand, r_rand):
        return self.params.ipa_rounds_transcript(p_prime, x3, z, challenge, l_rand, r_rand)

    def sync(self):
        if self._live:
            self._live[-1].download(1)

    def free(self):
        for p in self._live:
            p.close()
        self._live = []

    def close(self):
        self.free()
        self.params.close()


class CpuArm:
    """The reference algorithm, C restatement, `threads` host threads: best_multiexp per commitment (poly/commitment.rs:119-150),
    best_fft-based transforms, serial eval_polynomial / kate_division (arithmetic.rs:297-341), the IPA loop with
    parallel_generator_collapse.  Only these hot-path calls are timed (`hot_s`); the elementwise glue is not."""
    name = "cpu"

    def __init__(self, cref, pasta, k, g, g_lagrange, w, u, threads):
        self.cref, self.k, self.n, self.threads = cref, k, 1 << k, threads
        zeta = pasta.zeta_candidates(FIELD)[0]
        assert zeta == pow(5, (P_MOD - 1) // 3, P_MOD)
        self.d = pasta.EvaluationDomain(FIELD, DEGREE_J, k, zeta)
        self.zeta = zeta
        self.bases = np.concatenate([g, w])
        self.bases_l = np.concatenate([g_lagrange, w])
        self.gwu = np.concatenate([g, w, u])
        self.hot_s = 0.0
        self.by_kind = {}
        self.ipa_threads = threads

    def _t(self, kind, t0):
        dt = time.time() - t0
        self.hot_s += dt
        self.by_kind[kind] = self.by_kind.get(kind, 0.0) + dt

    def poly(self, values, length=None):
        arr = np.ascontiguousarray(values, dtype=np.uint8).reshape(-1, 32)
        if length and length > arr.shape[0]:
            arr = np.concatenate([arr, np.zeros((length - arr.shape[0], 32), dtype=np.uint8)])
        return arr

    def commit(self, polys, blinds, lagrange):
        t0 = time.time()
        out = np.stack([self.cref.best_multiexp(CURVE, np.concatenate([p[:self.n], self.cref.ints_to_bytes([b])]),
                                                self.bases_l if lagrange else self.bases, self.threads) for p, b in zip(polys, blinds)])
        self._t("commit_lagrange" if lagrange else "commit", t0)
        return out

    def l2c(self, p):
        t0 = time.time()
        out = self.cref.ifft(FIELD, p, self.d.omega_inv, self.k, self.d.ifft_divisor, self.threads)
        self._t("lagrange_to_coeff", t0)
        return out

    def c2e(self, p):
        t0 = time.time()
        out = self.cref.coeff_to_extended(FIELD, p, self.k, self.d.extended_k, self.zeta, self.d.extended_omega, self.threads)
        self._t("coeff_to_extended", t0)
        return out

    def e2c(self, p):
        t0 = time.time()
        out = self.cref.extended_to_coeff(FIELD, p, self.d.extended_k, self.d.extended_omega_inv, self.d.extended_ifft_divisor, self.zeta,
                                          self.n * (DEGREE_J - 1), self.threads)
        self._t("extended_to_coeff", t0)
        return out

    def vanish(self, p):
        tev = self.cref.ints_to_bytes(self.d.t_evaluations)
        tfull = tev[np.arange(1 << self.d.extended_k) % len(self.d.t_evaluations)]
        return self.cref.ast_eval(FIELD, np.stack([p, tfull]), self.d.extended_k,
                                  np.array([[0, 0, 0, 0], [0, 1, 0, 0], [4, 0, 0, 0]], dtype=np.uint32), [], self.d.extended_omega, self.zeta, self.threads)

    def ast(self, kind, polys, ch, extended):
        from halo2_b200.evaluator import AstLeaf, compile_ast      # the pure-host flattener of the Ast (no GPU involved)
        log_n = self.d.extended_k if extended else self.k
        stride = 1 << (self.d.extended_k - self.k) if extended else 1
        code, consts = compile_ast(_schedule_ast(kind, [AstLeaf(i) for i in range(len(polys))], ch), P_MOD, stride)
        omega = self.d.extended_omega if extended else self.d.omega
        return self.cref.ast_eval(FIELD, np.stack([p[:1 << log_n] for p in polys]), log_n, code, consts, omega, self.zeta if extended else 1, self.threads)

    def evals(self, polys, points):
        t0 = time.time()
        out = [self.cref.eval_polynomial(FIELD, p[:self.n], x) for p, x in zip(polys, points)]
        self._t("eval_polynomial", t0)
        return out

    def kate(self, p, point):
        t0 = time.time()
        q = self.cref.kate_division(FIELD, p[:self.n], point)
        self._t("kate_division", t0)
        return np.concatenate([q, np.zeros((1, 32), dtype=np.uint8)])       # multiopen/prover.rs: poly.push(ZERO)

    def pieces(self, p, count):
        return [p[i * self.n:(i + 1) * self.n] for i in range(count)]

    def add_at(self, p, idx, delta):
        v = (int.from_bytes(p[idx].tobytes(), "little") + delta) % P_MOD
        p[idx] = np.frombuffer(v.to_bytes(32, "little"), dtype=np.uint8)

    def ipa(self, p_prime, x3, z, challenge, l_rand, r_rand):
        t0 = time.time()
        out = self.cref.ipa_rounds_transcript(CURVE, self.gwu, self.k, p_prime[:self.n], x3, z, challenge, self.cref.ints_to_bytes(l_rand),
                                              self.cref.ints_to_bytes(r_rand), self.ipa_threads)
        self._t("ipa", t0)
        return out

    def sync(self):
        pass

    def free(self):
        pass

    def close(self):
        pass


def replay_inputs(cref, k, seed):
    """Synthetic witness of the replay: three advice columns and the base of the permutation product (Lagrange values), the
    vanishing argument's random polynomial and the opening's s_poly (coefficients), every blind and the per-round randomness
    -- all from the seeded generator of SURVEY.md section 8(d)."""
    n = 1 << k
    cols = [cref.gen_scalars(FIELD, seed + 10 + i, n) for i in range(3)]
    zbase = cref.gen_scalars(FIELD, seed + 20, n)
    rand_poly = cref.gen_scalars(FIELD, seed + 21, n)
    s_poly = cref.gen_scalars(FIELD, seed + 22, n)
    blinds = cref.bytes_to_ints(cref.gen_scalars(FIELD, seed + 23, 16))
    l_rand = cref.bytes_to_ints(cref.gen_scalars(FIELD, seed + 24, k))
    r_rand = cref.bytes_to_ints(cref.gen_scalars(FIELD, seed + 25, k))
    return {"cols": cols, "zbase": zbase, "rand_poly": rand_poly, "s_poly": s_poly, "blinds": blinds, "l_rand": l_rand, "r_rand": r_rand}


def run(arm, inp, k, omega):
    """One proof-shaped pass; returns the proof bytes.  `omega`: the 2^k-th root of unity of the domain."""
    T = Blake2bTranscript()
    n = 1 << k
    bl = list(inp["blinds"])
    m = P_MOD
    # 1. advice columns
    adv_l = [arm.poly(c) for c in inp["cols"]]
    for pt in arm.commit(adv_l, bl[0:3], lagrange=True):
        T.write_point(pt)
    adv = [arm.l2c(p) for p in adv_l]
    adv_e = [arm.c2e(p) for p in adv]
    # 2. permutation product
    ch = {"theta": T.squeeze_challenge(), "beta": T.squeeze_challenge(), "gamma": T.squeeze_challenge()}
    z_l = arm.ast("perm_z", [arm.poly(inp["zbase"])], ch, extended=False)
    T.write_point(arm.commit([z_l], bl[3:4], lagrange=True)[0])
    z = arm.l2c(z_l)
    z_e = arm.c2e(z)
    # 3. vanishing argument: random polynomial
    rnd = arm.poly(inp["rand_poly"])
    T.write_point(arm.commit([rnd], bl[4:5], lagrange=False)[0])
    # 4. h(X)
    ch["y"] = T.squeeze_challenge()
    h_e = arm.vanish(arm.ast("h", adv_e + [z_e], ch, extended=True))
    h = arm.e2c(h_e)
    hp = arm.pieces(h, DEGREE_J - 1)
    for pt in arm.commit(hp, bl[5:9], lagrange=False):
        T.write_point(pt)
    # 5. evaluations at x (advice at x and x*omega, z at x, x*omega, x*omega^-1... : 3 + 3 + 3 + 4 + 1 = 14 serial Horner loops)
    x = T.squeeze_challenge()
    xw, xwi = x * omega % m, x * pow(omega, -1, m) % m
    ev_polys = adv + adv + [z, z, z] + hp + [rnd]
    ev_points = [x] * 3 + [xw] * 3 + [x, xw, xwi] + [x] * 4 + [x]
    evals = arm.evals(ev_polys, ev_points)
    for e in evals:
        T.write_scalar(e)
    # 6. multiopen (poly/multiopen/prover.rs:38-123): two point sets {x}: advice, h pieces, random poly;  {x omega}: advice, z
    x1 = T.squeeze_challenge()
    x2 = T.squeeze_challenge()
    set0, b0 = adv + hp + [rnd], bl[0:3] + bl[5:9] + [bl[4]]
    set1, b1 = adv + [z], bl[0:3] + [bl[3]]
    # q_i = Horner in x_1 over the set's polynomials, first polynomial first (:53-63); the blinds fold the same way (:60-61)
    c0 = {"coeffs": [pow(x1, len(set0) - 1 - i, m) for i in range(len(set0))]}
    c1 = {"coeffs": [pow(x1, len(set1) - 1 - i, m) for i in range(len(set1))]}
    q0 = arm.ast("lincomb", set0, c0, extended=False)
    q1 = arm.ast("lincomb", set1, c1, extended=False)
    qb0 = sum(cf * b for cf, b in zip(c0["coeffs"], b0)) % m
    qb1 = sum(cf * b for cf, b in zip(c1["coeffs"], b1)) % m
    k0, k1 = arm.kate(q0, x), arm.kate(q1, xw)               # :78-84: kate_division drops the remainder q_i(point)
    f = arm.ast("lincomb", [k0, k1], {"coeffs": [x2, 1]}, extended=False)      # :91-95  q' = q'_0 * x_2 + q'_1
    T.write_point(arm.commit([f], bl[9:10], lagrange=False)[0])                # :99-102
    x3 = T.squeeze_challenge()
    for e in arm.evals([q0, q1], [x3, x3]):                  # :108-110
        T.write_scalar(e)
    x4 = T.squeeze_challenge()
    p = arm.ast("lincomb", [f, q0, q1], {"coeffs": [x4 * x4 % m, x4, 1]}, extended=False)   # :114-122  ((q' x_4) + q_0) x_4 + q_1
    p_blind = (bl[9] * x4 % m * x4 + qb0 * x4 + qb1) % m
    # 7. the opening, poly/commitment/prover.rs:36-145
    s = arm.poly(inp["s_poly"])
    s_at = arm.evals([s], [x3])[0]
    arm.add_at(s, 0, -s_at)                                  # :51
    s_blind = bl[12]
    T.write_point(arm.commit([s], [s_blind], lagrange=False)[0])
    xi = T.squeeze_challenge()
    zc = T.squeeze_challenge()
    pp = arm.ast("lincomb", [s, p], {"coeffs": [xi, 1]}, extended=False)      # :76
    v = arm.evals([pp], [x3])[0]
    arm.add_at(pp, 0, -v)                                    # :78
    fsyn = (s_blind * xi + p_blind) % m                      # :79

    us = []

    def challenge(j, l_xy, r_xy):                            # :124-128
        T.write_point(l_xy)
        T.write_point(r_xy)
        us.append(T.squeeze_challenge())
        return us[-1]

    ls, rs, c = arm.ipa(pp, x3, zc, challenge, inp["l_rand"], inp["r_rand"])
    for j, u in enumerate(us):                               # :143-144
        fsyn = (fsyn + inp["l_rand"][j] * pow(u, -1, m) + inp["r_rand"][j] * u) % m
    T.write_scalar(c)                                        # :150
    T.write_scalar(fsyn)                                     # :151
    arm.sync()
    return bytes(T.proof)


# ------------------------------------------------------------------------------------------------------------------------
# The verifier's side: the proof bytes of run() checked the way plonk::verify_proof's tail does it -- multiopen::verify_proof
# (poly/multiopen/verifier.rs:29-140) building the MSM of the commitment being opened from the proof's own commitments and
# evaluations, commitment::verify_proof (poly/commitment/verifier.rs:67-141) reading the opening, and the final
# `guard.use_challenges().eval()` of SingleVerifier (plonk/verifier.rs:53-62): ONE multiexp over all 2^k generators.  Two
# interchangeable arms again; what is NOT checked is the vanishing argument's identity (plonk/verifier.rs:294-357): the
# replay's gate expressions are stand-ins that do not vanish on the domain.
# ------------------------------------------------------------------------------------------------------------------------
class GpuVerifierArm:
    """halo2_b200.verifier: g_scalars resident, compute_s / scale / add on the device, eval over the resident generator table."""
    name = "gpu"

    def __init__(self, h2, k, g, g_lagrange, w, u, params=None):
        self.h2, self.k = h2, k
        self._own = params is None
        self.params = params if params is not None else h2.Params(CURVE, k, g, g_lagrange, w, u=u)

    def prepare(self, proof: bytes, point_offsets) -> None:
        """All of the proof's points through ONE h2_points_decompress call (the layout of a proof is known before it is read);
        if any encoding is invalid the batch fails and read_point meets the bad one on its own."""
        self._pts = {}
        enc = [proof[o:o + 32] for o in point_offsets if o + 32 <= len(proof)]
        if not enc:
            return
        try:
            xy = self.h2.decompress_points(np.frombuffer(b"".join(enc), dtype=np.uint8).reshape(-1, 32), CURVE)
        except self.h2.H2Error:
            return
        self._pts = {e: xy[i] for i, e in enumerate(enc)}

    def decompress(self, b32: bytes) -> np.ndarray:
        hit = getattr(self, "_pts", {}).get(b32)
        if hit is not None:
            return hit
        return self.h2.decompress_points(np.frombuffer(b32, dtype=np.uint8).reshape(1, 32), CURVE)[0]

    def msm(self):
        return self.h2.MSM(self.params)

    def append(self, msm, scalar, xy):
        msm.append_term(scalar, xy)

    def ipa_verify(self, msm, T, x, v):
        return self.h2.verify_proof(self.params, msm, T, x, v)

    def finish(self, guard) -> bool:                          # plonk/verifier.rs:57-58
        msm = guard.use_challenges()
        try:
            return msm.eval()
        finally:
            msm.close()

    def close(self):
        if self._own:
            self.params.close()


class _TupleTranscript:
    """The oracle speaks affine tuples; the transcripts of this file speak (64,) uint8 arrays."""

    def __init__(self, T, cref):
        self.T, self.cref = T, cref

    def read_point(self):
        return self.cref.bytes_to_affine(self.T.read_point())

    def read_scalar(self):
        return self.T.read_scalar()

    def squeeze_challenge(self):
        return self.T.squeeze_challenge()


class CpuVerifierArm:
    """oracle/pasta.py's restatement of MSM / verify_proof / Guard; the two hot calls -- compute_s (verifier.rs:156-171) and
    the final best_multiexp (msm.rs:175) -- run through the C restatement and are the only ones timed (`hot_s`)."""
    name = "cpu"

    def __init__(self, cref, pasta, k, g, g_lagrange, w, u, threads):
        self.cref, self.pasta, self.k, self.threads = cref, pasta, k, threads
        self.c = pasta.CURVES[CURVE]
        self.g_bytes = np.ascontiguousarray(g, dtype=np.uint8).reshape(-1, 64)
        self.w_xy, self.u_xy = cref.bytes_to_affine(np.asarray(w).reshape(64)), cref.bytes_to_affine(np.asarray(u).reshape(64))
        self.hot_s = 0.0

    def decompress(self, b32: bytes) -> np.ndarray:
        return self.cref.affines_to_bytes([self.pasta.decompress(self.c, b32)])[0]

    def msm(self):
        return self.pasta.MSM(self.c, [None] * (1 << self.k), self.w_xy, self.u_xy)    # the generators stay in self.g_bytes

    def append(self, msm, scalar, xy):
        msm.append_term(scalar, self.cref.bytes_to_affine(np.asarray(xy).reshape(64)))

    def ipa_verify(self, msm, T, x, v):
        return self.pasta.ipa_verify_proof(self.k, msm, _TupleTranscript(T, self.cref), x, v)

    def finish(self, guard) -> bool:
        cref, msm = self.cref, guard.msm
        t0 = time.time()
        s = cref.compute_s(FIELD, guard.u, guard.neg_c)                       # Guard::use_challenges, verifier.rs:36
        self.hot_s += time.time() - t0
        if msm.g_scalars is not None:                                         # add_to_g_scalars, msm.rs:99-109 (glue: a handful of non-zeros)
            for i, gv in enumerate(msm.g_scalars):
                if gv:
                    cur = int.from_bytes(s[i].tobytes(), "little")
                    s[i] = np.frombuffer(((cur + gv) % P_MOD).to_bytes(32, "little"), dtype=np.uint8)
        msm.g_scalars = None
        sc, bs = msm.terms()                                                  # other, w, u in the reference's order (msm.rs:150-166)
        scalars = np.concatenate([cref.ints_to_bytes(sc), s])
        bases = np.concatenate([cref.affines_to_bytes(bs), self.g_bytes])
        t0 = time.time()
        res = cref.best_multiexp(CURVE, scalars, bases, self.threads)          # msm.rs:175
        self.hot_s += time.time() - t0
        return not res.any()

    def close(self):
        pass


def verify(arm, proof: bytes, k: int, omega: int) -> bool:
    """Reads the proof run() wrote and checks its openings; returns msm.eval() of the final MSM (False also on a proof that
    cannot be parsed: Error::OpeningError / SamplingError / an invalid encoding)."""
    m = P_MOD
    if hasattr(arm, "prepare"):
        npt = 5 + DEGREE_J - 1                                                # 3 advice, z, the random polynomial, the h pieces
        arm.prepare(proof, [32 * i for i in range(npt)] + [32 * (npt + 14)] + [32 * (npt + 17 + i) for i in range(1 + 2 * k)])
    T = Blake2bRead(proof, arm.decompress)
    try:
        adv_c = [T.read_point() for _ in range(3)]
        for _ in range(3):
            T.squeeze_challenge()                                             # theta, beta, gamma
        z_c = T.read_point()
        rnd_c = T.read_point()
        T.squeeze_challenge()                                                 # y
        h_c = [T.read_point() for _ in range(DEGREE_J - 1)]
        x = T.squeeze_challenge()
        ev = [T.read_scalar() for _ in range(14)]
        xw = x * omega % m
        # multiopen::verify_proof, poly/multiopen/verifier.rs:29-140, for the replay's two single-point sets
        x1 = T.squeeze_challenge()
        x2 = T.squeeze_challenge()
        sets = [(x, adv_c + h_c + [rnd_c], ev[0:3] + ev[9:13] + [ev[13]]),     # commitments and their evaluations at the set's point
                (xw, adv_c + [z_c], ev[3:6] + [ev[7]])]
        q_commitments, q_evals = [], []
        for _, comms, evals in sets:                                          # :39-87: increasing powers of x_1 from the LAST commitment
            q, qe, power = arm.msm(), 0, 1
            for cm, e in zip(reversed(comms), reversed(evals)):
                arm.append(q, power, cm)
                qe = (qe + e * power) % m
                power = power * x1 % m
            q_commitments.append(q)
            q_evals.append(qe)
        f_c = T.read_point()                                                  # :90
        x3 = T.squeeze_challenge()
        u_ev = [T.read_scalar() for _ in sets]                                # :98-101
        msm_eval = 0
        for (point, _, _), r_eval, proof_eval in zip(sets, q_evals, u_ev):    # :105-119; one point: r(X) is the constant q_i(point)
            msm_eval = (msm_eval * x2 + (proof_eval - r_eval) * pow(x3 - point, -1, m)) % m
        x4 = T.squeeze_challenge()
        msm = arm.msm()
        arm.append(msm, 1, f_c)                                               # :126
        v = msm_eval
        for q, qe in zip(q_commitments, u_ev):                                # :127-134
            msm.scale(x4)
            msm.add_msm(q)
            v = (v * x4 + qe) % m
        guard = arm.ipa_verify(msm, T, x3, v)                                 # :137
    except Exception as e:                                                    # any parse / opening error: the proof is rejected
        if isinstance(e, AssertionError):
            raise
        return False
    finally:
        for q in locals().get("q_commitments", []):
            if hasattr(q, "close"):
                q.close()
    return arm.finish(guard)
