"""plonk::create_proof with the vanishing argument from halo2_b200.vanishing, for the vanishing tests: create_proof_engine's
own source with its vanishing lines (the random polynomial, h(X) and its pieces, the fold of h_poly, random_eval and the two
queries) replaced by vanishing_commit / construct / evaluate / open, and everything else unchanged.  Each replaced block must
occur exactly once, so a change to create_proof_engine that moves them fails here loudly instead of comparing something else.

record() runs either prover and returns what the comparison needs: the points and scalars written, the proof bytes, and the
last two queries (h_poly with h_blind, random_poly with random_blind) as bytes."""
from __future__ import annotations

import contextlib
import ctypes
import inspect

import numpy as np

from oracle import cref
from tests import fake_engine
from tests import plonk_prover as PP
from tests import prover_replay as R

_PATCHES = [
    ("""        random_poly = rng.poly(n)
        random_poly = random_poly if isinstance(random_poly, eng.ResidentPoly) else eng.ResidentPoly(field, n, random_poly)
        live.append(random_poly)
        random_blind = rng.scalar()
        transcript.write_point(commit([random_poly], [random_blind], False)[0])
""", """        vanishing, cm = eng.vanishing_commit(params, D, rng)
        live.append(vanishing.random_poly)
        transcript.write_point(cm)
"""),
    ("""        h_ext = ev_e.evaluate(Ast.distribute_powers(exprs, y), out=RP(None, L))
        D.divide_by_vanishing_poly_resident(h_ext)
        h = D.extended_to_coeff_resident(h_ext, out=RP(None, n * (cs_degree - 1)))
        h_pieces = [RP(None).copy_from(h, n, src_off=a * n) for a in range(cs_degree - 1)]
        h_blinds = [rng.scalar() for _ in h_pieces]
        for cm in commit(h_pieces, h_blinds, False):
            transcript.write_point(cm)
""", """        vanishing, cms = vanishing.construct(params, D, ev_e, exprs, y, rng)
        live.extend(vanishing.h_pieces)
        for cm in cms:
            transcript.write_point(cm)
"""),
    ("""        ev_list.append((random_poly, x))
""", """        random_at = len(ev_list)
"""),
    ("""        for e in eng.eval_polynomial_resident([p for p, _ in ev_list], [pt for _, pt in ev_list], n=n):
            transcript.write_scalar(e)
""", """        evals = eng.eval_polynomial_resident([p for p, _ in ev_list], [pt for _, pt in ev_list], n=n)
        vanishing, random_eval = vanishing.evaluate(D, x)
        live.append(vanishing.h_poly)
        evals.insert(random_at, random_eval)
        for e in evals:
            transcript.write_scalar(e)
"""),
    ("""        h_poly = RP(None).copy_from(h_pieces[-1], n)
        h_blind = h_blinds[-1]
        for piece, b in zip(reversed(h_pieces[:-1]), reversed(h_blinds[:-1])):
            eng.opening._scale_add(h_poly, xn, piece, 1, n)
            h_blind = (h_blind * xn + b) % m
""", ""),
    ("""        queries.append(Q(x, h_poly, Blind(h_blind)))
        queries.append(Q(x, random_poly, Blind(random_blind)))
""", """        queries += vanishing.open(x)
"""),
]


def _module_prover():
    src = inspect.getsource(PP.create_proof_engine)
    for old, new in _PATCHES:
        assert src.count(old) == 1, old
        src = src.replace(old, new)
    src = src.replace("def create_proof_engine(", "def create_proof_module(", 1)
    ns = dict(vars(PP))
    exec(compile(src, PP.__file__ + " (vanishing module)", "exec"), ns)
    return ns["create_proof_module"]


create_proof_module = _module_prover()


def record(h2, prover, params, vk, fixed, sigma, advice, instances, rng, zeta: int, delta: int, pk=None) -> dict:
    """Runs `prover` (create_proof_engine or create_proof_module) and returns the points and scalars it wrote, its proof, and
    the bytes of the last two queries it opened."""
    rec = {"points": [], "scalars": [], "queries": []}

    class T(R.Blake2bTranscript):
        def write_point(self, xy):
            rec["points"].append(np.array(xy, dtype=np.uint8).reshape(64).copy())
            super().write_point(xy)

        def write_scalar(self, v):
            rec["scalars"].append(int(v))
            super().write_scalar(v)

    class Multiopen:
        def __getattr__(self, name):
            return getattr(h2.multiopen, name)

        def create_proof(self, params_, rng_, transcript, queries):
            rec["queries"] = [(q.point, q.poly.download(), q.blind.value) for q in queries[-2:]]
            return h2.multiopen.create_proof(params_, rng_, transcript, queries)

    class Eng:
        multiopen = Multiopen()

        def __getattr__(self, name):
            return getattr(h2, name)

    t = T(vk.scalar_modulus)
    prover(Eng(), params, vk, fixed, sigma, advice, instances, rng, t, zeta, delta, pk=pk)
    rec["proof"] = bytes(t.proof)
    return rec


class VanishingFake(fake_engine.FakeLib):
    """The ABI stand-in with h2_poly_vanishing_quotient: the fused pass bodies on the host emulation (emul_vanishing.cpp),
    after the library's argument checks that the host mirror can reach."""

    def h2_poly_vanishing_quotient(self, pieces, count, src, k, ext_k, ext_omega_inv, ext_divisor, zeta, t_evals, t_len, repr_):
        who = "h2_poly_vanishing_quotient"
        self._log(who)
        count, src, k, ext_k, t_len = (fake_engine._v(x) for x in (count, src, k, ext_k, t_len))
        why = self.emu.emu_vanishing_quotient_sizes(k, ext_k, ctypes.c_uint64(count), t_len)
        if why:
            return self._fail(f"{who}: {ctypes.string_at(why).decode()}")
        hs = [int(pieces[i]) for i in range(count)]
        short = [i for i, h in enumerate(hs) if self.polys[h][1].shape[0] < 1 << k]
        if short:
            return self._fail(f"{who}: pieces[{short[0]}]: a polynomial holds fewer than 2^k elements")
        c = fake_engine.clash(fake_engine.args("pieces", hs, True) + [("src", src, False)])
        if c:
            return self._fail(f"{who}: {c}")
        f, a = self.polys[src]
        rd = fake_engine._rd
        out = np.zeros((count, 1 << k, 32), dtype=np.uint8)
        rc = self.emu.emu_vanishing_quotient(cref.FIELD_ID[f], cref._p(np.ascontiguousarray(a[:1 << ext_k])), k, ext_k, ctypes.c_uint64(count),
                                             cref._p(rd(ext_omega_inv, 32)), cref._p(rd(ext_divisor, 32)), cref._p(rd(zeta, 32)),
                                             cref._p(rd(t_evals, 32 * t_len)), t_len, cref._p(out), 0, 64)
        assert rc > 0, rc
        for i, h in enumerate(hs):
            self.polys[h][1][:1 << k] = out[i]
        return 0


@contextlib.contextmanager
def installed():
    """halo2_b200.lib bound to a VanishingFake for the duration of the block (and back to whatever it was afterwards)."""
    from halo2_b200 import lib as L
    saved = (L._lib, L._inited_device)
    fake = VanishingFake()
    L._lib, L._inited_device = fake, 0
    try:
        yield fake
    finally:
        L._lib, L._inited_device = saved
