"""TEST-ONLY: the ABI stand-in (tests/fake_engine.FakeLib) with the device draws of the prover's random polynomials,
h2_poly_random.  The library's checks run first, in its order and with its messages: count, null arguments, the word offset,
handles, fields, lengths, aliasing and the end of the keystream.  Then the K26 body (csrc/chacha.cuh) runs over the launch's
whole grid on the host emulation.  Install it with `installed()`, as fake_engine's."""
from __future__ import annotations

import contextlib
import ctypes

import numpy as np

from oracle import cref
from tests.fake_engine import FakeLib, _rd, _v, args, clash


class RandomFake(FakeLib):
    def h2_poly_random(self, polys, count, lens, seed32, stream, block, word):
        who = "h2_poly_random"
        count, stream, block, word = _v(count), _v(stream), _v(block), _v(word)
        if count == 0:
            return self._fail(f"{who}: count == 0")
        if polys is None or lens is None:
            return self._fail(f"{who}: null argument")
        if seed32 is None or not _v(seed32):
            return self._fail(f"{who}: null seed32")
        if word >= 16:
            return self._fail(f"{who}: word >= 16")
        hs, ls = [int(polys[i]) for i in range(count)], [int(lens[i]) for i in range(count)]
        for i, h in enumerate(hs):
            if h not in self.polys:
                return self._fail(f"{who}: polys[{i}]: unknown polynomial handle")
            if h in self.shared:
                return self._fail(f"{who}: polys[{i}]: the polynomial is shared (read-only)")
            if self.polys[h][0] != self.polys[hs[0]][0]:
                return self._fail(f"{who}: polys[{i}]: the polynomials live in different fields")
            if ls[i] > self.polys[h][1].shape[0]:
                return self._fail(f"{who}: polys[{i}]: a polynomial holds fewer than lens[{i}] elements")
        c = clash(args("polys", hs, True))
        if c:
            return self._fail(f"{who}: {c}")
        total = sum(ls)
        if total == 0:
            return 0
        if block + total - 1 + (word != 0) >= 1 << 64:
            return self._fail(f"{who}: the draws run past keystream block 2^64 - 1")
        self._log(who)
        f = cref.FIELD_ID[self.polys[hs[0]][0]]
        out = np.zeros((total, 32), dtype=np.uint8)
        self.emu.emu_chacha_random(f, cref._p(_rd(seed32, 32)), ctypes.c_uint64(stream), ctypes.c_uint64(block), ctypes.c_uint32(word),
                                   ctypes.c_uint64(count), (ctypes.c_uint64 * count)(*ls), cref._p(out))
        at = 0
        for h, n in zip(hs, ls):
            self.polys[h][1][:n] = out[at:at + n]
            at += n
        return 0


@contextlib.contextmanager
def installed():
    """halo2_b200.lib bound to a RandomFake for the duration of the block (and back to whatever it was afterwards)."""
    from halo2_b200 import lib as L
    saved = (L._lib, L._inited_device)
    fake = RandomFake()
    L._lib, L._inited_device = fake, 0
    try:
        yield fake
    finally:
        L._lib, L._inited_device = saved
