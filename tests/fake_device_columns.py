"""TEST-ONLY: the ABI stand-in (tests/fake_engine.FakeLib) with the two device-memory column transfers,
h2_poly_upload_dev / h2_poly_download_dev.  Host addresses stand for device pointers.  The library's checks that do not need a
device run first: handles, lengths, aliasing, null pointers, alignment and overlapping destinations.  Then the K25 body
(csrc/columns_io.cuh) runs on the host emulation, through Montgomery form both ways.  Install it with `installed()`, as
fake_engine's."""
from __future__ import annotations

import contextlib
import ctypes

import numpy as np

from oracle import cref
from tests.fake_engine import FakeLib, _v, args, clash


class DeviceColumnsFake(FakeLib):
    def _dev_io(self, who, up, polys, count, ptrs, lens, repr_):
        count, canon = _v(count), int(_v(repr_) == 0)
        if count == 0:
            return 0
        pname = "d_src" if up else "d_dst"
        hs, ls, ps = [int(polys[i]) for i in range(count)], [int(lens[i]) for i in range(count)], [_v(ptrs[i] or 0) for i in range(count)]
        for i, h in enumerate(hs):
            if h not in self.polys:
                return self._fail(f"{who}: polys[{i}]: unknown polynomial handle")
            if up and h in self.shared:
                return self._fail(f"{who}: polys[{i}]: the polynomial is shared (read-only)")
            if self.polys[h][0] != self.polys[hs[0]][0]:
                return self._fail(f"{who}: polys[{i}]: the polynomials live in different fields")
            if ls[i] > self.polys[h][1].shape[0]:
                return self._fail(f"{who}: polys[{i}]: a polynomial holds fewer than lens[{i}] elements")
        if up:
            c = clash(args("polys", hs, True))
            if c:
                return self._fail(f"{who}: {c}")
        live = [i for i in range(count) if ls[i]]
        for i in live:
            if not ps[i]:
                return self._fail(f"{who}: {pname}[{i}]: null pointer")
            if ps[i] % 16:
                return self._fail(f"{who}: {pname}[{i}]: not 16-byte aligned")
        if not up:
            rs = sorted(live, key=lambda i: ps[i])
            for a, b in zip(rs, rs[1:]):
                if ps[b] < ps[a] + 32 * ls[a]:
                    return self._fail(f"{who}: {pname}[{max(a, b)}]: overlaps {pname}[{min(a, b)}]")
        if not live:
            return 0
        self._log(who)
        f = cref.FIELD_ID[self.polys[hs[0]][0]]
        for i in live:
            mont = np.zeros((ls[i], 32), dtype=np.uint8)
            store = self.polys[hs[i]][1]
            if up:
                self._emu_io(f, 1, canon, mont, ps[i], ls[i])                 # caller -> Montgomery
                buf = np.zeros((ls[i], 32), dtype=np.uint8)
                self._emu_io(f, 0, 1, mont, buf.ctypes.data, ls[i])           # the stand-in keeps canonical values
                store[:ls[i]] = buf
            else:
                src = np.ascontiguousarray(store[:ls[i]])
                self._emu_io(f, 1, 1, mont, src.ctypes.data, ls[i])
                self._emu_io(f, 0, canon, mont, ps[i], ls[i])                 # Montgomery -> caller
        return 0

    def _emu_io(self, field, to_dev, canon, res, addr, n):
        self.emu.emu_columns_io(field, to_dev, canon, ctypes.c_uint64(1), (ctypes.c_void_p * 1)(res.ctypes.data), (ctypes.c_void_p * 1)(addr),
                                (ctypes.c_uint64 * 1)(n))

    def h2_poly_upload_dev(self, polys, count, d_src, lens, repr_, stream):
        return self._dev_io("h2_poly_upload_dev", True, polys, count, d_src, lens, repr_)

    def h2_poly_download_dev(self, polys, count, d_dst, lens, repr_, stream):
        return self._dev_io("h2_poly_download_dev", False, polys, count, d_dst, lens, repr_)


@contextlib.contextmanager
def installed():
    """halo2_b200.lib bound to a DeviceColumnsFake for the duration of the block (and back to whatever it was afterwards)."""
    from halo2_b200 import lib as L
    saved = (L._lib, L._inited_device)
    fake = DeviceColumnsFake()
    L._lib, L._inited_device = fake, 0
    try:
        yield fake
    finally:
        L._lib, L._inited_device = saved
