"""Raw C-ABI helpers for the tests that call the library's entry points directly: the loaded library and its last error,
the lane calls, a sigma call on raw handles, the symbols the header declares, and a way to run work on several host
threads at once."""
from __future__ import annotations

import ctypes
import os
import re
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from halo2_b200 import lib as L
    return L.load()


def _err() -> str:
    return _lib().h2_last_error().decode()


def _create() -> int:
    h = ctypes.c_uint64(0)
    assert _lib().h2_lane_create(ctypes.byref(h)) == 0, _err()
    return h.value


def _bind(h: int) -> int:
    return _lib().h2_lane_bind(ctypes.c_uint64(h))


def _destroy(h: int) -> int:
    return _lib().h2_lane_destroy(ctypes.c_uint64(h))


def _run_parallel(fns):
    """Runs every fn on its own host thread at once; returns the results in order, or raises the first exception."""
    res, errs = [None] * len(fns), []
    start = threading.Barrier(len(fns))

    def run(i):
        try:
            start.wait()
            res[i] = fns[i]()
        except BaseException as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=run, args=(i,)) for i in range(len(fns))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errs:
        raise errs[0]
    return res


def _sigma_call(polys, k: int, mapping, omega: int, delta: int, repr_: int = 0, cols=None) -> int:
    """h2_poly_permutation_sigma on raw handles / mapping; omega and delta as given (already in `repr_`)."""
    from halo2_b200 import lib as L
    hs = [p if isinstance(p, int) else p._h.value for p in polys]
    arr = (ctypes.c_uint64 * max(len(hs), 1))(*hs)
    mp = None if mapping is None else np.ascontiguousarray(mapping, dtype=np.uint32)
    return _lib().h2_poly_permutation_sigma(arr if hs else None, ctypes.c_size_t(len(hs) if cols is None else cols), ctypes.c_uint32(k),
                                            None if mp is None else mp.ctypes.data_as(ctypes.c_void_p), L.ptr(L.fe_bytes(omega)),
                                            L.ptr(L.fe_bytes(delta)), repr_)


def _header_symbols():
    with open(os.path.join(ROOT, "include", "halo2_b200.h")) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(h2_[a-z0-9_]+)\s*\(", text)))
