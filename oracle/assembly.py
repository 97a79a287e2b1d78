"""ctypes front-end for oracle/assembly_oracle.c (TEST INFRASTRUCTURE ONLY -- see pasta.py): the reference's sequential
Assembly::copy loop in C, the oracle of the device copy-cycle computation (csrc/assembly.cuh) and its timed CPU baseline."""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "assembly_oracle.c")
_SO = os.path.join(_HERE, "_build", "libassembly_oracle.so")
_lib: Optional[ctypes.CDLL] = None


def build(force: bool = False) -> str:
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fPIC", "-Wall", "-Wextra", "-shared", "-o", _SO, _SRC])
    return _SO


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        build()                  # no-op unless the source is newer than the library
        _lib = ctypes.CDLL(_SO)
        _lib.orc_assembly.restype = ctypes.c_int
    return _lib


def assembly(copies, cols: int, k: int):
    """Assembly::new + Assembly::copy (plonk/permutation/keygen.rs:24-100, see orc_assembly) over an (m, 4) array of copies
    (left column, left row, right column, right row).  Returns (mapping, None) with mapping a (cols, 2^k, 2) uint32 array of
    (column, row) pairs, or (None, (kind, index)) for the first bad copy, kind "column" or "row"."""
    cp = np.ascontiguousarray(np.asarray(copies, dtype=np.uint32).reshape(-1, 4))
    out = np.empty((cols, 1 << k, 2), dtype=np.uint32)
    bad = ctypes.c_size_t(0)
    rc = lib().orc_assembly(cp.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(cp.shape[0]), ctypes.c_uint32(cols), ctypes.c_uint32(k),
                            out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(bad))
    if rc:
        return None, ("column" if rc == 1 else "row", bad.value)
    return out, None
