"""CPU-only checks of the boundary: the C-ABI library builds, loads and exports every symbol
include/halo2_b200.h declares; the product path fails loudly without a GPU (no CPU fallback)."""
import os
import re

import numpy as np
import pytest

from tests.abi_cases import _header_symbols

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from halo2_b200 import build, lib
    build.build()
    handle = lib.load()
    declared = _header_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(handle, name), f"{name} declared in include/halo2_b200.h but not exported"
    assert sorted(lib.SYMBOLS) == declared
    assert handle.h2_abi_version() == 1


def test_no_cpu_fallback():
    """Without a CUDA device every operation must raise, never compute on the host."""
    import halo2_b200
    from halo2_b200 import lib
    if lib.load().h2_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(halo2_b200.H2Error):
        halo2_b200.best_multiexp(np.zeros((2, 32), np.uint8), np.zeros((2, 64), np.uint8), "pallas")
    a = np.zeros((4, 32), np.uint8)
    with pytest.raises(halo2_b200.H2Error):
        halo2_b200.best_fft(a, 1, 2, "fp")
    # ... and so must everything either side of the two kernels
    for call in (lambda: halo2_b200.lagrange_generators("vesta", 2, np.zeros((4, 64), np.uint8)),
                 lambda: halo2_b200.best_fft_curve(np.zeros((4, 96), np.uint8), 1, 2, "vesta"),
                 lambda: halo2_b200.batch_normalize(np.zeros((3, 96), np.uint8), "pallas"),
                 lambda: halo2_b200.hash_to_curve("pallas", "Halo2-Parameters")(b"\x01"),
                 lambda: halo2_b200.Params.new("vesta", 2),
                 lambda: halo2_b200.compress_points(np.zeros((3, 64), np.uint8), "pallas"),
                 lambda: halo2_b200.decompress_points(np.zeros((3, 32), np.uint8), "vesta"),
                 lambda: halo2_b200.eval_polynomial(a, 3, "fp"),
                 lambda: halo2_b200.kate_division(a, 3, "fq"),
                 lambda: halo2_b200.compute_inner_product(a, a, "fp"),
                 lambda: halo2_b200.ResidentPoly("fp", 4),
                 lambda: halo2_b200.small_multiexp(np.zeros((2, 32), np.uint8), np.zeros((2, 64), np.uint8), "vesta")):
        with pytest.raises(halo2_b200.H2Error):
            call()


def test_product_does_not_import_oracle():
    """The package must not reference oracle/ or the test-only emulation."""
    pkg = os.path.join(ROOT, "halo2_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                with open(os.path.join(dirpath, fn)) as f:
                    src = f.read()
                for pat in (r"(from|import)\s+oracle", r"halo2_oracle", r"oracle[/.](pasta|cref|_build|_ref)",
                            r"(from|import)\s+tests", r"libh2_kernel_emul", r"fake_engine", r"FakeLib"):
                    assert not re.search(pat, src), (fn, pat)
