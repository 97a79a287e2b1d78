"""ctypes binding of include/halo2_b200.h.  Fails loudly when the CUDA library is missing or no
GPU is usable -- there is deliberately no other backend."""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_lib", "libhalo2_b200.so")
_lib: Optional[ctypes.CDLL] = None
_inited_device: Optional[int] = None

CURVE_ID = {"pallas": 0, "vesta": 1}
FIELD_ID = {"fp": 0, "fq": 1}
REPR_CANONICAL, REPR_MONTGOMERY = 0, 1
SCALAR_FIELD = {"pallas": "fq", "vesta": "fp"}
BASE_FIELD = {"pallas": "fp", "vesta": "fq"}

# every symbol the header declares (tests check the export list against include/halo2_b200.h)
SYMBOLS = [
    "h2_init", "h2_shutdown", "h2_last_error", "h2_device_count", "h2_abi_version", "h2_msm", "h2_bases_register", "h2_bases_register_ex",
    "h2_bases_release", "h2_msm_registered", "h2_msm_registered_batch", "h2_msm_registered_batch_affine", "h2_ipa_begin", "h2_ipa_round", "h2_ipa_fold", "h2_ipa_finish", "h2_poly_alloc", "h2_poly_free", "h2_poly_share", "h2_poly_upload", "h2_poly_download", "h2_poly_lagrange_to_coeff",
    "h2_poly_coeff_to_extended", "h2_poly_extended_to_coeff", "h2_msm_registered_polys", "h2_msm_registered_polys_affine", "h2_ipa_begin_poly", "h2_ipa_round_affine", "h2_poly_add_at", "h2_poly_copy", "h2_poly_eval", "h2_poly_inner_product", "h2_poly_kate_division", "h2_poly_divide_by_vanishing", "h2_poly_eval_ast", "h2_poly_batch_invert", "h2_poly_lookup_permute", "h2_poly_running_product", "h2_poly_compute_s", "h2_poly_scale_add", "h2_poly_permutation_sigma", "h2_poly_permutation_sigma_copies", "h2_poly_permutation_product", "h2_poly_lookup_product", "h2_poly_lookup_permuted", "h2_poly_lagrange_to_coeff_batch", "h2_poly_coeff_to_extended_batch", "h2_poly_set_rows", "h2_poly_vanishing_quotient", "h2_set_window_bits", "h2_set_glv", "h2_set_sort_mode", "h2_msm_dev", "h2_point_sum", "h2_point_sum_dev", "h2_multi_init", "h2_multi_count", "h2_msm_multi_gpu", "h2_multi_bases_register", "h2_multi_bases_release", "h2_msm_multi_registered", "h2_test_set_staging", "h2_test_set_copy_threads", "h2_test_set_batched_affine", "h2_test_set_ntt_tma", "h2_ntt",
    "h2_intt_scaled", "h2_coeff_to_extended", "h2_extended_to_coeff", "h2_ntt_dev", "h2_ntt_clear_cache",
    "h2_ec_fft", "h2_batch_normalize", "h2_params_lagrange", "h2_hash_to_curve", "h2_params_new", "h2_points_compress", "h2_points_decompress",
    "h2_dev_gen_points", "h2_dev_convert", "h2_test_last_msm_flags", "h2_test_last_msm_plan", "h2_test_set_chunk_threshold", "h2_test_set_chunk_cuts", "h2_test_set_graphs", "h2_test_set_poly_cta", "h2_test_set_fast_fixed", "h2_test_set_ecfft_quad", "h2_test_set_accum_ways", "h2_test_field_op", "h2_test_curve_op", "h2_bench_field_mul", "h2_bench_latency",
    "h2_launch_count", "h2_profile_enable", "h2_profile_read", "h2_lane_create", "h2_lane_bind", "h2_lane_destroy",
]


class H2Error(RuntimeError):
    pass


def lib_path() -> str:
    return _LIB_PATH


def load() -> ctypes.CDLL:
    """Loads the CUDA library (does not touch the GPU)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise H2Error(f"{_LIB_PATH} is missing: build it with `python -m halo2_b200.build` "
                      "(needs nvcc).  halo2_b200 has no CPU fallback.")
    lib = ctypes.CDLL(_LIB_PATH)
    for name in SYMBOLS:
        getattr(lib, name)  # AttributeError if the export is missing
    lib.h2_last_error.restype = ctypes.c_char_p
    lib.h2_abi_version.restype = ctypes.c_uint32
    lib.h2_launch_count.restype = ctypes.c_uint64
    for name in SYMBOLS:
        if name not in ("h2_last_error", "h2_abi_version", "h2_launch_count"):
            getattr(lib, name).restype = ctypes.c_int
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        raise H2Error(load().h2_last_error().decode("utf-8", "replace"))


def init(device: Optional[int] = None) -> ctypes.CDLL:
    """Binds the engine to a CUDA device (default: LOCAL_RANK or 0).  Raises H2Error without a GPU."""
    global _inited_device
    lib = load()
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    if _inited_device is None:
        check(lib.h2_init(int(device)))
        _inited_device = int(device)
    elif _inited_device != int(device):
        raise H2Error(f"engine already bound to device {_inited_device} (one process per GPU)")
    return lib


class Lane:
    """An independent prover context on the GPU: its own streams, scratch, caches, settings, resident polynomials and IPA
    sessions (include/halo2_b200.h, "lanes").  Every call from a thread bound to it runs there, concurrently with threads
    on other lanes; base sets (Params) are shared by all lanes.  Binding is per host thread.

        with Lane():          # created, bound to this thread; unbound and destroyed on exit
            prove(...)
    """

    def __init__(self, device: Optional[int] = None):
        lib = init(device)
        h = ctypes.c_uint64(0)
        check(lib.h2_lane_create(ctypes.byref(h)))
        self.handle = int(h.value)

    def bind(self) -> "Lane":
        """Binds the calling thread: its later calls run on this lane."""
        if not self.handle:
            raise H2Error("the lane is closed")
        check(load().h2_lane_bind(ctypes.c_uint64(self.handle)))
        return self

    def close(self) -> None:
        """Destroys the lane and everything created on it; the calling thread, if bound to it, goes back to the primary
        context.  Fails while another thread is bound to it."""
        if self.handle:
            check(load().h2_lane_destroy(ctypes.c_uint64(self.handle)))
            self.handle = 0

    def __enter__(self) -> "Lane":
        try:
            return self.bind()
        except BaseException:
            self.close()
            raise

    def __exit__(self, *exc) -> None:
        self.close()


def launch_count() -> int:
    return int(load().h2_launch_count())


# ---- buffer helpers ---------------------------------------------------------------------------
def as_u8(a, width: int) -> np.ndarray:
    arr = np.ascontiguousarray(a, dtype=np.uint8)
    if arr.ndim == 1:
        arr = arr.reshape(-1, width)
    if arr.ndim != 2 or arr.shape[1] != width:
        raise ValueError(f"expected an (n, {width}) uint8 array, got shape {arr.shape}")
    return arr


def ptr(a: Optional[np.ndarray]):
    if a is None:
        return None
    return a.ctypes.data_as(ctypes.c_void_p)


def fe_bytes(x) -> np.ndarray:
    """int or 32 bytes -> (32,) uint8 little-endian."""
    if isinstance(x, (int, np.integer)):
        return np.frombuffer(int(x).to_bytes(32, "little"), dtype=np.uint8).copy()
    arr = np.ascontiguousarray(x, dtype=np.uint8).reshape(-1)
    if arr.size != 32:
        raise ValueError("field element must be 32 bytes")
    return arr
