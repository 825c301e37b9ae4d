"""ctypes binding of ``libsvsb200.so`` (the C ABI in ``include/svsb200.h``).

The library is CUDA-only.  There is deliberately no fallback: if the shared object is
missing or no sm_90-class device is usable, importing succeeds but every operation raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SVSB200_LIB lets experiments point at an alternative build; the default is the in-tree library.
LIB_PATH = os.environ.get("SVSB200_LIB") or os.path.join(_HERE, "libsvsb200.so")

#: every symbol ``include/svsb200.h`` declares (checked by tests/test_abi.py)
SYMBOLS = [
    "svsb200_last_error", "svsb200_version", "svsb200_device_count", "svsb200_device_sm",
    "svsb200_index_create", "svsb200_index_destroy", "svsb200_index_size",
    "svsb200_index_dimensions", "svsb200_index_max_degree", "svsb200_index_device_bytes",
    "svsb200_index_device", "svsb200_search", "svsb200_search_device", "svsb200_set_counting",
    "svsb200_get_counters", "svsb200_get_fetched", "svsb200_last_kernel_ms", "svsb200_launch_count", "svsb200_set_option", "svsb200_get_option",
    "svsb200_merge_topk_device", "svsb200_exhaustive_device", "svsb200_lvq8_row_stride", "svsb200_lvq8_compress",
    "svsb200_index_create_multi", "svsb200_index_num_devices", "svsb200_search_cancellable", "svsb200_set_id_offset",
    "svsb200_search_sharded", "svsb200_build_vamana", "svsb200_flat_search_device", "svsb200_flat_search", "svsb200_index_assemble", "svsb200_toml_get", "svsb200_search_filtered", "svsb200_range_search", "svsb200_free", "svsb200_set_entry_points",
    "svsb200_flat_plan",
]

_lib = None
#: the cancellation predicate of svsb200_search_cancellable: int (*)(void*)
CANCEL_FN = C.CFUNCTYPE(C.c_int, C.c_void_p)


class Svsb200Error(RuntimeError):
    """Raised for every non-zero return code of the C ABI (the C++ adapter throws ANNException)."""


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Svsb200Error(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(make -C scalablevectorsearch_b200/csrc). There is no CPU fallback.")
    l = C.CDLL(LIB_PATH)
    vp, sz, i32, u32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
    l.svsb200_last_error.restype = C.c_char_p
    l.svsb200_launch_count.restype = C.c_uint64
    l.svsb200_device_sm.argtypes = [i32, C.POINTER(i32)]
    l.svsb200_flat_plan.argtypes = [C.c_size_t, C.c_size_t, i32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                    C.POINTER(C.c_uint32), C.c_void_p]
    l.svsb200_index_create.argtypes = [vp, i32, sz, sz, sz, vp, sz, u32, i32, i32, vp, i32, C.POINTER(vp)]
    l.svsb200_index_destroy.argtypes = [vp]
    for name in ("size", "dimensions", "max_degree", "device_bytes"):
        fn = getattr(l, f"svsb200_index_{name}")
        fn.restype, fn.argtypes = sz, [vp]
    l.svsb200_index_device.argtypes = [vp]
    l.svsb200_search.argtypes = [vp, vp, i32, sz, sz, sz, sz, i32, vp, i32, vp, vp]
    l.svsb200_search_device.argtypes = [vp, vp, i32, sz, sz, sz, sz, i32, vp, i32, vp, vp]
    l.svsb200_set_counting.argtypes = [vp, i32]
    l.svsb200_get_counters.argtypes = [vp, sz, vp, vp]
    l.svsb200_get_fetched.argtypes = [vp, sz, vp]
    l.svsb200_last_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
    l.svsb200_set_option.argtypes = [vp, C.c_char_p, C.c_long]
    l.svsb200_get_option.argtypes = [vp, C.c_char_p, C.POINTER(C.c_long)]
    l.svsb200_merge_topk_device.argtypes = [vp, vp, sz, sz, sz, i32, vp, vp, i32, vp]
    l.svsb200_lvq8_row_stride.restype, l.svsb200_lvq8_row_stride.argtypes = sz, [sz]
    l.svsb200_lvq8_compress.argtypes = [vp, sz, sz, vp, vp, i32]
    l.svsb200_exhaustive_device.argtypes = [vp, vp, i32, sz, sz, vp, vp, vp]
    l.svsb200_index_create_multi.argtypes = [vp, i32, sz, sz, sz, vp, sz, u32, i32, i32, vp, C.POINTER(i32), sz,
                                             C.POINTER(vp)]
    l.svsb200_index_num_devices.restype, l.svsb200_index_num_devices.argtypes = sz, [vp]
    l.svsb200_search_cancellable.argtypes = [vp, vp, i32, sz, sz, sz, sz, i32, vp, i32, vp, vp, CANCEL_FN, vp]
    l.svsb200_set_id_offset.argtypes = [vp, C.c_uint64]
    l.svsb200_search_sharded.argtypes = [C.POINTER(vp), sz, vp, i32, sz, sz, sz, sz, vp, vp]
    l.svsb200_flat_search_device.argtypes = [vp, vp, i32, sz, sz, vp, vp, vp, C.POINTER(u32)]
    l.svsb200_flat_search.argtypes = [vp, vp, i32, sz, sz, vp, vp]
    l.svsb200_index_assemble.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, i32, sz, i32, C.POINTER(i32), sz, C.POINTER(vp)]
    l.svsb200_toml_get.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, sz]
    l.svsb200_search_filtered.argtypes = [vp, vp, i32, sz, sz, sz, vp, vp, vp, vp]
    l.svsb200_range_search.argtypes = [vp, vp, i32, sz, C.c_float, sz, vp, C.POINTER(vp), C.POINTER(vp)]
    l.svsb200_free.argtypes = [vp]
    l.svsb200_free.restype = None
    l.svsb200_set_entry_points.argtypes = [vp, vp, sz]
    l.svsb200_build_vamana.argtypes = [vp, i32, sz, sz, sz, i32, C.c_float, sz, sz, sz, sz, i32, vp, C.POINTER(u32)]
    _lib = l
    return l


def check(rc: int) -> None:
    if rc != 0:
        raise Svsb200Error(lib().svsb200_last_error().decode(errors="replace"))
