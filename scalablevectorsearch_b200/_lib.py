"""ctypes binding of ``libsvsb200.so`` (the C ABI in ``include/svsb200.h``).

The library is CUDA-only.  There is deliberately no fallback: if the shared object is
missing or no sm_90-class device is usable, importing succeeds but every operation raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

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
    "svsb200_search_sharded", "svsb200_build_vamana", "svsb200_build_vamana_sq", "svsb200_flat_search_device", "svsb200_flat_search", "svsb200_index_assemble", "svsb200_toml_get", "svsb200_search_filtered", "svsb200_range_search", "svsb200_free", "svsb200_set_entry_points",
    "svsb200_flat_plan", "svsb200_flat_plan_k",
    "svsb200_flat_index_create", "svsb200_flat_index_destroy", "svsb200_flat_index_size", "svsb200_flat_index_dimensions",
    "svsb200_flat_index_device_bytes", "svsb200_flat_index_search", "svsb200_flat_index_search_device",
    "svsb200_dynamic_create", "svsb200_dynamic_delete", "svsb200_dynamic_ids", "svsb200_dynamic_has_id",
    "svsb200_dynamic_export", "svsb200_dynamic_set_build_parameters", "svsb200_dynamic_get_build_parameters",
    "svsb200_dynamic_add", "svsb200_dynamic_consolidate", "svsb200_dynamic_compact", "svsb200_dynamic_build",
    "svsb200_dynamic_flat_create", "svsb200_dynamic_flat_destroy", "svsb200_dynamic_flat_size",
    "svsb200_dynamic_flat_num_slots", "svsb200_dynamic_flat_dimensions", "svsb200_dynamic_flat_device_bytes",
    "svsb200_dynamic_flat_add", "svsb200_dynamic_flat_delete", "svsb200_dynamic_flat_compact", "svsb200_dynamic_flat_ids",
    "svsb200_dynamic_flat_has_id", "svsb200_dynamic_flat_export", "svsb200_dynamic_flat_search",
    "svsb200_dynamic_flat_search_device",
    "svsb200_flat_index_search_filtered", "svsb200_flat_index_search_filtered_device", "svsb200_flat_filter_plan",
    "svsb200_dynamic_flat_search_filtered", "svsb200_dynamic_flat_search_filtered_device",
    "svsb200_ivf_random", "svsb200_ivf_cluster", "svsb200_ivf_create", "svsb200_ivf_destroy", "svsb200_ivf_size",
    "svsb200_ivf_dimensions", "svsb200_ivf_num_clusters", "svsb200_ivf_device_bytes", "svsb200_ivf_cluster_sizes",
    "svsb200_ivf_centroids", "svsb200_ivf_search", "svsb200_ivf_search_device", "svsb200_sq_compress",
    "svsb200_ivf_create_sq", "svsb200_ivf_search_filtered", "svsb200_ivf_search_filtered_device",
    "svsb200_dynamic_ivf_create", "svsb200_dynamic_ivf_destroy", "svsb200_dynamic_ivf_size",
    "svsb200_dynamic_ivf_num_slots", "svsb200_dynamic_ivf_dimensions", "svsb200_dynamic_ivf_num_clusters",
    "svsb200_dynamic_ivf_device_bytes", "svsb200_dynamic_ivf_cluster_sizes", "svsb200_dynamic_ivf_centroids",
    "svsb200_dynamic_ivf_add", "svsb200_dynamic_ivf_delete", "svsb200_dynamic_ivf_compact", "svsb200_dynamic_ivf_ids",
    "svsb200_dynamic_ivf_has_id", "svsb200_dynamic_ivf_export", "svsb200_dynamic_ivf_search",
    "svsb200_dynamic_ivf_search_device", "svsb200_dynamic_ivf_create_sq", "svsb200_dynamic_ivf_search_filtered",
    "svsb200_dynamic_ivf_search_filtered_device",
]

_lib = None
#: the C ABI's element-type codes (SVSB200_F32 .. SVSB200_U8)
_DTYPE_CODE = {np.dtype(np.float32): 0, np.dtype(np.float16): 1, np.dtype(np.int8): 2, np.dtype(np.uint8): 3}
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
    l.svsb200_flat_plan_k.argtypes = [sz, sz, sz, i32, C.POINTER(u32), C.POINTER(u32), C.POINTER(u32), C.POINTER(u32), vp]
    l.svsb200_flat_index_create.argtypes = [vp, i32, sz, sz, sz, i32, i32, C.POINTER(vp)]
    l.svsb200_flat_index_destroy.argtypes = [vp]
    for name in ("size", "dimensions", "device_bytes"):
        fn = getattr(l, f"svsb200_flat_index_{name}")
        fn.restype, fn.argtypes = sz, [vp]
    l.svsb200_flat_index_search.argtypes = [vp, vp, i32, sz, sz, vp, vp]
    l.svsb200_flat_index_search_device.argtypes = [vp, vp, i32, sz, sz, vp, vp, vp, C.POINTER(u32)]
    l.svsb200_flat_index_search_filtered.argtypes = [vp, vp, i32, sz, sz, vp, vp, vp, C.POINTER(sz)]
    l.svsb200_flat_index_search_filtered_device.argtypes = [vp, vp, i32, sz, sz, vp, vp, vp, vp, C.POINTER(sz),
                                                            C.POINTER(u32)]
    l.svsb200_flat_filter_plan.argtypes = [sz, sz, C.POINTER(i32)]
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
    l.svsb200_build_vamana_sq.argtypes = [vp, i32, sz, sz, i32, C.c_float, C.c_float, C.c_float, sz, sz, sz, sz, i32, vp,
                                          C.POINTER(u32)]
    l.svsb200_dynamic_create.argtypes = [vp, i32, sz, sz, vp, sz, u32, i32, vp, i32, C.POINTER(vp)]
    l.svsb200_dynamic_delete.argtypes = [vp, vp, sz]
    l.svsb200_dynamic_ids.argtypes = [vp, vp, C.POINTER(sz)]
    l.svsb200_dynamic_has_id.argtypes = [vp, C.c_uint64, C.POINTER(i32)]
    l.svsb200_dynamic_export.argtypes = [vp, vp, vp, vp, C.POINTER(u32)]
    l.svsb200_dynamic_set_build_parameters.argtypes = [vp, C.c_float, sz, sz, sz]
    l.svsb200_dynamic_get_build_parameters.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]
    l.svsb200_dynamic_add.argtypes = [vp, vp, i32, sz, vp, i32, vp]
    l.svsb200_dynamic_consolidate.argtypes = [vp]
    l.svsb200_dynamic_compact.argtypes = [vp]
    l.svsb200_dynamic_build.argtypes = [vp, i32, sz, sz, i32, C.c_float, sz, sz, sz, sz, vp, i32, C.POINTER(vp)]
    l.svsb200_dynamic_flat_create.argtypes = [vp, i32, sz, sz, i32, vp, i32, C.POINTER(vp)]
    l.svsb200_dynamic_flat_destroy.argtypes = [vp]
    for name in ("size", "num_slots", "dimensions", "device_bytes"):
        fn = getattr(l, f"svsb200_dynamic_flat_{name}")
        fn.restype, fn.argtypes = sz, [vp]
    l.svsb200_dynamic_flat_add.argtypes = [vp, vp, i32, sz, vp, i32, vp]
    l.svsb200_dynamic_flat_delete.argtypes = [vp, vp, sz]
    l.svsb200_dynamic_flat_compact.argtypes = [vp]
    l.svsb200_dynamic_flat_ids.argtypes = [vp, vp, C.POINTER(sz)]
    l.svsb200_dynamic_flat_has_id.argtypes = [vp, C.c_uint64, C.POINTER(i32)]
    l.svsb200_dynamic_flat_export.argtypes = [vp, vp, vp]
    l.svsb200_dynamic_flat_search.argtypes = [vp, vp, i32, sz, sz, vp, vp]
    l.svsb200_dynamic_flat_search_device.argtypes = [vp, vp, i32, sz, sz, vp, vp, vp, C.POINTER(u32)]
    l.svsb200_dynamic_flat_search_filtered.argtypes = [vp, vp, i32, sz, sz, vp, vp, vp, C.POINTER(sz)]
    l.svsb200_dynamic_flat_search_filtered_device.argtypes = [vp, vp, i32, sz, sz, vp, vp, vp, vp, C.POINTER(sz),
                                                              C.POINTER(u32)]
    l.svsb200_ivf_random.argtypes = [C.c_uint64, sz, vp]
    l.svsb200_ivf_cluster.argtypes = [vp, i32, sz, sz, i32, sz, sz, sz, i32, C.c_float, C.c_uint64, i32, vp, vp]
    l.svsb200_ivf_create.argtypes = [vp, i32, sz, sz, i32, vp, sz, vp, i32, C.POINTER(vp)]
    l.svsb200_ivf_create_sq.argtypes = [vp, i32, sz, sz, i32, C.c_float, C.c_float, vp, sz, vp, i32, C.POINTER(vp)]
    l.svsb200_sq_compress.argtypes = [vp, sz, sz, i32, i32, vp, vp, vp]
    l.svsb200_ivf_destroy.argtypes = [vp]
    for name in ("size", "dimensions", "num_clusters", "device_bytes"):
        fn = getattr(l, f"svsb200_ivf_{name}")
        fn.restype, fn.argtypes = sz, [vp]
    l.svsb200_ivf_cluster_sizes.argtypes = [vp, vp]
    l.svsb200_ivf_centroids.argtypes = [vp, vp]
    l.svsb200_ivf_search.argtypes = [vp, vp, i32, sz, sz, sz, vp, vp]
    l.svsb200_ivf_search_device.argtypes = [vp, vp, i32, sz, sz, sz, vp, vp, vp]
    l.svsb200_ivf_search_filtered.argtypes = [vp, vp, i32, sz, sz, sz, vp, vp, vp, vp, vp, vp]
    l.svsb200_ivf_search_filtered_device.argtypes = [vp, vp, i32, sz, sz, sz, vp, vp, vp, vp, vp, vp, vp]
    l.svsb200_dynamic_ivf_create.argtypes = [vp, i32, sz, sz, i32, vp, sz, vp, vp, i32, C.POINTER(vp)]
    l.svsb200_dynamic_ivf_create_sq.argtypes = [vp, i32, sz, sz, i32, C.c_float, C.c_float, vp, sz, vp, vp, i32,
                                                C.POINTER(vp)]
    l.svsb200_dynamic_ivf_destroy.argtypes = [vp]
    for name in ("size", "num_slots", "dimensions", "num_clusters", "device_bytes"):
        fn = getattr(l, f"svsb200_dynamic_ivf_{name}")
        fn.restype, fn.argtypes = sz, [vp]
    l.svsb200_dynamic_ivf_cluster_sizes.argtypes = [vp, vp]
    l.svsb200_dynamic_ivf_centroids.argtypes = [vp, vp]
    l.svsb200_dynamic_ivf_add.argtypes = [vp, vp, i32, sz, vp, i32, vp]
    l.svsb200_dynamic_ivf_delete.argtypes = [vp, vp, sz]
    l.svsb200_dynamic_ivf_compact.argtypes = [vp]
    l.svsb200_dynamic_ivf_ids.argtypes = [vp, vp, C.POINTER(sz)]
    l.svsb200_dynamic_ivf_has_id.argtypes = [vp, C.c_uint64, C.POINTER(i32)]
    l.svsb200_dynamic_ivf_export.argtypes = [vp, vp, vp, vp]
    l.svsb200_dynamic_ivf_search.argtypes = [vp, vp, i32, sz, sz, sz, vp, vp]
    l.svsb200_dynamic_ivf_search_device.argtypes = [vp, vp, i32, sz, sz, sz, vp, vp, vp]
    l.svsb200_dynamic_ivf_search_filtered.argtypes = [vp, vp, i32, sz, sz, sz, vp, vp, vp, vp, vp, vp]
    l.svsb200_dynamic_ivf_search_filtered_device.argtypes = [vp, vp, i32, sz, sz, sz, vp, vp, vp, vp, vp, vp, vp]
    _lib = l
    return l


def check(rc: int) -> None:
    if rc != 0:
        raise Svsb200Error(lib().svsb200_last_error().decode(errors="replace"))


def _bitmap(allowed, n: int):
    """A boolean mask of n entries -> the uint32 bitmap of the filtered searches ((n + 31) / 32 words)."""
    mask = np.ascontiguousarray(allowed, dtype=bool)
    if mask.shape != (n,):
        raise ValueError(f"allowed must hold {n} booleans")
    b = np.packbits(mask, bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, dtype=np.uint8)]).view(np.uint32)


class _Slots:
    """``has_id``, ``all_ids``, ``delete`` and the argument checks of ``add``, shared by the dynamic indexes over their
    C functions ``{_ABI}_has_id``, ``_ids``, ``_delete`` and ``_add``."""

    _ABI = ""

    def _fn(self, name: str):
        return getattr(self._lib, f"{self._ABI}_{name}")

    def has_id(self, id: int) -> bool:
        out = C.c_int()
        check(self._fn("has_id")(self._h, int(id), C.byref(out)))
        return bool(out.value)

    def all_ids(self):
        """External ids of every Valid slot, in slot order."""
        n = C.c_size_t(self.size)
        out = np.empty(n.value, dtype=np.uint64)
        check(self._fn("ids")(self._h, out.ctypes.data, C.byref(n)))
        return out[: n.value]

    def delete(self, ids) -> int:
        """Deletes the entries of these external ids (what becomes of their slots: the class's docstring).  Fails
        without changing anything unless every id is present, once.  Returns the number of deleted entries."""
        ids = np.ascontiguousarray(np.atleast_1d(ids), dtype=np.uint64)
        check(self._fn("delete")(self._h, ids.ctypes.data, len(ids)))
        return len(ids)

    def _add(self, points, ids, reuse_empty: bool):
        """The body of ``add``: rows [count, dimensions] with one new external id each; returns the slots used."""
        pts = np.ascontiguousarray(points)
        ids = np.ascontiguousarray(np.atleast_1d(ids), dtype=np.uint64)
        if pts.ndim != 2 or pts.shape[1] != self.dimensions:
            raise ValueError(f"points must be [count, {self.dimensions}]")
        if pts.shape[0] != len(ids):
            raise ValueError(f"Number of points ({pts.shape[0]}) not equal to the number of external ids ({len(ids)})!")
        if pts.dtype not in _DTYPE_CODE:
            raise TypeError(f"unsupported data type {pts.dtype}")
        slots = np.empty(len(ids), dtype=np.uint64)
        check(self._fn("add")(self._h, pts.ctypes.data, _DTYPE_CODE[pts.dtype], len(ids), ids.ctypes.data,
                              int(bool(reuse_empty)), slots.ctypes.data))
        return slots


def _flat_search_filtered(fn, h, dims: int, queries, n_neighbors: int, bitmap, with_counts: bool):
    """The host form of the Flat and DynamicFlat filtered searches: (ids, dists, found[, allowed rows])."""
    q = np.ascontiguousarray(queries)
    if q.ndim != 2 or q.shape[1] != dims:
        raise ValueError(f"queries must be [nq, {dims}]")
    if q.dtype not in _DTYPE_CODE:
        raise TypeError(f"unsupported query type {q.dtype}")
    nq, k = q.shape[0], int(n_neighbors)
    ids = np.empty((nq, k), dtype=np.uint64)
    dists = np.empty((nq, k), dtype=np.float32)
    allowed = C.c_size_t()
    check(fn(h, q.ctypes.data, _DTYPE_CODE[q.dtype], nq, k, bitmap.ctypes.data, ids.ctypes.data, dists.ctypes.data,
             C.byref(allowed)))
    found = np.full(nq, min(k, allowed.value), dtype=np.uint32)
    if with_counts:
        return ids, dists, found, int(allowed.value)
    return ids, dists, found
