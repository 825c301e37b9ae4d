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

_lib = None
#: the C ABI's element-type codes (SVSB200_F32 .. SVSB200_U8)
_DTYPE_CODE = {np.dtype(np.float32): 0, np.dtype(np.float16): 1, np.dtype(np.int8): 2, np.dtype(np.uint8): 3}
#: the cancellation predicate of svsb200_search_cancellable: int (*)(void*)
CANCEL_FN = C.CFUNCTYPE(C.c_int, C.c_void_p)

vp, sz, i32, u32, u64, f32, cs = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32, C.c_uint64, C.c_float, C.c_char_p
P = C.POINTER
_GET, _H = (sz, [vp]), (i32, [vp])   # a size_t getter of a handle; a call on a handle alone
#: every function ``include/svsb200.h`` declares -> (restype, argtypes) (checked by tests/test_abi.py)
ABI = {
    "svsb200_last_error": (cs, []), "svsb200_version": (i32, []), "svsb200_device_count": (i32, []),
    "svsb200_device_sm": (i32, [i32, P(i32)]), "svsb200_launch_count": (u64, []),
    "svsb200_index_create": (i32, [vp, i32, sz, sz, sz, vp, sz, u32, i32, i32, vp, i32, P(vp)]),
    "svsb200_index_create_multi": (i32, [vp, i32, sz, sz, sz, vp, sz, u32, i32, i32, vp, P(i32), sz, P(vp)]),
    "svsb200_index_assemble": (i32, [cs, cs, cs, i32, sz, i32, P(i32), sz, P(vp)]),
    "svsb200_index_destroy": _H, "svsb200_index_size": _GET, "svsb200_index_dimensions": _GET,
    "svsb200_index_max_degree": _GET, "svsb200_index_device_bytes": _GET, "svsb200_index_num_devices": _GET,
    "svsb200_index_device": _H,
    "svsb200_search": (i32, [vp, vp, i32, sz, sz, sz, sz, i32, vp, i32, vp, vp]),
    "svsb200_search_device": (i32, [vp, vp, i32, sz, sz, sz, sz, i32, vp, i32, vp, vp]),
    "svsb200_search_cancellable": (i32, [vp, vp, i32, sz, sz, sz, sz, i32, vp, i32, vp, vp, CANCEL_FN, vp]),
    "svsb200_search_sharded": (i32, [P(vp), sz, vp, i32, sz, sz, sz, sz, vp, vp]),
    "svsb200_search_filtered": (i32, [vp, vp, i32, sz, sz, sz, vp, vp, vp, vp]),
    "svsb200_range_search": (i32, [vp, vp, i32, sz, f32, sz, vp, P(vp), P(vp)]), "svsb200_free": (None, [vp]),
    "svsb200_exhaustive_device": (i32, [vp, vp, i32, sz, sz, vp, vp, vp]),
    "svsb200_index_distances": (i32, [vp, vp, i32, sz, vp, vp]), "svsb200_index_reconstruct": (i32, [vp, vp, sz, vp]),
    "svsb200_flat_search": (i32, [vp, vp, i32, sz, sz, vp, vp]),
    "svsb200_flat_search_device": (i32, [vp, vp, i32, sz, sz, vp, vp, vp, P(u32)]),
    "svsb200_merge_topk_device": (i32, [vp, vp, sz, sz, sz, i32, vp, vp, i32, vp]),
    "svsb200_set_counting": (i32, [vp, i32]), "svsb200_get_counters": (i32, [vp, sz, vp, vp]),
    "svsb200_get_fetched": (i32, [vp, sz, vp]), "svsb200_last_kernel_ms": (i32, [vp, P(f32)]),
    "svsb200_set_option": (i32, [vp, cs, C.c_long]), "svsb200_get_option": (i32, [vp, cs, P(C.c_long)]),
    "svsb200_set_id_offset": (i32, [vp, u64]), "svsb200_set_entry_points": (i32, [vp, vp, sz]),
    "svsb200_toml_get": (i32, [cs, cs, cs, sz]),
    "svsb200_lvq8_row_stride": (sz, [sz]), "svsb200_lvq8_compress": (i32, [vp, sz, sz, vp, vp, i32]),
    "svsb200_build_vamana": (i32, [vp, i32, sz, sz, sz, i32, f32, sz, sz, sz, sz, i32, vp, P(u32)]),
    "svsb200_build_vamana_sq": (i32, [vp, i32, sz, sz, i32, f32, f32, f32, sz, sz, sz, sz, i32, vp, P(u32)]),
    "svsb200_dynamic_create": (i32, [vp, i32, sz, sz, vp, sz, u32, i32, vp, i32, P(vp)]),
    "svsb200_dynamic_build": (i32, [vp, i32, sz, sz, i32, f32, sz, sz, sz, sz, vp, i32, P(vp)]),
    "svsb200_dynamic_create_sq": (i32, [vp, i32, sz, sz, f32, f32, vp, sz, u32, i32, vp, i32, P(vp)]),
    "svsb200_dynamic_build_sq": (i32, [vp, i32, sz, sz, i32, f32, f32, f32, sz, sz, sz, sz, vp, i32, P(vp)]),
    "svsb200_dynamic_add": (i32, [vp, vp, i32, sz, vp, i32, vp]), "svsb200_dynamic_delete": (i32, [vp, vp, sz]),
    "svsb200_dynamic_ids": (i32, [vp, vp, P(sz)]), "svsb200_dynamic_has_id": (i32, [vp, u64, P(i32)]),
    "svsb200_dynamic_export": (i32, [vp, vp, vp, vp, P(u32)]),
    "svsb200_dynamic_consolidate": _H, "svsb200_dynamic_compact": _H,
    "svsb200_dynamic_set_build_parameters": (i32, [vp, f32, sz, sz, sz]),
    "svsb200_dynamic_get_build_parameters": (i32, [vp, P(f32), P(sz), P(sz), P(sz)]),
    "svsb200_flat_plan": (i32, [sz, sz, i32, P(u32), P(u32), P(u32), vp]),
    "svsb200_flat_plan_k": (i32, [sz, sz, sz, i32, P(u32), P(u32), P(u32), P(u32), vp]),
    "svsb200_flat_filter_plan": (i32, [sz, sz, P(i32)]),
    "svsb200_flat_index_create": (i32, [vp, i32, sz, sz, sz, i32, i32, P(vp)]),
    "svsb200_flat_index_destroy": _H, "svsb200_flat_index_size": _GET, "svsb200_flat_index_dimensions": _GET,
    "svsb200_flat_index_device_bytes": _GET,
    "svsb200_flat_index_search": (i32, [vp, vp, i32, sz, sz, vp, vp]),
    "svsb200_flat_index_search_device": (i32, [vp, vp, i32, sz, sz, vp, vp, vp, P(u32)]),
    "svsb200_flat_index_search_filtered": (i32, [vp, vp, i32, sz, sz, vp, vp, vp, P(sz)]),
    "svsb200_flat_index_search_filtered_device": (i32, [vp, vp, i32, sz, sz, vp, vp, vp, vp, P(sz), P(u32)]),
    "svsb200_dynamic_flat_create": (i32, [vp, i32, sz, sz, i32, vp, i32, P(vp)]),
    "svsb200_dynamic_flat_destroy": _H, "svsb200_dynamic_flat_size": _GET, "svsb200_dynamic_flat_num_slots": _GET,
    "svsb200_dynamic_flat_dimensions": _GET, "svsb200_dynamic_flat_device_bytes": _GET,
    "svsb200_dynamic_flat_add": (i32, [vp, vp, i32, sz, vp, i32, vp]),
    "svsb200_dynamic_flat_delete": (i32, [vp, vp, sz]), "svsb200_dynamic_flat_compact": _H,
    "svsb200_dynamic_flat_ids": (i32, [vp, vp, P(sz)]), "svsb200_dynamic_flat_has_id": (i32, [vp, u64, P(i32)]),
    "svsb200_dynamic_flat_export": (i32, [vp, vp, vp]),
    "svsb200_dynamic_flat_search": (i32, [vp, vp, i32, sz, sz, vp, vp]),
    "svsb200_dynamic_flat_search_device": (i32, [vp, vp, i32, sz, sz, vp, vp, vp, P(u32)]),
    "svsb200_dynamic_flat_search_filtered": (i32, [vp, vp, i32, sz, sz, vp, vp, vp, P(sz)]),
    "svsb200_dynamic_flat_search_filtered_device": (i32, [vp, vp, i32, sz, sz, vp, vp, vp, vp, P(sz), P(u32)]),
    "svsb200_ivf_random": (i32, [u64, sz, vp]),
    "svsb200_ivf_cluster": (i32, [vp, i32, sz, sz, i32, sz, sz, sz, i32, f32, u64, i32, vp, vp]),
    "svsb200_ivf_cluster_hierarchical": (i32, [vp, i32, sz, sz, i32, sz, sz, sz, sz, f32, u64, i32, vp, vp, vp]),
    "svsb200_sq_compress": (i32, [vp, sz, sz, i32, i32, vp, vp, vp]),
    "svsb200_ivf_create": (i32, [vp, i32, sz, sz, i32, vp, sz, vp, i32, P(vp)]),
    "svsb200_ivf_create_sq": (i32, [vp, i32, sz, sz, i32, f32, f32, vp, sz, vp, i32, P(vp)]),
    "svsb200_ivf_destroy": _H, "svsb200_ivf_size": _GET, "svsb200_ivf_dimensions": _GET,
    "svsb200_ivf_num_clusters": _GET, "svsb200_ivf_device_bytes": _GET,
    "svsb200_ivf_cluster_sizes": (i32, [vp, vp]), "svsb200_ivf_centroids": (i32, [vp, vp]),
    "svsb200_ivf_search": (i32, [vp, vp, i32, sz, sz, sz, vp, vp]),
    "svsb200_ivf_search_device": (i32, [vp, vp, i32, sz, sz, sz, vp, vp, vp]),
    "svsb200_ivf_search_filtered": (i32, [vp, vp, i32, sz, sz, sz, vp, vp, vp, vp, vp, vp]),
    "svsb200_ivf_search_filtered_device": (i32, [vp, vp, i32, sz, sz, sz, vp, vp, vp, vp, vp, vp, vp]),
    "svsb200_ivf_plan": (i32, [sz, i32, i32, i32, sz, sz, sz, i32] + [P(u32)] * 7 + [P(u64)]),
    "svsb200_ivf_group_plan": (i32, [sz, P(u32), P(u32), P(u64)]),
    "svsb200_dynamic_ivf_create": (i32, [vp, i32, sz, sz, i32, vp, sz, vp, vp, i32, P(vp)]),
    "svsb200_dynamic_ivf_create_sq": (i32, [vp, i32, sz, sz, i32, f32, f32, vp, sz, vp, vp, i32, P(vp)]),
    "svsb200_dynamic_ivf_destroy": _H, "svsb200_dynamic_ivf_size": _GET, "svsb200_dynamic_ivf_num_slots": _GET,
    "svsb200_dynamic_ivf_dimensions": _GET, "svsb200_dynamic_ivf_num_clusters": _GET,
    "svsb200_dynamic_ivf_device_bytes": _GET,
    "svsb200_dynamic_ivf_cluster_sizes": (i32, [vp, vp]), "svsb200_dynamic_ivf_centroids": (i32, [vp, vp]),
    "svsb200_dynamic_ivf_add": (i32, [vp, vp, i32, sz, vp, i32, vp]),
    "svsb200_dynamic_ivf_delete": (i32, [vp, vp, sz]), "svsb200_dynamic_ivf_compact": _H,
    "svsb200_dynamic_ivf_ids": (i32, [vp, vp, P(sz)]), "svsb200_dynamic_ivf_has_id": (i32, [vp, u64, P(i32)]),
    "svsb200_dynamic_ivf_export": (i32, [vp, vp, vp, vp]),
    "svsb200_dynamic_ivf_search": (i32, [vp, vp, i32, sz, sz, sz, vp, vp]),
    "svsb200_dynamic_ivf_search_device": (i32, [vp, vp, i32, sz, sz, sz, vp, vp, vp]),
    "svsb200_dynamic_ivf_search_filtered": (i32, [vp, vp, i32, sz, sz, sz, vp, vp, vp, vp, vp, vp]),
    "svsb200_dynamic_ivf_search_filtered_device": (i32, [vp, vp, i32, sz, sz, sz, vp, vp, vp, vp, vp, vp, vp]),
}
SYMBOLS = list(ABI)
del vp, sz, i32, u32, u64, f32, cs, P, _GET, _H


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
    for name, (restype, argtypes) in ABI.items():
        fn = getattr(l, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = l
    return l


def check(rc: int) -> None:
    if rc != 0:
        raise Svsb200Error(lib().svsb200_last_error().decode(errors="replace"))


def _rows(data, dtypes=_DTYPE_CODE, ndim_error: str | None = "data must be a 2-D array",
          dtype_error: str = "unsupported data type {}") -> np.ndarray:
    """The rows of an index or a codec: ``data`` (an array, or a loader with ``load()``) as a contiguous 2-D array of
    one of ``dtypes``.  ``dtype_error`` is formatted with the dtype; without ``ndim_error`` a wrong rank raises it too."""
    x = np.ascontiguousarray(data.load() if hasattr(data, "load") else data)
    if x.ndim != 2 and ndim_error is not None:
        raise ValueError(ndim_error)
    if x.ndim != 2 or x.dtype not in dtypes:
        raise TypeError(dtype_error.format(x.dtype))
    return x


def _queries(queries, dims: int, width: str | None = None) -> np.ndarray:
    """The queries of a host-buffer search: 2-D, ``dims`` wide and of a supported type, returned contiguous (the
    library reads nq x dims elements).  ``width`` words the width in the error where it is not the number."""
    q = np.ascontiguousarray(queries)
    if q.ndim != 2 or q.shape[1] != dims:
        raise ValueError(f"queries must be [nq, {width or dims}]")
    if q.dtype not in _DTYPE_CODE:
        raise TypeError(f"unsupported query type {q.dtype}")
    return q


def _results(nq: int, k: int):
    """The (ids uint64, distances float32) [nq, k] of a host-buffer search."""
    return np.empty((nq, k), dtype=np.uint64), np.empty((nq, k), dtype=np.float32)


def _search(fn, head: tuple, q: np.ndarray, n_neighbors: int, mid: tuple = (), tail: tuple = ()):
    """Runs the host-buffer search ``fn(*head, queries, qtype, nq, k, *mid, ids, dists, *tail)`` over queries from
    :func:`_queries`; returns (ids, dists) of :func:`_results`."""
    nq, k = q.shape[0], int(n_neighbors)
    ids, dists = _results(nq, k)
    check(fn(*head, q.ctypes.data, _DTYPE_CODE[q.dtype], nq, k, *mid, ids.ctypes.data, dists.ctypes.data, *tail))
    return ids, dists


def _bitmap(allowed, n: int):
    """A boolean mask of n entries -> the uint32 bitmap of the filtered searches ((n + 31) / 32 words)."""
    mask = np.ascontiguousarray(allowed, dtype=bool)
    if mask.shape != (n,):
        raise ValueError(f"allowed must hold {n} booleans")
    b = np.packbits(mask, bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, dtype=np.uint8)]).view(np.uint32)


class _Handle:
    """An index behind the handle ``_h`` of the C functions ``{_PREFIX}_*``: ``_destroy`` when it is collected, the
    ``size``, ``dimensions`` and ``device_bytes`` getters, and ``num_threads``, kept for interface parity (the
    reference's thread pool is replaced by the grid)."""

    _PREFIX = ""

    def _cfn(self, name: str):
        return getattr(self._lib, f"{self._PREFIX}_{name}")

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._cfn("destroy")(h)
            self._h = None

    @property
    def size(self) -> int:
        return self._cfn("size")(self._h)

    @property
    def dimensions(self) -> int:
        return self._cfn("dimensions")(self._h)

    @property
    def device_bytes(self) -> int:
        return self._cfn("device_bytes")(self._h)

    @property
    def num_threads(self) -> int:
        return self._num_threads

    @num_threads.setter
    def num_threads(self, n: int):
        self._num_threads = int(n)


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
