"""Exact flat index on the GPU, mirroring the reference's ``svs.Flat`` (bindings/python/src/flat.cpp):

    index = Flat(data, distance=DistanceType.L2)      # [n, dim] array or a VectorDataLoader
    I, D = index.search(queries, 100)                  # numpy (nq, k) uint64 / float32

Backed by the graph-free handle of ``libsvsb200.so`` (``svsb200_flat_index_*``): k <= 25 and 26 <= k <= 121 run on the
tensor cores, everything else on the exact scan, and the result always equals the exact scan bit for bit.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .vamana import _DTYPE_CODE, DistanceType


class Flat:
    """``svs.Flat(data, distance, num_threads)`` on one CUDA device."""

    def __init__(self, data, distance: DistanceType = DistanceType.L2, num_threads: int = 1, device: int = 0):
        data = data.load() if hasattr(data, "load") else data
        data = np.ascontiguousarray(data)
        if data.ndim != 2:
            raise ValueError("data must be a 2-D array")
        if data.dtype not in _DTYPE_CODE:
            raise TypeError(f"unsupported data type {data.dtype}")
        self._lib = _lib.lib()
        self._distance = DistanceType(distance)
        self._num_threads = int(num_threads)
        handle = C.c_void_p()
        _lib.check(self._lib.svsb200_flat_index_create(data.ctypes.data, _DTYPE_CODE[data.dtype], data.shape[0],
                                                        data.shape[1], 0, int(self._distance), int(device),
                                                        C.byref(handle)))
        self._h = handle

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._lib.svsb200_flat_index_destroy(h)
            self._h = None

    @property
    def size(self) -> int:
        return self._lib.svsb200_flat_index_size(self._h)

    @property
    def dimensions(self) -> int:
        return self._lib.svsb200_flat_index_dimensions(self._h)

    @property
    def device_bytes(self) -> int:
        """Device memory held by the rows (no graph is stored)."""
        return self._lib.svsb200_flat_index_device_bytes(self._h)

    @property
    def num_threads(self) -> int:
        """Kept for interface parity: the reference's thread pool is replaced by the grid."""
        return self._num_threads

    @num_threads.setter
    def num_threads(self, n: int):
        self._num_threads = int(n)

    def search(self, queries: np.ndarray, n_neighbors: int):
        """``svs.Flat.search(queries, n_neighbors)`` -> (ids uint64 [nq,k], distances float32 [nq,k]): the exact top k."""
        q = np.ascontiguousarray(queries)
        if q.ndim != 2 or q.shape[1] != self.dimensions:
            raise ValueError(f"queries must be [nq, {self.dimensions}]")
        if q.dtype not in _DTYPE_CODE:
            raise TypeError(f"unsupported query type {q.dtype}")
        nq, k = q.shape[0], int(n_neighbors)
        ids = np.empty((nq, k), dtype=np.uint64)
        dists = np.empty((nq, k), dtype=np.float32)
        _lib.check(self._lib.svsb200_flat_index_search(self._h, q.ctypes.data, _DTYPE_CODE[q.dtype], nq, k,
                                                       ids.ctypes.data, dists.ctypes.data))
        return ids, dists

    def search_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_ids: int, d_dists: int,
                      stream: int = 0) -> int:
        """Device-buffer form (raw pointers, e.g. ``tensor.data_ptr()``; ids uint64); returns how many queries ran on
        the exact scan."""
        fb = C.c_uint32()
        _lib.check(self._lib.svsb200_flat_index_search_device(self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq,
                                                              int(n_neighbors), d_ids, d_dists, stream or None,
                                                              C.byref(fb)))
        return int(fb.value)

    def search_filtered(self, queries: np.ndarray, n_neighbors: int, allowed: np.ndarray, with_counts: bool = False):
        """``FlatIndex::search`` with a predicate (flat.h:421-465): ``allowed`` is a boolean mask over the ids.  Returns
        (ids uint64 [nq,k], distances float32 [nq,k], found per query = min(k, allowed rows)): the exact top k over the
        allowed rows, equal to :meth:`search` on a Flat of those rows with its ids mapped back; short rows are padded
        with 2^64 - 1 / +inf for every metric.  ``with_counts`` adds the number of allowed rows."""
        return _lib._flat_search_filtered(self._lib.svsb200_flat_index_search_filtered, self._h, self.dimensions,
                                          queries, n_neighbors, _lib._bitmap(allowed, self.size), with_counts)

    def search_filtered_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_bitmap: int,
                               d_ids: int, d_dists: int, stream: int = 0) -> int:
        """Device-buffer form of :meth:`search_filtered` (raw pointers; the uint32 bitmap has (size + 31) / 32 words,
        bit i = id i); returns how many queries ran on a scan."""
        fb = C.c_uint32()
        _lib.check(self._lib.svsb200_flat_index_search_filtered_device(
            self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq, int(n_neighbors), d_bitmap, d_ids, d_dists,
            stream or None, None, C.byref(fb)))
        return int(fb.value)


def filter_route(n: int, allowed: int) -> str:
    """The route a filtered flat search takes with ``allowed`` of ``n`` rows allowed: "sparse" (the allowed rows are
    gathered and scanned alone) or "dense" (the index's own routing with the other rows masked)."""
    route = C.c_int()
    _lib.check(_lib.lib().svsb200_flat_filter_plan(int(n), int(allowed), C.byref(route)))
    return "sparse" if route.value == 1 else "dense"
