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
from ._lib import _DTYPE_CODE
from .vamana import DistanceType


class _FlatSearch(_lib._Handle):
    """The search forms of Flat and DynamicFlat over ``{_PREFIX}_search*``.  The filter mask has one entry per
    ``_MASK`` (``size`` or ``num_slots``), and the bitmap of the device form (_MASK + 31) / 32 uint32 words."""

    _MASK = "size"

    def search(self, queries: np.ndarray, n_neighbors: int):
        """``search(queries, n_neighbors)`` -> (ids uint64 [nq,k], distances float32 [nq,k]): the exact top k."""
        q = _lib._queries(queries, self.dimensions)
        return _lib._search(self._cfn("search"), (self._h,), q, n_neighbors)

    def search_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_ids: int, d_dists: int,
                      stream: int = 0) -> int:
        """Device-buffer form (raw pointers, e.g. ``tensor.data_ptr()``; ids uint64); returns how many queries ran on
        the exact scan."""
        fb = C.c_uint32()
        _lib.check(self._cfn("search_device")(self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq, int(n_neighbors),
                                              d_ids, d_dists, stream or None, C.byref(fb)))
        return int(fb.value)

    def search_filtered(self, queries: np.ndarray, n_neighbors: int, allowed: np.ndarray, with_counts: bool = False):
        """``search`` with a predicate: ``allowed`` is a boolean mask (see the class).  Returns (ids uint64 [nq,k],
        distances float32 [nq,k], found per query = min(k, allowed rows)): the exact top k over the allowed rows; short
        rows are padded with 2^64 - 1 / +inf for every metric.  ``with_counts`` adds the number of allowed rows."""
        dims = self.dimensions
        bitmap = _lib._bitmap(allowed, getattr(self, self._MASK))
        q = _lib._queries(queries, dims)
        n_allowed = C.c_size_t()
        ids, dists = _lib._search(self._cfn("search_filtered"), (self._h,), q, n_neighbors, (bitmap.ctypes.data,),
                                  (C.byref(n_allowed),))
        found = np.full(q.shape[0], min(int(n_neighbors), n_allowed.value), dtype=np.uint32)
        if with_counts:
            return ids, dists, found, int(n_allowed.value)
        return ids, dists, found

    def search_filtered_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_bitmap: int,
                               d_ids: int, d_dists: int, stream: int = 0) -> int:
        """Device-buffer form of :meth:`search_filtered` (raw pointers; the uint32 bitmap: see the class); returns how
        many queries ran on a scan."""
        fb = C.c_uint32()
        _lib.check(self._cfn("search_filtered_device")(
            self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq, int(n_neighbors), d_bitmap, d_ids, d_dists,
            stream or None, None, C.byref(fb)))
        return int(fb.value)


class Flat(_FlatSearch):
    """``svs.Flat(data, distance, num_threads)`` on one CUDA device.  ``device_bytes`` counts the rows (no graph is
    stored).  The filtered search is ``FlatIndex::search`` with a predicate (flat.h:421-465): ``allowed`` is a boolean
    mask over the ids, and the result equals :meth:`search` on a Flat of the allowed rows with its ids mapped back; the
    device form's bitmap has (size + 31) / 32 words, bit i = id i."""

    _PREFIX = "svsb200_flat_index"

    def __init__(self, data, distance: DistanceType = DistanceType.L2, num_threads: int = 1, device: int = 0):
        data = _lib._rows(data)
        self._lib = _lib.lib()
        self._distance = DistanceType(distance)
        self._num_threads = int(num_threads)
        handle = C.c_void_p()
        _lib.check(self._lib.svsb200_flat_index_create(data.ctypes.data, _DTYPE_CODE[data.dtype], data.shape[0],
                                                        data.shape[1], 0, int(self._distance), int(device),
                                                        C.byref(handle)))
        self._h = handle


def filter_route(n: int, allowed: int) -> str:
    """The route a filtered flat search takes with ``allowed`` of ``n`` rows allowed: "sparse" (the allowed rows are
    gathered and scanned alone) or "dense" (the index's own routing with the other rows masked)."""
    route = C.c_int()
    _lib.check(_lib.lib().svsb200_flat_filter_plan(int(n), int(allowed), C.byref(route)))
    return "sparse" if route.value == 1 else "dense"
