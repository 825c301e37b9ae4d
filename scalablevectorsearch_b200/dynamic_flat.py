"""Dynamic exact flat index on the GPU, mirroring the reference's ``svs.DynamicFlat``
(bindings/python/src/dynamic_flat.cpp, include/svs/index/flat/dynamic_flat.h):

    index = DynamicFlat.build(data, ids, DistanceType.L2)
    slots = index.add(points, new_ids)                 # reuse_empty=False as in the reference
    index.delete(old_ids)                              # the slots are Empty at once
    I, D = index.search(queries, 100)                  # external ids (uint64), float32 distances

Backed by ``svsb200_dynamic_flat_*`` in ``libsvsb200.so``: the Flat index's exact search (tensor cores for k <= 121, the
exact scan otherwise) over the Valid slots only.  Mutations must not run concurrently with searches of the same index.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .vamana import _DTYPE_CODE, DistanceType


class DynamicFlat(_lib._Slots):
    """``svs.DynamicFlat`` on one CUDA device: float32 / float16 / int8 / uint8 rows, L2 / MIP / cosine.  A delete
    (``delete_entries``, dynamic_flat.h:292-307) empties the slots at once."""

    _ABI = "svsb200_dynamic_flat"

    @classmethod
    def build(cls, data, ids, distance_type: DistanceType = DistanceType.L2, num_threads: int = 1,
              device: int = 0) -> "DynamicFlat":
        """``svs.DynamicFlat.build(data, ids, distance_type, num_threads)``: one external id per row of ``data``.  An
        empty ``data`` ([0, dim]) makes an empty index to be filled with :meth:`add`."""
        data = data.load() if hasattr(data, "load") else data
        data = np.ascontiguousarray(data)
        ids = np.ascontiguousarray(np.atleast_1d(ids), dtype=np.uint64)
        if data.ndim != 2:
            raise ValueError("Expected points to have 2 dimensions!")
        if ids.ndim != 1:
            raise ValueError("Expected ids to have 1 dimension!")
        if data.shape[0] != len(ids):
            raise ValueError("Expected IDs to be the same length as the number of rows in points!")
        if data.dtype not in _DTYPE_CODE:
            raise TypeError(f"unsupported data type {data.dtype}")
        self = cls.__new__(cls)
        self._lib = _lib.lib()
        self._distance = DistanceType(distance_type)
        self._num_threads = int(num_threads)
        self._dtype = data.dtype
        handle = C.c_void_p()
        _lib.check(self._lib.svsb200_dynamic_flat_create(data.ctypes.data, _DTYPE_CODE[data.dtype], data.shape[0],
                                                          data.shape[1], int(self._distance), ids.ctypes.data,
                                                          int(device), C.byref(handle)))
        self._h = handle
        return self

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._lib.svsb200_dynamic_flat_destroy(h)
            self._h = None

    @property
    def size(self) -> int:
        """Valid rows."""
        return self._lib.svsb200_dynamic_flat_size(self._h)

    @property
    def num_slots(self) -> int:
        """Slots, Valid or Empty."""
        return self._lib.svsb200_dynamic_flat_num_slots(self._h)

    @property
    def dimensions(self) -> int:
        return self._lib.svsb200_dynamic_flat_dimensions(self._h)

    @property
    def device_bytes(self) -> int:
        """Device memory held by the rows, statuses and external ids of the allocated slots."""
        return self._lib.svsb200_dynamic_flat_device_bytes(self._h)

    @property
    def num_threads(self) -> int:
        """Kept for interface parity: the reference's thread pool is replaced by the grid."""
        return self._num_threads

    @num_threads.setter
    def num_threads(self, n: int):
        self._num_threads = int(n)

    def add(self, points, ids, reuse_empty: bool = False) -> np.ndarray:
        """``add_points`` (dynamic_flat.h:214-276): rows of the index's dtype with new external ids.  Empty slots are
        used first (from slot 0 with ``reuse_empty``, else from the first slot past the last add), then the index
        grows.  Fails without changing anything on a repeated, present or reserved id.  Returns the slots used."""
        return self._add(points, ids, reuse_empty)

    def consolidate(self) -> None:
        """No-op, as in the reference: deletion is direct."""

    def compact(self, batchsize: int = 1000) -> None:
        """``compact`` (dynamic_flat.h:335-367): the Valid slots move, in order, to the front.  ``batchsize`` only
        tunes the reference's copy and is ignored."""
        _lib.check(self._lib.svsb200_dynamic_flat_compact(self._h))

    def export(self):
        """(status uint8 (0 Empty, 1 Valid), external ids (2^64 - 1 where Empty)) over every slot."""
        n = self.num_slots
        status = np.empty(n, dtype=np.uint8)
        ids = np.empty(n, dtype=np.uint64)
        _lib.check(self._lib.svsb200_dynamic_flat_export(self._h, status.ctypes.data, ids.ctypes.data))
        return status, ids

    def search(self, queries: np.ndarray, n_neighbors: int):
        """``svs.DynamicFlat.search(queries, n_neighbors)`` -> (external ids uint64 [nq,k], distances float32 [nq,k]):
        the exact top k over the Valid rows, ties by slot; short rows padded with 2^64 - 1 and +-inf."""
        q = np.ascontiguousarray(queries)
        if q.ndim != 2 or q.shape[1] != self.dimensions:
            raise ValueError(f"queries must be [nq, {self.dimensions}]")
        if q.dtype not in _DTYPE_CODE:
            raise TypeError(f"unsupported query type {q.dtype}")
        nq, k = q.shape[0], int(n_neighbors)
        ids = np.empty((nq, k), dtype=np.uint64)
        dists = np.empty((nq, k), dtype=np.float32)
        _lib.check(self._lib.svsb200_dynamic_flat_search(self._h, q.ctypes.data, _DTYPE_CODE[q.dtype], nq, k,
                                                         ids.ctypes.data, dists.ctypes.data))
        return ids, dists

    def search_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_ids: int, d_dists: int,
                      stream: int = 0) -> int:
        """Device-buffer form (raw pointers, e.g. ``tensor.data_ptr()``; ids uint64); returns how many queries ran on
        the exact scan."""
        fb = C.c_uint32()
        _lib.check(self._lib.svsb200_dynamic_flat_search_device(self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq,
                                                                int(n_neighbors), d_ids, d_dists, stream or None,
                                                                C.byref(fb)))
        return int(fb.value)

    def search_filtered(self, queries: np.ndarray, n_neighbors: int, allowed: np.ndarray, with_counts: bool = False):
        """``search`` with a predicate over the data index (dynamic_flat.h:513-573): ``allowed`` is a boolean mask over
        the slots, in :meth:`export` order; Empty slots' entries are ignored.  Returns (external ids, distances, found
        per query = min(k, allowed Valid slots)); ties by slot, short rows padded with 2^64 - 1 / +inf for every
        metric.  ``with_counts`` adds the number of allowed Valid slots."""
        return _lib._flat_search_filtered(self._lib.svsb200_dynamic_flat_search_filtered, self._h, self.dimensions,
                                          queries, n_neighbors, _lib._bitmap(allowed, self.num_slots), with_counts)

    def search_filtered_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_bitmap: int,
                               d_ids: int, d_dists: int, stream: int = 0) -> int:
        """Device-buffer form of :meth:`search_filtered` (raw pointers; the uint32 bitmap has (num_slots + 31) / 32
        words, bit i = slot i); returns how many queries ran on a scan.  A mutation may follow it at once."""
        fb = C.c_uint32()
        _lib.check(self._lib.svsb200_dynamic_flat_search_filtered_device(
            self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq, int(n_neighbors), d_bitmap, d_ids, d_dists,
            stream or None, None, C.byref(fb)))
        return int(fb.value)
