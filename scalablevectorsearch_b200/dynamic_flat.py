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
from ._lib import _DTYPE_CODE
from .flat import _FlatSearch
from .vamana import DistanceType


class DynamicFlat(_lib._Slots, _FlatSearch):
    """``svs.DynamicFlat`` on one CUDA device: float32 / float16 / int8 / uint8 rows, L2 / MIP / cosine.  A delete
    (``delete_entries``, dynamic_flat.h:292-307) empties the slots at once.  ``size`` counts the Valid rows,
    ``num_slots`` the slots, Valid or Empty, and ``device_bytes`` the rows, statuses and external ids of the allocated
    slots.  A search returns external ids: the exact top k over the Valid rows, ties by slot; short rows are padded
    with 2^64 - 1 and +-inf.  The filtered search (dynamic_flat.h:513-573) takes a boolean mask over the SLOTS, in
    :meth:`export` order, and ignores the Empty slots' entries; its found and allowed counts are of allowed Valid
    slots, and the device form's bitmap has (num_slots + 31) / 32 words, bit i = slot i (a mutation may follow it at
    once)."""

    _ABI = _PREFIX = "svsb200_dynamic_flat"
    _MASK = "num_slots"

    @classmethod
    def build(cls, data, ids, distance_type: DistanceType = DistanceType.L2, num_threads: int = 1,
              device: int = 0) -> "DynamicFlat":
        """``svs.DynamicFlat.build(data, ids, distance_type, num_threads)``: one external id per row of ``data``.  An
        empty ``data`` ([0, dim]) makes an empty index to be filled with :meth:`add`."""
        data = _lib._rows(data, ndim_error="Expected points to have 2 dimensions!")
        ids = np.ascontiguousarray(np.atleast_1d(ids), dtype=np.uint64)
        if ids.ndim != 1:
            raise ValueError("Expected ids to have 1 dimension!")
        if data.shape[0] != len(ids):
            raise ValueError("Expected IDs to be the same length as the number of rows in points!")
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

    @property
    def num_slots(self) -> int:
        return self._lib.svsb200_dynamic_flat_num_slots(self._h)

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
