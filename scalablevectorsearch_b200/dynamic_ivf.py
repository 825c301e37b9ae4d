"""Dynamic IVF index on the GPU, mirroring the reference's ``svs.DynamicIVF`` (bindings/python/src/dynamic_ivf.cpp,
include/svs/index/ivf/dynamic_ivf.h):

    clustering = Clustering.build(IVFBuildParameters(num_centroids=1024), data, DistanceType.L2)
    index = DynamicIVF.assemble_from_clustering(clustering, data, ids, DistanceType.L2)
    slots = index.add(points, new_ids)                 # appended to their nearest clusters
    index.delete(old_ids)                              # tombstones at once
    index.search_parameters = IVFSearchParameters(n_probes=16)
    I, D = index.search(queries, 10)                   # external ids (uint64), float32 distances

Scalar-quantised rows (the reference's ``StorageKind::SQI8`` and its uint8 twin) take four times less device memory.
The index keeps the scale and bias it was assembled with; later adds take float32 rows and encode them with those:

    codes, scale, bias = sq_compress(data)             # int8 codes, one global scale and bias
    index = DynamicIVF.assemble_from_clustering(clustering, codes, ids, DistanceType.L2, sq=(scale, bias))
    index.add(points, new_ids)                         # float32 rows, encoded on the device (values past the range clamp)

Backed by ``svsb200_dynamic_ivf_*`` of ``libsvsb200.so``: the IVF index's exact cluster-probed search over the Valid rows,
ties by slot.  The centroids never move after assembly.  Mutations must not run concurrently with searches of the same
index.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import _DTYPE_CODE
from .ivf import Clustering, IVFSearchParameters, _index_rows, _IVFSearch
from .vamana import DistanceType


class DynamicIVF(_lib._Slots, _IVFSearch):
    """``svs.DynamicIVF`` on one CUDA device: float32 / float16 rows or int8 / uint8 SQ codes, L2 / MIP / cosine.  A
    delete empties the slots at once and leaves tombstones in their clusters.  ``size`` counts the Valid rows,
    ``num_slots`` the slots, Valid or Empty, and ``device_bytes`` the device memory held, the regions that clusters left
    when they grew included until :meth:`compact`.  A search returns external ids: the exact top k over the Valid rows
    of the probed clusters, ties by slot; short rows are padded with 2^64 - 1 and +-inf.  The filtered search is
    :meth:`IVF.search_filtered` over the Valid rows: ``allowed`` is a boolean mask over the SLOTS (``num_slots``
    entries, in the order of :meth:`export`; the device form's bitmap has (num_slots + 31) / 32 words), Empty slots are
    never returned, and ``with_counts`` adds (probes used, allowed rows, Valid rows)."""

    _ABI = _PREFIX = "svsb200_dynamic_ivf"
    _MASK = "num_slots"

    @classmethod
    def assemble_from_clustering(cls, clustering: Clustering, data, ids, distance: DistanceType = DistanceType.L2,
                                 num_threads: int = 1, intra_query_threads: int = 1, device: int = 0,
                                 sq: tuple | None = None) -> "DynamicIVF":
        """``svs.DynamicIVF.assemble_from_clustering``: one external id per row of ``data``, the rows grouped as the
        clustering says (a clustering without assignments puts every row in its nearest cluster).  An empty ``data``
        ([0, dim]) makes an empty index to be filled with :meth:`add`.  ``sq=(scale, bias)`` marks ``data`` as int8 /
        uint8 SQ codes (see :func:`sq_compress`); the clustering must then carry assignments unless ``data`` is empty.
        The thread counts are kept for interface parity only."""
        x = _index_rows(data, sq)
        ids = np.ascontiguousarray(np.atleast_1d(ids), dtype=np.uint64)
        if ids.shape != (x.shape[0],):
            raise ValueError("Expected IDs to be the same length as the number of rows in points!")
        cent = clustering.centroids
        if cent.shape[1] != x.shape[1]:
            raise ValueError(f"centroids have {cent.shape[1]} dimensions, data {x.shape[1]}")
        a = clustering.assignments
        if a is not None and a.shape != (x.shape[0],):
            raise ValueError("the clustering has one assignment per data row")
        self = cls.__new__(cls)
        self._lib = _lib.lib()
        self._distance = DistanceType(distance)
        self._dtype = x.dtype
        self.num_threads, self.intra_query_threads = int(num_threads), int(intra_query_threads)
        self.search_parameters = IVFSearchParameters()
        handle = C.c_void_p()
        a_ptr = None if a is None else a.ctypes.data
        if sq is not None:
            _lib.check(self._lib.svsb200_dynamic_ivf_create_sq(
                x.ctypes.data, _DTYPE_CODE[x.dtype], x.shape[0], x.shape[1], int(self._distance), float(sq[0]),
                float(sq[1]), cent.ctypes.data, cent.shape[0], a_ptr, ids.ctypes.data, int(device), C.byref(handle)))
        else:
            _lib.check(self._lib.svsb200_dynamic_ivf_create(
                x.ctypes.data, _DTYPE_CODE[x.dtype], x.shape[0], x.shape[1], int(self._distance), cent.ctypes.data,
                cent.shape[0], a_ptr, ids.ctypes.data, int(device), C.byref(handle)))
        self._h = handle
        return self

    @property
    def num_slots(self) -> int:
        return self._lib.svsb200_dynamic_ivf_num_slots(self._h)

    def add(self, points, ids, reuse_empty: bool = False) -> np.ndarray:
        """``add_points``: rows with new external ids, each appended to its nearest centroid's cluster.  Without
        ``reuse_empty`` every row takes a new slot at the end; with it, Empty slots from slot 0 come first.  Rows of the
        index's dtype; float32 rows given to a float16 index are rounded to nearest even.  An SQ index takes float32
        rows (finite) and encodes them with its scale and bias.  Fails without changing anything on a repeated, present
        or reserved id.  Returns the slots used."""
        pts = np.ascontiguousarray(points)
        if pts.dtype == np.float32 and self._dtype == np.float16:
            pts = pts.astype(np.float16)
        return self._add(pts, ids, reuse_empty)

    def consolidate(self) -> None:
        """No-op, as in the reference: deletion is direct."""

    def compact(self, batchsize: int = 1_000_000) -> None:
        """``compact``: the Valid slots are renumbered in order and the clusters laid out without tombstones.
        ``batchsize`` only tunes the reference's copy and is ignored."""
        _lib.check(self._lib.svsb200_dynamic_ivf_compact(self._h))

    def export(self):
        """Per slot: (status uint8 (0 Empty, 1 Valid), external id (2^64 - 1 where Empty), cluster uint32 (2^32 - 1
        where Empty))."""
        n = self.num_slots
        status = np.empty(n, dtype=np.uint8)
        ids = np.empty(n, dtype=np.uint64)
        cluster = np.empty(n, dtype=np.uint32)
        _lib.check(self._lib.svsb200_dynamic_ivf_export(self._h, status.ctypes.data, ids.ctypes.data, cluster.ctypes.data))
        return status, ids, cluster
