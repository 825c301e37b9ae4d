"""IVF index on the GPU, mirroring the reference's ``svs.IVF`` and ``svs.Clustering`` (bindings/python/src/ivf.cpp):

    clustering = Clustering.build(IVFBuildParameters(num_centroids=1024), data, DistanceType.L2)
    index = IVF.assemble_from_clustering(clustering, data, DistanceType.L2)
    index.search_parameters = IVFSearchParameters(n_probes=16)
    I, D = index.search(queries, 10)                   # numpy (nq, k) uint64 / float32

Scalar-quantised rows (the reference's ``StorageKind::SQI8`` and its uint8 twin) take four times less device memory:

    codes, scale, bias = sq_compress(data)             # int8 codes, one global scale and bias
    index = IVF.assemble_from_clustering(clustering, codes, DistanceType.L2, sq=(scale, bias))

The reference's default, hierarchical k-means, is a method of its own here (``is_hierarchical`` is not read by it):

    clustering = Clustering.build_hierarchical(IVFBuildParameters(num_centroids=16384), data, DistanceType.L2)

Backed by ``svsb200_ivf_*`` of ``libsvsb200.so``.  Both k-means are the reference's made deterministic (an own
documented random sequence, float32 sums in row order).  ``Clustering.build`` is the flat k-means, so
``is_hierarchical`` defaults to False here and True is refused by it.  A search returns the exact top k over the probed
clusters, bit for bit the distances of the exact scan.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib
from ._lib import _DTYPE_CODE
from .vamana import DistanceType


@dataclass
class IVFBuildParameters:
    """``svs.IVFBuildParameters`` (index/ivf/common.h:70-118); ``is_hierarchical`` defaults to False (see module)."""
    num_centroids: int = 1000
    minibatch_size: int = 10_000
    num_iterations: int = 10
    is_hierarchical: bool = False
    training_fraction: float = 0.1
    hierarchical_level1_clusters: int = 0
    seed: int = 0xC0FFEE


@dataclass
class IVFSearchParameters:
    """``svs.IVFSearchParameters``: clusters probed per query, and ``k_reorder`` (>= 1), which cannot change the top k
    of uncompressed rows (the reference only widens its leaf buffer to k_reorder * k and returns the first k)."""
    n_probes: int = 1
    k_reorder: float = 1.0


def sq_compress(data, dtype=np.int8, device: int = 0):
    """``SQDataset<int8_t / uint8_t>::compress`` on the GPU (``svsb200_sq_compress``): float32 rows [n, dim] ->
    (codes [n, dim] of ``dtype``, scale, bias).  NaN, infinite and constant data are refused."""
    x = _lib._rows(data, (np.float32,), dtype_error="sq_compress takes float32 rows, got {}")
    dtype = np.dtype(dtype)
    if dtype not in (np.dtype(np.int8), np.dtype(np.uint8)):
        raise TypeError(f"SQ codes are int8 or uint8, got {dtype}")
    codes = np.empty(x.shape, dtype=dtype)
    scale, bias = C.c_float(), C.c_float()
    _lib.check(_lib.lib().svsb200_sq_compress(x.ctypes.data, x.shape[0], x.shape[1], _DTYPE_CODE[dtype], int(device),
                                              codes.ctypes.data, C.byref(scale), C.byref(bias)))
    return codes, float(np.float32(scale.value)), float(np.float32(bias.value))


def _index_rows(data, sq) -> np.ndarray:
    """The rows of an ``assemble_from_clustering``: int8 / uint8 SQ codes with ``sq=(scale, bias)``."""
    if sq is None:
        return _lib._rows(data)
    x = _lib._rows(data, (np.int8, np.uint8),
                   dtype_error="with sq=(scale, bias) the data are int8 or uint8 codes, got {}")
    if len(sq) != 2:
        raise ValueError("sq must be (scale, bias)")
    return x


class Clustering:
    """``svs.Clustering``: centroids float32 [C, dim] and one cluster per data row (uint32 [n]); a hierarchical one also
    the level-2 centroids of every level-1 group (uint32 [L1], ``level2_counts``, else None)."""

    def __init__(self, centroids, assignments=None, level2_counts=None):
        self.centroids = np.ascontiguousarray(centroids, dtype=np.float32)
        if self.centroids.ndim != 2:
            raise ValueError("centroids must be [C, dim]")
        self.assignments = None if assignments is None else np.ascontiguousarray(assignments, dtype=np.uint32)
        self.level2_counts = level2_counts

    @property
    def num_clusters(self) -> int:
        return self.centroids.shape[0]

    @staticmethod
    def build(build_parameters: IVFBuildParameters, data, distance: DistanceType = DistanceType.L2,
              device: int = 0) -> "Clustering":
        """``svs.Clustering.build``: the flat k-means on the GPU (``svsb200_ivf_cluster``)."""
        x = _lib._rows(data)
        bp = build_parameters
        n, dim = x.shape
        centroids = np.empty((int(bp.num_centroids), dim), dtype=np.float32)
        assignments = np.empty(n, dtype=np.uint32)
        _lib.check(_lib.lib().svsb200_ivf_cluster(
            x.ctypes.data, _DTYPE_CODE[x.dtype], n, dim, int(DistanceType(distance)), int(bp.num_centroids),
            int(bp.minibatch_size), int(bp.num_iterations), int(bool(bp.is_hierarchical)), float(bp.training_fraction),
            int(bp.seed), int(device), centroids.ctypes.data, assignments.ctypes.data))
        return Clustering(centroids, assignments)

    @staticmethod
    def build_hierarchical(build_parameters: IVFBuildParameters, data, distance: DistanceType = DistanceType.L2,
                           device: int = 0) -> "Clustering":
        """``hierarchical_kmeans_clustering`` on the GPU (``svsb200_ivf_cluster_hierarchical``): a flat k-means of
        ``hierarchical_level1_clusters`` centroids (0: sqrt(num_centroids)), then a k-means inside every level-1 group
        with centroids in proportion to its training rows, all groups trained together.  A row's cluster is the nearest
        centroid of its own level-1 group.  ``is_hierarchical`` is not read.  The level-2 centroids per level-1 group
        are kept as ``level2_counts``."""
        x = _lib._rows(data)
        bp = build_parameters
        n, dim = x.shape
        C = int(bp.num_centroids)
        centroids = np.empty((C, dim), dtype=np.float32)
        assignments = np.empty(n, dtype=np.uint32)
        counts = np.zeros(int(bp.hierarchical_level1_clusters) or int(np.sqrt(float(C))), dtype=np.uint32)
        _lib.check(_lib.lib().svsb200_ivf_cluster_hierarchical(
            x.ctypes.data, _DTYPE_CODE[x.dtype], n, dim, int(DistanceType(distance)), C,
            int(bp.hierarchical_level1_clusters), int(bp.minibatch_size), int(bp.num_iterations),
            float(bp.training_fraction), int(bp.seed), int(device), centroids.ctypes.data, assignments.ctypes.data,
            counts.ctypes.data))
        return Clustering(centroids, assignments, level2_counts=counts)


class _IVFSearch(_lib._Handle):
    """The search forms, probes and cluster accessors of IVF and DynamicIVF over ``{_PREFIX}_*``.  The filter mask has
    one entry per ``_MASK`` (``size`` or ``num_slots``), and the bitmap of the device form (_MASK + 31) / 32 uint32
    words."""

    _MASK = "size"

    @property
    def num_clusters(self) -> int:
        return self._cfn("num_clusters")(self._h)

    @property
    def cluster_sizes(self) -> np.ndarray:
        """Rows per cluster (Valid rows, in a DynamicIVF)."""
        out = np.empty(self.num_clusters, dtype=np.uint32)
        _lib.check(self._cfn("cluster_sizes")(self._h, out.ctypes.data))
        return out

    @property
    def centroids(self) -> np.ndarray:
        out = np.empty((self.num_clusters, self.dimensions), dtype=np.float32)
        _lib.check(self._cfn("centroids")(self._h, out.ctypes.data))
        return out

    def _n_probes(self) -> int:
        sp = self.search_parameters
        if not sp.k_reorder >= 1.0:
            raise ValueError(f"k_reorder must be at least 1, got {sp.k_reorder}")
        return int(sp.n_probes)

    def search(self, queries: np.ndarray, n_neighbors: int):
        """``search(queries, n_neighbors)`` -> (ids uint64 [nq,k], distances float32 [nq,k]): the exact top k over the
        probed clusters."""
        n_probes = self._n_probes()
        q = _lib._queries(queries, self.dimensions)
        return _lib._search(self._cfn("search"), (self._h,), q, n_neighbors, (n_probes,))

    def search_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_ids: int, d_dists: int,
                      stream: int = 0) -> None:
        """Device-buffer form (raw pointers, e.g. ``tensor.data_ptr()``; ids uint64), enqueued on ``stream``."""
        n_probes = self._n_probes()
        _lib.check(self._cfn("search_device")(self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq, int(n_neighbors),
                                              n_probes, d_ids, d_dists, stream or None))

    def search_filtered(self, queries: np.ndarray, n_neighbors: int, allowed: np.ndarray, with_counts: bool = False):
        """``svs::runtime::IVFIndex::search(..., IDFilter*)``: ``allowed`` is a boolean mask (see the class).  Each
        query probes ``search_parameters.n_probes`` clusters, four times more while they hold fewer than k allowed rows
        (at most min(C, 1024)), and gets the exact top k over the allowed rows of those clusters.  Returns (ids uint64,
        distances, found per query); short rows are padded with all-ones / +inf for every metric.  ``with_counts``
        adds (probes used, allowed rows, rows) of the probed clusters per query."""
        dims, n_probes = self.dimensions, self._n_probes()
        bitmap = _lib._bitmap(allowed, getattr(self, self._MASK))
        q = _lib._queries(queries, dims)
        counts = tuple(np.empty(q.shape[0], dtype=np.uint32) for _ in range(3))   # probes, allowed rows, rows
        ids, dists = _lib._search(self._cfn("search_filtered"), (self._h,), q, n_neighbors,
                                  (n_probes, bitmap.ctypes.data), tuple(c.ctypes.data for c in counts))
        found = np.minimum(counts[1], np.uint32(int(n_neighbors)))
        if with_counts:
            return ids, dists, found, counts
        return ids, dists, found

    def search_filtered_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_bitmap: int,
                               d_ids: int, d_dists: int, d_probes: int = 0, d_allowed: int = 0, d_rows: int = 0,
                               stream: int = 0) -> None:
        """Device-buffer form of :meth:`search_filtered`: the uint32 bitmap (see the class) and the outputs are raw
        device pointers (the per-query uint32 outputs may be 0), enqueued on ``stream`` apart from the probes and the
        growth decisions."""
        _lib.check(self._cfn("search_filtered_device")(
            self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq, int(n_neighbors), self._n_probes(), d_bitmap, d_ids,
            d_dists, d_probes or None, d_allowed or None, d_rows or None, stream or None))


class IVF(_IVFSearch):
    """``svs.IVF`` on one CUDA device.  The filter mask of the filtered searches is over the ids: ``size`` entries,
    bit i of the device form's bitmap = id i."""

    _PREFIX = "svsb200_ivf"

    def __init__(self, handle, lib, distance: DistanceType):
        self._h, self._lib, self._distance = handle, lib, distance
        self.search_parameters = IVFSearchParameters()

    @staticmethod
    def assemble_from_clustering(clustering: Clustering, data, distance: DistanceType = DistanceType.L2,
                                 device: int = 0, sq: tuple | None = None) -> "IVF":
        """``svs.IVF.assemble_from_clustering``: the rows grouped as the clustering says (a clustering without
        assignments puts every row in its nearest cluster).  ``sq=(scale, bias)`` marks ``data`` as int8 / uint8 SQ
        codes (see :func:`sq_compress`); the clustering must then carry assignments."""
        x = _index_rows(data, sq)
        cent = clustering.centroids
        if cent.shape[1] != x.shape[1]:
            raise ValueError(f"centroids have {cent.shape[1]} dimensions, data {x.shape[1]}")
        a = clustering.assignments
        if a is not None and a.shape != (x.shape[0],):
            raise ValueError("the clustering has one assignment per data row")
        lib = _lib.lib()
        handle = C.c_void_p()
        if sq is not None:
            _lib.check(lib.svsb200_ivf_create_sq(x.ctypes.data, _DTYPE_CODE[x.dtype], x.shape[0], x.shape[1],
                                                 int(DistanceType(distance)), float(sq[0]), float(sq[1]), cent.ctypes.data,
                                                 cent.shape[0], None if a is None else a.ctypes.data, int(device),
                                                 C.byref(handle)))
            return IVF(handle, lib, DistanceType(distance))
        _lib.check(lib.svsb200_ivf_create(x.ctypes.data, _DTYPE_CODE[x.dtype], x.shape[0], x.shape[1],
                                          int(DistanceType(distance)), cent.ctypes.data, cent.shape[0],
                                          None if a is None else a.ctypes.data, int(device), C.byref(handle)))
        return IVF(handle, lib, DistanceType(distance))
