"""IVF index on the GPU, mirroring the reference's ``svs.IVF`` and ``svs.Clustering`` (bindings/python/src/ivf.cpp):

    clustering = Clustering.build(IVFBuildParameters(num_centroids=1024), data, DistanceType.L2)
    index = IVF.assemble_from_clustering(clustering, data, DistanceType.L2)
    index.search_parameters = IVFSearchParameters(n_probes=16)
    I, D = index.search(queries, 10)                   # numpy (nq, k) uint64 / float32

Scalar-quantised rows (the reference's ``StorageKind::SQI8`` and its uint8 twin) take four times less device memory:

    codes, scale, bias = sq_compress(data)             # int8 codes, one global scale and bias
    index = IVF.assemble_from_clustering(clustering, codes, DistanceType.L2, sq=(scale, bias))

Backed by ``svsb200_ivf_*`` of ``libsvsb200.so``.  The k-means is the reference's flat k-means made deterministic (an own
documented random sequence, float32 sums in row order), so ``is_hierarchical`` defaults to False here and True is
refused.  A search returns the exact top k over the probed clusters, bit for bit the distances of the exact scan.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib
from ._lib import _bitmap
from .vamana import _DTYPE_CODE, DistanceType


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


def _rows(data) -> np.ndarray:
    data = data.load() if hasattr(data, "load") else data
    data = np.ascontiguousarray(data)
    if data.ndim != 2:
        raise ValueError("data must be a 2-D array")
    if data.dtype not in _DTYPE_CODE:
        raise TypeError(f"unsupported data type {data.dtype}")
    return data


def sq_compress(data, dtype=np.int8, device: int = 0):
    """``SQDataset<int8_t / uint8_t>::compress`` on the GPU (``svsb200_sq_compress``): float32 rows [n, dim] ->
    (codes [n, dim] of ``dtype``, scale, bias).  NaN, infinite and constant data are refused."""
    x = np.ascontiguousarray(data.load() if hasattr(data, "load") else data)
    if x.ndim != 2:
        raise ValueError("data must be a 2-D array")
    if x.dtype != np.float32:
        raise TypeError(f"sq_compress takes float32 rows, got {x.dtype}")
    dtype = np.dtype(dtype)
    if dtype not in (np.dtype(np.int8), np.dtype(np.uint8)):
        raise TypeError(f"SQ codes are int8 or uint8, got {dtype}")
    codes = np.empty(x.shape, dtype=dtype)
    scale, bias = C.c_float(), C.c_float()
    _lib.check(_lib.lib().svsb200_sq_compress(x.ctypes.data, x.shape[0], x.shape[1], _DTYPE_CODE[dtype], int(device),
                                              codes.ctypes.data, C.byref(scale), C.byref(bias)))
    return codes, float(np.float32(scale.value)), float(np.float32(bias.value))


def _search_filtered(fn, h, dims: int, queries, n_neighbors: int, n_probes: int, bitmap: np.ndarray, with_counts: bool):
    """The host form of both indexes' filtered searches."""
    q = np.ascontiguousarray(queries)
    if q.ndim != 2 or q.shape[1] != dims:
        raise ValueError(f"queries must be [nq, {dims}]")
    if q.dtype not in _DTYPE_CODE:
        raise TypeError(f"unsupported query type {q.dtype}")
    nq, k = q.shape[0], int(n_neighbors)
    ids = np.empty((nq, k), dtype=np.uint64)
    dists = np.empty((nq, k), dtype=np.float32)
    probes, allowed, rows = (np.empty(nq, dtype=np.uint32) for _ in range(3))
    _lib.check(fn(h, q.ctypes.data, _DTYPE_CODE[q.dtype], nq, k, n_probes, bitmap.ctypes.data, ids.ctypes.data,
                  dists.ctypes.data, probes.ctypes.data, allowed.ctypes.data, rows.ctypes.data))
    found = np.minimum(allowed, np.uint32(k))
    if with_counts:
        return ids, dists, found, (probes, allowed, rows)
    return ids, dists, found


def _sq_codes(data, sq) -> np.ndarray:
    """The codes of an SQ ``assemble_from_clustering``: int8 / uint8 rows."""
    x = np.ascontiguousarray(data.load() if hasattr(data, "load") else data)
    if x.ndim != 2:
        raise ValueError("data must be a 2-D array")
    if x.dtype not in (np.dtype(np.int8), np.dtype(np.uint8)):
        raise TypeError(f"with sq=(scale, bias) the data are int8 or uint8 codes, got {x.dtype}")
    if len(sq) != 2:
        raise ValueError("sq must be (scale, bias)")
    return x


class Clustering:
    """``svs.Clustering``: centroids float32 [C, dim] and one cluster per data row (uint32 [n])."""

    def __init__(self, centroids, assignments=None):
        self.centroids = np.ascontiguousarray(centroids, dtype=np.float32)
        if self.centroids.ndim != 2:
            raise ValueError("centroids must be [C, dim]")
        self.assignments = None if assignments is None else np.ascontiguousarray(assignments, dtype=np.uint32)

    @property
    def num_clusters(self) -> int:
        return self.centroids.shape[0]

    @staticmethod
    def build(build_parameters: IVFBuildParameters, data, distance: DistanceType = DistanceType.L2,
              device: int = 0) -> "Clustering":
        """``svs.Clustering.build``: the flat k-means on the GPU (``svsb200_ivf_cluster``)."""
        x = _rows(data)
        bp = build_parameters
        n, dim = x.shape
        centroids = np.empty((int(bp.num_centroids), dim), dtype=np.float32)
        assignments = np.empty(n, dtype=np.uint32)
        _lib.check(_lib.lib().svsb200_ivf_cluster(
            x.ctypes.data, _DTYPE_CODE[x.dtype], n, dim, int(DistanceType(distance)), int(bp.num_centroids),
            int(bp.minibatch_size), int(bp.num_iterations), int(bool(bp.is_hierarchical)), float(bp.training_fraction),
            int(bp.seed), int(device), centroids.ctypes.data, assignments.ctypes.data))
        return Clustering(centroids, assignments)


class IVF:
    """``svs.IVF`` on one CUDA device."""

    def __init__(self, handle, lib, distance: DistanceType):
        self._h, self._lib, self._distance = handle, lib, distance
        self.search_parameters = IVFSearchParameters()

    @staticmethod
    def assemble_from_clustering(clustering: Clustering, data, distance: DistanceType = DistanceType.L2,
                                 device: int = 0, sq: tuple | None = None) -> "IVF":
        """``svs.IVF.assemble_from_clustering``: the rows grouped as the clustering says (a clustering without
        assignments puts every row in its nearest cluster).  ``sq=(scale, bias)`` marks ``data`` as int8 / uint8 SQ
        codes (see :func:`sq_compress`); the clustering must then carry assignments."""
        x = _rows(data) if sq is None else _sq_codes(data, sq)
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

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._lib.svsb200_ivf_destroy(h)
            self._h = None

    @property
    def size(self) -> int:
        return self._lib.svsb200_ivf_size(self._h)

    @property
    def dimensions(self) -> int:
        return self._lib.svsb200_ivf_dimensions(self._h)

    @property
    def num_clusters(self) -> int:
        return self._lib.svsb200_ivf_num_clusters(self._h)

    @property
    def device_bytes(self) -> int:
        return self._lib.svsb200_ivf_device_bytes(self._h)

    @property
    def cluster_sizes(self) -> np.ndarray:
        out = np.empty(self.num_clusters, dtype=np.uint32)
        _lib.check(self._lib.svsb200_ivf_cluster_sizes(self._h, out.ctypes.data))
        return out

    @property
    def centroids(self) -> np.ndarray:
        out = np.empty((self.num_clusters, self.dimensions), dtype=np.float32)
        _lib.check(self._lib.svsb200_ivf_centroids(self._h, out.ctypes.data))
        return out

    def _n_probes(self) -> int:
        sp = self.search_parameters
        if not sp.k_reorder >= 1.0:
            raise ValueError(f"k_reorder must be at least 1, got {sp.k_reorder}")
        return int(sp.n_probes)

    def search(self, queries: np.ndarray, n_neighbors: int):
        """``svs.IVF.search(queries, n_neighbors)`` -> (ids uint64 [nq,k], distances float32 [nq,k])."""
        n_probes = self._n_probes()
        q = np.ascontiguousarray(queries)
        if q.ndim != 2 or q.shape[1] != self.dimensions:
            raise ValueError(f"queries must be [nq, {self.dimensions}]")
        if q.dtype not in _DTYPE_CODE:
            raise TypeError(f"unsupported query type {q.dtype}")
        nq, k = q.shape[0], int(n_neighbors)
        ids = np.empty((nq, k), dtype=np.uint64)
        dists = np.empty((nq, k), dtype=np.float32)
        _lib.check(self._lib.svsb200_ivf_search(self._h, q.ctypes.data, _DTYPE_CODE[q.dtype], nq, k, n_probes,
                                                ids.ctypes.data, dists.ctypes.data))
        return ids, dists

    def search_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_ids: int, d_dists: int,
                      stream: int = 0) -> None:
        """Device-buffer form (raw pointers, e.g. ``tensor.data_ptr()``; ids uint64), enqueued on ``stream``."""
        n_probes = self._n_probes()
        _lib.check(self._lib.svsb200_ivf_search_device(self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq,
                                                       int(n_neighbors), n_probes, d_ids, d_dists, stream or None))

    def search_filtered(self, queries: np.ndarray, n_neighbors: int, allowed: np.ndarray, with_counts: bool = False):
        """``svs::runtime::IVFIndex::search(..., IDFilter*)``: ``allowed`` is a boolean mask over the ids.  Each query
        probes ``search_parameters.n_probes`` clusters, four times more while they hold fewer than k allowed rows (at
        most min(C, 1024)), and gets the exact top k over the allowed rows of those clusters.  Returns (ids uint64,
        distances, found per query); short rows are padded with all-ones / +inf for every metric.  ``with_counts``
        adds (probes used, allowed rows, rows) of the probed clusters per query."""
        return _search_filtered(self._lib.svsb200_ivf_search_filtered, self._h, self.dimensions, queries, n_neighbors,
                                self._n_probes(), _bitmap(allowed, self.size), with_counts)

    def search_filtered_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_bitmap: int,
                               d_ids: int, d_dists: int, d_probes: int = 0, d_allowed: int = 0, d_rows: int = 0,
                               stream: int = 0) -> None:
        """Device-buffer form of :meth:`search_filtered`: the uint32 bitmap ((size + 31) / 32 words, bit i = id i) and
        the outputs are raw device pointers (the per-query uint32 outputs may be 0), enqueued on ``stream`` apart from
        the probes and the growth decisions."""
        _lib.check(self._lib.svsb200_ivf_search_filtered_device(
            self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq, int(n_neighbors), self._n_probes(), d_bitmap, d_ids,
            d_dists, d_probes or None, d_allowed or None, d_rows or None, stream or None))
