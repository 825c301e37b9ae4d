"""Host-side mirror of the reference's Vamana search interface, backed by ``libsvsb200.so``.

Names, argument meaning and error behaviour follow the reference's Python binding of
``svs::Vamana`` (``/root/reference/bindings/python/src/vamana.cpp:340-348,409-451``,
``include/svs/python/manager.h:34-58,85-142``, ``src/vamana_common.cpp:88-160``):

    index = Vamana(config_path, GraphLoader(dir), VectorDataLoader(path, DataType.float32),
                   distance=DistanceType.L2)
    index.search_window_size = 128
    I, D = index.search(queries, 10)          # numpy (nq, k) uint64 / float32

Everything that is not batch search (build, save, reconstruct, calibrate ...) stays on the
reference's CPU code and is out of scope here (SURVEY.md §8).
"""
from __future__ import annotations

import ctypes as C
import enum
import os
from dataclasses import dataclass, field

import numpy as np

from . import _lib, io
from ._lib import _DTYPE_CODE


class DistanceType(enum.IntEnum):
    """``svs.DistanceType`` (core/distance.h:41-60)."""
    L2 = 0
    MIP = 1
    Cosine = 2


class DataType(enum.Enum):
    """``svs.DataType`` restricted to the element types the search path supports."""
    float32 = np.dtype(np.float32)
    float16 = np.dtype(np.float16)
    int8 = np.dtype(np.int8)
    uint8 = np.dtype(np.uint8)


_STORAGE_PLAIN, _STORAGE_SQ, _STORAGE_LVQ8 = 0, 1, 2


@dataclass
class SearchBufferConfig:
    """``svs.SearchBufferConfig`` (index/vamana/search_buffer.h:39-96)."""
    search_window_size: int = 0
    search_buffer_capacity: int | None = None

    def __post_init__(self):
        if self.search_buffer_capacity is None:
            self.search_buffer_capacity = self.search_window_size
        if self.search_window_size > self.search_buffer_capacity:
            raise ValueError(
                f"Improper configuration for search buffer! Effective size ({self.search_window_size}) "
                f"cannot be less than capacity ({self.search_buffer_capacity}).")


@dataclass
class VamanaSearchParameters:
    """``svs.VamanaSearchParameters`` (index/vamana/search_params.h:27-128).

    ``prefetch_*`` are accepted for interface parity; the GPU hides latency with warps in
    flight instead of software prefetch (lib/prefetch.h)."""
    buffer_config: SearchBufferConfig = field(default_factory=SearchBufferConfig)
    search_buffer_visited_set: bool = False
    prefetch_lookahead: int = 4
    prefetch_step: int = 1


@dataclass
class VectorDataLoader:
    """``svs.VectorDataLoader``: a ``.svs`` / ``.fvecs`` style file plus its element type."""
    path: str
    data_type: DataType = DataType.float32
    dims: int = 0

    def load(self) -> np.ndarray:
        dt = self.data_type.value
        ext = os.path.splitext(self.path)[1]
        if os.path.isdir(self.path):
            path = os.path.join(self.path, "data_0.svs") if os.path.exists(os.path.join(self.path, "data_0.svs")) \
                else self.path
            return io.read_svs(path, dt)
        if ext in (".fvecs", ".ivecs", ".bvecs", ".hvecs"):
            return io.read_vecs(self.path, dt)
        return io.read_svs(self.path, dt)


@dataclass
class GraphLoader:
    """``svs.GraphLoader``: a native graph file (or the directory holding ``graph_0.svs``)."""
    path: str

    def load(self) -> np.ndarray:
        path = self.path
        if os.path.isdir(path):
            path = os.path.join(path, "graph_0.svs")
        return io.read_graph(path)


def toml_get(path: str, dotted_key: str) -> str:
    """Raw text of ``table.key`` in a TOML file, read by the library's own subset parser (``svsb200_toml_get``)."""
    buf = C.create_string_buffer(4096)
    _lib.check(_lib.lib().svsb200_toml_get(os.fsencode(path), dotted_key.encode(), buf, len(buf)))
    return buf.value.decode()


def _read_entry_point(config_path: str) -> int:
    """``entry_point`` of a ``vamana_index_parameters`` TOML (index/vamana/index.h:53-178)."""
    path = config_path
    if os.path.isdir(path):
        path = os.path.join(path, "svs_config.toml")
    return int(toml_get(path, "object.entry_point"))


def lvq8_compress(data: np.ndarray, mean: np.ndarray | None = None, device: int = 0):
    """LVQ-8 encode float32 vectors on the GPU (own specification, DESIGN.md §10; stands where the
    reference's closed ``LVQDataset<8>::compress(data, threadpool, padding)`` would).
    Returns ``(rows uint8 [n, stride], mean float32 [dim])``.  Raises :class:`Svsb200Error`, naming the first offending
    row, when a value minus the mean is not finite or a row's delta or lower bound does not fit in float16."""
    data = np.ascontiguousarray(data, dtype=np.float32)
    if mean is None:
        mean = data.mean(axis=0, dtype=np.float64).astype(np.float32)
    mean = np.ascontiguousarray(mean, dtype=np.float32)
    lib = _lib.lib()
    stride = lib.svsb200_lvq8_row_stride(data.shape[1])
    rows = np.empty((data.shape[0], stride), dtype=np.uint8)
    _lib.check(lib.svsb200_lvq8_compress(data.ctypes.data, data.shape[0], data.shape[1], mean.ctypes.data,
                                         rows.ctypes.data, int(device)))
    return rows, mean


@dataclass
class VamanaBuildParameters:
    """``svs.VamanaBuildParameters`` (index/vamana/build_params.h; defaults lib/preprocessor.h:179-183,
    index/vamana/index.h:1079-1095): 0 / None select the reference's defaults."""
    alpha: float = 0.0
    graph_max_degree: int = 32
    window_size: int = 200
    max_candidate_pool_size: int = 0
    prune_to: int = 0
    use_full_search_history: bool = True


def build_graph(data: np.ndarray, distance: "DistanceType", parameters: VamanaBuildParameters, device: int = 0,
                sq: tuple | None = None):
    """Vamana graph construction on the GPU (``svsb200_build_vamana``; stands where ``svs.Vamana.build`` /
    ``index::vamana::auto_build`` runs the reference's CPU builder).  Returns ``(graph uint32[n][R+1] in the
    reference's degree-first layout, entry_point)``.  int8 / uint8 rows are built with exact integer distances, as the
    reference builds ``SimpleData<int8_t / uint8_t>``.  ``sq=(scale, bias)`` marks ``data`` as scalar-quantised
    int8 / uint8 codes (from :func:`scalablevectorsearch_b200.ivf.sq_compress`), built as the reference builds
    ``SQDataset`` (``svsb200_build_vamana_sq``)."""
    data = _lib._rows(data, ndim_error=None,
                      dtype_error="build_graph takes a 2-D float32 / float16 / int8 / uint8 array")
    if sq is not None and data.dtype not in (np.int8, np.uint8):
        raise TypeError("SQ codes are int8 or uint8")
    if not parameters.use_full_search_history:
        raise ValueError("the GPU builder always keeps the full search history (the reference's default)")
    lib = _lib.lib()
    n, R = data.shape[0], int(parameters.graph_max_degree)
    graph = np.empty((n, R + 1), dtype=np.uint32)
    ep = C.c_uint32()
    tail = (float(parameters.alpha), R, int(parameters.window_size), int(parameters.max_candidate_pool_size),
            int(parameters.prune_to), int(device), graph.ctypes.data, C.byref(ep))
    if sq is None:
        _lib.check(lib.svsb200_build_vamana(data.ctypes.data, _DTYPE_CODE[data.dtype], n, data.shape[1], 0, int(distance),
                                            *tail))
    else:
        _lib.check(lib.svsb200_build_vamana_sq(data.ctypes.data, _DTYPE_CODE[data.dtype], n, data.shape[1], int(distance),
                                               float(sq[0]), float(sq[1]), *tail))
    return graph, int(ep.value)


class Vamana(_lib._Handle):
    """GPU-backed static Vamana index exposing the reference's search surface."""

    _PREFIX = "svsb200_index"

    @classmethod
    def build(cls, parameters: VamanaBuildParameters, data: np.ndarray, distance: "DistanceType" = None, device=0,
              num_threads: int = 1, sq: tuple | None = None) -> "Vamana":
        """``svs.Vamana.build(parameters, data_loader, distance_type, num_threads)``
        (bindings/python/src/vamana.cpp:171-240): graph construction and the resulting index, all on the GPU.
        ``sq=(scale, bias)`` as in :meth:`from_arrays`: ``data`` are SQ codes, and the result is an SQ index."""
        distance = DistanceType.L2 if distance is None else distance
        dev0 = device[0] if isinstance(device, (list, tuple)) else device
        graph, ep = build_graph(data, distance, parameters, dev0, sq=sq)
        self = cls.from_arrays(data, graph, ep, distance, device=device, sq=sq, num_threads=num_threads)
        self.build_parameters = parameters
        return self

    def __init__(self, config_path, graph_loader, data_loader, distance: DistanceType = DistanceType.L2,
                 query_type: DataType = DataType.float32, enforce_dims: bool = False, num_threads: int = 1,
                 device: int = 0):
        self._query_type = query_type
        self._enforce_dims = bool(enforce_dims)
        if isinstance(graph_loader, GraphLoader) and isinstance(data_loader, VectorDataLoader):
            # files: streamed straight into HBM by the library (svsb200_index_assemble), no host copy
            self._lib = _lib.lib()
            self._distance = DistanceType(distance)
            self._dtype = data_loader.data_type.value
            self._params = VamanaSearchParameters()
            self._num_threads = int(num_threads)
            devices = [int(d) for d in device] if isinstance(device, (list, tuple)) else [int(device)]
            handle = C.c_void_p()
            _lib.check(self._lib.svsb200_index_assemble(
                os.fsencode(str(config_path)), os.fsencode(graph_loader.path), os.fsencode(data_loader.path),
                _DTYPE_CODE[self._dtype], int(data_loader.dims), int(self._distance), (C.c_int * len(devices))(*devices),
                len(devices), C.byref(handle)))
            self._h = handle
            # index.apply(config): the saved search parameters become the defaults (index.h:1047-1048)
            w, c = self.get_option("config_search_window_size"), self.get_option("config_search_buffer_capacity")
            self._params.buffer_config = SearchBufferConfig(w, max(w, c))
            self._params.search_buffer_visited_set = bool(self.get_option("config_search_buffer_visited_set"))
            return
        graph = graph_loader.load() if hasattr(graph_loader, "load") else np.asarray(graph_loader)
        data = data_loader.load() if hasattr(data_loader, "load") else np.asarray(data_loader)
        if getattr(data_loader, "dims", 0) and data.shape[1] != data_loader.dims:
            raise ValueError(f"the data file holds {data.shape[1]}-dimensional vectors, {data_loader.dims} expected")
        self._init(data, graph, _read_entry_point(config_path), distance, device, num_threads)

    @classmethod
    def from_arrays(cls, data: np.ndarray, graph: np.ndarray, entry_point: int,
                    distance: DistanceType = DistanceType.L2, device=0, sq: tuple | None = None,
                    num_threads: int = 1, lvq8: tuple | None = None) -> "Vamana":
        """Assemble from in-memory parts: ``VamanaIndex(graph, data, entry_point, distance, threads)``
        (index/vamana/index.h:364-378).  ``graph`` is ``uint32[n][max_degree+1]``, degree first.
        ``sq=(scale, bias)`` marks ``data`` as scalar-quantised int8/uint8 codes;
        ``lvq8=(dim, mean)`` marks ``data`` as LVQ-8 rows from :func:`lvq8_compress`.
        ``device`` is one CUDA ordinal or a list of them: a list replicates the index and every batch is
        split over the devices with the reference's ``threads::balance`` (one process, no collective)."""
        self = cls.__new__(cls)
        self._init(data, graph, entry_point, distance, device, num_threads, sq, lvq8)
        return self

    def _init(self, data, graph, entry_point, distance, device, num_threads, sq=None, lvq8=None):
        graph = np.ascontiguousarray(graph, dtype=np.uint32)
        if graph.ndim != 2:
            raise ValueError("data and graph must be 2-D")
        data = _lib._rows(data, ndim_error="data and graph must be 2-D")
        if graph.shape[0] != data.shape[0]:
            raise ValueError("Wrong sizes!")  # index/vamana/index.h:417-419
        self._lib = _lib.lib()
        self._distance = DistanceType(distance)
        self._dtype = data.dtype
        self._params = VamanaSearchParameters()
        self._num_threads = int(num_threads)
        handle = C.c_void_p()
        aux = None
        storage = _STORAGE_PLAIN
        dim, stride = data.shape[1], 0
        if sq is not None:
            aux = (C.c_float * 2)(float(sq[0]), float(sq[1]))
            storage = _STORAGE_SQ
        if lvq8 is not None:
            dim, mean = int(lvq8[0]), np.ascontiguousarray(lvq8[1], dtype=np.float32)
            aux = (C.c_float * dim)(*mean.tolist())
            storage, stride = _STORAGE_LVQ8, data.shape[1]
        devices = [int(d) for d in device] if isinstance(device, (list, tuple)) else [int(device)]
        dev_arr = (C.c_int * len(devices))(*devices)
        _lib.check(self._lib.svsb200_index_create_multi(
            data.ctypes.data, _DTYPE_CODE[data.dtype], data.shape[0], dim, stride, graph.ctypes.data,
            graph.shape[1], int(entry_point), int(self._distance), storage,
            C.cast(aux, C.c_void_p) if aux is not None else None, dev_arr, len(devices), C.byref(handle)))
        self._h = handle

    # ---- properties (bindings/python/include/svs/python/manager.h:85-110) -------------
    @property
    def graph_max_degree(self) -> int:
        return self._lib.svsb200_index_max_degree(self._h)

    @property
    def search_parameters(self) -> VamanaSearchParameters:
        return self._params

    @search_parameters.setter
    def search_parameters(self, p: VamanaSearchParameters):
        self._params = p

    @property
    def search_window_size(self) -> int:
        return self._params.buffer_config.search_window_size

    @search_window_size.setter
    def search_window_size(self, w: int):
        # orchestrators/vamana.h set_search_window_size: window == capacity
        self._params.buffer_config = SearchBufferConfig(int(w))

    # ---- search ------------------------------------------------------------------------
    @property
    def num_devices(self) -> int:
        return self._lib.svsb200_index_num_devices(self._h)

    def search(self, queries: np.ndarray, n_neighbors: int, cancel=None):
        """``svs.Vamana.search(queries, n_neighbors)`` -> (ids uint64 [nq,k], distances float32 [nq,k]).
        ``cancel`` is an optional zero-argument predicate, polled while the batch runs (the reference's
        ``lib::DefaultPredicate`` of index/vamana/index.h:568): once it returns True the kernels stop at their
        next query / hop boundary and the rows of unfinished queries are unspecified."""
        q = np.ascontiguousarray(queries)
        if q.ndim != 2:
            raise ValueError("queries must be a 2-D array")
        if q.dtype not in _DTYPE_CODE:
            raise TypeError(f"unsupported query type {q.dtype}")
        qt = getattr(self, "_query_type", None)
        if qt is not None and q.dtype != qt.value:
            # the reference compiles one specialisation per declared query type (bindings/python/src/vamana.cpp:88-160)
            raise TypeError(f"this index was assembled for {qt.name} queries, got {q.dtype}")
        if q.shape[1] != self.dimensions:
            raise ValueError(f"Query has dimension {q.shape[1]}, index has {self.dimensions}")
        nq, k = q.shape[0], int(n_neighbors)
        ids, dists = _lib._results(nq, k)
        cfg = self._params.buffer_config
        if cancel is None:
            _lib.check(self._lib.svsb200_search(
                self._h, q.ctypes.data, _DTYPE_CODE[q.dtype], nq, k, cfg.search_window_size,
                cfg.search_buffer_capacity, int(self._params.search_buffer_visited_set), ids.ctypes.data, 8,
                dists.ctypes.data, None))
        else:
            fn = _lib.CANCEL_FN(lambda _arg: 1 if cancel() else 0)
            _lib.check(self._lib.svsb200_search_cancellable(
                self._h, q.ctypes.data, _DTYPE_CODE[q.dtype], nq, k, cfg.search_window_size,
                cfg.search_buffer_capacity, int(self._params.search_buffer_visited_set), ids.ctypes.data, 8,
                dists.ctypes.data, None, fn, None))
        return ids, dists

    def search_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_ids: int, d_dists: int,
                      stream: int = 0, id_bytes: int = 8):
        """Enqueue a search over device-resident buffers (raw pointers, e.g. ``tensor.data_ptr()``)."""
        cfg = self._params.buffer_config
        _lib.check(self._lib.svsb200_search_device(
            self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq, int(n_neighbors), cfg.search_window_size,
            cfg.search_buffer_capacity, int(self._params.search_buffer_visited_set), d_ids, id_bytes, d_dists,
            stream or None))

    def exhaustive_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_ids: int, d_dists: int,
                          stream: int = 0):
        """Exact top-k of every query against all base vectors (same distance code; ties by id) -- the
        harness's ground truth, standing where the reference uses ``svs::Flat`` (index/flat/flat.h:159)."""
        _lib.check(self._lib.svsb200_exhaustive_device(self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq,
                                                       int(n_neighbors), d_ids, d_dists, stream or None))

    def search_filtered(self, queries: np.ndarray, n_neighbors: int, allowed: np.ndarray):
        """``svs::runtime::VamanaIndex::search(..., IDFilter*)`` (bindings/cpp/include/svs/runtime/vamana_index.h:75-83):
        ``allowed`` is a boolean mask over the ids (the filter's ``is_member``), evaluated on the device.
        Returns (ids uint64, distances, found per query); short rows are padded with all-ones / +inf."""
        bitmap = _lib._bitmap(allowed, self._lib.svsb200_index_size(self._h))   # rows held, deleted ones included
        q = _lib._queries(queries, self.dimensions)
        found = np.empty(q.shape[0], dtype=np.uint32)
        ids, dists = _lib._search(self._lib.svsb200_search_filtered, (self._h,), q, n_neighbors,
                                  (self._params.buffer_config.search_window_size, bitmap.ctypes.data),
                                  (found.ctypes.data,))
        return ids, dists, found

    def range_search(self, queries: np.ndarray, radius: float):
        """``svs::runtime::VamanaIndex::range_search`` (vamana_index.h:85-92): per query, every graph-search result
        closer than ``radius`` (greater than, for MIP).  Returns a list of (ids, distances) pairs."""
        q = _lib._queries(queries, self.dimensions)
        nq = q.shape[0]
        if nq == 0:
            return []
        counts = np.empty(nq, dtype=np.uint32)
        pi, pd = C.c_void_p(), C.c_void_p()
        _lib.check(self._lib.svsb200_range_search(self._h, q.ctypes.data, _DTYPE_CODE[q.dtype], nq, float(radius),
                                                  self._params.buffer_config.search_window_size, counts.ctypes.data,
                                                  C.byref(pi), C.byref(pd)))
        total = int(counts.sum())
        ids = np.ctypeslib.as_array(C.cast(pi, C.POINTER(C.c_uint64)), shape=(max(total, 1),))[:total].copy()
        dd = np.ctypeslib.as_array(C.cast(pd, C.POINTER(C.c_float)), shape=(max(total, 1),))[:total].copy()
        self._lib.svsb200_free(pi)
        self._lib.svsb200_free(pd)
        offs = np.concatenate([[0], np.cumsum(counts.astype(np.int64))])
        return [(ids[offs[i]:offs[i + 1]], dd[offs[i]:offs[i + 1]]) for i in range(nq)]

    # ---- stored rows (bindings/python/include/svs/python/vamana.h:217, manager.h:141) --------------------------
    def get_distance(self, external_id: int, query_vector: np.ndarray) -> float:
        """``svs.Vamana.get_distance(external_id, query_vector)``: the distance the search computes between the query
        (a 1-D array of the index's dimension; float32 unless it already has a query type the search takes) and the
        stored row that a search returns as ``external_id``."""
        q = np.asarray(query_vector)
        if q.dtype not in _DTYPE_CODE:
            q = q.astype(np.float32)
        q = np.ascontiguousarray(q.reshape(-1))
        if q.shape[0] != self.dimensions:
            raise ValueError(f"Incompatible dimensions. Query has {q.shape[0]} while the index expects {self.dimensions}.")
        ids = np.array([int(external_id)], dtype=np.uint64)
        out = np.empty(1, dtype=np.float32)
        _lib.check(self._lib.svsb200_index_distances(self._h, q.ctypes.data, _DTYPE_CODE[q.dtype], 1, ids.ctypes.data,
                                                     out.ctypes.data))
        return float(out[0])

    def reconstruct(self, ids) -> np.ndarray:
        """``svs.Vamana.reconstruct(ids)``: the stored rows named by ``ids`` (any shape) as float32, shaped
        ``ids.shape + (dimensions,)``; SQ codes come back decompressed (scale * c + bias)."""
        ids = np.asarray(ids, dtype=np.uint64)
        flat = np.ascontiguousarray(ids.reshape(-1))
        out = np.empty((flat.shape[0], self.dimensions), dtype=np.float32)
        _lib.check(self._lib.svsb200_index_reconstruct(self._h, flat.ctypes.data, flat.shape[0], out.ctypes.data))
        return out.reshape(ids.shape + (self.dimensions,))

    def flat_search(self, queries: np.ndarray, n_neighbors: int):
        """Exact top-k of every query over ALL base vectors -- what ``svs.Flat(...).search`` computes
        (index/flat/flat.h:421-465) -- on the tensor cores, with the graph search's bit-exact distances
        (``svsb200_flat_search``)."""
        q = _lib._queries(queries, self.dimensions, "dim")
        return _lib._search(self._lib.svsb200_flat_search, (self._h,), q, n_neighbors)

    def flat_search_device(self, d_queries: int, qdtype: np.dtype, nq: int, n_neighbors: int, d_ids: int, d_dists: int,
                           stream: int = 0) -> int:
        """Device-buffer form; returns how many queries needed the exact-scan fallback."""
        fb = C.c_uint32()
        _lib.check(self._lib.svsb200_flat_search_device(self._h, d_queries, _DTYPE_CODE[np.dtype(qdtype)], nq,
                                                        int(n_neighbors), d_ids, d_dists, stream or None, C.byref(fb)))
        return int(fb.value)

    # ---- instrumentation ---------------------------------------------------------------
    def set_counting(self, enabled: bool):
        _lib.check(self._lib.svsb200_set_counting(self._h, int(enabled)))

    def counters(self, nq: int):
        hops = np.empty(nq, dtype=np.uint32)
        evals = np.empty(nq, dtype=np.uint32)
        _lib.check(self._lib.svsb200_get_counters(self._h, nq, hops.ctypes.data, evals.ctypes.data))
        return hops, evals

    def fetched(self, nq: int):
        out = np.empty(nq, dtype=np.uint32)
        _lib.check(self._lib.svsb200_get_fetched(self._h, nq, out.ctypes.data))
        return out

    def last_kernel_ms(self) -> float:
        ms = C.c_float()
        _lib.check(self._lib.svsb200_last_kernel_ms(self._h, C.byref(ms)))
        return float(ms.value)

    def set_entry_points(self, entry_points):
        """Several distinct entry points (``VamanaIndex::entry_point_`` is a vector, index/vamana/index.h:304-312)."""
        eps = np.ascontiguousarray(entry_points, dtype=np.uint32)
        _lib.check(self._lib.svsb200_set_entry_points(self._h, eps.ctypes.data, len(eps)))

    def set_option(self, name: str, value: int):
        _lib.check(self._lib.svsb200_set_option(self._h, name.encode(), int(value)))

    def get_option(self, name: str) -> int:
        out = C.c_long()
        _lib.check(self._lib.svsb200_get_option(self._h, name.encode(), C.byref(out)))
        return int(out.value)


class ShardedVamana:
    """One dataset split into contiguous id ranges, one single-device :class:`Vamana` (own graph, own entry
    point) per range -- SURVEY.md 8e mode B inside one process (``svsb200_search_sharded``).  Every query runs
    on every shard; the per-shard top-k rows are gathered on the first shard's device over NVLink and merged
    with the reference's ``TotalOrder`` (distance, then id; lib/neighbor.h:143-155)."""

    def __init__(self, shards: list, id_offsets: list):
        if len(shards) != len(id_offsets) or not shards:
            raise ValueError("one id offset per shard")
        self._shards = list(shards)
        self._lib = _lib.lib()
        for sh, off in zip(self._shards, id_offsets):
            _lib.check(self._lib.svsb200_set_id_offset(sh._h, int(off)))
        self.search_parameters = VamanaSearchParameters()

    @property
    def size(self) -> int:
        return sum(sh.size for sh in self._shards)

    def search(self, queries: np.ndarray, n_neighbors: int):
        q = _lib._queries(queries, self._shards[0].dimensions, "dim")
        cfg = self.search_parameters.buffer_config
        handles = (C.c_void_p * len(self._shards))(*[sh._h for sh in self._shards])
        return _lib._search(self._lib.svsb200_search_sharded, (handles, len(self._shards)), q, n_neighbors,
                            (cfg.search_window_size, cfg.search_buffer_capacity))


class DynamicVamana(_lib._Slots, Vamana):
    """GPU-backed dynamic Vamana index: the reference's ``svs.DynamicVamana`` / ``MutableVamanaIndex``
    (bindings/python/src/dynamic_vamana.cpp, include/svs/index/vamana/dynamic_index.h) built on the GPU or assembled
    from a graph, its data and one external id per row, with ``add``, soft ``delete``, ``consolidate`` and
    ``compact``.  Searches return external ids and never return a deleted one, while the walk still goes through
    deleted rows, exactly as ``MutableVamanaIndex::search`` does.  Mutations must not run concurrently with searches
    of the same index.  float32 / float16 data, or scalar-quantised int8 / uint8 codes (``sq=(scale, bias)``: the
    reference's ``MutableVamanaIndex`` over ``SQDataset``), one device.  A delete (``delete_entries``,
    dynamic_index.h:773-788) is soft: the slots are Deleted, and keep their rows and external ids until
    :meth:`consolidate`."""

    _ABI = "svsb200_dynamic"

    @classmethod
    def build(cls, parameters: VamanaBuildParameters, data: np.ndarray, ids=None, distance: "DistanceType" = None,
              device: int = 0, num_threads: int = 1, sq: tuple | None = None) -> "DynamicVamana":
        """``svs.DynamicVamana.build(parameters, data, ids, distance)`` (``MutableVamanaIndex(parameters, data,
        external_ids, distance)``, dynamic_index.h:208-261): the GPU builder's graph, with ``parameters`` kept as the
        mutation parameters.  ``ids`` defaults to ``0 .. n-1``.  ``sq=(scale, bias)`` marks ``data`` as SQ codes (as
        in :meth:`from_arrays`), built as :meth:`Vamana.build` builds them."""
        distance = DistanceType.L2 if distance is None else DistanceType(distance)
        if sq is not None:
            data = _lib._rows(data, (np.int8, np.uint8), ndim_error=None,
                              dtype_error="SQ codes are a 2-D int8 / uint8 array")
        else:
            data = _lib._rows(data, (np.float32, np.float16), ndim_error=None,
                              dtype_error="DynamicVamana.build takes a 2-D float32 / float16 array")
        if not parameters.use_full_search_history:
            raise ValueError("the GPU builder always keeps the full search history (the reference's default)")
        n = data.shape[0]
        ids = np.arange(n, dtype=np.uint64) if ids is None else np.ascontiguousarray(ids, dtype=np.uint64)
        if ids.shape != (n,):
            raise ValueError("one external id per row")
        self = cls.__new__(cls)
        self._lib = _lib.lib()
        self._distance = distance
        self._dtype = data.dtype
        self._params = VamanaSearchParameters()
        self._num_threads = int(num_threads)
        handle = C.c_void_p()
        tail = (float(parameters.alpha), int(parameters.graph_max_degree), int(parameters.window_size),
                int(parameters.max_candidate_pool_size), int(parameters.prune_to), ids.ctypes.data, int(device),
                C.byref(handle))
        if sq is None:
            _lib.check(self._lib.svsb200_dynamic_build(data.ctypes.data, _DTYPE_CODE[data.dtype], n, data.shape[1],
                                                       int(distance), *tail))
        else:
            _lib.check(self._lib.svsb200_dynamic_build_sq(data.ctypes.data, _DTYPE_CODE[data.dtype], n, data.shape[1],
                                                          int(distance), float(sq[0]), float(sq[1]), *tail))
        self._h = handle
        self.build_parameters = parameters
        return self

    @classmethod
    def from_arrays(cls, data: np.ndarray, graph: np.ndarray, entry_point: int, ids=None,
                    distance: DistanceType = DistanceType.L2, device: int = 0, num_threads: int = 1,
                    sq: tuple | None = None) -> "DynamicVamana":
        """``MutableVamanaIndex(graph, data, entry_point, distance, external_ids, threadpool)``
        (dynamic_index.h:178-202); ``ids`` defaults to ``0 .. n-1``.  ``sq=(scale, bias)`` marks ``data`` as
        scalar-quantised int8 / uint8 codes (from :func:`scalablevectorsearch_b200.ivf.sq_compress`): the scale and
        bias stay fixed, and :meth:`add` then takes float32 rows, encoded with them as ``SQDataset::set_datum`` does."""
        graph = np.ascontiguousarray(graph, dtype=np.uint32)
        if graph.ndim != 2:
            raise ValueError("data and graph must be 2-D")
        if sq is not None:
            data = _lib._rows(data, (np.int8, np.uint8), "data and graph must be 2-D", "SQ codes are int8 or uint8")
        else:
            data = _lib._rows(data, (np.float32, np.float16), "data and graph must be 2-D",
                              "a dynamic index takes float32 / float16 data")
        if graph.shape[0] != data.shape[0]:
            raise ValueError("Wrong sizes!")
        n = data.shape[0]
        ids = np.arange(n, dtype=np.uint64) if ids is None else np.ascontiguousarray(ids, dtype=np.uint64)
        if ids.shape != (n,):
            raise ValueError("one external id per row")
        self = cls.__new__(cls)
        self._lib = _lib.lib()
        self._distance = DistanceType(distance)
        self._dtype = data.dtype
        self._params = VamanaSearchParameters()
        self._num_threads = int(num_threads)
        handle = C.c_void_p()
        tail = (graph.ctypes.data, graph.shape[1], int(entry_point), int(self._distance), ids.ctypes.data, int(device),
                C.byref(handle))
        if sq is None:
            _lib.check(self._lib.svsb200_dynamic_create(data.ctypes.data, _DTYPE_CODE[data.dtype], n, data.shape[1], *tail))
        else:
            _lib.check(self._lib.svsb200_dynamic_create_sq(data.ctypes.data, _DTYPE_CODE[data.dtype], n, data.shape[1],
                                                           float(sq[0]), float(sq[1]), *tail))
        self._h = handle
        return self

    @property
    def size(self) -> int:
        """Number of valid (searchable) entries (``MutableVamanaIndex::size``)."""
        n = C.c_size_t(0)
        _lib.check(self._lib.svsb200_dynamic_ids(self._h, None, C.byref(n)))
        return int(n.value)

    @property
    def num_slots(self) -> int:
        """Rows held on the device, deleted ones included."""
        return self._lib.svsb200_index_size(self._h)

    def add(self, points: np.ndarray, ids, reuse_empty: bool = False) -> np.ndarray:
        """``add_points`` (dynamic_index.h:657-749): insert rows of the index's dtype (float32 rows into an SQ index,
        encoded with its scale and bias; a NaN or an infinity is refused) with new external ids.  Empty slots are used
        first (from the start with ``reuse_empty``), then the index grows.  Fails without changing anything on a
        repeated, present or reserved id.  Returns the slots used."""
        return self._add(points, ids, reuse_empty)

    def consolidate(self):
        """``consolidate`` (dynamic_index.h:976-1013): unlink the deleted entries from the graph; their slots become
        empty.  A deleted entry point is replaced by the medoid of the valid rows."""
        _lib.check(self._lib.svsb200_dynamic_consolidate(self._h))

    def compact(self):
        """``compact`` (dynamic_index.h:817-916): move the valid entries to slots ``0 .. size-1``, in slot order.
        Fails without changing anything while deleted entries are present (call :meth:`consolidate` first)."""
        _lib.check(self._lib.svsb200_dynamic_compact(self._h))

    def _build_parameters(self):
        a, w, m, p = C.c_float(), C.c_size_t(), C.c_size_t(), C.c_size_t()
        _lib.check(self._lib.svsb200_dynamic_get_build_parameters(self._h, C.byref(a), C.byref(w), C.byref(m), C.byref(p)))
        return {"alpha": float(a.value), "construction_window_size": int(w.value), "max_candidates": int(m.value),
                "prune_to": int(p.value)}

    def _set_build_parameter(self, name, value):
        cur = self._build_parameters()
        cur[name] = value
        _lib.check(self._lib.svsb200_dynamic_set_build_parameters(
            self._h, float(cur["alpha"]), int(cur["construction_window_size"]), int(cur["max_candidates"]),
            int(cur["prune_to"])))

    # mutation parameters (dynamic_vamana.cpp; 0 restores the default)
    alpha = property(lambda self: self._build_parameters()["alpha"],
                     lambda self, v: self._set_build_parameter("alpha", v))
    construction_window_size = property(lambda self: self._build_parameters()["construction_window_size"],
                                        lambda self, v: self._set_build_parameter("construction_window_size", v))
    max_candidates = property(lambda self: self._build_parameters()["max_candidates"],
                              lambda self, v: self._set_build_parameter("max_candidates", v))
    prune_to = property(lambda self: self._build_parameters()["prune_to"],
                        lambda self, v: self._set_build_parameter("prune_to", v))

    def search_filtered(self, queries: np.ndarray, n_neighbors: int, allowed: np.ndarray):
        """Filtered search: ``allowed`` is a boolean mask over the SLOTS (``num_slots`` entries, in the order of
        :meth:`export`); entries that are not valid are never returned.  Returns external ids, distances and the
        number found per query."""
        return super().search_filtered(queries, n_neighbors, allowed)

    def export(self):
        """(graph uint32[n][R+1] degree first, status uint8[n] (0 Empty, 1 Valid, 2 Deleted), external ids, entry
        point) over every slot."""
        n, R = self.num_slots, self.graph_max_degree
        graph = np.empty((n, R + 1), dtype=np.uint32)
        status = np.empty(n, dtype=np.uint8)
        ids = np.empty(n, dtype=np.uint64)
        ep = C.c_uint32()
        _lib.check(self._lib.svsb200_dynamic_export(self._h, graph.ctypes.data, status.ctypes.data, ids.ctypes.data,
                                                    C.byref(ep)))
        return graph, status, ids, int(ep.value)
