"""ctypes bindings for the two parity checkers.  TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may import
this module; the product package (``scalablevectorsearch_b200``) never does.

* :class:`RefLib`    -- ``oracle/_ref/libsvsref.so``: the unmodified reference headers compiled
  from ``/root/reference`` (``make -C oracle ref``).  It is built in the authoring container
  and travels to the GPU box as a binary.
* :class:`OracleLib` -- ``oracle/liboracle.so``: the plain-C restatement (``vamana_oracle.c``).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

DTYPE_CODES = {np.dtype(np.float32): 0, np.dtype(np.float16): 1, np.dtype(np.int8): 2, np.dtype(np.uint8): 3}
METRIC_CODES = {"l2": 0, "ip": 1, "cosine": 2}


def effective_cpus() -> int:
    """min(affinity, cgroup quota): the reference's spin-waiting pool must not be oversubscribed."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            n = min(n, max(1, int(int(quota) / int(period))))
    except (OSError, ValueError):
        pass
    return max(1, n)


def _code(arr: np.ndarray) -> int:
    return DTYPE_CODES[arr.dtype]


def _ptr(arr: np.ndarray):
    return arr.ctypes.data_as(C.c_void_p)


def _c(arr: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(arr)


class _Index:
    def __init__(self, lib, prefix: str, handle):
        self._lib, self._p, self._h = lib, prefix, handle

    def close(self):
        if self._h:
            getattr(self._lib, f"{self._p}_index_destroy")(self._h)
            self._h = None

    __del__ = close

    def set_entry_points(self, entry_points):
        """Several distinct entry points (oracle only; the compiled reference takes one)."""
        eps = np.ascontiguousarray(entry_points, dtype=np.uint32)
        fn = getattr(self._lib, f"{self._p}_index_set_entry_points")
        fn.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        if fn(self._h, eps.ctypes.data, len(eps)):
            raise RuntimeError("set_entry_points failed")

    def set_threads(self, n: int):
        fn = getattr(self._lib, f"{self._p}_index_set_threads", None)
        if fn is not None:
            fn(self._h, C.c_size_t(n))

    def search(self, queries: np.ndarray, k: int, window: int, capacity: int | None = None,
               visited_set: bool = False):
        q = _c(queries)
        nq = q.shape[0]
        capacity = window if capacity is None else capacity
        ids = np.empty((nq, k), dtype=np.uint64)
        dists = np.empty((nq, k), dtype=np.float32)
        rc = getattr(self._lib, f"{self._p}_index_search")(
            self._h, _code(q), _ptr(q), C.c_size_t(nq), C.c_size_t(k), C.c_size_t(window),
            C.c_size_t(capacity), int(visited_set), _ptr(ids), _ptr(dists))
        if rc:
            raise RuntimeError(getattr(self._lib, f"{self._p}_last_error")().decode())
        return ids, dists

    def counts(self, queries: np.ndarray, window: int, capacity: int | None = None):
        q = _c(queries)
        nq = q.shape[0]
        capacity = window if capacity is None else capacity
        hops = np.empty(nq, dtype=np.uint64)
        evals = np.empty(nq, dtype=np.uint64)
        rc = getattr(self._lib, f"{self._p}_index_counts")(
            self._h, _code(q), _ptr(q), C.c_size_t(nq), C.c_size_t(window), C.c_size_t(capacity),
            _ptr(hops), _ptr(evals))
        if rc:
            raise RuntimeError(getattr(self._lib, f"{self._p}_last_error")().decode())
        return hops, evals


class _Base:
    prefix = ""
    path = ""

    def __init__(self, path: str | None = None):
        path = path or self.path
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = C.CDLL(path)
        p = self.prefix
        getattr(self.lib, f"{p}_last_error").restype = C.c_char_p
        getattr(self.lib, f"{p}_index_create").restype = C.c_void_p
        getattr(self.lib, f"{p}_index_destroy").argtypes = [C.c_void_p]
        getattr(self.lib, f"{p}_index_search").argtypes = [
            C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int,
            C.c_void_p, C.c_void_p]
        getattr(self.lib, f"{p}_index_counts").argtypes = [
            C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p]
        getattr(self.lib, f"{p}_distance_rows").argtypes = [
            C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p]

    @classmethod
    def available(cls) -> bool:
        return os.path.exists(cls.path)

    def _err(self) -> str:
        return getattr(self.lib, f"{self.prefix}_last_error")().decode()

    def distance_rows(self, metric: str, query: np.ndarray, rows: np.ndarray) -> np.ndarray:
        q, r = _c(query), _c(rows)
        out = np.empty(r.shape[0], dtype=np.float32)
        rc = getattr(self.lib, f"{self.prefix}_distance_rows")(
            METRIC_CODES[metric], _code(q), _code(r), _ptr(q), _ptr(r), C.c_size_t(r.shape[0]),
            C.c_size_t(r.shape[1]), _ptr(out))
        if rc:
            raise RuntimeError(self._err())
        return out

    def index(self, data: np.ndarray, graph: np.ndarray, entry_point: int, metric: str,
              threads: int = 1) -> _Index:
        """``graph`` is the reference layout: uint32[n][max_degree+1], degree first."""
        d, g = _c(data), _c(graph.astype(np.uint32, copy=False))
        fn = getattr(self.lib, f"{self.prefix}_index_create")
        fn.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_uint32,
                       C.c_int, C.c_size_t]
        h = fn(_code(d), _ptr(d), d.shape[0], d.shape[1], _ptr(g), g.shape[1] - 1, int(entry_point),
               METRIC_CODES[metric], threads)
        if not h:
            raise RuntimeError(self._err())
        idx = _Index(self.lib, self.prefix, h)
        idx._keep = (d, g)
        return idx

    def sq_index(self, data: np.ndarray, graph: np.ndarray, entry_point: int, metric: str,
                 code_dtype=np.int8, threads: int = 1):
        """Scalar-quantised index; returns (index, codes, scale, bias)."""
        d, g = _c(data.astype(np.float32, copy=False)), _c(graph.astype(np.uint32, copy=False))
        codes = np.empty(d.shape, dtype=code_dtype)
        scale, bias = C.c_float(), C.c_float()
        fn = getattr(self.lib, f"{self.prefix}_sq_index_create")
        fn.restype = C.c_void_p
        fn.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_uint32,
                       C.c_int, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
        h = fn(DTYPE_CODES[np.dtype(code_dtype)], _ptr(d), d.shape[0], d.shape[1], _ptr(g), g.shape[1] - 1,
               int(entry_point), METRIC_CODES[metric], threads, C.byref(scale), C.byref(bias), _ptr(codes))
        if not h:
            raise RuntimeError(self._err())
        idx = _Index(self.lib, self.prefix, h)
        idx._keep = (d, g)
        return idx, codes, float(np.float32(scale.value)), float(np.float32(bias.value))


class RefLib(_Base):
    """The compiled reference (``oracle/_ref/libsvsref.so``)."""
    prefix = "svsref"
    path = os.path.join(HERE, "_ref", "libsvsref.so")

    def __init__(self, path=None):
        super().__init__(path)
        self.lib.svsref_to_float16.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]

    def avx512(self) -> bool:
        return bool(self.lib.svsref_avx512())

    def avx512vnni(self) -> bool:
        return bool(self.lib.svsref_avx512vnni())

    def to_float16(self, x: np.ndarray) -> np.ndarray:
        """float32 -> float16 through the reference's own ``Float16(float)`` (lib/float16.h:54-79)."""
        x = _c(x.astype(np.float32, copy=False))
        out = np.empty(x.shape, dtype=np.uint16)
        self.lib.svsref_to_float16(_ptr(x), x.size, _ptr(out))
        return out.view(np.float16)

    def build(self, data: np.ndarray, metric: str, max_degree: int, window: int, alpha: float | None = None,
              max_candidates: int | None = None, prune_to: int | None = None, threads: int = 0):
        """Reference ``auto_build``; returns (graph uint32[n][R+1] degree-first, entry_point)."""
        d = _c(data)
        n = d.shape[0]
        threads = threads or effective_cpus()
        if alpha is None:
            alpha = 1.2 if metric == "l2" else 0.95
        # Defaults of index/vamana/index.h:1081-1095.
        max_candidates = max_candidates or 3 * window
        prune_to = prune_to or (max_degree - 4 if max_degree >= 16 else max_degree)
        graph = np.zeros((n, max_degree + 1), dtype=np.uint32)
        ep = C.c_uint32()
        fn = self.lib.svsref_build
        fn.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_float, C.c_size_t, C.c_size_t,
                       C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p]
        rc = fn(_code(d), _ptr(d), n, d.shape[1], METRIC_CODES[metric], alpha, max_degree, window,
                max_candidates, prune_to, threads, _ptr(graph), C.byref(ep))
        if rc:
            raise RuntimeError(self._err())
        return graph, int(ep.value)


class OracleLib(_Base):
    """The plain-C restatement (``oracle/liboracle.so``)."""
    prefix = "oracle"
    path = os.path.join(HERE, "liboracle.so")

    def sq_distance_rows(self, metric: str, query: np.ndarray, codes: np.ndarray, scale: float,
                         bias: float) -> np.ndarray:
        """:meth:`distance_rows` over SQ int8 / uint8 codes, as the SQ index search computes them."""
        q, r = _c(query), _c(codes)
        out = np.empty(r.shape[0], dtype=np.float32)
        fn = self.lib.oracle_sq_distance_rows
        fn.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_size_t,
                       C.c_size_t, C.c_void_p]
        if fn(METRIC_CODES[metric], _code(q), _code(r), float(scale), float(bias), _ptr(q), _ptr(r),
              C.c_size_t(r.shape[0]), C.c_size_t(r.shape[1]), _ptr(out)):
            raise RuntimeError(self._err())
        return out

    # ---- LVQ-8 (own specification; parity with Intel's closed LVQ is unpinned) ----
    def lvq8_distance_rows(self, metric: str, query: np.ndarray, rows: np.ndarray, dim: int,
                           mean: np.ndarray) -> np.ndarray:
        """:meth:`distance_rows` over LVQ-8 rows (from :meth:`lvq8_compress`), as the LVQ-8 index search computes them."""
        q, r, m = _c(query), _c(rows), _c(mean.astype(np.float32, copy=False))
        out = np.empty(r.shape[0], dtype=np.float32)
        fn = self.lib.oracle_lvq8_distance_rows
        fn.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p]
        if fn(METRIC_CODES[metric], _code(q), _ptr(q), _ptr(r), C.c_size_t(r.shape[0]), C.c_size_t(dim), _ptr(m),
              _ptr(out)):
            raise RuntimeError(self._err())
        return out

    def lvq8_compress(self, data: np.ndarray, mean: np.ndarray) -> np.ndarray:
        """Raises RuntimeError, naming the first offending row, where a residual or a float16 constant is not finite."""
        d, m = _c(data.astype(np.float32, copy=False)), _c(mean.astype(np.float32, copy=False))
        self.lib.oracle_lvq8_row_stride.restype = C.c_size_t
        self.lib.oracle_lvq8_row_stride.argtypes = [C.c_size_t]
        stride = self.lib.oracle_lvq8_row_stride(d.shape[1])
        rows = np.zeros((d.shape[0], stride), dtype=np.uint8)
        self.lib.oracle_lvq8_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p]
        if self.lib.oracle_lvq8_compress(_ptr(d), d.shape[0], d.shape[1], _ptr(m), _ptr(rows)):
            raise RuntimeError(self._err())
        return rows

    def lvq8_index(self, rows: np.ndarray, dim: int, mean: np.ndarray, graph: np.ndarray, entry_point: int,
                   metric: str) -> _Index:
        r, m, g = _c(rows), _c(mean.astype(np.float32, copy=False)), _c(graph.astype(np.uint32, copy=False))
        fn = self.lib.oracle_lvq8_index_create
        fn.restype = C.c_void_p
        fn.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_int]
        h = fn(_ptr(r), r.shape[0], dim, _ptr(m), _ptr(g), g.shape[1] - 1, int(entry_point), METRIC_CODES[metric])
        if not h:
            raise RuntimeError(self._err())
        idx = _Index(self.lib, self.prefix, h)
        idx._keep = (r, m, g)
        return idx
