"""ctypes binding of ``oracle/_ref/libsvsref_dynamic_flat.so``: the reference's ``DynamicFlatIndex``
(index/flat/dynamic_flat.h) compiled from the unmodified headers (``make -C oracle -f dynamic_flat.mk dynamic_flat``).
TEST INFRASTRUCTURE ONLY: the product package never imports it."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .bindings import HERE, METRIC_CODES, _c, _code, _ptr, effective_cpus


class RefDynamicFlat:
    """The reference's ``DynamicFlatIndex`` behind ``svsref_dynamic_flat_*``."""

    def __init__(self, lib, handle, dtype):
        self._lib, self._h, self._dtype = lib, handle, np.dtype(dtype)

    def close(self):
        if self._h:
            self._lib.svsref_dynamic_flat_destroy(self._h)
            self._h = None

    __del__ = close

    def _check(self, rc):
        if rc:
            raise RuntimeError(self._lib.svsref_dynamic_flat_last_error().decode())

    def add(self, points, ids, reuse_empty=False) -> np.ndarray:
        pts = _c(np.asarray(points).astype(self._dtype, copy=False))
        ids = _c(np.atleast_1d(np.asarray(ids, dtype=np.uint64)))
        slots = np.empty(len(ids), dtype=np.uint64)
        self._check(self._lib.svsref_dynamic_flat_add(self._h, _ptr(pts), len(ids), _ptr(ids), int(reuse_empty),
                                                      _ptr(slots)))
        return slots

    def delete(self, ids):
        ids = _c(np.atleast_1d(np.asarray(ids, dtype=np.uint64)))
        self._check(self._lib.svsref_dynamic_flat_delete(self._h, _ptr(ids), len(ids)))

    def compact(self):
        self._check(self._lib.svsref_dynamic_flat_compact(self._h))

    @property
    def size(self) -> int:
        return self._lib.svsref_dynamic_flat_size(self._h)

    def all_ids(self) -> np.ndarray:
        out = np.empty(self.size, dtype=np.uint64)
        self._check(self._lib.svsref_dynamic_flat_all_ids(self._h, _ptr(out)))
        return out

    def export(self):
        """(status uint8 (0 Empty, 1 Valid), external ids (2^64 - 1 where Empty)) over every slot."""
        n = self._lib.svsref_dynamic_flat_slots(self._h)
        status = np.zeros(n, dtype=np.uint8)
        ext = np.zeros(n, dtype=np.uint64)
        self._check(self._lib.svsref_dynamic_flat_export(self._h, _ptr(status), _ptr(ext)))
        return status, ext

    def search(self, queries, k):
        """Exact top k over the Valid slots, external ids.  Queries: float32 over float rows, the rows' own type over
        int8 / uint8 rows.  Needs at least k Valid slots (the reference translates every result id)."""
        qt = self._dtype if self._dtype in (np.int8, np.uint8) else np.float32
        q = _c(np.asarray(queries, dtype=qt))
        ids = np.empty((q.shape[0], k), dtype=np.uint64)
        dists = np.empty((q.shape[0], k), dtype=np.float32)
        self._check(self._lib.svsref_dynamic_flat_search(self._h, _ptr(q), q.shape[0], k, _ptr(ids), _ptr(dists)))
        return ids, dists


class RefDynamicFlatLib:
    """The compiled façade (``oracle/_ref/libsvsref_dynamic_flat.so``)."""
    path = os.path.join(HERE, "_ref", "libsvsref_dynamic_flat.so")

    @classmethod
    def available(cls) -> bool:
        return os.path.exists(cls.path)

    def __init__(self, path=None):
        path = path or self.path
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = L = C.CDLL(path)
        sz, vp = C.c_size_t, C.c_void_p
        L.svsref_dynamic_flat_last_error.restype = C.c_char_p
        L.svsref_dynamic_flat_create.restype = vp
        L.svsref_dynamic_flat_create.argtypes = [C.c_int, vp, sz, sz, C.c_int, vp, sz]
        L.svsref_dynamic_flat_destroy.argtypes = [vp]
        L.svsref_dynamic_flat_add.argtypes = [vp, vp, sz, vp, C.c_int, vp]
        L.svsref_dynamic_flat_delete.argtypes = [vp, vp, sz]
        L.svsref_dynamic_flat_compact.argtypes = [vp]
        L.svsref_dynamic_flat_slots.restype, L.svsref_dynamic_flat_slots.argtypes = sz, [vp]
        L.svsref_dynamic_flat_size.restype, L.svsref_dynamic_flat_size.argtypes = sz, [vp]
        L.svsref_dynamic_flat_all_ids.argtypes = [vp, vp]
        L.svsref_dynamic_flat_export.argtypes = [vp, vp, vp]
        L.svsref_dynamic_flat_search.argtypes = [vp, vp, sz, sz, vp, vp]

    def dynamic_flat(self, data, ids, metric, threads: int = 0) -> RefDynamicFlat:
        """``DynamicFlatIndex(data, ids, distance, threads)``; ``data`` may have no rows."""
        d, e = _c(data), _c(np.asarray(ids, dtype=np.uint64))
        h = self.lib.svsref_dynamic_flat_create(_code(d), _ptr(d), d.shape[0], d.shape[1], METRIC_CODES[metric],
                                                _ptr(e), threads or effective_cpus())
        if not h:
            raise RuntimeError(self.lib.svsref_dynamic_flat_last_error().decode())
        return RefDynamicFlat(self.lib, h, d.dtype)
