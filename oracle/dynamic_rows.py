"""ctypes binding of ``oracle/_ref/libsvsref_dynamic_rows.so`` and ``libsvsref_dynamic_sq_rows.so``: the façades of
:mod:`oracle.dynamic` and :mod:`oracle.dynamic_sq`, each compiled with the reference's stored-row reads
(``MutableVamanaIndex::get_distance`` / ``reconstruct_at``, index/vamana/dynamic_index.h) added
(``make -C oracle -f dynamic_rows.mk dynamic_rows``).  TEST INFRASTRUCTURE ONLY: the product package never imports it."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .bindings import HERE, _c, _ptr
from .dynamic import RefDynamicLib
from .dynamic_sq import RefDynamicSQLib


def _bind(lib, prefix):
    vp, sz = C.c_void_p, C.c_size_t
    getattr(lib, prefix + "_get_distance").argtypes = [vp, C.c_uint64, vp, vp]
    getattr(lib, prefix + "_reconstruct").argtypes = [vp, vp, sz, vp]


class RefDynamicRowsLib(RefDynamicLib):
    """:class:`oracle.dynamic.RefDynamicLib` whose handles also answer :func:`get_distance` and :func:`reconstruct`."""
    path = os.path.join(HERE, "_ref", "libsvsref_dynamic_rows.so")
    prefix = "svsref_dynamic"

    def __init__(self, path=None):
        super().__init__(path)
        _bind(self.lib, self.prefix)


class RefDynamicSQRowsLib(RefDynamicSQLib):
    """:class:`oracle.dynamic_sq.RefDynamicSQLib` whose handles also answer :func:`get_distance` and
    :func:`reconstruct` (the rows decompressed as scale * c + bias)."""
    path = os.path.join(HERE, "_ref", "libsvsref_dynamic_sq_rows.so")
    prefix = "svsref_dynamic_sq"

    def __init__(self, path=None):
        super().__init__(path)
        _bind(self.lib, self.prefix)


def _prefix(ref):
    return "svsref_dynamic_sq" if hasattr(ref._lib, "svsref_dynamic_sq_create") else "svsref_dynamic"


def get_distance(ref, external_id, query) -> float:
    """``MutableVamanaIndex::get_distance(external_id, query)`` with a float32 query, on a handle of either library."""
    q = _c(np.asarray(query, dtype=np.float32).reshape(-1))
    out = C.c_float()
    ref._check(getattr(ref._lib, _prefix(ref) + "_get_distance")(ref._h, int(external_id), _ptr(q), C.byref(out)))
    return float(out.value)


def reconstruct(ref, ids, dim) -> np.ndarray:
    """The rows of external ids ``ids`` as float32 [len(ids), dim] (``reconstruct_at``), on a handle of either library."""
    e = _c(np.asarray(ids, dtype=np.uint64).reshape(-1))
    out = np.empty((e.shape[0], dim), dtype=np.float32)
    ref._check(getattr(ref._lib, _prefix(ref) + "_reconstruct")(ref._h, _ptr(e), e.shape[0], _ptr(out)))
    return out
