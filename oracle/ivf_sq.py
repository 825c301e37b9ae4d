"""ctypes wrapper of ``_ref/libsvsref_ivf_sq.so`` (ref/ivf_sq_capi.cpp): the reference's own IVF index over
SQDataset<int8_t / uint8_t> behind a test-only façade.  TEST INFRASTRUCTURE ONLY (see README.md)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libsvsref_ivf_sq.so")
CODE_TYPES = {np.dtype(np.int8): 2, np.dtype(np.uint8): 3}


class RefIVFSQ:
    """``SQDataset::compress`` + ``assemble_from_clustering`` + ``IVFIndex::search`` of the reference, float32 rows and
    queries."""

    def __init__(self, path: str = PATH):
        self.lib = C.CDLL(path)
        self.lib.svsref_ivf_sq_last_error.restype = C.c_char_p
        sz, vp = C.c_size_t, C.c_void_p
        self.lib.svsref_ivf_sq_search.argtypes = [vp, sz, sz, C.c_int, C.c_int, vp, sz, vp, vp, sz, sz, sz, vp, vp, vp,
                                                  vp, vp]

    @staticmethod
    def available() -> bool:
        return os.path.exists(PATH)

    def search(self, data, code_dtype, metric: int, centroids, assignments, queries, k: int, n_probes: int):
        """-> (ids, distances, codes, scale, bias)."""
        x = np.ascontiguousarray(data, dtype=np.float32)
        c = np.ascontiguousarray(centroids, dtype=np.float32)
        a = np.ascontiguousarray(assignments, dtype=np.uint32)
        q = np.ascontiguousarray(queries, dtype=np.float32)
        ids = np.empty((q.shape[0], k), dtype=np.uint64)
        dists = np.empty((q.shape[0], k), dtype=np.float32)
        codes = np.empty(x.shape, dtype=code_dtype)
        scale, bias = C.c_float(), C.c_float()
        rc = self.lib.svsref_ivf_sq_search(x.ctypes.data, x.shape[0], x.shape[1], CODE_TYPES[np.dtype(code_dtype)],
                                           int(metric), c.ctypes.data, c.shape[0], a.ctypes.data, q.ctypes.data,
                                           q.shape[0], k, n_probes, ids.ctypes.data, dists.ctypes.data,
                                           codes.ctypes.data, C.byref(scale), C.byref(bias))
        if rc:
            raise RuntimeError(self.lib.svsref_ivf_sq_last_error().decode())
        return ids, dists, codes, float(np.float32(scale.value)), float(np.float32(bias.value))
