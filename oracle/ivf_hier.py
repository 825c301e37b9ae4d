"""ctypes wrapper of ``_ref/libsvsref_ivf_hier.so`` (ref/ivf_hier_capi.cpp): the reference's own hierarchical k-means
behind a test-only façade.  TEST INFRASTRUCTURE ONLY (see README.md)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libsvsref_ivf_hier.so")


class RefHierarchicalKMeans:
    """``hierarchical_kmeans_clustering<float>`` of the reference over float32 rows."""

    def __init__(self, path: str = PATH):
        self.lib = C.CDLL(path)
        self.lib.svsref_ivf_hier_last_error.restype = C.c_char_p
        sz, vp = C.c_size_t, C.c_void_p
        self.lib.svsref_ivf_cluster_hierarchical.argtypes = [vp, sz, sz, C.c_int, sz, sz, sz, sz, C.c_float, C.c_uint64,
                                                             vp, vp]

    @staticmethod
    def available() -> bool:
        return os.path.exists(PATH)

    def cluster(self, data, metric: int, num_centroids: int, level1_clusters: int, num_iterations: int,
                training_fraction: float, seed: int, minibatch_size: int = 10_000):
        """(centroids float32 [C][dim], assignments uint32 [n])."""
        x = np.ascontiguousarray(data, dtype=np.float32)
        cent = np.empty((num_centroids, x.shape[1]), dtype=np.float32)
        assign = np.empty(x.shape[0], dtype=np.uint32)
        rc = self.lib.svsref_ivf_cluster_hierarchical(x.ctypes.data, x.shape[0], x.shape[1], int(metric), num_centroids,
                                                      level1_clusters, minibatch_size, num_iterations,
                                                      float(training_fraction), int(seed), cent.ctypes.data,
                                                      assign.ctypes.data)
        if rc:
            raise RuntimeError(self.lib.svsref_ivf_hier_last_error().decode())
        return cent, assign
