"""A numpy model of the dynamic IVF index over SQ codes (include/svsb200.h, svsb200_dynamic_ivf_create_sq; DESIGN.md §16,
SQ storage), needing no GPU.

The slot rules are the float model's (tests/dynamic_ivf_model.py) over int8 / uint8 codes under a scale and bias fixed
at assembly.  An add takes finite float32 rows: each joins the centroid nearest to its float32 values, and is stored as
``ivf_sq_model.encode`` of them.  A search is the exact top k over the Valid codes of the probed clusters with
``ivf_sq_model.distances``, ordered by (distance, slot), the slots mapped to external ids.
"""
from __future__ import annotations

import numpy as np

import ivf_model as M
import ivf_sq_model as S
from dynamic_ivf_model import NONE32, RESERVED, DynamicIVFModel, Refused


class DynamicIVFSQModel(DynamicIVFModel):
    def __init__(self, oracle, metric: int, centroids: np.ndarray, code_dtype, dim: int, scale: float, bias: float):
        super().__init__(oracle, metric, centroids, code_dtype, dim)
        self.scale, self.bias = float(np.float32(scale)), float(np.float32(bias))

    @classmethod
    def assemble(cls, oracle, metric, centroids, codes, ids, scale, bias, assignments=None):
        """Codes with one external id each; assignments are required unless there are no codes."""
        if codes.shape[0] and assignments is None:
            raise Refused("SQ rows need assignments")
        m = cls(oracle, metric, centroids, codes.dtype, codes.shape[1], scale, bias)
        ids = [int(i) for i in ids]
        m._check_new(ids)
        for i, (row, a) in enumerate(zip(codes, assignments if codes.shape[0] else [])):
            m.valid.append(True)
            m.ext.append(ids[i])
            m.cluster.append(int(a))
            m.rows[i] = row
            m.stored[int(a)].append(i)
            m.translator[ids[i]] = i
        return m

    def encode(self, points: np.ndarray) -> np.ndarray:
        return S.encode(points, self.dtype, self.scale, self.bias)

    def add(self, points: np.ndarray, ids, reuse_empty: bool = False) -> list[int]:
        ids = [int(i) for i in ids]
        if np.dtype(points.dtype) != np.float32:
            raise Refused("float32")
        if not np.isfinite(points).all():
            raise Refused("NaN or infinity")
        self._check_new(ids)
        slots = []
        if reuse_empty:
            slots = [s for s, v in enumerate(self.valid) if not v][:len(ids)]
        n = len(self.valid)
        slots += list(range(n, n + len(ids) - len(slots)))
        assign = self.nearest_cluster(points)
        codes = self.encode(points)
        grow = max(slots, default=-1) + 1 - n
        self.valid += [False] * max(grow, 0)
        self.ext += [RESERVED] * max(grow, 0)
        self.cluster += [NONE32] * max(grow, 0)
        for s, i, row, a in zip(slots, ids, codes, assign):
            self.valid[s] = True
            self.ext[s] = i
            self.cluster[s] = int(a)
            self.rows[s] = row
            self.stored[int(a)].append(s)
            self.translator[i] = s
        return slots

    def search(self, queries: np.ndarray, k: int, n_probes: int):
        nq = queries.shape[0]
        ids = np.full((nq, k), RESERVED, dtype=np.uint64)
        dists = np.full((nq, k), np.inf if self.metric == 0 else -np.inf, dtype=np.float32)
        live = self.live_slots()
        if live.size == 0:
            return ids, dists
        codes = self.live_rows()
        live_cluster = np.array([self.cluster[s] for s in live])
        probes = M.nearest(self.oracle, self.metric, queries, self.centroids, n_probes)
        ext = np.array(self.ext, dtype=np.uint64)
        for i, q in enumerate(queries):
            sel = np.flatnonzero(np.isin(live_cluster, probes[i]))
            if sel.size == 0:
                continue
            d = S.distances(self.oracle, self.metric, q, codes[sel], self.scale, self.bias)
            key = d if self.metric == 0 else -d
            order = np.lexsort((live[sel], key))[:k]
            ids[i, :order.size] = ext[live[sel][order]]
            dists[i, :order.size] = d[order]
        return ids, dists
