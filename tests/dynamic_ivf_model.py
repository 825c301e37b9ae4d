"""A numpy model of the dynamic IVF index's contract (include/svsb200.h, svsb200_dynamic_ivf_*; DESIGN.md §16), needing
no GPU.

Slots follow the reference's rules (dynamic_ivf.h): a slot is Valid or Empty; a delete empties it at once and leaves a
tombstone in its cluster; an add without reuse_empty appends new slots, with reuse_empty it takes Empty slots from slot
0 first; every added row is appended to its nearest centroid's cluster in input order; compaction renumbers the Valid
slots in slot order and keeps every cluster's stored order.  A search is the static IVF model's (tests/ivf_model.py)
over the Valid rows of the probed clusters, ordered by (distance, slot), with the slots mapped to external ids.
Distances and the nearest centroids come from the C oracle through ivf_model.
"""
from __future__ import annotations

import numpy as np

import ivf_model as M

RESERVED = 2**64 - 1
NONE32 = 2**32 - 1


class Refused(ValueError):
    """A call the library refuses without changing anything."""


class DynamicIVFModel:
    def __init__(self, oracle, metric: int, centroids: np.ndarray, dtype, dim: int):
        self.oracle, self.metric = oracle, metric
        self.centroids = np.ascontiguousarray(centroids, dtype=np.float32)
        self.C = self.centroids.shape[0]
        self.dtype, self.dim = np.dtype(dtype), dim
        self.valid: list[bool] = []
        self.ext: list[int] = []
        self.cluster: list[int] = []          # per slot: its cluster (NONE32 when Empty)
        self.rows: dict[int, np.ndarray] = {}  # per Valid slot: its row
        self.stored: list[list[int]] = [[] for _ in range(self.C)]   # per cluster: slots in stored order, None = tombstone
        self.translator: dict[int, int] = {}

    # ---- assembly ----
    @classmethod
    def assemble(cls, oracle, metric, centroids, data, ids, assignments=None):
        m = cls(oracle, metric, centroids, data.dtype, data.shape[1])
        ids = [int(i) for i in ids]
        m._check_new(ids)
        if assignments is None:
            assignments = m.nearest_cluster(data)
        for i, (row, a) in enumerate(zip(data, assignments)):
            m.valid.append(True)
            m.ext.append(ids[i])
            m.cluster.append(int(a))
            m.rows[i] = row
            m.stored[int(a)].append(i)
            m.translator[ids[i]] = i
        return m

    def nearest_cluster(self, rows: np.ndarray) -> np.ndarray:
        if rows.shape[0] == 0:
            return np.empty(0, dtype=np.int64)
        return M.nearest(self.oracle, self.metric, rows, self.centroids, 1)[:, 0]

    # ---- mutations ----
    def _check_new(self, ids):
        if len(set(ids)) != len(ids):
            raise Refused("repeated id")
        for i in ids:
            if i == RESERVED:
                raise Refused("reserved id")
            if i in self.translator:
                raise Refused(f"id {i} already exists")

    def add(self, points: np.ndarray, ids, reuse_empty: bool = False) -> list[int]:
        ids = [int(i) for i in ids]
        if np.dtype(points.dtype) != self.dtype:
            raise Refused("dtype")
        self._check_new(ids)
        slots = []
        if reuse_empty:
            slots = [s for s, v in enumerate(self.valid) if not v][:len(ids)]
        n = len(self.valid)
        slots += list(range(n, n + len(ids) - len(slots)))
        if slots and slots[-1] >= 2**31 - 1:
            raise Refused("too many slots")
        assign = self.nearest_cluster(points)
        grow = max(slots, default=-1) + 1 - n
        self.valid += [False] * max(grow, 0)
        self.ext += [RESERVED] * max(grow, 0)
        self.cluster += [NONE32] * max(grow, 0)
        for s, i, row, a in zip(slots, ids, points, assign):
            self.valid[s] = True
            self.ext[s] = i
            self.cluster[s] = int(a)
            self.rows[s] = row
            self.stored[int(a)].append(s)
            self.translator[i] = s
        return slots

    def delete(self, ids) -> None:
        ids = [int(i) for i in ids]
        if len(set(ids)) != len(ids) or any(i not in self.translator for i in ids):
            raise Refused("absent or repeated id")
        for i in ids:
            s = self.translator.pop(i)
            c = self.cluster[s]
            self.stored[c][self.stored[c].index(s)] = None
            self.valid[s] = False
            self.ext[s] = RESERVED
            self.cluster[s] = NONE32
            del self.rows[s]

    def compact(self) -> None:
        renum = {}
        for s, v in enumerate(self.valid):
            if v:
                renum[s] = len(renum)
        m = len(renum)
        ext, cluster, rows = [RESERVED] * m, [NONE32] * m, {}
        for s, t in renum.items():
            ext[t], cluster[t], rows[t] = self.ext[s], self.cluster[s], self.rows[s]
        self.stored = [[renum[s] for s in st if s is not None] for st in self.stored]
        self.valid, self.ext, self.cluster, self.rows = [True] * m, ext, cluster, rows
        self.translator = {e: t for t, e in enumerate(ext)}

    # ---- inspection ----
    @property
    def size(self) -> int:
        return len(self.translator)

    def all_ids(self) -> np.ndarray:
        return np.array([e for e, v in zip(self.ext, self.valid) if v], dtype=np.uint64)

    def export(self):
        return (np.array(self.valid, dtype=np.uint8), np.array(self.ext, dtype=np.uint64),
                np.array(self.cluster, dtype=np.uint32))

    def cluster_sizes(self) -> np.ndarray:
        return np.array([sum(s is not None for s in st) for st in self.stored], dtype=np.uint32)

    def live_slots(self) -> np.ndarray:
        return np.flatnonzero(np.array(self.valid, dtype=bool))

    def live_rows(self) -> np.ndarray:
        live = self.live_slots()
        if live.size == 0:
            return np.empty((0, self.dim), dtype=self.dtype)
        return np.stack([self.rows[s] for s in live]).astype(self.dtype)

    # ---- search ----
    def search(self, queries: np.ndarray, k: int, n_probes: int):
        """The exact top k over the Valid rows of the n_probes nearest clusters, by (distance, slot), as external ids;
        padded with all-ones ids and +-inf."""
        nq = queries.shape[0]
        ids = np.full((nq, k), RESERVED, dtype=np.uint64)
        dists = np.full((nq, k), np.inf if self.metric == 0 else -np.inf, dtype=np.float32)
        live = self.live_slots()
        if live.size == 0:
            return ids, dists
        rows = self.live_rows()
        live_cluster = np.array([self.cluster[s] for s in live])
        probes = M.nearest(self.oracle, self.metric, queries, self.centroids, n_probes)
        ext = np.array(self.ext, dtype=np.uint64)
        for i, q in enumerate(queries):
            sel = np.flatnonzero(np.isin(live_cluster, probes[i]))
            if sel.size == 0:
                continue
            d = self.oracle.distance_rows(M.METRICS[self.metric], q, rows[sel])
            key = d if self.metric == 0 else -d
            order = np.lexsort((live[sel], key))[:k]
            ids[i, :order.size] = ext[live[sel][order]]
            dists[i, :order.size] = d[order]
        return ids, dists
