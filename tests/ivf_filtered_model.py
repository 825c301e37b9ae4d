"""A numpy model of the IVF filtered search's contract (include/svsb200.h, svsb200_ivf_search_filtered and
svsb200_dynamic_ivf_search_filtered; DESIGN.md §15), needing no GPU.

Query q probes the clusters in the plain search's order (``ivf_model.nearest``: the flat search over the centroids,
ties to the lower centroid).  P_0 = n_probes, P_{j+1} = min(4 P_j, P_max), P_max = min(C, 1024); q uses the first P_j
whose nearest P_j clusters hold at least k allowed rows, or P_max when none does, independently of the other queries.
Its row is the exact top k over the allowed rows of those clusters, ordered by (distance, key) -- the key is the
original id, or the slot of the dynamic index, whose ids are then mapped to external ids -- and padded with all-ones
ids and +inf for every metric.  Per query it also reports the P used, the allowed rows and the rows of those clusters.
Distances are those of ivf_model / ivf_sq_model / the dynamic models, so they are the scan's bit-exact ones.
"""
from __future__ import annotations

import numpy as np

import ivf_model as M
import ivf_sq_model as S

PAD_ID = M.PAD_ID
NONE32 = 2**32 - 1
P_LIMIT = 1024


def p_max(C: int) -> int:
    return min(C, P_LIMIT)


def growth(n_probes: int, C: int) -> list[int]:
    """The sequence P_0, P_1, ... up to and including P_max."""
    seq = [int(n_probes)]
    while seq[-1] < p_max(C):
        seq.append(min(4 * seq[-1], p_max(C)))
    return seq


def choose(order: np.ndarray, allowed_per_cluster: np.ndarray, k: int, n_probes: int) -> int:
    """The P one query uses, its probe order being `order` (at least P_max clusters)."""
    C = allowed_per_cluster.shape[0]
    for P in growth(n_probes, C):
        if int(allowed_per_cluster[order[:P]].sum()) >= k:
            return P
    return p_max(C)


def search(metric: int, order: np.ndarray, key_cluster: np.ndarray, present: np.ndarray, keep: np.ndarray, distances,
           k: int, n_probes: int, out_ids: np.ndarray | None, C: int):
    """The filtered search over rows addressed by keys 0 .. len(key_cluster) - 1.

    order: [nq][P_max] probe order per query; key_cluster: cluster of every key; present: the key holds a row (an
    Empty slot does not); keep: present and allowed; distances(i, keys) -> float32 distances of query i to those keys'
    rows; out_ids: the id returned for every key (None: the key itself).
    Returns (ids uint64 [nq][k], dists float32 [nq][k], probes, allowed, rows uint32 [nq])."""
    nq = order.shape[0]
    allowed_c = np.bincount(key_cluster[keep], minlength=C)[:C]
    rows_c = np.bincount(key_cluster[present], minlength=C)[:C]
    ids = np.full((nq, k), PAD_ID, dtype=np.uint64)
    dists = np.full((nq, k), np.inf, dtype=np.float32)
    probes = np.zeros(nq, dtype=np.uint32)
    n_allowed = np.zeros(nq, dtype=np.uint32)
    n_rows = np.zeros(nq, dtype=np.uint32)
    for i in range(nq):
        P = choose(order[i], allowed_c, k, n_probes)
        probed = order[i, :P]
        probes[i] = P
        n_allowed[i] = allowed_c[probed].sum()
        n_rows[i] = rows_c[probed].sum()
        keys = np.flatnonzero(keep & np.isin(key_cluster, probed))
        if keys.size == 0:
            continue
        d = np.asarray(distances(i, keys), dtype=np.float32)
        sort_key = d if metric == 0 else -d
        top = np.lexsort((keys, sort_key))[:k]
        ids[i, :top.size] = keys[top] if out_ids is None else out_ids[keys[top]]
        dists[i, :top.size] = d[top]
    return ids, dists, probes, n_allowed, n_rows


def probe_order(oracle, metric: int, queries: np.ndarray, centroids: np.ndarray) -> np.ndarray:
    """Every query's nearest P_max clusters, in probe order."""
    return M.nearest(oracle, metric, queries, centroids, p_max(centroids.shape[0]))


def static(oracle, metric: int, data: np.ndarray, centroids: np.ndarray, assignments: np.ndarray, queries: np.ndarray,
           k: int, n_probes: int, allowed: np.ndarray):
    """svsb200_ivf_search_filtered on a float index; `allowed` is bool [n] over original ids."""
    order = probe_order(oracle, metric, queries, centroids)
    cl = np.asarray(assignments, dtype=np.int64)
    return search(metric, order, cl, np.ones(cl.shape[0], dtype=bool), np.asarray(allowed, dtype=bool),
                   lambda i, keys: oracle.distance_rows(M.METRICS[metric], queries[i], data[keys]), k, n_probes, None,
                   C=centroids.shape[0])


def static_sq(oracle, metric: int, codes: np.ndarray, scale: float, bias: float, centroids: np.ndarray,
              assignments: np.ndarray, queries: np.ndarray, k: int, n_probes: int, allowed: np.ndarray):
    """svsb200_ivf_search_filtered on an SQ index."""
    order = probe_order(oracle, metric, queries, centroids)
    cl = np.asarray(assignments, dtype=np.int64)
    return search(metric, order, cl, np.ones(cl.shape[0], dtype=bool), np.asarray(allowed, dtype=bool),
                   lambda i, keys: S.distances(oracle, metric, queries[i], codes[keys], scale, bias), k, n_probes, None,
                   C=centroids.shape[0])


def dynamic(model, queries: np.ndarray, k: int, n_probes: int, allowed_slots: np.ndarray):
    """svsb200_dynamic_ivf_search_filtered on a DynamicIVFModel or DynamicIVFSQModel; `allowed_slots` is bool
    [num_slots] (bits of Empty slots are ignored).  Ids are external."""
    oracle, metric = model.oracle, model.metric
    order = probe_order(oracle, metric, queries, model.centroids)
    n = len(model.valid)
    present = np.array(model.valid, dtype=bool)
    cl = np.array([model.cluster[s] if model.valid[s] else NONE32 for s in range(n)], dtype=np.int64)
    keep = present & np.asarray(allowed_slots, dtype=bool)[:n]
    sq = hasattr(model, "scale")

    def distances(i, keys):
        rows = np.stack([model.rows[int(s)] for s in keys])
        if sq:
            return S.distances(oracle, metric, queries[i], rows.astype(model.dtype), model.scale, model.bias)
        return oracle.distance_rows(M.METRICS[metric], queries[i], rows.astype(model.dtype))

    return search(metric, order, cl, present, keep, distances, k, n_probes, np.array(model.ext, dtype=np.uint64),
                   C=model.C)


def bitmap(allowed: np.ndarray) -> np.ndarray:
    """bool [n] -> uint32 [(n + 31) / 32], bit i of word i / 32 = allowed[i]."""
    b = np.packbits(np.asarray(allowed, dtype=bool), bitorder="little")
    b = np.concatenate([b, np.zeros((-len(b)) % 4, dtype=np.uint8)])
    return b.view(np.uint32)
