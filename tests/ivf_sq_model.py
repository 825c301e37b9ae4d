"""A numpy model of the SQ IVF index (include/svsb200.h, svsb200_sq_compress and svsb200_ivf_create_sq; DESIGN.md §15),
needing no GPU.

Compression is SQDataset::compress spelt out in float32.  Distances are the SQ search path's: L2 is the exact integer
sum scaled by scale^2; MIP and cosine come from the C oracle's float trees (``oracle_distance_rows``) over the codes
as float32 rows, with the query preparation of InnerProductCompressed / CosineSimilarityCompressed spelt out here.  The
probe and the union top k are tests/ivf_model.py's.
"""
from __future__ import annotations

import numpy as np

import ivf_model as M

RANGE = {np.dtype(np.int8): (-128.0, 127.0), np.dtype(np.uint8): (0.0, 255.0)}


def compress(data: np.ndarray, dtype=np.int8):
    """svsb200_sq_compress: (codes, scale, bias) with every operation rounded to float32 on its own."""
    x = np.ascontiguousarray(data, dtype=np.float32).reshape(-1)
    lo, hi = (np.float32(v) for v in RANGE[np.dtype(dtype)])
    mn, mx = x.min(), x.max()
    if mn == 0:   # the sequential `x < mn ? x : mn` keeps the first zero it meets
        mn = x[np.flatnonzero(x == 0)[0]]
    scale = np.float32(np.float32(mx - mn) / np.float32(hi - lo))
    bias = np.float32(mn - np.float32(lo * scale))
    return encode(data, dtype, scale, bias), float(scale), float(bias)


def encode(data: np.ndarray, dtype, scale: float, bias: float) -> np.ndarray:
    """detail::compress: clamp(roundf((x - bias) / scale), MIN, MAX), halves away from zero."""
    lo, hi = RANGE[np.dtype(dtype)]
    r = (np.asarray(data, dtype=np.float32) - np.float32(bias)).astype(np.float32) / np.float32(scale)
    r = r.astype(np.float32).astype(np.float64)
    r = np.sign(r) * np.floor(np.abs(r) + 0.5)   # exact in float64 for float32 inputs
    return np.clip(r, lo, hi).astype(dtype)


def query_f32(q: np.ndarray) -> np.ndarray:
    """The SQ queries as float32, element by element: the reference's scalar float16 conversion flushes subnormals."""
    if q.dtype == np.float16:
        f = q.astype(np.float32)
        return np.where(np.abs(f) < np.float32(2.0**-14), np.copysign(np.float32(0), f), f).astype(np.float32)
    return q.astype(np.float32)


def _reduce4(q: np.ndarray) -> np.float32:
    """std::reduce over float32 (libstdc++: four at a time, (x0 + x1) + (x2 + x3), then the tail)."""
    acc = np.float32(0)
    n = q.shape[0]
    i = 0
    while i + 4 <= n:
        acc = np.float32(acc + np.float32(np.float32(q[i] + q[i + 1]) + np.float32(q[i + 2] + q[i + 3])))
        i += 4
    for j in range(i, n):
        acc = np.float32(acc + q[j])
    return acc


def distances(oracle, metric: int, query: np.ndarray, codes: np.ndarray, scale: float, bias: float) -> np.ndarray:
    """The SQ search path's distances of one query to every code row."""
    q = query_f32(query)
    s, b = np.float32(scale), np.float32(bias)
    if metric == 0:   # EuclideanCompressed: scale^2 * float(sum (qc - x)^2), int32
        qc = encode(q, codes.dtype, scale, bias).astype(np.int64)
        l2 = ((codes.astype(np.int64) - qc) ** 2).sum(axis=1)
        l2 = ((l2 + 2**31) % 2**32 - 2**31).astype(np.int32)
        return (np.float32(s * s) * l2.astype(np.float32)).astype(np.float32)
    if metric == 1:   # InnerProductCompressed: scale * <q, x> + bias * sum(q)
        ip = oracle.distance_rows("ip", q, codes.astype(np.float32))
        return ((s * ip).astype(np.float32) + np.float32(b * _reduce4(q))).astype(np.float32)
    rows = ((s * codes.astype(np.float32)).astype(np.float32) + b).astype(np.float32)   # decompress, then cosine
    return oracle.distance_rows("cosine", q, rows)


def search(oracle, metric: int, codes: np.ndarray, scale: float, bias: float, centroids: np.ndarray,
           assignments: np.ndarray, queries: np.ndarray, k: int, n_probes: int):
    """svsb200_ivf_search on an SQ index: the exact top k over the probed clusters' rows, by (distance, id)."""
    nq = queries.shape[0]
    ids = np.full((nq, k), M.PAD_ID, dtype=np.uint64)
    dists = np.full((nq, k), np.inf if metric == 0 else -np.inf, dtype=np.float32)
    probes = M.nearest(oracle, metric, queries, centroids, n_probes)
    for i, q in enumerate(queries):
        rows = np.flatnonzero(np.isin(assignments, probes[i]))
        if rows.size == 0:
            continue
        d = distances(oracle, metric, q, codes[rows], scale, bias)
        key = d if metric == 0 else -d
        order = np.lexsort((rows, key))[:k]
        ids[i, :order.size] = rows[order]
        dists[i, :order.size] = d[order]
    return ids, dists
