"""A numpy model of the IVF index's contract (include/svsb200.h, svsb200_ivf_*; DESIGN.md §15), needing no GPU.

Distances come from the C oracle (``oracle_distance_rows``), so they are the search path's bit-exact ones; every other
step (the random sequence, the training sample, the float32 k-means sums, the split, the normalisation, the probe, the
union top k) is spelt out here in float32 as the library does it.
"""
from __future__ import annotations

import math

import numpy as np

MASK64 = (1 << 64) - 1
EPSILON = 1.0 / 1024.0
MIN_TRAINING_SAMPLE_MULTIPLIER = 2
METRICS = {0: "l2", 1: "ip", 2: "cosine"}
PAD_ID = np.uint64(2**64 - 1)


class Rng:
    """splitmix64, the library's documented sequence (svsb200_ivf_random)."""

    def __init__(self, seed: int):
        self.state = int(seed) & MASK64

    def next(self) -> int:
        self.state = (self.state + 0x9E3779B97F4A7C15) & MASK64
        z = self.state
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
        return z ^ (z >> 31)

    def uniform(self) -> np.float32:
        return np.float32((self.next() >> 40) * 2.0**-24)

    def shuffle_prefix(self, n: int, m: int) -> np.ndarray:
        """The first m of a Fisher-Yates shuffle of [0, n)."""
        perm = np.arange(n, dtype=np.int64)
        for i in range(m):
            j = i + self.next() % (n - i)
            perm[i], perm[j] = perm[j], perm[i]
        return perm[:m].copy()


def random_sequence(seed: int, count: int) -> list[int]:
    r = Rng(seed)
    return [r.next() for _ in range(count)]


def num_training_rows(n: int, num_centroids: int, training_fraction: float) -> int:
    lo = min(num_centroids * MIN_TRAINING_SAMPLE_MULTIPLIER, n)
    return min(n, max(lo, int(math.ceil(np.float32(n) * np.float32(training_fraction)))))


def to_f32(x: np.ndarray) -> np.ndarray:
    return np.asarray(x).astype(np.float32)


def normalize(cent: np.ndarray) -> np.ndarray:
    """normalize_centroids: x * (1 / sqrt(sequential float32 sum of squares)); zero rows untouched."""
    cent = cent.astype(np.float32, copy=True)
    acc = np.zeros(cent.shape[0], dtype=np.float32)
    for d in range(cent.shape[1]):
        acc = (acc + cent[:, d] * cent[:, d]).astype(np.float32)
    norm = np.sqrt(acc).astype(np.float32)
    nz = norm != 0
    inv = (np.float32(1.0) / norm[nz]).astype(np.float32)
    cent[nz] = (cent[nz] * inv[:, None]).astype(np.float32)
    return cent


def nearest(oracle, metric: int, queries: np.ndarray, centroids: np.ndarray, count: int) -> np.ndarray:
    """The `count` centroids nearest to each query under the metric, ties to the lower index: [nq][count]."""
    out = np.empty((queries.shape[0], count), dtype=np.int64)
    idx = np.arange(centroids.shape[0])
    for i, q in enumerate(queries):
        d = oracle.distance_rows(METRICS[metric], q, centroids)
        key = d if metric == 0 else -d
        out[i] = np.lexsort((idx, key))[:count]
    return out


def split(cent: np.ndarray, counts: np.ndarray, m: int, rng: Rng) -> None:
    """centroid_split with the documented sequence, in place."""
    C, dim = cent.shape
    up, down = 1.0 + EPSILON, 1.0 - EPSILON
    even = np.arange(dim) % 2 == 0
    for i in range(C):
        if counts[i] != 0:
            continue
        j = 0
        while True:
            if counts[j] != 0:
                p = np.float32(np.float32(counts[j]) / np.float32(m))
                if rng.uniform() < p:
                    break
            j = (j + 1) % C
        cent[i] = cent[j]
        ci, cj = cent[i].astype(np.float64), cent[j].astype(np.float64)
        cent[i] = (ci * np.where(even, up, down)).astype(np.float32)
        cent[j] = (cj * np.where(even, down, up)).astype(np.float32)
        counts[i] = counts[j] // 2
        counts[j] -= counts[i]


def kmeans(oracle, data: np.ndarray, metric: int, num_centroids: int, num_iterations: int, training_fraction: float,
           seed: int):
    """svsb200_ivf_cluster: (centroids float32 [C][dim], assignments uint32 [n])."""
    n = data.shape[0]
    C = num_centroids
    m = num_training_rows(n, C, training_fraction)
    if m < C:
        raise ValueError("insufficient data for clustering")
    rng = Rng(seed)
    sample = np.sort(rng.shuffle_prefix(n, m))
    init = rng.shuffle_prefix(m, C)
    train = data[sample]
    train32 = to_f32(train)
    cent = train32[init].copy()
    ip_like = metric != 0
    if ip_like:
        cent = normalize(cent)
    for _ in range(num_iterations):
        assign = nearest(oracle, metric, train, cent, 1)[:, 0]
        new = cent.copy()
        counts = np.zeros(C, dtype=np.int64)
        for i in range(m):   # float32, ascending row order, onto the old centroid
            a = assign[i]
            new[a] = (new[a] + train32[i]).astype(np.float32)
            counts[a] += 1
        for c in range(C):
            if counts[c]:
                new[c] = (new[c] * np.float32(1.0 / (counts[c] + 1))).astype(np.float32)
        cent = new
        split(cent, counts, m, rng)
        if ip_like:
            cent = normalize(cent)
    assign = nearest(oracle, metric, data, cent, 1)[:, 0].astype(np.uint32)
    return cent, assign


def search(oracle, metric: int, data: np.ndarray, centroids: np.ndarray, assignments: np.ndarray, queries: np.ndarray,
           k: int, n_probes: int):
    """svsb200_ivf_search: the exact top k over the union of the n_probes nearest clusters' rows, ordered by
    (distance, id), padded with all-ones ids and +-inf."""
    nq = queries.shape[0]
    ids = np.full((nq, k), PAD_ID, dtype=np.uint64)
    dists = np.full((nq, k), np.inf if metric == 0 else -np.inf, dtype=np.float32)
    probes = nearest(oracle, metric, queries, centroids, n_probes)
    for i, q in enumerate(queries):
        rows = np.flatnonzero(np.isin(assignments, probes[i]))
        if rows.size == 0:
            continue
        d = oracle.distance_rows(METRICS[metric], q, data[rows])
        key = d if metric == 0 else -d
        order = np.lexsort((rows, key))[:k]
        ids[i, :order.size] = rows[order]
        dists[i, :order.size] = d[order]
    return ids, dists
