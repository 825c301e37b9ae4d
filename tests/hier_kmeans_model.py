"""A numpy model of the hierarchical k-means contract (include/svsb200.h, svsb200_ivf_cluster_hierarchical; DESIGN.md
§15), needing no GPU, built on the flat k-means model of tests/ivf_model.py: the same random sequence, training sample,
float32 update, split and normalisation, and the oracle's exact distances with ties to the lower centroid."""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

import ivf_model as M


@dataclass
class Result:
    centroids: np.ndarray       # float32 [C][dim], level-1 groups in order
    assignments: np.ndarray     # uint32 [n]
    level2_counts: np.ndarray   # uint32 [L1]: c_g
    train_counts: np.ndarray    # [L1]: t_g
    train_level1: np.ndarray    # [m]: every training row's level-1 group
    level1: np.ndarray          # [n]: every row's level-1 group
    seeds: list                 # the groups' stream seeds
    discarded: int              # remainder draws discarded by the allocation guard
    level1_centroids: np.ndarray = None   # float32 [L1][dim]: the final level-1 centroids


def level1_clusters(num_centroids: int, level1: int) -> int:
    return level1 or int(math.sqrt(float(num_centroids)))


def allocate(t, m: int, C: int, rng: M.Rng):
    """Step 5: c_g = size_t(double(t_g) / m * C), then remainder draws j = r % L1, discarded when t_j = 0 or c_j = t_j.
    Returns (c, discarded draws)."""
    L1 = len(t)
    c = [int(float(tg) / m * C) for tg in t]
    total, discarded = sum(c), 0
    while total < C:
        j = rng.next() % L1
        if t[j] == 0 or c[j] == t[j]:
            discarded += 1
            continue
        c[j] += 1
        total += 1
    return c, discarded


def iterate(oracle, metric: int, rows, rows32, cent, num_iterations: int, m: int, rng: M.Rng):
    """svsb200_ivf_cluster's step 3 over the rows and centroids given, splits drawing from `rng` with m as denominator."""
    C = cent.shape[0]
    for _ in range(num_iterations):
        assign = M.nearest(oracle, metric, rows, cent, 1)[:, 0]
        new = cent.copy()
        counts = np.zeros(C, dtype=np.int64)
        for i in range(rows.shape[0]):   # float32, ascending row order, onto the old centroid
            a = assign[i]
            new[a] = (new[a] + rows32[i]).astype(np.float32)
            counts[a] += 1
        for c in range(C):
            if counts[c]:
                new[c] = (new[c] * np.float32(1.0 / (counts[c] + 1))).astype(np.float32)
        cent = new
        M.split(cent, counts, m, rng)
        if metric != 0:
            cent = M.normalize(cent)
    return cent


def hierarchical_kmeans(oracle, data: np.ndarray, metric: int, num_centroids: int, level1: int, num_iterations: int,
                        training_fraction: float, seed: int) -> Result:
    n, dim = data.shape
    C = num_centroids
    m = M.num_training_rows(n, C, training_fraction)
    if m < C:
        raise ValueError("insufficient data for clustering")
    L1 = level1_clusters(C, level1)
    if L1 > C:
        raise ValueError("level1_clusters must be at most num_centroids")
    ip_like = metric != 0
    rng = M.Rng(seed)
    # 1-3. the sample and the level-1 flat k-means
    sample = np.sort(rng.shuffle_prefix(n, m))
    train = data[sample]
    train32 = M.to_f32(train)
    cent1 = train32[rng.shuffle_prefix(m, L1)].copy()
    if ip_like:
        cent1 = M.normalize(cent1)
    cent1 = iterate(oracle, metric, train, train32, cent1, num_iterations, m, rng)
    # 4-5. the sample's groups, the allocation, the groups' seeds
    tl1 = M.nearest(oracle, metric, train, cent1, 1)[:, 0]
    t = np.bincount(tl1, minlength=L1)
    c, discarded = allocate([int(v) for v in t], m, C, rng)
    seeds = [rng.next() for _ in range(L1)]
    start = np.concatenate([[0], np.cumsum(c)]).astype(np.int64)
    # 7. every group's own k-means
    cent = np.zeros((C, dim), dtype=np.float32)
    for g in range(L1):
        if c[g] == 0:
            continue
        rows = np.flatnonzero(tl1 == g)
        grng = M.Rng(seeds[g])
        cg = train32[rows[grng.shuffle_prefix(int(t[g]), c[g])]].copy()
        if ip_like:
            cg = M.normalize(cg)
        cent[start[g]:start[g + 1]] = iterate(oracle, metric, train[rows], train32[rows], cg, num_iterations, int(t[g]),
                                              grng)
    # 6. every row to the nearest populated level-1 centroid, then 7. to the nearest of its group's centroids
    pop = np.array([g for g in range(L1) if c[g] > 0])
    level1_of = pop[M.nearest(oracle, metric, data, cent1[pop], 1)[:, 0]]
    assign = np.empty(n, dtype=np.uint32)
    for g in pop:
        rows = np.flatnonzero(level1_of == g)
        if rows.size:
            assign[rows] = start[g] + M.nearest(oracle, metric, data[rows], cent[start[g]:start[g + 1]], 1)[:, 0]
    return Result(cent, assign, np.array(c, dtype=np.uint32), t, tl1, level1_of, seeds, discarded, cent1)
