#!/usr/bin/env python
"""bench_dynamic.py -- cost of the dynamic index's mutations on the GPU, one JSON line.

    python bench_dynamic.py

Workload: bench.py's C2 data (synthetic 1M x 96 float32, L2, 10k queries, k = 10; GPU builder R = 64, window 128,
alpha 1.2).  DynamicVamana.build over the first 90 % of the rows, `add` of the last 10 % in calls of 10 000, deletion
of a random 10 %, `consolidate`, `compact`.  Reported: points inserted per second (host clock around the blocking
`add` calls), consolidate and compact milliseconds (host clock around each blocking call), recall@10 at window 128
after every stage against exact ground truth over the live rows (a DynamicFlat, the library's exact flat index, mutated
in step with the graph index, outside the timed calls), and the card's name and power limit read in the same run.
Nothing is written to disk.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

# bench.py's "c2-1Mx96-f32-L2-w128"
C2 = dict(n=1_000_000, dim=96, nq=10_000, k=10, window=128, max_degree=64, build_window=128, alpha=1.2)


def main():
    from scalablevectorsearch_b200 import DistanceType, DynamicFlat, DynamicVamana, SearchBufferConfig, VamanaBuildParameters
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    w = C2
    base, queries = clustered_unit_vectors(w["n"], w["nq"], w["dim"])
    n, n0, k = w["n"], int(0.9 * w["n"]), w["k"]
    # ground truth: the exact top k over the live rows, from a dynamic flat index given the same mutations
    exact = DynamicFlat.build(base[:n0], np.arange(n0), DistanceType.L2)

    def recall(index):
        """recall@k at window 128 against the exact top k over the live rows."""
        gt = exact.search(queries, k)[0].astype(np.int64)
        index.search_parameters.buffer_config = SearchBufferConfig(w["window"], w["window"])
        ids = index.search(queries, k)[0].astype(np.int64)
        return float(np.mean([len(set(a.tolist()) & set(b.tolist())) for a, b in zip(ids, gt)]) / k)

    t0 = time.time()
    index = DynamicVamana.build(VamanaBuildParameters(alpha=w["alpha"], graph_max_degree=w["max_degree"],
                                                      window_size=w["build_window"]), base[:n0], np.arange(n0),
                                DistanceType.L2)
    build_s = time.time() - t0
    rec = {"build": recall(index)}
    add_s = 0.0
    for lo in range(n0, n, 10_000):
        hi = min(n, lo + 10_000)
        t0 = time.time()
        index.add(base[lo:hi], np.arange(lo, hi))
        add_s += time.time() - t0
        exact.add(base[lo:hi], np.arange(lo, hi))
    rec["add"] = recall(index)
    gone = np.random.default_rng(0).choice(n, n // 10, replace=False)
    index.delete(gone)
    exact.delete(gone)
    rec["delete"] = recall(index)
    t0 = time.time()
    index.consolidate()
    consolidate_ms = (time.time() - t0) * 1e3
    exact.consolidate()
    rec["consolidate"] = recall(index)
    t0 = time.time()
    index.compact()
    compact_ms = (time.time() - t0) * 1e3
    exact.compact()
    rec["compact"] = recall(index)
    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({
        "metric": "dynamic_mutations", "workload": "c2-1Mx96-f32-L2-w128", "gpu": card,
        "build_points": n0, "build_s": round(build_s, 3), "added_points": n - n0,
        "insert_points_per_s": round((n - n0) / add_s, 1), "deleted_points": len(gone),
        "consolidate_ms": round(consolidate_ms, 2), "compact_ms": round(compact_ms, 2),
        "recall_at_10_w128": rec, "size": index.size, "slots": index.num_slots,
        "mutation_parameters": {"alpha": index.alpha, "window": index.construction_window_size,
                                "max_candidates": index.max_candidates, "prune_to": index.prune_to},
    }), flush=True)


if __name__ == "__main__":
    main()
