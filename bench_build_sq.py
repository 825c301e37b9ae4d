#!/usr/bin/env python
"""bench_build_sq.py -- the Vamana graph built and searched over SQ int8 codes against float32 rows, one JSON line.

    python bench_build_sq.py [--n 1000000] [--repeats 2]

Workload: bench.py's clustered unit vectors, n x 96 float32, and 10 000 queries of the same law; L2, R = 64, window 128,
alpha 1.2.  The SQ side compresses the rows to int8 codes with one global scale and bias (sq_compress, not timed) and
builds over the codes (svsb200_build_vamana_sq); the float32 side builds over the rows (svsb200_build_vamana).  Each
build is timed with a host clock around the blocking call, after one small warm-up build of each kind; the two kinds
alternate, `--repeats` times each.  Both indexes are then searched with the float32 queries at window 128, k = 10:
queries per second from a host clock around blocking searches (best of three after a warm-up), recall@10 against the
exact flat scan over the float32 rows.  Device bytes are each index's HBM footprint.  The card's name and power limit
are read in the same run.  Nothing is written to disk.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    from scalablevectorsearch_b200 import (DistanceType, SearchBufferConfig, Vamana, VamanaBuildParameters,
                                           build_graph)
    from scalablevectorsearch_b200.ivf import sq_compress
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    x, q = clustered_unit_vectors(args.n, 10_000, 96)
    codes, scale, bias = sq_compress(x)
    params = VamanaBuildParameters(alpha=1.2, graph_max_degree=64, window_size=128)
    kinds = {"float32": (x, None), "sq_int8": (codes, (scale, bias))}   # float32 first: its exact scan is the truth
    for data, sq in kinds.values():   # module loads, first-launch costs
        build_graph(data[:20_000], DistanceType.L2, params, sq=sq)
    times = {k: [] for k in kinds}
    graphs = {}
    for _ in range(args.repeats):
        for name, (data, sq) in kinds.items():
            t0 = time.time()
            graphs[name] = build_graph(data, DistanceType.L2, params, sq=sq)
            times[name].append(round(time.time() - t0, 3))
    result = {}
    gt = None
    for name, (data, sq) in kinds.items():
        graph, ep = graphs[name]
        index = Vamana.from_arrays(data, graph, ep, DistanceType.L2, sq=sq)
        if gt is None:
            gt = index.flat_search(q, 10)[0]
        index.search_parameters.buffer_config = SearchBufferConfig(128)
        ids, _ = index.search(q, 10)
        best = float("inf")
        for _ in range(3):
            t0 = time.time()
            index.search(q, 10)
            best = min(best, time.time() - t0)
        recall = float(np.mean([len(set(a.tolist()) & set(b.tolist())) / 10.0 for a, b in zip(ids, gt)]))
        result[name] = {"build_s": times[name], "device_bytes": int(index.device_bytes),
                        "qps_w128": round(q.shape[0] / best), "recall10_w128": round(recall, 4),
                        "mean_degree": round(float(graph[:, 0].mean()), 3)}
        del index
    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({"metric": "build_wall_s", "workload": f"synthetic-{args.n}x96-L2", "gpu": card,
                      "parameters": {"graph_max_degree": 64, "window_size": 128, "alpha": 1.2, "search_window": 128},
                      **result}), flush=True)


if __name__ == "__main__":
    main()
