#!/usr/bin/env python
"""bench_dynamic_sq.py -- the dynamic Vamana index over int8 SQ codes next to the float32 one, through
bench_dynamic.py's mutation script; one JSON line.

    python bench_dynamic_sq.py [--n 1000000] [--repeats 3]

Workload: bench_dynamic.py's (bench.py's C2 data: synthetic n x 96 float32, L2, 10 000 queries, k = 10; GPU builder
R = 64, window 128, alpha 1.2), run once on a float32 DynamicVamana and once on an int8 SQ one (sq_compress of the first
90 % of the rows; the scale and bias stay fixed from there on, and the added float32 rows are encoded with them):
  1. DynamicVamana.build over the first 90 % of the rows;
  2. `add` of the last 10 % in calls of 10 000;
  3. deletion of a random 10 % of the ids;
  4. `consolidate`, then `compact`.
Reported per index: inserted points per second, consolidate and compact milliseconds (host clock around each blocking
call; the build runs the same builder kernels first, so none of them is a cold launch), search QPS at window 128 with
no Deleted slot (after the adds) and with 10 % Deleted (after the deletion) -- best of `--repeats` blocking searches of
all 10 000 queries after one warm-up search --, recall@10 at window 128 after every stage against the exact top 10 over
the live float32 rows (a DynamicFlat mutated in step, outside the timed calls), and device bytes after every stage.
The card's name and power limit are read in the same run.  Nothing is written to disk.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

# bench_dynamic.py's workload (bench.py's "c2-1Mx96-f32-L2-w128")
C2 = dict(dim=96, nq=10_000, k=10, window=128, max_degree=64, build_window=128, alpha=1.2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    from scalablevectorsearch_b200 import (DistanceType, DynamicFlat, DynamicVamana, SearchBufferConfig,
                                           VamanaBuildParameters, _lib, sq_compress)
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    if _lib.lib().svsb200_device_count() == 0:
        raise SystemExit("bench_dynamic_sq.py needs a CUDA device")
    w = C2
    n, k = args.n, w["k"]
    base, queries = clustered_unit_vectors(n, w["nq"], w["dim"])
    n0 = int(0.9 * n)
    gone = np.random.default_rng(0).choice(n, n // 10, replace=False)
    params = VamanaBuildParameters(alpha=w["alpha"], graph_max_degree=w["max_degree"], window_size=w["build_window"])

    def run(kind):
        exact = DynamicFlat.build(base[:n0], np.arange(n0), DistanceType.L2)
        out = {"recall_at_10_w128": {}, "device_bytes": {}, "search_qps_w128": {}}

        def stage(name, index):
            gt = exact.search(queries, k)[0].astype(np.int64)
            index.search_parameters.buffer_config = SearchBufferConfig(w["window"], w["window"])
            ids = index.search(queries, k)[0].astype(np.int64)
            out["recall_at_10_w128"][name] = round(float(np.mean([len(set(a.tolist()) & set(b.tolist()))
                                                                  for a, b in zip(ids, gt)]) / k), 4)
            out["device_bytes"][name] = index.device_bytes

        def qps(name, index):
            index.search_parameters.buffer_config = SearchBufferConfig(w["window"], w["window"])
            index.search(queries, k)   # warm-up
            best = float("inf")
            for _ in range(args.repeats):
                t0 = time.perf_counter()
                index.search(queries, k)
                best = min(best, time.perf_counter() - t0)
            out["search_qps_w128"][name] = round(len(queries) / best, 1)

        t0 = time.perf_counter()
        if kind == "sq_int8":
            codes, scale, bias = sq_compress(base[:n0])
            index = DynamicVamana.build(params, codes, np.arange(n0), DistanceType.L2, sq=(scale, bias))
            out["sq"] = {"scale": scale, "bias": bias}
        else:
            index = DynamicVamana.build(params, base[:n0], np.arange(n0), DistanceType.L2)
        out["build_s"] = round(time.perf_counter() - t0, 3)
        stage("build", index)
        add_s = 0.0
        for lo in range(n0, n, 10_000):
            hi = min(n, lo + 10_000)
            t0 = time.perf_counter()
            index.add(base[lo:hi], np.arange(lo, hi))
            add_s += time.perf_counter() - t0
            exact.add(base[lo:hi], np.arange(lo, hi))
        out["insert_points_per_s"] = round((n - n0) / add_s, 1)
        stage("add", index)
        qps("no_deleted", index)
        index.delete(gone)
        exact.delete(gone)
        stage("delete", index)
        qps("deleted_10pct", index)
        t0 = time.perf_counter()
        index.consolidate()
        out["consolidate_ms"] = round((time.perf_counter() - t0) * 1e3, 2)
        exact.consolidate()
        stage("consolidate", index)
        t0 = time.perf_counter()
        index.compact()
        out["compact_ms"] = round((time.perf_counter() - t0) * 1e3, 2)
        exact.compact()
        stage("compact", index)
        out["size"] = index.size
        return out

    results = {kind: run(kind) for kind in ("float32", "sq_int8")}
    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({"metric": "dynamic_sq_mutations", "workload": f"c2-{n}x96-L2-w128", "gpu": card,
                      "build_points": n0, "added_points": n - n0, "deleted_points": len(gone), **results}), flush=True)


if __name__ == "__main__":
    main()
