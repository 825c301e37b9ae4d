#!/usr/bin/env python
"""bench_build_int.py -- wall time of the GPU graph builder on uint8 rows and on the same values as float32, one JSON
line.

    python bench_build_int.py [--n 1000000] [--repeats 2]

Workload: BIGANN-shaped, n x 128 uint8 (bench.py's clustered unit vectors, mapped affinely onto 0..255), L2, R = 64,
window 128, alpha 1.2 (the builder settings of bench.py's C2).  The same values as float32 take four times the device
memory and the float expression tree; the uint8 build runs exact int32 distances.  Each build is timed with a host
clock around the blocking svsb200_build_vamana call (build_graph), after one small warm-up build of each type; the two
types alternate, `--repeats` times each.  The card's name and power limit are read in the same run.  Nothing is written
to disk.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def uint8_rows(n, dim, nq=0):
    """n base rows; with nq > 0, also nq queries of the same law through the same mapping (clipped to 0..255)."""
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(n, max(nq, 1), dim)
    lo, hi = float(base.min()), float(base.max())
    rows = np.rint((base - lo) * (255.0 / (hi - lo))).astype(np.uint8)
    if nq == 0:
        return rows
    return rows, np.rint(np.clip((queries - lo) * (255.0 / (hi - lo)), 0.0, 255.0)).astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    from scalablevectorsearch_b200 import DistanceType, VamanaBuildParameters, build_graph
    params = VamanaBuildParameters(alpha=1.2, graph_max_degree=64, window_size=128)
    u8 = uint8_rows(args.n, args.dim)
    f32 = u8.astype(np.float32)
    for x in (u8[:20_000], f32[:20_000]):   # module loads, first-launch costs
        build_graph(x, DistanceType.L2, params)
    times = {"uint8": [], "float32": []}
    degree = {}
    for _ in range(args.repeats):
        for name, x in (("uint8", u8), ("float32", f32)):
            t0 = time.time()
            graph, _ = build_graph(x, DistanceType.L2, params)
            times[name].append(round(time.time() - t0, 3))
            degree[name] = round(float(graph[:, 0].mean()), 3)
    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({
        "metric": "build_wall_s", "workload": f"synthetic-{args.n}x{args.dim}-u8-L2", "gpu": card,
        "parameters": {"graph_max_degree": 64, "window_size": 128, "alpha": 1.2},
        "uint8_s": times["uint8"], "float32_s": times["float32"], "mean_degree": degree,
    }), flush=True)


if __name__ == "__main__":
    main()
