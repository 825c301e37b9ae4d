#!/usr/bin/env python
"""bench_ivf_hier.py -- hierarchical against flat k-means for the IVF index: clustering time and recall; one JSON line.

    python bench_ivf_hier.py [--n 1000000] [--clusters 1024,4096,16384] [--probes 1,4,16]

Workload: bench.py's clustered unit vectors, n x 96 float32, and its 10 000 float32 queries, L2, k = 10.  For every C:
  * Clustering.build (flat) and Clustering.build_hierarchical (level-1 groups: sqrt(C)), default IVFBuildParameters
    otherwise (10 iterations, a 10 % training sample), each timed on the host around the blocking call;
  * an IVF over each clustering, searched at every n_probes; recall@10 against Flat.search over the same rows.
The flat k-means assigns every row against all C centroids per pass; the hierarchical one against sqrt(C) level-1
centroids, then against the ~sqrt(C) centroids of its own group, which is why it should gain as C grows.  The card's
name and power limit are read in the same run.  Nothing is written.
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
    ap.add_argument("--clusters", default="1024,4096,16384")
    ap.add_argument("--probes", default="1,4,16")
    args = ap.parse_args()
    import torch
    from scalablevectorsearch_b200 import IVF, Clustering, DistanceType, Flat, IVFBuildParameters, IVFSearchParameters
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    if not torch.cuda.is_available():
        raise SystemExit("bench_ivf_hier.py needs a CUDA device")
    k = 10
    x, q = clustered_unit_vectors(args.n, 10_000, 96)
    gt, _ = Flat(x, DistanceType.L2).search(q, k)

    def recall(ids):
        return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / k for a, b in zip(ids, gt)]))

    builders = {"flat": Clustering.build, "hierarchical": Clustering.build_hierarchical}
    out = {}
    for C in (int(c) for c in args.clusters.split(",")):
        bp = IVFBuildParameters(num_centroids=C)
        row = {}
        for name, build in builders.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            clustering = build(bp, x, DistanceType.L2)
            seconds = time.perf_counter() - t0
            index = IVF.assemble_from_clustering(clustering, x, DistanceType.L2)
            sizes = index.cluster_sizes
            rec = {}
            for n_probes in (int(p) for p in args.probes.split(",")):
                index.search_parameters = IVFSearchParameters(n_probes=n_probes)
                rec[f"n_probes_{n_probes}"] = round(recall(index.search(q, k)[0]), 4)
            row[name] = {"clustering_s": round(seconds, 3), "recall_at_10": rec,
                         "cluster_sizes": {"min": int(sizes.min()), "max": int(sizes.max()),
                                           "empty": int((sizes == 0).sum())}}
            del index
        row["speedup"] = round(row["flat"]["clustering_s"] / row["hierarchical"]["clustering_s"], 2)
        out[f"C_{C}"] = row

    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({"metric": "ivf_clustering_s", "n": args.n, "dim": 96, "k": k, "gpu": card, "workloads": out}),
          flush=True)


if __name__ == "__main__":
    main()
