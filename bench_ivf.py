#!/usr/bin/env python
"""bench_ivf.py -- the IVF index (k-means build and cluster-probed search) against the exact flat search; one JSON line.

    python bench_ivf.py [--n 1000000] [--clusters 1024] [--repeats 3] [--profile DIR]

Workload: bench.py's clustered unit vectors, n x 96 float32, and its 10 000 float32 queries, L2, k = 10.
  * the clustering: Clustering.build with C = --clusters and the default IVFBuildParameters (10 iterations, a 10 %
    training sample), timed on the host around the blocking call;
  * ground truth: Flat.search at k = 10 over the same rows;
  * for n_probes in 1, 4, 16, 64: IVF.search_device and Flat.search_device at k = 10 on device buffers, timed with CUDA
    events, alternating, `--repeats` calls each after one warm-up call of each; recall@10 against the flat result.
With --profile the n_probes = 16 search runs once more under torch.profiler and the per-kernel CUDA times are written
to DIR/ivf_profile.json.  The card's name and power limit are read in the same run.  Nothing else is written.
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
    ap.add_argument("--clusters", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    import torch
    from scalablevectorsearch_b200 import IVF, Clustering, DistanceType, Flat, IVFBuildParameters, IVFSearchParameters
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    if not torch.cuda.is_available():
        raise SystemExit("bench_ivf.py needs a CUDA device")
    stream = torch.cuda.current_stream()
    k = 10
    x, q = clustered_unit_vectors(args.n, 10_000, 96)

    t0 = time.perf_counter()
    clustering = Clustering.build(IVFBuildParameters(num_centroids=args.clusters), x, DistanceType.L2)
    cluster_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    index = IVF.assemble_from_clustering(clustering, x, DistanceType.L2)
    assemble_s = time.perf_counter() - t0
    sizes = index.cluster_sizes
    flat = Flat(x, DistanceType.L2)
    gt, _ = flat.search(q, k)

    dq = torch.from_numpy(q).cuda()

    def call(fn):
        ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
        d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn(dq.data_ptr(), np.float32, q.shape[0], k, ids.data_ptr(), d.data_ptr(), stream=stream.cuda_stream or 1)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), ids.cpu().numpy().view(np.uint64)

    def recall(ids):
        return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / k for a, b in zip(ids, gt)]))

    out = {}
    for n_probes in (1, 4, 16, 64):
        index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        runs = {"ivf": index.search_device, "flat": flat.search_device}
        for fn in runs.values():
            call(fn)
        times = {name: [] for name in runs}
        for _ in range(args.repeats):
            for name, fn in runs.items():
                ms, ids = call(fn)
                times[name].append(round(ms, 3))
                if name == "ivf":
                    r = recall(ids)
        out[f"n_probes_{n_probes}"] = {"times_ms": times, "recall_at_10": r}

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        index.search_parameters = IVFSearchParameters(n_probes=16)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(index.search_device)
        kernels = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA":
                kernels[ev.key] = round(ev.device_time_total / 1000.0, 3)
        os.makedirs(args.profile, exist_ok=True)
        with open(os.path.join(args.profile, "ivf_profile.json"), "w") as f:
            json.dump(kernels, f, indent=1)

    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({"metric": "ivf_search_ms", "n": args.n, "clusters": args.clusters, "k": k, "gpu": card,
                      "clustering_s": round(cluster_s, 3), "assemble_s": round(assemble_s, 3),
                      "cluster_sizes": {"min": int(sizes.min()), "max": int(sizes.max()), "empty": int((sizes == 0).sum())},
                      "workloads": out}), flush=True)


if __name__ == "__main__":
    main()
