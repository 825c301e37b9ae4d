#!/usr/bin/env python
"""bench_ivf_sq.py -- the IVF index over float32 rows against the same index over SQ int8 codes; one JSON line.

    python bench_ivf_sq.py [--n 1000000] [--clusters 1024] [--repeats 3] [--profile DIR]

Workload: bench_ivf.py's clustered unit vectors, n x 96 float32, and its 10 000 float32 queries, k = 10, L2 and MIP.
  * one Clustering.build per metric (C = --clusters, default IVFBuildParameters); sq_compress timed on the host around
    the blocking call; both indexes assembled from the same clustering;
  * ground truth: Flat.search at k = 10 over the float32 rows;
  * for n_probes in 1, 4, 16, 64: IVF.search_device of the float32 and the SQ index at k = 10 on device buffers, timed
    with CUDA events, alternating, two rounds of `--repeats` calls each after one warm-up call of each; recall@10
    against the flat result; device_bytes of both indexes.  Progress goes to stderr.
With --profile the n_probes = 16 searches run once more under torch.profiler and the per-kernel CUDA times are written
to DIR/ivf_sq_profile.json.  The card's name and power limit are read in the same run.  Nothing else is written.
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
    from scalablevectorsearch_b200 import (IVF, Clustering, DistanceType, Flat, IVFBuildParameters, IVFSearchParameters,
                                           sq_compress)
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    if not torch.cuda.is_available():
        raise SystemExit("bench_ivf_sq.py needs a CUDA device")
    stream = torch.cuda.current_stream()
    k = 10
    x, q = clustered_unit_vectors(args.n, 10_000, 96)
    dq = torch.from_numpy(q).cuda()
    t0 = time.perf_counter()
    codes, scale, bias = sq_compress(x, np.int8)
    compress_s = time.perf_counter() - t0

    def call(fn):
        ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
        d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn(dq.data_ptr(), np.float32, q.shape[0], k, ids.data_ptr(), d.data_ptr(), stream=stream.cuda_stream or 1)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), ids.cpu().numpy().view(np.uint64)

    out, profiles = {}, {}
    for metric in (DistanceType.L2, DistanceType.MIP):
        clustering = Clustering.build(IVFBuildParameters(num_centroids=args.clusters), x, metric)
        indexes = {"f32": IVF.assemble_from_clustering(clustering, x, metric),
                   "sq_i8": IVF.assemble_from_clustering(clustering, codes, metric, sq=(scale, bias))}
        gt, _ = Flat(x, metric).search(q, k)

        def recall(ids):
            return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / k for a, b in zip(ids, gt)]))

        res = {"device_bytes": {name: ix.device_bytes for name, ix in indexes.items()}}
        for n_probes in (1, 4, 16, 64):
            for ix in indexes.values():
                ix.search_parameters = IVFSearchParameters(n_probes=n_probes)
                call(ix.search_device)
            times = {name: [[], []] for name in indexes}
            rec = {}
            for rnd in range(2):
                for _ in range(args.repeats):
                    for name, ix in indexes.items():
                        ms, ids = call(ix.search_device)
                        times[name][rnd].append(round(ms, 3))
                        rec[name] = recall(ids)
            res[f"n_probes_{n_probes}"] = {"times_ms": times, "recall_at_10": rec}
            print(f"{metric.name} n_probes={n_probes}: {res[f'n_probes_{n_probes}']}", file=sys.stderr, flush=True)
        out[metric.name] = res
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            for name, ix in indexes.items():
                ix.search_parameters = IVFSearchParameters(n_probes=16)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    call(ix.search_device)
                profiles[f"{metric.name}_{name}"] = {ev.key: round(ev.device_time_total / 1000.0, 3)
                                                     for ev in prof.key_averages() if ev.device_type.name == "CUDA"}
    if args.profile:
        os.makedirs(args.profile, exist_ok=True)
        with open(os.path.join(args.profile, "ivf_sq_profile.json"), "w") as f:
            json.dump(profiles, f, indent=1)

    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({"metric": "ivf_sq_search_ms", "n": args.n, "clusters": args.clusters, "k": k, "gpu": card,
                      "sq_compress_s": round(compress_s, 3), "workloads": out}), flush=True)


if __name__ == "__main__":
    main()
