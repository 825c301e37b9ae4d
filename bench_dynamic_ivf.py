#!/usr/bin/env python
"""bench_dynamic_ivf.py -- the dynamic IVF index through a mutation script, against the static IVF index; one JSON line.

    python bench_dynamic_ivf.py [--n 1000000] [--clusters 1024] [--repeats 3]

Workload: bench_ivf.py's clustered unit vectors, n x 96 float32, and its 10 000 float32 queries, L2, k = 10.
  1. Clustering.build (C = --clusters, default parameters) over the first 90 % of the rows; DynamicIVF and IVF assembled
     from it;
  2. searches at n_probes 1, 4 and 16, DynamicIVF.search_device alternating with IVF.search_device on device buffers,
     timed with CUDA events, `--repeats` calls each after one warm-up call of each;
  3. two adds of 1 % of n rows each (the device memory before and after shows whether clusters moved);
  4. deletes of 1 % and then 9 % of n ids;
  5. an add of 5 % of n rows with reuse_empty;
  6. the searches again, now against an IVF assembled over the live rows with the same centroids;
  7. compact, and the searches once more.
Mutations are timed on the host around the blocking call.  Every stage reports recall@10 against a DynamicFlat mutated
alongside.  The card's name and power limit are read in the same run.  Nothing is written.
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
    args = ap.parse_args()
    import torch
    from scalablevectorsearch_b200 import (IVF, Clustering, DistanceType, DynamicFlat, DynamicIVF, IVFBuildParameters,
                                           IVFSearchParameters)
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    if not torch.cuda.is_available():
        raise SystemExit("bench_dynamic_ivf.py needs a CUDA device")
    stream = torch.cuda.current_stream()
    k, n = 10, args.n
    x, q = clustered_unit_vectors(n, 10_000, 96)
    n0, a = n * 9 // 10, n // 100
    ids = np.arange(n, dtype=np.uint64)

    t0 = time.perf_counter()
    clustering = Clustering.build(IVFBuildParameters(num_centroids=args.clusters), x[:n0], DistanceType.L2)
    cluster_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    dyn = DynamicIVF.assemble_from_clustering(clustering, x[:n0], ids[:n0], DistanceType.L2)
    assemble_s = time.perf_counter() - t0
    static = IVF.assemble_from_clustering(clustering, x[:n0], DistanceType.L2)
    truth = DynamicFlat.build(x[:n0], ids[:n0], DistanceType.L2)
    dq = torch.from_numpy(q).cuda()

    def call(fn):
        out_i = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
        out_d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn(dq.data_ptr(), np.float32, q.shape[0], k, out_i.data_ptr(), out_d.data_ptr(), stream=stream.cuda_stream or 1)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out_i.cpu().numpy().view(np.uint64)

    def searches(static_index, static_ids):
        gt, _ = truth.search(q, k)
        res = {}
        for n_probes in (1, 4, 16):
            dyn.search_parameters = IVFSearchParameters(n_probes=n_probes)
            static_index.search_parameters = IVFSearchParameters(n_probes=n_probes)
            runs = {"dynamic": dyn.search_device, "static": static_index.search_device}
            for fn in runs.values():
                call(fn)
            times = {name: [] for name in runs}
            got = {}
            for _ in range(args.repeats):
                for name, fn in runs.items():
                    ms, out = call(fn)
                    times[name].append(round(ms, 3))
                    got[name] = out
            ok = got["static"] != np.uint64(2**64 - 1)
            mapped = np.full_like(got["static"], np.uint64(2**64 - 1))
            mapped[ok] = static_ids[got["static"][ok].astype(np.int64)]
            rec = {name: float(np.mean([len(set(r.tolist()) & set(g.tolist())) / k for r, g in zip(v, gt)]))
                   for name, v in (("dynamic", got["dynamic"]), ("static", mapped))}
            res[f"n_probes_{n_probes}"] = {"times_ms": times, "recall_at_10": rec}
        return res

    def timed(fn):
        t0 = time.perf_counter()
        fn()
        return round(time.perf_counter() - t0, 4)

    stages, mutations = {}, {}
    stages["assembled"] = searches(static, ids[:n0])
    for i, (lo, hi) in enumerate(((n0, n0 + a), (n0 + a, n0 + 2 * a))):
        before = dyn.device_bytes
        mutations[f"add_{i}"] = {"rows": hi - lo, "s": timed(lambda: dyn.add(x[lo:hi], ids[lo:hi])),
                                 "device_bytes_before": before, "device_bytes_after": dyn.device_bytes}
        truth.add(x[lo:hi], ids[lo:hi])
    rng = np.random.default_rng(0)
    live = dyn.all_ids()
    gone = rng.choice(live, 10 * a, replace=False)
    for name, part in (("delete_small", gone[:a]), ("delete_large", gone[a:])):
        mutations[name] = {"ids": len(part), "s": timed(lambda: dyn.delete(part))}
        truth.delete(part)
    lo, hi = n0 + 2 * a, min(n, n0 + 7 * a)
    mutations["add_reuse"] = {"rows": hi - lo, "s": timed(lambda: dyn.add(x[lo:hi], ids[lo:hi], reuse_empty=True))}
    truth.add(x[lo:hi], ids[lo:hi], reuse_empty=True)
    status, ext, _ = dyn.export()
    live_ids = ext[status == 1]
    tombstones = 1.0 - len(live_ids) / (len(live_ids) + 10 * a)
    live_static = IVF.assemble_from_clustering(Clustering(clustering.centroids), x[live_ids.astype(np.int64)],
                                               DistanceType.L2)
    stages["tombstones"] = {"share": round(tombstones, 4), "device_bytes": dyn.device_bytes,
                            **searches(live_static, live_ids)}
    mutations["compact"] = {"s": timed(dyn.compact)}
    stages["compacted"] = {"device_bytes": dyn.device_bytes, **searches(live_static, live_ids)}

    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({"metric": "dynamic_ivf_search_ms", "n": n, "clusters": args.clusters, "k": k, "gpu": card,
                      "clustering_s": round(cluster_s, 3), "assemble_s": round(assemble_s, 3), "mutations": mutations,
                      "stages": stages}), flush=True)


if __name__ == "__main__":
    main()
