#!/usr/bin/env python
"""bench_ivf_filtered.py -- the IVF index's filtered search against its plain search; one JSON line.

    python bench_ivf_filtered.py [--n 1000000] [--clusters 1024] [--repeats 3]

Workload: bench.py's clustered unit vectors, n x 96 float32, and its 10 000 float32 queries, L2, k = 10, an IVF index
over C = --clusters k-means clusters (default IVFBuildParameters).
  * masks: random masks over the ids letting 100 %, 50 %, 10 %, 1 % and 0.1 % of the rows through, and one letting
    through the rows of a random 10 % of the clusters;
  * ground truth per mask: Flat.search at k = 10 over the allowed rows only, ids mapped back;
  * for n_probes in 1, 4, 16 and every mask: IVF.search_filtered_device and the plain IVF.search_device at k = 10 on
    device buffers, timed with CUDA events, alternating, `--repeats` calls each after one warm-up call of each; the
    mean probe count the filtered search used, and its recall@10 against the filtered ground truth.
The card's name and power limit are read in the same run.  Nothing is written.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--clusters", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    from scalablevectorsearch_b200 import IVF, Clustering, DistanceType, Flat, IVFBuildParameters, IVFSearchParameters
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    if not torch.cuda.is_available():
        raise SystemExit("bench_ivf_filtered.py needs a CUDA device")
    stream = torch.cuda.current_stream()
    k, nq = 10, 10_000
    x, q = clustered_unit_vectors(args.n, nq, 96)
    clustering = Clustering.build(IVFBuildParameters(num_centroids=args.clusters), x, DistanceType.L2)
    index = IVF.assemble_from_clustering(clustering, x, DistanceType.L2)
    rng = np.random.default_rng(0)
    masks = {f"random_{p}%": rng.random(args.n) < p / 100.0 for p in (100, 50, 10, 1, 0.1)}
    some = rng.choice(args.clusters, max(1, args.clusters // 10), replace=False)
    masks["clusters_10%"] = np.isin(clustering.assignments, some)

    dq = torch.from_numpy(q).cuda()
    ids = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    d = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    probes = torch.empty(nq, dtype=torch.int32, device="cuda")

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return round(e0.elapsed_time(e1), 3)

    def plain():
        index.search_device(dq.data_ptr(), np.float32, nq, k, ids.data_ptr(), d.data_ptr(), stream=stream.cuda_stream or 1)

    out = {}
    for name, mask in masks.items():
        allowed = np.flatnonzero(mask)
        gt_local, _ = Flat(np.ascontiguousarray(x[allowed]), DistanceType.L2).search(q, k)
        gt = np.where(gt_local < len(allowed), allowed[np.minimum(gt_local, len(allowed) - 1).astype(np.int64)], -1)
        bitmap = np.packbits(mask, bitorder="little")
        bitmap = np.concatenate([bitmap, np.zeros((-len(bitmap)) % 4, dtype=np.uint8)]).view(np.int32)
        dbm = torch.from_numpy(bitmap.copy()).cuda()

        def filtered():
            index.search_filtered_device(dq.data_ptr(), np.float32, nq, k, dbm.data_ptr(), ids.data_ptr(), d.data_ptr(),
                                         probes.data_ptr(), stream=stream.cuda_stream or 1)

        for n_probes in (1, 4, 16):
            index.search_parameters = IVFSearchParameters(n_probes=n_probes)
            runs = {"filtered": filtered, "plain": plain}
            for fn in runs.values():
                timed(fn)
            times = {r: [] for r in runs}
            for _ in range(args.repeats):
                for r, fn in runs.items():
                    times[r].append(timed(fn))
            timed(filtered)
            got = ids.cpu().numpy()
            p = probes.cpu().numpy()
            rec = float(np.mean([len(set(a.tolist()) & set(b.tolist()) - {-1}) / k for a, b in zip(got, gt)]))
            out[f"{name}/n_probes_{n_probes}"] = {"times_ms": times, "mean_probes": round(float(p.mean()), 2),
                                                  "recall_at_10": round(rec, 4), "allowed": int(len(allowed))}

    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({"metric": "ivf_filtered_search_ms", "n": args.n, "clusters": args.clusters, "k": k, "nq": nq,
                      "gpu": card, "workloads": out}), flush=True)


if __name__ == "__main__":
    main()
