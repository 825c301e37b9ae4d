#!/usr/bin/env python
"""bench_dynamic_ivf_sq.py -- the dynamic IVF index over int8 SQ codes next to the float32 one, through
bench_dynamic_ivf.py's mutation script; one JSON line.

    python bench_dynamic_ivf_sq.py [--n 1000000] [--clusters 1024] [--repeats 3]

Workload: bench_ivf.py's clustered unit vectors, n x 96 float32, and its 10 000 float32 queries, L2, k = 10.
  1. Clustering.build (C = --clusters, default parameters) over the first 90 % of the rows; a float32 DynamicIVF and an
     int8 SQ DynamicIVF (sq_compress of those rows: the scale and bias stay fixed from here on) assembled from it;
  2. searches at n_probes 1, 4 and 16, the two indexes' search_device alternating on device buffers, timed with CUDA
     events, `--repeats` calls each after one warm-up call of each;
  3. two adds of 1 % of n rows each (float32 rows to both; the SQ index encodes them);
  4. deletes of 1 % and then 9 % of n ids;
  5. an add of 5 % of n rows with reuse_empty;
  6. the searches again;
  7. compact, and the searches once more.
Mutations are timed on the host around the blocking call.  Every stage reports recall@10 against a DynamicFlat mutated
alongside, and the recall of a static SQ IVF over the live codes (in slot order, each in the cluster the dynamic index
holds it in), which the SQ dynamic index must equal; device_bytes of both indexes at every stage.  The card's name and
power limit are read in the same run.  Nothing is written.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

PAD = np.uint64(2**64 - 1)


def encode(x, scale, bias):
    """SQDataset::set_datum into int8: clamp(roundf((x - bias) / scale), -128, 127), halves away from zero."""
    r = ((x - np.float32(bias)).astype(np.float32) / np.float32(scale)).astype(np.float32).astype(np.float64)
    return np.clip(np.sign(r) * np.floor(np.abs(r) + 0.5), -128, 127).astype(np.int8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--clusters", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    from scalablevectorsearch_b200 import (IVF, Clustering, DistanceType, DynamicFlat, DynamicIVF, IVFBuildParameters,
                                           IVFSearchParameters, sq_compress)
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    if not torch.cuda.is_available():
        raise SystemExit("bench_dynamic_ivf_sq.py needs a CUDA device")
    stream = torch.cuda.current_stream()
    k, n = 10, args.n
    x, q = clustered_unit_vectors(n, 10_000, 96)
    n0, a = n * 9 // 10, n // 100
    ids = np.arange(n, dtype=np.uint64)

    clustering = Clustering.build(IVFBuildParameters(num_centroids=args.clusters), x[:n0], DistanceType.L2)
    t0 = time.perf_counter()
    codes, scale, bias = sq_compress(x[:n0])
    compress_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    sq = DynamicIVF.assemble_from_clustering(clustering, codes, ids[:n0], DistanceType.L2, sq=(scale, bias))
    assemble_sq_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    f32 = DynamicIVF.assemble_from_clustering(clustering, x[:n0], ids[:n0], DistanceType.L2)
    assemble_f32_s = time.perf_counter() - t0
    truth = DynamicFlat.build(x[:n0], ids[:n0], DistanceType.L2)
    indexes = {"float32": f32, "sq_int8": sq}
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

    def recall(found, gt):
        return float(np.mean([len(set(r.tolist()) & set(g.tolist())) / k for r, g in zip(found, gt)]))

    def stage():
        """Searches of both indexes, recall against the flat truth and against a static SQ IVF over the live codes."""
        gt, _ = truth.search(q, k)
        status, ext, cluster = sq.export()
        live = status == 1
        live_ids = ext[live]
        static = IVF.assemble_from_clustering(Clustering(clustering.centroids, cluster[live]),
                                              encode(x[live_ids.astype(np.int64)], scale, bias), DistanceType.L2,
                                              sq=(scale, bias))
        res = {"device_bytes": {name: index.device_bytes for name, index in indexes.items()},
               "live_rows": int(live.sum()), "empty_slots": int(sq.num_slots - live.sum())}
        for n_probes in (1, 4, 16):
            for index in (*indexes.values(), static):
                index.search_parameters = IVFSearchParameters(n_probes=n_probes)
            runs = {name: index.search_device for name, index in indexes.items()}
            for fn in runs.values():
                call(fn)
            times = {name: [] for name in runs}
            got = {}
            for _ in range(args.repeats):
                for name, fn in runs.items():
                    ms, out = call(fn)
                    times[name].append(round(ms, 3))
                    got[name] = out
            s_ids, _ = static.search(q, k)
            mapped = np.full_like(s_ids, PAD)
            ok = s_ids != PAD
            mapped[ok] = live_ids[s_ids[ok].astype(np.int64)]
            rec = {name: recall(v, gt) for name, v in got.items()}
            rec["sq_int8_static"] = recall(mapped, gt)
            res[f"n_probes_{n_probes}"] = {"times_ms": times, "recall_at_10": rec,
                                           "sq_equals_static": bool(np.array_equal(got["sq_int8"], mapped))}
        return res

    def timed(fn):
        t0 = time.perf_counter()
        fn()
        return round(time.perf_counter() - t0, 4)

    def mutate(name, what, fn):
        entry = {}
        for label, index in indexes.items():
            entry[label] = {"s": timed(lambda: fn(index)), "device_bytes": index.device_bytes}
        mutations[name] = {**what, **entry}

    stages, mutations = {}, {}
    stages["assembled"] = stage()
    for i, (lo, hi) in enumerate(((n0, n0 + a), (n0 + a, n0 + 2 * a))):
        mutate(f"add_{i}", {"rows": hi - lo}, lambda index: index.add(x[lo:hi], ids[lo:hi]))
        truth.add(x[lo:hi], ids[lo:hi])
    rng = np.random.default_rng(0)
    gone = rng.choice(sq.all_ids(), 10 * a, replace=False)
    for name, part in (("delete_small", gone[:a]), ("delete_large", gone[a:])):
        mutate(name, {"ids": len(part)}, lambda index: index.delete(part))
        truth.delete(part)
    lo, hi = n0 + 2 * a, min(n, n0 + 7 * a)
    mutate("add_reuse", {"rows": hi - lo}, lambda index: index.add(x[lo:hi], ids[lo:hi], reuse_empty=True))
    truth.add(x[lo:hi], ids[lo:hi], reuse_empty=True)
    stages["tombstones"] = stage()
    mutate("compact", {}, lambda index: index.compact())
    stages["compacted"] = stage()

    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({"metric": "dynamic_ivf_sq_search_ms", "n": n, "clusters": args.clusters, "k": k, "gpu": card,
                      "sq_compress_s": round(compress_s, 3), "assemble_s": {"float32": round(assemble_f32_s, 3),
                                                                            "sq_int8": round(assemble_sq_s, 3)},
                      "mutations": mutations, "stages": stages}), flush=True)


if __name__ == "__main__":
    main()
