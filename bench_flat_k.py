#!/usr/bin/env python
"""bench_flat_k.py -- the exact search of the flat index (Flat.search_device) against the exact scan, at k = 10 and at
the 100-deep lists users take ground truth with; one JSON line.

    python bench_flat_k.py [--n 1000000] [--repeats 3]

Workloads (L2; k = 10 runs the FLAT_KC lists, k = 100 the deep ones):
  * f32_nq10000_k10 / f32_nq10000_k100: bench.py's clustered unit vectors, n x 96 float32, 10 000 float32 queries;
  * u8_nq10000_k100: bench_build_int.py's BIGANN-shaped n x 128 uint8 rows and uint8 queries (the integer GEMM);
  * f32_nq100_k100, f32_nq256_k100 / f32_nq384_k100: the float32 rows with 100, 256 and 384 queries, the two sides of
    the routing rule: one query tile keeps only 7 CTAs busy with the deep lists, so batches of one or two tiles
    (nq <= 256) run the scan and three tiles or more the GEMM.
Each workload times Flat.search_device and Vamana.exhaustive_device (a graph of zeros: the scan never reads it) over the
same rows with CUDA events on device buffers, alternating, `--repeats` calls each after one warm-up call of each (which
also builds the GEMM's base tiles).  Reported: the times, the fallback counts of the flat calls, and whether every call
returned the same ids and distance bits as the scan.  The card's name and power limit are read in the same run.
Nothing is written to disk.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_build_int import uint8_rows  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    from scalablevectorsearch_b200 import DistanceType, Flat, Vamana
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    if not torch.cuda.is_available():
        raise SystemExit("bench_flat_k.py needs a CUDA device")
    stream = torch.cuda.current_stream()

    def call(fn, dq, k):
        nq = dq.shape[0]
        ids = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        d = torch.empty((nq, k), dtype=torch.float32, device="cuda")
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        r = fn(dq.data_ptr(), np.dtype(str(dq.dtype).replace("torch.", "")), nq, k, ids.data_ptr(), d.data_ptr(),
               stream=stream.cuda_stream or 1)
        t1.record(stream)
        torch.cuda.synchronize()
        return t0.elapsed_time(t1), ids.cpu().numpy(), d.cpu().numpy().view(np.uint32), r

    def measure(x, q, k):
        flat = Flat(x, DistanceType.L2)
        scan = Vamana.from_arrays(x, np.zeros((x.shape[0], 2), dtype=np.uint32), 0, DistanceType.L2)
        dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
        runs = {"flat": flat.search_device, "scan": scan.exhaustive_device}
        for fn in runs.values():
            call(fn, dq, k)
        times, fallbacks, identical = {name: [] for name in runs}, [], True
        for _ in range(args.repeats):
            res = {}
            for name, fn in runs.items():
                ms, ids, b, r = call(fn, dq, k)
                times[name].append(round(ms, 3))
                res[name] = (ids, b)
                if name == "flat":
                    fallbacks.append(int(r))
            identical &= np.array_equal(res["flat"][0], res["scan"][0]) and np.array_equal(res["flat"][1], res["scan"][1])
        del flat, scan
        torch.cuda.empty_cache()
        return {"times_ms": times, "fallback_queries": fallbacks, "identical_ids_and_distance_bits": bool(identical),
                "flat_faster": max(times["flat"]) < min(times["scan"])}

    out = {}
    xf, qf = clustered_unit_vectors(args.n, 10_000, 96)
    out["f32_nq10000_k10"] = measure(xf, qf, 10)
    out["f32_nq10000_k100"] = measure(xf, qf, 100)
    out["f32_nq100_k100"] = measure(xf, qf[:100], 100)
    out["f32_nq256_k100"] = measure(xf, qf[:256], 100)
    out["f32_nq384_k100"] = measure(xf, qf[:384], 100)
    del xf, qf
    xu, qu = uint8_rows(args.n, 128, 10_000)
    out["u8_nq10000_k100"] = measure(xu, qu, 100)
    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({"metric": "flat_index_search_ms", "n": args.n, "gpu": card, "workloads": out}), flush=True)
    if not all(w["identical_ids_and_distance_bits"] for w in out.values()):
        raise SystemExit("bench_flat_k.py: the flat index and the scan returned different results")


if __name__ == "__main__":
    main()
