#!/usr/bin/env python
"""bench_flat_filtered.py -- the Flat index's filtered exact search against its plain search and against what a caller
does without it; one JSON line.

    python bench_flat_filtered.py [--n 1000000] [--repeats 3]

Workload: bench.py's clustered unit vectors, n x 96 float32, and its 10 000 float32 queries, L2, k = 10 and 100.
Masks: random masks over the ids letting 100 %, 50 %, 10 %, 5 %, 1 %, 0.1 % and 0.01 % of the rows through.  For
every (mask, k), alternating, `--repeats` calls each after one warm-up call of each, timed with CUDA events:
  * filtered: Flat.search_filtered_device on device buffers;
  * plain:    Flat.search_device (no filter) on device buffers;
  * rebuild:  a Flat built from the allowed rows (host copy, upload, first-search tiling) and searched on device
              buffers, the ids mapped back on the device: what a caller does today.
The route the filtered search takes (filter_route), its fallback count, and whether its ids and distance bits equal
the rebuild's are reported.  The card's name and power limit are read in the same run.  Nothing is written.
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
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    from scalablevectorsearch_b200 import DistanceType, Flat
    from scalablevectorsearch_b200._lib import _bitmap
    from scalablevectorsearch_b200.flat import filter_route
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    if not torch.cuda.is_available():
        raise SystemExit("bench_flat_filtered.py needs a CUDA device")
    stream = torch.cuda.current_stream()
    sid = stream.cuda_stream or 1
    nq = 10_000
    x, q = clustered_unit_vectors(args.n, nq, 96)
    flat = Flat(x, DistanceType.L2)
    dq = torch.from_numpy(q).cuda()
    rng = np.random.default_rng(0)
    masks = {f"random_{p}%": rng.random(args.n) < p / 100.0 for p in (100, 50, 10, 5, 1, 0.1, 0.01)}

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return round(e0.elapsed_time(e1), 3)

    out = {}
    for k in (10, 100):
        ids = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        d = torch.empty((nq, k), dtype=torch.float32, device="cuda")
        rids = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        rd = torch.empty((nq, k), dtype=torch.float32, device="cuda")
        for name, mask in masks.items():
            allowed = np.flatnonzero(mask)
            dbm = torch.from_numpy(_bitmap(mask, args.n).view(np.int32).copy()).cuda()
            fallback = [0]

            def filtered():
                fallback[0] = flat.search_filtered_device(dq.data_ptr(), np.float32, nq, k, dbm.data_ptr(), ids.data_ptr(),
                                                          d.data_ptr(), stream=sid)

            def plain():
                flat.search_device(dq.data_ptr(), np.float32, nq, k, ids.data_ptr(), d.data_ptr(), stream=sid)

            def rebuild():
                sub = Flat(np.ascontiguousarray(x[allowed]), DistanceType.L2)
                sub.search_device(dq.data_ptr(), np.float32, nq, k, rids.data_ptr(), rd.data_ptr(), stream=sid)
                pad = rids == -1
                back = torch.from_numpy(allowed).cuda()[rids.clamp(min=0)]
                rids.copy_(torch.where(pad, rids, back))
                rd.masked_fill_(pad, float("inf"))

            runs = {"filtered": filtered, "plain": plain}
            if len(allowed):
                runs["rebuild"] = rebuild
            for fn in runs.values():
                timed(fn)
            times = {r: [] for r in runs}
            for _ in range(args.repeats):
                for r, fn in runs.items():
                    times[r].append(timed(fn))
            timed(filtered)
            same = None
            if len(allowed):
                timed(rebuild)
                same = bool(torch.equal(ids, rids) and torch.equal(d.view(torch.int32), rd.view(torch.int32)))
            out[f"{name}/k_{k}"] = {"times_ms": times, "allowed": int(len(allowed)),
                                    "route": filter_route(args.n, len(allowed)), "fallback_queries": int(fallback[0]),
                                    "equal_to_rebuild": same}

    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({"metric": "flat_filtered_search_ms", "n": args.n, "nq": nq, "gpu": card, "workloads": out}),
          flush=True)


if __name__ == "__main__":
    main()
