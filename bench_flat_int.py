#!/usr/bin/env python
"""bench_flat_int.py -- the exact flat search over uint8 rows on the integer tensor cores, against the fp16 path over
the same values and the exact scan; one JSON line.

    python bench_flat_int.py [--n 1000000] [--nq 10000] [--repeats 3]

Workload: bench_build_int.py's BIGANN-shaped rows (bench.py's clustered unit vectors mapped affinely onto 0..255),
n x 128 uint8, with nq uint8 queries of the same law through the same mapping, k = 10, L2.  Each index comes from
Vamana.from_arrays with a graph of zeros (the flat search never reads it).  Three calls are timed with CUDA events
on device buffers, alternating, `--repeats` times each:
  * flat_search_device on the uint8 index: the integer GEMM (wgmma s8/u8, exact int32 keys);
  * flat_search_device on a float32 index of the same values with the same queries as float32: the fp16 GEMM;
  * exhaustive_device on the uint8 index: the exact scan (dp4a, one warp per query and base range).
The first flat call of each index also builds its base tiles: the tile build is reported as that call's time less
the median of the same call's timed repeats (for the fp16 index both include its scan fallbacks, which cancel).  At dim
128 every distance is below 2^24, so all three must return the same ids and distance bits, which is checked.  The
rate is 2 nq n dim / time, against the data-sheet dense INT8 (and FP16) rate of the H100 SXM.  The card's name and
power limit are read in the same run.  Nothing is written to disk.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_build_int import uint8_rows  # noqa: E402

DATASHEET_DENSE_INT8_TOPS = 1979.0   # H100 SXM, 700 W
DATASHEET_DENSE_FP16_TFLOPS = 989.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    from scalablevectorsearch_b200 import DistanceType, Vamana
    if not torch.cuda.is_available():
        raise SystemExit("bench_flat_int.py needs a CUDA device")
    x, q = uint8_rows(args.n, args.dim, args.nq)
    graph = np.zeros((args.n, 2), dtype=np.uint32)
    u8 = Vamana.from_arrays(x, graph, 0, DistanceType.L2)
    f32 = Vamana.from_arrays(x.astype(np.float32), graph, 0, DistanceType.L2)
    dq = {"u8": torch.from_numpy(q).cuda(), "f32": torch.from_numpy(q.astype(np.float32)).cuda()}
    qdtype = {"u8": np.dtype(np.uint8), "f32": np.dtype(np.float32)}
    stream = torch.cuda.current_stream()
    nq, k = args.nq, args.k

    def call(index, fn, qk):
        ids = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        d = torch.empty((nq, k), dtype=torch.float32, device="cuda")
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        r = getattr(index, fn)(dq[qk].data_ptr(), qdtype[qk], nq, k, ids.data_ptr(), d.data_ptr(),
                               stream=stream.cuda_stream or 1)
        t1.record(stream)
        torch.cuda.synchronize()
        return t0.elapsed_time(t1), ids.cpu().numpy(), d.cpu().numpy(), r

    runs = {"int_gemm": (u8, "flat_search_device", "u8"), "fp16_gemm": (f32, "flat_search_device", "f32"),
            "exact_scan": (u8, "exhaustive_device", "u8")}
    first = {name: round(call(*runs[name])[0], 3) for name in ("int_gemm", "fp16_gemm")}   # also builds the base tiles
    call(*runs["exact_scan"])
    times = {name: [] for name in runs}
    fallbacks = {"int_gemm": [], "fp16_gemm": []}
    results = {}
    for _ in range(args.repeats):
        for name, spec in runs.items():
            ms, ids, d, r = call(*spec)
            times[name].append(round(ms, 3))
            if name in fallbacks:
                fallbacks[name].append(int(r))
            results[name] = (ids, d.view(np.uint32))
    ref_ids, ref_bits = results["exact_scan"]
    identical = all(np.array_equal(i, ref_ids) and np.array_equal(b, ref_bits) for i, b in results.values())
    ops = 2.0 * nq * args.n * args.dim
    best = {name: min(t) for name, t in times.items()}
    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    tile_build = {name: round(first[name] - float(np.median(times[name])), 3) for name in first}
    print(json.dumps({
        "metric": "flat_search_ms", "workload": f"synthetic-{args.n}x{args.dim}-u8-L2-nq{nq}-k{k}", "gpu": card,
        "times_ms": times, "first_call_ms": first, "tile_build_ms": tile_build, "fallback_queries": fallbacks,
        "identical_ids_and_distance_bits": identical,
        "tops_at_best": {name: round(ops / (t * 1e-3) / 1e12, 1) for name, t in best.items()},
        "datasheet_dense_tops": {"int8": DATASHEET_DENSE_INT8_TOPS, "fp16": DATASHEET_DENSE_FP16_TFLOPS},
        "int_gemm_share_of_int8_datasheet": round(ops / (best["int_gemm"] * 1e-3) / 1e12 / DATASHEET_DENSE_INT8_TOPS, 4),
    }), flush=True)
    if not identical:
        raise SystemExit("bench_flat_int.py: the three paths returned different results")


if __name__ == "__main__":
    main()
