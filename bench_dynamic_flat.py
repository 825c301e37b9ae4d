#!/usr/bin/env python
"""bench_dynamic_flat.py -- the dynamic flat index's mutations and searches on the GPU, one JSON line.

    python bench_dynamic_flat.py [--repeats 5]

Workload: bench.py's C2 data (synthetic 1M x 96 float32, L2, 10 000 queries).  DynamicFlat.build over the first 900 000
rows and one search (which tiles them for the tensor cores); `add` of the last 100 000 rows in calls of 10 000; deletion
of a random 10 % of the 1M (in two calls, 10 000 and 90 000 ids); `add` of 50 000 new rows with reuse_empty; `compact`.
Reported:
  * milliseconds of every add call, of the deletion, of the reuse_empty add and of the compaction (host clock around
    each blocking call; the tiles are kept exact by every mutation, so the adds include their re-tiling);
  * after the deletion (1M slots, 10 % Empty): search_device at k = 10, k = 100 and k = 200 (the scan route: the masked
    scan over the slots) against a static Flat over 1M rows (the same number of slots) and against the exact scan
    (Vamana.exhaustive_device over the same 1M rows), timed with CUDA events, alternating, `--repeats` calls each after
    one warm-up call of each; the fallback counts;
  * after every stage: whether the index returned the ids and distance bits of a static Flat over the live rows in slot
    order, ids mapped to the external ids (k = 10, 100 and 200);
  * the card's name and power limit, read in the same run.
Nothing is written to disk.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

# bench.py's "c2-1Mx96-f32-L2-w128" rows and queries
C2 = dict(n=1_000_000, dim=96, nq=10_000)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    from scalablevectorsearch_b200 import DistanceType, DynamicFlat, Flat, Vamana
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    if not torch.cuda.is_available():
        raise SystemExit("bench_dynamic_flat.py needs a CUDA device")
    stream = torch.cuda.current_stream()
    n, n0 = C2["n"], int(0.9 * C2["n"])
    base, queries = clustered_unit_vectors(n, C2["nq"], C2["dim"])
    extra, _ = clustered_unit_vectors(n + 50_000, 1, C2["dim"])
    extra = extra[n:]                              # rows for the reuse_empty add, outside the 1M
    dq = torch.from_numpy(queries).cuda()
    rows_of = np.full(n + 50_000, -1, dtype=np.int64)   # external id -> its row in `base` / `extra` (stacked)
    pool = np.concatenate([base, extra])

    def call(fn, k):
        nq = dq.shape[0]
        ids = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        d = torch.empty((nq, k), dtype=torch.float32, device="cuda")
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        r = fn(dq.data_ptr(), np.float32, nq, k, ids.data_ptr(), d.data_ptr(), stream=stream.cuda_stream or 1)
        t1.record(stream)
        torch.cuda.synchronize()
        return t0.elapsed_time(t1), ids.cpu().numpy().view(np.uint64), d.cpu().numpy().view(np.uint32), r

    def identical(index):
        """The index's result == a static Flat over the live rows in slot order, ids mapped (k = 10, 100 and 200)."""
        ext = index.all_ids()
        flat = Flat(pool[rows_of[ext.astype(np.int64)]], DistanceType.L2)
        ok = True
        for k in (10, 100, 200):
            _, gi, gd, _ = call(index.search_device, k)
            _, fi, fd, _ = call(flat.search_device, k)
            ok &= np.array_equal(gi, ext[fi.astype(np.int64)]) and np.array_equal(gd, fd)
        del flat
        torch.cuda.empty_cache()
        return bool(ok)

    def timed(f):
        t0 = time.time()
        f()
        return round((time.time() - t0) * 1e3, 3)

    out = {}
    index = DynamicFlat.build(base[:n0], np.arange(n0), DistanceType.L2)
    rows_of[:n0] = np.arange(n0)
    out["first_search_ms"] = round(call(index.search_device, 10)[0], 3)   # includes tiling the 900 000 rows
    same = {"build": identical(index)}
    out["add_ms"] = []
    for lo in range(n0, n, 10_000):
        out["add_ms"].append(timed(lambda: index.add(base[lo:lo + 10_000], np.arange(lo, lo + 10_000))))
        rows_of[lo:lo + 10_000] = np.arange(lo, lo + 10_000)
    same["add"] = identical(index)
    gone = np.random.default_rng(0).choice(n, n // 10, replace=False)
    out["delete_ms"] = [timed(lambda: index.delete(gone[:10_000])), timed(lambda: index.delete(gone[10_000:]))]
    same["delete"] = identical(index)

    # 1M slots, 10 % Empty: this index against a static Flat over 1M rows and against the scan over them
    flat = Flat(base, DistanceType.L2)
    scan = Vamana.from_arrays(base, np.zeros((n, 2), dtype=np.uint32), 0, DistanceType.L2)
    runs = {"dynamic_flat": index.search_device, "flat_1M": flat.search_device, "scan_1M": scan.exhaustive_device}
    out["search"] = {}
    for k in (10, 100, 200):
        for fn in runs.values():
            call(fn, k)
        times, fallbacks = {name: [] for name in runs}, {"dynamic_flat": [], "flat_1M": []}
        for _ in range(args.repeats):
            for name, fn in runs.items():
                ms, _, _, r = call(fn, k)
                times[name].append(round(ms, 3))
                if name in fallbacks:
                    fallbacks[name].append(int(r))
        out["search"][f"k{k}"] = {"times_ms": times, "fallback_queries": fallbacks}
    del flat, scan
    torch.cuda.empty_cache()

    new_ids = np.arange(n, n + 50_000)
    out["add_reuse_empty_50000_ms"] = timed(lambda: index.add(extra, new_ids, reuse_empty=True))
    rows_of[n:] = np.arange(n, n + 50_000)
    same["add_reuse_empty"] = identical(index)
    out["compact_ms"] = timed(lambda: index.compact())
    same["compact"] = identical(index)
    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or None
    print(json.dumps({"metric": "dynamic_flat", "workload": "c2-1Mx96-f32-L2", "gpu": card, "build_points": n0,
                      "add_ms_mean": round(float(np.mean(out["add_ms"])), 3), **out, "size": index.size,
                      "slots": index.num_slots, "identical_to_static_flat_over_live_rows": same}), flush=True)
    if not all(same.values()):
        raise SystemExit("bench_dynamic_flat.py: the dynamic flat index and the static Flat returned different results")


if __name__ == "__main__":
    main()
