"""Generate the committed golden fixtures under tests/golden/ (run in the authoring container).

Inputs : /root/reference/data/test_dataset (the reference's own 10k x 128 fixtures, prebuilt
         Vamana graph, ground truth) and oracle/_ref/libsvsref.so (the reference compiled
         from /root/reference by `make -C oracle ref`).
Outputs: test_dataset.npz   compact copy of the fixtures the parity tests need on the GPU box
         ref_outputs.npz    ids / distances / work counters the *reference itself* produces
         golden_recalls.json the 17 (window, capacity) -> recall@10 goldens of
                            data/test_dataset/reference/vamana_reference.toml (vamana_test_search)
         ref_builder.json   entry point, mean degree and recall@10 of graphs from the reference's own
                            builder, for the GPU builder's tests (tests/test_gpu_build.py)

    python tests/golden/make_golden.py [--builder-only]
"""
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.bindings import RefLib  # noqa: E402
from scalablevectorsearch_b200 import io  # noqa: E402

SRC = "/root/reference/data/test_dataset"
OUT = os.path.dirname(os.path.abspath(__file__))


def parse_goldens(path):
    """Pull (distance, window, capacity, recall) of every vamana_test_search entry."""
    text = open(path).read()
    out = {}
    for block in text.split("[[vamana_test_search]]")[1:]:
        block = block.split("[[vamana_test_build]]")[0]
        dist = re.search(r"distance = '(\w+)'", block).group(1)
        entries = []
        for sub in block.split("[[vamana_test_search.config_and_recall]]")[1:]:
            recall = float(re.search(r"^\s*recall = ([0-9.eE+-]+)", sub, re.M).group(1))
            cap = int(re.search(r"search_buffer_capacity = (\d+)", sub).group(1))
            win = int(re.search(r"search_window_size = (\d+)", sub).group(1))
            k = int(re.search(r"num_neighbors = (\d+)", sub).group(1))
            nq = int(re.search(r"num_queries = (\d+)", sub).group(1))
            entries.append({"window": win, "capacity": cap, "recall": recall, "k": k, "num_queries": nq})
        out[{"L2": "l2", "MIP": "ip", "Cosine": "cosine"}[dist]] = entries
    return out


def recall_at_k(ids, gt, k=10):
    return sum(len(set(r[:k].tolist()) & set(t[:k].tolist())) for r, t in zip(ids, gt)) / (k * len(ids))


def builder_goldens(ref):
    """The reference builder's side of tests/test_gpu_build.py, searched with the reference's own search (bit-exact
    with the GPU search, so these are the recalls that test would measure on the reference's graphs)."""
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    z = np.load(f"{OUT}/test_dataset.npz")
    X, Q = z["data"].astype(np.float32), z["queries"].astype(np.float32)
    out = {"test_dataset": {}}
    for metric in ("l2", "ip", "cosine"):
        alpha = 1.2 if metric == "l2" else 0.95
        g, ep = ref.build(X, metric, 32, 64, alpha=alpha, threads=4)
        idx = ref.index(X, g, ep, metric, threads=4)
        out["test_dataset"][metric] = {
            "max_degree": 32, "window_size": 64, "alpha": alpha, "entry_point": int(ep),
            "mean_degree": float(g[:, 0].mean()),
            "recall": {str(w): recall_at_k(idx.search(Q, 10, w, w)[0], z[f"gt_{metric}"]) for w in (10, 30)}}
    base, queries = clustered_unit_vectors(30_000, 500, 96)
    base16 = base.astype(np.float16)
    x = base16.astype(np.float32)
    d = (queries ** 2).sum(1)[:, None] + (x ** 2).sum(1)[None, :] - 2.0 * queries @ x.T
    gt = np.argsort(d, axis=1, kind="stable")[:, :10]
    g, ep = ref.build(base16, "l2", 64, 128, alpha=1.2, threads=8)
    ids = ref.index(base16, g, ep, "l2", threads=8).search(queries, 10, 64, 64)[0]
    out["synthetic_30000x96_f16_l2"] = {"max_degree": 64, "window_size": 128, "alpha": 1.2, "search_window": 64,
                                         "recall": recall_at_k(ids, gt)}
    json.dump(out, open(f"{OUT}/ref_builder.json", "w"), indent=1)


def main():
    ref = RefLib()
    assert ref.avx512(), "goldens must come from the AVX-512 expression tree"
    if "--builder-only" in sys.argv:
        builder_goldens(ref)
        return
    X = io.read_svs(f"{SRC}/data_f32.svs", np.float32)
    G = io.read_graph(f"{SRC}/graph_128.svs")
    Q = io.read_vecs(f"{SRC}/queries_f32.fvecs")
    assert np.array_equal(X, np.round(X)) and np.abs(X).max() <= 127
    assert np.array_equal(Q, np.round(Q)) and np.abs(Q).max() <= 127
    ep = int(re.search(r"entry_point = (\d+)", open(f"{SRC}/vamana_config.toml").read()).group(1))
    gts = {m: io.read_vecs(f"{SRC}/groundtruth_{f}.ivecs")[:, :10].astype(np.uint32)
           for m, f in (("l2", "euclidean"), ("ip", "mip"), ("cosine", "cosine"))}
    np.savez_compressed(f"{OUT}/test_dataset.npz", data=X.astype(np.int8), graph=G, queries=Q.astype(np.int8),
                        entry_point=np.uint32(ep), gt_l2=gts["l2"], gt_ip=gts["ip"], gt_cosine=gts["cosine"])

    goldens = parse_goldens(f"{SRC}/reference/vamana_reference.toml")
    json.dump(goldens, open(f"{OUT}/golden_recalls.json", "w"), indent=1)

    outs = {}
    threads = os.cpu_count() or 1
    # (a) the 17 golden configurations, f32 data / f32 queries, last 900 queries
    for metric, entries in goldens.items():
        idx = ref.index(X, G, ep, metric, threads=threads)
        for e in entries:
            ids, dists = idx.search(Q[100:], 10, e["window"], e["capacity"])
            tag = f"{metric}_f32_f32_w{e['window']}_c{e['capacity']}"
            outs[tag + "_ids"] = ids.astype(np.uint32)
            outs[tag + "_dists"] = dists
        hops, evals = idx.counts(Q[:64], 32, 48)
        outs[f"{metric}_counts_w32_c48_hops"] = hops.astype(np.uint32)
        outs[f"{metric}_counts_w32_c48_evals"] = evals.astype(np.uint32)
    # (b) every supported (query, data) element-type pair at one split-buffer configuration
    variants = {
        "f32_f16": (Q, X.astype(np.float16)), "f16_f16": (Q.astype(np.float16), X.astype(np.float16)),
        "f16_f32": (Q.astype(np.float16), X), "f32_i8": (Q, X.astype(np.int8)),
        "i8_i8": (Q.astype(np.int8), X.astype(np.int8)),
        "f32_u8": (Q, (X + 127).astype(np.uint8)),
        "u8_u8": ((Q + 127).astype(np.uint8), (X + 127).astype(np.uint8)),
    }
    for metric in goldens:
        for name, (q, x) in variants.items():
            idx = ref.index(x, G, ep, metric, threads=threads)
            ids, dists = idx.search(q[:256], 10, 24, 40)
            outs[f"{metric}_{name}_w24_c40_ids"] = ids.astype(np.uint32)
            outs[f"{metric}_{name}_w24_c40_dists"] = dists
        # (c) scalar quantisation: the reference compresses, we keep codes + scale/bias
        for code in (np.int8, np.uint8):
            idx, codes, scale, bias = ref.sq_index(X * np.float32(0.37) + np.float32(1.5), G, ep, metric, code,
                                                   threads=threads)
            cname = np.dtype(code).name
            if metric == "l2":
                outs[f"sq_{cname}_codes"] = codes
                outs[f"sq_{cname}_scale_bias"] = np.array([scale, bias], dtype=np.float32)
            for qn, q in (("f32", Q * np.float32(0.37) + np.float32(1.5)),
                          ("f16", (Q * np.float32(0.37) + np.float32(1.5)).astype(np.float16))):
                ids, dists = idx.search(q[:256], 10, 24, 40)
                outs[f"{metric}_sq_{cname}_{qn}_w24_c40_ids"] = ids.astype(np.uint32)
                outs[f"{metric}_sq_{cname}_{qn}_w24_c40_dists"] = dists
    np.savez_compressed(f"{OUT}/ref_outputs.npz", **outs)
    builder_goldens(ref)
    for f in ("test_dataset.npz", "ref_outputs.npz", "golden_recalls.json", "ref_builder.json"):
        print(f, os.path.getsize(f"{OUT}/{f}") // 1024, "KiB")


if __name__ == "__main__":
    main()
