"""Pin the oracle: the plain-C restatement vs (a) the reference's 17 golden recalls, (b) the committed
outputs of the reference itself, (c) the compiled reference live (when oracle/_ref loads here),
(d) a double-precision model with the reference's own tolerance."""
import numpy as np
import pytest

from conftest import bits, knn_graph, recall_at_k


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
def test_oracle_reproduces_golden_recalls_and_reference_outputs(oracle, dataset, ref_outputs, golden_recalls, metric):
    idx = oracle.index(dataset.data, dataset.graph, dataset.entry_point, metric)
    for e in golden_recalls[metric]:
        ids, dists = idx.search(dataset.queries[100:], 10, e["window"], e["capacity"])
        # tests/integration/vamana/index_search.cpp:138,189-190
        assert abs(recall_at_k(ids, dataset.gt[metric][100:]) - e["recall"]) < 0.0005
        tag = f"{metric}_f32_f32_w{e['window']}_c{e['capacity']}"
        assert np.array_equal(ids, ref_outputs[tag + "_ids"].astype(np.uint64)), tag
        assert np.array_equal(bits(dists), bits(ref_outputs[tag + "_dists"])), tag
    hops, evals = idx.counts(dataset.queries[:64], 32, 48)
    assert np.array_equal(hops, ref_outputs[f"{metric}_counts_w32_c48_hops"])
    assert np.array_equal(evals, ref_outputs[f"{metric}_counts_w32_c48_evals"])


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("pair", ["f32_f16", "f16_f16", "f16_f32", "f32_i8", "i8_i8", "f32_u8", "u8_u8"])
def test_oracle_element_type_pairs(oracle, dataset, ref_outputs, metric, pair):
    q, x = dataset.variant(pair)
    ids, dists = oracle.index(x, dataset.graph, dataset.entry_point, metric).search(q[:256], 10, 24, 40)
    tag = f"{metric}_{pair}_w24_c40"
    assert np.array_equal(ids, ref_outputs[tag + "_ids"].astype(np.uint64)), tag
    assert np.array_equal(bits(dists), bits(ref_outputs[tag + "_dists"])), tag


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("code", [np.int8, np.uint8])
def test_oracle_scalar_quantisation(oracle, dataset, ref_outputs, metric, code):
    raw = dataset.data * np.float32(0.37) + np.float32(1.5)
    idx, codes, scale, bias = oracle.sq_index(raw, dataset.graph, dataset.entry_point, metric, code)
    name = np.dtype(code).name
    assert np.array_equal(codes, ref_outputs[f"sq_{name}_codes"])
    assert np.array_equal(np.array([scale, bias], dtype=np.float32), ref_outputs[f"sq_{name}_scale_bias"])
    qf = dataset.queries * np.float32(0.37) + np.float32(1.5)
    for qn, q in (("f32", qf), ("f16", qf.astype(np.float16))):
        ids, dists = idx.search(q[:256], 10, 24, 40)
        tag = f"{metric}_sq_{name}_{qn}_w24_c40"
        assert np.array_equal(ids, ref_outputs[tag + "_ids"].astype(np.uint64)), tag
        assert np.array_equal(bits(dists), bits(ref_outputs[tag + "_dists"])), tag


def test_oracle_distances_vs_double_precision(oracle):
    """tests/svs/core/distances/distance_euclidean.cpp:42-78: D = 160 and ragged 223, every pair, against a
    double reference with Catch::Approx's default epsilon (100 * FLT_EPSILON relative)."""
    rng = np.random.default_rng(5)
    eps = 100 * np.finfo(np.float32).eps
    for dim in (160, 223):
        for qd, xd in ((np.float32, np.float32), (np.float32, np.float16), (np.float16, np.float16),
                       (np.float32, np.int8), (np.int8, np.int8), (np.uint8, np.uint8)):
            def draw(dt, shape):
                if np.issubdtype(dt, np.integer):
                    info = np.iinfo(dt)
                    return rng.integers(info.min, info.max + 1, shape).astype(dt)
                return rng.standard_normal(shape).astype(dt)
            q, x = draw(qd, dim), draw(xd, (64, dim))
            qq, xx = q.astype(np.float64), x.astype(np.float64)
            want = {"l2": ((xx - qq) ** 2).sum(1), "ip": xx @ qq,
                    "cosine": (xx @ qq) / (np.sqrt((xx * xx).sum(1)) * np.sqrt((qq * qq).sum()))}
            for metric, w in want.items():
                got = oracle.distance_rows(metric, q, x).astype(np.float64)
                scale = np.maximum(np.abs(w), 1.0) if metric != "l2" else np.abs(w)
                assert np.all(np.abs(got - w) <= eps * np.maximum(scale, 1e-30) * 4), (dim, qd, xd, metric)


def test_oracle_matches_compiled_reference_live(oracle, reflib):
    """Bit-exact distances and searches against oracle/_ref on fresh random inputs (non-integer data)."""
    rng = np.random.default_rng(11)
    for dim in (17, 96, 100, 768):
        q = rng.standard_normal(dim).astype(np.float32)
        x = rng.standard_normal((40, dim)).astype(np.float32)
        for metric in ("l2", "ip", "cosine"):
            for qq, xx in ((q, x), (q, x.astype(np.float16)), (q.astype(np.float16), x.astype(np.float16))):
                assert np.array_equal(bits(oracle.distance_rows(metric, qq, xx)), bits(reflib.distance_rows(metric, qq, xx)))
    n, dim = 1200, 48
    x = rng.standard_normal((n, dim)).astype(np.float32)
    qs = rng.standard_normal((100, dim)).astype(np.float32)
    graph = knn_graph(x, 12, rng)
    for metric in ("l2", "ip", "cosine"):
        a = oracle.index(x, graph, 5, metric).search(qs, 5, 9, 14)
        b = reflib.index(x, graph, 5, metric).search(qs, 5, 9, 14)
        assert np.array_equal(a[0], b[0]) and np.array_equal(bits(a[1]), bits(b[1]))
        a = oracle.index(x, graph, 5, metric).search(qs, 5, 9, 14, visited_set=True)
        assert np.array_equal(a[0], b[0]) and np.array_equal(bits(a[1]), bits(b[1]))


def test_oracle_edge_cases(oracle):
    """Isolated entry point (fewer than k reachable), zero-degree nodes, capacity < k bump, window 1."""
    rng = np.random.default_rng(3)
    x = rng.standard_normal((50, 16)).astype(np.float32)
    q = rng.standard_normal((7, 16)).astype(np.float32)
    graph = np.zeros((50, 5), dtype=np.uint32)
    graph[0, :3] = (2, 1, 2)      # 0 -> {1, 2}; 1 and 2 have no out-edges
    idx = oracle.index(x, graph, 0, "l2")
    ids, dists = idx.search(q, 5, 4, 4)          # capacity 4 < k 5  -> both become 5
    assert np.all(ids[:, 3:] == np.uint64(0xFFFFFFFFFFFFFFFF)) and np.all(np.isposinf(dists[:, 3:]))
    assert np.all(np.sort(ids[:, :3], axis=1) == np.array([0, 1, 2]))
    assert np.all(np.diff(dists[:, :3], axis=1) >= 0)
    with pytest.raises(RuntimeError):
        idx.search(q, 5, 8, 4)                   # window > capacity (SearchBufferConfig::check_invariants)


def test_oracle_lvq8_codec_roundtrip(oracle):
    """LVQ-8 own spec: decode error is bounded by half a quantisation step (+ float16 rounding of the
    per-vector constants); constant vectors and the float16 clamp edge are handled."""
    rng = np.random.default_rng(8)
    x = (rng.standard_normal((200, 100)) * 0.4 + 2.0).astype(np.float32)
    mean = x.mean(axis=0, dtype=np.float64).astype(np.float32)
    x[5] = mean + np.float32(0.75)                # constant after centring: delta == 0
    rows = oracle.lvq8_compress(x, mean)
    assert rows.shape == (200, 128)               # 100 codes + 4 constant bytes, padded to 32
    delta = rows[:, 100:102].copy().view(np.float16).astype(np.float32)
    lower = rows[:, 102:104].copy().view(np.float16).astype(np.float32)
    dec = delta * rows[:, :100].astype(np.float32) + lower + mean
    step = np.maximum(delta, 1e-3)
    assert np.all(np.abs(dec - x) <= 0.5 * step + 1e-5)
    assert np.all(rows[5, :100] == 0) and float(delta[5, 0]) == 0.0
    assert np.all(rows[:, 104:] == 0)


def _complete_graph(n):
    graph = np.zeros((n, n), dtype=np.uint32)
    graph[:, 0] = n - 1
    for i in range(n):
        graph[i, 1:] = [j for j in range(n) if j != i]
    return graph


def _assert_search_is_sorted_distances(index, q, d, metric, tag):
    """window = capacity = n on a complete graph: the search returns every row, ordered by the comparator, with the
    distances the search computes -- which must be `d`'s bits."""
    n = len(d)
    ids, dists = index.search(q[None, :], n, n, n)
    ids, dists = ids[0].astype(np.int64), dists[0]
    assert np.array_equal(np.sort(ids), np.arange(n)), tag
    assert np.array_equal(bits(dists), bits(d[ids])), tag
    want = np.sort(d) if metric == "l2" else -np.sort(-d)
    assert np.array_equal(bits(dists), bits(want)), tag


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("code", [np.int8, np.uint8])
@pytest.mark.parametrize("dim", [3, 100])
def test_oracle_sq_distance_rows_match_its_pinned_search(oracle, metric, code, dim):
    """oracle_sq_distance_rows is the SQ search's distance: every distance the pinned SQ index search returns over a
    complete graph."""
    rng = np.random.default_rng(dim)
    n = 60
    x = (rng.standard_normal((n, dim)) * 2 + 0.3).astype(np.float32)
    graph = _complete_graph(n)
    index, codes, scale, bias = oracle.sq_index(x, graph, 0, metric, code)
    for qt in (np.float32, np.float16):
        for q in (rng.standard_normal((4, dim)) * 2 + 0.3).astype(qt):
            d = oracle.sq_distance_rows(metric, q, codes, scale, bias)
            _assert_search_is_sorted_distances(index, q, d, metric, f"sq {np.dtype(code).name} {metric} {np.dtype(qt).name}")


@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("dim", [5, 96, 100])
def test_oracle_lvq8_distance_rows_match_its_search(oracle, metric, dim):
    """oracle_lvq8_distance_rows is the LVQ-8 search's distance, over a complete graph."""
    rng = np.random.default_rng(dim + 1)
    n = 60
    x = (rng.standard_normal((n, dim)) * 0.5 + 1.0).astype(np.float32)
    mean = x.mean(axis=0, dtype=np.float64).astype(np.float32)
    rows = oracle.lvq8_compress(x, mean)
    index = oracle.lvq8_index(rows, dim, mean, _complete_graph(n), 0, metric)
    for qt in (np.float32, np.float16):
        for q in (rng.standard_normal((4, dim)) + 1.0).astype(qt):
            d = oracle.lvq8_distance_rows(metric, q, rows, dim, mean)
            _assert_search_is_sorted_distances(index, q, d, metric, f"lvq8 {metric} {np.dtype(qt).name}")
    with pytest.raises(RuntimeError):
        oracle.lvq8_distance_rows("cosine", x[0], rows, dim, mean)


def test_oracle_lvq8_refuses_what_float16_cannot_hold(oracle):
    """A residual that is not finite, a delta of 65520 or more or a lower bound at or below -65520 would decode to NaN
    or -inf: the encoder refuses the data, naming the first such row.  65504 - epsilon and subnormal deltas encode."""
    mean = np.zeros(8, np.float32)
    good = np.linspace(-1, 1, 32, dtype=np.float32).reshape(4, 8)
    for tag, row in (("NaN", [np.nan] + [0.0] * 7), ("+inf", [np.inf] + [0.0] * 7), ("-inf", [0.0] * 7 + [-np.inf]),
                     ("delta16 overflow", [0.0] * 7 + [255 * 65520.0]), ("lower16 overflow", [-65520.0] + [0.0] * 7)):
        x = good.copy()
        x[1] = row
        x[3] = row
        with pytest.raises(RuntimeError, match="row 1 "):
            oracle.lvq8_compress(x, mean)
    x = good.copy()
    x[1] = [-65503.0] + [0.0] * 7
    x[2] = [0.0] * 7 + [255 * 65504.0 * (1 - 2.0 ** -12)]
    x[3] = np.linspace(0, 255 * 2.0 ** -20, 8, dtype=np.float32)    # delta16 in float16's subnormals
    rows = oracle.lvq8_compress(x, mean)
    consts = rows[:, 8:12].copy().view(np.float16).astype(np.float32)
    assert np.all(np.isfinite(consts)) and consts[3, 0] == np.float32(2.0 ** -20)
