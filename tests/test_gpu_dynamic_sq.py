"""Dynamic Vamana index over scalar-quantised int8 / uint8 codes on the GPU, against the compiled reference's
MutableVamanaIndex over SQDataset (``refdynsq``: oracle/_ref/libsvsref_dynamic_sq.so), both sides started from the
same codes, scale, bias and graph and driven through the same calls.

Searches are compared bit for bit (external ids and distance bits).  Insertion is compared row for row in adds of at
most 40 points, where every round of the reference's builder holds one node and its result is deterministic;
consolidation row for row, except where a node's candidates hold exactly equal distances (the reference orders those
arbitrarily); larger adds by the slots they pick and by recall."""
import functools

import numpy as np
import pytest

from conftest import bits, recall_at_k

pytestmark = pytest.mark.gpu

METRIC = {"l2": 0, "ip": 1, "cosine": 2}
NONE = np.uint64(2**64 - 1)


@pytest.fixture(scope="module")
def refdynsq(reflib):
    from oracle.dynamic_sq import RefDynamicSQLib
    if not RefDynamicSQLib.available():
        pytest.skip("oracle/_ref/libsvsref_dynamic_sq.so not built (needs /root/reference)")
    if not reflib.avx512vnni():
        pytest.skip("host lacks AVX-512 VNNI: the reference would take its float fallback for integer rows")
    return RefDynamicSQLib()


@pytest.fixture(scope="module")
def refbuild(refdynsq):
    from oracle.build_sq import RefSQBuildLib
    if not RefSQBuildLib.available():
        pytest.skip("oracle/_ref/libsvsref_sq_build.so not built (needs /root/reference)")
    return RefSQBuildLib()


@pytest.fixture(scope="module")
def setdatum():
    from oracle.sq_set_datum import RefSQSetDatum
    if not RefSQSetDatum.available():
        pytest.skip("oracle/_ref/libsvsref_sq_set_datum.so not built (needs /root/reference)")
    return RefSQSetDatum()


@functools.lru_cache(maxsize=None)
def rows_of(n, dim, seed):
    """n x dim float32 rows with some structure (cluster centres plus noise) and a few queries near them."""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((32, dim)).astype(np.float32)
    x = centres[rng.integers(0, 32, n)] + 0.5 * rng.standard_normal((n, dim)).astype(np.float32)
    q = centres[rng.integers(0, 32, 24)] + 0.5 * rng.standard_normal((24, dim)).astype(np.float32)
    return x.astype(np.float32), q.astype(np.float32)


@functools.lru_cache(maxsize=None)
def sq_graph(n, dim, code, metric, R):
    """The SQ codes of rows_of(n, dim), their scale and bias, and the GPU SQ builder's graph over them."""
    from scalablevectorsearch_b200 import DistanceType, VamanaBuildParameters, build_graph
    from scalablevectorsearch_b200.ivf import sq_compress
    x, _ = rows_of(n, dim, dim)
    codes, scale, bias = sq_compress(x, code)
    graph, ep = build_graph(codes, DistanceType(METRIC[metric]), VamanaBuildParameters(graph_max_degree=R, window_size=2 * R),
                            sq=(scale, bias))
    return codes, scale, bias, graph, ep


def pair(refdynsq, codes, scale, bias, graph, ep, ids, metric):
    """The GPU index and the reference's, with the same mutation parameters (the GPU defaults)."""
    from scalablevectorsearch_b200 import DistanceType, DynamicVamana
    gpu = DynamicVamana.from_arrays(codes, graph, ep, ids, DistanceType(METRIC[metric]), sq=(scale, bias))
    ref = refdynsq.dynamic(codes, scale, bias, graph, ep, ids, metric, gpu.alpha, gpu.construction_window_size,
                           gpu.max_candidates, gpu.prune_to)
    return gpu, ref


def rows(graph):
    return [tuple(r[1:1 + r[0]].tolist()) for r in graph]


def same_search(gpu, ref, queries, window, capacity, k, tag=""):
    from scalablevectorsearch_b200 import SearchBufferConfig
    gpu.search_parameters.buffer_config = SearchBufferConfig(window, capacity)
    gi, gd = gpu.search(queries, k)
    ri, rd = ref.search(queries, k, window, capacity)
    for qi in range(len(queries)):
        m = int((ri[qi] != NONE).sum())
        assert gi[qi, :m].tolist() == ri[qi, :m].tolist(), (tag, qi)
        assert np.array_equal(bits(gd[qi, :m]), bits(rd[qi, :m])), (tag, qi)
        assert (gi[qi, m:] == NONE).all(), (tag, qi)
    return gi, gd


def encode(x, code, scale, bias):
    """SQDataset::set_datum's rule in numpy: clamp(roundf((x - bias) / scale)), each step rounded in float32."""
    info = np.iinfo(code)
    v = np.round((np.asarray(x, dtype=np.float32) - np.float32(bias)) / np.float32(scale))
    return np.clip(v, info.min, info.max).astype(code)


# ---------------------------------------------------------------- search parity

@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("code", [np.int8, np.uint8])
@pytest.mark.parametrize("dim", [96, 128, 256, 101])
def test_search_matches_the_reference(refdynsq, metric, code, dim):
    """0 %, 1 %, 10 % (with the entry point) and 50 % of the slots Deleted, every buffer shape, forced re-runs."""
    from scalablevectorsearch_b200 import DistanceType, SearchBufferConfig, Vamana
    n = 3000
    codes, scale, bias, graph, ep = sq_graph(n, dim, code, metric, 32)
    _, queries = rows_of(n, dim, dim)
    rng = np.random.default_rng(dim + METRIC[metric])
    ext = rng.permutation(np.arange(10**9, 10**9 + n, dtype=np.uint64))
    gpu, ref = pair(refdynsq, codes, scale, bias, graph, ep, ext, metric)
    # no Deleted slot: the static SQ index over the same codes and graph, with external ids
    static = Vamana.from_arrays(codes, graph, ep, DistanceType(METRIC[metric]), sq=(scale, bias))
    for w, c, k in [(10, 20, 10), (100, 100, 100)]:
        gi, gd = same_search(gpu, ref, queries, w, c, k, "0%")
        static.search_parameters.buffer_config = SearchBufferConfig(w, c)
        si, sd = static.search(queries, k)
        assert np.array_equal(gi, ext[si.astype(np.int64)]) and np.array_equal(bits(gd), bits(sd))
    order = rng.permutation(n)
    dead = np.zeros(n, dtype=bool)
    for frac in (0.0, 0.01, 0.1, 0.5):
        gone = order[:int(frac * n)]
        if frac == 0.1:
            gone = np.append(gone, ep)
        gone = np.unique(gone[~dead[gone]])
        if len(gone):
            gpu.delete(ext[gone])
            ref.delete(ext[gone])
            dead[gone] = True
        for w, c, k in [(1, 10, 1), (10, 20, 10), (15, 15, 10), (100, 100, 100)]:
            same_search(gpu, ref, queries, w, c, k, f"{frac}")
    # no room for Deleted entries: most queries are re-run, with the same answers
    before = gpu.get_option("dynamic_reruns")
    gpu.set_option("dynamic_slack", 0)
    same_search(gpu, ref, queries, 10, 20, 10, "slack 0")
    assert gpu.get_option("dynamic_reruns") > before
    gpu.set_option("dynamic_slack", -1)


# ---------------------------------------------------------------- mutations

def tie_in_candidates(refbuild, metric, codes, scale, bias, graph, status, v):
    """Whether node v's consolidation candidates hold an exactly repeated builder distance."""
    cand = set()
    for u in graph[v, 1:1 + graph[v, 0]].tolist():
        cand |= {u} if status[u] == 1 else set(graph[u, 1:1 + graph[u, 0]].tolist())
    cand = sorted(c for c in cand if status[c] == 1)
    d = refbuild.distance(codes, scale, bias, metric, np.array([(v, c) for c in cand], dtype=np.uint32))
    return len(np.unique(d)) < len(d)


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("code", [np.int8, np.uint8])
@pytest.mark.parametrize("R", [32, 128])
def test_mutation_script_matches_the_reference(refdynsq, refbuild, setdatum, metric, code, R):
    """build_sq; add float32 rows (values outside the compressed range included); delete (the entry point included);
    consolidate; compact; a large add into the Empty slots -- checked after every step."""
    from scalablevectorsearch_b200 import DistanceType, DynamicVamana, Svsb200Error, VamanaBuildParameters
    from scalablevectorsearch_b200.ivf import sq_compress
    dim, n0 = 96, 2000
    x, queries = rows_of(2600, dim, 7)
    codes, scale, bias = sq_compress(x[:n0], code)
    ids = np.arange(n0, dtype=np.uint64) + np.uint64(10**6)
    gpu = DynamicVamana.build(VamanaBuildParameters(graph_max_degree=R, window_size=2 * R), codes, ids,
                              DistanceType(METRIC[metric]), sq=(scale, bias))
    graph, status, ext, ep = gpu.export()
    assert (status == 1).all() and np.array_equal(ext, ids)
    ref = refdynsq.dynamic(codes, scale, bias, graph, ep, ids, metric, gpu.alpha, gpu.construction_window_size,
                           gpu.max_candidates, gpu.prune_to)

    def check(tag, exact_rows=True):
        g_graph, g_status, g_ext, g_ep = gpu.export()
        r_graph, r_status, r_ext, r_ep, r_codes = ref.export()
        valid = g_status == 1   # (a Deleted slot keeps its external id here until consolidation)
        assert np.array_equal(g_status, r_status) and np.array_equal(g_ext[valid], r_ext[valid]) and g_ep == r_ep, tag
        if exact_rows:
            assert rows(g_graph) == rows(r_graph), tag
            same_search(gpu, ref, queries, 20, 20, 10, tag)
        return r_codes

    # adds of at most 40 points: every round holds one node, so the reference's rows are deterministic
    by_slot_codes = codes.copy()
    for step, (lo, hi, stretch) in enumerate([(n0, n0 + 30, 1.0), (n0 + 30, n0 + 70, 3.0)]):
        pts = (x[lo:hi] * np.float32(stretch)).astype(np.float32)   # 3x: most values leave the compressed range
        new = np.arange(lo, hi, dtype=np.uint64) + np.uint64(10**6)
        s_gpu, s_ref = gpu.add(pts, new), ref.add(pts, new)
        assert np.array_equal(s_gpu, s_ref), f"add {step}: slots"
        r_codes = check(f"add {step}")
        want = setdatum.set_datum(pts, code, scale, bias)
        assert np.array_equal(want, encode(pts, code, scale, bias))
        assert np.array_equal(r_codes[s_ref.astype(np.int64)], want), f"add {step}: the reference's codes"
        by_slot_codes = np.concatenate([by_slot_codes, want])
        # the added rows as queries: each one's own code decides its nearest distances
        same_search(gpu, ref, pts, 20, 20, 10, f"add {step} self")
    if stretch == 3.0:
        info = np.iinfo(code)
        assert ((want == info.min) | (want == info.max)).mean() > 0.1   # the clamp was exercised

    # delete 10 %, the entry point included; consolidate
    n = gpu.num_slots
    rng = np.random.default_rng(R + METRIC[metric])
    gone = rng.choice(n, n // 10, replace=False)
    ep = gpu.export()[3]
    if ep not in gone:
        gone = np.append(gone, ep)
    ext_all = gpu.export()[2]
    gpu.delete(ext_all[gone])
    ref.delete(ext_all[gone])
    check("delete")
    before_graph, before_status = gpu.export()[:2]
    with pytest.raises(Svsb200Error, match="consolidate first"):
        gpu.compact()
    gpu.consolidate()
    ref.consolidate()
    g_graph, g_status, _, g_ep = gpu.export()
    r_graph, r_status, _, r_ep, _ = ref.export()
    assert np.array_equal(g_status, r_status) and g_ep == r_ep != ep
    differ = [v for v, (a, b) in enumerate(zip(rows(g_graph), rows(r_graph))) if a != b]
    assert len(differ) < 0.01 * n, differ[:10]
    for v in differ:
        assert tie_in_candidates(refbuild, metric, by_slot_codes, scale, bias, before_graph, before_status, v), v
    check("consolidate", exact_rows=not differ)

    gpu.compact()
    ref.compact()
    r_codes = check("compact", exact_rows=not differ)
    live = np.ones(n, dtype=bool)
    live[gone] = False
    assert np.array_equal(r_codes, by_slot_codes[live])
    assert gpu.num_slots == gpu.size == int(live.sum())

    # a large add into the Empty slots after one more delete and consolidate: slots equal, recall equivalent
    more = rng.choice(gpu.size, 200, replace=False)
    gone_ids = gpu.all_ids()[more]
    gpu.delete(gone_ids)
    ref.delete(gone_ids)
    gpu.consolidate()
    ref.consolidate()
    pts = x[n0 + 70:n0 + 600]
    new = np.arange(n0 + 70, n0 + 600, dtype=np.uint64) + np.uint64(10**6)
    assert np.array_equal(gpu.add(pts, new, reuse_empty=True), ref.add(pts, new, reuse_empty=True))
    check("large add", exact_rows=False)
    _, status, ext, _ = gpu.export()
    xs = x[:n0 + 600].copy()
    xs[n0 + 30:n0 + 70] *= np.float32(3.0)   # as the second add stretched them
    all_ids = np.arange(n0 + 600, dtype=np.uint64) + np.uint64(10**6)
    keep = np.isin(all_ids, ext[status == 1])
    if metric == "l2":
        d = (xs * xs).sum(1)[None, :] - 2.0 * queries @ xs.T
    elif metric == "ip":
        d = -(queries @ xs.T)
    else:
        d = -(queries @ xs.T) / np.linalg.norm(xs, axis=1)[None, :]
    d[:, ~keep] = np.inf
    gt = all_ids[np.argsort(d, axis=1, kind="stable")[:, :10]]
    for w in (20, 50):
        gpu.search_window_size = w
        a = recall_at_k(gpu.search(queries, 10)[0], gt)
        b = recall_at_k(ref.search(queries, 10, w)[0], gt)
        assert abs(a - b) <= 0.05, (w, a, b)


# ---------------------------------------------------------------- filtered and range searches

@pytest.mark.parametrize("metric,code", [("l2", np.int8), ("ip", np.uint8), ("cosine", np.int8)])
def test_filtered_and_range_match_the_host_model(metric, code):
    from test_gpu_filtered_range import Dynamic
    from scalablevectorsearch_b200 import DistanceType, DynamicVamana
    n = 5000
    codes, scale, bias, graph, ep = sq_graph(n, 96, code, metric, 32)
    _, q = rows_of(n, 96, 96)
    rng = np.random.default_rng(5)
    ext = rng.permutation(np.arange(n, dtype=np.uint64) + np.uint64(7 * 10**6))
    index = DynamicVamana.from_arrays(codes, graph, ep, ext, DistanceType(METRIC[metric]), sq=(scale, bias))
    gone = rng.choice(n, n // 5, replace=False)
    if ep not in gone:
        gone = np.append(gone, ep)
    index.delete(ext[gone])
    dyn = Dynamic(index, metric)
    assert dyn.status[ep] == 2
    dyn.battery(q[:16], f"sq {metric} deleted")
    index.consolidate()
    index.delete(rng.choice(index.all_ids(), 300, replace=False))
    dyn.refresh()
    assert (dyn.status == 0).any() and (dyn.status == 2).sum() == 300
    dyn.battery(q[:16], f"sq {metric} empty+deleted")


# ---------------------------------------------------------------- refusals and memory

def test_refusals_change_nothing():
    from scalablevectorsearch_b200 import DistanceType, DynamicVamana, ShardedVamana, Svsb200Error
    n = 2000
    codes, scale, bias, graph, ep = sq_graph(n, 96, np.int8, "l2", 32)
    x, q = rows_of(n, 96, 96)
    ext = np.arange(n, dtype=np.uint64)
    index = DynamicVamana.from_arrays(codes, graph, ep, ext, DistanceType.L2, sq=(scale, bias))
    index.delete(ext[:100])
    state = index.export()
    index.search_window_size = 30
    want = index.search(q, 10)
    pts, new = x[:2] + 0.1, [5 * 10**6, 5 * 10**6 + 1]
    for bad, match in [(pts.astype(np.float16), "float32"), (codes[:2], "float32"), (codes[:2].astype(np.uint8), "float32")]:
        with pytest.raises(Svsb200Error, match=match):
            index.add(bad, new)
    for value in (np.nan, np.inf, -np.inf):
        bad = pts.copy()
        bad[1, 7] = value
        with pytest.raises(Svsb200Error, match="NaN or an infinity"):
            index.add(bad, new)
    for ids, match in [([9, 9], "repeat"), ([200, 6 * 10**6], "exists"), ([2**64 - 1, 6 * 10**6], "reserved")]:
        with pytest.raises(Svsb200Error, match=match):
            index.add(pts, np.array(ids, dtype=np.uint64))
    with pytest.raises(Svsb200Error, match="consolidate first"):
        index.compact()
    with pytest.raises(Svsb200Error, match="dynamic index"):
        index.flat_search(q[:2], 10)
    with pytest.raises(Svsb200Error, match="exhaustive search is not available"):
        index.exhaustive_device(0, np.float32, 0, 10, 0, 0)
    with pytest.raises(Svsb200Error):   # a dynamic index takes no id offset and is no shard
        ShardedVamana([index], [0]).search(q[:2], 10)
    after = index.export()
    assert all(np.array_equal(a, b) for a, b in zip(state[:3], after[:3])) and state[3] == after[3]
    got = index.search(q, 10)
    assert np.array_equal(got[0], want[0]) and np.array_equal(bits(got[1]), bits(want[1]))


def test_device_bytes_are_a_quarter_for_the_rows():
    from scalablevectorsearch_b200 import DistanceType, DynamicVamana
    n, dim = 2000, 96
    codes, scale, bias, graph, ep = sq_graph(n, dim, np.int8, "l2", 32)
    x, _ = rows_of(n, dim, dim)
    ids = np.arange(n, dtype=np.uint64)
    sq = DynamicVamana.from_arrays(codes, graph, ep, ids, DistanceType.L2, sq=(scale, bias))
    f32 = DynamicVamana.from_arrays(x, graph, ep, ids, DistanceType.L2)
    assert f32.device_bytes - sq.device_bytes == 3 * dim * n
