"""Dynamic index mutations on the GPU -- add, consolidate, compact, build -- against the compiled reference's
MutableVamanaIndex (``refdyn``: oracle/_ref/libsvsref_dynamic.so), both sides started from the same graph and driven through the same calls.

Consolidation and compaction are deterministic and compared row by row; insertion runs the graph builder, whose
reference result depends on thread timing, so its bar is the slots it picks plus recall equivalence.  After every
mutation the GPU search must still equal the MutableBuffer restatement (tests/mutable_model.py) over the exported
graph, ids and distance bits."""
import functools

import numpy as np
import pytest

from conftest import bits, recall_at_k
from mutable_model import mutable_search

pytestmark = pytest.mark.gpu

METRIC = {"l2": 0, "ip": 1, "cosine": 2}
NONE = np.uint64(2**64 - 1)


@pytest.fixture(scope="module")
def refdyn(reflib):
    """The reference's MutableVamanaIndex, where the compiled reference (``reflib``) runs here."""
    from oracle.dynamic import RefDynamicLib
    if not RefDynamicLib.available():
        pytest.skip("oracle/_ref/libsvsref_dynamic.so not built (needs /root/reference)")
    return RefDynamicLib()


@functools.lru_cache(maxsize=None)
def gaussian(dtype, R, metric):
    """5000 x 100 (a ragged dimension) Gaussian rows and the GPU builder's graph over them."""
    from scalablevectorsearch_b200 import DistanceType, VamanaBuildParameters, build_graph
    x = np.random.default_rng(R).standard_normal((5000, 100)).astype(np.float32).astype(dtype)
    graph, ep = build_graph(x, DistanceType(METRIC[metric]), VamanaBuildParameters(graph_max_degree=R, window_size=2 * R))
    return x, graph, ep


def pair(refdyn, data, graph, ep, ids, metric):
    """The GPU index and the reference's, with the same mutation parameters (the GPU defaults)."""
    from scalablevectorsearch_b200 import DistanceType, DynamicVamana
    gpu = DynamicVamana.from_arrays(data, graph, ep, ids, DistanceType(METRIC[metric]))
    ref = refdyn.dynamic(data, graph, ep, ids, metric, gpu.alpha, gpu.construction_window_size, gpu.max_candidates,
                         gpu.prune_to)
    return gpu, ref


def rows(graph):
    return [tuple(r[1:1 + r[0]].tolist()) for r in graph]


def tie_in_candidates(reflib, metric, data, graph, status, v):
    """Whether node v's consolidation candidates (before consolidation) hold an exactly repeated distance."""
    cand = set()
    for u in graph[v, 1:1 + graph[v, 0]].tolist():
        cand |= {u} if status[u] == 1 else set(graph[u, 1:1 + graph[u, 0]].tolist())
    cand = sorted(c for c in cand if status[c] == 1)
    d = reflib.distance_rows(metric, data[v], data[cand])
    return len(np.unique(d)) < len(d)


def check_structure(index):
    graph, status, _, ep = index.export()
    R, n = index.graph_max_degree, index.num_slots
    assert status[ep] == 1
    for v in np.flatnonzero(status == 1):
        row = graph[v, 1:1 + graph[v, 0]]
        assert 1 <= len(row) <= R and v not in row and len(set(row.tolist())) == len(row) and (row < n).all(), v


def check_search(oracle, index, data_by_slot, metric, queries, window=20, k=10):
    """GPU search == the MutableBuffer restatement over the exported graph and entry point (ids and distance bits)."""
    from scalablevectorsearch_b200 import SearchBufferConfig
    graph, status, ext, ep = index.export()
    index.search_parameters.buffer_config = SearchBufferConfig(window, window)
    ids, dists = index.search(queries, k)
    sign = np.float32(-1.0 if metric != "l2" else 1.0)
    for qi, q in enumerate(queries):
        keys = oracle.distance_rows(metric, q, data_by_slot[:len(status)]) * sign
        res = mutable_search(ep, lambda v: graph[v, 1:1 + graph[v, 0]], lambda s: keys[s], lambda v: status[v] == 1,
                             window, window, k)
        m = len(res)
        assert ids[qi, :m].tolist() == [int(ext[s]) for s, _ in res], qi
        assert np.array_equal(bits(dists[qi, :m]), bits(np.array([key for _, key in res], dtype=np.float32) * sign)), qi
        assert (ids[qi, m:] == NONE).all()


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16])
@pytest.mark.parametrize("R", [32, 128])
@pytest.mark.parametrize("frac", [0.01, 0.1, 0.5])
def test_consolidate_and_compact_match_the_reference(reflib, refdyn, oracle, metric, dtype, R, frac):
    from scalablevectorsearch_b200 import Svsb200Error
    data, graph, ep = gaussian(dtype, R, metric)
    n = len(data)
    rng = np.random.default_rng(int(frac * 100) + R)
    ids = rng.permutation(n).astype(np.uint64) + np.uint64(10**6)
    gpu, ref = pair(refdyn, data, graph, ep, ids, metric)
    gone = rng.choice(n, int(frac * n), replace=False)
    if frac == 0.1 and ep not in gone:
        gone = np.append(gone, ep)   # a deleted entry point: replaced by the medoid of the Valid rows
    gpu.delete(ids[gone])
    ref.delete(ids[gone])
    before_graph, before_status, _, _ = gpu.export()
    # compaction needs consolidation first, and changes nothing when refused
    with pytest.raises(Svsb200Error, match="consolidate first"):
        gpu.compact()
    assert gpu.num_slots == n and np.array_equal(gpu.export()[1], before_status)

    gpu.consolidate()
    ref.consolidate()
    g_graph, g_status, _, g_ep = gpu.export()
    r_graph, r_status, _, r_ep = ref.export()
    assert np.array_equal(g_status, r_status) and g_ep == r_ep
    assert not (g_status == 2).any()
    differ = [v for v, (a, b) in enumerate(zip(rows(g_graph), rows(r_graph))) if a != b]
    # only nodes whose candidates tie exactly may differ: the reference orders equal distances arbitrarily
    assert len(differ) < 0.01 * n, differ[:10]
    for v in differ:
        assert tie_in_candidates(reflib, metric, data, before_graph, before_status, v), v
    check_structure(gpu)
    check_search(oracle, gpu, data, metric, data[:4].astype(np.float32) + 0.5)

    gpu.compact()
    ref.compact()
    g_graph, g_status, g_ext, g_ep = gpu.export()
    r_graph, r_status, r_ext, r_ep = ref.export()
    assert gpu.num_slots == gpu.size == int((r_status == 1).sum())
    assert np.array_equal(g_status, r_status) and np.array_equal(g_ext, r_ext) and g_ep == r_ep
    assert sum(a != b for a, b in zip(rows(g_graph), rows(r_graph))) <= len(differ)
    assert np.array_equal(gpu.all_ids(), g_ext)
    live = np.ones(n, dtype=bool)
    live[gone] = False
    check_search(oracle, gpu, data[np.flatnonzero(live)], metric, data[:4].astype(np.float32) + 0.5)


@pytest.mark.parametrize("metric,dtype", [("l2", np.float32), ("ip", np.float16), ("cosine", np.float32)])
def test_add_picks_the_reference_slots_and_validates_first(refdyn, oracle, metric, dtype):
    from scalablevectorsearch_b200 import Svsb200Error
    data, graph, ep = gaussian(dtype, 32, metric)
    n0 = 2000   # the first 2000 rows with the graph restricted to them; the other rows are added
    gpu, ref = pair(refdyn, data[:n0], _subgraph(graph, n0), ep if ep < n0 else 0, np.arange(n0, dtype=np.uint64), metric)
    by_slot = np.zeros((4000, 100), dtype=dtype)
    by_slot[:n0] = data[:n0]
    q = data[:4].astype(np.float32) + 0.25
    todo = list(range(n0, len(data)))

    def add(count, reuse):
        rows_, todo[:] = todo[:count], todo[count:]
        pts, ids = data[rows_], np.array(rows_, dtype=np.uint64)
        s_gpu = gpu.add(pts, ids, reuse_empty=reuse)
        s_ref = ref.add(pts, ids, reuse_empty=reuse)
        assert np.array_equal(s_gpu, s_ref), (s_gpu[:8], s_ref[:8])
        by_slot[s_gpu.astype(np.int64)] = pts
        check_structure(gpu)
        check_search(oracle, gpu, by_slot, metric, q)

    add(50, False)                                  # appended
    gone = np.random.default_rng(1).choice(n0, 200, replace=False).astype(np.uint64)
    gpu.delete(gone)
    ref.delete(gone)
    gpu.consolidate()
    ref.consolidate()
    check_search(oracle, gpu, by_slot, metric, q)
    add(60, False)                                  # Empty slots exist, but below first_empty: appended
    add(300, True)                                  # reuses the 200 Empty slots, then grows
    assert gpu.num_slots == n0 + 50 + 60 + 100
    more = data[todo]

    # every validation failure leaves the index as it was
    state = gpu.export()
    size, slots, all_ids = gpu.size, gpu.num_slots, gpu.all_ids()
    present = int(all_ids[0])
    for pts, ids, what in [(more[:2], [9 * 10**6, 9 * 10**6], "repeat"), (more[:2], [present, 5 * 10**6], "exists"),
                           (more[:1], [2**64 - 1], "reserved"), (more[:1].astype(np.float64), [6 * 10**6], "type")]:
        with pytest.raises((Svsb200Error, TypeError), match=what if what != "type" else None):
            gpu.add(pts, ids)
    with pytest.raises(Svsb200Error, match="dtype"):
        other = np.float16 if dtype == np.float32 else np.float32
        gpu.add(more[:1].astype(other), [6 * 10**6])
    assert gpu.size == size and gpu.num_slots == slots and np.array_equal(gpu.all_ids(), all_ids)
    after = gpu.export()
    assert all(np.array_equal(a, b) for a, b in zip(state[:3], after[:3])) and state[3] == after[3]


def _subgraph(graph, n):
    """Rows 0..n-1 of a degree-first graph with the neighbours >= n removed."""
    out = np.zeros((n, graph.shape[1]), dtype=np.uint32)
    for v in range(n):
        row = [u for u in graph[v, 1:1 + graph[v, 0]].tolist() if u < n]
        out[v, 0] = len(row)
        out[v, 1:1 + len(row)] = row
    return out


def test_insertion_recall_matches_the_reference(refdyn, dataset):
    """80 % of the test dataset from one graph, the other 20 % added in four calls on both sides."""
    from scalablevectorsearch_b200 import DistanceType, VamanaBuildParameters, build_graph
    n = len(dataset.data)
    n0 = int(0.8 * n)
    graph, ep = build_graph(dataset.data[:n0], DistanceType.L2, VamanaBuildParameters(graph_max_degree=64, window_size=128))
    gpu, ref = pair(refdyn, dataset.data[:n0], graph, ep, np.arange(n0, dtype=np.uint64), "l2")
    for lo in range(n0, n, (n - n0) // 4):
        hi = min(n, lo + (n - n0) // 4)
        ids = np.arange(lo, hi, dtype=np.uint64)
        assert np.array_equal(gpu.add(dataset.data[lo:hi], ids), ref.add(dataset.data[lo:hi], ids))
    check_structure(gpu)
    for w in (10, 30):
        gpu.search_window_size = w
        got = recall_at_k(gpu.search(dataset.queries, 10)[0], dataset.gt["l2"])
        want = recall_at_k(ref.search(dataset.queries, 10, w)[0], dataset.gt["l2"])
        assert abs(got - want) <= 0.01, (w, got, want)


def test_lifecycle_through_python_matches_the_reference(refdyn, dataset):
    """DynamicVamana.build, delete 30 %, add 30 % new points into the emptied slots, consolidate, compact."""
    from scalablevectorsearch_b200 import DistanceType, DynamicVamana, Svsb200Error, VamanaBuildParameters
    x, queries = dataset.data, dataset.queries[:300]
    n0 = 7000
    params = VamanaBuildParameters(graph_max_degree=32, window_size=64)
    gpu = DynamicVamana.build(params, x[:n0], np.arange(n0), DistanceType.L2)
    assert (gpu.alpha, gpu.construction_window_size, gpu.max_candidates, gpu.prune_to) == (np.float32(1.2), 64, 192, 28)
    ref = refdyn.dynamic_build(x[:n0], np.arange(n0), "l2", gpu.alpha, 32, 64, 192, 28)
    live = np.zeros(len(x), dtype=bool)
    live[:n0] = True

    def recalls():
        xs = x[live]
        d = (xs * xs).sum(1)[None, :] - 2.0 * queries @ xs.T
        gt = np.flatnonzero(live)[np.argsort(d, axis=1, kind="stable")[:, :10]]
        gpu.search_window_size = 30
        return (recall_at_k(gpu.search(queries, 10)[0], gt), recall_at_k(ref.search(queries, 10, 30)[0], gt))

    a, b = recalls()
    assert abs(a - b) <= 0.01, (a, b)
    gone = np.random.default_rng(2).choice(n0, int(0.3 * n0), replace=False)
    gpu.delete(gone)
    ref.delete(gone)
    live[gone] = False
    new = np.arange(n0, n0 + len(gone))
    assert np.array_equal(gpu.add(x[new], new, reuse_empty=True), ref.add(x[new], new, reuse_empty=True))
    live[new] = True
    with pytest.raises(Svsb200Error, match="consolidate first"):
        gpu.compact()
    for step in ("consolidate", "compact"):
        getattr(gpu, step)()
        getattr(ref, step)()
        a, b = recalls()
        assert abs(a - b) <= 0.01, (step, a, b)
    assert gpu.size == gpu.num_slots == n0 and sorted(gpu.all_ids().tolist()) == np.flatnonzero(live).tolist()
    check_structure(gpu)


def test_mutation_parameters(dataset):
    from scalablevectorsearch_b200 import DistanceType, DynamicVamana, Svsb200Error
    index = DynamicVamana.from_arrays(dataset.data, dataset.graph, dataset.entry_point, distance=DistanceType.MIP)
    R = index.graph_max_degree   # 128: the reference's 3 * window default (768) is clamped to the GPU pool
    assert (index.alpha, index.construction_window_size, index.max_candidates, index.prune_to) == \
        (np.float32(0.95), 2 * R, 512, R - 4)
    index.max_candidates = 100
    index.prune_to = 60
    assert (index.max_candidates, index.prune_to) == (100, 60)
    for name, value in [("max_candidates", 513), ("alpha", 1.1), ("prune_to", R + 1), ("construction_window_size", 400)]:
        with pytest.raises(Svsb200Error):
            setattr(index, name, value)
    assert (index.alpha, index.max_candidates, index.prune_to) == (np.float32(0.95), 100, 60)
    index.max_candidates = 0
    assert index.max_candidates == 512
