"""Dynamic (mutable) index on the GPU: MutableVamanaIndex::search bit for bit, soft deletion, and the API around it.

The expected results come from the one-by-one MutableBuffer restatement (tests/mutable_model.py, pinned to the
reference's known answers in test_mutable_buffer.py) driving greedy search over the reference's distances
(the oracle's ``distance_rows``).  The index is tests/golden/test_dataset.npz (10k x 128, the reference's graph) with
permuted external ids."""
import numpy as np
import pytest

from conftest import bits
from mutable_model import mutable_search

pytestmark = pytest.mark.gpu

METRIC = {"l2": 0, "ip": 1, "cosine": 2}


def make_index(dataset, metric, dtype, frac, rng, delete_entry=False):
    from scalablevectorsearch_b200 import DistanceType, DynamicVamana
    data = dataset.data.astype(dtype)
    n = data.shape[0]
    ext = rng.permutation(np.arange(10**9, 10**9 + n, dtype=np.uint64))
    index = DynamicVamana.from_arrays(data, dataset.graph, dataset.entry_point, ext, DistanceType(METRIC[metric]))
    deleted = rng.choice(n, size=int(frac * n), replace=False)
    if delete_entry and dataset.entry_point not in deleted:
        deleted = np.append(deleted, dataset.entry_point)
    if len(deleted):
        index.delete(ext[deleted])
    valid = np.ones(n, dtype=bool)
    valid[deleted] = False
    return index, data, ext, valid


def expected(oracle, dataset, data, valid, metric, queries, window, capacity, k):
    sign = -1.0 if metric != "l2" else 1.0
    graph = dataset.graph
    out_ids, out_keys = [], []
    for q in queries:
        keys = oracle.distance_rows(metric, q, data) * np.float32(sign)
        res = mutable_search(dataset.entry_point, lambda v: graph[v, 1:1 + graph[v, 0]], lambda ids: keys[ids],
                             lambda v: bool(valid[v]), window, capacity, k)
        out_ids.append([s for s, _ in res])
        out_keys.append([key for _, key in res])
    return out_ids, out_keys


def check_against_model(oracle, dataset, index, data, ext, valid, metric, queries, window, capacity, k):
    from scalablevectorsearch_b200 import SearchBufferConfig
    index.search_parameters.buffer_config = SearchBufferConfig(window, capacity)
    ids, dists = index.search(queries, k)
    want_slots, want_keys = expected(oracle, dataset, data, valid, metric, queries, window, capacity, k)
    sign = np.float32(-1.0 if metric != "l2" else 1.0)
    for qi in range(len(queries)):
        m = len(want_slots[qi])
        assert ids[qi, :m].tolist() == ext[want_slots[qi]].tolist(), qi
        assert np.array_equal(bits(dists[qi, :m]), bits(np.array(want_keys[qi], dtype=np.float32) * sign)), qi
        assert (ids[qi, m:] == np.uint64(2**64 - 1)).all()
    return ids, dists


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16])
@pytest.mark.parametrize("frac", [0.0, 0.01, 0.1, 0.5])
@pytest.mark.parametrize("window,capacity,k", [(1, 10, 1), (10, 20, 10), (15, 15, 10), (100, 100, 100)])
def test_search_matches_mutable_buffer(oracle, dataset, metric, dtype, frac, window, capacity, k):
    rng = np.random.default_rng(int(frac * 1000) + window)
    index, data, ext, valid = make_index(dataset, metric, dtype, frac, rng, delete_entry=frac == 0.1)
    nq = 4 if window == 100 else 12
    queries = dataset.queries[rng.choice(len(dataset.queries), nq, replace=False)]
    check_against_model(oracle, dataset, index, data, ext, valid, metric, queries, window, capacity, k)


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_forced_small_slack_reruns_and_agrees(oracle, dataset, metric):
    """With no room for Deleted entries most queries overflow and are re-run: the answers stay exact."""
    rng = np.random.default_rng(7)
    index, data, ext, valid = make_index(dataset, metric, np.float32, 0.5, rng)
    queries = dataset.queries[:16]
    index.set_option("dynamic_slack", 0)
    before = index.get_option("dynamic_reruns")
    check_against_model(oracle, dataset, index, data, ext, valid, metric, queries, 10, 20, 10)
    assert index.get_option("dynamic_reruns") > before
    # and the default slack gives the same rows
    index.set_option("dynamic_slack", -1)
    a = index.search(queries, 10)
    index.set_option("dynamic_slack", 0)
    b = index.search(queries, 10)
    assert np.array_equal(a[0], b[0]) and np.array_equal(bits(a[1]), bits(b[1]))


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16])
def test_no_deletions_equals_static_index(dataset, metric, dtype):
    from scalablevectorsearch_b200 import DistanceType, SearchBufferConfig, Vamana
    rng = np.random.default_rng(3)
    index, data, ext, _ = make_index(dataset, metric, dtype, 0.0, rng)
    static = Vamana.from_arrays(data, dataset.graph, dataset.entry_point, DistanceType(METRIC[metric]))
    for w, c, k in [(10, 20, 10), (50, 50, 10), (100, 100, 100)]:
        index.search_parameters.buffer_config = SearchBufferConfig(w, c)
        static.search_parameters.buffer_config = SearchBufferConfig(w, c)
        ids, dists = index.search(dataset.queries, k)
        sids, sdists = static.search(dataset.queries, k)
        assert np.array_equal(ids, ext[sids.astype(np.int64)])
        assert np.array_equal(bits(dists), bits(sdists))


def test_deleted_ids_never_returned_and_bookkeeping(dataset):
    from scalablevectorsearch_b200 import Svsb200Error
    rng = np.random.default_rng(11)
    index, data, ext, valid = make_index(dataset, "l2", np.float32, 0.2, rng, delete_entry=True)
    n = len(ext)
    assert index.size == int(valid.sum()) and index.num_slots == n
    assert np.array_equal(index.all_ids(), ext[valid])
    assert not index.has_id(ext[dataset.entry_point]) and index.has_id(ext[np.flatnonzero(valid)[0]])
    graph, status, ids, ep = index.export()
    assert np.array_equal(status, np.where(valid, 1, 2)) and np.array_equal(ids, ext) and ep == dataset.entry_point
    for v in rng.choice(n, 200, replace=False):   # the rows as given (repeated ids are stored once)
        row = dataset.graph[v, 1:1 + dataset.graph[v, 0]]
        assert sorted(graph[v, 1:1 + graph[v, 0]].tolist()) == sorted(set(row.tolist()))
    index.search_window_size = 50
    got, _ = index.search(dataset.queries, 10)
    live = set(ext[valid].tolist())
    assert all(int(i) in live for i in got.ravel() if i != np.uint64(2**64 - 1))
    # an unknown or already deleted id fails and changes nothing
    with pytest.raises(Svsb200Error, match="does not exist"):
        index.delete([ext[np.flatnonzero(valid)[0]], ext[dataset.entry_point]])
    assert index.size == int(valid.sum())
    with pytest.raises(Svsb200Error, match="single entry point"):
        index.set_entry_points([0, 1])
    with pytest.raises(Svsb200Error, match="dynamic index"):
        index.flat_search(dataset.queries[:2], 10)


def test_cancellation_is_polled_during_a_dynamic_search(dataset):
    rng = np.random.default_rng(8)
    index, data, ext, valid = make_index(dataset, "l2", np.float32, 0.5, rng)
    index.search_window_size = 200
    q = np.tile(dataset.queries, (20, 1))
    calls = []

    def cancel():   # False for the check before any work, True once the kernels run
        calls.append(1)
        return len(calls) >= 2

    index.search(q, 10, cancel=cancel)   # rows unspecified, but the call returns cleanly
    assert len(calls) >= 2
    # the index is intact: the same search without a predicate matches a fresh run
    a = index.search(dataset.queries[:100], 10)
    b = index.search(dataset.queries[:100], 10)
    assert np.array_equal(a[0], b[0]) and np.array_equal(bits(a[1]), bits(b[1]))
    assert (a[0] != np.uint64(2**64 - 1)).all()


def test_duplicate_external_ids_are_rejected(dataset):
    from scalablevectorsearch_b200 import DynamicVamana, Svsb200Error
    ids = np.arange(len(dataset.data), dtype=np.uint64)
    ids[5] = ids[6]
    with pytest.raises(Svsb200Error, match="repeat"):
        DynamicVamana.from_arrays(dataset.data, dataset.graph, dataset.entry_point, ids)
    ids = np.arange(len(dataset.data), dtype=np.uint64)
    ids[3] = np.uint64(2**64 - 1)
    with pytest.raises(Svsb200Error, match="reserved"):
        DynamicVamana.from_arrays(dataset.data, dataset.graph, dataset.entry_point, ids)
