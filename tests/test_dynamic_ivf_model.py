"""The numpy model of the dynamic IVF index (tests/dynamic_ivf_model.py) on hand-made scripts, no GPU: the slot rules
(reuse from slot 0, append-only without reuse, compaction order), the refusals, tombstones never returned, whole
clusters and the whole index deleted, and the search at n_probes = C equal to the exact search over the live rows in
slot order."""
import numpy as np
import pytest

import ivf_model as M
from dynamic_ivf_model import NONE32, RESERVED, DynamicIVFModel, Refused


def _two_clusters(oracle, metric=0):
    """Six rows in two well separated clusters (rows 0, 2, 4 near centroid 0; 1, 3, 5 near centroid 1), ids 10-15."""
    cent = np.array([[0.0, 0.0], [10.0, 10.0]], dtype=np.float32)
    x = np.array([[0, 1], [10, 11], [1, 0], [11, 10], [1, 1], [9, 9]], dtype=np.float32)
    return DynamicIVFModel.assemble(oracle, metric, cent, x, np.arange(10, 16)), x


def test_assembly_groups_rows_by_nearest_centroid(oracle):
    m, _ = _two_clusters(oracle)
    assert m.stored == [[0, 2, 4], [1, 3, 5]]
    assert list(m.cluster_sizes()) == [3, 3]
    assert list(m.all_ids()) == [10, 11, 12, 13, 14, 15]


def test_add_without_reuse_appends(oracle):
    m, _ = _two_clusters(oracle)
    m.delete([11, 12])
    slots = m.add(np.array([[0.5, 0.5], [10.5, 10.5]], dtype=np.float32), [20, 21])
    assert slots == [6, 7]
    status, ext, cluster = m.export()
    assert list(status) == [1, 0, 0, 1, 1, 1, 1, 1]
    assert list(ext[[1, 2]]) == [RESERVED, RESERVED]
    assert list(cluster) == [0, NONE32, NONE32, 1, 0, 1, 0, 1]
    assert m.stored == [[0, None, 4, 6], [None, 3, 5, 7]]


def test_add_with_reuse_takes_empty_slots_from_zero(oracle):
    m, _ = _two_clusters(oracle)
    m.delete([13, 11])
    slots = m.add(np.array([[0.5, 0.5], [10.5, 10.5], [0.2, 0.2]], dtype=np.float32), [20, 21, 22], reuse_empty=True)
    assert slots == [1, 3, 6]
    assert list(m.all_ids()) == [10, 20, 12, 21, 14, 15, 22]
    # the reused slots' entries are appended; the old ones stay tombstones
    assert m.stored == [[0, 2, 4, 1, 6], [None, None, 5, 3]]


def test_compact_renumbers_in_slot_order_and_keeps_the_stored_order(oracle):
    m, x = _two_clusters(oracle)
    m.delete([10, 13])
    m.add(np.array([[0.5, 0.5]], dtype=np.float32), [20], reuse_empty=True)   # slot 0, stored last in cluster 0
    before = m.search(x, 6, 2)
    m.compact()
    assert list(m.all_ids()) == [20, 11, 12, 14, 15]
    assert m.stored == [[2, 3, 0], [1, 4]]   # cluster 0 held slots 0 (tombstone), 2, 4, then 0 again
    assert list(m.export()[0]) == [1] * 5
    got = m.search(x, 6, 2)
    assert np.array_equal(got[0], before[0]) and np.array_equal(got[1].view(np.uint32), before[1].view(np.uint32))


def test_refusals_change_nothing(oracle):
    m, _ = _two_clusters(oracle)
    snap = (m.export(), [list(s) for s in m.stored])
    p = np.zeros((2, 2), dtype=np.float32)
    for call in (lambda: m.add(p, [20, 20]), lambda: m.add(p, [20, 12]), lambda: m.add(p, [20, RESERVED]),
                 lambda: m.add(p.astype(np.float16), [20, 21]), lambda: m.delete([99]), lambda: m.delete([10, 10])):
        with pytest.raises(Refused):
            call()
        exp = m.export()
        assert all(np.array_equal(a, b) for a, b in zip(exp, snap[0]))
        assert [list(s) for s in m.stored] == snap[1]


@pytest.mark.parametrize("metric", [0, 1, 2])
def test_deleted_rows_never_come_back(oracle, metric):
    m, x = _two_clusters(oracle, metric)
    m.delete([11, 13, 15])                              # the whole of cluster 1
    ids, d = m.search(x, 6, 2)
    assert not np.isin(ids, [11, 13, 15]).any()
    assert (ids[:, 3:] == RESERVED).all()
    assert np.isinf(d[:, 3:]).all()
    m.delete([10, 12, 14])                              # everything
    ids, d = m.search(x, 4, 1)
    assert (ids == RESERVED).all() and np.isinf(d).all()
    assert m.size == 0 and list(m.cluster_sizes()) == [0, 0]
    m.add(x[:2], [30, 31])
    assert m.add(x[2:3], [32], reuse_empty=True) == [0]
    m.compact()
    assert list(m.all_ids()) == [32, 30, 31]


@pytest.mark.parametrize("metric", [0, 1, 2])
def test_all_probes_equal_the_exact_search_over_the_live_rows(oracle, metric):
    rng = np.random.default_rng(metric)
    x = rng.standard_normal((300, 12)).astype(np.float32)
    q = rng.standard_normal((20, 12)).astype(np.float32)
    cent = x[rng.choice(300, 9, replace=False)]
    m = DynamicIVFModel.assemble(oracle, metric, cent, x[:200], np.arange(1000, 1200))
    m.delete(np.arange(1000, 1200, 3))
    m.add(x[200:260], np.arange(2000, 2060), reuse_empty=True)
    m.add(x[260:], np.arange(3000, 3040))
    live = m.live_slots()
    ext = np.array(m.ext, dtype=np.uint64)
    # the static model over the live rows in slot order, every row in one cluster
    want_i, want_d = M.search(oracle, metric, m.live_rows(), np.zeros((1, 12), np.float32), np.zeros(live.size, np.int64),
                              q, 50, 1)
    got_i, got_d = m.search(q, 50, 9)
    assert np.array_equal(got_i, ext[live[want_i.astype(np.int64)]])
    assert np.array_equal(got_d.view(np.uint32), want_d.view(np.uint32))
