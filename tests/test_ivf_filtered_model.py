"""The IVF filtered search's numpy model (tests/ivf_filtered_model.py) from first principles, without a GPU: the plain
search under an all-ones mask, a brute force over the allowed rows at P = C, hand-computed growth sequences, the
empty mask, per-query choices, and the bitmap layout."""
import numpy as np
import pytest

import dynamic_ivf_model as D
import ivf_filtered_model as F
import ivf_model as M


def clustered(n, dim, C, seed, spread=0.2):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((C, dim)).astype(np.float32) * 3
    return (centres[rng.integers(0, C, n)] + spread * rng.standard_normal((n, dim))).astype(np.float32)


@pytest.fixture(scope="module")
def small(oracle):
    x = clustered(600, 8, 12, seed=1)
    cent = clustered(12, 8, 12, seed=1, spread=0.0)
    assign = M.nearest(oracle, 0, x, cent, 1)[:, 0].astype(np.uint32)
    q = clustered(9, 8, 12, seed=2)
    return x, cent, assign, q


def test_growth_sequences():
    assert F.growth(1, 5000) == [1, 4, 16, 64, 256, 1024]
    assert F.growth(3, 100) == [3, 12, 48, 100]          # clipped to C
    assert F.growth(1024, 5000) == [1024]
    assert F.growth(7, 7) == [7]
    order = np.arange(2000)
    allowed = np.zeros(2000, dtype=np.int64)
    allowed[70] = 1
    assert F.choose(order, allowed, 1, 1) == 256         # 1 -> 4 -> 16 -> 64 -> 256 reaches cluster 70
    assert F.choose(order, allowed, 2, 1) == 1024        # never k: P_max = min(C, 1024)
    allowed[1500] = 5
    assert F.choose(order, allowed, 2, 1) == 1024        # cluster 1500 lies past P_max
    allowed[:] = 0
    allowed[0] = 10
    assert F.choose(order, allowed, 10, 1) == 1          # n_probes already enough (>= k, not > k)
    assert F.choose(order, allowed, 11, 1) == 1024
    allowed[5] = 1
    assert F.choose(order, allowed, 11, 1) == 16         # 4 clusters hold 10, 16 hold 11
    allowed = np.zeros(100, dtype=np.int64)
    allowed[99] = 3
    assert F.choose(np.arange(100), allowed, 3, 2) == 100   # 2 -> 8 -> 32 -> 100 (clip)


def test_all_ones_mask_is_the_plain_search(oracle, small):
    x, cent, assign, q = small
    for metric in (0, 1, 2):
        for k, n_probes in ((5, 1), (40, 3), (600, 12)):
            ids, dists, probes, allowed, rows = F.static(oracle, metric, x, cent, assign, q, k, n_probes,
                                                         np.ones(len(x), dtype=bool))
            for i in range(len(q)):
                want_i, want_d = M.search(oracle, metric, x, cent, assign, q[i:i + 1], k, int(probes[i]))
                real = want_i[0] != M.PAD_ID
                np.testing.assert_array_equal(ids[i], want_i[0])
                np.testing.assert_array_equal(dists[i, real], want_d[0, real])
                assert (dists[i, ~real] == np.inf).all()      # +inf padding for every metric
                assert allowed[i] == rows[i]
                assert (probes[i] == n_probes) == (allowed[i] >= k or n_probes == 12)


def test_all_clusters_is_a_brute_force_over_the_allowed_rows(oracle, small):
    x, cent, assign, q = small
    rng = np.random.default_rng(3)
    for metric in (0, 1, 2):
        for frac in (1.0, 0.5, 0.1, 0.01):
            mask = rng.random(len(x)) < frac
            k = 17
            ids, dists, probes, allowed, rows = F.static(oracle, metric, x, cent, assign, q, k, 12, mask)
            assert (probes == 12).all() and (allowed == mask.sum()).all() and (rows == len(x)).all()
            keys = np.flatnonzero(mask)
            for i in range(len(q)):
                d = oracle.distance_rows(M.METRICS[metric], q[i], x[keys])
                order = np.lexsort((keys, d if metric == 0 else -d))[:k]
                m = order.size
                assert ids[i, :m].tolist() == keys[order].tolist()
                np.testing.assert_array_equal(dists[i, :m], d[order])
                assert (ids[i, m:] == F.PAD_ID).all() and (dists[i, m:] == np.inf).all()


def test_empty_mask_pads_everything_at_p_max(oracle, small):
    x, cent, assign, q = small
    for metric in (0, 1):
        ids, dists, probes, allowed, rows = F.static(oracle, metric, x, cent, assign, q, 4, 1, np.zeros(len(x), bool))
        assert (ids == F.PAD_ID).all() and (dists == np.inf).all()
        assert (probes == 12).all() and (allowed == 0).all() and (rows == len(x)).all()


def test_growth_is_per_query_and_counts_the_probed_clusters(oracle, small):
    x, cent, assign, q = small
    c = int(np.argmax(np.bincount(assign, minlength=12)))
    mask = assign == c                       # one cluster allowed: queries near it stop early, the others grow
    k = 3
    ids, _, probes, allowed, rows = F.static(oracle, 0, x, cent, assign, q, k, 1, mask)
    order = F.probe_order(oracle, 0, q, cent)
    sizes = np.bincount(assign, minlength=12)
    for i in range(len(q)):
        P = int(probes[i])
        assert P in F.growth(1, 12)
        assert c in order[i, :P].tolist()    # k <= cluster c's size, so it is reached
        earlier = [p for p in F.growth(1, 12) if p < P]
        assert all(c not in order[i, :p].tolist() for p in earlier)
        assert allowed[i] == sizes[c] and rows[i] == sizes[order[i, :P]].sum()
        assert set(ids[i].tolist()) <= set(np.flatnonzero(mask).tolist())
    alone = [F.static(oracle, 0, x, cent, assign, q[i:i + 1], k, 1, mask) for i in range(len(q))]
    assert [int(a[2][0]) for a in alone] == probes.tolist()
    assert len(set(probes.tolist())) > 1


def test_dynamic_index_ignores_empty_slots_and_returns_external_ids(oracle, small):
    x, cent, assign, q = small
    ext = np.arange(len(x), dtype=np.uint64) * 3 + 11
    m = D.DynamicIVFModel.assemble(oracle, 0, cent, x, ext, assign)
    m.delete(ext[::4])
    allowed = np.ones(len(x), dtype=bool)     # Empty slots' bits set too
    ids, dists, probes, n_allowed, rows = F.dynamic(m, q, 10, 2, allowed)
    pid, _ = m.search(q, 10, 2)
    enough = probes == 2
    np.testing.assert_array_equal(ids[enough], pid[enough])
    live = m.live_slots()
    assert not np.isin(ids[ids != F.PAD_ID], ext[::4]).any()
    assert (n_allowed == rows).all() and rows.max() <= len(live)
    half = np.zeros(len(x), dtype=bool)
    half[::2] = True
    ids, _, _, n_allowed, rows = F.dynamic(m, q, 10, 12, half)
    want = set((ext[::2][np.isin(np.arange(0, len(x), 2), live)]).tolist())
    assert set(ids[ids != F.PAD_ID].tolist()) <= want and (n_allowed == len(want)).all()


def test_bitmap_layout():
    mask = np.zeros(70, dtype=bool)
    mask[[0, 31, 32, 63, 69]] = True
    b = F.bitmap(mask)
    assert b.dtype == np.uint32 and b.tolist() == [0x80000001, 0x80000001, 1 << 5]
