"""The IVF contract's numpy model (tests/ivf_model.py) on hand-made cases, without a GPU: the random sequence against the
library's own, the probe's ties, the union top k's padding, the k-means update, split and normalisation."""
import numpy as np
import pytest

import ivf_model as M


@pytest.fixture(scope="module")
def oracle():
    from oracle.bindings import OracleLib
    if not OracleLib.available():
        pytest.skip("oracle/liboracle.so not built")
    return OracleLib()


def test_random_sequence_matches_the_library():
    from scalablevectorsearch_b200 import _lib
    for seed in (0, 1, 0xC0FFEE, 2**64 - 1):
        out = np.empty(64, dtype=np.uint64)
        _lib.check(_lib.lib().svsb200_ivf_random(seed, 64, out.ctypes.data))
        assert [int(v) for v in out] == M.random_sequence(seed, 64)
    # splitmix64's published first output for seed 0
    assert M.random_sequence(0, 1)[0] == 0xE220A8397B1DCDAF


def test_training_sample_size_rules():
    assert M.num_training_rows(1000, 10, 0.1) == 100
    assert M.num_training_rows(1000, 80, 0.1) == 160        # at least 2 C
    assert M.num_training_rows(100, 80, 0.1) == 100         # capped at n
    assert M.num_training_rows(1001, 1, 0.5) == 501         # ceil


def test_probe_ties_go_to_the_lower_centroid(oracle):
    cent = np.array([[1, 0], [0, 1], [1, 0], [0, 1]], dtype=np.float32)
    q = np.array([[1, 1]], dtype=np.float32)          # equidistant from all four
    for metric in (0, 1, 2):
        assert M.nearest(oracle, metric, q, cent, 4).tolist() == [[0, 1, 2, 3]]
    q = np.array([[0, 2]], dtype=np.float32)
    assert M.nearest(oracle, 0, q, cent, 2).tolist() == [[1, 3]]


def test_union_smaller_than_k_is_padded(oracle):
    data = np.array([[0, 0], [1, 0], [5, 5], [6, 5], [7, 5]], dtype=np.float32)
    cent = np.array([[0.5, 0], [6, 5]], dtype=np.float32)
    assign = np.array([0, 0, 1, 1, 1], dtype=np.uint32)
    q = np.array([[0, 0.1]], dtype=np.float32)
    ids, dists = M.search(oracle, 0, data, cent, assign, q, 4, 1)
    assert ids[0].tolist() == [0, 1, 2**64 - 1, 2**64 - 1]
    assert np.isinf(dists[0, 2:]).all() and (dists[0, 2:] > 0).all()
    ids, dists = M.search(oracle, 1, data, cent, assign, q, 4, 1)   # MIP pads with -inf
    assert (dists[0, ids[0] == 2**64 - 1] == -np.inf).all()
    ids, _ = M.search(oracle, 0, data, cent, assign, q, 4, 2)
    assert ids[0].tolist() == [0, 1, 2, 3]


def test_equal_distances_order_by_id(oracle):
    data = np.array([[1, 0], [0, 1], [-1, 0], [0, -1]], dtype=np.float32)
    cent = np.array([[0, 0], [9, 9]], dtype=np.float32)
    assign = np.array([1, 0, 1, 0], dtype=np.uint32)
    ids, dists = M.search(oracle, 0, data, cent, assign, np.zeros((1, 2), np.float32), 4, 2)
    assert ids[0].tolist() == [0, 1, 2, 3] and (dists == 1).all()


def test_update_sums_in_float32_onto_the_old_centroid():
    # the (old + sum) / (count + 1) rule, in float32 and in row order: 1e8 + 1 + 1 + ... loses every 1
    cent = np.array([[1e8]], dtype=np.float32)
    s = cent[0].copy()
    for _ in range(4):
        s = (s + np.float32(1.0)).astype(np.float32)
    assert s[0] == np.float32(1e8)
    assert np.float32(1.0 / 5) * s[0] == np.float32(np.float32(0.2) * np.float32(1e8))


def test_split_copies_and_perturbs(oracle):
    cent = np.array([[2.0, 4.0, 8.0], [0.0, 0.0, 0.0]], dtype=np.float32)
    counts = np.array([7, 0])
    M.split(cent, counts, 7, M.Rng(5))       # p = 7 / 7 = 1: the first draw accepts cluster 0
    up, down = 1 + 2**-10, 1 - 2**-10
    assert cent[1].tolist() == [np.float32(2 * up), np.float32(4 * down), np.float32(8 * up)]
    assert cent[0].tolist() == [np.float32(2 * down), np.float32(4 * up), np.float32(8 * down)]
    assert counts.tolist() == [4, 3]


def test_kmeans_splits_an_empty_cluster(oracle):
    # 40 identical rows and 2 others, with a seed whose four initial centroids are all the repeated row: ties send every
    # row to centroid 0, so 1, 2 and 3 empty and must be split off a populated one
    data = np.zeros((42, 4), dtype=np.float32)
    data[:40] = [1, 2, 3, 4]
    data[40] = [9, 9, 9, 9]
    data[41] = [-9, 0, 9, 0]
    seed = next(s for s in range(1000) if _init_rows(s, 42, 4) == {0})
    cent, assign = M.kmeans(oracle, data, 0, 4, 1, 1.0, seed)
    assert len(np.unique(cent, axis=0)) == 4             # no two centroids left equal
    assert assign.shape == (42,) and assign.max() < 4


def _init_rows(seed, n, C):
    r = M.Rng(seed)
    sample = np.sort(r.shuffle_prefix(n, n))
    init = r.shuffle_prefix(n, C)
    return {0 if sample[i] < 40 else 1 for i in init}


@pytest.mark.parametrize("metric", [1, 2])
def test_kmeans_normalises_for_mip_and_cosine(oracle, metric):
    rng = np.random.default_rng(3)
    data = (rng.standard_normal((200, 8)) * 5 + 1).astype(np.float32)
    cent, assign = M.kmeans(oracle, data, metric, 6, 3, 0.5, 11)
    norms = np.sqrt((cent.astype(np.float64) ** 2).sum(1))
    assert np.allclose(norms, 1.0, atol=1e-6)
    assert np.array_equal(assign, M.nearest(oracle, metric, data, cent, 1)[:, 0])


# ---- the model against the reference's own IVF index (oracle/ivf.mk façade) on the reference's test dataset ----

@pytest.fixture(scope="module")
def ref_ivf():
    from oracle.ivf import RefIVF
    if not RefIVF.available():
        pytest.skip("oracle/_ref/libsvsref_ivf.so not built (needs the reference at build time)")
    return RefIVF()


@pytest.fixture(scope="module")
def dataset():
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "test_dataset.npz"))
    return z["data"].astype(np.float32), z["queries"].astype(np.float32), z


def _same_up_to_kth_ties(ids_a, d_a, ids_b, d_b):
    """Distance bits equal everywhere; the same ids at every distance above the k-th (the reference leaves the order
    inside a tie group unspecified, so a group compares as a set); ids at the k-th distance may differ (the group may
    continue past k)."""
    assert np.array_equal(d_a.view(np.uint32), d_b.view(np.uint32))
    for ia, ib, d in zip(ids_a, ids_b, d_a):
        for v in np.unique(d[d != d[-1]]):
            assert set(ia[d == v].tolist()) == set(ib[d == v].tolist())


@pytest.mark.parametrize("metric", [0, 1, 2])
def test_model_equals_the_reference_with_every_probe(oracle, ref_ivf, dataset, metric):
    x, q, _ = dataset
    cent, assign = M.kmeans(oracle, x, metric, 32, 3, 0.1, 1)
    ri, rd = ref_ivf.search(x, metric, cent, assign, q, 10, 32)
    mi, md = M.search(oracle, metric, x, cent, assign, q, 10, 32)
    _same_up_to_kth_ties(mi, md, ri, rd)


@pytest.mark.parametrize("metric,gt", [(0, "gt_l2"), (1, "gt_ip"), (2, "gt_cosine")])
def test_model_recall_matches_the_reference_with_fewer_probes(oracle, ref_ivf, dataset, metric, gt):
    # The reference ranks centroids from its GEMM, so its probe sets may differ at near-ties: recall@10 agrees within
    # 0.005, and the number of queries whose ids differ is reported.
    x, q, z = dataset
    truth = z[gt]
    cent, assign = M.kmeans(oracle, x, metric, 32, 3, 0.1, 1)

    def recall(ids):
        return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / 10 for a, b in zip(ids, truth)]))

    for n_probes in (2, 8):
        ri, _ = ref_ivf.search(x, metric, cent, assign, q, 10, n_probes)
        mi, _ = M.search(oracle, metric, x, cent, assign, q, 10, n_probes)
        print(f"metric {metric} n_probes {n_probes}: recall model {recall(mi):.4f} reference {recall(ri):.4f}, "
              f"{int((mi != ri).any(1).sum())} of {len(q)} queries with different ids")
        assert abs(recall(mi) - recall(ri)) <= 0.005
