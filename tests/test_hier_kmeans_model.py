"""The hierarchical k-means contract's numpy model (tests/hier_kmeans_model.py) without a GPU: the random streams, the
allocation of level-2 centroids and its guard, empty level-1 groups, the group ranges of the output; the model against
the reference's own hierarchical k-means (oracle/ivf_hier.mk façade) by the recall of an IVF over each clustering; and
the ctypes call of Clustering.build_hierarchical against a recording stub."""
import os

import numpy as np
import pytest

import hier_kmeans_model as H
import ivf_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def oracle():
    from oracle.bindings import OracleLib
    if not OracleLib.available():
        pytest.skip("oracle/liboracle.so not built")
    return OracleLib()


def blobs(n, dim, centres, seed):
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((centres, dim)).astype(np.float32) * 3
    return (c[rng.integers(0, centres, n)] + 0.4 * rng.standard_normal((n, dim))).astype(np.float32)


def _check_structure(res, C, L1):
    c = res.level2_counts.astype(np.int64)
    assert c.sum() == C
    assert (c <= res.train_counts).all()
    assert (c[res.train_counts == 0] == 0).all()
    start = np.concatenate([[0], np.cumsum(c)])
    g = res.level1
    assert (c[g] > 0).all()                                        # no row in a group without centroids
    assert ((res.assignments >= start[g]) & (res.assignments < start[g + 1])).all()


def test_streams_in_the_documented_order(oracle):
    x = blobs(600, 8, 6, seed=1)
    n, C, L1, seed = 600, 20, 4, 77
    res = H.hierarchical_kmeans(oracle, x, 0, C, L1, 0, 0.1, seed)   # no iterations: no split draws
    m = M.num_training_rows(n, C, 0.1)
    r = M.Rng(seed)
    r.shuffle_prefix(n, m)
    r.shuffle_prefix(m, L1)
    c, discarded = H.allocate([int(v) for v in res.train_counts], m, C, r)
    assert c == res.level2_counts.tolist() and discarded == res.discarded
    assert res.seeds == [r.next() for _ in range(L1)]
    # a group's stream starts with its init shuffle: group g's first centroid is its training row p[0]
    sample = np.sort(M.Rng(seed).shuffle_prefix(n, m))
    g = int(np.flatnonzero(res.level2_counts)[0])
    start = int(res.level2_counts[:g].sum())
    first = M.Rng(res.seeds[g]).shuffle_prefix(int(res.train_counts[g]), int(res.level2_counts[g]))[0]
    members = np.flatnonzero(res.train_level1 == g)
    assert np.array_equal(res.centroids[start], x[sample[members[first]]])


def test_allocation_floors_and_remainder():
    c, discarded = H.allocate([0, 1, 5, 4], 10, 10, M.Rng(1))
    assert c == [0, 1, 5, 4] and discarded == 0                       # floors exact: no draw
    c, _ = H.allocate([3, 3, 3, 1], 10, 5, M.Rng(2))                  # floors 1, 1, 1, 0 and two draws
    assert sum(c) == 5 and [min(v, 1) for v in c[:3]] == [1, 1, 1] and all(a >= b for a, b in zip(c, [1, 1, 1, 0]))
    # the draws follow the sequence: replay them
    r, want, total = M.Rng(2), [1, 1, 1, 0], 3
    while total < 5:
        j = r.next() % 4
        want[j] += 1
        total += 1
    assert c == want


def test_allocation_guard():
    # t = [1, 2, 2], m = 5, C = 4: floors 0, 1, 1; group 0 takes at most one of the two extra centroids
    seen_discard = False
    for seed in range(200):
        c, discarded = H.allocate([1, 2, 2], 5, 4, M.Rng(seed))
        assert sum(c) == 4 and c[0] <= 1 and c[1] <= 2 and c[2] <= 2
        seen_discard |= discarded > 0
    assert seen_discard
    for seed in range(50):                                            # a group without training rows gets nothing
        c, _ = H.allocate([0, 3, 3], 6, 5, M.Rng(seed))
        assert c[0] == 0 and sum(c) == 5


def test_empty_level1_group_rows_go_to_the_nearest_populated(oracle):
    # repeated rows: with no iterations two initial level-1 centroids coincide, ties send every row to the lower one,
    # and the higher one's group has no training rows and no centroids
    rng = np.random.default_rng(0)
    base = rng.standard_normal((3, 6)).astype(np.float32) * 4
    x = base[rng.integers(0, 3, 400)]
    x[:20] += 0.01 * rng.standard_normal((20, 6)).astype(np.float32)
    found = False
    for seed in range(40):
        res = H.hierarchical_kmeans(oracle, x, 0, 12, 4, 0, 0.5, seed)
        _check_structure(res, 12, 4)
        if (res.train_counts == 0).any():
            found = True
            empty = np.flatnonzero(res.level2_counts == 0)
            assert not np.isin(res.level1, empty).any()
            break
    assert found


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("C,L1", [(30, 0), (24, 5), (12, 12), (12, 1)])
def test_outputs_lie_in_their_groups_ranges(oracle, metric, C, L1):
    x = blobs(500, 8, 7, seed=C + L1)
    res = H.hierarchical_kmeans(oracle, x, metric, C, L1, 2, 0.2, seed=3)
    _check_structure(res, C, H.level1_clusters(C, L1))
    if metric:
        norms = np.sqrt((res.centroids.astype(np.float64) ** 2).sum(1))
        assert np.allclose(norms, 1.0, atol=1e-6)


def test_refusals(oracle):
    x = blobs(50, 4, 3, seed=0)
    with pytest.raises(ValueError, match="insufficient"):
        H.hierarchical_kmeans(oracle, x, 0, 51, 0, 1, 0.1, 0)
    with pytest.raises(ValueError, match="level1"):
        H.hierarchical_kmeans(oracle, x, 0, 10, 11, 1, 0.1, 0)


# ---- the model against the reference's hierarchical k-means on the reference's test dataset ----

@pytest.fixture(scope="module")
def ref_hier():
    from oracle.ivf_hier import RefHierarchicalKMeans
    if not RefHierarchicalKMeans.available():
        pytest.skip("oracle/_ref/libsvsref_ivf_hier.so not built (needs the reference at build time)")
    return RefHierarchicalKMeans()


@pytest.fixture(scope="module")
def dataset():
    z = np.load(os.path.join(ROOT, "tests", "golden", "test_dataset.npz"))
    return z["data"].astype(np.float32), z["queries"].astype(np.float32), z


# recall@10 of an IVF over the model's clustering against one over the reference's, at equal probes: the two draw
# different random sequences, so the clusterings differ; the bound is set from CPU runs of this test (DESIGN.md §15)
RECALL_TOLERANCE = 0.06


@pytest.mark.parametrize("metric,gt", [(0, "gt_l2"), (1, "gt_ip"), (2, "gt_cosine")])
def test_model_recall_matches_the_reference(oracle, ref_hier, dataset, metric, gt):
    x, q, z = dataset
    truth = z[gt]
    C, L1, iters = 64, 8, 10

    def recall(ids):
        return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / 10 for a, b in zip(ids, truth)]))

    model = H.hierarchical_kmeans(oracle, x, metric, C, L1, iters, 0.1, 1)
    rc, ra = ref_hier.cluster(x, metric, C, L1, iters, 0.1, 1)
    fc, fa = M.kmeans(oracle, x, metric, C, iters, 0.1, 1)
    assert np.bincount(ra, minlength=C).sum() == x.shape[0]
    for n_probes in (2, 8):
        got = recall(M.search(oracle, metric, x, model.centroids, model.assignments, q, 10, n_probes)[0])
        ref = recall(M.search(oracle, metric, x, rc, ra, q, 10, n_probes)[0])
        flat = recall(M.search(oracle, metric, x, fc, fa, q, 10, n_probes)[0])
        print(f"metric {metric} n_probes {n_probes}: recall@10 model {got:.4f} reference {ref:.4f} flat {flat:.4f}")
        assert abs(got - ref) <= RECALL_TOLERANCE
        assert abs(got - flat) <= RECALL_TOLERANCE


# ---- the binding's C call, against a recording stub ----

def test_build_hierarchical_binding(monkeypatch):
    from test_bindings_cpu import Stub, _calls, _rows
    from scalablevectorsearch_b200 import Clustering, DistanceType, IVFBuildParameters, _lib
    stub = Stub()
    monkeypatch.setattr(_lib, "_lib", stub)
    bp = IVFBuildParameters(num_centroids=5, minibatch_size=64, num_iterations=3, training_fraction=0.5,
                            hierarchical_level1_clusters=2, is_hierarchical=False, seed=9)
    got = Clustering.build_hierarchical(bp, _rows(dtype=np.float16), DistanceType.MIP, device=1)
    assert _calls(stub, False) == [("svsb200_ivf_cluster_hierarchical", "p", 1, 6, 4, 1, 5, 2, 64, 3, 0.5, 9, 1, "p", "p",
                                    "p")]
    assert got.centroids.shape == (5, 4) and got.assignments.shape == (6,) and got.level2_counts.shape == (2,)
    stub.calls.clear()
    bp.hierarchical_level1_clusters = 0                        # sqrt(5) = 2 level-1 groups
    got = Clustering.build_hierarchical(bp, _rows(), DistanceType.L2)
    assert _calls(stub, False) == [("svsb200_ivf_cluster_hierarchical", "p", 0, 6, 4, 0, 5, 0, 64, 3, 0.5, 9, 0, "p", "p",
                                    "p")]
    assert got.level2_counts.shape == (2,)
