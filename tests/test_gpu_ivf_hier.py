"""Hierarchical k-means on the GPU (svsb200_ivf_cluster_hierarchical: csrc/ivf.cu, ivf_group_assign_kernel and
ivf_kmeans_group_update_kernel in ivf_kernel.cuh) against the numpy model of tests/hier_kmeans_model.py: centroid bits,
assignments and level-2 counts; an IVF over the result at n_probes = C against the exact scan; recall on the reference
dataset; the refusals; and the runtime IVFIndex with is_hierarchical = true."""
import os
import subprocess

import numpy as np
import pytest

import hier_kmeans_model as H
from scalablevectorsearch_b200 import (IVF, Clustering, DistanceType, IVFBuildParameters, IVFSearchParameters,
                                       Svsb200Error, Vamana)
from test_gpu_ivf import _recall, _same, _scan, clustered

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIST = {0: DistanceType.L2, 1: DistanceType.MIP, 2: DistanceType.Cosine}


@pytest.fixture(scope="module")
def oracle():
    from oracle.bindings import OracleLib
    if not OracleLib.available():
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "oracle"])
    return OracleLib()


def _build(x, metric, C, L1, iters, frac, seed, minibatch):
    bp = IVFBuildParameters(num_centroids=C, hierarchical_level1_clusters=L1, num_iterations=iters,
                            training_fraction=frac, seed=seed, minibatch_size=minibatch)
    return Clustering.build_hierarchical(bp, x, DIST[metric])


def _same_as_model(got, want):
    assert np.array_equal(got.level2_counts, want.level2_counts)
    assert np.array_equal(got.centroids.view(np.uint32), want.centroids.view(np.uint32)), "centroid bits differ"
    assert np.array_equal(got.assignments, want.assignments), \
        f"{int((got.assignments != want.assignments).sum())} assignments differ"


@pytest.mark.parametrize("iters", [0, 4])
@pytest.mark.parametrize("C,L1,frac", [(64, 0, 0.1), (100, 7, 0.1), (40, 40, 0.01), (40, 1, 0.1)])
@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dtype", [np.float32, np.float16])
def test_clustering_matches_the_model_bit_for_bit(oracle, dtype, metric, C, L1, frac, iters):
    x = clustered(1500, 24, 12, seed=C + L1 + metric, dtype=dtype)
    want = H.hierarchical_kmeans(oracle, x, metric, C, L1, iters, frac, seed=5)
    if L1 == C:   # m = 2 C training rows: some groups get as many centroids as training rows
        assert (want.level2_counts == want.train_counts).any()
    for minibatch in (1000, 10_000):   # pieces of the assignment passes change no result
        _same_as_model(_build(x, metric, C, L1, iters, frac, 5, minibatch), want)


@pytest.mark.parametrize("metric", [0, 2])
def test_wide_rows_match_the_model(oracle, metric):
    # dimension 96 (the kernels' static shape) and 130 (generic, a masked tail)
    for dim in (96, 130):
        x = clustered(1200, dim, 10, seed=dim + metric)
        want = H.hierarchical_kmeans(oracle, x, metric, 30, 4, 3, 0.2, seed=8)
        _same_as_model(_build(x, metric, 30, 4, 3, 0.2, 8, 500), want)


def test_an_empty_level1_group(oracle):
    # repeated rows with no iterations: coinciding level-1 centroids leave a group without training rows, whose rows
    # go to the nearest populated group
    rng = np.random.default_rng(0)
    base = rng.standard_normal((3, 6)).astype(np.float32) * 4
    x = base[rng.integers(0, 3, 400)]
    x[:20] += 0.01 * rng.standard_normal((20, 6)).astype(np.float32)
    seed = next(s for s in range(40) if (H.hierarchical_kmeans(oracle, x, 0, 12, 4, 0, 0.5, s).train_counts == 0).any())
    want = H.hierarchical_kmeans(oracle, x, 0, 12, 4, 0, 0.5, seed)
    assert (want.level2_counts == 0).any()
    _same_as_model(_build(x, 0, 12, 4, 0, 0.5, seed, 100), want)


@pytest.mark.parametrize("metric", [0, 1, 2])
def test_all_probes_equal_the_exact_scan(metric):
    import torch
    x = clustered(5000, 96, 40, seed=metric)
    q = clustered(64, 96, 40, seed=metric + 100)
    clustering = _build(x, metric, 100, 0, 4, 0.2, 1, 10_000)
    index = IVF.assemble_from_clustering(clustering, x, DIST[metric])
    index.search_parameters = IVFSearchParameters(n_probes=100)
    scan = Vamana.from_arrays(x, np.zeros((x.shape[0], 2), dtype=np.uint32), 0, DIST[metric])
    for k in (1, 10, 100):
        _same(index.search(q, k), _scan(scan, q, k))
    torch.cuda.synchronize()


def test_recall_on_the_reference_dataset_grows_with_the_probes():
    z = np.load(os.path.join(ROOT, "tests", "golden", "test_dataset.npz"))
    x, q, gt = z["data"].astype(np.float32), z["queries"].astype(np.float32), z["gt_l2"]
    clustering = _build(x, 0, 64, 8, 10, 0.1, 0xC0FFEE, 10_000)
    index = IVF.assemble_from_clustering(clustering, x, DistanceType.L2)
    recalls = {}
    for n_probes in (1, 2, 4, 8, 16, 32, 64):
        index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        recalls[n_probes] = _recall(index.search(q, 10)[0], gt)
    print("hierarchical recall@10 by n_probes:", recalls)
    r = list(recalls.values())
    assert all(a <= b for a, b in zip(r, r[1:]))
    assert recalls[64] == 1.0


def test_refusals():
    x = clustered(600, 16, 8, seed=1)
    with pytest.raises(Svsb200Error, match="level1_clusters"):
        _build(x, 0, 8, 9, 1, 0.1, 0, 100)
    with pytest.raises(Svsb200Error, match="insufficient data"):
        _build(x, 0, 601, 0, 1, 0.1, 0, 100)
    for bad in (x.astype(np.int8), x.astype(np.uint8)):
        with pytest.raises(Svsb200Error, match="float32 or float16"):
            _build(bad, 0, 8, 0, 1, 0.1, 0, 100)
    with pytest.raises(Svsb200Error, match="is_hierarchical"):   # the flat entry point still refuses it
        Clustering.build(IVFBuildParameters(num_centroids=8, is_hierarchical=True), x, DistanceType.L2)


def test_runtime_ivf_index_demo_matches_the_c_abi(tmp_path):
    """cpp/ivf_hier_demo (svs::runtime::v0::IVFIndex with is_hierarchical = true, FP32 and SQI8 storage) prints the
    same results as Clustering.build_hierarchical + IVF.search with the same parameters."""
    from scalablevectorsearch_b200 import sq_compress
    exe = os.path.join(ROOT, "scalablevectorsearch_b200", "cpp", "_build", "ivf_hier_demo")
    if not os.path.exists(exe):
        pytest.skip("ivf_hier_demo not built (needs the reference's runtime headers at build time)")
    n, nq, dim, k, C, L1, iters, n_probes = 6000, 50, 48, 20, 64, 6, 4, 5
    x = clustered(n, dim, 25, seed=21)
    q = clustered(nq, dim, 25, seed=22)
    x.tofile(tmp_path / "x.f32")
    q.tofile(tmp_path / "q.f32")
    out = subprocess.run([exe, str(tmp_path / "x.f32"), str(n), str(dim), str(tmp_path / "q.f32"), str(nq), str(k), str(C),
                          str(L1), str(iters), str(n_probes)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    rows = {}
    for line in out.stdout.splitlines():
        tag, *rest = line.split()
        rows.setdefault(tag, []).append(rest)
    bp = IVFBuildParameters(num_centroids=C, hierarchical_level1_clusters=L1, num_iterations=iters)
    clustering = Clustering.build_hierarchical(bp, x, DistanceType.L2)
    codes, scale, bias = sq_compress(x)
    for tag, index in (("fp32", IVF.assemble_from_clustering(clustering, x, DistanceType.L2)),
                       ("sqi8", IVF.assemble_from_clustering(clustering, codes, DistanceType.L2, sq=(scale, bias)))):
        got_ids = np.array([int(r[0]) for r in rows[tag]], dtype=np.uint64).reshape(nq, k)
        got_d = np.array([float(r[1]) for r in rows[tag]]).astype(np.float32).reshape(nq, k)
        index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        _same((got_ids, got_d), index.search(q, k))
