"""The IVF index on the GPU (csrc/ivf.cu, ivf_kernel.cuh) against the numpy model of tests/ivf_model.py: search ids
and distance bits for every query, equality with the exact scan at n_probes = C, k-means centroids and assignments bit
for bit, recall on the reference dataset, and the refusals."""
import os

import numpy as np
import pytest

import ivf_model as M
from scalablevectorsearch_b200 import (IVF, Clustering, DistanceType, IVFBuildParameters, IVFSearchParameters,
                                       Svsb200Error, Vamana)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIST = {0: DistanceType.L2, 1: DistanceType.MIP, 2: DistanceType.Cosine}


@pytest.fixture(scope="module")
def oracle():
    from oracle.bindings import OracleLib
    if not OracleLib.available():
        import subprocess
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "oracle"])
    return OracleLib()


def clustered(n, dim, centres, seed, dtype=np.float32, spread=0.3):
    """Rows around `centres` random centres, cluster sizes skewed (some clusters far larger than the ring's 64 rows)."""
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((centres, dim)).astype(np.float32) * 3
    w = rng.pareto(1.5, centres) + 0.2
    which = rng.choice(centres, n, p=w / w.sum())
    x = c[which] + spread * rng.standard_normal((n, dim)).astype(np.float32)
    return x.astype(dtype)


def centroids_for(x, C, seed):
    """C centroids from the rows, two of them far away so that their clusters stay empty."""
    rng = np.random.default_rng(seed)
    cent = x[rng.choice(x.shape[0], C, replace=False)].astype(np.float32)
    cent[C // 3] = 1000.0
    cent[C // 2] = -1000.0
    return cent


def _same(got, want):
    gi, gd = got
    wi, wd = want
    assert np.array_equal(gi, wi), f"ids differ in {np.flatnonzero((gi != wi).any(1))[:10]} queries"
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32)), "distance bits differ"


@pytest.mark.parametrize("C", [40, 520])
@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dtype,qdtype,dim", [(np.float32, np.float32, 96), (np.float32, np.float16, 40),
                                              (np.float16, np.float32, 33), (np.float16, np.float16, 96)])
def test_search_matches_the_model(oracle, C, metric, dtype, qdtype, dim):
    x = clustered(4000, dim, 30, seed=C + metric + dim, dtype=dtype)
    q = clustered(24, dim, 30, seed=C + metric + dim, dtype=qdtype)
    cent = centroids_for(x.astype(np.float32), C, seed=7)
    index = IVF.assemble_from_clustering(Clustering(cent), x, DIST[metric])   # assignment on the device
    want_assign = M.nearest(oracle, metric, x, cent, 1)[:, 0]
    assert np.array_equal(index.cluster_sizes, np.bincount(want_assign, minlength=C))
    if C == 40:
        assert index.cluster_sizes.max() > 64                # clusters larger than the ring
    if metric == 0:
        assert (index.cluster_sizes == 0).any()               # empty clusters
    for k in (1, 10, 100, 1024):
        for n_probes in (1, 8, C):
            index.search_parameters = IVFSearchParameters(n_probes=n_probes)
            got = index.search(q, k)
            want = M.search(oracle, metric, x, cent, want_assign, q, k, n_probes)
            _same(got, want)


def _device_search(index, q, k):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
    d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
    index.search_device(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), d.data_ptr(),
                        stream=torch.cuda.current_stream().cuda_stream or 1)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint64), d.cpu().numpy()


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("C", [33, 600])
def test_all_probes_equal_the_exact_scan(metric, C):
    x = clustered(5000, 96, 40, seed=metric)
    q = clustered(64, 96, 40, seed=metric + 100)
    cent = centroids_for(x, C, seed=1)
    index = IVF.assemble_from_clustering(Clustering(cent), x, DIST[metric])
    index.search_parameters = IVFSearchParameters(n_probes=C)
    scan = Vamana.from_arrays(x, np.zeros((x.shape[0], 2), dtype=np.uint32), 0, DIST[metric])
    for k in (1, 10, 100, 1024):
        got = _device_search(index, q, k)
        _same(got, _scan(scan, q, k))
        _same(index.search(q, k), got)


def _scan(scan, q, k):
    import torch
    dq = torch.from_numpy(q).cuda()
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
    d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
    scan.exhaustive_device(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), d.data_ptr(),
                           stream=torch.cuda.current_stream().cuda_stream or 1)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint64), d.cpu().numpy()


def test_a_large_batch_crosses_the_query_chunks(oracle):
    # 10 000 queries at n_probes = 64 and k = 100: the per-(query, probe) lists take several chunks of the budget
    x = clustered(20000, 96, 60, seed=5)
    q = clustered(10000, 96, 60, seed=6)
    cent = centroids_for(x, 128, seed=2)
    assign = M.nearest(oracle, 0, x, cent, 1)[:, 0].astype(np.uint32)
    index = IVF.assemble_from_clustering(Clustering(cent, assign), x, DistanceType.L2)
    index.search_parameters = IVFSearchParameters(n_probes=64)
    ids, dists = index.search(q, 100)
    for lo in (0, 3333, 6667, 9900):   # the same queries in small batches
        _same((ids[lo:lo + 100], dists[lo:lo + 100]), index.search(q[lo:lo + 100], 100))
    pick = np.arange(0, 10000, 250)
    _same((ids[pick], dists[pick]), M.search(oracle, 0, x, cent, assign, q[pick], 100, 64))
    index.search_parameters = IVFSearchParameters(n_probes=8)
    pick = np.arange(0, 10000, 97)
    got = index.search(q, 10)
    _same((got[0][pick], got[1][pick]), M.search(oracle, 0, x, cent, assign, q[pick], 10, 8))


@pytest.mark.parametrize("metric", [0, 1, 2])
def test_clustering_matches_the_model_bit_for_bit(oracle, metric):
    x = clustered(3000, 24, 20, seed=metric + 40)
    bp = IVFBuildParameters(num_centroids=30, num_iterations=5, training_fraction=0.5, seed=metric + 9)
    got = Clustering.build(bp, x, DIST[metric])
    cent, assign = M.kmeans(oracle, x, metric, 30, 5, 0.5, metric + 9)
    assert np.array_equal(got.centroids.view(np.uint32), cent.view(np.uint32))
    assert np.array_equal(got.assignments, assign)
    bp.minibatch_size = 77   # only bounds the assignment batches
    again = Clustering.build(bp, x, DIST[metric])
    assert np.array_equal(again.centroids.view(np.uint32), got.centroids.view(np.uint32))
    assert np.array_equal(again.assignments, got.assignments)


@pytest.mark.parametrize("C", [24, 520])
def test_clustering_splits_empty_clusters(oracle, C):
    # most rows repeat a handful of values: initial centroids coincide, ties empty all but the lowest of each group,
    # and the split has to refill them (C = 520 assigns on the tensor cores)
    rng = np.random.default_rng(C)
    base = rng.standard_normal((6, 16)).astype(np.float32)
    x = base[rng.integers(0, 6, 2400)]
    x[:200] = rng.standard_normal((200, 16)).astype(np.float32)
    x = x.astype(np.float16)
    bp = IVFBuildParameters(num_centroids=C, num_iterations=3, training_fraction=0.3, seed=3)
    got = Clustering.build(bp, x, DistanceType.L2)
    cent, assign = M.kmeans(oracle, x, 0, C, 3, 0.3, 3)
    assert np.array_equal(got.centroids.view(np.uint32), cent.view(np.uint32))
    assert np.array_equal(got.assignments, assign)


def _recall(ids, gt):
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / gt.shape[1] for a, b in zip(ids, gt)]))


def test_recall_on_the_reference_dataset_grows_with_the_probes():
    z = np.load(os.path.join(ROOT, "tests", "golden", "test_dataset.npz"))
    x, q, gt = z["data"].astype(np.float32), z["queries"].astype(np.float32), z["gt_l2"]
    clustering = Clustering.build(IVFBuildParameters(num_centroids=64, num_iterations=10), x, DistanceType.L2)
    index = IVF.assemble_from_clustering(clustering, x, DistanceType.L2)
    scan = Vamana.from_arrays(x, np.zeros((x.shape[0], 2), dtype=np.uint32), 0, DistanceType.L2)
    exact = _recall(_scan(scan, q, 10)[0], gt)
    recalls = {}
    for n_probes in (1, 2, 4, 8, 16, 32, 64):
        index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        recalls[n_probes] = _recall(index.search(q, 10)[0], gt)
    print("recall@10 by n_probes:", recalls, "exact scan:", exact)
    r = list(recalls.values())
    assert all(a <= b for a, b in zip(r, r[1:]))
    assert recalls[64] == exact == 1.0


def test_refusals_leave_nothing_changed():
    x = clustered(600, 16, 8, seed=1)
    q = x[:5]
    cent = centroids_for(x, 8, seed=1)
    index = IVF.assemble_from_clustering(Clustering(cent), x, DistanceType.L2)
    index.search_parameters = IVFSearchParameters(n_probes=3)
    before = index.search(q, 10)
    for k in (0, 1025):
        with pytest.raises(Svsb200Error, match="k must be"):
            index.search(q, k)
    for n_probes in (0, 9):
        index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        with pytest.raises(Svsb200Error, match="n_probes"):
            index.search(q, 10)
    index.search_parameters = IVFSearchParameters(n_probes=3, k_reorder=0.5)
    with pytest.raises(ValueError, match="k_reorder"):
        index.search(q, 10)
    index.search_parameters = IVFSearchParameters(n_probes=3)
    with pytest.raises(ValueError):
        index.search(q[:, :15], 10)
    with pytest.raises(Svsb200Error, match="float32 or float16"):
        index.search(q.astype(np.int8), 10)
    _same(index.search(q, 10), before)
    for bad in (x.astype(np.int8), x.astype(np.uint8)):
        with pytest.raises(Svsb200Error, match="float32 or float16"):
            IVF.assemble_from_clustering(Clustering(cent), bad, DistanceType.L2)
        with pytest.raises(Svsb200Error, match="float32 or float16"):
            Clustering.build(IVFBuildParameters(num_centroids=8), bad, DistanceType.L2)
    with pytest.raises(Svsb200Error, match="is_hierarchical"):
        Clustering.build(IVFBuildParameters(num_centroids=8, is_hierarchical=True), x, DistanceType.L2)
    with pytest.raises(Svsb200Error, match="insufficient data"):
        Clustering.build(IVFBuildParameters(num_centroids=601), x, DistanceType.L2)
    with pytest.raises(Svsb200Error, match="not a cluster"):
        IVF.assemble_from_clustering(Clustering(cent, np.full(600, 8, np.uint32)), x, DistanceType.L2)
    _same(index.search(q, 10), before)


def test_runtime_ivf_index_demo_matches_the_c_abi(tmp_path):
    """cpp/ivf_demo, written against the reference's runtime header only (svs::runtime::v0::IVFIndex) and linked with
    libsvsb200_runtime.so, prints the same results as Clustering.build + IVF.search with the same parameters, LVQ
    storage NOT_IMPLEMENTED (3) and k = 0 INVALID_ARGUMENT (2)."""
    import subprocess
    exe = os.path.join(ROOT, "scalablevectorsearch_b200", "cpp", "_build", "ivf_demo")
    if not os.path.exists(exe):
        pytest.skip("ivf_demo not built (needs the reference's runtime headers at build time)")
    n, nq, dim, k, C, iters, n_probes = 6000, 50, 48, 20, 40, 4, 5
    x = clustered(n, dim, 25, seed=21)
    q = clustered(nq, dim, 25, seed=22)
    x.tofile(tmp_path / "x.f32")
    q.tofile(tmp_path / "q.f32")
    out = subprocess.run([exe, str(tmp_path / "x.f32"), str(n), str(dim), str(tmp_path / "q.f32"), str(nq), str(k), str(C),
                          str(iters), str(n_probes)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    rows = {}
    for line in out.stdout.splitlines():
        tag, *rest = line.split()
        rows.setdefault(tag, []).append(rest)
    assert rows["storage_lvq8"] == [["3"]] and rows["k0"] == [["2"]]
    got_ids = np.array([int(r[0]) for r in rows["result"]], dtype=np.uint64).reshape(nq, k)
    got_d = np.array([float(r[1]) for r in rows["result"]]).astype(np.float32).reshape(nq, k)
    clustering = Clustering.build(IVFBuildParameters(num_centroids=C, num_iterations=iters), x, DistanceType.L2)
    index = IVF.assemble_from_clustering(clustering, x, DistanceType.L2)
    index.search_parameters = IVFSearchParameters(n_probes=n_probes)
    _same((got_ids, got_d), index.search(q, k))
