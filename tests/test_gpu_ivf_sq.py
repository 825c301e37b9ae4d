"""The SQ IVF index on the GPU (svsb200_sq_compress, svsb200_ivf_create_sq; the tensor-core L2 leaf and the float-tree
MIP / cosine leaves of csrc/ivf_kernel.cuh) against the model of tests/ivf_sq_model.py and the C oracle: compression
bit for bit, search ids and distance bits, equality with the exact scan at n_probes = C, and the refusals."""
import os

import numpy as np
import pytest

import ivf_model as M
import ivf_sq_model as S
from scalablevectorsearch_b200 import (IVF, Clustering, DistanceType, IVFSearchParameters, Svsb200Error, Vamana,
                                       sq_compress)

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
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((centres, dim)).astype(np.float32) * 3
    w = rng.pareto(1.5, centres) + 0.2
    which = rng.choice(centres, n, p=w / w.sum())
    return (c[which] + spread * rng.standard_normal((n, dim)).astype(np.float32)).astype(dtype)


def centroids_for(x, C, seed):
    """C centroids from the rows, two far away so that their clusters stay empty."""
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


@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
@pytest.mark.parametrize("shape", [(10000, 128), (333, 37), (1, 5)])
def test_compression_equals_the_oracle(oracle, dtype, shape):
    rng = np.random.default_rng(shape[1])
    x = rng.standard_normal(shape).astype(np.float32)
    x.reshape(-1)[:2] = [-0.0, 0.0]
    codes, scale, bias = sq_compress(x, dtype)
    graph = np.zeros((shape[0], 2), dtype=np.uint32)
    index, want_codes, want_scale, want_bias = oracle.sq_index(x, graph, 0, "l2", code_dtype=dtype)
    index.close()
    assert np.float32(scale).view(np.uint32) == np.float32(want_scale).view(np.uint32)
    assert np.float32(bias).view(np.uint32) == np.float32(want_bias).view(np.uint32)
    assert np.array_equal(codes, want_codes)


def test_compression_refusals():
    with pytest.raises(Svsb200Error, match="constant"):
        sq_compress(np.full((10, 4), 2.5, dtype=np.float32))
    x = np.ones((10, 4), dtype=np.float32)
    x[3, 1] = np.nan
    with pytest.raises(Svsb200Error, match="NaN"):
        sq_compress(x)
    x[3, 1] = np.inf
    with pytest.raises(Svsb200Error, match="NaN"):
        sq_compress(x)


def _sq_index(x, C, metric, dtype, oracle):
    codes, scale, bias = S.compress(x, dtype)
    cent = centroids_for(x, C, seed=7)
    assign = M.nearest(oracle, metric, x, cent, 1)[:, 0].astype(np.uint32)
    index = IVF.assemble_from_clustering(Clustering(cent, assign), codes, DIST[metric], sq=(scale, bias))
    return index, codes, scale, bias, cent, assign


@pytest.mark.parametrize("C", [40, 520])
@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dtype,qdtype,dim", [(np.int8, np.float32, 96), (np.uint8, np.float16, 128),
                                              (np.int8, np.float16, 45), (np.uint8, np.float32, 96)])
def test_search_matches_the_model(oracle, C, metric, dtype, qdtype, dim):
    x = clustered(3000, dim, 30, seed=C + metric + dim)
    q = clustered(16, dim, 30, seed=C + metric + dim + 1, dtype=qdtype)
    index, codes, scale, bias, cent, assign = _sq_index(x, C, metric, dtype, oracle)
    assert np.array_equal(index.cluster_sizes, np.bincount(assign, minlength=C))
    if metric == 0:
        assert (index.cluster_sizes == 0).any()           # empty clusters
    if C == 40:
        assert index.cluster_sizes.max() > 64              # clusters larger than the ring
    for k in (1, 10, 100, 1024):
        for n_probes in (1, 8, C):
            index.search_parameters = IVFSearchParameters(n_probes=n_probes)
            got = index.search(q, k)
            want = S.search(oracle, metric, codes, scale, bias, cent, assign, q, k, n_probes)
            _same(got, want)


def _scan(scan, q, k):
    import torch
    dq = torch.from_numpy(q).cuda()
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
    d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
    scan.exhaustive_device(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), d.data_ptr(),
                           stream=torch.cuda.current_stream().cuda_stream or 1)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint64), d.cpu().numpy()


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
@pytest.mark.parametrize("dim", [96, 200])
def test_all_probes_equal_the_exact_scan(oracle, metric, dtype, dim):
    x = clustered(5000, dim, 40, seed=metric + dim)
    q = clustered(64, dim, 40, seed=metric + 100)
    index, codes, scale, bias, cent, assign = _sq_index(x, 50, metric, dtype, oracle)
    index.search_parameters = IVFSearchParameters(n_probes=50)
    scan = Vamana.from_arrays(codes, np.zeros((x.shape[0], 2), dtype=np.uint32), 0, DIST[metric], sq=(scale, bias))
    for k in (1, 10, 100, 1024):
        _same(index.search(q, k), _scan(scan, q, k))
        _same(index.search(q.astype(np.float16), k), _scan(scan, q.astype(np.float16), k))


def test_a_large_batch_crosses_the_query_chunks(oracle):
    # 10 000 queries at n_probes = 64 and k = 100: the per-(query, probe) lists take several chunks
    x = clustered(20000, 96, 60, seed=5)
    q = clustered(10000, 96, 60, seed=6)
    index, codes, scale, bias, cent, assign = _sq_index(x, 128, 0, np.int8, oracle)
    index.search_parameters = IVFSearchParameters(n_probes=64)
    ids, dists = index.search(q, 100)
    for lo in (0, 4999, 9990):
        _same((ids[lo:lo + 10], dists[lo:lo + 10]),
              S.search(oracle, 0, codes, scale, bias, cent, assign, q[lo:lo + 10], 100, 64))


def test_unions_smaller_than_k_are_padded(oracle):
    x = clustered(300, 64, 5, seed=9)
    q = clustered(8, 64, 5, seed=10)
    index, codes, scale, bias, cent, assign = _sq_index(x, 40, 1, np.int8, oracle)
    index.search_parameters = IVFSearchParameters(n_probes=2)
    ids, dists = index.search(q, 1024)
    assert (ids == M.PAD_ID).any() and np.isneginf(dists[ids == M.PAD_ID]).all()
    _same((ids, dists), S.search(oracle, 1, codes, scale, bias, cent, assign, q, 1024, 2))


def test_refusals():
    x = np.random.default_rng(0).standard_normal((100, 16)).astype(np.float32)
    codes, scale, bias = sq_compress(x)
    cent = x[:4].copy()
    with pytest.raises(Svsb200Error, match="need assignments"):
        IVF.assemble_from_clustering(Clustering(cent), codes, DistanceType.L2, sq=(scale, bias))
    assign = np.zeros(100, dtype=np.uint32)
    for bad in ((0.0, bias), (-1.0, bias), (float("nan"), bias), (scale, float("inf"))):
        with pytest.raises(Svsb200Error, match="scale"):
            IVF.assemble_from_clustering(Clustering(cent, assign), codes, DistanceType.L2, sq=bad)
    with pytest.raises(TypeError, match="codes"):
        IVF.assemble_from_clustering(Clustering(cent, assign), x, DistanceType.L2, sq=(scale, bias))
    with pytest.raises(Svsb200Error, match="float32 or float16"):   # integer rows without sq= as before
        IVF.assemble_from_clustering(Clustering(cent, assign), codes, DistanceType.L2)


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dim,k", [(2048, 10), (2048, 1024), (4096, 1024)])
def test_wide_rows(oracle, metric, dim, k):
    # rows over 1536 bytes stage 16- or 8-row tiles (the tensor-core leaf's second row block is idle); with k = 1024 the
    # code slots still fit a CTA wherever the float leaf's query slots do
    x = clustered(400, dim, 6, seed=dim + k)
    q = clustered(20, dim, 6, seed=dim + k + 1)
    index, codes, scale, bias, cent, assign = _sq_index(x, 12, metric, np.int8, oracle)
    scan = Vamana.from_arrays(codes, np.zeros((x.shape[0], 2), dtype=np.uint32), 0, DIST[metric], sq=(scale, bias))
    index.search_parameters = IVFSearchParameters(n_probes=12)
    _same(index.search(q, k), _scan(scan, q, k))
    index.search_parameters = IVFSearchParameters(n_probes=3)
    _same(index.search(q, k), S.search(oracle, metric, codes, scale, bias, cent, assign, q, k, 3))
