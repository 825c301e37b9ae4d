"""The filtered search of the IVF and dynamic IVF indexes on the GPU (svsb200_ivf_search_filtered,
svsb200_dynamic_ivf_search_filtered and their device forms) against the numpy model of tests/ivf_filtered_model.py, bit
for bit: ids, distance bits, and per query the probes used, the allowed rows and the rows of the probed clusters.
Covers every metric, row type, query type and storage kind, k up to 1024, selectivities from everything to nothing,
growth up to and past P_max, per-query independence, a batch across the query chunks, the dynamic index through its
mutations, a delete right after a device search, the refusals, and the runtime classes through an IDFilter."""
import os
import subprocess

import numpy as np
import pytest

import ivf_filtered_model as F
import ivf_model as M
from dynamic_ivf_model import DynamicIVFModel
from dynamic_ivf_sq_model import DynamicIVFSQModel
from scalablevectorsearch_b200 import (IVF, Clustering, DistanceType, DynamicIVF, IVFBuildParameters,
                                       IVFSearchParameters, Svsb200Error, _lib, sq_compress)
from scalablevectorsearch_b200.vamana import _DTYPE_CODE

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIST = {0: DistanceType.L2, 1: DistanceType.MIP, 2: DistanceType.Cosine}
KS = (1, 10, 100, 1024)


@pytest.fixture(scope="module")
def oracle():
    from oracle.bindings import OracleLib
    if not OracleLib.available():
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "oracle"])
    return OracleLib()


def clustered(n, dim, centres, seed, dtype=np.float32, spread=0.3):
    """Rows around `centres` random centres, cluster sizes skewed."""
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((centres, dim)).astype(np.float32) * 3
    w = rng.pareto(1.5, centres) + 0.2
    which = rng.choice(centres, n, p=w / w.sum())
    return (c[which] + spread * rng.standard_normal((n, dim)).astype(np.float32)).astype(dtype)


def centroids_for(x, C, seed):
    """C centroids from the rows, two of them far away so that their clusters stay empty."""
    rng = np.random.default_rng(seed)
    cent = x[rng.choice(x.shape[0], C, replace=False)].astype(np.float32)
    cent[C // 3] = 1000.0
    cent[C // 2] = -1000.0
    return cent


def _same(got, want, what=""):
    gi, gd, gp, ga, gr = got
    wi, wd, wp, wa, wr = want
    assert np.array_equal(gi, wi), f"{what}: ids differ in queries {np.flatnonzero((gi != wi).any(1))[:10]}"
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32)), f"{what}: distance bits differ"
    assert np.array_equal(gp, wp), f"{what}: probes {gp[:8]} != {wp[:8]}"
    assert np.array_equal(ga, wa), f"{what}: allowed counts differ"
    assert np.array_equal(gr, wr), f"{what}: row counts differ"


def _host(index, q, k, mask):
    ids, dists, found, (probes, allowed, rows) = index.search_filtered(q, k, mask, with_counts=True)
    assert np.array_equal(found, np.minimum(allowed, k))
    return ids, dists, probes, allowed, rows


def _device(index, q, k, mask):
    import torch
    nq = q.shape[0]
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    bm = torch.from_numpy(F.bitmap(mask).view(np.int32).copy()).cuda()
    ids = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    d = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    cnt = torch.empty((3, nq), dtype=torch.int32, device="cuda")
    index.search_filtered_device(dq.data_ptr(), q.dtype, nq, k, bm.data_ptr(), ids.data_ptr(), d.data_ptr(),
                                 cnt[0].data_ptr(), cnt[1].data_ptr(), cnt[2].data_ptr(),
                                 stream=torch.cuda.current_stream().cuda_stream or 1)
    torch.cuda.synchronize()
    c = cnt.cpu().numpy().view(np.uint32)
    return ids.cpu().numpy().view(np.uint64), d.cpu().numpy(), c[0], c[1], c[2]


def _static(oracle, metric, dtype=np.float32, n=3000, dim=40, C=40, seed=0):
    x = clustered(n, dim, 30, seed=seed + metric + dim, dtype=dtype)
    cent = centroids_for(x.astype(np.float32), C, seed=7)
    assign = M.nearest(oracle, metric, x, cent, 1)[:, 0].astype(np.uint32)
    return x, cent, assign, IVF.assemble_from_clustering(Clustering(cent, assign), x, DIST[metric])


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dtype,qdtype,dim", [(np.float32, np.float32, 96), (np.float32, np.float16, 40),
                                              (np.float16, np.float32, 33), (np.float16, np.float16, 96)])
def test_every_metric_row_and_query_type(oracle, metric, dtype, qdtype, dim):
    x, cent, assign, index = _static(oracle, metric, dtype, dim=dim)
    q = clustered(16, dim, 30, seed=metric + dim + 50, dtype=qdtype)
    mask = np.random.default_rng(metric + dim).random(len(x)) < 0.5
    for n_probes in (1, 3, 40):
        index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        for k in KS:
            want = F.static(oracle, metric, x, cent, assign, q, k, n_probes, mask)
            _same(_host(index, q, k, mask), want, f"k={k} n_probes={n_probes}")
    index.search_parameters = IVFSearchParameters(n_probes=3)
    _same(_device(index, q, 100, mask), _host(index, q, 100, mask), "device form")


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("code", [np.int8, np.uint8])
def test_sq_storage(oracle, metric, code):
    x = clustered(3000, 48, 30, seed=metric + 11)
    q = clustered(16, 48, 30, seed=metric + 12)
    codes, scale, bias = sq_compress(x, code)
    cent = centroids_for(x, 40, seed=3)
    assign = M.nearest(oracle, metric, x, cent, 1)[:, 0].astype(np.uint32)
    index = IVF.assemble_from_clustering(Clustering(cent, assign), codes, DIST[metric], sq=(scale, bias))
    mask = np.random.default_rng(metric).random(len(x)) < 0.3
    for qq in (q, q.astype(np.float16)):
        for n_probes in (1, 3, 40):
            index.search_parameters = IVFSearchParameters(n_probes=n_probes)
            for k in KS:
                want = F.static_sq(oracle, metric, codes, scale, bias, cent, assign, qq, k, n_probes, mask)
                _same(_host(index, qq, k, mask), want, f"{qq.dtype} k={k} n_probes={n_probes}")


def _masks(x, assign, cent, q, oracle, metric):
    rng = np.random.default_rng(5)
    n = len(x)
    one = np.zeros(n, dtype=bool)
    one[n // 2] = True
    order = F.probe_order(oracle, metric, q, cent)
    late = set.intersection(*(set(o[4:].tolist()) for o in order))   # clusters no query ranks in its first 4: growth
    bits = np.zeros(n, dtype=bool)
    bits[31::32] = True                                  # bit 31 of full words ...
    bits[n - (n % 32):] = True                           # ... and the last, partial word
    return {"all": np.ones(n, dtype=bool), "50%": rng.random(n) < 0.5, "10%": rng.random(n) < 0.1,
            "1%": rng.random(n) < 0.01, "one id": one, "none": np.zeros(n, dtype=bool),
            "clusters": np.isin(assign, list(late)), "bit 31 and the last word": bits}


@pytest.mark.parametrize("metric", [0, 1])
def test_selectivity(oracle, metric):
    x, cent, assign, index = _static(oracle, metric, n=3001, dim=32, C=60)
    q = clustered(24, 32, 30, seed=metric + 77)
    for name, mask in _masks(x, assign, cent, q, oracle, metric).items():
        for n_probes, k in ((1, 10), (2, 100)):
            index.search_parameters = IVFSearchParameters(n_probes=n_probes)
            want = F.static(oracle, metric, x, cent, assign, q, k, n_probes, mask)
            got = _host(index, q, k, mask)
            _same(got, want, f"{name} k={k} n_probes={n_probes}")
            if name == "clusters" and n_probes == 1:
                assert (got[2] >= 16).all(), "the cluster-correlated mask forces growth"
            if name == "none":
                assert (got[0] == F.PAD_ID).all() and (got[1] == np.inf).all() and (got[2] == 60).all()


def test_all_ones_mask_keeps_the_plain_rows(oracle):
    for metric in (0, 1, 2):
        x, cent, assign, index = _static(oracle, metric, n=3000, dim=32, C=40)
        q = clustered(32, 32, 30, seed=metric + 5)
        for n_probes in (1, 3):
            index.search_parameters = IVFSearchParameters(n_probes=n_probes)
            ids, dists, probes, allowed, rows = _host(index, q, 50, np.ones(len(x), dtype=bool))
            pi, pd = index.search(q, 50)
            assert (allowed == rows).all()
            for i in np.flatnonzero(probes == n_probes):   # (a query short of k rows probes further)
                real = ids[i] != F.PAD_ID
                assert np.array_equal(ids[i], pi[i])
                assert np.array_equal(dists[i, real].view(np.uint32), pd[i, real].view(np.uint32))
                assert (dists[i, ~real] == np.inf).all()


def test_growth_clips_at_p_max(oracle):
    # C = 1100 > 1024: the allowed cluster ranks past 1024 for the first query, which stays short at P_max
    x = clustered(6000, 16, 200, seed=9, spread=1.0)
    cent = x[np.random.default_rng(1).choice(6000, 1100, replace=False)].astype(np.float32)
    assign = M.nearest(oracle, 0, x, cent, 1)[:, 0].astype(np.uint32)
    index = IVF.assemble_from_clustering(Clustering(cent, assign), x, DistanceType.L2)
    q = clustered(48, 16, 200, seed=10, spread=1.0)
    late = M.nearest(oracle, 0, q[:1], cent, 1100)[0, 1024:]
    sizes = np.bincount(assign, minlength=1100)
    c = int(late[np.argmax(sizes[late])])
    mask = assign == c
    for n_probes in (1, 3):   # 1, 4, ..., 1024 and 3, 12, 48, 192, 768, then 1024 (not 3072 or C)
        index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        want = F.static(oracle, 0, x, cent, assign, q, 5, n_probes, mask)
        got = _host(index, q, 5, mask)
        _same(got, want, f"clip from {n_probes}")
        assert got[2][0] == 1024 and got[3][0] == 0 and (got[0][0] == F.PAD_ID).all()
        assert (got[2] <= 1024).all()


def test_each_query_alone_equals_its_row(oracle):
    x, cent, assign, index = _static(oracle, 0, n=3000, dim=32, C=60)
    q = clustered(20, 32, 30, seed=41)
    mask = np.isin(assign, np.arange(0, 60, 7))
    index.search_parameters = IVFSearchParameters(n_probes=1)
    batch = _host(index, q, 30, mask)
    assert len(set(batch[2].tolist())) > 1, "the batch mixes probe counts"
    for i in range(len(q)):
        alone = _host(index, q[i:i + 1], 30, mask)
        _same(alone, tuple(a[i:i + 1] for a in batch), f"query {i}")


def test_a_large_batch_crosses_the_query_chunks(oracle):
    x = clustered(20000, 64, 60, seed=5)
    q = clustered(10000, 64, 60, seed=6)
    cent = centroids_for(x, 128, seed=2)
    assign = M.nearest(oracle, 0, x, cent, 1)[:, 0].astype(np.uint32)
    index = IVF.assemble_from_clustering(Clustering(cent, assign), x, DistanceType.L2)
    mask = np.random.default_rng(1).random(len(x)) < 0.05
    index.search_parameters = IVFSearchParameters(n_probes=16)
    got = _host(index, q, 100, mask)
    assert set(got[2].tolist()) == {16, 64}, "most queries stay at 16 probes (over several chunks), some grow to 64"
    _same(_device(index, q, 100, mask), got, "device form")
    for lo in (0, 4321, 9900):
        _same(_host(index, q[lo:lo + 100], 100, mask), tuple(a[lo:lo + 100] for a in got), f"queries {lo}..")
    pick = np.arange(0, 10000, 400)
    _same(tuple(a[pick] for a in got), F.static(oracle, 0, x, cent, assign, q[pick], 100, 16, mask), "model")


def _dynamic_pair(oracle, metric, sq, x, n0, ids, C):
    cent = centroids_for(x, C, seed=4)
    assign = M.nearest(oracle, metric, x[:n0], cent, 1)[:, 0].astype(np.uint32)
    if sq:
        codes, scale, bias = sq_compress(x, np.int8)
        index = DynamicIVF.assemble_from_clustering(Clustering(cent, assign), codes[:n0], ids[:n0], DIST[metric],
                                                    sq=(scale, bias))
        model = DynamicIVFSQModel.assemble(oracle, metric, cent, codes[:n0], ids[:n0], scale, bias, assign)
    else:
        index = DynamicIVF.assemble_from_clustering(Clustering(cent, assign), x[:n0], ids[:n0], DIST[metric])
        model = DynamicIVFModel.assemble(oracle, metric, cent, x[:n0], ids[:n0], assign)
    return index, model


def _dynamic_equal(index, model, q, mask_of, what):
    status, ext, _ = index.export()
    mask = mask_of(status, ext)
    for n_probes, k in ((1, 10), (3, 100), (40, 1024)):
        index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        want = F.dynamic(model, q, k, n_probes, mask)
        _same(_host(index, q, k, mask), want, f"{what} k={k} n_probes={n_probes}")
    index.search_parameters = IVFSearchParameters(n_probes=3)
    _same(_device(index, q, 10, mask), F.dynamic(model, q, 10, 3, mask), f"{what} device form")


@pytest.mark.parametrize("sq", [False, True])
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("deleted", [0.2, 0.6])
def test_dynamic_index(oracle, sq, metric, deleted):
    n, n0, C = 3000, 2400, 40
    x = clustered(n, 32, 30, seed=int(deleted * 10) + metric)
    q = clustered(16, 32, 30, seed=99)
    ids = np.arange(n, dtype=np.uint64) * 5 + 3
    index, model = _dynamic_pair(oracle, metric, sq, x, n0, ids, C)
    rng = np.random.default_rng(metric)
    gone = ids[:n0][rng.random(n0) < deleted]
    index.delete(gone)
    model.delete(gone)
    # every slot's bit set, Empty ones included, or a random half of them; and half of the external ids
    half = rng.random(n) < 0.5
    masks = {"all": lambda s, e: np.ones(len(s), dtype=bool), "half of the slots": lambda s, e: half[:len(s)],
             "ids % 3": lambda s, e: (e % 3 == 0) & (s == 1)}
    for name, mask_of in masks.items():
        _dynamic_equal(index, model, q, mask_of, f"deleted {deleted}, {name}")
    index.add(x[n0:], ids[n0:], reuse_empty=True)   # (float32 rows: an SQ index encodes them)
    model.add(x[n0:], ids[n0:], reuse_empty=True)
    _dynamic_equal(index, model, q, masks["half of the slots"], "after reuse_empty adds")
    index.compact()
    model.compact()
    _dynamic_equal(index, model, q, masks["ids % 3"], "after compact")


def test_a_delete_right_after_a_device_search(oracle):
    import torch
    n, C = 4000, 40
    x = clustered(n, 64, 30, seed=3)
    q = clustered(2000, 64, 30, seed=4)
    ids = np.arange(n, dtype=np.uint64) + 100
    index, model = _dynamic_pair(oracle, 0, False, x, n, ids, C)
    index.search_parameters = IVFSearchParameters(n_probes=8)
    mask = np.random.default_rng(2).random(n) < 0.3
    dq = torch.from_numpy(q).cuda()
    bm = torch.from_numpy(F.bitmap(mask).view(np.int32).copy()).cuda()
    di = torch.empty((len(q), 100), dtype=torch.int64, device="cuda")
    dd = torch.empty((len(q), 100), dtype=torch.float32, device="cuda")
    index.search_filtered_device(dq.data_ptr(), q.dtype, len(q), 100, bm.data_ptr(), di.data_ptr(), dd.data_ptr(),
                                 stream=torch.cuda.current_stream().cuda_stream or 1)
    index.delete(ids[::2])                       # no synchronisation in between: the delete waits for the search
    torch.cuda.synchronize()
    pick = np.arange(0, len(q), 50)
    want = F.dynamic(model, q[pick], 100, 8, mask)
    got = (di.cpu().numpy().view(np.uint64)[pick], dd.cpu().numpy()[pick])
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
    model.delete(ids[::2])
    _dynamic_equal(index, model, q[:16], lambda s, e: mask[:len(s)], "after the delete")


def test_refusals_change_nothing(oracle):
    x, cent, assign, index = _static(oracle, 0, n=2000, dim=32, C=40)
    q = clustered(8, 32, 30, seed=1)
    mask = np.random.default_rng(0).random(len(x)) < 0.5
    index.search_parameters = IVFSearchParameters(n_probes=2)
    before = _host(index, q, 10, mask)
    lib = _lib.lib()
    F32 = _DTYPE_CODE[np.dtype(np.float32)]
    out = np.empty((8, 10), dtype=np.uint64)
    dist = np.empty((8, 10), dtype=np.float32)
    bitmap = F.bitmap(mask)
    for args, what in (((10, 2, None), "NULL bitmap"), ((0, 2, bitmap.ctypes.data), "k = 0"),
                       ((1025, 2, bitmap.ctypes.data), "k > 1024"), ((10, 0, bitmap.ctypes.data), "n_probes = 0"),
                       ((10, 41, bitmap.ctypes.data), "n_probes > P_max")):
        k, n_probes, bm = args
        rc = lib.svsb200_ivf_search_filtered(index._h, q.ctypes.data, F32, 8, k, n_probes, bm, out.ctypes.data,
                                             dist.ctypes.data, None, None, None)
        assert rc != 0, what
    with pytest.raises(Svsb200Error):
        index.search_filtered(q.astype(np.int8), 10, mask)           # integer queries
    with pytest.raises(ValueError):
        index.search_filtered(q, 10, mask[:-1])                       # a mask of the wrong size
    dyn = DynamicIVF.assemble_from_clustering(Clustering(cent, assign), x, np.arange(len(x)), DistanceType.L2)
    dyn.search_parameters = IVFSearchParameters(n_probes=2)
    assert lib.svsb200_dynamic_ivf_search_filtered(dyn._h, q.ctypes.data, F32, 8, 10, 2, None, out.ctypes.data,
                                                   dist.ctypes.data, None, None, None) != 0
    _same(_host(index, q, 10, mask), before, "after the refusals")
    ids, dists, found = index.search_filtered(q[:0], 10, mask)
    assert ids.shape == (0, 10) and found.shape == (0,)


def test_runtime_filtered_demo_matches_the_c_abi(tmp_path):
    """cpp/ivf_filter_demo, written against the reference's runtime headers only, prints the C ABI's filtered rows for
    IVFIndex (FP32, SQI8) and DynamicIVFIndex through IDFilters; filter_stop = 0.5 on a 10 % filter pads every row with
    status OK; with filter_estimate_batch = false and filter_stop = 0.05 the rows below that hit rate are padded."""
    exe = os.path.join(ROOT, "scalablevectorsearch_b200", "cpp", "_build", "ivf_filter_demo")
    if not os.path.exists(exe):
        pytest.skip("ivf_filter_demo not built (needs the reference's runtime headers at build time)")
    n, n0, nq, dim, k, C, iters, n_probes = 4000, 4000, 40, 32, 20, 40, 4, 2
    x = clustered(n, dim, 25, seed=31)
    q = clustered(nq, dim, 25, seed=32)
    x.tofile(tmp_path / "x.f32")
    q.tofile(tmp_path / "q.f32")
    out = subprocess.run([exe, str(tmp_path / "x.f32"), str(n), str(dim), str(tmp_path / "q.f32"), str(nq), str(k), str(C),
                          str(iters), str(n_probes), str(n0)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    rows, status = {}, {}
    for line in out.stdout.splitlines():
        tag, a, b = line.split()
        if a == "status":
            status[tag] = int(b)
        else:
            rows.setdefault(tag, []).append((int(a), float(b)))
    assert all(v == 0 for v in status.values()), status

    def parsed(tag):
        r = rows[tag]
        return (np.array([a for a, _ in r], dtype=np.uint64).reshape(nq, k),
                np.array([b for _, b in r]).astype(np.float32).reshape(nq, k))

    def same(tag, want):
        gi, gd = parsed(tag)
        assert np.array_equal(gi, want[0]), tag
        assert np.array_equal(gd.view(np.uint32), want[1].view(np.uint32)), tag

    def thirty(ids):
        ids = np.asarray(ids, dtype=np.uint64)
        return ((ids * np.uint64(2654435761)) % np.uint64(2**32)) >> np.uint64(22) < 307

    clustering = Clustering.build(IVFBuildParameters(num_centroids=C, num_iterations=iters), x[:n0], DistanceType.L2)
    sp = IVFSearchParameters(n_probes=n_probes)
    idx = np.arange(n0)
    rng_mask, bit_mask = (idx >= n0 // 4) & (idx < n0 // 2), thirty(idx)
    fp32 = IVF.assemble_from_clustering(clustering, x[:n0], DistanceType.L2)
    codes, scale, bias = sq_compress(x[:n0])
    sqi8 = IVF.assemble_from_clustering(clustering, codes, DistanceType.L2, sq=(scale, bias))
    for tag, index in (("fp32", fp32), ("sqi8", sqi8)):
        index.search_parameters = sp
        same(f"{tag}_range", index.search_filtered(q, k, rng_mask))
        same(f"{tag}_bitmap", index.search_filtered(q, k, bit_mask))
    gi, gd = parsed("stop")
    assert (gi == F.PAD_ID).all() and (gd == np.inf).all()
    ids, dists, _, (probes, allowed, nrows) = fp32.search_filtered(q, k, idx % 10 == 3, with_counts=True)
    low = (allowed == 0) | (allowed.astype(np.float32) / nrows.astype(np.float32) < np.float32(0.05))
    ids[low], dists[low] = F.PAD_ID, np.inf
    same("no_estimate", (ids, dists))
    labels = np.arange(n0, dtype=np.uint64) + 1000
    dyn = DynamicIVF.assemble_from_clustering(clustering, x[:n0], labels, DistanceType.L2)
    dyn.search_parameters = sp
    dyn.delete(labels[::3])
    st, ext, _ = dyn.export()
    live = st == 1
    same("dynamic_range", dyn.search_filtered(q, k, live & (ext >= 1000 + n0 // 4) & (ext < 1000 + n0 // 2)))
    same("dynamic_bitmap", dyn.search_filtered(q, k, live & thirty(ext)))
