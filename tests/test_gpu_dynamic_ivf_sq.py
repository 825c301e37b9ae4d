"""The dynamic IVF index over SQ codes on the GPU (svsb200_dynamic_ivf_create_sq; float32 adds encoded on the device; the
DYN forms of the tensor-core L2 leaf and of the SQ float-tree MIP / cosine leaves) against the numpy model of
tests/dynamic_ivf_sq_model.py: after every step of a mutation script the slot state, cluster sizes and every search (ids
and distance bits) equal the model's.  Also: the exact scan over the live codes at n_probes = C, equality with the
static SQ IVF index, adds that clamp, wide rows, a batch that crosses the query chunks, a delete right after a device
search, the refusals, the device memory against a float32 index, and the runtime classes with SQI8 storage."""
import os

import numpy as np
import pytest

import ivf_model as M
import ivf_sq_model as S
from dynamic_ivf_model import RESERVED
from dynamic_ivf_sq_model import DynamicIVFSQModel
from scalablevectorsearch_b200 import (IVF, Clustering, DistanceType, DynamicIVF, IVFSearchParameters, Svsb200Error,
                                       Vamana, sq_compress)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIST = {0: DistanceType.L2, 1: DistanceType.MIP, 2: DistanceType.Cosine}
KS = (1, 10, 100, 1024)


def clustered(n, dim, centres, seed, dtype=np.float32, spread=0.3):
    """Rows around `centres` random centres, cluster sizes skewed (some clusters far larger than the ring's 64 rows)."""
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
    gi, gd = got
    wi, wd = want
    assert np.array_equal(gi, wi), f"{what}: ids differ in {np.flatnonzero((gi != wi).any(1))[:10]} queries"
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32)), f"{what}: distance bits differ"


def _state_equal(index, model, what):
    status, ext, cluster = index.export()
    ws, we, wc = model.export()
    assert np.array_equal(status, ws), what
    assert np.array_equal(ext, we), what
    assert np.array_equal(cluster, wc), what
    assert np.array_equal(index.all_ids(), model.all_ids()), what
    assert np.array_equal(index.cluster_sizes, model.cluster_sizes()), what
    assert index.size == model.size and index.num_slots == len(ws), what


def _searches_equal(index, model, q, C, what, deep=True, ks=KS):
    """Every k at n_probes 1, 8 and C; without `deep`, the largest k at n_probes = C is left out."""
    for n_probes in sorted({1, min(8, C), C}):
        index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        wi, wd = model.search(q, max(ks), n_probes)   # (the top k is a prefix of the top max(ks))
        for k in ks:
            if deep or k < max(ks) or n_probes < C:
                _same(index.search(q, k), (wi[:, :k], wd[:, :k]), f"{what}, k={k}, n_probes={n_probes}")


def _assembled(oracle, x, n0, ids, C, metric, dtype, seed=7):
    """The first n0 rows compressed (the scale and bias of all of x) and assembled with nearest-centroid assignments."""
    codes, scale, bias = sq_compress(x, dtype)
    cent = centroids_for(x, C, seed)
    assign = M.nearest(oracle, metric, x[:n0], cent, 1)[:, 0].astype(np.uint32)
    index = DynamicIVF.assemble_from_clustering(Clustering(cent, assign), codes[:n0], ids[:n0], DIST[metric],
                                                sq=(scale, bias))
    model = DynamicIVFSQModel.assemble(oracle, metric, cent, codes[:n0], ids[:n0], scale, bias, assign)
    return index, model, codes, scale, bias, cent


@pytest.mark.parametrize("C", [40, 520])
@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dtype,qdtype,dim", [(np.int8, np.float32, 96), (np.uint8, np.float16, 128),
                                              (np.int8, np.float16, 45), (np.uint8, np.float32, 96)])
def test_mutation_script_matches_the_model(oracle, C, metric, dtype, qdtype, dim):
    seed = C + metric + dim
    x = clustered(4000, dim, 30, seed=seed)
    q = clustered(24, dim, 30, seed=seed + 1, dtype=qdtype)
    rng = np.random.default_rng(seed)
    ids = rng.permutation(10**6)[:4100].astype(np.uint64) + 5   # distinct external ids in no particular order
    index, model, _, _, _, _ = _assembled(oracle, x, 2500, ids, C, metric, dtype)

    def check(what, deep=False):
        _state_equal(index, model, what)
        _searches_equal(index, model, q, C, what, deep)

    check("assembled", deep=True)
    for lo, hi, what in ((2500, 2505, "small add"), (2505, 3700, "add that relocates clusters")):
        before = index.device_bytes
        got = index.add(x[lo:hi], ids[lo:hi])
        assert list(got) == model.add(x[lo:hi], ids[lo:hi])
        if hi == 3700 and C == 40:
            assert index.device_bytes > before   # clusters overflowed and the pool grew
        check(what, deep=hi == 3700)
    gone = rng.choice(model.all_ids(), 1400, replace=False)
    index.delete(gone)
    model.delete(gone)
    check("delete")
    got = index.add(x[3700:3900], ids[3700:3900], reuse_empty=True)
    assert list(got) == model.add(x[3700:3900], ids[3700:3900], reuse_empty=True)
    check("add with reuse_empty", deep=True)
    index.compact()
    model.compact()
    check("compact", deep=True)
    got = index.add(x[3900:4000], ids[3900:4000])
    assert list(got) == model.add(x[3900:4000], ids[3900:4000])
    check("add after compact")
    status, ext, cluster = index.export()
    biggest = np.bincount(cluster[status == 1], minlength=C).argmax()
    whole = ext[(status == 1) & (cluster == biggest)]
    index.delete(whole)
    model.delete(whole)
    assert index.cluster_sizes[biggest] == 0
    check("delete a whole cluster")
    everything = index.all_ids()
    index.delete(everything)
    model.delete(everything)
    assert index.size == 0
    check("delete everything")
    got = index.add(x[:50], ids[4000:4050], reuse_empty=bool(metric % 2))
    assert list(got) == model.add(x[:50], ids[4000:4050], reuse_empty=bool(metric % 2))
    check("add again")


def _device_search(index, q, k, stream=None):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
    d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
    s = stream or torch.cuda.current_stream()
    index.search_device(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), d.data_ptr(), stream=s.cuda_stream or 1)
    return dq, ids, d


def _scan(scan, q, k):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
    d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
    scan.exhaustive_device(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), d.data_ptr(),
                           stream=torch.cuda.current_stream().cuda_stream or 1)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint64), d.cpu().numpy()


def _scan_over_live(index, model, metric, q, k):
    """svsb200_exhaustive_device on an SQ index over the Valid slots' codes in slot order, ids mapped through the slots."""
    status, ext, _ = index.export()
    live = np.flatnonzero(status == 1)
    codes = np.ascontiguousarray(model.live_rows())
    scan = Vamana.from_arrays(codes, np.zeros((live.size, 2), dtype=np.uint32), 0, DIST[metric],
                              sq=(model.scale, model.bias))
    wi, wd = _scan(scan, q, k)
    want = np.full(wi.shape, RESERVED, dtype=np.uint64)
    ok = wi != np.uint64(RESERVED)
    want[ok] = ext[live[wi[ok].astype(np.int64)]]
    return want, wd


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
def test_all_probes_equal_the_exact_scan_over_the_live_codes(oracle, metric, dtype):
    import torch
    x = clustered(5000, 96, 40, seed=metric)
    q = clustered(64, 96, 40, seed=metric + 100)
    C = 50
    ids = np.arange(5000, dtype=np.uint64) * 7
    index, model, _, _, _, _ = _assembled(oracle, x, 3000, ids, C, metric, dtype, seed=1)
    for m in (index, model):
        m.delete(ids[:3000:4])
        m.add(x[3000:4000], ids[3000:4000], reuse_empty=True)
        m.add(x[4000:], ids[4000:])
    index.search_parameters = IVFSearchParameters(n_probes=C)
    for k in KS:
        for qq in (q, q.astype(np.float16)):
            want = _scan_over_live(index, model, metric, qq, k)
            _, gi, gd = _device_search(index, qq, k)
            torch.cuda.synchronize()
            got = (gi.cpu().numpy().view(np.uint64), gd.cpu().numpy())
            _same(got, want, f"k={k}, {qq.dtype} queries")
            _same(index.search(qq, k), got, f"host k={k}")


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
def test_equalities_with_the_static_sq_ivf(oracle, metric, dtype):
    x = clustered(3000, 48, 25, seed=metric + 3)
    q = clustered(40, 48, 25, seed=metric + 4)
    C, n0 = 37, 1800
    cent = centroids_for(x, C, seed=2)
    codes, scale, bias = sq_compress(x, dtype)
    near = M.nearest(oracle, metric, x, cent, 1)[:, 0].astype(np.uint32)
    given = ((near + np.arange(3000) % 3) % C).astype(np.uint32)   # assignments other than the nearest
    sq = (scale, bias)
    # 2. an unmutated index with ids 0 .. n-1 equals the static SQ index over the same codes and clustering
    static_given = IVF.assemble_from_clustering(Clustering(cent, given), codes, DIST[metric], sq=sq)
    unmutated = DynamicIVF.assemble_from_clustering(Clustering(cent, given), codes, np.arange(3000), DIST[metric], sq=sq)
    # 3. the first n0 codes assembled, the remaining rows added as float32
    mixed = np.concatenate([given[:n0], near[n0:]])
    static_mixed = IVF.assemble_from_clustering(Clustering(cent, mixed), codes, DIST[metric], sq=sq)
    prefix = DynamicIVF.assemble_from_clustering(Clustering(cent, given[:n0]), codes[:n0], np.arange(n0), DIST[metric],
                                                 sq=sq)
    assert list(prefix.add(x[n0:], np.arange(n0, 3000))) == list(range(n0, 3000))
    # 4. an empty index filled by one add equals the static SQ index over encode(x) with the nearest centroids
    static_near = IVF.assemble_from_clustering(Clustering(cent, near), S.encode(x, dtype, scale, bias), DIST[metric],
                                               sq=sq)
    empty = DynamicIVF.assemble_from_clustering(Clustering(cent), codes[:0], np.arange(0), DIST[metric], sq=sq)
    assert empty.size == 0 and empty.num_slots == 0
    empty.search_parameters = IVFSearchParameters(n_probes=3)
    assert (empty.search(q, 10)[0] == RESERVED).all()
    assert list(empty.add(x, np.arange(3000))) == list(range(3000))
    assert np.array_equal(empty.cluster_sizes, static_near.cluster_sizes)
    assert np.array_equal(prefix.cluster_sizes, static_mixed.cluster_sizes)
    pairs = ((unmutated, static_given, "unmutated"), (prefix, static_mixed, "prefix + add"),
             (empty, static_near, "filled by one add"))
    for n_probes in (1, 5, C):
        for index in (static_given, static_mixed, static_near, unmutated, prefix, empty):
            index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        for k in KS:
            for dyn, static, what in pairs:
                _same(dyn.search(q, k), static.search(q, k), f"{what}, k={k}, n_probes={n_probes}")


@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
def test_adds_beyond_the_compressed_range_clamp(oracle, dtype):
    x = clustered(2000, 64, 20, seed=12)
    ids = np.arange(2400, dtype=np.uint64)
    index, model, codes, scale, bias, cent = _assembled(oracle, x, 2000, ids, 24, 0, dtype)
    rng = np.random.default_rng(3)
    far = (clustered(400, 64, 20, seed=13) * 4 + rng.standard_normal((400, 64)).astype(np.float32) * 20)
    lo, hi = S.RANGE[np.dtype(dtype)]
    enc = S.encode(far, dtype, scale, bias)
    assert (enc == lo).any() and (enc == hi).any()
    index.add(far, ids[2000:])
    model.add(far, ids[2000:])
    q = clustered(30, 64, 20, seed=14) * 3
    _state_equal(index, model, "clamped add")
    _searches_equal(index, model, q, 24, "clamped add", ks=(1, 10, 100))
    index.search_parameters = IVFSearchParameters(n_probes=24)
    _same(index.search(q, 100), _scan_over_live(index, model, 0, q, 100), "clamped add, exact scan")


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dim", [2048, 4096])
def test_wide_rows(oracle, metric, dim):
    # rows of 2048 and 4096 codes stage 16- and 8-row tiles, with k = 1024
    x = clustered(500, dim, 6, seed=dim + metric)
    q = clustered(12, dim, 6, seed=dim + metric + 1)
    ids = np.arange(500, dtype=np.uint64) + 3
    index, model, _, _, _, _ = _assembled(oracle, x, 350, ids, 12, metric, np.int8)
    for m in (index, model):
        m.delete(ids[:350:5])
        m.add(x[350:], ids[350:], reuse_empty=True)
    index.search_parameters = IVFSearchParameters(n_probes=12)
    _same(index.search(q, 1024), _scan_over_live(index, model, metric, q, 1024), "n_probes = C")
    index.search_parameters = IVFSearchParameters(n_probes=3)
    _same(index.search(q, 1024), model.search(q, 1024, 3), "n_probes = 3")


def test_a_large_batch_crosses_the_query_chunks(oracle):
    x = clustered(20000, 96, 60, seed=5)
    q = clustered(10000, 96, 60, seed=6)
    ids = np.arange(20000, dtype=np.uint64)
    index, model, _, _, _, _ = _assembled(oracle, x, 15000, ids, 128, 0, np.int8, seed=2)
    for m in (index, model):
        m.delete(np.arange(0, 15000, 5))
        m.add(x[15000:], ids[15000:], reuse_empty=True)
    index.search_parameters = IVFSearchParameters(n_probes=64)
    got_ids, got_d = index.search(q, 100)
    for lo in (0, 3333, 6667, 9900):   # the same queries in small batches
        _same((got_ids[lo:lo + 100], got_d[lo:lo + 100]), index.search(q[lo:lo + 100], 100))
    pick = np.arange(0, 10000, 250)
    _same((got_ids[pick], got_d[pick]), model.search(q[pick], 100, 64))


def test_a_delete_may_follow_a_device_search_without_a_synchronisation(oracle):
    import torch
    x = clustered(8000, 64, 30, seed=9)
    q = clustered(2000, 64, 30, seed=10)
    index, _, _, _, _, _ = _assembled(oracle, x, 8000, np.arange(8000, dtype=np.uint64) + 1, 64, 0, np.int8, seed=3)
    index.search_parameters = IVFSearchParameters(n_probes=16)
    want = index.search(q, 100)
    gone = np.unique(want[0][:, 0])[:500]
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        keep = _device_search(index, q, 100, stream)
        index.delete(gone)            # at once: the delete waits for the search
    stream.synchronize()
    _, gi, gd = keep
    _same((gi.cpu().numpy().view(np.uint64), gd.cpu().numpy()), want)
    assert not np.isin(index.search(q, 100)[0], gone).any()


def test_refusals_leave_nothing_changed(oracle):
    x = clustered(600, 16, 8, seed=1)
    q = x[:5]
    ids = np.arange(600, dtype=np.uint64)
    index, _, codes, scale, bias, cent = _assembled(oracle, x, 500, ids, 8, 0, np.int8, seed=1)
    index.delete([3, 4])
    index.search_parameters = IVFSearchParameters(n_probes=3)
    before, state = index.search(q, 10), index.export()

    def unchanged():
        _same(index.search(q, 10), before)
        for a, b in zip(index.export(), state):
            assert np.array_equal(a, b)

    p = x[500:502].copy()
    for pts, match in ((p.astype(np.float16), "float32"), (codes[500:502], "float32")):
        with pytest.raises(Svsb200Error, match=match):
            index.add(pts, [600, 601])
        unchanged()
    for bad in (np.nan, np.inf, -np.inf):
        p2 = p.copy()
        p2[1, 7] = bad
        with pytest.raises(Svsb200Error, match="NaN or an infinity"):
            index.add(p2, [600, 601])
        unchanged()
    for new, match in (([600, 600], "repeat"), ([600, 7], "already exists"), ([600, RESERVED], "reserved")):
        with pytest.raises(Svsb200Error, match=match):
            index.add(p, np.array(new, dtype=np.uint64))
        unchanged()
    for gone in ([3], [9, 9], [9, 12345]):
        with pytest.raises(Svsb200Error, match="does not exist"):
            index.delete(gone)
        unchanged()
    with pytest.raises(Svsb200Error, match="need assignments"):
        DynamicIVF.assemble_from_clustering(Clustering(cent), codes, ids, DistanceType.L2, sq=(scale, bias))
    assign = np.zeros(600, dtype=np.uint32)
    for bad in ((0.0, bias), (-1.0, bias), (float("nan"), bias), (scale, float("inf"))):
        with pytest.raises(Svsb200Error, match="scale"):
            DynamicIVF.assemble_from_clustering(Clustering(cent, assign), codes, ids, DistanceType.L2, sq=bad)
    with pytest.raises(TypeError, match="codes"):
        DynamicIVF.assemble_from_clustering(Clustering(cent, assign), x, ids, DistanceType.L2, sq=(scale, bias))
    with pytest.raises(Svsb200Error, match="repeat"):
        DynamicIVF.assemble_from_clustering(Clustering(cent, assign[:2]), codes[:2], [1, 1], DistanceType.L2,
                                            sq=(scale, bias))
    unchanged()


def test_device_bytes_below_the_float32_index(oracle):
    x = clustered(20000, 128, 40, seed=15)
    ids = np.arange(20000, dtype=np.uint64)
    cent = centroids_for(x, 64, seed=4)
    assign = M.nearest(oracle, 0, x[:15000], cent, 1)[:, 0].astype(np.uint32)
    codes, scale, bias = sq_compress(x)
    f32 = DynamicIVF.assemble_from_clustering(Clustering(cent, assign), x[:15000], ids[:15000], DistanceType.L2)
    sq = DynamicIVF.assemble_from_clustering(Clustering(cent, assign), codes[:15000], ids[:15000], DistanceType.L2,
                                             sq=(scale, bias))
    assert sq.device_bytes < f32.device_bytes
    for index in (f32, sq):
        index.add(x[15000:], ids[15000:])
    assert sq.device_bytes < f32.device_bytes / 2


def test_runtime_ivf_sq_demo_matches_the_c_abi(tmp_path):
    """cpp/ivf_sq_demo, written against the reference's runtime headers only (IVFIndex and DynamicIVFIndex with
    StorageKind::SQI8), prints the same results as Clustering.build + sq_compress + assemble_from_clustering(..., sq=)
    with the same parameters and mutations; check_storage_kind(SQI8) is 0 for both classes, and constant rows, which
    have no SQ scale, are an error status (RUNTIME_ERROR, 5) with no index."""
    import subprocess
    from scalablevectorsearch_b200 import IVFBuildParameters
    exe = os.path.join(ROOT, "scalablevectorsearch_b200", "cpp", "_build", "ivf_sq_demo")
    if not os.path.exists(exe):
        pytest.skip("ivf_sq_demo not built (needs the reference's runtime headers at build time)")
    n, n0, nq, dim, k, C, iters, n_probes = 6000, 4500, 50, 48, 20, 40, 4, 5
    x = clustered(n, dim, 25, seed=21)
    q = clustered(nq, dim, 25, seed=22)
    x.tofile(tmp_path / "x.f32")
    q.tofile(tmp_path / "q.f32")
    out = subprocess.run([exe, str(tmp_path / "x.f32"), str(n), str(dim), str(tmp_path / "q.f32"), str(nq), str(k), str(C),
                          str(iters), str(n_probes), str(n0)], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    rows = {}
    for line in out.stdout.splitlines():
        tag, *rest = line.split()
        rows.setdefault(tag, []).append(rest)
    assert rows["storage_sqi8"] == [["0", "0"]]
    assert rows["constant"] == [["5", "1"]]

    def parsed(tag):
        return (np.array([int(r[0]) for r in rows[tag]], dtype=np.uint64).reshape(nq, k),
                np.array([float(r[1]) for r in rows[tag]]).astype(np.float32).reshape(nq, k))

    labels = np.arange(n, dtype=np.uint64) + 1000
    clustering = Clustering.build(IVFBuildParameters(num_centroids=C, num_iterations=iters), x[:n0], DistanceType.L2)
    codes, scale, bias = sq_compress(x[:n0])
    static = IVF.assemble_from_clustering(clustering, codes, DistanceType.L2, sq=(scale, bias))
    static.search_parameters = IVFSearchParameters(n_probes=n_probes)
    _same(parsed("ivf"), static.search(q, k), "IVFIndex")
    index = DynamicIVF.assemble_from_clustering(clustering, codes, labels[:n0], DistanceType.L2, sq=(scale, bias))
    index.search_parameters = IVFSearchParameters(n_probes=n_probes)
    _same(parsed("initial"), index.search(q, k), "built empty, filled by one add")
    index.delete(labels[:n0:3])
    index.add(x[n0:], labels[n0:], reuse_empty=True)
    sevens = index.all_ids()[index.all_ids() % 7 == 0]
    index.delete(sevens)
    assert rows["removed"] == [[str(len(sevens))]]
    index.compact()
    _same(parsed("result"), index.search(q, k), "mutated")
