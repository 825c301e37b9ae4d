"""The dynamic IVF index on the GPU (csrc/dynamic_ivf.cu, the DYN form of ivf_scan_kernel) against the numpy model of
tests/dynamic_ivf_model.py: after every step of a mutation script the slot state, cluster sizes and every search (ids
and distance bits) equal the model's.  Also: the exact scan over the live rows at n_probes = C, equality with the static
IVF index, a batch that crosses the query chunks, a delete right after a device search, the refusals, and float32 rows
added to a float16 index."""
import os

import numpy as np
import pytest

import ivf_model as M
from dynamic_ivf_model import RESERVED, DynamicIVFModel
from scalablevectorsearch_b200 import (IVF, Clustering, DistanceType, DynamicIVF, IVFSearchParameters, Svsb200Error,
                                       Vamana)

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
    x = c[which] + spread * rng.standard_normal((n, dim)).astype(np.float32)
    return x.astype(dtype)


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


def _searches_equal(index, model, q, C, what, deep=True):
    """Every k of KS at n_probes 1, 8 and C; without `deep`, k = 1024 at n_probes = C (the slowest merge) is left out."""
    for n_probes in (1, 8, C):
        index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        wi, wd = model.search(q, max(KS), n_probes)   # (the top k is a prefix of the top 1024)
        for k in KS:
            if deep or k < max(KS) or n_probes < C:
                _same(index.search(q, k), (wi[:, :k], wd[:, :k]), f"{what}, k={k}, n_probes={n_probes}")


@pytest.mark.parametrize("C", [40, 520])
@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dtype,qdtype,dim", [(np.float32, np.float32, 96), (np.float32, np.float16, 40),
                                              (np.float16, np.float32, 33), (np.float16, np.float16, 96)])
def test_mutation_script_matches_the_model(oracle, C, metric, dtype, qdtype, dim):
    seed = C + metric + dim
    x = clustered(4000, dim, 30, seed=seed, dtype=dtype)
    q = clustered(24, dim, 30, seed=seed + 1, dtype=qdtype)
    cent = centroids_for(x.astype(np.float32), C, seed=7)
    rng = np.random.default_rng(seed)
    ids = rng.permutation(10**6)[:4100].astype(np.uint64) + 5   # distinct external ids in no particular order
    index = DynamicIVF.assemble_from_clustering(Clustering(cent), x[:2500], ids[:2500], DIST[metric])
    model = DynamicIVFModel.assemble(oracle, metric, cent, x[:2500], ids[:2500])

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


@pytest.mark.parametrize("metric", [0, 1, 2])
def test_all_probes_equal_the_exact_scan_over_the_live_rows(oracle, metric):
    import torch
    x = clustered(5000, 96, 40, seed=metric)
    q = clustered(64, 96, 40, seed=metric + 100)
    C = 50
    cent = centroids_for(x, C, seed=1)
    index = DynamicIVF.assemble_from_clustering(Clustering(cent), x[:3000], np.arange(3000) * 7, DIST[metric])
    index.delete(np.arange(0, 3000, 4) * 7)
    index.add(x[3000:4000], np.arange(3000, 4000) * 7, reuse_empty=True)
    index.add(x[4000:], np.arange(4000, 5000) * 7)
    index.search_parameters = IVFSearchParameters(n_probes=C)
    status, ext, _ = index.export()
    live = np.flatnonzero(status == 1)
    rows = np.empty((status.size, 96), np.float32)
    rows[:3000], rows[3000:] = x[:3000], 0
    slots_of = {int(e): s for s, e in enumerate(ext) if status[s]}
    for i in range(3000, 5000):
        rows[slots_of[i * 7]] = x[i]
    scan = Vamana.from_arrays(np.ascontiguousarray(rows[live]), np.zeros((live.size, 2), dtype=np.uint32), 0, DIST[metric])
    for k in KS:
        dq = torch.from_numpy(q).cuda()
        si = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
        sd = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
        scan.exhaustive_device(dq.data_ptr(), q.dtype, q.shape[0], k, si.data_ptr(), sd.data_ptr(),
                               stream=torch.cuda.current_stream().cuda_stream or 1)
        torch.cuda.synchronize()
        wi, wd = si.cpu().numpy().view(np.uint64), sd.cpu().numpy()
        want = np.full(wi.shape, RESERVED, dtype=np.uint64)
        ok = wi != np.uint64(RESERVED)
        want[ok] = ext[live[wi[ok].astype(np.int64)]]
        _, gi, gd = _device_search(index, q, k)
        torch.cuda.synchronize()
        got = (gi.cpu().numpy().view(np.uint64), gd.cpu().numpy())
        _same(got, (want, wd), f"k={k}")
        _same(index.search(q, k), got, f"host k={k}")


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("dtype", [np.float32, np.float16])
def test_unmutated_and_refilled_indexes_equal_the_static_ivf(oracle, metric, dtype):
    x = clustered(3000, 48, 25, seed=metric + 3, dtype=dtype)
    q = clustered(40, 48, 25, seed=metric + 4)
    C = 37
    cent = centroids_for(x.astype(np.float32), C, seed=2)
    assign = M.nearest(oracle, metric, x, cent, 1)[:, 0].astype(np.uint32)
    static = IVF.assemble_from_clustering(Clustering(cent), x, DIST[metric])
    given = DynamicIVF.assemble_from_clustering(Clustering(cent, assign), x, np.arange(3000), DIST[metric])
    empty = DynamicIVF.assemble_from_clustering(Clustering(cent), x[:0], np.arange(0), DIST[metric])
    assert empty.size == 0 and empty.num_slots == 0
    for index in (given, empty):
        index.search_parameters = IVFSearchParameters(n_probes=3)
        ids, d = index.search(q, 10)
        assert (ids == RESERVED).all() == (index is empty)
    assert list(empty.add(x, np.arange(3000))) == list(range(3000))
    assert np.array_equal(empty.cluster_sizes, static.cluster_sizes)
    for n_probes in (1, 5, C):
        for index in (static, given, empty):
            index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        for k in (1, 10, 100, 1024):
            want = static.search(q, k)
            _same(given.search(q, k), want, f"assembled, k={k}, n_probes={n_probes}")
            _same(empty.search(q, k), want, f"filled by one add, k={k}, n_probes={n_probes}")


def test_a_large_batch_crosses_the_query_chunks(oracle):
    x = clustered(20000, 96, 60, seed=5)
    q = clustered(10000, 96, 60, seed=6)
    cent = centroids_for(x, 128, seed=2)
    index = DynamicIVF.assemble_from_clustering(Clustering(cent), x[:15000], np.arange(15000), DistanceType.L2)
    model = DynamicIVFModel.assemble(oracle, 0, cent, x[:15000], np.arange(15000))
    index.delete(np.arange(0, 15000, 5))
    model.delete(np.arange(0, 15000, 5))
    index.add(x[15000:], np.arange(15000, 20000), reuse_empty=True)
    model.add(x[15000:], np.arange(15000, 20000), reuse_empty=True)
    index.search_parameters = IVFSearchParameters(n_probes=64)
    ids, dists = index.search(q, 100)
    for lo in (0, 3333, 6667, 9900):   # the same queries in small batches
        _same((ids[lo:lo + 100], dists[lo:lo + 100]), index.search(q[lo:lo + 100], 100))
    pick = np.arange(0, 10000, 250)
    _same((ids[pick], dists[pick]), model.search(q[pick], 100, 64))


def test_a_delete_may_follow_a_device_search_without_a_synchronisation(oracle):
    import torch
    x = clustered(8000, 64, 30, seed=9)
    q = clustered(2000, 64, 30, seed=10)
    cent = centroids_for(x, 64, seed=3)
    index = DynamicIVF.assemble_from_clustering(Clustering(cent), x, np.arange(8000) + 1, DistanceType.L2)
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


def test_refusals_leave_nothing_changed():
    x = clustered(600, 16, 8, seed=1)
    q = x[:5]
    cent = centroids_for(x, 8, seed=1)
    index = DynamicIVF.assemble_from_clustering(Clustering(cent), x[:500], np.arange(500), DistanceType.L2)
    index.delete([3, 4])
    index.search_parameters = IVFSearchParameters(n_probes=3)
    before, state = index.search(q, 10), index.export()

    def unchanged():
        _same(index.search(q, 10), before)
        for a, b in zip(index.export(), state):
            assert np.array_equal(a, b)

    p = x[500:502]
    for ids, match in (([600, 600], "repeat"), ([600, 7], "already exists"), ([600, RESERVED], "reserved")):
        with pytest.raises(Svsb200Error, match=match):
            index.add(p, np.array(ids, dtype=np.uint64))
        unchanged()
    with pytest.raises(Svsb200Error, match="dtype"):
        index.add(p.astype(np.float16), [600, 601])
    unchanged()
    for ids in ([3], [9, 9], [9, 12345]):
        with pytest.raises(Svsb200Error, match="does not exist"):
            index.delete(ids)
        unchanged()
    for k in (0, 1025):
        with pytest.raises(Svsb200Error, match="k must be"):
            index.search(q, k)
    for n_probes in (0, 9):
        index.search_parameters = IVFSearchParameters(n_probes=n_probes)
        with pytest.raises(Svsb200Error, match="n_probes"):
            index.search(q, 10)
    index.search_parameters = IVFSearchParameters(n_probes=3)
    with pytest.raises(Svsb200Error, match="float32 or float16"):
        DynamicIVF.assemble_from_clustering(Clustering(cent), x.astype(np.int8), np.arange(600), DistanceType.L2)
    with pytest.raises(Svsb200Error, match="repeat"):
        DynamicIVF.assemble_from_clustering(Clustering(cent), x[:2], [1, 1], DistanceType.L2)
    unchanged()


def test_float32_points_are_rounded_into_a_float16_index():
    x = clustered(1000, 24, 10, seed=11)
    cent = centroids_for(x, 12, seed=4)
    a = DynamicIVF.assemble_from_clustering(Clustering(cent), x[:500].astype(np.float16), np.arange(500), DistanceType.L2)
    b = DynamicIVF.assemble_from_clustering(Clustering(cent), x[:500].astype(np.float16), np.arange(500), DistanceType.L2)
    a.add(x[500:], np.arange(500, 1000))                       # float32, rounded to nearest even
    b.add(x[500:].astype(np.float16), np.arange(500, 1000))
    for index in (a, b):
        index.search_parameters = IVFSearchParameters(n_probes=12)
    _same(a.search(x[::7], 50), b.search(x[::7], 50))
    for u, v in zip(a.export(), b.export()):
        assert np.array_equal(u, v)


def test_runtime_dynamic_ivf_index_demo_matches_the_c_abi(tmp_path):
    """cpp/dynamic_ivf_demo, written against the reference's runtime header only (svs::runtime::v0::DynamicIVFIndex) and
    linked with libsvsb200_runtime.so, prints the same results as Clustering.build + DynamicIVF with the same parameters
    and mutations, for an index built with rows and for one built empty and filled by its first add; plus the refusals:
    LVQ storage NOT_IMPLEMENTED (3), search and compact before initialisation NOT_INITIALIZED (4, labels -1), k = 0
    INVALID_ARGUMENT (2)."""
    import subprocess
    from scalablevectorsearch_b200 import IVFBuildParameters
    exe = os.path.join(ROOT, "scalablevectorsearch_b200", "cpp", "_build", "dynamic_ivf_demo")
    if not os.path.exists(exe):
        pytest.skip("dynamic_ivf_demo not built (needs the reference's runtime headers at build time)")
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
    assert rows["storage_lvq8"] == [["3"]] and rows["k0"] == [["2"]] and rows["empty_compact"] == [["4"]]
    assert rows["empty_search"] == [["4", str(2**64 - 1)]]

    def parsed(tag):
        return (np.array([int(r[0]) for r in rows[tag]], dtype=np.uint64).reshape(nq, k),
                np.array([float(r[1]) for r in rows[tag]]).astype(np.float32).reshape(nq, k))

    labels = np.arange(n, dtype=np.uint64) + 1000
    clustering = Clustering.build(IVFBuildParameters(num_centroids=C, num_iterations=iters), x[:n0], DistanceType.L2)
    index = DynamicIVF.assemble_from_clustering(clustering, x[:n0], labels[:n0], DistanceType.L2)
    index.search_parameters = IVFSearchParameters(n_probes=n_probes)
    _same(parsed("initial"), index.search(q, k), "built empty, filled by one add")
    index.delete(labels[:n0:3])
    index.add(x[n0:], labels[n0:], reuse_empty=True)
    sevens = index.all_ids()[index.all_ids() % 7 == 0]
    index.delete(sevens)
    assert rows["removed"] == [[str(len(sevens))]]
    index.compact()
    assert rows["has_id"] == [["0", str(int(index.has_id(1001)))]]
    _same(parsed("result"), index.search(q, k), "mutated")
