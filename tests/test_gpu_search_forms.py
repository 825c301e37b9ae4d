"""The host form (host buffers, blocking, a pooled scratch) and the device form (device buffers, enqueued on the caller's
stream) of every search outside the Vamana graph search agree bit for bit: ids, distance bits, the per-query counts of
the filtered IVF searches and the allowed-row count of the filtered flat search.  Also: the host calls of one index
give their scratch sets back to the pool on every return path, and a delete issued right after an unfiltered device
search of a dynamic flat index waits for it."""
import ctypes as C

import numpy as np
import pytest

from conftest import bits

pytestmark = pytest.mark.gpu

NQ = 300   # more than two 128-query tiles: the Flat handle's deep lists (k > 25) run on the GEMM


def _rows(n, dim, dtype, seed):
    rng = np.random.default_rng(seed)
    if dtype in (np.int8, np.uint8):
        lo, hi = (-128, 128) if dtype == np.int8 else (0, 256)
        return rng.integers(lo, hi, (n, dim)).astype(dtype)
    return rng.standard_normal((n, dim)).astype(dtype)


def _to_device(*arrays):
    """The arrays on the GPU, their copies finished before any other stream reads them."""
    import torch
    out = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    torch.cuda.synchronize()
    return out


def _outputs(nq, k, counts=0):
    import torch
    ids = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    dists = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    cnt = torch.empty((max(counts, 1), nq), dtype=torch.int32, device="cuda")
    return ids, dists, cnt


def _host_view(ids, dists):
    return ids.cpu().numpy().view(np.uint64), dists.cpu().numpy()


def _same(host, device, tag):
    hi, hd = host
    di, dd = device
    assert np.array_equal(hi, di), f"{tag}: ids differ in {np.count_nonzero(hi != di)} entries"
    assert np.array_equal(bits(hd), bits(dd)), f"{tag}: distance bits differ"


def _plain(index, q, k, tag):
    """index.search (host form) == index.search_device on a side stream (device form)."""
    import torch
    (dq,) = _to_device(q)
    ids, dists, _ = _outputs(q.shape[0], k)
    s = torch.cuda.Stream()
    index.search_device(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), dists.data_ptr(), stream=s.cuda_stream)
    torch.cuda.synchronize()
    _same(index.search(q, k), _host_view(ids, dists), tag)


@pytest.mark.parametrize("dtype,k", [(np.float32, 10), (np.int8, 50)])
def test_flat(dtype, k):
    from scalablevectorsearch_b200 import DistanceType, Flat
    x = _rows(3000, 64, dtype, 1)
    _plain(Flat(x, DistanceType.L2), _rows(NQ, 64, dtype, 2), k, f"Flat {np.dtype(dtype).name} k={k}")


def test_dynamic_flat_after_deletes():
    from scalablevectorsearch_b200 import DistanceType, DynamicFlat
    n = 3000
    ids = np.arange(n, dtype=np.uint64) * 7 + 3
    dyn = DynamicFlat.build(_rows(n, 48, np.float32, 3), ids, DistanceType.L2)
    dyn.delete(ids[np.random.default_rng(4).choice(n, 700, replace=False)])
    _plain(dyn, _rows(NQ, 48, np.float32, 5), 10, "DynamicFlat")


@pytest.mark.parametrize("frac", [0.5, 0.005])   # the dense and the sparse route
@pytest.mark.parametrize("dynamic", [False, True])
def test_flat_filtered(frac, dynamic):
    import torch
    from scalablevectorsearch_b200 import DistanceType, DynamicFlat, Flat, _lib
    from scalablevectorsearch_b200._lib import _bitmap
    from scalablevectorsearch_b200.flat import filter_route
    from scalablevectorsearch_b200.vamana import _DTYPE_CODE
    n, k = 6000, 10
    x, q = _rows(n, 32, np.float32, 6), _rows(NQ, 32, np.float32, 7)
    rng = np.random.default_rng(8)
    if dynamic:
        index = DynamicFlat.build(x, np.arange(n, dtype=np.uint64), DistanceType.L2)
        index.delete(rng.choice(n, 500, replace=False).astype(np.uint64))
        fn, slots = index._lib.svsb200_dynamic_flat_search_filtered_device, index.num_slots
    else:
        index = Flat(x, DistanceType.L2)
        fn, slots = index._lib.svsb200_flat_index_search_filtered_device, index.size
    mask = rng.random(slots) < frac
    hi, hd, _, allowed = index.search_filtered(q, k, mask, with_counts=True)
    assert filter_route(n, allowed) == ("dense" if frac > 0.1 else "sparse")
    dq, bm = _to_device(q, _bitmap(mask, slots).view(np.int32))
    ids, dists, _ = _outputs(NQ, k)
    s = torch.cuda.Stream()
    d_allowed, fallback = C.c_size_t(), C.c_uint32()
    from scalablevectorsearch_b200 import _lib
    _lib.check(fn(index._h, dq.data_ptr(), _DTYPE_CODE[q.dtype], NQ, k, bm.data_ptr(), ids.data_ptr(), dists.data_ptr(),
                  s.cuda_stream, C.byref(d_allowed), C.byref(fallback)))
    torch.cuda.synchronize()
    assert d_allowed.value == allowed
    _same((hi, hd), _host_view(ids, dists), f"filtered {'DynamicFlat' if dynamic else 'Flat'} frac={frac}")


def _ivf_data(sq=False, seed=10):
    from scalablevectorsearch_b200 import Clustering, sq_compress
    n, dim, C_ = 4000, 32, 40
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((C_, dim)).astype(np.float32) * 3
    x = (centres[rng.integers(0, C_, n)] + 0.5 * rng.standard_normal((n, dim))).astype(np.float32)
    cent = x[rng.choice(n, C_, replace=False)]
    assign = np.argmin(((x[:, None, :] - cent[None]) ** 2).sum(-1), axis=1).astype(np.uint32)
    q = _rows(NQ, dim, np.float32, seed + 1) * 3
    if sq:
        codes, scale, bias = sq_compress(x)
        return Clustering(cent, assign), codes, (scale, bias), q
    return Clustering(cent, assign), x, None, q


@pytest.mark.parametrize("sq", [False, True])
def test_ivf(sq):
    from scalablevectorsearch_b200 import IVF
    clustering, rows, sqp, q = _ivf_data(sq)
    index = IVF.assemble_from_clustering(clustering, rows, sq=sqp)
    index.search_parameters.n_probes = 5
    _plain(index, q, 10, f"IVF sq={sq}")


def _ivf_filtered(index, q, k, mask, tag):
    import torch
    from scalablevectorsearch_b200._lib import _bitmap
    hi, hd, _, (hp, ha, hr) = index.search_filtered(q, k, mask, with_counts=True)
    dq, bm = _to_device(q, _bitmap(mask, mask.shape[0]).view(np.int32))
    ids, dists, cnt = _outputs(q.shape[0], k, counts=3)
    s = torch.cuda.Stream()
    index.search_filtered_device(dq.data_ptr(), q.dtype, q.shape[0], k, bm.data_ptr(), ids.data_ptr(), dists.data_ptr(),
                                 cnt[0].data_ptr(), cnt[1].data_ptr(), cnt[2].data_ptr(), stream=s.cuda_stream)
    torch.cuda.synchronize()
    _same((hi, hd), _host_view(ids, dists), tag)
    counts = cnt.cpu().numpy().view(np.uint32)
    for name, h, d in zip(("probes", "allowed", "rows"), (hp, ha, hr), counts):
        assert np.array_equal(h, d), f"{tag}: per-query {name} differ"


def test_ivf_filtered():
    from scalablevectorsearch_b200 import IVF
    clustering, rows, _, q = _ivf_data(seed=20)
    index = IVF.assemble_from_clustering(clustering, rows)
    index.search_parameters.n_probes = 2
    mask = np.random.default_rng(21).random(index.size) < 0.05   # sparse enough that queries grow their probes
    _ivf_filtered(index, q, 10, mask, "filtered IVF")


def test_dynamic_ivf_and_filtered():
    from scalablevectorsearch_b200 import DynamicIVF
    clustering, rows, _, q = _ivf_data(seed=30)
    n = rows.shape[0]
    ids = np.arange(n, dtype=np.uint64) * 5 + 1
    index = DynamicIVF.assemble_from_clustering(clustering, rows, ids)
    index.search_parameters.n_probes = 3
    rng = np.random.default_rng(31)
    index.delete(ids[rng.choice(n, 900, replace=False)])
    _plain(index, q, 10, "DynamicIVF")
    _ivf_filtered(index, q, 10, rng.random(index.num_slots) < 0.05, "filtered DynamicIVF")


def test_host_calls_give_their_scratch_back(dataset):
    """Every kind of host call on one index, and calls that fail before and after checking out a scratch: none leaves a
    scratch set checked out, so the pool's size stays where the first call left it.  Each kind runs alone more times
    than the pool holds sets, so a single call kind that kept its set would have to grow the pool."""
    from scalablevectorsearch_b200 import DistanceType, SearchBufferConfig, Svsb200Error, Vamana
    index = Vamana.from_arrays(dataset.data, dataset.graph, dataset.entry_point, DistanceType.L2)
    index.search_parameters.buffer_config = SearchBufferConfig(22, 23)
    q = dataset.queries[:100]
    mask = np.random.default_rng(40).random(dataset.data.shape[0]) < 0.3

    def refused(call):
        with pytest.raises(Svsb200Error):
            call()

    kinds = {
        "search": lambda: index.search(q, 10),
        "search_filtered": lambda: index.search_filtered(q, 10, mask),
        "range_search": lambda: index.range_search(q[:10], 1e9),
        "flat_search": lambda: index.flat_search(q, 10),
        "refused before checkout": lambda: refused(lambda: index.search_filtered(q, 0, mask)),
        "filtered, refused by the body": lambda: refused(lambda: index.search_filtered(q.astype(np.int8), 10, mask)),
        "range, refused by the body": lambda: refused(lambda: index.range_search(q.astype(np.int8), 1.0)),
        "flat, refused by the body": lambda: refused(lambda: index.flat_search(q.astype(np.int8), 10)),
    }
    index.search(np.tile(q, (50, 1)), 10)   # 5000 queries: the batch runs in several pieces, one scratch set each
    streams = index.get_option("streams")
    assert streams > 1
    for name, call in kinds.items():
        for _ in range(streams + 1):
            call()
        assert index.get_option("streams") == streams, f"{name} kept a scratch set"


def test_dynamic_flat_delete_right_after_a_device_search():
    """An unfiltered device search, then at once a delete of the rows it returns: the delete waits for the search.  The
    search runs on the exact scan (cosine never takes the GEMM), which has nothing to synchronise, and the caller's
    stream is held by a spin kernel, so the whole scan -- it reads the slots' statuses, which the delete rewrites -- is
    still queued when the delete reaches the device.  Without the search's completion event the delete would clear the
    statuses before the scan starts."""
    import torch
    from scalablevectorsearch_b200 import DistanceType, DynamicFlat
    n, nq, k = 20000, 2000, 10
    x, q = _rows(n + nq, 64, np.float32, 50), _rows(nq, 64, np.float32, 51)
    dyn = DynamicFlat.build(x, np.arange(n + nq, dtype=np.uint64), DistanceType.Cosine)
    # nq rows deleted first: the delete below then fits the staging and allocates nothing (a cudaFree would synchronise
    # the device, and so wait for the search whatever the completion event says)
    dyn.delete(np.arange(n, n + nq, dtype=np.uint64))
    want = dyn.search(q, k)
    (dq,) = _to_device(q)
    ids, dists, _ = _outputs(nq, k)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)   # about 0.1 s of one thread spinning: the search below starts after it
    scanned = dyn.search_device(dq.data_ptr(), q.dtype, nq, k, ids.data_ptr(), dists.data_ptr(), stream=s.cuda_stream)
    dyn.delete(np.unique(want[0][:, 0]))   # no synchronisation: every query's nearest row goes at once
    torch.cuda.synchronize()
    assert scanned == nq, "every query should run on the exact scan"
    _same(want, _host_view(ids, dists), "device search before a delete")
