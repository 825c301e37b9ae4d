"""The graph-free flat index (svsb200_flat_index_*, Python Flat) == the exact scan, bit for bit.

For 26 <= k <= 121 the index runs the tensor-core GEMM with deep candidate lists (129 entries per query and base range,
csrc/flat.cu).  The checker is Vamana.exhaustive_device over the same rows (dummy graph), as in tests/test_gpu_flat.py:
ids and distance bits must be equal, and on the shapes where the error bound proves every query (clustered vectors,
integer rows below 2^24) no query may fall back to the scan."""
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits

pytestmark = pytest.mark.gpu

METRICS = {"l2": 0, "ip": 1, "cosine": 2}


def _flat(x, metric):
    from scalablevectorsearch_b200 import DistanceType, Flat
    return Flat(x, DistanceType(METRICS[metric]))


def _scan_index(x, metric):
    from scalablevectorsearch_b200 import DistanceType, Vamana
    return Vamana.from_arrays(x, np.zeros((x.shape[0], 2), dtype=np.uint32), 0, DistanceType(METRICS[metric]))


def _device_call(fn, q, k):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
    d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
    r = fn(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), d.data_ptr(),
           stream=torch.cuda.current_stream().cuda_stream or 1)
    torch.cuda.synchronize()
    return ids.cpu().numpy(), d.cpu().numpy(), r


def _check(x, q, metric, ks, fallbacks=0):
    """Flat.search_device == exhaustive_device over the same rows for every k; returns the fallback counts."""
    flat, scan = _flat(x, metric), _scan_index(x, metric)
    out = []
    for k in ks:
        ei, ed, _ = _device_call(scan.exhaustive_device, q, k)
        fi, fd, nfb = _device_call(flat.search_device, q, k)
        assert np.array_equal(fi, ei), (metric, k)
        assert np.array_equal(bits(fd), bits(ed)), (metric, k)
        if fallbacks is not None:
            assert nfb == fallbacks, f"k={k}: {nfb} of {q.shape[0]} queries fell back to the scan (expected {fallbacks})"
        out.append(nfb)
    return out


def _clustered_int(n, nq, dim, dtype):
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(n, nq, dim)
    lo, hi = float(min(base.min(), queries.min())), float(max(base.max(), queries.max()))
    if dtype == np.uint8:
        f = lambda v: np.rint((v - lo) * (255.0 / (hi - lo))).astype(np.uint8)   # noqa: E731
    else:
        m = max(abs(lo), abs(hi))
        f = lambda v: np.rint(v * (127.0 / m)).astype(np.int8)   # noqa: E731
    return f(base), f(queries)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("dtype,qtype", [(np.float32, np.float32), (np.float32, np.float16), (np.float16, np.float32),
                                         (np.float16, np.float16)])
def test_deep_lists_equal_the_scan_on_clustered_vectors(metric, dtype, qtype):
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(40_000, 333, 96)
    _check(base.astype(dtype), queries.astype(qtype), metric, (26, 50, 100, 121))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
def test_deep_integer_lists_equal_the_scan(metric, dtype):
    base, queries = _clustered_int(40_000, 333, 96, dtype)
    _check(base, queries, metric, (100,))
    # float32 queries over integer rows take the fp16 GEMM
    if dtype == np.uint8:
        _check(base, queries.astype(np.float32) + np.float32(0.25), metric, (100,))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_deep_integer_lists_with_ties_everywhere(metric):
    """int8 values in [-3, 3]: nearly every key is tied with many others; the (key, id) lists stay exact."""
    rng = np.random.default_rng(5)
    x = rng.integers(-3, 4, size=(20_000, 64)).astype(np.int8)
    q = rng.integers(-3, 4, size=(300, 64)).astype(np.int8)
    _check(x, q, metric, (100,))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("n,nq,dim", [(40_000, 1100, 96), (30_000, 600, 256), (20_000, 1300, 272), (12_000, 600, 520)])
def test_deep_lists_row_groups_pacing_and_ragged_k_blocks(n, nq, dim):
    """The row-group, pacing and ragged k-block shapes of test_gpu_flat.py / test_gpu_flat_int.py at k = 100."""
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(n, nq, dim)
    for metric in ("l2", "ip"):
        _check(base, queries, metric, (100,))
    xb, xq = _clustered_int(n, nq, dim, np.uint8)
    _check(xb, xq, "l2", (100,))


@pytest.mark.timeout(600)
def test_deep_lists_small_batches_over_many_rows():
    """Over 200k rows, batches of one or two query tiles (nq <= 256) take the scan at deep k (one tile keeps only 7 CTAs
    busy with the deep lists); from three tiles on (nq = 257, 300) the deep lists run, each tile cut into as many
    pieces as the rescoring kernel holds."""
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(200_000, 300, 96)
    for nq in (1, 7, 100, 129, 256):
        _check(base, queries[:nq], "l2", (100,), fallbacks=nq)
        _check(base, queries[:nq], "l2", (25,))
    for nq in (257, 300):
        _check(base, queries[:nq], "l2", (26, 100))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_small_k_takes_the_existing_path(metric):
    """k = 10 and 25 on the Flat handle == Vamana.flat_search on the same rows (host forms, ids and distance bits)."""
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(40_000, 200, 96)
    flat, scan = _flat(base, metric), _scan_index(base, metric)
    for k in (10, 25):
        fi, fd = flat.search(queries, k)
        vi, vd = scan.flat_search(queries, k)
        assert fi.dtype == np.uint64 and np.array_equal(fi, vi) and np.array_equal(bits(fd), bits(vd))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
def test_reference_ground_truth_at_k100(dataset, metric):
    """Flat(...).search(queries, 100) over the reference's test dataset returns its 100-deep ground truth
    (groundtruth_*.ivecs, tests/golden/flat_gt100.npz): the same ids as sets except inside the tie group at the 100th
    distance.  L2 / MIP distances are integers below 2^24, so they must equal the exact integer distances of the
    returned ids, be the 100 smallest exact distances of the query, and end at the exact distance of the reference's
    100th id; cosine ids outside the reference's set must tie the 100th distance."""
    gt = np.load(os.path.join(GOLDEN, "flat_gt100.npz"))[metric].astype(np.int64)
    x, q = dataset.data, dataset.queries
    ids, d = _flat(x, metric).search(q, 100)
    ids = ids.astype(np.int64)
    if metric != "cosine":
        xi, qi = x.astype(np.int64), q.astype(np.int64)
        exact = -(qi @ xi.T) if metric == "ip" else (qi * qi).sum(1)[:, None] + (xi * xi).sum(1)[None, :] - 2 * qi @ xi.T
        want = np.take_along_axis(exact, ids, 1)
        assert np.array_equal(d.astype(np.float64), (-want if metric == "ip" else want).astype(np.float64))
        # an exact top 100: the keys are the 100 smallest of the query, the last one the key of the reference's 100th
        assert np.array_equal(want, np.sort(exact, axis=1)[:, :100])
        assert np.array_equal(want[:, 99], exact[np.arange(q.shape[0]), gt[:, 99]])
    for i in range(q.shape[0]):
        a, b = set(ids[i].tolist()), set(gt[i].tolist())
        if a == b:
            continue
        # every id outside the reference's set sits at the 100th distance (a tie the reference broke otherwise)
        for j in np.flatnonzero([v not in b for v in ids[i]]):
            assert bits(d[i, j]) == bits(d[i, 99]), (metric, i)


@pytest.mark.timeout(600)
def test_shapes_that_keep_the_scan():
    """k = 122, cosine and n < 512 run the scan for every query."""
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(4_000, 100, 64)
    _check(base, queries, "l2", (122,), fallbacks=100)
    _check(base, queries, "cosine", (10, 100), fallbacks=100)
    _check(base[:500], queries, "l2", (10, 100), fallbacks=100)


@pytest.mark.timeout(600)
def test_api_memory_and_errors():
    from scalablevectorsearch_b200 import Svsb200Error
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(2_000, 10, 100)
    flat = _flat(base, "l2")
    assert flat.size == 2_000 and flat.dimensions == 100
    assert flat.device_bytes == 2_000 * 400   # the rows only (400-byte rows are already 16-byte aligned)
    for k in (0, 1025):
        with pytest.raises(Svsb200Error, match="k must be in"):
            flat.search(queries, k)
    xi = _flat(np.rint(base * 100).astype(np.int8), "l2")
    with pytest.raises(Svsb200Error, match="float16 queries"):
        xi.search(queries.astype(np.float16), 10)
    ids, _ = _flat(base[:5], "l2").search(queries, 8)   # k > n: padded rows
    assert (ids[:, 5:] == np.iinfo(np.uint64).max).all()


@pytest.mark.timeout(600)
def test_runtime_flat_index_demo_matches_the_c_abi(tmp_path):
    """cpp/flat_demo, written against the reference's runtime header only (svs::runtime::v0::FlatIndex) and linked with
    libsvsb200_runtime.so, prints the same top-100 as the C ABI, and the runtime's error codes: FP16 storage
    INVALID_ARGUMENT (2), search before add NOT_INITIALIZED (4) with label -1 / +inf, a second add NOT_IMPLEMENTED (3),
    k = 0 INVALID_ARGUMENT."""
    exe = os.path.join(ROOT, "scalablevectorsearch_b200", "cpp", "_build", "flat_demo")
    if not os.path.exists(exe):
        pytest.skip("flat_demo not built (needs the reference's runtime headers at build time)")
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    n, nq, dim, k = 20_000, 300, 96, 100
    base, queries = clustered_unit_vectors(n, nq, dim)
    base.tofile(tmp_path / "x.f32")
    queries.tofile(tmp_path / "q.f32")
    out = subprocess.run([exe, str(tmp_path / "x.f32"), str(n), str(dim), str(tmp_path / "q.f32"), str(nq), str(k)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    rows = {}
    for line in out.stdout.splitlines():
        tag, *rest = line.split()
        rows.setdefault(tag, []).append(rest)
    assert rows["storage_fp16"] == [["2"]]
    assert rows["search_before_add"] == [["4", str(2 ** 64 - 1), "inf"]]
    assert rows["second_add"] == [["3"]] and rows["k0"] == [["2"]]
    got_ids = np.array([int(r[0]) for r in rows["result"]], dtype=np.uint64).reshape(nq, k)
    got_d = np.array([float(r[1]) for r in rows["result"]]).astype(np.float32).reshape(nq, k)
    ids, d = _flat(base, "l2").search(queries, k)
    assert np.array_equal(got_ids, ids) and np.array_equal(bits(got_d), bits(d))
