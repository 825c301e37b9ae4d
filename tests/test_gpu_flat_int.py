"""Exact flat search over int8 / uint8 data (svsb200_flat_search*, csrc/flat.cu) == the exact scan, bit for bit.

(int8, int8) and (uint8, uint8) run the integer tensor-core GEMM, whose keys are exact: its per-range lists hold the
smallest (key, id) pairs, and wherever the distances stay below 2^24 the certificate holds for every query, ties
included -- so those cases also require that no query fell back to the scan.  float32 queries over integer data take
the fp16 GEMM.  The checker is svsb200_exhaustive_device, as in tests/test_gpu_flat.py."""
import numpy as np
import pytest

from conftest import bits

pytestmark = pytest.mark.gpu


def _both(index, q, k):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    out = []
    for fn in ("exhaustive_device", "flat_search_device"):
        ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
        d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
        r = getattr(index, fn)(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), d.data_ptr(),
                               stream=torch.cuda.current_stream().cuda_stream or 1)
        torch.cuda.synchronize()
        out.append((ids.cpu().numpy(), d.cpu().numpy(), r))
    return out


def _index(x, metric):
    from scalablevectorsearch_b200 import DistanceType, Vamana
    graph = np.zeros((x.shape[0], 2), dtype=np.uint32)
    return Vamana.from_arrays(x, graph, 0, {"l2": DistanceType.L2, "ip": DistanceType.MIP,
                                            "cosine": DistanceType.Cosine}[metric])


def _check(index, q, k, fallbacks=0):
    (ei, ed, _), (fi, fd, nfb) = _both(index, q, k)
    assert np.array_equal(fi, ei)
    assert np.array_equal(bits(fd), bits(ed))
    if fallbacks is not None:
        assert nfb == fallbacks, f"{nfb} of {q.shape[0]} queries fell back to the scan (expected {fallbacks})"
    return ei, ed, nfb


def _clustered(n, nq, dim, dtype):
    """Clustered unit vectors mapped affinely onto the integer range of `dtype`."""
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(n, nq, dim)
    lo, hi = float(min(base.min(), queries.min())), float(max(base.max(), queries.max()))
    if dtype == np.uint8:
        f = lambda v: np.rint((v - lo) * (255.0 / (hi - lo))).astype(np.uint8)   # noqa: E731
    else:
        m = max(abs(lo), abs(hi))
        f = lambda v: np.rint(v * (127.0 / m)).astype(np.int8)   # noqa: E731
    return f(base), f(queries)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
def test_int_flat_equals_exact_scan_on_clustered_vectors(metric, dtype):
    base, queries = _clustered(40_000, 333, 96, dtype)
    index = _index(base, metric)
    ei, ed, _ = _check(index, queries, 10)
    hi, hd = index.flat_search(queries[:50], 10)          # host-buffer form
    assert np.array_equal(hi.astype(np.int64), ei[:50]) and np.array_equal(bits(hd), bits(ed[:50]))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("variant", ["i8_i8", "u8_u8"])
def test_int_flat_on_the_reference_dataset_with_ties(dataset, variant):
    """Integer-valued data with exact distance ties everywhere: the (key, id) lists and the certificate leave no
    query to the scan; n = 9999 is not a multiple of the tile, 130 queries not a multiple of 128."""
    q, x = dataset.variant(variant)
    x = x[:9999]
    for metric in ("l2", "ip"):
        index = _index(x, metric)
        for qq, k in ((q[:130], 25), (q[:7], 1)):
            _check(index, qq, k)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_int_flat_narrow_range_ties(metric):
    """int8 values in [-3, 3]: nearly every key is tied with many others."""
    rng = np.random.default_rng(5)
    x = rng.integers(-3, 4, size=(20_000, 64)).astype(np.int8)
    q = rng.integers(-3, 4, size=(300, 64)).astype(np.int8)
    _check(_index(x, metric), q, 10)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n,nq,dim", [(40_000, 1100, 96), (30_000, 600, 256), (20_000, 1300, 272), (5_000, 200, 17),
                                      (5_000, 200, 100), (20_000, 1100, 576), (12_000, 600, 520)])
def test_int_flat_row_groups_pacing_and_ragged_k_blocks(n, nq, dim):
    """Row groups of 2 and 4 query tiles, rows that are not a multiple of the 64-element k-block, and the producers'
    pacing, which runs for rows of >= 8 integer k-blocks (dim > 448) with row groups: 576 (9 k-blocks, groups of 4)
    and 520 (9 k-blocks, the last one ragged, groups of 2)."""
    for dtype in (np.int8, np.uint8):
        base, queries = _clustered(n, nq, dim, dtype)
        for metric in ("l2", "ip"):
            _check(_index(base, metric), queries, 10)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_int_flat_in_the_rounding_regime(metric):
    """uint8 at dim 300 with values near 0 and 255: every distance is above 2^24, where float32 rounds it and exact
    ties appear that the integers do not have.  The result is still exact; queries whose certificate fails there
    take the scan (their number is only reported)."""
    rng = np.random.default_rng(11)
    x = rng.integers(248, 256, size=(6_000, 300)).astype(np.uint8)
    q = rng.integers(0, 8, size=(150, 300)) if metric == "l2" else rng.integers(248, 256, size=(150, 300))
    _, ed, nfb = _check(_index(x, metric), q.astype(np.uint8), 10, fallbacks=None)
    assert np.abs(ed).min() > 1 << 24
    print(f"{metric}: {nfb} of {q.shape[0]} queries fell back")


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_int_flat_equals_the_float_path_on_the_same_values(metric):
    """Below 2^24 the uint8 path (integer GEMM) and the float32 path (fp16 GEMM) over the same values agree bit for
    bit."""
    base, queries = _clustered(30_000, 200, 128, np.uint8)
    ui, ud, _ = _check(_index(base, metric), queries, 10)
    fi, fd, _ = _check(_index(base.astype(np.float32), metric), queries.astype(np.float32), 10, fallbacks=None)
    assert np.array_equal(ui, fi) and np.array_equal(bits(ud), bits(fd))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("dtype", [np.int8, np.uint8])
def test_float32_queries_over_int_data(metric, dtype):
    """float32 queries over int8 / uint8 data take the fp16 GEMM: the data is exact in fp16, only the query rounds.
    (uint8 rows as non-negative features, like SIFT's: the magnitudes of clustered vectors.)"""
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(40_000, 333, 96)
    if dtype == np.uint8:
        base, queries = np.abs(base), np.abs(queries)
    s = (255.0 if dtype == np.uint8 else 127.0) / float(np.abs(base).max())
    x = np.rint(base * s).astype(dtype)
    q = (queries * s).astype(np.float32)
    _check(_index(x, metric), q, 10)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_int_flat_wide_rows(metric):
    """dim 10 000: the rescoring kernel stages the query in more than the default 48 KB of shared memory (float32
    queries) or close to it (integer codes), for both GEMM routes.  Distances pass 2^24 here, so fallbacks are
    allowed; the results must still equal the scan's."""
    rng = np.random.default_rng(17)
    x = rng.integers(0, 256, size=(1_000, 10_000)).astype(np.uint8)
    q = rng.integers(0, 256, size=(20, 10_000)).astype(np.uint8)
    index = _index(x, metric)
    _check(index, q, 10, fallbacks=None)
    _check(index, q.astype(np.float32) + np.float32(0.25), 10, fallbacks=None)


@pytest.mark.timeout(300)
def test_int_shapes_that_keep_the_scan():
    """Integer cosine, k > 25 and n < 512 stay on the exact scan."""
    base, queries = _clustered(4_000, 100, 64, np.uint8)
    _check(_index(base, "cosine"), queries, 10, fallbacks=100)
    _check(_index(base, "l2"), queries, 26, fallbacks=100)
    _check(_index(base[:500], "l2"), queries, 10, fallbacks=100)
