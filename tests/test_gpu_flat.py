"""Tensor-core exhaustive search (svsb200_flat_search*, csrc/flat.cu) == the exact scan, bit for bit.

The checker is svsb200_exhaustive_device (the search path's distance code over every base vector, itself checked
against the oracle in test_gpu_parity.py::test_exhaustive_scan_is_exact_topk): ids and distance bits must be equal
for every query, whether the GEMM candidates verified or the query fell back to the scan.  The fallback keeps the
result exact even when the GEMM is wrong, so on clustered vectors (where the error bound proves every query) the tests
also require that no query fell back: a defect in the GEMM or its accumulator layout, even in a single query row of a
tile, sends that row's queries to the scan and fails them."""
import numpy as np
import pytest

from conftest import bits

pytestmark = pytest.mark.gpu


def _both(index, q, k):
    import torch
    dq = torch.from_numpy(q).cuda()
    out = []
    for fn in ("exhaustive_device", "flat_search_device"):
        ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
        d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
        r = getattr(index, fn)(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), d.data_ptr(),
                               stream=torch.cuda.current_stream().cuda_stream or 1)
        torch.cuda.synchronize()
        out.append((ids.cpu().numpy(), d.cpu().numpy(), r))
    return out


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16])
def test_flat_equals_exact_scan_on_clustered_vectors(metric, dtype):
    from scalablevectorsearch_b200 import DistanceType, Vamana
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(40_000, 333, 96)
    base = base.astype(dtype)
    graph = np.zeros((base.shape[0], 2), dtype=np.uint32)
    index = Vamana.from_arrays(base, graph, 0, {"l2": DistanceType.L2, "ip": DistanceType.MIP}[metric])
    (ei, ed, _), (fi, fd, nfb) = _both(index, queries, 10)
    assert np.array_equal(fi, ei), (metric, dtype)
    assert np.array_equal(bits(fd), bits(ed))
    assert nfb == 0, f"{nfb} of {queries.shape[0]} queries fell back to the scan"
    hi, hd = index.flat_search(queries[:50], 10)          # host-buffer form
    assert np.array_equal(hi.astype(np.int64), ei[:50]) and np.array_equal(bits(hd), bits(ed[:50]))


@pytest.mark.timeout(300)
def test_flat_on_the_reference_dataset_with_ties_and_odd_shapes(dataset):
    """Integer-valued data (exact ties everywhere, large norms: most queries take the verified-or-fallback route),
    dim 128, n not a multiple of the tile, nq not a multiple of 128, f16 queries, k = 1 and 25."""
    from scalablevectorsearch_b200 import DistanceType, Vamana
    x = dataset.data[:9999]
    graph = np.zeros((x.shape[0], 2), dtype=np.uint32)
    for metric in (DistanceType.L2, DistanceType.MIP):
        index = Vamana.from_arrays(x, graph, 0, metric)
        for q, k in ((dataset.queries[:130], 25), (dataset.queries[:7].astype(np.float16), 1)):
            (ei, ed, _), (fi, fd, _) = _both(index, q, k)
            assert np.array_equal(fi, ei) and np.array_equal(bits(fd), bits(ed)), (metric, k)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n,nq,dim", [(40_000, 1100, 96), (30_000, 600, 256), (20_000, 1300, 272)])
def test_flat_row_groups_and_pacing(n, nq, dim):
    """Batches of >= 4 query tiles are walked in row groups (2 or 4 CTAs on the same base tiles, csrc/flat.cu): 9 tiles =
    two full groups and one with three absent tiles; 5 tiles = pairs with one absent; rows of >= 256 elements switch
    the producers' pacing on; 272 is not a multiple of the 32-element k-block."""
    from scalablevectorsearch_b200 import DistanceType, Vamana
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    base, queries = clustered_unit_vectors(n, nq, dim)
    graph = np.zeros((n, 2), dtype=np.uint32)
    for metric in (DistanceType.L2, DistanceType.MIP):
        index = Vamana.from_arrays(base, graph, 0, metric)
        (ei, ed, _), (fi, fd, nfb) = _both(index, queries, 10)
        assert np.array_equal(fi, ei), (metric, n, nq, dim)
        assert np.array_equal(bits(fd), bits(ed))
        assert nfb == 0, f"{nfb} of {nq} queries fell back to the scan"
