"""The fp16 flat search beyond float16's range: elements that overflow fp16, and elements in its subnormals.

Both fp16 entry points -- Vamana.flat_search_device (k = 10 and 25, the 33-entry lists) and Flat.search_device (k = 100
over 300 queries, the deep lists) -- must return, for every query, the ids and distance bits of
  * the exact scan over the same rows (exhaustive_device), and
  * the C oracle's distances (oracle.distance_rows, the pinned restatement of the reference) sorted by (distance, id).
The second check also holds the scan itself to the oracle on values this small, where a scan that flushed denormals
would agree with the flat path and still be wrong.  Where a fixture was designed around one answer (a row beyond fp16's
range, the zero row), every affected query's top 1 must be that row, which float64 distances confirm.

The fixtures (tests/flat_range_fixtures.py) defeat an error bound that assumes a relative fp16 rounding of 2^-11: on
them, such a bound accepts candidate lists that miss the answer (tests/test_flat_bound_model.py shows it on a model).
A query or base with an element that overflows fp16 must fall back to the scan; the tightness control -- ordinary
clustered data that merely touches fp16's subnormals -- must not fall back at all."""
import numpy as np
import pytest

import flat_range_fixtures as fx
from conftest import bits

pytestmark = pytest.mark.gpu

NQ = 300   # > 256: Flat.search_device runs the deep lists at k = 100


def _device_call(fn, q, k):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
    d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
    r = fn(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), d.data_ptr(),
           stream=torch.cuda.current_stream().cuda_stream or 1)
    torch.cuda.synchronize()
    return ids.cpu().numpy(), d.cpu().numpy(), r


def _oracle_topk(oracle, metric, q, x, k):
    ids = np.empty((q.shape[0], k), dtype=np.int64)
    dists = np.empty((q.shape[0], k), dtype=np.float32)
    for i in range(q.shape[0]):
        d = oracle.distance_rows(metric, q[i], x)
        ids[i] = np.lexsort((np.arange(x.shape[0]), d if metric == "l2" else -d))[:k]
        dists[i] = d[ids[i]]
    return ids, dists


def _check(oracle, x, q, metric, nearest=None, affected=None):
    """Both entry points against the scan and the oracle; returns the fallback counts {(entry point, k): count}."""
    from scalablevectorsearch_b200 import DistanceType, Flat, Vamana
    dist = {"l2": DistanceType.L2, "ip": DistanceType.MIP}[metric]
    scan = Vamana.from_arrays(x, np.zeros((x.shape[0], 2), dtype=np.uint32), 0, dist)
    flat = Flat(x, dist)
    oi, od = _oracle_topk(oracle, metric, q, x, 100)
    fallbacks = {}
    for name, fn, k in (("flat_search_device", scan.flat_search_device, 10),
                        ("flat_search_device", scan.flat_search_device, 25), ("Flat.search_device", flat.search_device, 100)):
        ei, ed, _ = _device_call(scan.exhaustive_device, q, k)
        fi, fd, nfb = _device_call(fn, q, k)
        bad = np.flatnonzero((fi != ei).any(1) | (bits(fd) != bits(ed)).any(1))
        assert bad.size == 0, f"{name} k={k}: queries {bad[:10]} differ from the exact scan ({nfb} fell back)"
        assert np.array_equal(ei, oi[:, :k]) and np.array_equal(bits(ed), bits(od[:, :k])), \
            f"k={k}: the exact scan differs from the oracle"
        if nearest is not None:
            rows = np.arange(q.shape[0]) if affected is None else np.flatnonzero(affected)
            assert (fi[rows, 0] == nearest).all(), f"{name} k={k}: the designed top 1 is missing"
        fallbacks[name, k] = nfb
    return fallbacks


def _designed(x, q, metric, nearest, rows):
    """float64 distances confirm that row `nearest` is the exact top 1 of queries `rows`."""
    x64, q64 = x.astype(np.float64), q[rows].astype(np.float64)
    d = ((q64[:, None, :] - x64[None, :, :]) ** 2).sum(2) if metric == "l2" else -(q64 @ x64.T)
    assert (d.argmin(1) == nearest).all()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("qtype", [np.float32, np.float16])
def test_data_beyond_fp16_falls_back_and_stays_exact(oracle, metric, qtype):
    """float32 rows, one of them (the exact top 1 of every query) beyond fp16's range: no query may be verified."""
    x, q, z = fx.data_overflow(metric, NQ)
    q = q.astype(qtype)
    _designed(x, q, metric, z, np.arange(NQ))
    for (name, k), nfb in _check(oracle, x, q, metric, nearest=z).items():
        assert nfb == NQ, f"{name} k={k}: only {nfb} of {NQ} queries fell back"


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16, np.uint8, np.int8])
def test_queries_beyond_fp16_fall_back_and_stay_exact(oracle, metric, dtype):
    """float32 queries with an element >= 65520, mixed in one batch with in-range queries: every overflowing query
    falls back (under L2 its exact top 1 is the zero row, which its fp16 key -- NaN -- hides from the lists)."""
    x, q, z = fx.query_overflow(metric, dtype, NQ)
    over = fx.overflowing(q)
    assert 0 < over.sum() < NQ
    if z is not None:
        _designed(x, q, metric, z, np.flatnonzero(over))
    for (name, k), nfb in _check(oracle, x, q, metric, nearest=z, affected=over).items():
        assert nfb >= over.sum(), f"{name} k={k}: {nfb} fell back, {over.sum()} queries overflow fp16"


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("inf_row", [False, True])
def test_the_65504_boundary(oracle, metric, inf_row):
    """Elements of +-65504 and +-65519 (finite in fp16) and +-65520 (inf), in rows and queries: exact either way."""
    x, q, _ = fx.boundary(inf_row, NQ)
    fallbacks = _check(oracle, x, q, metric)
    if inf_row:
        assert all(nfb == NQ for nfb in fallbacks.values()), fallbacks
    else:
        assert all(nfb >= fx.overflowing(q).sum() for nfb in fallbacks.values()), fallbacks


@pytest.mark.timeout(300)
@pytest.mark.parametrize("scale", [1e-6, 3e-7, 1e-7])
@pytest.mark.parametrize("dim", [16, 32, 96, 100])
def test_thin_shell_in_fp16_subnormals(oracle, scale, dim):
    """Rows on a thin shell with elements of about `scale`, queries 0 and 0.01 x a row; (query, data) types f32/f32,
    f16/f32 and f32/f16; L2 and MIP.  Exact, whatever falls back."""
    x, q, _ = fx.thin_shell(scale, dim, nq=NQ)
    for xt, qt in ((np.float32, np.float32), (np.float32, np.float16), (np.float16, np.float32)):
        for metric in ("l2", "ip"):
            _check(oracle, x.astype(xt), q.astype(qt), metric)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_subnormal_queries_over_uint8(oracle, metric):
    x, q, _ = fx.subnormal_queries_u8(NQ)
    _check(oracle, x, q, metric)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_ordinary_data_touching_subnormals_still_verifies(oracle, metric):
    """The tightness control: a bound made sound by being loose would send these queries to the scan."""
    x, q, _ = fx.tightness_control()
    for (name, k), nfb in _check(oracle, x, q, metric).items():
        assert nfb == 0, f"{name} k={k}: {nfb} of {q.shape[0]} queries fell back to the scan"
