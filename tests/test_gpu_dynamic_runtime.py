"""Stored-row access on the GPU (svsb200_index_distances / svsb200_index_reconstruct, Vamana.get_distance /
reconstruct) and the runtime DynamicVamanaIndex built on it.

* Every (query, returned neighbour) pair of a search has exactly the search's distance bits, on static float32,
  float16, int8, uint8 and SQ handles and on dynamic float32, float16 and SQ int8 / uint8 handles after every step of a
  mutation script, over L2, MIP and cosine at dims 96, 101, 128 and 256.
* On a static handle the distance to every row, reached by the walk or not, equals the exhaustive scan's.
* get_distance and reconstruct of the dynamic float32 / float16 / SQ indexes equal the reference's MutableVamanaIndex
  (the façades over its unmodified headers) bit for bit after the same mutations, compacted slots included.
* Absent, Deleted and out-of-range ids, LVQ-8 handles and wrong query types are refused, name the id, write nothing.
* cpp/dynamic_vamana_demo, written against the runtime header only, prints what DynamicVamana computes for the same
  script, storage kind by storage kind.
"""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

METRICS = ("l2", "mip", "cosine")
DIMS = (96, 101, 128, 256)
REF_METRIC = {"l2": "l2", "mip": "ip", "cosine": "cosine"}   # the façades' metric names


def _dt(metric):
    from scalablevectorsearch_b200 import DistanceType
    return {"l2": DistanceType.L2, "mip": DistanceType.MIP, "cosine": DistanceType.Cosine}[metric]


def _data(n, dim, seed):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((8, dim)).astype(np.float32) * 2
    return (centers[rng.integers(0, 8, n)] + rng.standard_normal((n, dim)).astype(np.float32)).astype(np.float32)


def _params(R=16, window=32):
    from scalablevectorsearch_b200 import VamanaBuildParameters
    p = VamanaBuildParameters()
    p.graph_max_degree, p.window_size = R, window
    return p


def _distances(index, queries, ids):
    """svsb200_index_distances for every (query row, id) pair of a [nq, k] id block (padding ids skipped)."""
    from scalablevectorsearch_b200 import _lib
    nq, k = ids.shape
    mask = ids != np.uint64(2**64 - 1)
    qq = np.ascontiguousarray(np.repeat(queries, k, axis=0)[mask.reshape(-1)])
    flat = np.ascontiguousarray(ids[mask])
    out = np.empty(flat.shape[0], dtype=np.float32)
    _lib.check(_lib.lib().svsb200_index_distances(index._h, qq.ctypes.data, _lib._DTYPE_CODE[qq.dtype], flat.shape[0],
                                                  flat.ctypes.data, out.ctypes.data))
    return out, mask


def _same_as_search(index, queries, k=10, what=""):
    ids, dists = index.search(queries, k)
    got, mask = _distances(index, queries, ids)
    assert mask.sum() > 0
    assert np.array_equal(got.view(np.uint32), dists[mask].view(np.uint32)), what


def _static(kind, metric, dim, seed=1):
    from scalablevectorsearch_b200 import Vamana
    from scalablevectorsearch_b200.ivf import sq_compress
    x = _data(600, dim, seed)
    if kind == "f32":
        return Vamana.build(_params(), x, _dt(metric)), x
    if kind == "f16":
        return Vamana.build(_params(), x.astype(np.float16), _dt(metric)), x
    if kind in ("i8", "u8"):
        rows = np.clip(np.rint(x * 20) + (0 if kind == "i8" else 128), -128 if kind == "i8" else 0,
                       127 if kind == "i8" else 255).astype(np.int8 if kind == "i8" else np.uint8)
        return Vamana.build(_params(), rows, _dt(metric)), rows
    codes, scale, bias = sq_compress(x, np.int8 if kind == "sq_i8" else np.uint8)
    return Vamana.build(_params(), codes, _dt(metric), sq=(scale, bias)), x


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("kind", ("f32", "f16", "i8", "u8", "sq_i8", "sq_u8"))
def test_static_distances_equal_the_search(kind, metric, dim):
    index, base = _static(kind, metric, dim)
    index.search_window_size = 40
    q = _data(24, dim, 7)
    _same_as_search(index, q, what="float32 queries")
    if kind != "f32" and kind[:2] != "sq":
        # float16 queries over float rows, the rows' own type over integer rows
        qq = q.astype(np.float16) if kind == "f16" else base[:24]
        _same_as_search(index, qq, what=f"{qq.dtype} queries")
    if kind in ("f32", "sq_i8"):
        _same_as_search(index, q.astype(np.float16), what="float16 queries")


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("kind", ("f32", "f16", "i8", "sq_u8"))
def test_rows_no_walk_reaches_match_the_exhaustive_scan(kind, metric):
    import torch
    index, _ = _static(kind, metric, 101, seed=3)
    n = index.size
    q = _data(4, 101, 9)
    dq = torch.from_numpy(q).cuda()
    d_ids = torch.empty((4, n), dtype=torch.int64, device="cuda")
    d_d = torch.empty((4, n), dtype=torch.float32, device="cuda")
    index.exhaustive_device(dq.data_ptr(), np.float32, 4, n, d_ids.data_ptr(), d_d.data_ptr())
    torch.cuda.synchronize()
    ids, dd = d_ids.cpu().numpy().view(np.uint64), d_d.cpu().numpy()
    got, mask = _distances(index, q, ids)
    assert mask.all()
    assert np.array_equal(got.view(np.uint32), dd.reshape(-1).view(np.uint32))
    # and with a shard's id offset: the same rows under the offset ids
    from scalablevectorsearch_b200 import _lib
    _lib.check(_lib.lib().svsb200_set_id_offset(index._h, 5000))
    assert index.get_distance(5000 + int(ids[0, 3]), q[0]) == float(dd[0, 3])


def _dynamic(kind, metric, dim, n=500, seed=11):
    """A GPU dynamic index and the reference's façade over the same rows and graph (None where no façade exists)."""
    from oracle.dynamic_rows import RefDynamicRowsLib, RefDynamicSQRowsLib
    from scalablevectorsearch_b200 import DynamicVamana
    from scalablevectorsearch_b200.ivf import sq_compress
    x = _data(n, dim, seed)
    ids = np.arange(n, dtype=np.uint64) * 3 + 100
    sq = None
    if kind in ("sq_i8", "sq_u8"):
        codes, scale, bias = sq_compress(x, np.int8 if kind == "sq_i8" else np.uint8)
        index = DynamicVamana.build(_params(), codes, ids, _dt(metric), sq=(scale, bias))
        sq = (codes, scale, bias)
    else:
        rows = x.astype(np.float16) if kind == "f16" else x
        index = DynamicVamana.build(_params(), rows, ids, _dt(metric))
    graph, _, _, ep = index.export()
    b = index._build_parameters()
    args = (b["alpha"], b["construction_window_size"], b["max_candidates"], b["prune_to"])
    ref = None
    if sq is not None and RefDynamicSQRowsLib.available():
        ref = RefDynamicSQRowsLib().dynamic(sq[0], sq[1], sq[2], graph, ep, ids, REF_METRIC[metric], *args)
    elif sq is None and RefDynamicRowsLib.available():
        ref = RefDynamicRowsLib().dynamic(x.astype(np.float16) if kind == "f16" else x, graph, ep, ids, REF_METRIC[metric], *args)
    return index, ref, x, ids


def _against_reference(index, ref, q, what):
    if ref is None:
        return
    from oracle import dynamic_rows
    valid = index.all_ids()
    for j, e in enumerate(valid[::7]):
        got = np.float32(index.get_distance(int(e), q[j % len(q)]))
        want = np.float32(dynamic_rows.get_distance(ref, int(e), q[j % len(q)]))
        assert got.view(np.uint32) == want.view(np.uint32), (what, int(e))
    got = index.reconstruct(valid)
    want = dynamic_rows.reconstruct(ref, valid, index.dimensions)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), what


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("kind", ("f32", "f16", "sq_i8", "sq_u8"))
def test_dynamic_distances_through_the_mutation_script(kind, metric, dim):
    index, ref, x, ids = _dynamic(kind, metric, dim)
    index.search_window_size = 40
    q = _data(16, dim, 5)

    def step(what):
        _same_as_search(index, q, what=what)
        _against_reference(index, ref, q, what)

    step("built")
    _, _, _, ep = index.export()
    slots_ids = index.export()[2]
    gone = np.unique(np.concatenate([[slots_ids[ep]], ids[1::4]]))   # the entry point among them
    index.delete(gone)
    if ref is not None:
        ref.delete(gone)
    step("deleted")
    new = _data(40, dim, 13)
    new_ids = np.arange(40, dtype=np.uint64) + 10**6
    index.add(new if kind != "f16" else new.astype(np.float16), new_ids)
    if ref is not None:
        ref.add(new if kind != "f16" else new.astype(np.float16), new_ids)
    _same_as_search(index, q, what="added")   # (the façade links the new rows with its own builder)
    index.consolidate()
    _same_as_search(index, q, what="consolidated")
    index.compact()
    _same_as_search(index, q, what="compacted")
    if ref is not None:
        ref.consolidate()
        ref.compact()
    _against_reference(index, ref, q, "compacted")


def test_refusals_name_the_id_and_write_nothing():
    from scalablevectorsearch_b200 import DistanceType, Svsb200Error, Vamana, _lib, lvq8_compress
    index, ref, x, ids = _dynamic("f32", "l2", 96, n=200)
    index.delete(ids[:3])
    out = np.full((2, 96), 7.0, dtype=np.float32)
    lib = _lib.lib()
    for bad, word in ((int(ids[1]), "not in the index"), (5, "not in the index"), (2**64 - 1, "not in the index")):
        pick = np.array([ids[10], bad], dtype=np.uint64)
        with pytest.raises(Svsb200Error, match=f"{bad} is {word}"):
            _lib.check(lib.svsb200_index_reconstruct(index._h, pick.ctypes.data, 2, out.ctypes.data))
        with pytest.raises(Svsb200Error, match=str(bad)):
            _lib.check(lib.svsb200_index_distances(index._h, x[:2].ctypes.data, 0, 2, pick.ctypes.data, out.ctypes.data))
        assert (out == 7.0).all()
    with pytest.raises(Svsb200Error, match="int8/uint8 queries need"):
        index.get_distance(int(ids[10]), x[0].astype(np.int8))
    static, _ = _static("f32", "l2", 96)
    with pytest.raises(Svsb200Error, match="id 600 is out of range"):
        static.reconstruct([3, 600])
    rows, mean = lvq8_compress(x)
    lvq = Vamana.from_arrays(rows, np.zeros((200, 9), dtype=np.uint32), 0, DistanceType.L2, lvq8=(96, mean))
    with pytest.raises(Svsb200Error, match="LVQ-8"):
        lvq.reconstruct([0])
    with pytest.raises(Svsb200Error, match="LVQ-8"):
        lvq.get_distance(0, x[0])
    assert index.reconstruct(np.zeros(0, dtype=np.uint64)).shape == (0, 96)


# ---- the runtime DynamicVamanaIndex ----
def _demo(tmp_path, kind, x, q, k, R, window, radius):
    exe = os.path.join(ROOT, "scalablevectorsearch_b200", "cpp", "_build", "dynamic_vamana_demo")
    if not os.path.exists(exe):
        pytest.skip("dynamic_vamana_demo not built (needs the reference's runtime headers at build time)")
    x.tofile(tmp_path / "x.f32")
    q.tofile(tmp_path / "q.f32")
    out = subprocess.run([exe, str(tmp_path / "x.f32"), str(len(x)), str(x.shape[1]), str(tmp_path / "q.f32"), str(len(q)),
                          str(k), kind, str(R), str(window), repr(float(radius))], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    rows = {}
    for line in out.stdout.splitlines():
        tag, *rest = line.split()
        rows.setdefault(tag, []).append(rest)
    return rows


@pytest.mark.parametrize("kind", ("fp32", "fp16", "sqi8"))
def test_runtime_dynamic_vamana_demo_matches_the_c_abi(tmp_path, kind):
    from scalablevectorsearch_b200 import DistanceType, DynamicVamana, Svsb200Error, _lib
    from scalablevectorsearch_b200.ivf import sq_compress
    n, nq, dim, k, R, window = 1200, 20, 40, 10, 16, 40
    x = _data(n, dim, 31)
    q = _data(nq, dim, 32)
    radius = float(np.median(((q[:, None, :] - x[None, :200, :]) ** 2).sum(-1)) * 0.5)
    rows = _demo(tmp_path, kind, x, q, k, R, window, radius)
    assert rows["storage_lvq8"] == [["3"]] and rows["build_lvq8"] == [["3"]] and rows["build_leanvec"] == [["3"]]
    assert rows["blocksize"] == [["2", "2"]] and rows["blocksize_bytes"] == [[str(2**20)]]
    assert rows["uninit"] == [["4", str(2**64 - 1)]] and rows["add_nolabels"] == [["3"]]
    assert rows["k0"] == [["2"]] and rows["range0"] == [["2"]]

    def parsed(tag):
        return (np.array([int(r[0]) for r in rows[tag]], dtype=np.uint64).reshape(nq, k),
                np.array([float(r[1]) for r in rows[tag]]).astype(np.float32).reshape(nq, k))

    def same(tag, got, what):
        ids, dd = parsed(tag)
        assert np.array_equal(ids, got[0]), what
        assert np.array_equal(dd.view(np.uint32), got[1].view(np.uint32)), what

    labels = np.arange(n, dtype=np.uint64) + 1000
    half = n // 2
    rows_of = (lambda v: v.astype(np.float16)) if kind == "fp16" else (lambda v: v)
    if kind == "sqi8":
        codes, scale, bias = sq_compress(x[:1], np.int8)
        index = DynamicVamana.from_arrays(codes, np.zeros((1, R + 1), np.uint32), 0, labels[:1], DistanceType.L2,
                                          sq=(scale, bias))
    else:
        index = DynamicVamana.from_arrays(rows_of(x[:1]), np.zeros((1, R + 1), np.uint32), 0, labels[:1], DistanceType.L2)
    _lib.check(_lib.lib().svsb200_dynamic_set_build_parameters(index._h, 0.0, window, 0, 0))   # as the class maps them
    index.add(rows_of(x[1:half]), labels[1:half])
    index.add(rows_of(x[half:]), labels[half:])
    index.search_window_size = 2 * k
    same("plain", index.search(q, k), "plain")
    slot_ids = index.export()[2]
    status = index.export()[1]
    allowed = (status == 1) & (slot_ids % 3 == 0)
    fi, fd, _ = index.search_filtered(q, k, allowed)
    same("filtered", (fi, fd), "filtered")
    got_range = index.range_search(q, radius)
    want = [(int(r[0]), int(r[1]), np.float32(float(r[2]))) for r in rows.get("range", [])]
    have = [(qi, int(i), np.float32(d)) for qi, (ii, dd) in enumerate(got_range) for i, d in zip(ii, dd) if int(i) % 3 == 0]
    assert [(a, b) for a, b, _ in want] == [(a, b) for a, b, _ in have]
    assert all(u.view(np.uint32) == v.view(np.uint32) for (_, _, u), (_, _, v) in zip(want, have))

    index.delete(labels[::10])   # below the clean-up threshold: soft deletions only
    assert int(rows["memory_remove1"][0][0]) == index.device_bytes
    odd = np.array([labels[i] for i in range(1, n, 2) if i % 10], dtype=np.uint64)
    index.delete(odd)            # above it: consolidate and compact
    index.consolidate()
    index.compact()
    assert index.num_slots == index.size
    assert int(rows["memory_remove2"][0][0]) == index.device_bytes
    sevens = index.all_ids()[index.all_ids() % 7 == 0]
    index.delete(sevens)   # remove_selected: below the threshold again
    assert rows["removed"] == [[str(len(sevens))]]
    same("after", index.search(q, k), "after the removals")
    for label, d in rows["distance"]:
        assert np.float32(float(d)).view(np.uint32) == np.float32(index.get_distance(int(label), q[0])).view(np.uint32)
    with pytest.raises(Svsb200Error):
        index.get_distance(1001, q[0])
    assert rows["distance_removed"][0][0] == "5"   # RUNTIME_ERROR
    recon = np.array([float(r[1]) for r in rows["row"]], dtype=np.float64).astype(np.float32).reshape(3, dim)
    assert np.array_equal(recon.view(np.uint32), index.reconstruct([1002, 1004, 1006]).view(np.uint32))
    total, graph, data, meta = (int(v) for v in rows["memory"][0])
    assert total == index.device_bytes and graph + data + meta == total and min(graph, data, meta) > 0
    assert rows["reset"] == [["4", "0"]]
    if kind == "sqi8":
        codes, scale, bias = sq_compress(x, np.int8)
        again = DynamicVamana.build(_params(R, window), codes, labels, DistanceType.L2, sq=(scale, bias))
    else:
        again = DynamicVamana.build(_params(R, window), rows_of(x), labels, DistanceType.L2)
    again.search_window_size = 2 * k
    same("rebuilt", again.search(q, k), "rebuilt")
