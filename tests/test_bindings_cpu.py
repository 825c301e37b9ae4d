"""The Python bindings against a recording stub in place of libsvsb200.so (no GPU needed).

Every class is built through its public constructors and every public method and property is called.  The stub
records each C call; the tables below pin, per call, the C symbols made, every scalar argument (ints, floats and
bytes), whether each pointer argument is NULL, and the dtypes and shapes (or values) returned.  The side-effect-free
getters (``*_size``, ``*_dimensions`` ...) are left out of the sequences, except where a property reads them.
"""
import ctypes as C
import re

import numpy as np
import pytest

from test_abi import header_prototypes

SIZE, SLOTS, DIM, CLUSTERS, DEVICE_BYTES, MAX_DEGREE, DEVICES, LVQ_STRIDE = 6, 8, 4, 2, 4096, 3, 1, 12
GETTER = re.compile(r"_(size|num_slots|dimensions|num_clusters|device_bytes|max_degree|num_devices)$")
_REPLY = {"size": SIZE, "num_slots": SLOTS, "dimensions": DIM, "num_clusters": CLUSTERS, "device_bytes": DEVICE_BYTES,
          "max_degree": MAX_DEGREE, "num_devices": DEVICES}
HANDLE = 0x1000
RANGE_COUNTS = (2, 0, 1)   # per query: the results svsb200_range_search reports


class Stub:
    """Records (symbol, arguments) and returns 0, or fixed values from the getters.  Creators get a non-NULL handle,
    and svsb200_range_search reports RANGE_COUNTS results per query."""

    def __init__(self):
        self.calls = []
        self._keep = []

    def __getattr__(self, name):
        if not name.startswith("svsb200_"):
            raise AttributeError(name)

        def fn(*args):
            self.calls.append((name, args))
            g = GETTER.search(name)
            if g:
                return _REPLY[g.group(1)]
            if name == "svsb200_lvq8_row_stride":
                return LVQ_STRIDE
            if name.endswith(("_create", "_create_sq", "_create_multi", "_assemble", "_dynamic_build")):
                args[-1]._obj.value = HANDLE
            if name == "svsb200_range_search" and args[3]:   # as in the library, nq = 0 sets no output
                nq = args[3]
                counts = (C.c_uint32 * nq).from_address(args[6])
                counts[:] = RANGE_COUNTS[:nq]
                total = sum(RANGE_COUNTS[:nq])
                ids, dists = (C.c_uint64 * max(total, 1))(), (C.c_float * max(total, 1))()
                self._keep += [ids, dists]
                args[7]._obj.value, args[8]._obj.value = C.addressof(ids), C.addressof(dists)
            return 0
        return fn


_PROTOS = header_prototypes()


def _arg(param: str, a):
    """A recorded argument: scalars as they are, pointers as None or "p" (bytes, the option names, as they are)."""
    if a is None or isinstance(a, bytes):
        return a
    if "*" in param:
        return "p"
    assert isinstance(a, (int, float)), (param, a)
    return a


def _calls(stub, getters: bool):
    out = []
    for name, args in stub.calls:
        if GETTER.search(name) and not getters:
            continue
        params = _PROTOS[name][1]
        assert len(params) == len(args), name
        out.append((name,) + tuple(_arg(p, a) for p, a in zip(params, args)))
    return out


def _summary(r):
    if isinstance(r, np.ndarray):
        return (r.dtype.str, r.shape)
    if isinstance(r, (tuple, list)):
        return type(r)(_summary(x) for x in r)
    if r is None or isinstance(r, (bool, int, float, str)):
        return r
    return type(r).__name__


@pytest.fixture
def stub(monkeypatch):
    from scalablevectorsearch_b200 import _lib
    s = Stub()
    monkeypatch.setattr(_lib, "_lib", s)
    return s


def _run(stub, steps):
    """steps: (label, thunk, whether the getters it reads are part of its record) -> {label: (calls, result)}."""
    out = {}
    for label, thunk, getters in steps:
        stub.calls.clear()
        result = _summary(thunk())
        out[label] = (_calls(stub, getters), result)
    return out


def _rows(n=SIZE, dtype=np.float32):
    return np.arange(n * DIM, dtype=np.float32).reshape(n, DIM).astype(dtype)


def _queries(nq=3, dtype=np.float32):
    return np.ones((nq, DIM), dtype=dtype)


def _mask(n):
    return np.arange(n) % 2 == 0


def _handle_steps(box, key, dynamic):
    """The handle properties every index class has; a dynamic one's num_slots too."""
    steps = [(f"{key}.size", lambda: box[key].size, True),
             (f"{key}.dimensions", lambda: box[key].dimensions, True),
             (f"{key}.device_bytes", lambda: box[key].device_bytes, True)]
    if dynamic:
        steps.append((f"{key}.num_slots", lambda: box[key].num_slots, True))
    return steps


def _slot_steps(box, key):
    return [(f"{key}.has_id", lambda: box[key].has_id(7), False),
            (f"{key}.all_ids", lambda: box[key].all_ids(), False),
            (f"{key}.delete", lambda: box[key].delete([1, 2]), False),
            (f"{key}.add", lambda: box[key].add(_rows(2), [10, 11]), False),
            (f"{key}.add_reuse", lambda: box[key].add(_rows(2), [12, 13], reuse_empty=True), False)]


def _flat_steps(box, key, n_mask):
    ix = lambda: box[key]  # noqa: E731
    return [(f"{key}.num_threads", lambda: ix().num_threads, False),
            (f"{key}.search", lambda: ix().search(_queries(), 5), False),
            (f"{key}.search_device", lambda: ix().search_device(0x10, np.float16, 3, 5, 0x20, 0x30), False),
            (f"{key}.search_device_stream", lambda: ix().search_device(0x10, np.int8, 3, 5, 0x20, 0x30, 0x40), False),
            (f"{key}.search_filtered", lambda: ix().search_filtered(_queries(), 5, _mask(n_mask)), False),
            (f"{key}.search_filtered_counts",
             lambda: ix().search_filtered(_queries(dtype=np.uint8), 5, _mask(n_mask), with_counts=True), False),
            (f"{key}.search_filtered_device",
             lambda: ix().search_filtered_device(0x10, np.float32, 3, 5, 0x50, 0x20, 0x30), False),
            (f"{key}.search_filtered_device_stream",
             lambda: ix().search_filtered_device(0x10, np.uint8, 3, 5, 0x50, 0x20, 0x30, stream=0x40), False)]


def _ivf_steps(box, key, n_mask):
    from scalablevectorsearch_b200 import IVFSearchParameters
    ix = lambda: box[key]  # noqa: E731

    def probes():
        ix().search_parameters = IVFSearchParameters(n_probes=3, k_reorder=2.0)
    return [(f"{key}.num_clusters", lambda: ix().num_clusters, True),
            (f"{key}.cluster_sizes", lambda: ix().cluster_sizes, True),
            (f"{key}.centroids", lambda: ix().centroids, True),
            (f"{key}.search", lambda: ix().search(_queries(), 5), False),
            (f"{key}.set_probes", probes, False),
            (f"{key}.search_probes", lambda: ix().search(_queries(dtype=np.float16), 5), False),
            (f"{key}.search_device", lambda: ix().search_device(0x10, np.float16, 3, 5, 0x20, 0x30), False),
            (f"{key}.search_device_stream", lambda: ix().search_device(0x10, np.int8, 3, 5, 0x20, 0x30, 0x40), False),
            (f"{key}.search_filtered", lambda: ix().search_filtered(_queries(), 5, _mask(n_mask)), False),
            (f"{key}.search_filtered_counts",
             lambda: ix().search_filtered(_queries(), 5, _mask(n_mask), with_counts=True), False),
            (f"{key}.search_filtered_device",
             lambda: ix().search_filtered_device(0x10, np.float32, 3, 5, 0x50, 0x20, 0x30), False),
            (f"{key}.search_filtered_device_outs",
             lambda: ix().search_filtered_device(0x10, np.float32, 3, 5, 0x50, 0x20, 0x30, 0x60, 0x70, 0x80, 0x40),
             False)]


def _delete(box, key):
    def run():
        del box[key]
    return (f"del {key}", run, False)


def test_flat_bindings(stub):
    from scalablevectorsearch_b200 import DistanceType, DynamicFlat, Flat
    from scalablevectorsearch_b200.flat import filter_route
    box = {}
    steps = [("Flat", lambda: box.__setitem__("flat", Flat(_rows(), DistanceType.MIP, num_threads=3, device=1)), False)]
    steps += _handle_steps(box, "flat", False) + _flat_steps(box, "flat", SIZE) + [_delete(box, "flat")]
    steps += [("filter_route", lambda: filter_route(100, 7), False),
              ("DynamicFlat.build", lambda: box.__setitem__("dyn", DynamicFlat.build(
                  _rows(dtype=np.float16), np.arange(SIZE) + 100, DistanceType.Cosine, num_threads=2)), False)]
    steps += _handle_steps(box, "dyn", True) + _slot_steps(box, "dyn") + _flat_steps(box, "dyn", SLOTS)
    steps += [("dyn.consolidate", lambda: box["dyn"].consolidate(), False),
              ("dyn.compact", lambda: box["dyn"].compact(), False),
              ("dyn.export", lambda: box["dyn"].export(), False), _delete(box, "dyn")]
    assert _run(stub, steps) == FLAT


def test_ivf_bindings(stub):
    from scalablevectorsearch_b200 import IVF, Clustering, DistanceType, DynamicIVF, IVFBuildParameters, sq_compress
    box = {}
    bp = IVFBuildParameters(num_centroids=CLUSTERS, minibatch_size=64, num_iterations=3, training_fraction=0.5, seed=9)
    clustering = Clustering(np.zeros((CLUSTERS, DIM), np.float32), np.zeros(SIZE, np.uint32))
    unassigned = Clustering(np.zeros((CLUSTERS, DIM), np.float32))
    steps = [("Clustering.build", lambda: Clustering.build(bp, _rows(dtype=np.float16), DistanceType.MIP, device=1),
              False),
             ("Clustering.build.result", lambda: Clustering.build(bp, _rows()).centroids, False),
             ("sq_compress", lambda: sq_compress(_rows()), False),
             ("sq_compress_u8", lambda: sq_compress(_rows(), np.uint8, device=1), False),
             ("IVF", lambda: box.__setitem__("ivf", IVF.assemble_from_clustering(
                 clustering, _rows(), DistanceType.L2, device=1)), False)]
    steps += _handle_steps(box, "ivf", False) + _ivf_steps(box, "ivf", SIZE) + [_delete(box, "ivf")]
    steps += [("IVF_sq", lambda: box.__setitem__("ivf_sq", IVF.assemble_from_clustering(
                 unassigned, _rows(dtype=np.int8), DistanceType.MIP, sq=(0.5, -1.0))), False),
              ("ivf_sq.search", lambda: box["ivf_sq"].search(_queries(), 2), False), _delete(box, "ivf_sq"),
              ("DynamicIVF", lambda: box.__setitem__("dyn", DynamicIVF.assemble_from_clustering(
                  clustering, _rows(dtype=np.float16), np.arange(SIZE) + 100, DistanceType.Cosine, num_threads=2,
                  intra_query_threads=3, device=1)), False),
              ("dyn.threads", lambda: (box["dyn"].num_threads, box["dyn"].intra_query_threads), False)]
    steps += _handle_steps(box, "dyn", True) + _slot_steps(box, "dyn") + _ivf_steps(box, "dyn", SLOTS)
    steps += [("dyn.add_f32_to_f16", lambda: box["dyn"].add(_rows(1), [20]), False),
              ("dyn.consolidate", lambda: box["dyn"].consolidate(), False),
              ("dyn.compact", lambda: box["dyn"].compact(), False),
              ("dyn.export", lambda: box["dyn"].export(), False), _delete(box, "dyn"),
              ("DynamicIVF_sq", lambda: box.__setitem__("dyn_sq", DynamicIVF.assemble_from_clustering(
                  unassigned, _rows(0, np.uint8), [], DistanceType.L2, sq=(0.25, 3.0))), False),
              ("dyn_sq.search", lambda: box["dyn_sq"].search(_queries(1), 1), False), _delete(box, "dyn_sq")]
    assert _run(stub, steps) == IVF_TABLE


def _vamana_steps(box, key):
    from scalablevectorsearch_b200 import SearchBufferConfig
    ix = lambda: box[key]  # noqa: E731

    def window():
        ix().search_parameters.buffer_config = SearchBufferConfig(16, 24)
        ix().search_parameters.search_buffer_visited_set = True
        return ix().search_window_size
    return [(f"{key}.graph_max_degree", lambda: ix().graph_max_degree, True),
            (f"{key}.num_devices", lambda: ix().num_devices, True),
            (f"{key}.num_threads", lambda: ix().num_threads, False),
            (f"{key}.search", lambda: ix().search(_queries(), 5), False),
            (f"{key}.window", window, False),
            (f"{key}.search_window", lambda: ix().search(_queries(), 5), False),
            (f"{key}.search_cancel", lambda: ix().search(_queries(), 5, cancel=lambda: False), False),
            (f"{key}.search_device", lambda: ix().search_device(0x10, np.float32, 3, 5, 0x20, 0x30), False),
            (f"{key}.search_device_ids4",
             lambda: ix().search_device(0x10, np.float16, 3, 5, 0x20, 0x30, stream=0x40, id_bytes=4), False),
            (f"{key}.exhaustive_device", lambda: ix().exhaustive_device(0x10, np.float32, 3, 5, 0x20, 0x30), False),
            (f"{key}.search_filtered", lambda: ix().search_filtered(_queries(), 5, _mask(SIZE)), False),
            (f"{key}.range_search", lambda: ix().range_search(_queries(), 0.5), False),
            (f"{key}.flat_search", lambda: ix().flat_search(_queries(), 5), False),
            (f"{key}.flat_search_device", lambda: ix().flat_search_device(0x10, np.float32, 3, 5, 0x20, 0x30), False),
            (f"{key}.set_counting", lambda: ix().set_counting(True), False),
            (f"{key}.counters", lambda: ix().counters(3), False),
            (f"{key}.fetched", lambda: ix().fetched(3), False),
            (f"{key}.last_kernel_ms", lambda: ix().last_kernel_ms(), False),
            (f"{key}.set_entry_points", lambda: ix().set_entry_points([0, 2]), False),
            (f"{key}.set_option", lambda: ix().set_option("lean", 1), False),
            (f"{key}.get_option", lambda: ix().get_option("lean"), False)]


def test_vamana_bindings(stub):
    from scalablevectorsearch_b200 import (DistanceType, ShardedVamana, Vamana, VamanaBuildParameters, build_graph,
                                           lvq8_compress)
    box = {}
    graph = np.zeros((SIZE, MAX_DEGREE + 1), np.uint32)
    bp = VamanaBuildParameters(alpha=1.2, graph_max_degree=MAX_DEGREE, window_size=20, max_candidate_pool_size=30,
                               prune_to=2)
    steps = [("build_graph", lambda: build_graph(_rows(), DistanceType.MIP, bp, device=1), False),
             ("build_graph_sq", lambda: build_graph(_rows(dtype=np.uint8), DistanceType.L2, bp, sq=(0.5, 2.0)), False),
             ("lvq8_compress", lambda: lvq8_compress(_rows()), False),
             ("lvq8_compress_mean", lambda: lvq8_compress(_rows(), np.ones(DIM), device=1), False),
             ("Vamana.from_arrays", lambda: box.__setitem__("v", Vamana.from_arrays(
                 _rows(), graph, 2, DistanceType.MIP, device=[0, 1], num_threads=4)), False)]
    steps += _handle_steps(box, "v", False) + _vamana_steps(box, "v") + [_delete(box, "v")]
    steps += [("Vamana.from_arrays_sq", lambda: box.__setitem__("vsq", Vamana.from_arrays(
                 _rows(dtype=np.int8), graph, 1, sq=(0.5, -2.0))), False),
              ("vsq.search", lambda: box["vsq"].search(_queries(), 2), False), _delete(box, "vsq"),
              ("Vamana.from_arrays_lvq8", lambda: box.__setitem__("vlvq", Vamana.from_arrays(
                  np.zeros((SIZE, LVQ_STRIDE), np.uint8), graph, 0, lvq8=(DIM, np.ones(DIM)))), False),
              _delete(box, "vlvq"),
              ("Vamana.build", lambda: box.__setitem__("vb", Vamana.build(bp, _rows(), DistanceType.L2)), False),
              ("vb.build_parameters", lambda: box["vb"].build_parameters.window_size, False), _delete(box, "vb"),
              ("ShardedVamana", lambda: box.__setitem__("sh", ShardedVamana(
                  [Vamana.from_arrays(_rows(), graph, 0), Vamana.from_arrays(_rows(), graph, 1)], [0, SIZE])), False),
              ("sh.size", lambda: box["sh"].size, True),
              ("sh.search", lambda: box["sh"].search(_queries(), 5), False), _delete(box, "sh")]
    assert _run(stub, steps) == VAMANA


def test_dynamic_vamana_bindings(stub):
    from scalablevectorsearch_b200 import DistanceType, DynamicVamana, VamanaBuildParameters
    box = {}
    graph = np.zeros((SIZE, MAX_DEGREE + 1), np.uint32)
    bp = VamanaBuildParameters(alpha=1.2, graph_max_degree=MAX_DEGREE, window_size=20, max_candidate_pool_size=30,
                               prune_to=2)
    steps = [("DynamicVamana.from_arrays", lambda: box.__setitem__("d", DynamicVamana.from_arrays(
                 _rows(dtype=np.float16), graph, 3, np.arange(SIZE) + 100, DistanceType.MIP, device=1)), False)]
    steps += _handle_steps(box, "d", True) + _slot_steps(box, "d") + _vamana_steps(box, "d")
    steps += [("d.consolidate", lambda: box["d"].consolidate(), False),
              ("d.compact", lambda: box["d"].compact(), False),
              ("d.export", lambda: box["d"].export(), False),
              ("d.alpha", lambda: box["d"].alpha, False),
              ("d.set_window", lambda: setattr(box["d"], "construction_window_size", 40), False),
              ("d.mutation_parameters", lambda: (box["d"].construction_window_size, box["d"].max_candidates,
                                                 box["d"].prune_to), False),
              _delete(box, "d"),
              ("DynamicVamana.build", lambda: box.__setitem__("db", DynamicVamana.build(
                  bp, _rows(), None, DistanceType.Cosine, device=1, num_threads=2)), False),
              ("db.search", lambda: box["db"].search(_queries(), 2), False), _delete(box, "db")]
    assert _run(stub, steps) == DYNAMIC_VAMANA


_BAD_QUERIES = {"narrow": (np.ones((3, DIM - 1), np.float32), ValueError),
                "1-D": (np.ones(DIM, np.float32), ValueError),
                "float64": (np.ones((3, DIM), np.float64), TypeError)}


@pytest.mark.parametrize("bad", sorted(_BAD_QUERIES))
@pytest.mark.parametrize("form", ["search_filtered", "range_search", "flat_search", "sharded"])
def test_host_searches_refuse_bad_queries_before_the_call(stub, form, bad):
    """Queries of the wrong width, rank or type never reach the C search (which reads nq x dimensions elements)."""
    from scalablevectorsearch_b200 import ShardedVamana, Vamana
    graph = np.zeros((SIZE, MAX_DEGREE + 1), np.uint32)
    index = Vamana.from_arrays(_rows(), graph, 0)
    queries, error = _BAD_QUERIES[bad]
    call = {"search_filtered": lambda: index.search_filtered(queries, 5, _mask(SIZE)),
            "range_search": lambda: index.range_search(queries, 0.5),
            "flat_search": lambda: index.flat_search(queries, 5),
            "sharded": lambda: ShardedVamana([index], [0]).search(queries, 5)}[form]
    stub.calls.clear()
    with pytest.raises(error):
        call()
    assert _calls(stub, False) == [("svsb200_set_id_offset", "p", 0)] * (form == "sharded")


def test_range_search_of_an_empty_batch(stub):
    from scalablevectorsearch_b200 import Vamana
    index = Vamana.from_arrays(_rows(), np.zeros((SIZE, MAX_DEGREE + 1), np.uint32), 0)
    assert index.range_search(np.ones((0, DIM), np.float32), 0.5) == []


# ---- the recorded tables ---------------------------------------------------------------------------------------
FLAT = {
    "Flat": ([("svsb200_flat_index_create", "p", 0, 6, 4, 0, 1, 1, "p")], None),
    "flat.size": ([("svsb200_flat_index_size", "p")], 6),
    "flat.dimensions": ([("svsb200_flat_index_dimensions", "p")], 4),
    "flat.device_bytes": ([("svsb200_flat_index_device_bytes", "p")], 4096),
    "flat.num_threads": ([], 3),
    "flat.search": ([("svsb200_flat_index_search", "p", "p", 0, 3, 5, "p", "p")], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "flat.search_device": ([("svsb200_flat_index_search_device", "p", "p", 1, 3, 5, "p", "p", None, "p")], 0),
    "flat.search_device_stream": ([("svsb200_flat_index_search_device", "p", "p", 2, 3, 5, "p", "p", "p", "p")], 0),
    "flat.search_filtered": ([
        ("svsb200_flat_index_search_filtered", "p", "p", 0, 3, 5, "p", "p", "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)), ("<u4", (3,)))),
    "flat.search_filtered_counts": ([
        ("svsb200_flat_index_search_filtered", "p", "p", 3, 3, 5, "p", "p", "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)), ("<u4", (3,)), 0)),
    "flat.search_filtered_device": ([
        ("svsb200_flat_index_search_filtered_device", "p", "p", 0, 3, 5, "p", "p", "p", None, None, "p"),
    ], 0),
    "flat.search_filtered_device_stream": ([
        ("svsb200_flat_index_search_filtered_device", "p", "p", 3, 3, 5, "p", "p", "p", "p", None, "p"),
    ], 0),
    "del flat": ([("svsb200_flat_index_destroy", "p")], None),
    "filter_route": ([("svsb200_flat_filter_plan", 100, 7, "p")], "dense"),
    "DynamicFlat.build": ([("svsb200_dynamic_flat_create", "p", 1, 6, 4, 2, "p", 0, "p")], None),
    "dyn.size": ([("svsb200_dynamic_flat_size", "p")], 6),
    "dyn.dimensions": ([("svsb200_dynamic_flat_dimensions", "p")], 4),
    "dyn.device_bytes": ([("svsb200_dynamic_flat_device_bytes", "p")], 4096),
    "dyn.num_slots": ([("svsb200_dynamic_flat_num_slots", "p")], 8),
    "dyn.has_id": ([("svsb200_dynamic_flat_has_id", "p", 7, "p")], False),
    "dyn.all_ids": ([("svsb200_dynamic_flat_ids", "p", "p", "p")], ("<u8", (6,))),
    "dyn.delete": ([("svsb200_dynamic_flat_delete", "p", "p", 2)], 2),
    "dyn.add": ([("svsb200_dynamic_flat_add", "p", "p", 0, 2, "p", 0, "p")], ("<u8", (2,))),
    "dyn.add_reuse": ([("svsb200_dynamic_flat_add", "p", "p", 0, 2, "p", 1, "p")], ("<u8", (2,))),
    "dyn.num_threads": ([], 2),
    "dyn.search": ([
        ("svsb200_dynamic_flat_search", "p", "p", 0, 3, 5, "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "dyn.search_device": ([("svsb200_dynamic_flat_search_device", "p", "p", 1, 3, 5, "p", "p", None, "p")], 0),
    "dyn.search_device_stream": ([("svsb200_dynamic_flat_search_device", "p", "p", 2, 3, 5, "p", "p", "p", "p")], 0),
    "dyn.search_filtered": ([
        ("svsb200_dynamic_flat_search_filtered", "p", "p", 0, 3, 5, "p", "p", "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)), ("<u4", (3,)))),
    "dyn.search_filtered_counts": ([
        ("svsb200_dynamic_flat_search_filtered", "p", "p", 3, 3, 5, "p", "p", "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)), ("<u4", (3,)), 0)),
    "dyn.search_filtered_device": ([
        ("svsb200_dynamic_flat_search_filtered_device", "p", "p", 0, 3, 5, "p", "p", "p", None, None, "p"),
    ], 0),
    "dyn.search_filtered_device_stream": ([
        ("svsb200_dynamic_flat_search_filtered_device", "p", "p", 3, 3, 5, "p", "p", "p", "p", None, "p"),
    ], 0),
    "dyn.consolidate": ([], None),
    "dyn.compact": ([("svsb200_dynamic_flat_compact", "p")], None),
    "dyn.export": ([("svsb200_dynamic_flat_export", "p", "p", "p")], (("|u1", (8,)), ("<u8", (8,)))),
    "del dyn": ([("svsb200_dynamic_flat_destroy", "p")], None),
}

IVF_TABLE = {
    "Clustering.build": ([("svsb200_ivf_cluster", "p", 1, 6, 4, 1, 2, 64, 3, 0, 0.5, 9, 1, "p", "p")], "Clustering"),
    "Clustering.build.result": ([
        ("svsb200_ivf_cluster", "p", 0, 6, 4, 0, 2, 64, 3, 0, 0.5, 9, 0, "p", "p"),
    ], ("<f4", (2, 4))),
    "sq_compress": ([("svsb200_sq_compress", "p", 6, 4, 2, 0, "p", "p", "p")], (("|i1", (6, 4)), 0.0, 0.0)),
    "sq_compress_u8": ([("svsb200_sq_compress", "p", 6, 4, 3, 1, "p", "p", "p")], (("|u1", (6, 4)), 0.0, 0.0)),
    "IVF": ([("svsb200_ivf_create", "p", 0, 6, 4, 0, "p", 2, "p", 1, "p")], None),
    "ivf.size": ([("svsb200_ivf_size", "p")], 6),
    "ivf.dimensions": ([("svsb200_ivf_dimensions", "p")], 4),
    "ivf.device_bytes": ([("svsb200_ivf_device_bytes", "p")], 4096),
    "ivf.num_clusters": ([("svsb200_ivf_num_clusters", "p")], 2),
    "ivf.cluster_sizes": ([
        ("svsb200_ivf_num_clusters", "p"),
        ("svsb200_ivf_cluster_sizes", "p", "p"),
    ], ("<u4", (2,))),
    "ivf.centroids": ([
        ("svsb200_ivf_num_clusters", "p"),
        ("svsb200_ivf_dimensions", "p"),
        ("svsb200_ivf_centroids", "p", "p"),
    ], ("<f4", (2, 4))),
    "ivf.search": ([("svsb200_ivf_search", "p", "p", 0, 3, 5, 1, "p", "p")], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "ivf.set_probes": ([], None),
    "ivf.search_probes": ([
        ("svsb200_ivf_search", "p", "p", 1, 3, 5, 3, "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "ivf.search_device": ([("svsb200_ivf_search_device", "p", "p", 1, 3, 5, 3, "p", "p", None)], None),
    "ivf.search_device_stream": ([("svsb200_ivf_search_device", "p", "p", 2, 3, 5, 3, "p", "p", "p")], None),
    "ivf.search_filtered": ([
        ("svsb200_ivf_search_filtered", "p", "p", 0, 3, 5, 3, "p", "p", "p", "p", "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)), ("<u4", (3,)))),
    "ivf.search_filtered_counts": ([
        ("svsb200_ivf_search_filtered", "p", "p", 0, 3, 5, 3, "p", "p", "p", "p", "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)), ("<u4", (3,)), (("<u4", (3,)), ("<u4", (3,)), ("<u4", (3,))))),
    "ivf.search_filtered_device": ([
        ("svsb200_ivf_search_filtered_device", "p", "p", 0, 3, 5, 3, "p", "p", "p", None, None, None, None),
    ], None),
    "ivf.search_filtered_device_outs": ([
        ("svsb200_ivf_search_filtered_device", "p", "p", 0, 3, 5, 3, "p", "p", "p", "p", "p", "p", "p"),
    ], None),
    "del ivf": ([("svsb200_ivf_destroy", "p")], None),
    "IVF_sq": ([("svsb200_ivf_create_sq", "p", 2, 6, 4, 1, 0.5, -1.0, "p", 2, None, 0, "p")], None),
    "ivf_sq.search": ([("svsb200_ivf_search", "p", "p", 0, 3, 2, 1, "p", "p")], (("<u8", (3, 2)), ("<f4", (3, 2)))),
    "del ivf_sq": ([("svsb200_ivf_destroy", "p")], None),
    "DynamicIVF": ([("svsb200_dynamic_ivf_create", "p", 1, 6, 4, 2, "p", 2, "p", "p", 1, "p")], None),
    "dyn.threads": ([], (2, 3)),
    "dyn.size": ([("svsb200_dynamic_ivf_size", "p")], 6),
    "dyn.dimensions": ([("svsb200_dynamic_ivf_dimensions", "p")], 4),
    "dyn.device_bytes": ([("svsb200_dynamic_ivf_device_bytes", "p")], 4096),
    "dyn.num_slots": ([("svsb200_dynamic_ivf_num_slots", "p")], 8),
    "dyn.has_id": ([("svsb200_dynamic_ivf_has_id", "p", 7, "p")], False),
    "dyn.all_ids": ([("svsb200_dynamic_ivf_ids", "p", "p", "p")], ("<u8", (6,))),
    "dyn.delete": ([("svsb200_dynamic_ivf_delete", "p", "p", 2)], 2),
    "dyn.add": ([("svsb200_dynamic_ivf_add", "p", "p", 1, 2, "p", 0, "p")], ("<u8", (2,))),
    "dyn.add_reuse": ([("svsb200_dynamic_ivf_add", "p", "p", 1, 2, "p", 1, "p")], ("<u8", (2,))),
    "dyn.num_clusters": ([("svsb200_dynamic_ivf_num_clusters", "p")], 2),
    "dyn.cluster_sizes": ([
        ("svsb200_dynamic_ivf_num_clusters", "p"),
        ("svsb200_dynamic_ivf_cluster_sizes", "p", "p"),
    ], ("<u4", (2,))),
    "dyn.centroids": ([
        ("svsb200_dynamic_ivf_num_clusters", "p"),
        ("svsb200_dynamic_ivf_dimensions", "p"),
        ("svsb200_dynamic_ivf_centroids", "p", "p"),
    ], ("<f4", (2, 4))),
    "dyn.search": ([
        ("svsb200_dynamic_ivf_search", "p", "p", 0, 3, 5, 1, "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "dyn.set_probes": ([], None),
    "dyn.search_probes": ([
        ("svsb200_dynamic_ivf_search", "p", "p", 1, 3, 5, 3, "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "dyn.search_device": ([("svsb200_dynamic_ivf_search_device", "p", "p", 1, 3, 5, 3, "p", "p", None)], None),
    "dyn.search_device_stream": ([("svsb200_dynamic_ivf_search_device", "p", "p", 2, 3, 5, 3, "p", "p", "p")], None),
    "dyn.search_filtered": ([
        ("svsb200_dynamic_ivf_search_filtered", "p", "p", 0, 3, 5, 3, "p", "p", "p", "p", "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)), ("<u4", (3,)))),
    "dyn.search_filtered_counts": ([
        ("svsb200_dynamic_ivf_search_filtered", "p", "p", 0, 3, 5, 3, "p", "p", "p", "p", "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)), ("<u4", (3,)), (("<u4", (3,)), ("<u4", (3,)), ("<u4", (3,))))),
    "dyn.search_filtered_device": ([
        ("svsb200_dynamic_ivf_search_filtered_device", "p", "p", 0, 3, 5, 3, "p", "p", "p", None, None, None, None),
    ], None),
    "dyn.search_filtered_device_outs": ([
        ("svsb200_dynamic_ivf_search_filtered_device", "p", "p", 0, 3, 5, 3, "p", "p", "p", "p", "p", "p", "p"),
    ], None),
    "dyn.add_f32_to_f16": ([("svsb200_dynamic_ivf_add", "p", "p", 1, 1, "p", 0, "p")], ("<u8", (1,))),
    "dyn.consolidate": ([], None),
    "dyn.compact": ([("svsb200_dynamic_ivf_compact", "p")], None),
    "dyn.export": ([
        ("svsb200_dynamic_ivf_export", "p", "p", "p", "p"),
    ], (("|u1", (8,)), ("<u8", (8,)), ("<u4", (8,)))),
    "del dyn": ([("svsb200_dynamic_ivf_destroy", "p")], None),
    "DynamicIVF_sq": ([
        ("svsb200_dynamic_ivf_create_sq", "p", 3, 0, 4, 0, 0.25, 3.0, "p", 2, None, "p", 0, "p"),
    ], None),
    "dyn_sq.search": ([
        ("svsb200_dynamic_ivf_search", "p", "p", 0, 1, 1, 1, "p", "p"),
    ], (("<u8", (1, 1)), ("<f4", (1, 1)))),
    "del dyn_sq": ([("svsb200_dynamic_ivf_destroy", "p")], None),
}

VAMANA = {
    "build_graph": ([
        ("svsb200_build_vamana", "p", 0, 6, 4, 0, 1, 1.2, 3, 20, 30, 2, 1, "p", "p"),
    ], (("<u4", (6, 4)), 0)),
    "build_graph_sq": ([
        ("svsb200_build_vamana_sq", "p", 3, 6, 4, 0, 0.5, 2.0, 1.2, 3, 20, 30, 2, 0, "p", "p"),
    ], (("<u4", (6, 4)), 0)),
    "lvq8_compress": ([
        ("svsb200_lvq8_row_stride", 4),
        ("svsb200_lvq8_compress", "p", 6, 4, "p", "p", 0),
    ], (("|u1", (6, 12)), ("<f4", (4,)))),
    "lvq8_compress_mean": ([
        ("svsb200_lvq8_row_stride", 4),
        ("svsb200_lvq8_compress", "p", 6, 4, "p", "p", 1),
    ], (("|u1", (6, 12)), ("<f4", (4,)))),
    "Vamana.from_arrays": ([
        ("svsb200_index_create_multi", "p", 0, 6, 4, 0, "p", 4, 2, 1, 0, None, "p", 2, "p"),
    ], None),
    "v.size": ([("svsb200_index_size", "p")], 6),
    "v.dimensions": ([("svsb200_index_dimensions", "p")], 4),
    "v.device_bytes": ([("svsb200_index_device_bytes", "p")], 4096),
    "v.graph_max_degree": ([("svsb200_index_max_degree", "p")], 3),
    "v.num_devices": ([("svsb200_index_num_devices", "p")], 1),
    "v.num_threads": ([], 4),
    "v.search": ([
        ("svsb200_search", "p", "p", 0, 3, 5, 0, 0, 0, "p", 8, "p", None),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "v.window": ([], 16),
    "v.search_window": ([
        ("svsb200_search", "p", "p", 0, 3, 5, 16, 24, 1, "p", 8, "p", None),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "v.search_cancel": ([
        ("svsb200_search_cancellable", "p", "p", 0, 3, 5, 16, 24, 1, "p", 8, "p", None, "p", None),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "v.search_device": ([("svsb200_search_device", "p", "p", 0, 3, 5, 16, 24, 1, "p", 8, "p", None)], None),
    "v.search_device_ids4": ([("svsb200_search_device", "p", "p", 1, 3, 5, 16, 24, 1, "p", 4, "p", "p")], None),
    "v.exhaustive_device": ([("svsb200_exhaustive_device", "p", "p", 0, 3, 5, "p", "p", None)], None),
    "v.search_filtered": ([
        ("svsb200_search_filtered", "p", "p", 0, 3, 5, 16, "p", "p", "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)), ("<u4", (3,)))),
    "v.range_search": ([
        ("svsb200_range_search", "p", "p", 0, 3, 0.5, 16, "p", "p", "p"),
        ("svsb200_free", "p"),
        ("svsb200_free", "p"),
    ], [(("<u8", (2,)), ("<f4", (2,))), (("<u8", (0,)), ("<f4", (0,))), (("<u8", (1,)), ("<f4", (1,)))]),
    "v.flat_search": ([("svsb200_flat_search", "p", "p", 0, 3, 5, "p", "p")], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "v.flat_search_device": ([("svsb200_flat_search_device", "p", "p", 0, 3, 5, "p", "p", None, "p")], 0),
    "v.set_counting": ([("svsb200_set_counting", "p", 1)], None),
    "v.counters": ([("svsb200_get_counters", "p", 3, "p", "p")], (("<u4", (3,)), ("<u4", (3,)))),
    "v.fetched": ([("svsb200_get_fetched", "p", 3, "p")], ("<u4", (3,))),
    "v.last_kernel_ms": ([("svsb200_last_kernel_ms", "p", "p")], 0.0),
    "v.set_entry_points": ([("svsb200_set_entry_points", "p", "p", 2)], None),
    "v.set_option": ([("svsb200_set_option", "p", b"lean", 1)], None),
    "v.get_option": ([("svsb200_get_option", "p", b"lean", "p")], 0),
    "del v": ([("svsb200_index_destroy", "p")], None),
    "Vamana.from_arrays_sq": ([
        ("svsb200_index_create_multi", "p", 2, 6, 4, 0, "p", 4, 1, 0, 1, "p", "p", 1, "p"),
    ], None),
    "vsq.search": ([
        ("svsb200_search", "p", "p", 0, 3, 2, 0, 0, 0, "p", 8, "p", None),
    ], (("<u8", (3, 2)), ("<f4", (3, 2)))),
    "del vsq": ([("svsb200_index_destroy", "p")], None),
    "Vamana.from_arrays_lvq8": ([
        ("svsb200_index_create_multi", "p", 3, 6, 4, 12, "p", 4, 0, 0, 2, "p", "p", 1, "p"),
    ], None),
    "del vlvq": ([("svsb200_index_destroy", "p")], None),
    "Vamana.build": ([
        ("svsb200_build_vamana", "p", 0, 6, 4, 0, 0, 1.2, 3, 20, 30, 2, 0, "p", "p"),
        ("svsb200_index_create_multi", "p", 0, 6, 4, 0, "p", 4, 0, 0, 0, None, "p", 1, "p"),
    ], None),
    "vb.build_parameters": ([], 20),
    "del vb": ([("svsb200_index_destroy", "p")], None),
    "ShardedVamana": ([
        ("svsb200_index_create_multi", "p", 0, 6, 4, 0, "p", 4, 0, 0, 0, None, "p", 1, "p"),
        ("svsb200_index_create_multi", "p", 0, 6, 4, 0, "p", 4, 1, 0, 0, None, "p", 1, "p"),
        ("svsb200_set_id_offset", "p", 0),
        ("svsb200_set_id_offset", "p", 6),
    ], None),
    "sh.size": ([("svsb200_index_size", "p"), ("svsb200_index_size", "p")], 12),
    "sh.search": ([
        ("svsb200_search_sharded", "p", 2, "p", 0, 3, 5, 0, 0, "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "del sh": ([("svsb200_index_destroy", "p"), ("svsb200_index_destroy", "p")], None),
}

DYNAMIC_VAMANA = {
    "DynamicVamana.from_arrays": ([("svsb200_dynamic_create", "p", 1, 6, 4, "p", 4, 3, 1, "p", 1, "p")], None),
    "d.size": ([("svsb200_dynamic_ids", "p", None, "p")], 0),
    "d.dimensions": ([("svsb200_index_dimensions", "p")], 4),
    "d.device_bytes": ([("svsb200_index_device_bytes", "p")], 4096),
    "d.num_slots": ([("svsb200_index_size", "p")], 6),
    "d.has_id": ([("svsb200_dynamic_has_id", "p", 7, "p")], False),
    "d.all_ids": ([("svsb200_dynamic_ids", "p", None, "p"), ("svsb200_dynamic_ids", "p", "p", "p")], ("<u8", (0,))),
    "d.delete": ([("svsb200_dynamic_delete", "p", "p", 2)], 2),
    "d.add": ([("svsb200_dynamic_add", "p", "p", 0, 2, "p", 0, "p")], ("<u8", (2,))),
    "d.add_reuse": ([("svsb200_dynamic_add", "p", "p", 0, 2, "p", 1, "p")], ("<u8", (2,))),
    "d.graph_max_degree": ([("svsb200_index_max_degree", "p")], 3),
    "d.num_devices": ([("svsb200_index_num_devices", "p")], 1),
    "d.num_threads": ([], 1),
    "d.search": ([
        ("svsb200_search", "p", "p", 0, 3, 5, 0, 0, 0, "p", 8, "p", None),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "d.window": ([], 16),
    "d.search_window": ([
        ("svsb200_search", "p", "p", 0, 3, 5, 16, 24, 1, "p", 8, "p", None),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "d.search_cancel": ([
        ("svsb200_search_cancellable", "p", "p", 0, 3, 5, 16, 24, 1, "p", 8, "p", None, "p", None),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "d.search_device": ([("svsb200_search_device", "p", "p", 0, 3, 5, 16, 24, 1, "p", 8, "p", None)], None),
    "d.search_device_ids4": ([("svsb200_search_device", "p", "p", 1, 3, 5, 16, 24, 1, "p", 4, "p", "p")], None),
    "d.exhaustive_device": ([("svsb200_exhaustive_device", "p", "p", 0, 3, 5, "p", "p", None)], None),
    "d.search_filtered": ([
        ("svsb200_search_filtered", "p", "p", 0, 3, 5, 16, "p", "p", "p", "p"),
    ], (("<u8", (3, 5)), ("<f4", (3, 5)), ("<u4", (3,)))),
    "d.range_search": ([
        ("svsb200_range_search", "p", "p", 0, 3, 0.5, 16, "p", "p", "p"),
        ("svsb200_free", "p"),
        ("svsb200_free", "p"),
    ], [(("<u8", (2,)), ("<f4", (2,))), (("<u8", (0,)), ("<f4", (0,))), (("<u8", (1,)), ("<f4", (1,)))]),
    "d.flat_search": ([("svsb200_flat_search", "p", "p", 0, 3, 5, "p", "p")], (("<u8", (3, 5)), ("<f4", (3, 5)))),
    "d.flat_search_device": ([("svsb200_flat_search_device", "p", "p", 0, 3, 5, "p", "p", None, "p")], 0),
    "d.set_counting": ([("svsb200_set_counting", "p", 1)], None),
    "d.counters": ([("svsb200_get_counters", "p", 3, "p", "p")], (("<u4", (3,)), ("<u4", (3,)))),
    "d.fetched": ([("svsb200_get_fetched", "p", 3, "p")], ("<u4", (3,))),
    "d.last_kernel_ms": ([("svsb200_last_kernel_ms", "p", "p")], 0.0),
    "d.set_entry_points": ([("svsb200_set_entry_points", "p", "p", 2)], None),
    "d.set_option": ([("svsb200_set_option", "p", b"lean", 1)], None),
    "d.get_option": ([("svsb200_get_option", "p", b"lean", "p")], 0),
    "d.consolidate": ([("svsb200_dynamic_consolidate", "p")], None),
    "d.compact": ([("svsb200_dynamic_compact", "p")], None),
    "d.export": ([
        ("svsb200_dynamic_export", "p", "p", "p", "p", "p"),
    ], (("<u4", (6, 4)), ("|u1", (6,)), ("<u8", (6,)), 0)),
    "d.alpha": ([("svsb200_dynamic_get_build_parameters", "p", "p", "p", "p", "p")], 0.0),
    "d.set_window": ([
        ("svsb200_dynamic_get_build_parameters", "p", "p", "p", "p", "p"),
        ("svsb200_dynamic_set_build_parameters", "p", 0.0, 40, 0, 0),
    ], None),
    "d.mutation_parameters": ([
        ("svsb200_dynamic_get_build_parameters", "p", "p", "p", "p", "p"),
        ("svsb200_dynamic_get_build_parameters", "p", "p", "p", "p", "p"),
        ("svsb200_dynamic_get_build_parameters", "p", "p", "p", "p", "p"),
    ], (0, 0, 0)),
    "del d": ([("svsb200_index_destroy", "p")], None),
    "DynamicVamana.build": ([("svsb200_dynamic_build", "p", 0, 6, 4, 2, 1.2, 3, 20, 30, 2, "p", 1, "p")], None),
    "db.search": ([
        ("svsb200_search", "p", "p", 0, 3, 2, 0, 0, 0, "p", 8, "p", None),
    ], (("<u8", (3, 2)), ("<f4", (3, 2)))),
    "del db": ([("svsb200_index_destroy", "p")], None),
}
