"""Every IVF leaf and k-means kernel shape the dispatch can choose (svsb200_ivf_plan, svsb200_ivf_group_plan), each case:
the plan it means to hit asserted first; ids and distance bits against the models (tests/ivf_model.py, ivf_sq_model.py,
the dynamic models, hier_kmeans_model.py); the exact scan at n_probes = C; and the float64 layer (tests/float64_layer.py):
every distance within its rounding bound of float64 (SQ L2 exact), no probed row left out that float64 says is nearer
than the k-th returned one beyond a near tie, and every k-means assignment the float64-nearest centroid up to a near tie.

Rows stay few at wide dimensions: the cases spend their time on shapes, not sizes."""
import ctypes as C

import numpy as np
import pytest

import dynamic_ivf_model as DM
import dynamic_ivf_sq_model as DSM
import float64_layer as F64
import hier_kmeans_model as H
import ivf_model as M
import ivf_sq_model as SM
from conftest import bits
from scalablevectorsearch_b200 import (IVF, Clustering, DistanceType, DynamicIVF, IVFBuildParameters,
                                       IVFSearchParameters, Svsb200Error, Vamana, _lib)

pytestmark = pytest.mark.gpu
DIST = {0: DistanceType.L2, 1: DistanceType.MIP, 2: DistanceType.Cosine}
NAME = {0: "l2", 1: "ip", 2: "cosine"}
CODE = {np.dtype(np.float32): 0, np.dtype(np.float16): 1, np.dtype(np.int8): 2, np.dtype(np.uint8): 3}


def ivf_plan(dim, dtype, metric, k, n_probes=1, nq=1, dynamic=False, sq=False):
    """(tile_rows, Q, ctas per SM, query chunk, leaf, static dim, rows per pass, smem bytes) of svsb200_ivf_plan."""
    out = [C.c_uint32() for _ in range(7)] + [C.c_uint64()]
    _lib.check(_lib.lib().svsb200_ivf_plan(dim, CODE[np.dtype(dtype)], int(sq), metric, k, n_probes, nq, int(dynamic),
                                           *[C.byref(o) for o in out]))
    return tuple(o.value for o in out)


def group_tile(dim):
    out = [C.c_uint32(), C.c_uint32(), C.c_uint64()]
    _lib.check(_lib.lib().svsb200_ivf_group_plan(dim, *[C.byref(o) for o in out]))
    return out[0].value


def f16(x):
    """float16 with subnormals flushed, so that every preparation (flushing or not) sees the same values."""
    h = np.asarray(x, dtype=np.float32).astype(np.float16)
    h[np.abs(h) < np.float16(2.0 ** -14)] = 0
    return h


def rows_of(rng, n, dim, dtype, centres):
    c = rng.standard_normal((centres, dim)).astype(np.float32)
    x = c[rng.integers(0, centres, n)] + 0.4 * rng.standard_normal((n, dim)).astype(np.float32)
    return f16(x) if dtype == np.float16 else x.astype(np.float32)


def layout(rng, n, sizes, C):
    """Assignments with the first clusters of exactly `sizes` rows and the rest spread over the other clusters."""
    a = np.empty(n, dtype=np.uint32)
    perm = rng.permutation(n)
    pos = 0
    for c, s in enumerate(sizes):
        a[perm[pos:pos + s]] = c
        pos += s
    a[perm[pos:]] = len(sizes) + rng.integers(0, C - len(sizes), n - pos)
    return a


def centroids_of(x, a, C, rng):
    cent = rng.standard_normal((C, x.shape[1])).astype(np.float32)
    for c in range(C):
        m = a == c
        if m.any():
            cent[c] = x[m].astype(np.float32).mean(0)
    return cent


def same(got, want, tag):
    gi, gd = got
    wi, wd = want
    assert np.array_equal(gi, wi), f"{tag}: ids differ in queries {np.flatnonzero((gi != wi).any(1))[:10]}"
    assert np.array_equal(bits(gd), bits(wd)), f"{tag}: distance bits differ"


def scan(rows, metric, q, k, sq=None):
    import torch
    v = Vamana.from_arrays(rows, np.zeros((rows.shape[0], 2), dtype=np.uint32), 0, DIST[metric], sq=sq)
    dq = torch.from_numpy(np.ascontiguousarray(q)).cuda()
    ids = torch.empty((q.shape[0], k), dtype=torch.int64, device="cuda")
    d = torch.empty((q.shape[0], k), dtype=torch.float32, device="cuda")
    v.exhaustive_device(dq.data_ptr(), q.dtype, q.shape[0], k, ids.data_ptr(), d.data_ptr(),
                        stream=torch.cuda.current_stream().cuda_stream or 1)
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint64), d.cpu().numpy()


def float64_layer(oracle, rows, sq, metric, cent, assign, q, got, P, tag, live=None):
    """Distances and the set of every query against float64 over the union of its probed clusters."""
    layer = F64.Rows(rows, sq)
    probes = M.nearest(oracle, metric, q, cent, P)
    ok = np.ones(rows.shape[0], bool) if live is None else live
    for i in range(q.shape[0]):
        cand = np.flatnonzero(np.isin(assign, probes[i]) & ok)
        layer.check_distances(NAME[metric], q[i], got[0][i], got[1][i], f"{tag} q{i}")
        layer.check_set(NAME[metric], q[i], got[0][i], cand, f"{tag} q{i}")


class Case:
    """One index over crafted clusters: rows, assignments (clusters of 0, 1, tile, tile + 1 and > 32 rows), centroids,
    queries."""

    def __init__(self, dim, dtype, qdtype, metric, n, C, nq, seed, sq_code=None):
        rng = np.random.default_rng(seed)
        self.dim, self.metric, self.C = dim, metric, C
        x = rows_of(rng, n, dim, np.float32 if sq_code else dtype, 6)
        self.sq = None
        if sq_code is not None:
            codes, scale, bias = SM.compress(x, sq_code)
            self.rows, self.sq = codes, (scale, bias)
        else:
            self.rows = x
        self.plan = ivf_plan(dim, self.rows.dtype, metric, 1, sq=sq_code is not None)
        t = self.plan[0]
        self.assign = layout(rng, n, [0, 1, t, t + 1, 40], C)
        self.cent = centroids_of(x.astype(np.float32), self.assign, C, rng)
        q = rows_of(rng, nq, dim, qdtype, 6)
        self.q = q

    def model(self, oracle, q, k, P):
        if self.sq is not None:
            return SM.search(oracle, self.metric, self.rows, *self.sq, self.cent, self.assign, q, k, P)
        return M.search(oracle, self.metric, self.rows, self.cent, self.assign, q, k, P)

    def index(self):
        return IVF.assemble_from_clustering(Clustering(self.cent, self.assign), self.rows, DIST[self.metric], sq=self.sq)

    def check(self, oracle, index, k, P, tag, q=None, want=None):
        q = self.q if q is None else q
        index.search_parameters = IVFSearchParameters(n_probes=P)
        got = index.search(q, k)
        same(got, self.model(oracle, q, k, P) if want is None else want, tag)
        if P == self.C:
            same(got, scan(self.rows, self.metric, q, k, self.sq), f"{tag} vs the exact scan")
        float64_layer(oracle, self.rows, self.sq, self.metric, self.cent, self.assign, q, got, P, tag)
        return got


# ---- 1. the float leaf, static form: every ring class, k from 1 to 1024, both CTA regimes -------------------------
# (dim, rows, expected (tile_rows, ctas per SM) at k = 10, ks); dims off and on the 16-element edges
FLOAT_DIMS = [(128, 3000, (32, 2), (1, 10, 100, 1024)), (385, 1500, (16, 2), (1, 10, 100)),
              (768, 1200, (16, 2), (10, 1024)), (769, 1000, (8, 2), (10, 100)), (1536, 800, (8, 2), (1, 10)),
              (1537, 600, (4, 2), (10, 100)), (3072, 500, (4, 2), (10, 1024)), (3073, 400, (2, 2), (1, 10)),
              (6144, 300, (2, 1), (10,)), (6145, 300, (1, 2), (10, 100)), (16384, 200, (1, 1), (1, 10))]
PAIRS = [(np.float32, np.float32), (np.float16, np.float32), (np.float32, np.float16), (np.float16, np.float16)]
# (tile_rows, ctas per SM) at k = 10 of the dims that run float16 rows: s = 2 dim, the float32 edges at twice the dims
FLOAT16_RING = {128: (32, 2), 768: (32, 2), 1536: (16, 2), 3072: (8, 2), 6144: (4, 1), 16384: (1, 1)}


@pytest.mark.parametrize("dim,n,ring,ks", FLOAT_DIMS)
def test_float_leaf(oracle, dim, n, ring, ks):
    for metric in (0, 1, 2):
        dtype, qdtype = PAIRS[(FLOAT_DIMS.index((dim, n, ring, ks)) + metric) % 4]
        if dtype == np.float16 and dim in (385, 769, 1537, 3073, 6145):
            dtype = np.float32   # the float16 ring edges sit at twice these dims; keep the float32 ring class
        case = Case(dim, dtype, qdtype, metric, n, 24, 0, seed=dim * 3 + metric)
        tag = f"d{dim} {np.dtype(dtype).name}/{np.dtype(qdtype).name} {NAME[metric]}"
        want_ring = ring if dtype == np.float32 else FLOAT16_RING[dim]
        assert ivf_plan(dim, dtype, metric, 10)[::2][:2] == want_ring, tag
        index = case.index()
        for k in ks:
            pl = ivf_plan(dim, dtype, metric, k)
            Q = pl[1]
            # per-cluster lists just under, at and over Q at n_probes = C (every query probes every cluster)
            rng = np.random.default_rng(dim + k)
            q = rows_of(rng, Q + 1, dim, qdtype, 6)
            want = case.model(oracle, q, k, case.C)
            for m in sorted({max(1, Q - 1), Q, Q + 1}):
                case.check(oracle, index, k, case.C, f"{tag} k{k} Q{Q} nq{m} P=C", q[:m],
                           (want[0][:m], want[1][:m]))
            case.check(oracle, index, k, 3, f"{tag} k{k} P3", q)


def test_one_cta_and_q1_regimes(oracle):
    """dim 3072 at k = 1024 (one CTA per SM, Q = 6), dim 768 at k = 1024 (Q = 1), dim 16384 (one CTA, Q = 1)."""
    for dim, dtype, k, want in ((3072, np.float32, 1024, (4, 6, 1)), (3072, np.float16, 1024, (8, 6, 1)),
                                (768, np.float32, 1024, (16, 1, 2)), (16384, np.float32, 100, (1, 1, 1))):
        for metric in (0, 2):
            assert ivf_plan(dim, dtype, metric, k)[:3] == want
            case = Case(dim, dtype, np.float32, metric, 1100 if dim < 16384 else 200, 8, 9, seed=dim + k + metric)
            index = case.index()
            case.check(oracle, index, k, case.C, f"d{dim} {np.dtype(dtype).name} k{k} {NAME[metric]} P=C")
            case.check(oracle, index, k, 2, f"d{dim} {np.dtype(dtype).name} k{k} {NAME[metric]} P2")


# ---- 2. the dynamic form: tombstones at the end of tiles -------------------------------------------------------
@pytest.mark.parametrize("dim,dtype,qdtype", [(128, np.float32, np.float32), (385, np.float32, np.float16),
                                              (769, np.float16, np.float32), (3073, np.float32, np.float32)])
def test_dynamic_leaf_after_deletes(oracle, dim, dtype, qdtype):
    for metric in (0, 1, 2):
        case = Case(dim, dtype, qdtype, metric, 900, 16, 12, seed=dim + 7 * metric)
        t, _, _, _, _, ds, nr, _ = ivf_plan(dim, dtype, metric, 10, dynamic=True)
        assert ds == (128 if dim == 128 else 0) and nr == (2 if dim == 128 and metric != 2 and dtype == np.float32
                                                          else 1)
        ids = np.arange(case.rows.shape[0], dtype=np.uint64)
        index = DynamicIVF.assemble_from_clustering(Clustering(case.cent, case.assign), case.rows, ids, DIST[metric])
        model = DM.DynamicIVFModel.assemble(oracle, metric, case.cent, case.rows, ids, case.assign)
        # delete the last row of every full tile and the last row of every cluster (clusters hold ascending ids)
        gone = []
        for c in range(case.C):
            members = np.flatnonzero(case.assign == c)
            gone += [int(members[j]) for j in range(t - 1, len(members), t)] + ([int(members[-1])] if len(members) else [])
        gone = sorted(set(gone))
        index.delete(np.array(gone, dtype=np.uint64))
        model.delete(gone)
        live = np.ones(case.rows.shape[0], bool)
        live[gone] = False
        for k, P in ((10, case.C), (100, 4), (1, 1)):
            index.search_parameters = IVFSearchParameters(n_probes=P)
            got = index.search(case.q, k)
            tag = f"dyn d{dim} {NAME[metric]} k{k} P{P}"
            same(got, model.search(case.q, k, P), tag)
            float64_layer(oracle, case.rows, None, metric, case.cent, case.assign, case.q, got, P, tag, live)


# ---- 3. the SQ leaves ------------------------------------------------------------------------------------------
# (dim, rows, tile at L2): rings of 4, 2 and 1 rows, dim % 32 in 1..16 (kpad past the row stride) and in 17..31
SQ_DIMS = [(6145, 300, 4), (6161, 300, 4), (12289, 200, 2), (12305, 200, 2), (24577, 120, 1), (24600, 120, 1)]


@pytest.mark.parametrize("dim,n,tile", SQ_DIMS)
@pytest.mark.parametrize("code", [np.int8, np.uint8])
def test_sq_l2_tensor_core_leaf(oracle, dim, n, tile, code):
    case = Case(dim, np.float32, np.float16 if code == np.uint8 else np.float32, 0, n, 8, 7, seed=dim, sq_code=code)
    assert case.plan[0] == tile and case.plan[4] == 1
    index = case.index()
    for k in (1, 10, 100):
        case.check(oracle, index, k, case.C, f"sq {np.dtype(code).name} d{dim} k{k} P=C")
    case.check(oracle, index, 10, 2, f"sq {np.dtype(code).name} d{dim} k10 P2")


@pytest.mark.parametrize("code", [np.int8, np.uint8])
def test_sq_float_tree_one_cta(oracle, code):
    """SQ MIP / cosine run the float tree on the decoded rows; at dim 3072, k = 1024 with one CTA per SM."""
    for metric in (1, 2):
        assert ivf_plan(3072, code, metric, 1024, sq=True)[:3] == (16, 6, 1)
        case = Case(3072, np.float32, np.float32, metric, 1100, 6, 8, seed=metric, sq_code=code)
        index = case.index()
        case.check(oracle, index, 1024, case.C, f"sq {np.dtype(code).name} {NAME[metric]} k1024 P=C")
        case.check(oracle, index, 10, 2, f"sq {np.dtype(code).name} {NAME[metric]} k10 P2")


@pytest.mark.parametrize("code", [np.int8, np.uint8])
def test_sq_dynamic_and_filtered_wide(oracle, code):
    for metric in (0, 1):
        dim = 6161
        case = Case(dim, np.float32, np.float32, metric, 300, 8, 6, seed=11 + metric, sq_code=code)
        ids = np.arange(case.rows.shape[0], dtype=np.uint64)
        index = DynamicIVF.assemble_from_clustering(Clustering(case.cent, case.assign), case.rows, ids, DIST[metric],
                                                    sq=case.sq)
        model = DSM.DynamicIVFSQModel.assemble(oracle, metric, case.cent, case.rows, ids, *case.sq, case.assign)
        gone = list(range(3, case.rows.shape[0], 7))
        index.delete(np.array(gone, dtype=np.uint64))
        model.delete(gone)
        live = np.ones(case.rows.shape[0], bool)
        live[gone] = False
        index.search_parameters = IVFSearchParameters(n_probes=case.C)
        got = index.search(case.q, 10)
        tag = f"dyn sq {np.dtype(code).name} d{dim} {NAME[metric]}"
        same(got, model.search(case.q, 10, case.C), tag)
        live_ids = np.flatnonzero(live)
        si, sd = scan(case.rows[live_ids], metric, case.q, 10, case.sq)   # the exact scan over the live rows
        same(got, (live_ids[si.astype(np.int64)].astype(np.uint64), sd), f"{tag} vs the exact scan")
        float64_layer(oracle, case.rows, case.sq, metric, case.cent, case.assign, case.q, got, case.C, tag, live)
        # filtered, on the static and on the dynamic index: every second row allowed, all clusters probed (the dynamic
        # mask is over slots, and slot i = row i)
        allowed = np.arange(case.rows.shape[0]) % 2 == 0
        keep = np.flatnonzero(allowed)
        sub = Case.__new__(Case)
        sub.__dict__.update(case.__dict__)
        sub.rows, sub.assign = case.rows[keep], case.assign[keep]
        wi, wd = sub.model(oracle, case.q, 10, case.C)
        st = case.index()
        st.search_parameters = IVFSearchParameters(n_probes=case.C)
        fi, fd, _ = st.search_filtered(case.q, 10, allowed)
        assert np.array_equal(fi, keep[wi.astype(np.int64)].astype(np.uint64)), f"filtered {tag}: ids"
        assert np.array_equal(bits(fd), bits(wd)), f"filtered {tag}: distances"
        float64_layer(oracle, case.rows, case.sq, metric, case.cent, case.assign, case.q, (fi, fd), case.C,
                      f"filtered {tag}", allowed)
        both = allowed & live
        keep = np.flatnonzero(both)
        sub.rows, sub.assign = case.rows[keep], case.assign[keep]
        wi, wd = sub.model(oracle, case.q, 10, case.C)
        di, dd, _ = index.search_filtered(case.q, 10, both)
        assert np.array_equal(di, keep[wi.astype(np.int64)].astype(np.uint64)), f"dyn filtered {tag}: ids"
        assert np.array_equal(bits(dd), bits(wd)), f"dyn filtered {tag}: distances"
        float64_layer(oracle, case.rows, case.sq, metric, case.cent, case.assign, case.q, (di, dd), case.C,
                      f"dyn filtered {tag}", both)


# ---- 4. refusals at the plan's edge ----------------------------------------------------------------------------
def test_refusal_edge_leaves_the_index_usable(oracle):
    for k, ok_dim, bad_dim in ((1024, 18432, 18433), (10, 19104, 19105)):
        with pytest.raises(Svsb200Error):
            ivf_plan(bad_dim, np.float32, 0, k)
        bad = Case(bad_dim, np.float32, np.float32, 0, 60, 8, 2, seed=k)
        index = bad.index()
        index.search_parameters = IVFSearchParameters(n_probes=2)
        with pytest.raises(Svsb200Error, match="k and the row size need more shared memory than a CTA has"):
            index.search(bad.q, k)
        bad.check(oracle, index, 1, 2, f"d{bad_dim} after the refusal")   # still usable at a k that fits
        case = Case(ok_dim, np.float32, np.float32, 0, 1100 if k == 1024 else 60, 8, 2, seed=k + 1)
        assert ivf_plan(ok_dim, np.float32, 0, k)[:3] == (1, 1, 1)
        case.check(oracle, case.index(), k, 2, f"d{ok_dim} k{k} one below the edge")


# ---- 5. query chunks and the probe's deep lists ------------------------------------------------------------------
def test_query_chunks(oracle):
    # nq = 8193 at n_probes = 1, k = 10: a full chunk of 8192 and one of one query
    case = Case(16, np.float32, np.float32, 0, 3000, 40, 8193, seed=5)
    assert ivf_plan(16, np.float32, 0, 10, 1, 8193)[3] == 8192
    index = case.index()
    got = case.check(oracle, index, 10, 1, "nq8193")
    index.search_parameters = IVFSearchParameters(n_probes=1)
    for i in (0, 8191, 8192):
        same(index.search(case.q[i:i + 1], 10), (got[0][i:i + 1], got[1][i:i + 1]), f"nq8193 q{i} alone")
    # nq = 43 at n_probes = k = 1024, C = 1024: chunks of 21, 21, 1
    case = Case(24, np.float32, np.float32, 1, 3000, 1024, 43, seed=6)
    assert ivf_plan(24, np.float32, 1, 1024, 1024, 43)[3] == 21
    index = case.index()
    got = case.check(oracle, index, 1024, 1024, "nq43 P=k=1024")
    for i in (0, 21, 42):
        same(index.search(case.q[i:i + 1], 1024), (got[0][i:i + 1], got[1][i:i + 1]), f"nq43 q{i} alone")


def test_probe_through_the_deep_lists(oracle):
    """C = 600, n_probes 26 and 121, 300 queries: the centroid flat search takes its deep-list split."""
    for metric in (0, 1):
        case = Case(32, np.float32, np.float32, metric, 4000, 600, 300, seed=40 + metric)
        index = case.index()
        for P in (26, 121):
            case.check(oracle, index, 10, P, f"deep lists P{P} {NAME[metric]}")


# ---- 6. hierarchical k-means: the grouped assignment's tiles and multi-chunk staging --------------------------------
def check_hier(oracle, x, metric, C, L1, tag):
    bp = IVFBuildParameters(num_centroids=C, hierarchical_level1_clusters=L1, num_iterations=3, training_fraction=0.5,
                            seed=C * 7 + L1)
    got = Clustering.build_hierarchical(bp, x, DIST[metric])
    want = H.hierarchical_kmeans(oracle, x, metric, C, L1, 3, 0.5, bp.seed)
    assert np.array_equal(got.level2_counts, want.level2_counts), f"{tag}: level2_counts"
    assert np.array_equal(bits(got.centroids), bits(want.centroids)), f"{tag}: centroid bits"
    assert np.array_equal(got.assignments, want.assignments), f"{tag}: assignments"
    start = np.concatenate([[0], np.cumsum(want.level2_counts)]).astype(np.int64)
    group = np.searchsorted(start, got.assignments, side="right") - 1
    F64.check_assignment(NAME[metric], x, got.centroids, got.assignments, f"{tag} level 2",
                         [np.arange(start[g], start[g + 1]) for g in group])
    pop = np.flatnonzero(want.level2_counts > 0)
    F64.check_assignment(NAME[metric], x, want.level1_centroids[pop], np.searchsorted(pop, group), f"{tag} level 1")
    return want.level2_counts


@pytest.mark.parametrize("dtype", [np.float32, np.float16])
@pytest.mark.parametrize("dim,C,L1,tile", [(96, 200, 2, 64), (128, 150, 2, 64), (177, 120, 2, 32), (384, 60, 2, 16),
                                           (768, 64, 4, 8)])
def test_hierarchical_kmeans_chunks(oracle, dim, C, L1, tile, dtype):
    """Groups with more centroids than one staged chunk (c_g > tile), and one with an exact multiple of it."""
    assert group_tile(dim) == tile
    rng = np.random.default_rng(dim)
    n = max(4 * C, 600)
    for metric in (0, 1, 2):
        x = rows_of(rng, n, dim, dtype, 5)
        counts = check_hier(oracle, x, metric, C, L1, f"hier d{dim} {np.dtype(dtype).name} {NAME[metric]}")
        assert counts.max() > tile, f"d{dim}: no group passes one chunk of {tile} centroids"


def test_hierarchical_group_at_a_multiple_of_the_chunk(oracle):
    """dim 768 (8 centroids per chunk), C = 16, L1 = 1: the one group holds exactly two chunks."""
    assert group_tile(768) == 8
    x = rows_of(np.random.default_rng(3), 400, 768, np.float32, 4)
    for metric in (0, 2):
        counts = check_hier(oracle, x, metric, 16, 1, f"hier multiple {NAME[metric]}")
        assert counts.tolist() == [16]


# ---- 7. flat k-means ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim,C", [(33, 40), (33, 520), (768, 40), (768, 520)])
def test_flat_kmeans(oracle, dim, C):
    rng = np.random.default_rng(dim + C)
    x = rows_of(rng, 2 * C + 400, dim, np.float32, 12)
    for metric in (0, 1):
        bp = IVFBuildParameters(num_centroids=C, num_iterations=2, training_fraction=0.6, seed=dim)
        got = Clustering.build(bp, x, DIST[metric])
        cent, assign = M.kmeans(oracle, x, metric, C, 2, 0.6, dim)
        tag = f"kmeans d{dim} C{C} {NAME[metric]}"
        assert np.array_equal(bits(got.centroids), bits(cent)), f"{tag}: centroid bits"
        assert np.array_equal(got.assignments, assign), f"{tag}: assignments"
        F64.check_assignment(NAME[metric], x, got.centroids, got.assignments, tag)
        # an assembly without assignments puts every row in the model's cluster, its float64-nearest: per row through
        # the dynamic index's export (slot i = row i), per cluster through the static index's sizes
        dyn = DynamicIVF.assemble_from_clustering(Clustering(got.centroids), x, np.arange(x.shape[0]), DIST[metric])
        status, _, cluster = dyn.export()
        assert np.all(status == 1) and np.array_equal(cluster, assign), f"{tag}: assembled assignments"
        F64.check_assignment(NAME[metric], x, got.centroids, cluster, f"{tag} assembled")
        index = IVF.assemble_from_clustering(Clustering(got.centroids), x, DIST[metric])
        assert np.array_equal(index.cluster_sizes, np.bincount(assign, minlength=C)), tag
