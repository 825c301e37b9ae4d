"""The shapes of the IVF leaf scan and of the hierarchical k-means' grouped assignment (csrc/ivf.cu: ivf_plan and
ivf_group_plan, the arithmetic ivf_search_on_device and ivf_group_assign run), checked through svsb200_ivf_plan and
svsb200_ivf_group_plan at and on both sides of every boundary.  No GPU needed.

The hand derivation (every size in bytes; L = 227 KB - 1 KB = 231424, the dynamic shared memory a CTA may use):
  row stride   s = round16(dim * element size)          query stride  qs = round16(dim) floats
  ring         tile_rows = 32, halved while 2 * tile_rows * s > 96 KB (98304)
  float leaf   fixed = 2 * tile_rows * s + 8 * 32 * 8,  slot = 4 qs + round16(8 k)
  SQ L2 leaf   fixed = 2 * tile_rows * s + 8 * 32 * 8 + 128,  slot = round32(dim) + round16(8 k) + 128
  Q            min(64, (L / 2 - fixed) / slot) with two CTAs per SM; where that is 0, min(64, (L - fixed) / slot) with one;
               where that is 0 too, the search is refused
  query chunk  max(1, min(8192, 256 MiB / (12 n_probes k)))
  group tile   64, halved while 2 tile * qs * 4 + 24 tile > 96 KB; chunk = tile; smem = 2 tile * qs * 4 + 12 tile <= L
"""
import ctypes as C

import pytest

from scalablevectorsearch_b200 import Svsb200Error, _lib

F32, F16, I8, U8 = 0, 1, 2, 3
PLAIN, SQ = 0, 1
L2, IP, COS = 0, 1, 2
LIMIT = 227 * 1024 - 1024
REFUSAL = "k and the row size need more shared memory than a CTA has"


def plan(dim, dtype=F32, metric=L2, k=10, n_probes=1, nq=1000, dynamic=False, storage=None):
    """(tile_rows, Q, ctas per SM, query chunk, leaf, static dim, rows per pass, smem bytes)."""
    if storage is None:
        storage = SQ if dtype in (I8, U8) else PLAIN
    out = [C.c_uint32() for _ in range(7)] + [C.c_uint64()]
    _lib.check(_lib.lib().svsb200_ivf_plan(dim, dtype, storage, metric, k, n_probes, nq, int(dynamic),
                                           *[C.byref(o) for o in out]))
    return tuple(o.value for o in out)


def group_plan(dim):
    out = [C.c_uint32(), C.c_uint32(), C.c_uint64()]
    _lib.check(_lib.lib().svsb200_ivf_group_plan(dim, *[C.byref(o) for o in out]))
    return tuple(o.value for o in out)


def ring(dim, dtype=F32, metric=L2, k=10):
    """(tile_rows, Q, ctas per SM)."""
    return plan(dim, dtype, metric, k)[:3]


def r16(x):
    return (x + 15) // 16 * 16


def derive(dim, esize, k, sq_l2):
    """The hand derivation above, for the invariants below: (tile_rows, Q, ctas, slot bytes)."""
    s, qs = r16(dim * esize), r16(dim)
    t = 32
    while t > 1 and 2 * t * s > 96 * 1024:
        t //= 2
    if sq_l2:
        fixed, slot = 2 * t * s + 8 * 32 * 8 + 128, (dim + 31) // 32 * 32 + r16(8 * k) + 128
    else:
        fixed, slot = 2 * t * s + 8 * 32 * 8, 4 * qs + r16(8 * k)
    for ctas, room in ((2, LIMIT // 2), (1, LIMIT)):
        if fixed < room and (room - fixed) // slot:
            return t, min(64, (room - fixed) // slot), ctas, slot
    return t, 0, 0, slot


# ---- the ring: where the row stride's 16-byte rounding passes 96 KB / (2 tile_rows) ---------------------------------
@pytest.mark.parametrize("dtype,dim,tile", [
    # float32: 2 * 32 * s <= 98304 while s <= 1536 bytes = 384 elements; 385 rounds s to 1552
    (F32, 384, 32), (F32, 385, 16), (F32, 768, 16), (F32, 769, 8), (F32, 1536, 8), (F32, 1537, 4),
    (F32, 3072, 4), (F32, 3073, 2), (F32, 6144, 2), (F32, 6145, 1), (F32, 16384, 1),
    # float16: the same byte edges at twice the elements (s = 2 dim)
    (F16, 768, 32), (F16, 769, 16), (F16, 1536, 16), (F16, 1537, 8), (F16, 3072, 8), (F16, 3073, 4),
    (F16, 6144, 4), (F16, 6145, 2), (F16, 12288, 2), (F16, 12289, 1),
    # SQ codes: one byte per element; 16-byte rounding makes 1537..1552 one stride
    (I8, 1536, 32), (I8, 1537, 16), (U8, 3072, 16), (U8, 3073, 8), (I8, 6144, 8), (I8, 6145, 4),
    (U8, 12288, 4), (U8, 12289, 2), (I8, 24576, 2), (I8, 24577, 1),
])
def test_ring_halves_at_the_row_stride_edges(dtype, dim, tile):
    for metric in (L2, IP, COS):
        assert plan(dim, dtype, metric, k=1)[0] == tile, (dtype, dim, metric)


def test_queries_per_item_and_ctas():
    # dim 96 float32: fixed = 2 * 32 * 384 + 2048 = 26624; slot = 384 + round16(8 k)
    assert ring(96, k=10) == (32, 64, 2)      # (115712 - 26624) / 464 = 192 -> 64
    assert ring(96, k=1024) == (32, 10, 2)    # (115712 - 26624) / 8576 = 10 (DESIGN §15's "k = 1024: 10 queries")
    # dim 128: slot 512 + 8192 at k = 1024 -> (115712 - 34816) / 8704 = 9
    assert ring(128, k=1024) == (32, 9, 2)
    # the embedding sizes at k = 10: 384 -> (115712 - 100352) / 1616 = 9; 768 (16 rows) -> 4; 1024 (8 rows) -> 11;
    # 1536 -> 2; 3072 (4 rows) -> 1
    assert [ring(d)[:2] for d in (384, 768, 1024, 1536, 3072)] == [(32, 9), (16, 4), (8, 11), (8, 2), (4, 1)]
    # Q = 1: dim 768 at k = 1024 -> (115712 - 100352) / 11280 = 1; dim 16384 at any k (ring 1 row, 65536 + 2048 fixed)
    assert ring(768, k=1024) == (16, 1, 2)
    for k in (1, 10, 100, 1024):
        assert ring(16384, k=k) == (1, 1, 1)
    # one CTA per SM: dim 3072, k = 1024: fixed 100352, slot 20480 -> (115712 - 100352) / 20480 = 0; one CTA:
    # (231424 - 100352) / 20480 = 6
    assert ring(3072, k=1024) == (4, 6, 1)
    assert ring(3072, k=100) == (4, 1, 2)
    # dim 6144: fixed 100352 and slot 24576 + 16 > 15360 at any k -> one CTA; 6145 returns to two with a 1-row ring
    for k in (1, 10, 100, 1024):
        assert ring(6144, k=k)[2] == 1
        assert ring(6145, k=k)[::2] == (1, 2)
    assert ring(12288, k=10) == (1, 2, 1)
    assert ring(12287, k=10) == (1, 2, 1)
    # float16 at 3072 / k = 1024 (8-row ring) and SQ MIP at 3072 / k = 1024 (float tree, 16-row ring): one CTA
    assert ring(3072, F16, k=1024) == (8, 6, 1)
    assert ring(3072, I8, IP, k=1024) == (16, 6, 1)
    assert ring(3072, U8, COS, k=1024) == (16, 6, 1)
    assert ring(3072, I8, L2, k=1024) == (16, 1, 2)   # the SQ L2 leaf: slot 3072 + 8192 + 128


@pytest.mark.parametrize("k,ok,refused", [
    # one CTA, ring 1 row: fixed = 2 s + 2048, slot = 4 qs + round16(8 k); refused where fixed + slot > 231424
    # k = 1024: 18432: 2 * 73728 + 2048 + 73728 + 8192 = 231424; 18433 rounds s to 73744 and qs to 18448
    (1024, 18432, 18433),
    # k = 10: 19104: 2 * 76416 + 2048 + 76416 + 80 = 231376; 19105: s 76432, qs 19120 -> 231472
    (10, 19104, 19105),
    # k = 1: 19108: s 76432, qs 19120 -> 152864 + 2048 + 76480 + 16 = 231408; 19109: s 76448 -> 231440
    (1, 19108, 19109),
])
def test_refusal_edge(k, ok, refused):
    assert plan(ok, k=k)[:3] == (1, 1, 1)
    with pytest.raises(Svsb200Error, match=REFUSAL):
        plan(refused, k=k)
    assert "svsb200_ivf_search" in _lib.lib().svsb200_last_error().decode()


def test_query_chunk():
    # 256 MiB / (12 P k): P = 1, k = 10 -> 2236962 -> 8192; a batch of 8193 is one full chunk and one of one query
    assert plan(96, k=10, n_probes=1, nq=8193)[3] == 8192
    assert plan(96, k=10, n_probes=1, nq=100)[3] == 100
    # P = k = 1024: 268435456 / 12582912 = 21 -> 43 queries are chunks of 21, 21 and 1
    assert plan(96, k=1024, n_probes=1024, nq=43)[3] == 21
    # P = 1024, k = 512: 268435456 / 6291456 = 42.7 -> 42; P = k = 1024 is the least chunk, so the floor of 1 is
    # never reached within the limits
    assert plan(96, k=512, n_probes=1024, nq=100)[3] == 42


def test_leaf_static_dim_and_rows_per_pass():
    # float32 L2 / MIP at 96 and 128: static dimension, two rows per pass; the dynamic form keeps two there
    for dim in (96, 128):
        for metric in (L2, IP):
            for dyn in (False, True):
                assert plan(dim, F32, metric, dynamic=dyn)[4:7] == (0, dim, 2)
        assert plan(dim, F32, COS)[4:7] == (0, dim, 1)        # cosine: one row
        assert plan(dim, F16, L2)[4:7] == (0, dim, 1)         # float16 rows: one row
        assert plan(dim, I8, IP)[4:7] == (0, dim, 1)          # SQ codes on the float tree: one row
    # the generic dimension: two rows per pass in the static form, one in the dynamic form
    assert plan(385, F32, L2)[4:7] == (0, 0, 2)
    assert plan(385, F32, L2, dynamic=True)[4:7] == (0, 0, 1)
    assert plan(127, F32, IP)[4:7] == (0, 0, 2)
    # SQ L2: the tensor-core leaf
    for dtype in (I8, U8):
        for dim in (96, 128, 6145):
            assert plan(dim, dtype, L2)[4:7] == (1, 0, 0)


def test_plan_invariants():
    """Over a sweep: the plan is the hand derivation, its shared memory fits a CTA (half of it with two CTAs per SM),
    and Q is the largest that fits (or 64)."""
    ks = (1, 10, 100, 1024)
    dims = sorted({d + e for d in (16, 96, 128, 384, 768, 1536, 3072, 6144, 12288, 16384) for e in (-1, 0, 1)})
    cases = [(F32, 4, L2), (F32, 4, COS), (F16, 2, IP), (I8, 1, L2), (U8, 1, IP)]
    for dtype, esize, metric in cases:
        sq_l2 = dtype in (I8, U8) and metric == L2
        for dim in dims:
            for k in ks:
                t, q, ctas, slot = derive(dim, esize, k, sq_l2)
                if q == 0:
                    with pytest.raises(Svsb200Error, match=REFUSAL):
                        plan(dim, dtype, metric, k)
                    continue
                got = plan(dim, dtype, metric, k)
                assert got[:3] == (t, q, ctas), (dtype, dim, metric, k)
                smem = got[7]
                room = LIMIT // ctas
                assert smem <= room
                assert q == 64 or smem + slot > room
                if ctas == 1:
                    assert smem - (q - 1) * slot > LIMIT // 2   # one query would not fit two CTAs


@pytest.mark.parametrize("dim,tile", [
    # 8 tile qs + 24 tile <= 98304: tile 64 while qs <= 189 -> dim 176 (qs 176); 177 rounds qs to 192
    # tile 32: qs <= 381 -> 368 | 369 (qs 384); 16: qs <= 765 -> 752 | 753; 8: qs <= 1533 -> 1520 | 1521;
    # 4: qs <= 3069 -> 3056 | 3057; 2: qs <= 6141 -> 6128 | 6129
    (130, 64), (176, 64), (177, 32), (368, 32), (369, 16), (384, 16), (752, 16), (753, 8), (768, 8), (1520, 8),
    (1521, 4), (3056, 4), (3057, 2), (6128, 2), (6129, 1), (16384, 1),
])
def test_group_tile(dim, tile):
    t, chunk, smem = group_plan(dim)
    qs = r16(dim)
    assert (t, chunk) == (tile, tile)
    assert smem == 2 * tile * qs * 4 + 12 * tile <= LIMIT


def test_group_refusal_edge():
    # tile 1: 8 qs + 12 <= 231424 while qs <= 28926 -> qs 28912 (dim 28912) fits, 28913 rounds qs to 28928
    assert group_plan(28912) == (1, 1, 8 * 28912 + 12)
    with pytest.raises(Svsb200Error, match="rows too wide for the grouped kernels"):
        group_plan(28913)


def test_plan_rejects_bad_arguments():
    lib = _lib.lib()
    out = [C.c_uint32() for _ in range(7)] + [C.c_uint64()]
    refs = [C.byref(o) for o in out]
    assert lib.svsb200_ivf_plan(96, I8, PLAIN, L2, 10, 1, 1, 0, *refs) != 0    # integer rows are not plain IVF rows
    assert lib.svsb200_ivf_plan(96, F32, SQ, L2, 10, 1, 1, 0, *refs) != 0      # SQ rows are codes
    assert lib.svsb200_ivf_plan(96, F32, PLAIN, 3, 10, 1, 1, 0, *refs) != 0
    assert lib.svsb200_ivf_plan(0, F32, PLAIN, L2, 10, 1, 1, 0, *refs) != 0
    assert lib.svsb200_ivf_plan(96, F32, PLAIN, L2, 0, 1, 1, 0, *refs) != 0
    assert lib.svsb200_ivf_plan(96, F32, PLAIN, L2, 1025, 1, 1, 0, *refs) != 0
    assert lib.svsb200_ivf_plan(96, F32, PLAIN, L2, 10, 0, 1, 0, *refs) != 0
    assert lib.svsb200_ivf_plan(96, F32, PLAIN, L2, 10, 1025, 1, 0, *refs) != 0
    assert lib.svsb200_ivf_plan(96, F32, PLAIN, L2, 10, 1, 0, 0, *refs) != 0
    assert b"svsb200_ivf_plan" in lib.svsb200_last_error()
    assert lib.svsb200_ivf_plan(96, F32, PLAIN, L2, 10, 1, 1, 0, *refs[:7], None) != 0
    assert lib.svsb200_ivf_group_plan(0, *refs[:2], refs[7]) != 0
