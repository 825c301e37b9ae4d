"""A numpy model of the fp16 flat search's certificate (csrc/flat.cu, flat_rescore_kernel), with the error bound E(q)
written as the kernel computes it: the earlier float32 formula, which assumed a relative fp16 rounding ("old"), beside
the current one ("new"; the kernel rounds each of its operations up in float32, the model evaluates it in double).
No GPU needed.

The model rounds both operands to fp16 as the tile kernel does (np.float16: round to nearest even, +-inf from 65520
on, subnormals below 2^-14), sums the rounded products in float64 (standing in for the tensor core's fp32 sum, whose
error the dim 2^-22 term covers), forms the fp32 key and keeps, per list, the KC smallest keys of the list's rows.  As
in the kernel, NaN and +inf keys are never offered to a list and -inf keys are.  The lists' row ranges come from
svsb200_flat_plan_k for a 132-SM device.  A query is "verified" when T > kth_approx + 2E, and the verification is
"wrong" when a row of the exact top k (float64 distances of the unrounded values, ties by id) is not a candidate.

The old bound assumed a relative rounding of 2^-11 per element: it verifies wrong candidate sets when an element
overflows fp16 or sits in fp16's subnormals.  The new bound adds 2^-25 sqrt(dim) per rounded operand and refuses to
verify a query whose ||q||, Xmax or E is not finite.  test_gpu_flat_range.py runs the same fixtures on the GPU."""
import ctypes as C
import math

import numpy as np
import pytest

import flat_range_fixtures as fx

SMS = 132


def list_rows(nq, n, k):
    """For each query tile, the row ids of each of its candidate lists (the plan's pieces, split into column halves for
    the 33-entry lists), and the list depth."""
    from scalablevectorsearch_b200 import _lib
    lib = _lib.lib()
    ctas, share, nl, kc = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
    out = (C.byref(ctas), C.byref(share), C.byref(nl), C.byref(kc))
    _lib.check(lib.svsb200_flat_plan_k(nq, n, k, SMS, *out, None))
    assert kc.value, "a batch that takes the scan has no lists"
    seg = np.zeros(ctas.value // share.value + 1, dtype=np.uint64)
    _lib.check(lib.svsb200_flat_plan_k(nq, n, k, SMS, *out, seg.ctypes.data))
    seg = seg.astype(np.int64)
    mtiles, ntiles = -(-nq // 128), -(-n // 256)
    tiles = []
    for m in range(mtiles):
        lo, hi = (m // share.value) * ntiles, (m // share.value + 1) * ntiles
        lists = []
        for b in range(len(seg) - 1):
            a, e = max(seg[b], lo) - lo, min(seg[b + 1], hi) - lo
            if a >= e:
                continue
            cols = np.arange(256) if kc.value == 129 else None
            for half in ([None] if kc.value == 129 else [0, 1]):
                c = cols if half is None else np.arange(128) + 128 * half
                r = (np.arange(a, e)[:, None] * 256 + c[None, :]).ravel()
                lists.append(r[r < n])
        assert sum(len(r) for r in lists) == n and len(lists) == nl.value
        tiles.append(lists)
    return tiles, kc.value


def f16(v):
    with np.errstate(over="ignore"):
        return v.astype(np.float32).astype(np.float16).astype(np.float64)


def norm32(v):
    """||v|| as flat_tile_kernel computes it (float32 sum, sqrtf, times 1.000001)."""
    s = (v.astype(np.float64) ** 2).sum(1).astype(np.float32)
    return np.sqrt(s).astype(np.float32) * np.float32(1.000001)


def old_bound(metric, dim, r, data_rounded, data_int, qn, xm):
    """The earlier E(q), in float32, operation by operation as flat_rescore_kernel wrote it: (r 2^-11 + dim 2^-22)
    ||q|| Xmax, for L2 doubled plus 2^-10 Xmax^2 for rounded data (2^-23 Xmax^2 for integer data)."""
    f = np.float32
    e_ip = (f(r) * f(4.8828125e-4) + f(dim) * f(2.384185791015625e-7)) * qn * xm * f(1.0001)
    if metric == "ip":
        return e_ip
    extra = f(9.765625e-4) * xm * xm if (r > 1 or data_rounded) else f(1.1920929e-7) * xm * xm if data_int else f(0)
    return f(2) * e_ip + extra


def new_bound(metric, dim, q_rounded, data_rounded, data_int, qn, xm):
    """E(q) of flat_rescore_kernel: per element |fl16(v) - v| <= 2^-11 |v| + 2^-25, so a rounded operand moves by at
    most 2^-11 ||v|| + 2^-25 sqrt(dim).  qn / xm are +inf when an element overflowed."""
    qn, xm = np.float64(qn), np.float64(xm)
    sd = 2.0 ** -25 * math.sqrt(dim)
    dq = 2.0 ** -11 * qn + sd if q_rounded else 0.0
    dx = 2.0 ** -11 * xm + sd if data_rounded else 0.0
    e_ip = dq * (xm + dx) + qn * dx + dim * 2.0 ** -22 * (qn + dq) * (xm + dx)
    e = e_ip if metric == "ip" else 2 * e_ip + dx * (2 * xm + dx) + (2.0 ** -23 * xm * xm if data_int else 0.0)
    return e * 1.0001


def model(x, q, metric, k):
    """(verified by the old bound, verified by the new bound, candidate set wrong), one entry per query."""
    q_rounded, data_rounded = q.dtype == np.float32, x.dtype == np.float32
    data_int = x.dtype in (np.int8, np.uint8)
    nq, n, dim = q.shape[0], x.shape[0], x.shape[1]
    qt = f16(q) if q_rounded else q.astype(np.float64)
    xt = f16(x) if data_rounded else x.astype(np.float64)
    with np.errstate(all="ignore"):
        dot = (qt @ xt.T).astype(np.float32).astype(np.float64)
        if metric == "l2":
            bias = (x.astype(np.int64) ** 2).sum(1) if data_int else (xt * xt).sum(1)
            key = (bias.astype(np.float32).astype(np.float64)[None, :] - 2 * dot).astype(np.float32)
        else:
            key = (-dot).astype(np.float32)
        q64, x64 = q.astype(np.float64), x.astype(np.float64)
        exact = ((q64 * q64).sum(1)[:, None] + (x64 * x64).sum(1)[None, :] - 2 * q64 @ x64.T
                 if metric == "l2" else -(q64 @ x64.T))
    qn, xn = norm32(q), norm32(x)
    xm = xn.max()
    qn_new = np.where(np.isinf(qt).any(1), np.float32(np.inf), qn)
    xm_new = np.float32(np.inf) if np.isinf(xt).any() else xm
    r = int(q_rounded) + int(data_rounded)
    tiles, kc = list_rows(nq, n, k)
    v_old, v_new, wrong = np.zeros(nq, bool), np.zeros(nq, bool), np.zeros(nq, bool)
    for i in range(nq):
        ki = key[i].astype(np.float64)
        offered = ki < np.inf          # NaN and +inf keys never enter a list; -inf keys do
        cand, T = [], np.inf
        for rows in tiles[i // 128]:
            rows = rows[offered[rows]]
            keep = rows[np.argsort(ki[rows], kind="stable")[:kc]]
            cand.append(keep)
            T = min(T, ki[keep].max() if len(keep) == kc else np.inf)
        cand = np.concatenate(cand)
        top = np.lexsort((np.arange(n), exact[i]))[:k]
        wrong[i] = not np.isin(top, cand).all()
        if len(cand) < k:
            continue
        kth = np.float32(np.sort(ki[cand])[k - 1])
        with np.errstate(all="ignore"):
            e_old = old_bound(metric, dim, r, data_rounded, data_int, qn[i], xm)
            v_old[i] = np.float32(T) > kth + np.float32(2) * e_old
            e_new = new_bound(metric, dim, q_rounded, data_rounded, data_int, qn_new[i], xm_new)
        v_new[i] = np.isfinite(e_new) and T > float(kth) + 2 * e_new
    return v_old, v_new, wrong


def _as(x, q, dtype, qtype):
    """The fixture's values as (data, query) types; float16 operands are clipped to its finite range first."""
    cast = lambda v, t: (np.clip(v, -fx.FP16_MAX, fx.FP16_MAX) if t == np.float16 else v).astype(t)   # noqa: E731
    return cast(x, dtype), cast(q, qtype)


# (name, metric, data, queries): every fixture of test_gpu_flat_range.py on which the parent's bound verified a wrong
# candidate set in this model
ADVERSARIAL = (
    [(f"data_overflow_{m}_{qt.__name__}", m, *_as(*fx.data_overflow(m)[:2], np.float32, qt))
     for m in ("l2", "ip") for qt in (np.float32, np.float16)]
    + [(f"query_overflow_{m}_{dt.__name__}", m, *fx.query_overflow(m, dt)[:2])
       for m in ("l2", "ip") for dt in (np.float32, np.float16, np.uint8, np.int8)]
    + [(f"thin_shell_1e-7_{d}", "l2", *fx.thin_shell(1e-7, d)[:2]) for d in (16, 32, 96, 100)]
)


@pytest.mark.parametrize("name,metric,x,q", ADVERSARIAL, ids=[a[0] for a in ADVERSARIAL])
def test_old_bound_verifies_wrong_sets_and_new_bound_does_not(name, metric, x, q):
    v_old, v_new, wrong = model(x, q, metric, 10)
    assert (v_old & wrong).any(), f"{name}: the fixture no longer defeats the old bound"
    assert not (v_new & wrong).any(), f"{name}: queries {np.flatnonzero(v_new & wrong)} verified a wrong set"


def _other_fixtures():
    for m in ("l2", "ip"):
        for inf_row in (False, True):
            yield f"boundary_{m}_{inf_row}", m, *fx.boundary(inf_row)[:2]
        for scale in (1e-6, 3e-7, 1e-7):
            for d in (16, 32, 96, 100):
                x, q, _ = fx.thin_shell(scale, d)
                for dt, qt in ((np.float32, np.float32), (np.float32, np.float16), (np.float16, np.float32)):
                    yield f"thin_shell_{m}_{scale}_{d}_{dt.__name__}_{qt.__name__}", m, *_as(x, q, dt, qt)
        yield f"subnormal_u8_{m}", m, *fx.subnormal_queries_u8()[:2]


def test_new_bound_is_sound_on_every_fixture():
    for name, metric, x, q in _other_fixtures():
        for k in (10, 25):
            _, v_new, wrong = model(x, q, metric, k)
            assert not (v_new & wrong).any(), (name, k, np.flatnonzero(v_new & wrong))


def test_new_bound_is_sound_over_the_float32_range():
    """Thin shells with elements of 2^-30 .. 2^18 (the top ones overflow fp16), dims 4 .. 272, L2 and MIP, one or two
    rounded operands (float16 operands clipped to fp16's finite range)."""
    checked = verified = 0
    for e in range(-30, 19, 3):
        for dim in (4, 16, 96, 272):
            x, q, _ = fx.thin_shell(2.0 ** e, dim, n=1024, seed=e)
            for dt, qt in ((np.float32, np.float32), (np.float32, np.float16), (np.float16, np.float32)):
                xx, qq = _as(x, q, dt, qt)
                for metric in ("l2", "ip"):
                    _, v_new, wrong = model(xx, qq, metric, 10)
                    assert not (v_new & wrong).any(), (e, dim, dt, qt, metric, np.flatnonzero(v_new & wrong))
                    checked += len(wrong)
                    verified += int(v_new.sum())
    assert verified > checked // 4, f"only {verified} of {checked} queries verified: the sweep proves little"


@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_new_bound_verifies_ordinary_data_that_touches_subnormals(metric):
    x, q, _ = fx.tightness_control()
    for k in (10, 100):
        v_old, v_new, wrong = model(x, q, metric, k)
        assert v_new.all(), f"k={k}: {int((~v_new).sum())} of {len(v_new)} queries no longer verify"
        assert not wrong.any()
