"""A float64 layer under the bit-exact checks: every returned distance recomputed in float64 from the operands the kernel
sees, held to a bound on its float32 rounding, so that a distance expression the kernel and the oracle share cannot
hide behind their agreement.  Used by tests/test_gpu_search_shapes.py (the exhaustive scan) and
tests/test_gpu_ivf_shapes.py (the IVF leaves and k-means assignments).

Bounds: a float32 sum of `dim` terms, each one rounding away from its float64 value, is within (dim + 8) 2^-24 of the
sum of their magnitudes (1% slack); cosine adds two relative roundings of the norms.  SQ L2 has no bound: the integer
sum is exact, so the distance must equal fl32(fl32(scale^2) * fl32(sum)) exactly.
"""
import numpy as np

U = 2.0 ** -24
ALL_ONES = np.uint64(0xFFFFFFFFFFFFFFFF)
SQ_RANGE = {np.dtype(np.int8): (-128, 127), np.dtype(np.uint8): (0, 255)}


def gamma(dim):
    return (dim + 8) * U * 1.01


def query_f32(q):
    """A query as the SQ and cosine preparation reads it (q_scalar): float16 subnormals flush to zero."""
    q = np.asarray(q)
    f = q.astype(np.float32)
    if q.dtype == np.float16:
        f = np.where(np.abs(f) < np.float32(2.0 ** -14), np.copysign(np.float32(0), f), f).astype(np.float32)
    return f


def sq_decode(codes, scale, bias):
    """fl32(scale * c + bias), one rounding per operation (scalar.h:44-46), as float64."""
    return (np.float32(scale) * np.asarray(codes).astype(np.float32) + np.float32(bias)).astype(np.float64)


def sq_l2_query_codes(q, code_dtype, scale, bias):
    """PREP_SQ_L2 (sq_compress_code over q_scalar): clamp(roundf(fl32(fl32(q - bias) / scale))), halves away from
    zero."""
    lo, hi = SQ_RANGE[np.dtype(code_dtype)]
    t = ((query_f32(q) - np.float32(bias)) / np.float32(scale)).astype(np.float64)   # fp32 subtract, then divide
    return np.clip(np.sign(t) * np.floor(np.abs(t) + 0.5), lo, hi).astype(np.int64)


def sq_l2_exact(q, codes, scale, bias):
    """The SQ L2 distances of one query to code rows: fl32(fl32(scale^2) * fl32(sum (qc - c)^2)), the sum in int64."""
    codes = np.asarray(codes)
    dim = codes.shape[1]
    assert dim * 255 ** 2 < 2 ** 31, "the int32 sum of the kernel wraps past dim 255^2 >= 2^31"
    qc = sq_l2_query_codes(q, codes.dtype, scale, bias)
    l2 = ((codes.astype(np.int64) - qc) ** 2).sum(1)
    return np.float32(np.float32(scale) * np.float32(scale)) * l2.astype(np.float32)


def float_tree(metric, q, y, lvq_mean=None):
    """(d64, bound) of the float tree of one float64 query q against float64 rows y; `lvq_mean` adds <q, mean> to MIP."""
    dim = y.shape[1]
    g = gamma(dim)
    if metric == "l2":
        t = (q[None, :] - y) ** 2
        d64 = t.sum(1)
        return d64, g * d64
    t = q[None, :] * y
    if metric == "ip":
        d64, terms = t.sum(1), np.abs(t).sum(1)
        if lvq_mean is not None:
            m = q * lvq_mean.astype(np.float64)
            d64, terms = d64 + m.sum(), terms + np.abs(m).sum()
        return d64, g * terms
    with np.errstate(invalid="ignore", divide="ignore"):
        norms = np.sqrt((y * y).sum(1)) * np.sqrt((q * q).sum())
        d64 = t.sum(1) / norms
        return d64, g * (np.abs(t).sum(1) / norms + 2 * np.abs(d64))


def sq_ip(q, codes, scale, bias):
    """(d64, bound) of the SQ inner product scale <q, c> + bias sum(q) against the decoded rows."""
    scale, bias = float(scale), float(bias)
    q, c = np.asarray(q).astype(np.float64), np.asarray(codes).astype(np.float64)
    d64 = (q * (scale * c + bias)).sum(1)
    terms = (np.abs(q) * (np.abs(scale * c) + abs(bias))).sum(1)
    return d64, gamma(c.shape[1]) * terms


def assert_within(d32, d64, bound, tag):
    err = np.abs(np.asarray(d32, dtype=np.float64) - d64)
    bad = ~(err <= bound)
    assert not np.any(bad), f"{tag}: off float64 by {err[bad][:4]} > {bound[bad][:4]}"


class Rows:
    """The rows of an index as the kernel sees them, for the float64 layer of its searches: float32 / float16 rows
    (`codes` None), or SQ codes with (scale, bias)."""

    def __init__(self, rows, sq=None):
        self.rows = np.asarray(rows)
        self.sq = None if sq is None else (np.float32(sq[0]), np.float32(sq[1]))

    def reference(self, metric, q, ids):
        """(d64, bound) of query q against rows `ids`; SQ L2 gives its exact float32 values and a zero bound."""
        ids = np.asarray(ids, dtype=np.int64)
        if self.sq is not None and metric == "l2":
            return sq_l2_exact(q, self.rows[ids], *self.sq).astype(np.float64), np.zeros(len(ids))
        if self.sq is not None and metric == "ip":
            return sq_ip(query_f32(q), self.rows[ids], *self.sq)
        q64 = (query_f32(q) if self.sq is not None else np.asarray(q).astype(np.float32)).astype(np.float64)
        y = sq_decode(self.rows[ids], *self.sq) if self.sq is not None else self.rows[ids].astype(np.float64)
        return float_tree(metric, q64, y)

    def check_distances(self, metric, q, ids, d32, tag):
        """Every returned (id, distance) of one query within its bound of float64 (SQ L2: equal)."""
        keep = ids != ALL_ONES
        ids, d32 = ids[keep].astype(np.int64), np.asarray(d32)[keep]
        if len(ids) == 0:
            return
        d64, bound = self.reference(metric, q, ids)
        if self.sq is not None and metric == "l2":
            assert np.array_equal(d32.astype(np.float32).view(np.uint32), d64.astype(np.float32).view(np.uint32)), \
                f"{tag}: SQ L2 is not scale^2 * int L2"
            return
        assert_within(d32, d64, bound, tag)

    def check_set(self, metric, q, ids, candidates, tag):
        """The returned ids of one query are candidates, and no candidate left out is nearer in float64 than the k-th
        returned row by the two rows' bounds added together or more (a near tie).  A short row holds every
        candidate."""
        keep = ids != ALL_ONES
        got = ids[keep].astype(np.int64)
        candidates = np.asarray(candidates, dtype=np.int64)
        assert np.all(np.isin(got, candidates)), f"{tag}: a returned row is not in a probed cluster"
        assert len(np.unique(got)) == len(got), f"{tag}: a row returned twice"
        if len(got) < len(ids):
            assert len(got) == len(candidates), f"{tag}: padded with {len(candidates) - len(got)} candidates left out"
            return
        out = np.setdiff1d(candidates, got)
        if len(out) == 0:
            return
        sign = 1.0 if metric == "l2" else -1.0
        dk, bk = self.reference(metric, q, got[-1:])
        d, b = self.reference(metric, q, out)
        nearer = sign * (dk[0] - d) - (bk[0] + b)
        assert not np.any(nearer > 0), f"{tag}: rows {out[nearer > 0][:4]} left out but nearer than the k-th row"


def check_assignment(metric, rows, centroids, assign, tag, allowed=None):
    """Every row's centroid is its float64-nearest (among `allowed[i]`, an index array per row, when given) up to a near
    tie: the chosen centroid's float64 distance is within the two bounds of the best one's."""
    rows = np.asarray(rows)
    cent = np.asarray(centroids, dtype=np.float64)
    sign = 1.0 if metric == "l2" else -1.0
    assign = np.asarray(assign, dtype=np.int64)
    for i in range(rows.shape[0]):
        cand = np.arange(cent.shape[0]) if allowed is None else np.asarray(allowed[i], dtype=np.int64)
        assert assign[i] in cand, f"{tag}: row {i} assigned outside its candidates"
        q64 = rows[i].astype(np.float32).astype(np.float64)
        d, b = float_tree(metric, q64, cent[cand])
        key = sign * d
        best = np.nanargmin(key)
        j = int(np.flatnonzero(cand == assign[i])[0])
        assert key[j] - key[best] <= b[j] + b[best], \
            f"{tag}: row {i} assigned to {assign[i]}, float64-nearest is {cand[best]} by {key[j] - key[best]}"
