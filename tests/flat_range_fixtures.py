"""Seeded data at the edges of float16's range for the fp16 flat search (csrc/flat.cu).

The GEMM rounds float32 operands to fp16.  Elements of magnitude >= 65520 become +-inf there, and elements below 2^-14
land in fp16's subnormals, where the rounding error is absolute (up to 2^-25) rather than 2^-11 of the value.  Each
fixture below is built so that one of these effects changes which rows the GEMM proposes.  They are shared by
test_gpu_flat_range.py (the GPU against the exact scan and the C oracle) and test_flat_bound_model.py (a numpy model of
the certificate that decides whether a query's candidates can be trusted).

A fixture is (x, q, nearest): rows, queries and, where the data was designed around one answer, the id every query's
exact top 1 must be (None otherwise).  `nq` sets the batch size, so that the same fixture also feeds the deep lists of
the Flat index, which need more than 256 queries.
"""
import numpy as np

FP16_MAX = 65504.0          # the largest finite fp16; 65519 still rounds to it, 65520 rounds to inf
OVERFLOW = (65520.0, 66000.0, 70000.0)


def data_overflow(metric, nq=8):
    """float32 rows with one row beyond fp16's range that is every query's exact top 1 (L2: (66000, 0, 0, 0) against
    queries near (60000, 0, 0, 0); MIP: (66000, 5000, 5000, 5000) against queries near (0, 1, 1, 1))."""
    rng = np.random.default_rng(101 if metric == "l2" else 102)
    n, z = 1024, 517
    if metric == "l2":
        x = rng.uniform(-30_000, 30_000, (n, 4))
        x[z] = (66_000, 0, 0, 0)
        q = np.column_stack([np.full(nq, 60_000.0), rng.uniform(-1, 1, (nq, 3))])
    else:
        x = rng.uniform(-1000, 1000, (n, 4))
        x[z] = (66_000, 5000, 5000, 5000)
        q = np.column_stack([np.zeros(nq), rng.uniform(0.5, 1.5, (nq, 3))])
    return x.astype(np.float32), q.astype(np.float32), z


def query_overflow(metric, dtype, nq=8):
    """Queries whose first element is >= 65520 (every other query of the batch stays in range) over rows whose first
    element is 0, except on every 8th row, where it is 1.  In fp16 such a query's key is NaN on most rows and -inf on
    the few others, so the lists hold only the rows with x0 = 1.  Under L2 the all-zero row 700 is the exact top 1 of
    every overflowing query (the designed answer returned; it says nothing of the in-range queries); under MIP the
    best rows are set by the other elements."""
    rng = np.random.default_rng(200 + {np.float32: 0, np.float16: 1, np.uint8: 2, np.int8: 3}[dtype])
    n, dim, z = 1024, 32, 700
    lo, hi = {np.float32: (600, 1000), np.float16: (600, 1000), np.uint8: (153, 255), np.int8: (110, 127)}[dtype]
    x = rng.uniform(lo, hi, (n, dim))
    if dtype != np.uint8:
        x = x * rng.choice((-1.0, 1.0), (n, dim))
    x = np.rint(x) if dtype in (np.uint8, np.int8) else x
    x[:, 0] = 0
    x[::8, 0] = 1
    x[z] = 0
    rest = 20.0 if metric == "l2" else 1000.0
    q = rng.uniform(-rest, rest, (nq, dim))
    q[:, 0] = rng.uniform(-1, 1, nq)
    over = np.arange(nq) % 2 == 0
    q[over, 0] = np.array(OVERFLOW)[np.arange(over.sum()) % len(OVERFLOW)]
    return x.astype(dtype), q.astype(np.float32), z if metric == "l2" else None


def overflowing(q):
    """Queries holding an element that rounds to inf in fp16."""
    return (np.abs(q.astype(np.float32)) >= 65520).any(axis=1)


def boundary(inf_row, nq=8):
    """Elements of exactly +-65504 and +-65519 (both round to the finite 65504) in rows and queries, queries holding
    +-65520 (rounds to inf), and -- with `inf_row` -- rows holding 65520 too."""
    rng = np.random.default_rng(300 + int(inf_row))
    n, dim = 1024, 8
    x = rng.uniform(-60_000, 60_000, (n, dim))
    edge = np.array([FP16_MAX, 65519.0, -FP16_MAX, -65519.0])
    x[rng.choice(n, 64, replace=False), rng.integers(0, dim, 64)] = edge[np.arange(64) % 4]
    if inf_row:
        x[[5, 333, 900], [0, 3, 7]] = (65_520.0, -65_520.0, 65_520.0)
    q = rng.uniform(-60_000, 60_000, (nq, dim))
    q[np.arange(nq), rng.integers(0, dim, nq)] = np.resize(np.array([FP16_MAX, 65519.0, 65520.0, -65520.0]), nq)
    return x.astype(np.float32), q.astype(np.float32), None


def thin_shell(scale, dim, n=2048, nq=8, seed=0):
    """Rows on a thin shell (|x|^2 spread over 1.0-1.2 of its smallest value) whose elements are about `scale`, below
    fp16's normal range for scale <= 6e-5.  Query 0 is the zero vector, the others 0.01 x a row."""
    rng = np.random.default_rng(400 + dim + seed)
    u = rng.standard_normal((n, dim))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    x = scale * np.sqrt(dim) * u * np.sqrt(1.0 + 0.2 * rng.random((n, 1)))
    q = 0.01 * x[rng.choice(n, nq, replace=False)]
    q[0] = 0
    return x.astype(np.float32), q.astype(np.float32), None


def subnormal_queries_u8(nq=8):
    """uint8 rows against float32 queries whose elements are 1e-7 .. 6e-5 (fp16 subnormals)."""
    rng = np.random.default_rng(500)
    x = rng.integers(0, 256, (4096, 16)).astype(np.uint8)
    q = np.exp(rng.uniform(np.log(1e-7), np.log(6e-5), (nq, 16))) * rng.choice((-1.0, 1.0), (nq, 16))
    return x, q.astype(np.float32), None


def touch_subnormals(v, rng, share=0.25):
    """About `share` of all elements replaced by values of magnitude 1e-7 .. 6e-5, random sign."""
    m = rng.random(v.shape) < share
    tiny = np.exp(rng.uniform(np.log(1e-7), np.log(6e-5), v.shape)) * rng.choice((-1.0, 1.0), v.shape)
    return np.where(m, tiny, v).astype(np.float32)


def tightness_control():
    """The clustered unit vectors of test_gpu_flat.py (40 000 x 96, 333 queries) with about a quarter of the elements,
    in rows and queries, replaced by fp16 subnormals: ordinary data on which every query must still verify."""
    from scalablevectorsearch_b200.synthetic import clustered_unit_vectors
    x, q = clustered_unit_vectors(40_000, 333, 96)
    rng = np.random.default_rng(600)
    return touch_subnormals(x, rng), touch_subnormals(q, rng), None
