"""float64 reference of the exact scan and a checker with a stated error bound (CPU only).

The device computes every returned distance in fp32, in an order that depends on the kernel (warp reduction, tile
micro-kernel, re-score).  Whatever the order, and with or without FMA, an fp32 sum of d terms is within
d * 2^-24 * S of the exact sum, S = the sum of the terms' magnitudes; the per-pair bound used here is

    beta(q, r) = 2 * (d + 2) * 2^-24 * S(q, r)      S = sum (x_i - q_i)^2 (L2), sum |x_i q_i| (IP, cosine)

(the +2 covers the rounding of x_i - q_i and of the product of a one-term sum), plus 2^-23 * (1 + S) for cosine's
`1 - dot`.  A returned distance must lie within beta of its float64 value, and a row the device left out is a miss when
its float64 distance is below the last returned one by more than both rows' bounds.

`helpers.exact_topk` stays the recall-only ground truth; this module is the one that decides exactness.
"""
import numpy as np

U = 2.0 ** -24
_CHUNK = 1 << 22  # float64 elements of one [rows x queries] block


def _as64(X, Q):
    return np.asarray(X, np.float32).astype(np.float64), np.atleast_2d(np.asarray(Q, np.float32)).astype(np.float64)


def direct(X, Q, metric, q, rows):
    """float64 distances and bounds beta of query q to `rows`, from the fp32 inputs, the direct form of each metric."""
    X64, Q64 = _as64(X, Q)
    x, y = X64[rows], Q64[q]
    d = X64.shape[1]
    if metric == "l2":
        diff = x - y[None, :]
        dist = (diff * diff).sum(1)
        S = dist
    else:
        prod = x * y[None, :]
        dot = prod.sum(1)
        S = np.abs(prod).sum(1)
        dist = -dot if metric == "ip" else 1.0 - dot
    beta = 2.0 * (d + 2) * U * S
    if metric == "cosine":
        beta = beta + 2.0 * U * (1.0 + S)
    return dist, beta


def _screen(X64, Q64, metric, q_idx, r0, r1):
    """float64 distances of queries q_idx to rows [r0, r1) by matrix product, with a bound on their own error:
    the L2 expansion |x|^2 + |q|^2 - 2 x.q loses up to ~d * 2^-52 * (|x| + |q|)^2 to cancellation."""
    x, y = X64[r0:r1], Q64[q_idx]
    g = y @ x.T
    d = X64.shape[1]
    if metric == "l2":
        xx, yy = (x * x).sum(1), (y * y).sum(1)
        dist = yy[:, None] + xx[None, :] - 2.0 * g
        err = 4.0 * (d + 4) * 2.0 ** -52 * (np.sqrt(xx)[None, :] + np.sqrt(yy)[:, None]) ** 2
    else:
        dist = -g if metric == "ip" else 1.0 - g
        err = 4.0 * (d + 4) * 2.0 ** -52 * (np.abs(y) @ np.abs(x).T + 1.0)
    return dist, err


def _rows(n, admissible, row_range):
    r0, r1 = (0, n) if row_range is None else row_range
    ok = np.zeros(n, bool)
    ok[r0:r1] = True
    if admissible is not None:
        ok &= np.asarray(admissible, bool)
    return ok


def _blocks(X64, Q64):
    n, d = X64.shape
    rstep = max(1, min(n, _CHUNK // max(1, d)))
    qstep = max(1, min(Q64.shape[0], _CHUNK // rstep))
    for r0 in range(0, n, rstep):
        for q0 in range(0, Q64.shape[0], qstep):
            yield r0, min(n, r0 + rstep), q0, min(Q64.shape[0], q0 + qstep)


def _kth_upper(X64, Q64, metric, ok, k):
    """Per query, an upper bound of the k-th smallest float64 distance over the admissible rows (+inf if fewer)."""
    best = np.full((Q64.shape[0], k), np.inf)
    for r0, r1, q0, q1 in _blocks(X64, Q64):
        m = ok[r0:r1]
        if not m.any():
            continue
        dist, err = _screen(X64, Q64, metric, np.arange(q0, q1), r0, r1)
        v = np.concatenate([best[q0:q1], (dist + err)[:, m]], axis=1)
        best[q0:q1] = np.partition(v, k - 1, axis=1)[:, :k] if v.shape[1] > k else v
    return best.max(axis=1)


def _suspects(X64, Q64, metric, ok, cut):
    """Per query, the admissible rows whose float64 distance may be <= cut[q]."""
    out = [[] for _ in range(Q64.shape[0])]
    for r0, r1, q0, q1 in _blocks(X64, Q64):
        m = ok[r0:r1]
        if not m.any():
            continue
        dist, err = _screen(X64, Q64, metric, np.arange(q0, q1), r0, r1)
        qi, ri = np.nonzero(m[None, :] & (dist - err <= cut[q0:q1, None]))
        for q in np.unique(qi):
            out[q0 + q].append(ri[qi == q] + r0)
    return [np.concatenate(o) if o else np.zeros(0, np.int64) for o in out]


def ref_topk(X, Q, metric, k, admissible=None, row_range=None):
    """Exact top-k by float64 distance (ties by id) over admissible rows of [row_range): ids [nq, k] (-1 padded),
    distances [nq, k] (+inf padded), counts [nq].  The matrix-product screen only preselects a superset (its own
    error bound is the margin); the candidates are then recomputed in the direct form."""
    X64, Q64 = _as64(X, Q)
    ok = _rows(X64.shape[0], admissible, row_range)
    nq = Q64.shape[0]
    ids = np.full((nq, k), -1, np.int64)
    dist = np.full((nq, k), np.inf)
    counts = np.zeros(nq, np.int64)
    sus = _suspects(X64, Q64, metric, ok, _kth_upper(X64, Q64, metric, ok, k))
    for q in range(nq):
        cand = sus[q]
        dd, _ = direct(X, Q, metric, q, cand)
        order = np.lexsort((cand, dd))[:k]
        c = len(order)
        ids[q, :c], dist[q, :c], counts[q] = cand[order], dd[order], c
    return ids, dist, counts


def check_exact(ids, dists, counts, X, Q, metric, k_eff, admissible=None, row_range=None, what=""):
    """Assert that (ids, dists, counts) is an exact answer for every query: count = min(k_eff, admissible rows) with
    -1 / +inf padding after it, unique admissible ids, distances within beta of float64, non-decreasing with equal
    distances by ascending id, and no admissible row left out that is closer than the last returned by more than
    both bounds."""
    X64, Q64 = _as64(X, Q)
    ids, dists, counts = np.atleast_2d(ids), np.atleast_2d(dists), np.atleast_1d(counts)
    ok = _rows(X64.shape[0], admissible, row_range)
    n_ok = int(ok.sum())
    want = min(k_eff, n_ok)
    cuts = np.full(Q64.shape[0], -np.inf)
    returned = []
    for q in range(Q64.shape[0]):
        tag = "%s query %d" % (what, q)
        c = int(counts[q])
        assert c == want, "%s: count %d, expected %d" % (tag, c, want)
        assert np.all(ids[q, c:] == -1) and np.all(np.isinf(dists[q, c:])), "%s: bad padding after %d" % (tag, c)
        got = ids[q, :c].astype(np.int64)
        returned.append(got)
        assert len(set(got.tolist())) == c, "%s: repeated ids" % tag
        assert np.all((got >= 0) & (got < X64.shape[0])) and ok[got].all(), "%s: id not admissible" % tag
        if c == 0:
            continue
        gd = dists[q, :c].astype(np.float64)
        d64, beta = direct(X, Q, metric, q, got)
        bad = np.nonzero(np.abs(gd - d64) > beta)[0]
        assert bad.size == 0, "%s pos %d id %d: distance %r, float64 %r, bound %r" % (
            tag, bad[0], got[bad[0]], gd[bad[0]], d64[bad[0]], beta[bad[0]])
        step = np.diff(gd)
        assert np.all(step >= 0), "%s: distances decrease at position %d" % (tag, int(np.argmax(step < 0)))
        tie = np.nonzero(step == 0)[0]
        assert np.all(got[tie] < got[tie + 1]), "%s: equal distances not ordered by id" % tag
        cuts[q] = d64[-1] - beta[-1]
    if want == n_ok:
        return  # every admissible row was returned
    for q, sus in enumerate(_suspects(X64, Q64, metric, ok, cuts)):
        sus = sus[~np.isin(sus, returned[q])]
        if sus.size:
            sd, sb = direct(X, Q, metric, q, sus)
            miss = np.nonzero(sd + sb < cuts[q])[0]
            assert miss.size == 0, "%s query %d: row %d (float64 %r) is missing; last returned id %d" % (
                what, q, sus[miss[0]], sd[miss[0]], returned[q][-1])


# ---- host model of the coarse pass ---------------------------------------------------------------------------------
def round_bf16(a):
    """fp32 -> bf16 (round to nearest even), returned as fp32 values."""
    b = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32)


def round_tf32(a, mode="rn"):
    """fp32 -> tf32 (10 mantissa bits): "rn" round to nearest even, "rz" truncation."""
    b = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    if mode == "rn":
        b = b + 0xFFF + ((b >> 13) & 1)
    return (b & 0xFFFFE000).astype(np.uint32).view(np.float32)


COARSE_MODELS = {"bf16": [round_bf16], "tf32": [lambda a: round_tf32(a, "rn"), lambda a: round_tf32(a, "rz")]}


def coarse_ip(X, Q, rnd):
    """Coarse -dot of the wgmma pass: operands rounded by `rnd`, products summed in float64."""
    return -(rnd(Q).astype(np.float64) @ rnd(X).astype(np.float64).T)


def guard_model(X, Q, k, kp, rnd):
    """The guard of the coarse pass on an IP table: per query the coarse top-k' list, the exact top-k inside it,
    T = the k'-th coarse value, E = the batch's largest |coarse - exact| over the re-scored rows, and whether the
    current rule (e_k + 2E <= T) calls the query safe.  Returns (lists [nq, k'], safe [nq])."""
    C = coarse_ip(X, Q, rnd)
    E64 = -(np.asarray(Q, np.float32).astype(np.float64) @ np.asarray(X, np.float32).astype(np.float64).T)
    lists = np.argsort(C, axis=1, kind="stable")[:, :kp]
    rows = np.arange(Q.shape[0])[:, None]
    err = np.abs(C[rows, lists] - E64[rows, lists]).max()
    T = C[rows, lists][:, -1]
    e_k = np.sort(E64[rows, lists], axis=1)[:, k - 1]
    return lists, e_k + 2.0 * err <= T


def planted_ip_table(n=100_000, d=64, nq=64, seed=0, scale=10_000.0, margin=0.2):
    """Unit rows (IP) and a batch of nq copies of one unit query q, plus one planted row
    x = (best + margin) q + scale z, z a unit vector orthogonal to q, written over the last row.  x is the exact top-1
    (its fp32 dot is off by at most ~scale * d * 2^-24, far below the margin), while rounding its large components to
    bf16 / tf32 drops its coarse dot far below its exact value: z is the seeded candidate that drops it most in the
    worst of the coarse models.  Returns X, Q, the planted id."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    q = rng.standard_normal(d)
    q = (q / np.linalg.norm(q)).astype(np.float32)
    q64 = q.astype(np.float64)
    best = float((X.astype(np.float64) @ q64).max())
    Z = rng.standard_normal((4096, d))
    Z -= (Z @ q64)[:, None] * q64[None, :]
    Z /= np.linalg.norm(Z, axis=1, keepdims=True)
    cand = ((best + margin) * q64[None, :] + scale * Z).astype(np.float32)
    worst = np.full(len(cand), -np.inf)
    for fns in COARSE_MODELS.values():
        for rnd in fns:
            worst = np.maximum(worst, rnd(cand).astype(np.float64) @ rnd(q).astype(np.float64))
    X[n - 1] = cand[int(np.argmin(worst))]
    return X, np.repeat(q[None, :], nq, axis=0), n - 1
