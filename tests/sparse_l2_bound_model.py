"""numpy restatement of the L2 screen's lower bound (sparse_l2_lower_bound, vectordb_b200/csrc/sparse_inverted.cu).

For a (row, query) pair with m_r and m_q elements, the fp32 dot of their matched elements `dot` (summed as the posting
lists sum it), the stored fp32 |row|^2 `rn` and the query's fp32 |q|^2 `qn`, with m = m_r + m_q, u = 2^-24,
eta = 2^-149 and 1 - gamma_k >= 1 - (9/8) k u (k u <= 2^-4):

    R2 >= max(0, (1 - gamma_{m_r}) (rn - m_r eta))          Q2 >= max(0, (1 - gamma_{m_q}) (qn - m_q eta))
    D  >= max(0, (1 - gamma_m) (R2 + Q2) - 2 dot - 2 m eta)
    LB  = (1 - gamma_{m+2}) D - m eta  <=  D_ref

every step rounded toward -inf in float64 (exactly: the rounding error of each add and multiply is recovered with
TwoSum / Dekker's product), and LB rounded toward -inf to float32.  Pairs with a non-finite input or m + 2 > 2^20 get
+inf (always re-scored)."""
import numpy as np

U = 2.0 ** -24
ETA = 2.0 ** -149
MAX_TERMS = 1 << 20
_SPLIT = 2.0 ** 27 + 1.0


def _add_rd(a, b):
    s = a + b
    bb = s - a
    err = (a - (s - bb)) + (b - bb)   # a + b = s + err exactly
    return np.where(err < 0, np.nextafter(s, -np.inf), s)


def _split(a):
    c = _SPLIT * a
    hi = c - (c - a)
    return hi, a - hi


def _mul_rd(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    err = ((ah * bh - p) + ah * bl + al * bh) + al * bl   # a * b = p + err exactly
    return np.where(err < 0, np.nextafter(p, -np.inf), p)


def _one_minus_gamma(k):
    return 1.0 - np.asarray(k, np.float64) * (1.125 * U)   # exact for k <= 2^20


def lower_bound(dot, rn, qn, m_r, m_q):
    """float32 LB of every pair (broadcast: dot [nq x n], rn and m_r [n], qn and m_q [nq, 1]); +inf where not covered."""
    dot = np.asarray(dot, np.float32)
    rn, qn = np.asarray(rn, np.float32), np.asarray(qn, np.float32)
    m_r, m_q = np.asarray(m_r, np.int64), np.asarray(m_q, np.int64)
    m = m_r + m_q
    covered = np.isfinite(dot) & np.isfinite(rn) & np.isfinite(qn) & (m + 2 <= MAX_TERMS)
    with np.errstate(all="ignore"):
        d64, r64, q64 = dot.astype(np.float64), rn.astype(np.float64), qn.astype(np.float64)
        r2 = np.maximum(0.0, _mul_rd(_one_minus_gamma(m_r), _add_rd(r64, -m_r * ETA)))
        q2 = np.maximum(0.0, _mul_rd(_one_minus_gamma(m_q), _add_rd(q64, -m_q * ETA)))
        d = _mul_rd(_one_minus_gamma(m), _add_rd(r2, q2))
        d = _add_rd(_add_rd(d, -2.0 * d64), -2.0 * m * ETA)
        lb = _add_rd(_mul_rd(_one_minus_gamma(m + 2), np.maximum(d, 0.0)), -m * ETA)
        f = lb.astype(np.float32)
        f = np.where(f.astype(np.float64) > lb, np.nextafter(f, np.float32(-np.inf)), f)
    return np.where(covered, f, np.float32(np.inf)).astype(np.float32)


def csr_norm2(csr):
    """Sequential fp32 sum of squares of each CSR row in index order (pack_sparse's |row|^2)."""
    off, _, val = csr
    lens = np.diff(off)
    s = np.zeros(lens.size, np.float32)
    with np.errstate(all="ignore"):
        for j in range(int(lens.max(initial=0))):
            has = np.nonzero(lens > j)[0]
            v = val[off[has] + j]
            s[has] = s[has] + v * v
    return s


def to_csr(rows):
    """[(indices, values)] -> (int64 offsets, int64 indices, float32 values)."""
    off = np.zeros(len(rows) + 1, np.int64)
    off[1:] = np.cumsum([len(r[0]) for r in rows])
    idx = np.concatenate([np.asarray(r[0], np.int64) for r in rows]) if off[-1] else np.zeros(0, np.int64)
    val = np.concatenate([np.asarray(r[1], np.float32) for r in rows]) if off[-1] else np.zeros(0, np.float32)
    return off, idx, val.astype(np.float32)


def adversarial(seed, n_plain=200):
    """Rows and queries (CSR, vocabulary 64) that stress the bound: values near 1e19 whose squares overflow once two are
    summed, values near 1e-23 whose products underflow, NaN and +-inf values, rows equal to a query and rows that are a
    query plus 1 ulp (in one element or in all: cancellation), 30 % empty rows, and ordinary rows."""
    vocab = 64
    rng = np.random.default_rng(seed)
    f32 = np.float32

    def plain(k, scale=1.0):
        idx = np.sort(rng.choice(vocab, size=k, replace=False))
        return idx, ((rng.random(k, dtype=f32) * 2 - 0.5) * f32(scale)).astype(f32)

    qs = [plain(12), plain(20, 0.1),
          (np.array([3, 9, 40]), np.array([1.1e19, -0.7e19, 2.0], f32)),          # |q|^2 ~ 1.7e38, finite
          (np.array([3, 9, 40, 41]), np.array([1.5e19, 1.5e19, 1.0, 1.0], f32)),  # |q|^2 overflows
          (np.array([1, 2, 5, 7]), np.array([1e-23, -3e-23, 2e-23, 1e-22], f32)),
          (np.array([1, 2, 50]), np.array([1e-23, 0.5, 1.0], f32)),
          (np.array([4, 8]), np.array([np.nan, 1.0], f32)),
          (np.array([4, 8]), np.array([np.inf, 1.0], f32)),
          (np.array([6]), np.array([-np.inf], f32)),
          (np.zeros(0, np.int64), np.zeros(0, f32))]
    rows = []
    for qi, qv in qs:
        rows.append((qi, qv.copy()))                                          # equal to the query
        if qi.size:
            one = qv.copy()
            one[0] = np.nextafter(one[0], f32(np.inf))
            rows.append((qi, one))                                            # + 1 ulp in one element
            rows.append((qi, np.nextafter(qv, f32(np.inf)).astype(f32)))      # + 1 ulp in every element
            rows.append((qi, (qv * f32(1.0000001)).astype(f32)))
    rows += [(np.array([3]), np.array([1e19], f32)), (np.array([3, 9]), np.array([1.5e19, 1.5e19], f32)),
             (np.array([3, 9, 40]), np.array([1.1e19, -0.7e19, 2.5], f32)), (np.array([9, 60]), np.array([-1e19, 3.0], f32)),
             (np.array([3]), np.array([-1.5e19], f32)),                       # (a - b)^2 overflows: D_ref = +inf
             (np.array([1, 2, 5]), np.array([1e-23, 1e-23, 1e-23], f32)), (np.array([1, 7, 9]), np.array([3e-23, -1e-22, 1e-30], f32)),
             (np.array([2, 4]), np.array([np.nan, 1.0], f32)), (np.array([4, 8]), np.array([np.inf, 0.0], f32)),
             (np.array([6, 8]), np.array([-np.inf, 1.0], f32)), (np.array([0, 63]), np.array([0.0, -0.0], f32))]
    rows += [plain(int(rng.integers(1, 30))) for _ in range(n_plain)]
    n_empty = int(0.3 * len(rows) / 0.7)
    rows += [(np.zeros(0, np.int64), np.zeros(0, f32))] * n_empty
    order = rng.permutation(len(rows))
    return to_csr([rows[i] for i in order]), to_csr(qs), vocab
