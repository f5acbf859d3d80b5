"""CPU check of the graph screen's lower bound (graph_search.cu screen_fresh, sketch.cu): restated in numpy with the
kernel's directed rounding, it must never exceed the fp32 L2 distance the graph kernel computes, emulated exactly
(32 lane fmaf chains over float4 chunks, then the 5-step butterfly).  A bound with one of its factors dropped must be
caught on some case, so that the check has teeth."""
import numpy as np
import pytest

U = 2.0 ** -24


def fmaf(a, b, c):
    """Exact fmaf(a, b, c) on fp32 arrays: the product is exact in float64; TwoSum keeps the sum exact."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    # correct the one case float64 -> fp32 rounding can get wrong: s exactly halfway between two fp32 values
    up = np.nextafter(r, np.float32(np.inf)).astype(np.float64)
    dn = np.nextafter(r, np.float32(-np.inf)).astype(np.float64)
    half_above = (r64 > s) & ((r64 - s) * 2 == (r64 - dn)) & (e < 0)
    half_below = (r64 < s) & ((s - r64) * 2 == (up - r64)) & (e > 0)
    r = np.where(half_above, np.nextafter(r, np.float32(-np.inf)), r)
    r = np.where(half_below, np.nextafter(r, np.float32(np.inf)), r)
    return r.astype(np.float32)


def kernel_l2(X, q):
    """The graph kernel's fp32 L2 distance of every row of X to q (warp_rows_vec4 + warp_sum)."""
    n, d = X.shape
    d4 = (d + 3) // 4
    Xp = np.zeros((n, d4 * 4), np.float32)
    Xp[:, :d] = X
    qp = np.zeros(d4 * 4, np.float32)
    qp[:d] = q
    acc = np.zeros((n, 32), np.float32)
    for c0 in range(0, d4, 32):
        for lane in range(32):
            c = c0 + lane
            if c >= d4:
                continue
            for k in range(4):
                dd = (Xp[:, 4 * c + k] - qp[4 * c + k]).astype(np.float32)
                acc[:, lane] = fmaf(dd, dd, acc[:, lane])
    for o in (16, 8, 4, 2, 1):
        acc = (acc + acc[:, np.arange(32) ^ o]).astype(np.float32)
    return acc[:, 0]


def round_down(x):
    f = np.float32(x)
    return np.nextafter(f, np.float32(0)) if float(f) > x else f


def rd(x64):
    """fp32 rounding toward -inf of exact float64 values."""
    f = x64.astype(np.float32)
    return np.where(f.astype(np.float64) > x64, np.nextafter(f, np.float32(-np.inf)), f).astype(np.float32)


def sqrt_rd(t):
    f = rd(np.sqrt(t.astype(np.float64)))
    return np.where(f.astype(np.float64) ** 2 > t.astype(np.float64), np.nextafter(f, np.float32(-np.inf)), f).astype(np.float32)


def basis(X, m):
    Xc = X.astype(np.float64) - X.astype(np.float64).mean(0)
    w, V = np.linalg.eigh(Xc.T @ Xc)
    P = V[:, ::-1][:, :m].T.astype(np.float32)  # [m x d]
    G = P.astype(np.float64) @ P.astype(np.float64).T
    eps = np.abs(G - np.eye(m)).sum(1).max() + m * X.shape[1] * 2.0 ** -52
    mu = X.astype(np.float64).mean(0).astype(np.float32)
    return P, mu, eps


def sketch(X, P, mu, eps):
    """sketch_rows_kernel: per component an fp32 fmaf chain over k of P~_jk fl(x_k - mu_k), and the bound
    ex = sqrt(m) (gamma_{d+2} sqrt(1 + eps) |x - mu| + d 2^-149) on its error, rounded up."""
    n, d = X.shape
    m = P.shape[0]
    Dh = (X - mu).astype(np.float32)
    v = np.zeros((n, m), np.float32)
    for k in range(d):
        v = fmaf(np.broadcast_to(P[:, k], (n, m)), np.broadcast_to(Dh[:, k:k + 1], (n, m)), v)
    gam = (d + 2) * U / (1 - (d + 2) * U)
    nrm = np.sqrt(((X.astype(np.float64) - mu.astype(np.float64)) ** 2).sum(1)) * (1 + 2.0 ** -40)
    ex = (nrm * np.sqrt(m) * gam * np.sqrt(1 + eps) + np.sqrt(m) * d * 2.0 ** -149) * (1 + 2.0 ** -40)
    ex32 = ex.astype(np.float32)
    ex32 = np.where(ex32.astype(np.float64) < ex, np.nextafter(ex32, np.float32(np.inf)), ex32)
    return v, ex32


def lower_bound(sx, ex, sq, eq, d, eps, drop=None):
    """screen_fresh: LB = [(sqrt(l^ (1 - gamma_{m+2})) - ex - E_q)+]^2 (1 - 2 (d + 2) 2^-24) / (1 + eps), rounded down."""
    m = sx.shape[1]
    g = round_down(1.0 - (m + 2) * U / (1.0 - (m + 2) * U))
    scale = round_down((1.0 - 2.0 * (d + 2) * U) / (1.0 + eps))
    if drop == "scale":
        scale = np.float32(1.0)
    # eight lanes per id: lane j chains sketch floats 4j .. 4j + 3 (+ 32 at m = 64), then a 3-step butterfly
    n = sx.shape[0]
    acc = np.zeros((n, 8), np.float32)
    for h in range(m // 32):
        for j in range(8):
            for k in range(4):
                i = 32 * h + 4 * j + k
                dd = (sx[:, i] - sq[i]).astype(np.float32)
                acc[:, j] = fmaf(dd, dd, acc[:, j])
    for o in (1, 2, 4):
        acc = (acc + acc[:, np.arange(8) ^ o]).astype(np.float32)
    lhat = acc[:, 0]
    r = sqrt_rd(rd(lhat.astype(np.float64) * float(g)))
    if drop != "ex":
        r = rd(r.astype(np.float64) - ex.astype(np.float64))
        r = rd(r.astype(np.float64) - float(eq))
    lb = rd(rd(r.astype(np.float64) ** 2).astype(np.float64) * float(scale))
    return np.where(r > 0, lb, np.float32(0)), lhat


def tables():
    rng = np.random.default_rng(7)
    out = []
    for d in (4, 36, 768):
        out.append(("random", d, rng.standard_normal((400, d)).astype(np.float32)))
        rank = min(d, 6)
        Z = rng.standard_normal((400, rank)) @ np.linalg.qr(rng.standard_normal((d, rank)))[0].T
        out.append(("low-rank", d, Z.astype(np.float32)))
        out.append(("offset", d, (1000.0 + 1e-2 * rng.standard_normal((400, d))).astype(np.float32)))
    return out


def cases():
    for name, d, X in tables():
        for m in (32, 64):
            yield name, d, X, m


def run_case(X, m, drop=None, queries="near", centred=True):
    d = X.shape[1]
    P, mu, eps = basis(X, min(m, d))
    if not centred:
        mu = np.zeros_like(mu)
    if P.shape[0] < m:  # fewer dimensions than sketch floats: zero rows keep sigma_max(P~)^2 <= 1 + eps
        P = np.vstack([P, np.zeros((m - P.shape[0], d), np.float32)])
    S, ex = sketch(X, P, mu, eps)
    worst = best_lb = -np.inf
    for qi in range(0, X.shape[0], 40):
        # "near": a row moved off the table by 1e-3 in every coordinate; "row": another row (in the table's subspace, so
        # the sketch carries the whole distance); "close": a row moved 1e-4 of the way to the next one (distances far
        # below the sketch's rounding, which only the error terms ex and E_q cover)
        x0, x1 = X[qi].astype(np.float64), X[qi + 1].astype(np.float64)
        q = {"near": x0 + 1e-3 * (qi % 3), "row": x1, "close": x0 + 1e-4 * (x1 - x0)}[queries].astype(np.float32)
        sq, eq = sketch(q[None, :].astype(np.float32), P, mu, eps)
        lb, _ = lower_bound(S, ex, sq[0], eq[0], d, eps, drop)
        D = kernel_l2(X, q)
        worst = max(worst, float(np.max(lb.astype(np.float64) - D.astype(np.float64))))
        best_lb = max(best_lb, float(lb.max()))
    return worst, best_lb


@pytest.mark.parametrize("name,d,m", [(n, d, m) for n, d, _, m in cases()])
def test_bound_never_exceeds_the_kernel_distance(name, d, m):
    X = {(n, dd): x for n, dd, x in tables()}[(name, d)]
    for queries in ("near", "row", "close"):
        worst, _ = run_case(X, m, queries=queries)
        assert worst <= 0.0, "LB exceeds the kernel's fp32 distance by %g" % worst


def test_offset_rows_collapse():
    """Rows at 1000 + N(0, 1e-2) sketched without taking the mean out: the rounding of sketches of norm ~2.8e4 is far
    above the distances (~0.4), so the bound must collapse to 0 for every pair, not lie."""
    X = [x for n, d, x in tables() if n == "offset" and d == 768][0]
    for m in (32, 64):
        worst, best_lb = run_case(X, m, centred=False)
        assert worst <= 0.0 and best_lb <= 0.0, (worst, best_lb)
    # with the mean out, the same rows keep a useful bound
    assert run_case(X, 32)[1] > 0.0


def test_weakened_bound_is_caught():
    caught = False
    for name, d, X in tables():
        if name != "low-rank" or d < 36:
            continue
        worst, _ = run_case(X, 32, drop="ex", queries="close")
        caught |= worst > 0.0
    assert caught, "dropping the sketches' error bounds went unnoticed: the check has no teeth"


def test_scale_factor_is_needed():
    """The factor (1 - 2 (d + 2) 2^-24) / (1 + eps) covers two facts, each shown here to occur: the kernel's fp32 sum can
    fall below the exact distance, and an fp32-rounded basis can stretch a vector (sigma_max(P~) > 1)."""
    below = stretch = False
    for name, d, X in tables():
        if d < 36:
            continue
        q = X[0] + np.float32(1e-3)
        exact = ((X.astype(np.float64) - q.astype(np.float64)) ** 2).sum(1)
        below |= bool(np.any(kernel_l2(X, q).astype(np.float64) < exact))
        P, _, eps = basis(X, 32)
        stretch |= float(np.linalg.svd(P.astype(np.float64), compute_uv=False)[0]) > 1.0
        assert float(np.linalg.svd(P.astype(np.float64), compute_uv=False)[0]) ** 2 <= 1.0 + eps
    assert below and stretch, (below, stretch)
