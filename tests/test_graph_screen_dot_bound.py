"""CPU check of the graph screen's dot-product bound for inner-product and cosine indexes (graph_search.cu screen_fresh,
kind kScreenDot; sketch.cu dot_terms_kernel).  LB is restated in numpy with the kernel's directed rounding and must never
exceed the distance the graph kernel computes, emulated exactly: the fp32 dot product of the float4 path (32 lane fmaf
chains over float4 chunks, then the 5-step butterfly) or, for d % 4 != 0, of the scalar path, finished as -acc (IP) or
fl(1 - acc) (cosine).  Dropping any one term of the bound must be caught on some case, so that the check has teeth."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_graph_screen_bound import U, basis, fmaf, sketch  # noqa: E402

F32_MAX = float(np.finfo(np.float32).max)


def butterfly(acc, offsets):
    for o in offsets:
        acc = (acc + acc[:, np.arange(acc.shape[1]) ^ o]).astype(np.float32)
    return acc[:, 0]


def kernel_dot(X, q):
    """The graph kernel's fp32 dot product of every row of X with q: warp_rows_vec4 (d % 4 == 0) or warp_rows_scalar."""
    n, d = X.shape
    acc = np.zeros((n, 32), np.float32)
    if d % 4 == 0:
        for c0 in range(0, d // 4, 32):
            for lane in range(32):
                c = c0 + lane
                if c >= d // 4:
                    continue
                for k in range(4):
                    acc[:, lane] = fmaf(X[:, 4 * c + k], np.broadcast_to(q[4 * c + k], (n,)), acc[:, lane])
    else:
        for lane in range(32):
            for i in range(lane, d, 32):
                acc[:, lane] = fmaf(X[:, i], np.broadcast_to(q[i], (n,)), acc[:, lane])
    return butterfly(acc, (16, 8, 4, 2, 1))  # warp_sum


def ru(x64):
    """fp32 rounding toward +inf of float64 values (taken as exact)."""
    x64 = np.asarray(x64, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        f = x64.astype(np.float32)
        return np.where(f.astype(np.float64) < x64, np.nextafter(f, np.float32(np.inf)), f).astype(np.float32)


def add_ru(a, b):
    """__fadd_ru on fp32 arrays: TwoSum gives the exact sum s + e, then round up."""
    a64, b64 = np.asarray(a, np.float64), np.asarray(b, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        s = a64 + b64
        bb = s - a64
        e = (a64 - (s - bb)) + (b64 - bb)
        f = s.astype(np.float32)
        up = (f.astype(np.float64) < s) | ((f.astype(np.float64) == s) & (e > 0))
        return np.where(up, np.nextafter(f, np.float32(np.inf)), f).astype(np.float32)


def mul_ru(a, b):
    with np.errstate(over="ignore", invalid="ignore"):
        return ru(np.asarray(a, np.float64) * np.asarray(b, np.float64))  # fp32 x fp32 is exact in float64


def consts(d, m, eps, mu):
    """DotConsts (sketch.cu dot_consts) for a sketch of m floats."""
    nc = 4 * ((d + 127) // 128) + 5
    ns = 4 * (m // 32) + 3  # the screen's lane chains + butterfly
    epn = np.sqrt(m) * ((d + 2) * U / (1 - (d + 2) * U)) * np.sqrt(1 + eps)
    k = (1 / epn) * (1 + (d + 8) * 2.0 ** -52) * (1 + 2.0 ** -40)
    return dict(
        ay_rel=((1 + eps) * (m + 2) * (d + m + 6) * 2.0 ** -52 + max(1.0, eps) * 2.0 ** -52) * (1 + 2.0 ** -40),
        mu_norm=np.sqrt((mu.astype(np.float64) ** 2).sum()) * (1 + (d + 8) * 2.0 ** -52),
        k=k, s1=(np.sqrt(1 + eps) * k + 1) * (1 + 2.0 ** -40), eps1=eps * (1 + eps) * (1 + 2.0 ** -40),
        g_c=nc * U / (1 - nc * U) * (1 + 2.0 ** -40), g_s=ns * U / (1 - ns * U) * (1 + 2.0 ** -40),
        tiny=(nc + 8) * 2.0 ** -149)


def terms(V, P, mu, c):
    """dot_terms_kernel in float64: |A y| and <mu, y> rounded up, and the pieces a query needs."""
    y = V.astype(np.float64) - mu.astype(np.float64)
    w = y @ P.astype(np.float64).T
    r = y - w @ P.astype(np.float64)
    d = V.shape[1]
    up = 1 + (d + 8) * 2.0 ** -52
    yn = np.sqrt((y * y).sum(1)) * up
    ay = (np.sqrt((r * r).sum(1)) * up + yn * c["ay_rel"]) * (1 + 2.0 ** -50)
    my = y @ mu.astype(np.float64)
    muy = my + (d + 6) * 2.0 ** -52 * c["mu_norm"] * yn
    return ay, muy + np.abs(muy) * 2.0 ** -50, yn


def query_consts(q, P, mu, c, pq, eq, base, drop):
    ay, _, yn = terms(q[None, :], P, mu, c)
    d = q.shape[0]
    q64 = q.astype(np.float64)
    qn = np.sqrt((q64 * q64).sum()) * (1 + (d + 8) * 2.0 ** -52)
    q1n = yn[0] * (1 + 2.0 ** -52)
    qm = q64 @ mu.astype(np.float64)
    qmu = qm + (d + 6) * 2.0 ** -52 * qn * c["mu_norm"]
    pn = np.sqrt((pq.astype(np.float64) ** 2).sum()) * (1 + 2.0 ** -45)
    eq = float(eq)
    qm_n = qn * c["mu_norm"] * (1 + 2.0 ** -50)
    g_c = 0.0 if drop == "consumer" else c["g_c"]
    c0 = qmu + g_c * qm_n + c["tiny"]
    c0 = c0 + abs(c0) * 2.0 ** -50 - base
    c0 += abs(c0) * 2.0 ** -50
    if drop == "sketch":
        cex = 0.0
    else:
        cex = pn + eq + c["s1"] * (eq + c["g_s"] * pn)
    eps1 = 0.0 if drop == "eps" else c["eps1"]
    cex = (cex + c["k"] * (eps1 * q1n + g_c * qn)) * (1 + 2.0 ** -40)
    kq = qn * c["k"] * (1 + 2.0 ** -50)
    if not qm_n < 2.0 ** 125:
        kq = np.inf
    if not np.isfinite(qn):
        c0 = np.nan
    return ru(c0), ru(cex), ru(0.0 if drop == "residual" else ay[0]), ru(kq)


def screen_dot(S, pq):
    """The screen's 8-lane fp32 dot product of the sketches: lane j chains floats 4j .. 4j + 3 (+ 32 at m = 64)."""
    n, m = S.shape
    acc = np.zeros((n, 8), np.float32)
    for h in range(m // 32):
        for j in range(8):
            for k in range(4):
                i = 32 * h + 4 * j + k
                acc[:, j] = fmaf(S[:, i], np.broadcast_to(pq[i], (n,)), acc[:, j])
    return butterfly(acc, (1, 2, 4))


def lower_bound(S, ex, ay, muy, pq, qc):
    """LB = -0 - UB rounded down, UB = s^ + (C0 - base) + <mu, y> + |A q'| |A y| + C_ex ex_x, each step rounded up;
    NaN where the id is kept whatever its key (UB not finite, or K ex_x >= 2^125)."""
    c0, cex, aq, kq = qc
    ub = add_ru(add_ru(screen_dot(S, pq), c0), muy)
    ub = add_ru(ub, mul_ru(aq, ay))
    ub = add_ru(ub, mul_ru(cex, ex))
    ok = (mul_ru(kq, ex) < np.float32(2.0 ** 125)) & (np.abs(ub) <= F32_MAX)
    return np.where(ok, -ub, np.float32(np.nan))


def setup(X, m, centred=True, stretch=1.0, mu=None):
    d = X.shape[1]
    P, mu0, eps = basis(X, min(m, d))
    if mu is None:
        mu = mu0 if centred else np.zeros_like(mu0)
    if P.shape[0] < m:  # fewer dimensions than sketch floats: zero rows keep sigma_max(P~)^2 <= 1 + eps
        P = np.vstack([P, np.zeros((m - P.shape[0], d), np.float32)])
    if stretch != 1.0:  # a basis that is not orthonormal: the bound holds for any P~ with its eps
        P = (P * np.float32(stretch)).astype(np.float32)
        G = P.astype(np.float64) @ P.astype(np.float64).T
        eps = np.abs(G - np.eye(m)).sum(1).max() + m * d * 2.0 ** -52
    return P, mu, eps


def run_case(X, m, metric, queries="near", drop=None, **kw):
    """Largest LB - D over the kept-or-dropped ids of a sweep of queries (<= 0: the bound holds) and the largest LB."""
    d = X.shape[1]
    P, mu, eps = setup(X, m, **kw)
    c = consts(d, m, eps, mu)
    S, ex = sketch(X, P, mu, eps)
    ay, muy, _ = terms(X, P, mu, c)
    ay, muy = ru(ay), ru(muy)
    base = 1.0 if metric == "cosine" else 0.0
    worst = best = -np.inf
    for qi in range(0, X.shape[0] - 1, 40):
        x0, x1 = X[qi].astype(np.float64), X[qi + 1].astype(np.float64)
        if queries == "far":  # a point unrelated to the table: its products with the rows cancel
            q = 1000.0 * np.random.default_rng(qi).standard_normal(d)
        else:
            q = {"near": x0 + 1e-3 * (qi % 3), "row": x1, "close": x0 + 1e-4 * (x1 - x0)}[queries]
        if metric == "cosine":
            q = q / np.linalg.norm(q)
        q = q.astype(np.float32)
        sq, eq = sketch(q[None, :], P, mu, eps)
        qc = query_consts(q, P, mu, c, sq[0], eq[0], base, drop)
        lb = lower_bound(S, ex, ay, muy, sq[0], qc)
        acc = kernel_dot(X, q)
        D = (np.float32(1) - acc).astype(np.float32) if metric == "cosine" else -acc
        diff = lb.astype(np.float64) - D.astype(np.float64)
        if np.any(np.isfinite(diff)):
            worst = max(worst, float(np.nanmax(diff)))
            best = max(best, float(np.nanmax(lb)))
    return worst, best


def normalise(X):
    return (X / np.linalg.norm(X.astype(np.float64), axis=1, keepdims=True)).astype(np.float32)


def tables():
    rng = np.random.default_rng(11)
    out = []
    for d in (4, 36, 130, 768):
        R = rng.standard_normal((300, d)).astype(np.float32)
        rank = min(d, 6)
        Z = (rng.standard_normal((300, rank)) @ np.linalg.qr(rng.standard_normal((d, rank)))[0].T).astype(np.float32)
        O = (1000.0 + 1e-2 * rng.standard_normal((300, d))).astype(np.float32)
        # rows whose norms spread over 10^6
        W = (Z.astype(np.float64) * 10.0 ** rng.uniform(-3, 3, size=(300, 1)) + 1e-3 * R).astype(np.float32)
        out += [("ip", "random", d, R), ("ip", "low-rank", d, Z), ("ip", "offset", d, O), ("ip", "norms", d, W)]
        out += [("cosine", "random", d, normalise(R)), ("cosine", "low-rank", d, normalise(Z + 0.3)),
                ("cosine", "offset", d, normalise(O))]
    return out


TABLES = {(mt, name, d): X for mt, name, d, X in tables()}


@pytest.mark.parametrize("metric,name,d", sorted(TABLES))
@pytest.mark.parametrize("m", [32, 64])
def test_bound_never_exceeds_the_kernel_distance(metric, name, d, m):
    X = TABLES[(metric, name, d)]
    for queries in ("near", "row", "close"):
        worst, _ = run_case(X, m, metric, queries)
        assert worst <= 0.0, "%s LB exceeds the kernel's distance by %g (%s queries)" % (metric, worst, queries)


def test_bound_is_useful_on_low_rank_rows():
    """A bound that never rises above the queue's worst distance would be valid and useless: on low-rank rows it comes
    within a small fraction of the distances."""
    for metric in ("ip", "cosine"):
        X = TABLES[(metric, "low-rank", 768)]
        P, mu, eps = setup(X, 32)
        c = consts(768, 32, eps, mu)
        S, ex = sketch(X, P, mu, eps)
        ay, muy, _ = terms(X, P, mu, c)
        q = X[5]
        sq, eq = sketch(q[None, :], P, mu, eps)
        lb = lower_bound(S, ex, ru(ay), ru(muy), sq[0], query_consts(q, P, mu, c, sq[0], eq[0], 1.0 if metric == "cosine" else 0.0, None))
        acc = kernel_dot(X, q)
        D = (np.float32(1) - acc) if metric == "cosine" else -acc
        spread = float(D.max() - D.min())
        assert np.all(np.isfinite(lb)) and float(np.max(D - lb)) < 0.01 * spread, (metric, float(np.max(D - lb)), spread)


def test_sketches_without_the_mean_collapse():
    """Offset rows (1000 + N(0, 1e-2)) sketched without taking the mean out: the sketches' error bounds (|y| ~ 2.8e4)
    dwarf the spread of the dot products, so the bound must fall below every distance by far, not lie."""
    X = TABLES[("ip", "offset", 768)]
    acc = np.concatenate([kernel_dot(X, X[i]) for i in (0, 40)])
    spread = float(acc.max() - acc.min())
    for m in (32, 64):
        worst, best = run_case(X, m, "ip", "near", centred=False)
        assert worst < -10 * spread, (worst, spread)
    assert run_case(X, 32, "ip", "near")[0] > -10 * spread  # with the mean out the same rows keep a useful bound


def caught(drop, cases):
    return any(run_case(X, m, metric, queries, drop=drop, **kw)[0] > 0.0 for X, m, metric, queries, kw in cases)


def test_residual_term_is_needed():
    cases = [(TABLES[("ip", "random", d)], 32, "ip", "row", {}) for d in (36, 768)]
    assert caught("residual", cases), "dropping |A q'| |A y| went unnoticed"


def test_eps_term_is_needed():
    """A basis scaled by 1.05 has eps ~ 0.1: the bound must pay eps (1 + eps) |q'| |y| for q'^T (A - A^2) y."""
    cases = [(TABLES[("ip", name, d)], 32, "ip", qk, {"stretch": 1.05}) for name in ("low-rank", "random")
             for d in (36, 768) for qk in ("row", "close")]
    assert caught("eps", cases), "dropping eps (1 + eps) |q'| |y| went unnoticed"


def test_sketch_error_terms_are_needed():
    """Rows whose norms spread over 10^6: against the largest rows, the sketches' rounding is the largest error."""
    cases = [(TABLES[("ip", "norms", 768)], 32, "ip", qk, {}) for qk in ("row", "close")]
    assert caught("sketch", cases), "dropping the sketches' error terms went unnoticed"


def test_consumer_rounding_term_is_needed():
    """Every row equal to the mean: the sketches, their errors and the residuals vanish, and UB is <q, mu> rounded up
    plus the consumer's own rounding, which queries whose products cancel make large."""
    rng = np.random.default_rng(23)
    cases = []
    for d in (130, 768):
        mu = (1000.0 * rng.standard_normal(d)).astype(np.float32)
        cases.append((np.tile(mu, (81, 1)), 32, "ip", "far", {"mu": mu}))
    assert caught("consumer", cases), "dropping gamma_{n_c} |q| |x| went unnoticed"


def test_overflowing_rows_and_non_finite_queries_are_kept():
    rng = np.random.default_rng(3)
    X = (rng.standard_normal((64, 128)) * 0.1).astype(np.float32)
    P, mu, eps = setup(X, 32)  # the basis and mean of the rows before row 7 grows, as after an extension
    X[7] *= np.float32(2e38) / np.abs(X[7]).max()  # |q| |x| beyond fp32 for a query of norm ~1
    c = consts(128, 32, eps, mu)
    S, ex = sketch(X, P, mu, eps)
    ay, muy, _ = terms(X, P, mu, c)
    q = X[3].copy()
    sq, eq = sketch(q[None, :], P, mu, eps)
    lb = lower_bound(S, ex, ru(ay), ru(muy), sq[0], query_consts(q, P, mu, c, sq[0], eq[0], 0.0, None))
    assert np.isnan(lb[7]) and np.isfinite(np.delete(lb, 7)).any()
    q[0] = np.inf
    with np.errstate(all="ignore"):
        sq, eq = sketch(q[None, :], P, mu, eps)
        lb = lower_bound(S, ex, ru(ay), ru(muy), sq[0], query_consts(q, P, mu, c, sq[0], eq[0], 0.0, None))
    assert np.all(np.isnan(lb))
