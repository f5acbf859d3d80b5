"""CPU tests of the float64 exact-scan reference and its checker (tests/exact_ref.py), and of the host model that
shows the coarse-pass guard's hole for large-norm rows."""
import numpy as np
import pytest

import exact_ref as er
from helpers import exact_topk


def _answer(X, Q, metric, k, admissible=None):
    ids, d64, cnt = er.ref_topk(X, Q, metric, k, admissible)
    dists = np.where(ids >= 0, d64, np.inf).astype(np.float32).astype(np.float64)
    return ids, dists, cnt


@pytest.mark.parametrize("metric", ["l2", "ip", "cosine"])
def test_ref_topk_matches_float64_argsort(metric):
    rng = np.random.default_rng(1)
    X, Q = rng.random((3000, 19), dtype=np.float32), rng.random((25, 19), dtype=np.float32)
    if metric == "cosine":
        X /= np.linalg.norm(X, axis=1, keepdims=True)
        Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    ids, _, cnt = er.ref_topk(X, Q, metric, 12)
    assert np.all(cnt == 12)
    assert np.array_equal(ids, exact_topk(X, Q, 12, metric))


def test_ref_topk_survives_large_offsets():
    """Rows at 1000 + N(0, 1e-2): the L2 expansion cancels ~7 digits, the reference must still rank exactly."""
    rng = np.random.default_rng(2)
    X = (1000.0 + 1e-2 * rng.standard_normal((4000, 32))).astype(np.float32)
    Q = (1000.0 + 1e-2 * rng.standard_normal((6, 32))).astype(np.float32)
    ids, d64, _ = er.ref_topk(X, Q, "l2", 10)
    X64, Q64 = X.astype(np.float64), Q.astype(np.float64)
    for q in range(6):
        full = ((X64 - Q64[q]) ** 2).sum(1)
        assert np.array_equal(ids[q], np.lexsort((np.arange(len(full)), full))[:10])
        assert np.array_equal(d64[q], full[ids[q]])


def test_ref_topk_admissible_and_row_range():
    rng = np.random.default_rng(3)
    X, Q = rng.random((500, 8), dtype=np.float32), rng.random((4, 8), dtype=np.float32)
    ok = rng.random(500) < 0.02
    ids, _, cnt = er.ref_topk(X, Q, "l2", 20, admissible=ok, row_range=(100, 500))
    n_ok = int(ok[100:].sum())
    assert np.all(cnt == min(20, n_ok))
    assert np.all(ids[:, n_ok:] == -1) and np.all(ok[ids[:, :n_ok]]) and ids[:, :n_ok].min() >= 100


@pytest.fixture(scope="module")
def table():
    rng = np.random.default_rng(4)
    X, Q = rng.random((2000, 24), dtype=np.float32), rng.random((8, 24), dtype=np.float32)
    X[1500] = X[200]                      # an exact tie: two ids at one distance
    Q[3] = X[200] + 1e-3
    return X, Q


def test_checker_accepts_correct_answers(table):
    X, Q = table
    for metric in ("l2", "ip"):
        ids, d, cnt = _answer(X, Q, metric, 10)
        er.check_exact(ids, d, cnt, X, Q, metric, 10)
    assert list(_answer(X, Q, "l2", 10)[0][3, :2]) == [200, 1500]
    ok = np.ones(len(X), bool)
    ok[:1000] = False
    ids, d, cnt = _answer(X, Q, "l2", 10, ok)
    er.check_exact(ids, d, cnt, X, Q, "l2", 10, admissible=ok)
    few = np.zeros(len(X), bool)
    few[[5, 77, 900]] = True              # fewer admissible rows than k: count 3, then -1 / +inf
    ids, d, cnt = _answer(X, Q, "l2", 10, few)
    er.check_exact(ids, d, cnt, X, Q, "l2", 10, admissible=few)


def _corrupt(kind, ids, d, cnt, X, Q):
    ids, d, cnt = ids.copy(), d.copy(), cnt.copy()
    q = 3
    if kind == "dropped":                 # the true 4th neighbour left out, the 11th taken in
        top, d11, _ = er.ref_topk(X, Q[q:q + 1], "l2", 11)
        keep = [0, 1, 2, 4, 5, 6, 7, 8, 9, 10]
        ids[q], d[q] = top[0, keep], d11[0, keep].astype(np.float32)
    elif kind == "swapped":
        ids[q, [4, 5]] = ids[q, [5, 4]]
        d[q, [4, 5]] = d[q, [5, 4]]
    elif kind == "distance":
        _, beta = er.direct(X, Q, "l2", q, ids[q, 2:3])
        d[q, 2] += 10 * beta[0]
    elif kind == "deleted":
        pass                              # ids unchanged; the caller marks one of them deleted
    elif kind == "count":
        cnt[q] -= 1
        ids[q, cnt[q]:], d[q, cnt[q]:] = -1, np.inf
    elif kind == "tie_order":
        ids[q, [0, 1]] = ids[q, [1, 0]]   # 200 and 1500 sit at the same distance
    return ids, d, cnt


@pytest.mark.parametrize("kind", ["dropped", "swapped", "distance", "deleted", "count", "tie_order"])
def test_checker_rejects_each_corruption(table, kind):
    X, Q = table
    ids, d, cnt = _answer(X, Q, "l2", 10)
    bad = _corrupt(kind, ids, d, cnt, X, Q)
    ok = None
    if kind == "deleted":
        ok = np.ones(len(X), bool)
        ok[ids[5, 7]] = False
    with pytest.raises(AssertionError):
        er.check_exact(*bad, X, Q, "l2", 10, admissible=ok)


def test_rounding_models():
    a = np.array([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -12 + 2 ** -13)], np.float32)
    assert list(er.round_bf16(a)) == [1.0, 1.0 + 2 ** -6, -1.0]              # halfway cases go to the even neighbour
    assert list(er.round_tf32(a, "rz")) == [1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -1.0]
    assert er.round_tf32(np.float32(1.0 + 2 ** -11 + 2 ** -12), "rn") == np.float32(1.0 + 2 ** -10)


@pytest.mark.parametrize("mode", ["bf16", "tf32"])
def test_planted_row_escapes_the_sampled_guard(mode):
    """The hole the large-norm guard closes, shown in a host model of the coarse pass (operands rounded to bf16 / tf32,
    dots in float64): the planted row is the exact top-1, lies outside the coarse top-k' of its query, and the rule
    e_k + 2E <= T with E sampled from the re-scored rows calls the query safe; the row's norm is ~10^4 times the
    sample's, so scaling E by that ratio flags it."""
    X, Q, p = er.planted_ip_table()
    ids, d64, _ = er.ref_topk(X, Q[:1], "ip", 10)
    assert ids[0, 0] == p
    _, beta = er.direct(X, Q, "ip", 0, ids[0, :2])
    assert d64[0, 0] + beta[0] < d64[0, 1] - beta[1]       # top-1 beyond any fp32 summation error
    norms = np.linalg.norm(X.astype(np.float64), axis=1)
    for rnd in er.COARSE_MODELS[mode]:
        lists, safe = er.guard_model(X, Q, 10, 128, rnd)
        assert not np.isin(p, lists).any() and safe.all()
        assert norms.max() / norms[lists].max() > 1000
