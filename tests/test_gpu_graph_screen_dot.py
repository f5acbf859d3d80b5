"""The graph-search screen on inner-product and cosine indexes (DESIGN.md §K2, the dot-product bound) never changes a
result: with the screen on and off, the dense kernel returns bitwise-equal ids, distances and counts, and the same
n_dist, n_expand, n_edges and n_seed, across the widths, ring sizes, CTAs per SM and queue lengths of
test_gpu_graph_screen.py, the bitmap path, a view, a graph installed with eps_index_set_graph, integer tables, rows whose
norms spread over orders of magnitude (some large enough to overflow the fp32 products), an extended graph and a
collect-mode filtered search.  Every case also requires the screen to drop ids, so that the equality says something;
an isotropic table stays unscreened under auto."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_graph_screen import CASES, assert_same, int_low_rank, low_rank, run  # noqa: E402

pytestmark = pytest.mark.gpu

OFF, ON, AUTO = 0, 1, 2
METRICS = ("ip", "cosine")


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200 as vdb
    assert vdb.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    return vdb


def rows_for(metric, X):
    if metric == "cosine":  # the rows a cosine index holds are normalised, as the drop-in does
        X = X / np.linalg.norm(X.astype(np.float64), axis=1, keepdims=True)
    return np.ascontiguousarray(X, np.float32)


def make(vdb, metric, X, n_build=None):
    ix = vdb.Index(metric, X.shape[1], host_vectors=X)
    ix.sync_rows(X.shape[0])
    ix.build(X.shape[0] if n_build is None else n_build)
    return ix


@pytest.fixture(scope="module", params=METRICS)
def lowrank(vdb, request):
    metric = request.param
    X = rows_for(metric, low_rank(20000, 256, 12, seed=1))
    Q = rows_for(metric, low_rank(48, 256, 12, seed=2))
    ix = make(vdb, metric, X)
    yield metric, X, ix, Q
    ix.close()


@pytest.mark.parametrize("W,tuning,L", CASES)
def test_low_rank_screen_is_invisible(lowrank, W, tuning, L):
    metric, X, ix, Q = lowrank
    on = run(ix, Q, L, W, tuning, ON)
    off = run(ix, Q, L, W, tuning, OFF)
    assert off[4] == 0
    assert_same(on, off, "%s W=%d tuning=%s L=%d" % (metric, W, tuning, L))
    assert on[4] > 0, "%s: the screen dropped nothing: the equality above says nothing" % metric
    ix.set_graph_screen(AUTO)
    ix.set_graph_tuning(0, 0)


@pytest.mark.parametrize("nq", [1, 2, 3, 5, 7])
def test_batch_sizes(lowrank, nq):
    """Batches of any size: the per-query terms start at a 16-byte boundary whatever nq is (sk_qterms_off)."""
    metric, X, ix, Q = lowrank
    for W, tuning, L in ((1, (0, 0), 128), (6, (0, 0), 768)):
        on = run(ix, Q[:nq], L, W, tuning, ON)
        off = run(ix, Q[:nq], L, W, tuning, OFF)
        assert_same(on, off, "%s nq=%d W=%d L=%d" % (metric, nq, W, L))
        assert on[4] > 0
    ix.set_graph_screen(AUTO)


@pytest.mark.parametrize("L", [12000, 13000])
def test_bitmap_path(lowrank, L):
    metric, X, ix, Q = lowrank
    on = run(ix, Q[:4], L, 4, (0, 0), ON)
    off = run(ix, Q[:4], L, 4, (0, 0), OFF)
    assert_same(on, off, "%s bitmap L=%d" % (metric, L))
    assert on[4] > 0
    ix.set_graph_screen(AUTO)


def test_views_and_installed_graph(vdb, lowrank):
    metric, X, ix, Q = lowrank
    n, off_t, nb, nav = ix.get_graph()
    ref = run(ix, Q, 256, 6, (0, 0), OFF)
    ix.set_graph_screen(ON)
    v = ix.view()
    try:
        assert v.graph_screen_info()["active"]
        v.config(256, 256)
        v.set_search_width(6)
        assert_same(v.search(Q, 10), ref, "%s view" % metric)
        assert v.graph_screen_info()["n_screened"] > 0
    finally:
        v.close()
    ix.set_graph_screen(AUTO)
    ix2 = vdb.Index(metric, X.shape[1], host_vectors=X)
    try:
        ix2.sync_rows(X.shape[0])
        ix2.set_graph(n, off_t, nb, nav)
        info = ix2.graph_screen_info()
        assert abs(info["share"] - ix.graph_screen_info()["share"]) < 1e-9 and info["share"] >= 0.9, info
        got = run(ix2, Q, 256, 6, (0, 0), ON)
        assert_same(got, ref, "%s set_graph" % metric)
        assert got[4] > 0
    finally:
        ix2.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [128, 130, 768])
def test_integer_tables(vdb, metric, d):
    """Integer rows (exact dot products in any order) with the screen forced on; d = 130 takes the scalar row path."""
    rng = np.random.default_rng(d)
    X = int_low_rank(3000, d, rng)
    Q = int_low_rank(16, d, rng)
    ix = make(vdb, metric, X)
    try:
        for W, tuning, L in ((1, (0, 0), 64), (8, (0, 7), 300), (4, (12, 4), 1500)):
            on = run(ix, Q, L, W, tuning, ON)
            off = run(ix, Q, L, W, tuning, OFF)
            assert_same(on, off, "int %s d=%d W=%d L=%d" % (metric, d, W, L))
            assert on[4] > 0, "int %s d=%d W=%d L=%d: the screen dropped nothing" % (metric, d, W, L)
    finally:
        ix.close()


def test_ip_norm_spread_and_overflow(vdb):
    """IP rows of a low-rank table scaled by 10^-3 .. 10^3, then a few rows appended by extend_graph (so that the kept
    basis and mean are those of the others) at ~10^37, whose products with the queries overflow fp32: they score -inf
    or NaN, and the screen must keep them."""
    n0, n = 20000, 20008
    rng = np.random.default_rng(17)
    X = low_rank(n, 256, 12, seed=3).astype(np.float64) * 10.0 ** rng.uniform(-3, 3, size=(n, 1))
    X[n0:] *= 3e37 / np.abs(X[n0:]).max(axis=1, keepdims=True)
    X = X.astype(np.float32)
    Q = low_rank(32, 256, 12, seed=4)
    with np.errstate(over="ignore", invalid="ignore"):
        assert not np.all(np.isfinite(X[n0:] @ Q.T))  # some products overflow
    ix = make(vdb, "ip", X, n_build=n0)
    try:
        ix.extend_graph(n)
        for W, tuning, L in ((1, (0, 0), 128), (4, (12, 4), 512), (8, (0, 7), 1024)):
            on = run(ix, Q, L, W, tuning, ON)
            off = run(ix, Q, L, W, tuning, OFF)
            assert_same(on, off, "norm spread W=%d L=%d" % (W, L))
            assert on[4] > 0
    finally:
        ix.close()


def test_extend_graph_ip(vdb):
    n0, n, d, nq = 12000, 20000, 256, 48
    X = low_rank(n, d, 12, seed=8)
    rng = np.random.default_rng(8)
    Q = X[n0 + rng.integers(0, n - n0, nq)] + 0.05 * rng.standard_normal((nq, d)).astype(np.float32)
    ix = make(vdb, "ip", X, n_build=n0)
    try:
        ix.config(200, 200)
        ix.search(Q, 10)
        info0 = ix.graph_screen_info()
        assert info0["active"] and info0["n_screened"] > 0, info0
        ix.extend_graph(n)
        info1 = ix.graph_screen_info()
        assert info1["active"] and info1["share"] == info0["share"]
        assert info1["n_screened"] == info0["n_screened"], "the extension's own searches were screened"
        on = run(ix, Q, 200, 4, (0, 0), ON)
        off = run(ix, Q, 200, 4, (0, 0), OFF)
        assert_same(on, off, "extended")
        assert on[4] > 0 and (on[0] >= n0).mean() > 0.2  # the searches reach, and screen, the new rows
    finally:
        ix.close()


def test_collect_mode_ip(vdb, monkeypatch):
    import test_gpu_filtered_search as fs
    monkeypatch.setenv("EPS_COLLECT_SCAN_ROWS", "0")  # every batch takes the graph search
    X, raw, _ = fs.make_table(fs.N, seed=1)
    Q = fs.queries(32, 16)
    ix = make(vdb, "ip", X)
    try:
        ix.set_attrs(raw.ravel(), fs.STRIDE, fs.N)
        nodes = fs.int_cmp(fs.em.LT, 0, fs.N // 10)
        ix.set_filter_search("collect")
        res = {}
        for mode in (ON, OFF):
            ix.set_graph_screen(mode)
            ix.config(128, 128)
            ix.set_search_width(4)
            before = ix.graph_screen_info()["n_screened"]
            res[mode] = ix.search(Q, 10, filter_nodes=nodes)
            res[mode] = res[mode] + (ix.graph_screen_info()["n_screened"] - before,)
        for x, y in zip(res[ON][:3], res[OFF][:3]):
            assert np.array_equal(x, y) and (x.dtype.kind != "f" or np.array_equal(x.view(np.uint32), y.view(np.uint32)))
        assert res[ON][4] > 0
    finally:
        ix.close()


def test_auto_off_on_isotropic_ip_table(vdb):
    rng = np.random.default_rng(5)
    X = rng.random((8000, 256), dtype=np.float32)
    Q = rng.random((16, 256), dtype=np.float32)
    ix = make(vdb, "ip", X)
    try:
        info = ix.graph_screen_info()
        assert not info["active"] and 0.0 <= info["share"] < 0.9, info
        ix.config(256, 256)
        ix.set_search_width(4)
        ix.search(Q, 10)
        assert ix.graph_screen_info()["n_screened"] == 0
    finally:
        ix.close()
