"""The graph-search screen (DESIGN.md §K2) never changes a result: with the screen on and off, the dense kernel returns
bitwise-equal ids, distances and counts, and the same n_dist, n_expand, n_edges and n_seed, across search widths, ring
sizes, both register instances (resident CTAs per SM), queue lengths, a query that moves to the bitmap, views, and a
graph installed with eps_index_set_graph.  The screen must also do something: it drops ids on a low-rank table, and
stays off under auto on an isotropic one, with the reason readable from the index."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

OFF, ON, AUTO = 0, 1, 2


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200 as vdb
    assert vdb.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    return vdb


def low_rank(n, d, rank, seed, noise=1e-3):
    rng = np.random.default_rng(seed)
    basis = np.linalg.qr(rng.standard_normal((d, rank)))[0].T
    z = rng.standard_normal((n, rank)) * (1.0 + rng.integers(0, 4, size=(n, 1)))
    return (z @ basis + noise * rng.standard_normal((n, d)) + 0.5).astype(np.float32)


@pytest.fixture(scope="module")
def lowrank(vdb):
    X = low_rank(20000, 256, 12, seed=1)
    ix = vdb.Index("l2", X.shape[1], host_vectors=X)
    ix.sync_rows(X.shape[0])
    ix.build(X.shape[0])
    Q = low_rank(48, 256, 12, seed=2)
    yield X, ix, Q
    ix.close()


def run(ix, Q, L, W, tuning, mode, k=10):
    ix.set_graph_screen(mode)
    ix.config(L, L)
    ix.set_search_width(W)
    ix.set_graph_tuning(*tuning)
    before = ix.graph_screen_info()["n_screened"]
    ids, ds, cnt, st = ix.search(Q, k)
    return ids, ds, cnt, st, ix.graph_screen_info()["n_screened"] - before


def assert_same(a, b, what):
    for x, y, name in zip(a[:3], b[:3], ("ids", "dists", "counts")):
        assert np.array_equal(x, y), "%s: %s differ with the screen" % (what, name)
        if x.dtype.kind == "f":
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), "%s: %s bits differ" % (what, name)
    for c in ("n_dist", "n_expand", "n_edges", "n_seed"):
        assert a[3][c] == b[3][c], "%s: %s %d != %d" % (what, c, a[3][c], b[3][c])


CASES = [  # (W, (ring slots, CTAs per SM), L)
    (1, (0, 0), 64),
    (2, (4, 7), 128),
    (3, (12, 4), 256),
    (4, (0, 4), 512),
    (5, (5, 7), 100),
    (6, (0, 0), 768),
    (7, (12, 1), 1024),
    (8, (4, 0), 2048),
]


@pytest.mark.parametrize("W,tuning,L", CASES)
def test_low_rank_screen_is_invisible(lowrank, W, tuning, L):
    X, ix, Q = lowrank
    info = ix.graph_screen_info()
    assert info["active"] and info["share"] >= 0.9, info
    on = run(ix, Q, L, W, tuning, ON)
    off = run(ix, Q, L, W, tuning, OFF)
    assert off[4] == 0
    assert_same(on, off, "W=%d tuning=%s L=%d" % (W, tuning, L))
    if L < 2048:
        assert on[4] > 0, "the screen dropped nothing: the equality above says nothing"
    ix.set_graph_screen(AUTO)
    ix.set_graph_tuning(0, 0)


@pytest.mark.parametrize("L", [12000, 13000])
def test_bitmap_path(lowrank, L):
    """At L = 12000 a query starts on its hash set (16384 entries, 12288 inserts) and moves to the bitmap mid-query,
    replaying the log of its fresh ids; at L > 12288 it starts on the bitmap."""
    X, ix, Q = lowrank
    on = run(ix, Q[:4], L, 4, (0, 0), ON)
    off = run(ix, Q[:4], L, 4, (0, 0), OFF)
    assert_same(on, off, "bitmap L=%d" % L)
    assert on[4] > 0
    ix.set_graph_screen(AUTO)


def test_bitmap_cleared_from_the_log(vdb):
    """A query that moves to the bitmap on a large table clears only the words of its seeds and logged fresh ids
    (10 (fresh + L) < bitmap words).  Random graph, low-rank rows; each query runs alone so that its own fresh count
    shows that both the migration and the log-based clear ran."""
    n, d, L, deg = 1 << 21, 128, 32, 24
    X = low_rank(n, d, 6, seed=6)
    rng = np.random.default_rng(6)
    off_t = np.arange(n + 1, dtype=np.int64) * deg
    nb = rng.integers(0, n, size=n * deg, dtype=np.int64)
    ix = vdb.Index("l2", d, host_vectors=X)
    try:
        ix.sync_rows(n)
        ix.set_graph(n, off_t, nb, 0)
        assert ix.graph_screen_info()["active"]
        Q = low_rank(8, d, 6, seed=7)
        vset_max, words, both = 768, (n + 31) // 32, 0  # hash set of 1024 entries at L = 32
        for i in range(Q.shape[0]):
            on = run(ix, Q[i:i + 1], L, 8, (0, 0), ON)
            off = run(ix, Q[i:i + 1], L, 8, (0, 0), OFF)
            assert_same(on, off, "log clear q%d" % i)
            fresh = on[3]["n_dist"] - L
            both += int(L + fresh > vset_max and 10 * (fresh + L) < words and on[4] > 0)
        assert both > 0, "no query took the migration and the log-based clear with the screen dropping ids"
        # the bitmaps were left clean: a repeat gives the same answer
        assert_same(run(ix, Q[:1], L, 8, (0, 0), ON), run(ix, Q[:1], L, 8, (0, 0), OFF), "repeat")
    finally:
        ix.close()


def test_views_and_installed_graph(vdb, lowrank):
    X, ix, Q = lowrank
    n, off_t, nb, nav = ix.get_graph()
    ref = run(ix, Q, 256, 6, (0, 0), OFF)
    ix.set_graph_screen(AUTO)
    v = ix.view()
    try:
        assert v.graph_screen_info()["active"]
        v.config(256, 256)
        v.set_search_width(6)
        got = v.search(Q, 10)
        assert_same(got, ref, "view")
        assert v.graph_screen_info()["n_screened"] > 0
    finally:
        v.close()
    ix2 = vdb.Index("l2", X.shape[1], host_vectors=X)
    try:
        ix2.sync_rows(X.shape[0])
        ix2.set_graph(n, off_t, nb, nav)
        info = ix2.graph_screen_info()
        assert info["active"] and abs(info["share"] - ix.graph_screen_info()["share"]) < 1e-9
        got = run(ix2, Q, 256, 6, (0, 0), AUTO)
        assert_same(got, ref, "set_graph")
        assert got[4] > 0
    finally:
        ix2.close()


def int_low_rank(n, d, rng):
    """Integer rows of a rank-4 integer space plus sparse +-1 noise: exact distances in any summation order."""
    Z = rng.integers(-3, 4, size=(n, 4))
    B = rng.integers(-2, 3, size=(4, d))
    return (Z @ B + (rng.random((n, d)) < 0.02) * rng.choice([-1, 1], size=(n, d))).astype(np.float32)


@pytest.mark.parametrize("d", [128, 130, 768])
def test_integer_tables(vdb, d):
    """Integer tables with the screen forced on; d = 130 takes the unstaged scalar row path (d % 4 != 0)."""
    rng = np.random.default_rng(d)
    X = int_low_rank(3000, d, rng)
    Q = int_low_rank(16, d, rng)
    ix = vdb.Index("l2", d, host_vectors=X)
    try:
        ix.sync_rows(X.shape[0])
        ix.build(X.shape[0])
        for W, tuning, L in ((1, (0, 0), 64), (8, (0, 7), 300), (4, (12, 4), 1500)):
            on = run(ix, Q, L, W, tuning, ON)
            off = run(ix, Q, L, W, tuning, OFF)
            assert_same(on, off, "int d=%d W=%d L=%d" % (d, W, L))
            assert on[4] > 0, "int d=%d W=%d L=%d: the screen dropped nothing" % (d, W, L)
    finally:
        ix.close()


def test_auto_off_on_isotropic_table(vdb):
    rng = np.random.default_rng(5)
    X = rng.random((8000, 256), dtype=np.float32)
    Q = rng.random((16, 256), dtype=np.float32)
    ix = vdb.Index("l2", 256, host_vectors=X)
    try:
        ix.sync_rows(X.shape[0])
        ix.build(X.shape[0])
        info = ix.graph_screen_info()
        assert not info["active"] and 0.0 <= info["share"] < 0.9, info
        ix.config(256, 256)
        ix.set_search_width(4)
        ix.search(Q, 10)
        assert ix.graph_screen_info()["n_screened"] == 0
    finally:
        ix.close()
