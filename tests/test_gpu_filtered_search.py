"""Collect mode of a filtered graph search (eps_index_set_filter_search, DESIGN.md §K3) on seeded tables, with numeric
and string filters built as expr_model node arrays: no row, one row, 0.1 %, 1 %, 10 %, 50 % and 100 % of the rows,
uncorrelated with the vectors or selecting whole clusters of them, with and without deleted rows.

  * count and validity: min(cap, P) rows per query, each passing the numpy model and not deleted, no duplicates,
    ascending by (distance, id);
  * prefix: with every row indexed, post mode's rows of a query are the first rows of collect mode's, ids and distance
    bits, at widths 1, 4 and 8, screen off / on / auto and two launch tunings; a query where they differ must be one
    the scan of the passing rows answered (at most n_redone of them, each equal to the exact answer);
  * counters: n_dist, n_seed, n_expand and n_edges equal post mode's when no query was scanned (screen off);
  * fallback: whole batches under the threshold, and 16-query batches (whose graph distances are the row kernel's
    bits) with at most cap passing rows, equal prefilter mode under set_coarse("fp32"): ids, distance bits, counts;
  * tail: after appends, every passing tail row closer than a query's last row is returned;
  * two runs agree, a view agrees with its base, and every refusal leaves the index usable."""
import numpy as np
import pytest

import expr_model as em

pytestmark = pytest.mark.gpu

BAD_ARG, UNSUPPORTED = 40005, 40006
N, D, RANK, CLUSTERS = 20000, 128, 12, 40
STRIDE = 8  # int32 u (a permutation of the rows: "u < m" passes exactly m rows), int32 cluster id
WORDS = ["w%d" % i for i in range(7)]  # string column 0: code = cluster % 7


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200 as vdb
    assert vdb.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    return vdb


def make_table(n, seed):
    """Clustered low-rank rows (the screen's basis carries most of the variance) and their attributes."""
    rng = np.random.default_rng(seed)
    basis = np.linalg.qr(rng.standard_normal((D, RANK)))[0].T
    centres = rng.standard_normal((CLUSTERS, RANK)) * 3.0
    lab = rng.integers(0, CLUSTERS, n)
    X = ((centres[lab] + rng.standard_normal((n, RANK))) @ basis + 1e-3 * rng.standard_normal((n, D)) + 0.5).astype(np.float32)
    raw = np.zeros((n, STRIDE), np.uint8)
    raw[:, 0:4] = rng.permutation(n).astype(np.int32).view(np.uint8).reshape(n, 4)
    raw[:, 4:8] = lab.astype(np.int32).view(np.uint8).reshape(n, 4)
    codes = (lab % 7).astype(np.int32)
    return X, raw, codes


def queries(nq, seed):
    X, _, _ = make_table(nq, seed)
    return X


def int_cmp(op, offset, value):
    return np.array([[em.INT4, em.VT_INT, -1, -1, 0, 0, 0, offset], [em.INT_CONST, em.VT_INT, -1, -1, value, 0, 0, -1],
                     [op, em.VT_BOOL, 0, 1, 0, 0, 0, -1]], np.int64)


def str_eq(code):
    return np.array([[em.STRING_ATTR, em.VT_STRING, -1, -1, 0, 0, 0, 0], [em.STRING_CONST, em.VT_STRING, -1, -1, code, 0, 0, -1],
                     [em.EQ, em.VT_BOOL, 0, 1, 0, 0, 0, -1]], np.int64)


def distance_lt(c):
    return np.array([[em.DOUBLE_ATTR, em.VT_DOUBLE, -1, -1, 0, 0, 0, -2],
                     [em.DOUBLE_CONST, em.VT_DOUBLE, -1, -1, 0, np.float64(c).view(np.int64), 0, -1],
                     [em.LT, em.VT_BOOL, 0, 1, 0, 0, 0, -1]], np.int64)


def filters(n):
    """name -> nodes: the uncorrelated selectivities on u, and filters that follow the clusters."""
    f = {"none": int_cmp(em.LT, 0, 0), "one": int_cmp(em.EQ, 0, 7)}
    for name, share in (("0.1%", 0.001), ("1%", 0.01), ("10%", 0.1), ("50%", 0.5)):
        f[name] = int_cmp(em.LT, 0, int(n * share))
    f["100%"] = int_cmp(em.GTE, 0, 0)
    f["cluster"] = int_cmp(em.EQ, 4, 3)
    f["clusters<4"] = int_cmp(em.LT, 4, 4)
    f["string"] = str_eq(2)
    return f


class Tab:
    def __init__(self, vdb, n, n_indexed, seed, deleted=None):
        self.X, raw, codes = make_table(n, seed)
        self.model = em.Table(raw.ravel(), STRIDE, n, codes[None, :], WORDS)
        self.deleted = np.zeros(n, bool) if deleted is None else deleted
        self.ix = vdb.Index("l2", D, host_vectors=self.X)
        self.ix.sync_rows(n_indexed)
        self.ix.build(n_indexed)
        self.ix.sync_rows(n)
        self.ix.append_string_dictionary(0, WORDS)
        self.ix.set_attrs(raw.ravel(), STRIDE, n)
        self.ix.set_string_codes(0, 0, codes)
        if deleted is not None:
            self.ix.set_deleted(np.packbits(deleted, bitorder="little"))

    def passing(self, nodes):
        return em.logical_eval(nodes, self.model, 0.0) & ~self.deleted

    def close(self):
        self.ix.close()


@pytest.fixture(scope="module")
def full(vdb):
    t = Tab(vdb, N, N, seed=1)
    yield t
    t.close()


@pytest.fixture(scope="module")
def with_deleted(vdb):
    rng = np.random.default_rng(5)
    t = Tab(vdb, N, N, seed=1, deleted=rng.random(N) < 0.2)
    yield t
    t.close()


@pytest.fixture(scope="module")
def with_tail(vdb):
    t = Tab(vdb, N, 16000, seed=3)
    yield t
    t.close()


@pytest.fixture
def graph_path(monkeypatch):
    """Every batch with a passing row takes the graph search (the threshold of step 2 set to 0)."""
    monkeypatch.setenv("EPS_COLLECT_SCAN_ROWS", "0")


def search(ix, Q, limit, nodes, mode, L=128, W=1, screen=0, tuning=(0, 0), prefilter=False, coarse="tf32"):
    ix.config(L, L, prefilter=prefilter)
    ix.set_search_width(W)
    ix.set_graph_screen(screen)
    ix.set_graph_tuning(*tuning)
    ix.set_coarse(coarse)
    ix.set_filter_search(mode)
    return ix.search(Q, limit, filter_nodes=nodes)


def exact(ix, Q, limit, nodes, L=128):
    """Prefilter mode with the coarse pass off."""
    return search(ix, Q, limit, nodes, "post", L=L, prefilter=True, coarse="fp32")


def bits(d):
    return np.asarray(d, np.float32).view(np.uint32)


def check_valid(t, X, Q, res, nodes, cap):
    ids, ds, cnt, _ = res
    ok = t.passing(nodes)
    P = int(ok.sum())
    assert (cnt == min(cap, P)).all(), "counts %s, expected min(%d, %d)" % (np.unique(cnt), cap, P)
    for q in range(len(Q)):
        c = int(cnt[q])
        row = ids[q, :c]
        assert (ids[q, c:] == -1).all() and np.isinf(ds[q, c:]).all()
        assert ok[row].all(), "query %d returned a row that fails the filter or is deleted" % q
        assert len(set(row.tolist())) == c, "query %d returned a row twice" % q
        d = ds[q, :c].astype(np.float32)
        assert all((d[i], row[i]) < (d[i + 1], row[i + 1]) for i in range(c - 1)), "query %d is not ascending" % q
        ref = ((X[row].astype(np.float64) - Q[q].astype(np.float64)) ** 2).sum(1)
        assert np.allclose(d, ref, rtol=1e-4, atol=1e-4)


def same(a, b, qs=slice(None)):
    return (np.array_equal(a[0][qs], b[0][qs]) and np.array_equal(bits(a[1][qs]), bits(b[1][qs]))
            and np.array_equal(a[2][qs], b[2][qs]))


@pytest.mark.parametrize("name", list(filters(N)))
def test_counts_and_validity(full, with_deleted, graph_path, name):
    Q = queries(64, 11)
    for t in (full, with_deleted):
        nodes = filters(N)[name]
        res = search(t.ix, Q, 10, nodes, "collect", W=4)
        check_valid(t, t.X, Q, res, nodes, 10)
        assert same(res, search(t.ix, Q, 10, nodes, "collect", W=4)), "two runs differ"


CONFIGS = [  # (W, screen, tuning)
    (1, 0, (0, 0)), (4, 0, (4, 7)), (8, 0, (0, 0)),
    (1, 1, (0, 0)), (4, 1, (4, 7)), (8, 2, (12, 4)),
]


@pytest.mark.parametrize("W,screen,tuning", CONFIGS)
@pytest.mark.parametrize("name", ["1%", "10%", "50%", "100%", "cluster", "clusters<4", "string"])
def test_post_is_a_prefix_of_collect(full, graph_path, W, screen, tuning, name):
    t, Q, limit = full, queries(64, 12), 20
    nodes = filters(N)[name]
    post = search(t.ix, Q, limit, nodes, "post", W=W, screen=screen, tuning=tuning)
    col = search(t.ix, Q, limit, nodes, "collect", W=W, screen=screen, tuning=tuning)
    check_valid(t, t.X, Q, col, nodes, limit)
    ex = exact(t.ix, Q, limit, nodes)
    off = []
    for q in range(len(Q)):
        c = int(post[2][q])
        if not (np.array_equal(post[0][q, :c], col[0][q, :c]) and np.array_equal(bits(post[1][q, :c]), bits(col[1][q, :c]))):
            off.append(q)
    assert len(off) <= col[3]["n_redone"], "%d queries break the prefix, %d were scanned" % (len(off), col[3]["n_redone"])
    for q in off:
        assert same(col, ex, q), "query %d breaks the prefix but is not the exact answer" % q
    if col[3]["n_redone"] == 0 and screen == 0:
        for c in ("n_dist", "n_seed", "n_expand", "n_edges"):
            assert post[3][c] == col[3][c], "%s: post %d, collect %d" % (c, post[3][c], col[3][c])


def test_some_batches_need_no_scan(full, graph_path):
    """The counter check above is not vacuous: unselective filters are answered by the graph alone."""
    Q = queries(64, 12)
    for name in ("50%", "100%"):
        assert search(full.ix, Q, 20, filters(N)[name], "collect")[3]["n_redone"] == 0


@pytest.mark.parametrize("name", list(filters(N)))
def test_whole_batch_under_threshold_is_prefilter(full, with_deleted, name):
    Q = queries(64, 13)
    for t in (full, with_deleted):
        nodes = filters(N)[name]
        col = search(t.ix, Q, 10, nodes, "collect", W=4)
        assert col[3]["n_redone"] == len(Q)  # 20 000 rows: every filter is under the threshold
        assert same(col, exact(t.ix, Q, 10, nodes)), name


@pytest.mark.parametrize("name", ["one", "0.1%"])
def test_short_queries_are_prefilter(full, with_deleted, graph_path, name):
    """16 queries: the graph kernel's distances are the row kernel's bits, so with P <= cap every query, scanned or
    not, is the exact answer."""
    Q = queries(16, 14)
    for t in (full, with_deleted):
        nodes = filters(N)[name]
        P = int(t.passing(nodes).sum())
        limit = 32
        assert P <= limit
        col = search(t.ix, Q, limit, nodes, "collect", L=256, W=2)
        assert same(col, exact(t.ix, Q, limit, nodes, L=256)), name
        if P > 0:
            assert col[3]["n_redone"] > 0


@pytest.mark.parametrize("name", ["1%", "10%", "cluster", "string", "100%"])
def test_tail_rows_are_merged(with_tail, graph_path, name):
    t, Q = with_tail, queries(32, 15)
    nodes = filters(N)[name]
    ids, ds, cnt, _ = col = search(t.ix, Q, 10, nodes, "collect", W=4)
    check_valid(t, t.X, Q, col, nodes, 10)
    ok = t.passing(nodes)
    tail = np.flatnonzero(ok[16000:]) + 16000
    for q in range(len(Q)):
        c = int(cnt[q])
        if c == 0:
            continue
        d = ((t.X[tail] - Q[q]) ** 2).sum(1)
        closer = set(tail[d < ds[q, c - 1] * (1 - 1e-5)].tolist())
        assert closer <= set(ids[q, :c].tolist()), "query %d misses passing tail rows" % q


def test_view_copies_the_mode(full, graph_path):
    t, Q, nodes = full, queries(32, 16), filters(N)["10%"]
    post = search(t.ix, Q, 10, nodes, "post", W=4)
    base = search(t.ix, Q, 10, nodes, "collect", W=4)
    v = t.ix.view()  # the base is not modified while the view lives
    try:
        assert same(v.search(Q, 10, filter_nodes=nodes), base)
        v.set_filter_search("post")
        assert same(v.search(Q, 10, filter_nodes=nodes), post)
        assert same(t.ix.search(Q, 10, filter_nodes=nodes), base)
    finally:
        v.close()


def test_refusals_leave_the_index_usable(vdb, full):
    from vectordb_b200.lib import EpsError
    t, Q = full, queries(8, 17)
    nodes = filters(N)["10%"]
    before = search(t.ix, Q, 10, nodes, "collect")
    L = t.ix.L
    for mode in (2, -1, 7):
        assert L.eps_index_set_filter_search(t.ix.h, mode) == BAD_ARG
    assert L.eps_index_set_filter_search(None, 1) == BAD_ARG
    with pytest.raises(EpsError) as e:
        t.ix.search(Q, 10, filter_nodes=distance_lt(1e9))
    assert e.value.code == UNSUPPORTED
    assert same(t.ix.search(Q, 10, filter_nodes=nodes), before)
    # outside the graph branch the mode changes nothing: prefilter with a distance filter runs
    t.ix.config(128, 128, prefilter=True)
    t.ix.search(Q, 10, filter_nodes=distance_lt(1e9))
    sp = vdb.SparseIndex("ip", 100)
    try:
        assert L.eps_index_set_filter_search(sp.h, 1) == BAD_ARG
    finally:
        sp.close()
