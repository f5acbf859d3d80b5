"""The dense graph kernel held to the exact width-W model (graph_model.py) on integer tables, where every distance is
exact in any summation order: ids, counts and distances must be bitwise equal, and n_dist, n_expand, n_edges and
n_seed must equal the model's sums.  The cases form a matrix over metric, dimension (staged and non-staged rows),
search width, ring size and resident CTAs per SM (both kernel instances), batch size (row-kernel and tile-kernel
seeds, several waves), queue length (unchecked-bitmap word edges, merge super-tiles, hash set and bitmap starts),
graph shape (the device's build, random CSRs with rows up to 300 ids, repeated ids and self-loops, ids that share one
hash bucket at the end of the table), the visited-set clean-up paths, and the Search wrapper around the kernel.

On one H100 80GB HBM3 (700 W power limit) the file runs in about 45 s.  Its largest table is 3000 x 4096 (49 MB);
the 2^20 x 4 table (16 MB) has the most rows."""
import numpy as np
import pytest

import graph_model as gm

pytestmark = pytest.mark.gpu

NT_INT_CONST, NT_DOUBLE_CONST, NT_INT4_ATTR, NT_DOUBLE_ATTR, NT_LT = 1, 3, 7, 10, 19
VLOG_CAP = 32768  # fresh ids a query logs (graph_search.cu prepare_visited)


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200 as vdb
    assert vdb.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    return vdb


def attr_lt(c):
    return np.array([[NT_INT4_ATTR, 1, -1, -1, 0, 0, 0, 0], [NT_INT_CONST, 1, -1, -1, c, 0, 0, -1],
                     [NT_LT, 3, 0, 1, 0, 0, 0, -1]], np.int64)


def distance_lt(c):
    return np.array([[NT_DOUBLE_ATTR, 2, -1, -1, 0, 0, 0, -2],
                     [NT_DOUBLE_CONST, 2, -1, -1, 0, np.float64(c).view(np.int64), 0, -1],
                     [NT_LT, 3, 0, 1, 0, 0, 0, -1]], np.int64)


class Table:
    """An integer table, its graph over the first n_indexed rows, and one device index per metric."""

    def __init__(self, vdb, X, graph, metrics=gm.METRICS):
        self.X, self.graph = X, graph
        n_indexed, off, nb, nav = graph
        self.ix = {}
        for m in metrics:
            ix = vdb.Index(m, X.shape[1], host_vectors=X)
            ix.sync_rows(X.shape[0])
            ix.set_graph(n_indexed, off, nb, nav)
            self.ix[m] = ix

    def close(self):
        for ix in self.ix.values():
            ix.close()


def check(t, metric, Q, L, limit, W=1, tuning=(0, 0), L_local=None, deleted=None, keep=None, nodes=None, what=""):
    """One device search against the model; returns (device ids, dists, counts, stats, model)."""
    gm.assert_exact(t.X, Q)
    ix = t.ix[metric]
    ix.config(L, L if L_local is None else L_local)
    ix.set_search_width(W)
    ix.set_graph_tuning(*tuning)
    ids, ds, cnt, st = ix.search(Q, limit, filter_nodes=nodes)
    m = gm.search(t.X, Q, metric, t.graph, L, limit, W=W, L_local=L_local, deleted=deleted, keep=keep)
    what = "%s %s d=%d W=%d ring/ctas=%s L=%d limit=%d nq=%d" % (what, metric, t.X.shape[1], W, tuning, L, limit, Q.shape[0])
    assert_match(ids, ds, cnt, st, m, what)
    return ids, ds, cnt, st, m


def assert_match(ids, ds, cnt, st, m, what):
    bad = np.flatnonzero((cnt != m.counts) | np.any(ids != m.ids, axis=1))
    assert bad.size == 0, "%s: %d queries differ, first q%d: ids %s vs model %s" % (
        what, bad.size, bad[0], ids[bad[0], :8], m.ids[bad[0], :8])
    v = ids >= 0
    assert np.all(np.isinf(ds[~v]))
    g = (ds[v].astype(np.float32) + np.float32(0)).view(np.uint32)
    w = (m.dists[v].astype(np.float32) + np.float32(0)).view(np.uint32)
    assert np.array_equal(g, w), "%s: distances are not bitwise equal" % what
    assert np.array_equal(ds[v], m.dists[v]), "%s: distances" % what
    for f in ("n_dist", "n_expand", "n_edges", "n_seed"):
        assert st[f] == int(getattr(m, f).sum()), "%s: %s %d != model %d" % (what, f, st[f], getattr(m, f).sum())


# ---- the device's own graph ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def built(vdb):
    n, d = 20000, 64
    X = gm.int_table(n, d, 1)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.build(n)
    graph = ix.get_graph()
    ix.close()
    t = Table(vdb, X, graph)
    yield t
    t.close()


# (metric, W, (ring slots, CTAs per SM), L, nq): every axis value at least once
BUILT_CASES = [
    ("l2", 1, (0, 0), 1, 16),
    ("l2", 1, (2, 0), 31, 17),
    ("l2", 2, (3, 1), 32, 1),
    ("l2", 3, (4, 4), 33, 17),
    ("l2", 4, (6, 5), 64, 1500),
    ("l2", 8, (7, 7), 1000, 16),
    ("l2", 8, (12, 4), 1025, 17),
    ("l2", 4, (13, 1), 4096, 3),
    ("l2", 2, (24, 0), 12288, 2),
    ("l2", 8, (0, 0), 12289, 2),
    ("l2", 1, (0, 0), 16384, 1),
    ("l2", 1, (0, 4), 64, 1000),
    ("ip", 1, (0, 0), 32, 17),
    ("ip", 3, (13, 5), 1025, 16),
    ("ip", 8, (24, 1), 64, 1500),
    ("ip", 2, (0, 0), 16384, 1),
    ("cosine", 1, (12, 7), 33, 16),
    ("cosine", 4, (2, 4), 1000, 17),
    ("cosine", 8, (3, 0), 12289, 1),
]


@pytest.mark.parametrize("metric,W,tuning,L,nq", BUILT_CASES,
                         ids=["%s-W%d-r%dc%d-L%d-nq%d" % (c[0], c[1], c[2][0], c[2][1], c[3], c[4]) for c in BUILT_CASES])
def test_built_graph(built, metric, W, tuning, L, nq):
    Q = gm.int_table(nq, built.X.shape[1], 1000 + L + W)
    check(built, metric, Q, L, min(L, 10), W=W, tuning=tuning, what="built")


def test_wide_results_do_not_depend_on_the_geometry(built):
    Q = gm.int_table(300, 64, 77)
    first = None
    for tuning in ((0, 0), (2, 1), (3, 4), (4, 5), (6, 7), (7, 0), (12, 4), (13, 1), (24, 7)):
        ix = built.ix["l2"]
        ix.config(256, 256)
        ix.set_search_width(4)
        ix.set_graph_tuning(*tuning)
        got = ix.search(Q, 20)
        if first is None:
            first = got
            continue
        for a, b, name in zip(got[:3], first[:3], ("ids", "dists", "counts")):
            assert np.array_equal(a, b), "W=4: %s with ring/ctas %s differ from auto geometry" % (name, tuning)
        for f in ("n_dist", "n_expand", "n_edges"):
            assert got[3][f] == first[3][f], "W=4: %s with ring/ctas %s" % (f, tuning)


# ---- synthetic graphs: long rows, repeated ids, self-loops, empty and long navigation rows, every dimension -------
def synthetic(n, seed):
    off, nb = gm.random_csr(n, 0, 300, seed, self_loops=0.05, dup=0.05)
    return off, nb


SYNTH_CASES = [  # (d, metric, W, tuning, L, nq, nav row)
    (1, "l2", 1, (0, 0), 32, 17, "long"),
    (1, "ip", 8, (0, 1), 64, 16, None),
    (3, "cosine", 2, (0, 5), 33, 17, "empty"),
    (3, "l2", 4, (0, 0), 1025, 3, None),
    (17, "ip", 3, (0, 4), 31, 16, "long"),
    (17, "l2", 8, (0, 7), 100, 17, None),
    (4, "l2", 8, (24, 0), 64, 16, "long"),
    (4, "cosine", 3, (13, 4), 32, 17, None),
    (768, "l2", 2, (7, 1), 64, 16, None),
    (768, "ip", 8, (12, 0), 33, 17, "long"),
    (4096, "l2", 4, (0, 0), 32, 16, None),
    (4096, "cosine", 1, (24, 4), 64, 3, "empty"),
]


@pytest.mark.parametrize("d,metric,W,tuning,L,nq,nav", SYNTH_CASES,
                         ids=["d%d-%s-W%d-r%dc%d-L%d-nq%d-%s" % (c[0], c[1], c[2], c[3][0], c[3][1], c[4], c[5], c[6]) for c in SYNTH_CASES])
def test_synthetic_graph(vdb, d, metric, W, tuning, L, nq, nav):
    n = 3000
    off, nb = synthetic(n, d)
    if nav == "empty":
        off, nb = gm.with_rows(off, nb, {5: []})
    elif nav == "long":
        off, nb = gm.with_rows(off, nb, {5: np.random.default_rng(d).integers(0, n, 2 * L + 7)})
    t = Table(vdb, gm.int_table(n, d, 2 + d), (n, off, nb, 5), metrics=(metric,))
    try:
        check(t, metric, gm.int_table(nq, d, 3 + d), L, 10, W=W, tuning=tuning, what="synthetic")
    finally:
        t.close()


def test_long_rows_picked_together_and_one_hash_bucket(vdb):
    """Rows of 65, 128, 129 and 300 ids (drained from the CSR in 128-id chunks, several picked in one step at W = 8),
    and rows whose ids all fall in the last bucket of the L = 64 hash table, so that probing wraps to entry 0."""
    n, d, L = 20000, 8, 64
    rng = np.random.default_rng(5)
    lens = np.array([65, 128, 129, 300, 20])[rng.integers(0, 5, n)]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    nb = rng.integers(0, n, off[-1]).astype(np.int64)
    cap, _, _ = gm.vset_geometry(L)
    same = np.flatnonzero(gm.vset_bucket(np.arange(n), L) == cap - 8)
    rng.shuffle(same)
    assert same.size > 100
    nav = int(same[0])
    rows = {nav: same[1:41]}                   # 40 seeds in one bucket
    for v in same[1:41]:
        rows[int(v)] = rng.permutation(same[41:])  # and rows of the other ids of that bucket
    off, nb = gm.with_rows(off, nb, rows)
    t = Table(vdb, gm.int_table(n, d, 6), (n, off, nb, nav))
    try:
        for metric, W, tuning in (("l2", 1, (0, 0)), ("ip", 8, (4, 1)), ("cosine", 8, (24, 7)), ("l2", 3, (7, 4))):
            Q = gm.int_table(40, d, 7 + W)
            check(t, metric, Q, L, 10, W=W, tuning=tuning, what="long rows / one bucket")
    finally:
        t.close()


# ---- the visited structures: hash set, move to the bitmap, touched-words and full clear, stale state --------------
def visited_paths(m, L, n_indexed):
    """Per query: 0 = stayed in the hash set, 1 = bitmap cleared word by word, 2 = bitmap cleared whole, -1 = not
    decidable from the totals (the move depends on the size of the last step)."""
    _, _, vmax = gm.vset_geometry(L)
    words = ((n_indexed + 31) // 32 + 3) & ~3
    out = []
    for r in m.runs:
        if L + r.fresh + 8 * 64 <= vmax:
            out.append(0)
        elif L + r.fresh > vmax or L > vmax:
            out.append(1 if r.fresh <= VLOG_CAP and 10 * (r.fresh + L) < words else 2)
        else:
            out.append(-1)
    return np.array(out)


@pytest.fixture(scope="module")
def million(vdb):
    n, d = 1 << 20, 4
    off, nb = gm.random_csr(n, 16, 16, 9)
    t = Table(vdb, gm.int_table(n, d, 10), (n, off, nb, 0), metrics=("l2",))
    yield t
    t.close()


@pytest.mark.parametrize("W,tuning", [(1, (0, 1)), (4, (12, 1)), (8, (0, 4))])
def test_visited_clean_up_paths(million, W, tuning):
    """Queries that stay hashed, move to the bitmap and clear only its touched words, or clear it whole (also past
    the log's capacity), each batch followed on the same index by different queries.  One CTA per SM: each CTA serves
    many queries in a row, inheriting what the previous one cleaned."""
    seen = set()
    for L, nq in ((24, 200), (48, 200), (300, 8), (3000, 2)):
        for batch in range(2):
            Q = gm.int_table(nq, 4, 11 + 2 * L + batch + W)
            *_, m = check(million, "l2", Q, L, 10, W=W, tuning=tuning, what="visited batch %d" % batch)
            seen.update(visited_paths(m, L, million.graph[0]).tolist())
    assert {0, 1, 2} <= seen, seen


# ---- the Search wrapper around the kernel --------------------------------------------------------------------------
@pytest.mark.parametrize("W", [1, 4])
def test_search_wrapper(vdb, W):
    n, total, d = 3000, 3400, 17
    off, nb = synthetic(n, 21)
    nav = 13
    X = gm.int_table(total, d, 22)
    attr = (np.arange(total) % 97).astype(np.int32)
    deleted = np.random.default_rng(23).random(total) < 0.1
    init = gm.prepare_init_ids(off, nb, nav, n, 48)
    deleted[[nav, *init[:5]]] = True
    t = Table(vdb, X, (n, off, nb, nav))
    try:
        Q = gm.int_table(33, d, 24)
        for metric, ix in t.ix.items():
            ix.set_deleted(np.packbits(deleted, bitorder="little"))
            ix.set_attrs(attr.view(np.uint8), 4, total)
            cut = float(np.median(gm.distances(metric, X, np.arange(200), Q[0]))) + 0.5
            check(t, metric, Q, 48, 10, W=W, deleted=deleted, what="tail+deleted")
            check(t, metric, Q, 48, 20, W=W, deleted=deleted, keep=lambda i, ds: attr[i] < 40, nodes=attr_lt(40),
                  what="numeric filter")
            check(t, metric, Q, 48, 20, W=W, deleted=deleted, keep=lambda i, ds: ds < cut, nodes=distance_lt(cut),
                  what="@distance filter")
            check(t, metric, Q, 48, 30, W=W, L_local=12, deleted=deleted, what="L_local < limit")
            check(t, metric, Q, 48, 100, W=W, deleted=deleted, what="limit > L")
    finally:
        t.close()


@pytest.mark.parametrize("n_indexed", [511, 512])
def test_brute_threshold(vdb, n_indexed):
    total, d = 700, 5
    off, nb = gm.random_csr(n_indexed, 1, 30, 25)
    t = Table(vdb, gm.int_table(total, d, 26), (n_indexed, off, nb, 3))
    try:
        for metric in gm.METRICS:
            check(t, metric, gm.int_table(17, d, 27), 64, 10, W=4, what="n_indexed=%d" % n_indexed)
    finally:
        t.close()
