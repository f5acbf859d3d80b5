"""GPU tests of eps_index_extend_graph (DESIGN.md §K4, B4): rows appended after a build linked into the installed graph
on the device.  The checkers are the reference's own known answer, a full build on the same rows, the oracle's search
on the same CSR, and the structural promises of the header."""
import numpy as np
import pytest

from helpers import assert_same_results, exact_topk, gen, recall

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200
    L = vectordb_b200.load_library()
    assert L.eps_device_count() > 0, "GPU tests need a CUDA device"
    return vectordb_b200


def reachable(n, off, nb, nav):
    """BFS of test_build_repair_does_not_grow_hubs: which vertices the navigation point reaches."""
    seen = np.zeros(n, bool)
    seen[nav] = True
    frontier = np.array([nav])
    while len(frontier):
        nxt = np.unique(nb[np.concatenate([np.arange(off[v], off[v + 1]) for v in frontier])])
        nxt = nxt[~seen[nxt]]
        seen[nxt] = True
        frontier = nxt
    return seen


def same_graph(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def quality(ix, Q, truth, L, width):
    ix.config(L, L)
    ix.set_search_width(width)
    ids, _, _, st = ix.search(Q, 10)
    return recall(ids, truth, 10), st["n_dist"] / len(Q)


# ---- the reference's own known answer (db_server.cpp:1232-1244, after its rebuild) --------------------------------
def test_extend_halfcircle_golden(vdb, golden):
    g = golden["halfcircle"]
    perm = g["perm"]
    ix = vdb.Index("cosine", 2, host_vectors=g["vectors"])
    ix.sync_rows(5000)
    ix.set_graph(5000, g["offsets"], g["nbrs"].astype(np.int64), int(g["nav"]))
    ix.config(500, 500)
    ix.sync_rows(10000)
    _, _, _, st_tail = ix.search(g["query"], 500)
    ix.extend_graph(10000)
    ni, off, nb, nav = ix.get_graph()
    assert ni == 10000 and nav == int(g["nav"]) and off[-1] == len(nb)
    ids, ds, cnt, st = ix.search(g["query"], 500)
    assert cnt[0] == 500
    assert np.array_equal(perm[ids[0]], np.arange(500)), "db_server.cpp:1232-1244"
    # the 5000 appended rows are no longer scanned as the tail: fewer evaluations than before, and than one full scan
    assert st["n_dist"] < min(st_tail["n_dist"], 10000), (st["n_dist"], st_tail["n_dist"])
    ix.close()


# ---- quality against a full build --------------------------------------------------------------------------------
@pytest.mark.parametrize("m", ("l2", "ip", "cosine"))
def test_extend_quality_vs_full_build(vdb, m):
    n0, n, d, nq = 20000, 60000, 64, 200
    X, Q = gen(n, d, 941, "cluster"), gen(nq, d, 942, "cluster")
    if m == "cosine":
        X /= np.linalg.norm(X, axis=1, keepdims=True)
        Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    truth = exact_topk(X, Q, 10, m)
    full = vdb.Index(m, d, host_vectors=X)
    full.sync_rows(n)
    full.build(n)
    ext = vdb.Index(m, d, host_vectors=X)
    ext.sync_rows(n)
    ext.build(n0)
    ext.extend_graph(n)
    assert ext.get_graph()[0] == n
    for width in (1, 4):
        rf, df = quality(full, Q, truth, 200, width)
        re, de = quality(ext, Q, truth, 200, width)
        assert re >= rf - 0.03, (m, width, re, rf)
        assert de <= 1.3 * df, (m, width, de, df)
    full.close()
    ext.close()


def test_extend_distribution_shift(vdb):
    """The appended rows come from other cluster centres than the indexed ones, and the queries lie near them."""
    n0, n1, d, nq = 20000, 30000, 64, 200
    X = np.concatenate([gen(n0, d, 951, "cluster"), gen(n1, d, 952, "cluster")])
    n = len(X)
    rng = np.random.default_rng(953)
    Q = X[n0 + rng.integers(0, n1, nq)] + 0.05 * rng.standard_normal((nq, d)).astype(np.float32)
    truth = exact_topk(X, Q, 10)
    assert (truth >= n0).mean() > 0.9
    full = vdb.Index("l2", d, host_vectors=X)
    full.sync_rows(n)
    full.build(n)
    ext = vdb.Index("l2", d, host_vectors=X)
    ext.sync_rows(n)
    ext.build(n0)
    ext.extend_graph(n)
    for width in (1, 4):
        rf, df = quality(full, Q, truth, 200, width)
        re, de = quality(ext, Q, truth, 200, width)
        assert re >= rf - 0.03, (width, re, rf)
    full.close()
    ext.close()


# ---- structure, over several chunks ------------------------------------------------------------------------------
def test_extend_structure_over_chunks(vdb):
    """140 000 appended rows = three chunks: reachability, degree bounds, untouched rows kept, and search quality
    against a full build (a hard table: 2 300 rows per 32-d Gaussian cluster, recall@10 at L = 200 is ~0.63 either way)."""
    n0, n, d, nq, R = 10000, 150000, 32, 200, 50
    X, Q = gen(n, d, 961, "cluster"), gen(nq, d, 962, "cluster")
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.build(n0)
    _, off0, nb0, nav0 = ix.get_graph()
    deg0 = np.diff(off0)
    ix.extend_graph(n)
    ni, off, nb, nav = ix.get_graph()
    assert ni == n and nav == nav0 and off[-1] == len(nb) and nb.min() >= 0 and nb.max() < n
    assert reachable(n, off, nb, nav).all()
    deg = np.diff(off)
    before = np.concatenate([deg0, np.zeros(n - n0, np.int64)])
    bound = np.maximum(before, R) + 16
    others = np.arange(n) != nav
    assert np.all(deg[others] <= bound[others]), np.max(deg[others] - bound[others])
    pointed = np.zeros(n, bool)
    src = np.repeat(np.arange(n), deg)
    pointed[nb[src >= n0]] = True  # old vertices some new row points to
    kept = 0
    for v in range(n0):
        if v == nav:
            continue
        row, old = nb[off[v]:off[v + 1]], nb0[off0[v]:off0[v + 1]]
        if np.array_equal(row[:len(old)], old):
            kept += 1
            continue
        # re-selected over its old row and new rows; anything else is a repair edge at the end (at most 16)
        foreign = np.nonzero(~np.isin(row, old) & (row < n0))[0]
        assert len(foreign) <= 16 and (len(foreign) == 0 or foreign[0] >= len(row) - 16), (v, row, old)
    untouched = [v for v in np.nonzero(~pointed[:n0])[0] if v != nav]
    for v in untouched:
        assert np.array_equal(nb[off[v]:off[v] + deg0[v]], nb0[off0[v]:off0[v + 1]]), v
    assert kept > 0 and len(untouched) > 0
    truth = exact_topk(X, Q, 10)
    full = vdb.Index("l2", d, host_vectors=X)
    full.sync_rows(n)
    full.build(n)
    for width in (1, 4):
        rf, df = quality(full, Q, truth, 200, width)
        re, de = quality(ix, Q, truth, 200, width)
        assert re >= rf - 0.03 and de <= 1.3 * df, (width, re, rf, de, df)
    full.close()
    ix.close()


# ---- graph format ------------------------------------------------------------------------------------------------
def test_extend_graph_format(vdb, port, have_ref):
    n0, n, d, nq = 8000, 20000, 64, 48
    X, Q = gen(n, d, 971, "cluster"), gen(nq, d, 972, "cluster")
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.build(n0)
    ix.extend_graph(n)
    ni, off, nb, nav = ix.get_graph()
    ix.config(500, 500)
    ix.set_search_width(1)
    ids, ds, cnt, st = ix.search(Q, 10)
    # the CSR stands on its own: installed on a fresh index it gives bitwise the same results
    fresh = vdb.Index("l2", d, host_vectors=X)
    fresh.sync_rows(n)
    fresh.set_graph(ni, off, nb, nav)
    fresh.config(500, 500)
    fresh.set_search_width(1)
    fids, fds, fcnt, fst = fresh.search(Q, 10)
    assert np.array_equal(ids, fids) and np.array_equal(ds, fds) and np.array_equal(cnt, fcnt)
    assert (st["n_dist"], st["n_expand"], st["n_edges"]) == (fst["n_dist"], fst["n_expand"], fst["n_edges"])
    fresh.close()
    # the oracle's search on the same CSR (test_graph_search_vs_port_same_graph)
    pids, pds, pcnt, pst = port.search_batch(metric="l2", vectors=X, queries=Q, limit=10, n_indexed=ni, offsets=off,
                                             nbrs=nb, nav=nav, L=500)
    assert assert_same_results(ids, ds, cnt, pids, pds, pcnt, "extended graph vs port") > 0.9
    assert abs(st["n_dist"] - pst[0]) <= 0.01 * pst[0]
    if have_ref:
        from oracle.oracle import Ref
        r = Ref("l2", d, n, [("ID", "int4")])
        r.set_rows(X)
        r.set_graph(ni, off, nb, nav)
        r.make_executors(1, 1, 500)
        rids, rds, rcnt = r.search_batch(Q, 10)
        assert_same_results(ids, ds, cnt, rids, rds, rcnt, "reference executor on the extended graph")
    ix.close()


# ---- determinism and deleted rows --------------------------------------------------------------------------------
@pytest.mark.parametrize("below", (60000, 1000))
def test_extend_deterministic_and_ignores_deleted_rows(vdb, below):
    n0, n, d = 4000, 9000, 32
    X = gen(n, d, 981, "cluster")

    def run(bits=None):
        ix = vdb.Index("l2", d, host_vectors=X)
        ix.sync_rows(n)
        ix.build(n0, exact_knn_below=below)
        if bits is not None:
            ix.set_deleted(bits)
        ix.extend_graph(n, exact_knn_below=below)
        g = ix.get_graph()
        ix.close()
        return g

    want = run()
    assert same_graph(run(), want), "two runs differ"
    bits = np.zeros(n // 8 + 1, np.uint8)
    bits[::3] = 0xA5
    nav = want[3]
    bits[nav >> 3] |= 1 << (nav & 7)
    assert same_graph(run(bits), want), "deleted rows changed the graph"


# ---- screen --------------------------------------------------------------------------------------------------------
def test_extend_keeps_the_screen(vdb):
    n0, n, d, nq = 30000, 50000, 128, 64
    rng = np.random.default_rng(991)
    W = rng.standard_normal((16, d)).astype(np.float32)
    X = (rng.standard_normal((n, 16)).astype(np.float32) @ W + 0.01 * rng.standard_normal((n, d)).astype(np.float32)).astype(np.float32)
    Q = X[n0 + rng.integers(0, n - n0, nq)] + 0.05 * rng.standard_normal((nq, d)).astype(np.float32)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.build(n0)
    ix.config(200, 200)
    ix.search(Q, 10)
    info0 = ix.graph_screen_info()
    assert info0["active"] and info0["n_screened"] > 0
    ix.extend_graph(n)
    info1 = ix.graph_screen_info()
    assert info1["active"] and info1["share"] == info0["share"]
    assert info1["n_screened"] == info0["n_screened"], "the extension's own searches were screened"
    ids, ds, cnt, st = ix.search(Q, 10)
    assert (ids >= n0).mean() > 0.2  # the searches reach the new rows
    info2 = ix.graph_screen_info()
    assert info2["n_screened"] > info1["n_screened"]
    ix.set_graph_screen(0)
    oids, ods, ocnt, ost = ix.search(Q, 10)
    assert np.array_equal(ids, oids) and np.array_equal(ds, ods) and np.array_equal(cnt, ocnt)
    for k in ("n_dist", "n_seed", "n_expand", "n_edges"):
        assert st[k] == ost[k], k
    ix.close()


# ---- errors and views --------------------------------------------------------------------------------------------
def test_extend_errors_and_views(vdb):
    from vectordb_b200 import EpsError
    n0, n, d = 3000, 5000, 32
    X = gen(n, d, 995, "cluster")
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n - 500)

    def refused(code, *args, on=None):
        with pytest.raises(EpsError) as e:
            (on or ix).extend_graph(*args)
        assert e.value.code == code, (args, e.value)
        return str(e.value)

    assert "eps_index_build" in refused(40005, n0)  # no graph installed
    ix.build(n0)
    g0 = ix.get_graph()
    refused(40005, n0 - 1)
    refused(40005, n)  # above the mirrored rows
    refused(40006, 1 << 31)
    v = ix.view()
    refused(40005, n - 500)  # live view
    refused(40005, n - 500, on=v)  # a view
    v.close()
    assert same_graph(ix.get_graph(), g0), "a refused call changed the graph"
    ix.extend_graph(n0)  # no-op
    assert same_graph(ix.get_graph(), g0)
    ix.extend_graph(n - 500)
    ix.sync_rows(n)
    ix.extend_graph(n)
    assert ix.get_graph()[0] == n
    Q = gen(32, d, 996, "cluster")
    ix.config(300, 300)
    ids, ds, cnt, _ = ix.search(Q, 10)
    v = ix.view()
    vids, vds, vcnt, _ = v.search(Q, 10)
    assert np.array_equal(ids, vids) and np.array_equal(ds, vds) and np.array_equal(cnt, vcnt)
    v.close()
    ix.close()
    sp = vdb.SparseIndex("l2", 100, capacity=10)
    with pytest.raises(EpsError) as e:
        sp.extend_graph(0)
    assert e.value.code == 40005
    sp.close()
