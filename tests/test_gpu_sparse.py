"""Sparse-vector fields on the GPU (eps_index_create_sparse / eps_search_sparse_batch / eps_index_build).

The expected results come from a restatement of the reference's sparse distances (engine/db/vector.cpp:7-100) in
numpy float32: every term and every partial sum is one IEEE fp32 operation, in the reference's order, so the device's
distances must be BITWISE equal (up to the sign of zero, which the (distance, id) keys fold), and ids identical."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

L2, COS, IP = 1, 2, 3
NT_INT_CONST, NT_DOUBLE_CONST, NT_INT4_ATTR, NT_STRING_ATTR, NT_STRING_CONST, NT_DOUBLE_ATTR = 1, 3, 7, 9, 2, 10
NT_LT, NT_EQ, NT_GT, NT_NE = 19, 21, 22, 24


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200
    assert vectordb_b200.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    return vectordb_b200


# ---- seeded sparse tables --------------------------------------------------------------------------------------
def sparse_rows(n, vocab, seed, max_nnz=60, empty_every=97, dup_every=53):
    """CSR rows with Zipf-like term ids, nnz spread over [0, max_nnz], some empty rows and exact duplicate rows."""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, vocab + 1) ** 0.9
    w /= w.sum()
    rows = []
    for r in range(n):
        if empty_every and r % empty_every == 5:
            rows.append((np.zeros(0, np.int64), np.zeros(0, np.float32)))
            continue
        if dup_every and r % dup_every == 7 and r > 10:
            rows.append(rows[r - 9])
            continue
        k = int(rng.integers(1, max_nnz + 1))
        idx = np.unique(rng.choice(vocab, size=k, p=w))
        val = (rng.random(idx.size, dtype=np.float32) * 2 - 0.5).astype(np.float32)
        rows.append((idx.astype(np.int64), val))
    off = np.zeros(n + 1, np.int64)
    off[1:] = np.cumsum([r[0].size for r in rows])
    idx = np.concatenate([r[0] for r in rows]) if off[-1] else np.zeros(0, np.int64)
    val = np.concatenate([r[1] for r in rows]) if off[-1] else np.zeros(0, np.float32)
    return off, idx, val.astype(np.float32)


def csr_slice(csr, lo, hi):
    off, idx, val = csr
    return off[lo:hi + 1] - off[lo], idx[off[lo]:off[hi]], val[off[lo]:off[hi]]


def densify(csr, vocab):
    off, idx, val = csr
    n = off.size - 1
    M = np.zeros((n, vocab), np.float32)
    rows = np.repeat(np.arange(n), np.diff(off))
    M[rows, idx] = val
    return M


def ref_distances(R, Qd, metric):
    """[nq x n] float32 distances of vector.cpp with row = v1, query = v2.  Summing over every column in increasing
    order reproduces the reference's merge order exactly: a column missing from both vectors adds an exact zero."""
    cols = np.nonzero((R != 0).any(0) | (Qd != 0).any(0))[0]
    acc = np.zeros((Qd.shape[0], R.shape[0]), np.float32)
    if metric == L2:
        for c in cols:
            d = R[None, :, c] - Qd[:, c, None]
            acc = acc + d * d
        return acc
    for c in cols:
        acc = acc + R[None, :, c] * Qd[:, c, None]
    if metric == IP:
        return -acc
    rn = np.zeros(R.shape[0], np.float32)
    qn = np.zeros(Qd.shape[0], np.float32)
    for c in cols:
        rn = rn + R[:, c] * R[:, c]
        qn = qn + Qd[:, c] * Qd[:, c]
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.float32(1) - acc / np.sqrt(rn[None, :] * qn[:, None])


def ref_search(D, k, cap, keep=None, dyn=None):
    """BruteForceSearch: drop deleted / failing rows (dyn sees the distance), sort by (distance, id), NaN last."""
    nq, n = D.shape
    ids = np.full((nq, k), -1, np.int64)
    ds = np.full((nq, k), np.inf, np.float64)
    cnt = np.zeros(nq, np.int64)
    for q in range(nq):
        ok = np.ones(n, bool) if keep is None else keep.copy()
        if dyn is not None:
            ok &= dyn(D[q].astype(np.float64))
        rows = np.nonzero(ok)[0]
        d = D[q, rows] + np.float32(0)
        order = np.lexsort((rows, d))[:min(k, cap)]
        cnt[q] = order.size
        ids[q, :order.size] = rows[order]
        ds[q, :order.size] = d[order]
    return ids, ds, cnt


def assert_bitwise(got, want, what):
    gi, gd, gc = got[:3]
    wi, wd, wc = want
    assert np.array_equal(gc, wc), what + ": counts"
    assert np.array_equal(gi, wi), what + ": ids"
    a = (gd.astype(np.float32) + np.float32(0)).view(np.uint32)
    b = (wd.astype(np.float32) + np.float32(0)).view(np.uint32)
    nan = np.isnan(wd)
    assert np.array_equal(np.isnan(gd), nan), what + ": NaN positions"
    assert np.array_equal(a[~nan], b[~nan]), what + ": distances are not bitwise equal"


def distance_lt(c):
    return np.array([[NT_DOUBLE_ATTR, 2, -1, -1, 0, 0, 0, -2],
                     [NT_DOUBLE_CONST, 2, -1, -1, 0, np.float64(c).view(np.int64), 0, -1],
                     [NT_LT, 3, 0, 1, 0, 0, 0, -1]], np.int64)


def attr_lt(c):
    return np.array([[NT_INT4_ATTR, 1, -1, -1, 0, 0, 0, 0], [NT_INT_CONST, 1, -1, -1, c, 0, 0, -1],
                     [NT_LT, 3, 0, 1, 0, 0, 0, -1]], np.int64)


# ---- exact scan: three metrics, every mode -----------------------------------------------------------------------
@pytest.mark.parametrize("metric", [L2, IP, COS])
def test_sparse_scan_bitwise_all_modes(vdb, metric):
    n, vocab, nq = 3000, 2000, 24
    rows = sparse_rows(n, vocab, 11)
    qs = sparse_rows(nq, vocab, 12, max_nnz=40, empty_every=0, dup_every=0)
    qs = (np.concatenate([qs[0], [qs[0][-1]]]), qs[1], qs[2])  # + one empty query
    R, Qd = densify(rows, vocab), densify(qs, vocab)
    D = ref_distances(R, Qd, metric)
    attr = (np.arange(n) * 7 % 100).astype(np.int32)
    deleted = np.zeros((n + 7) // 8, np.uint8)
    dead = np.arange(3, n, 41)
    np.bitwise_or.at(deleted, dead >> 3, (1 << (dead & 7)).astype(np.uint8))
    alive = np.ones(n, bool)
    alive[dead] = False

    ix = vdb.SparseIndex(metric, vocab, capacity=1000)
    ix.append(rows)
    ix.set_attrs(attr.view(np.uint8), 4, n)
    k = 10
    ix.config(500, 500, force_brute=True)
    got = ix.search(qs, k)
    assert_bitwise(got, ref_search(D, k, k), "force_brute")
    assert got[3]["n_dist"] == (nq + 1) * n
    ix.config(500, 7)   # brute-force branch of an un-indexed table: min(limit, L_local) results
    assert_bitwise(ix.search(qs, k), ref_search(D, k, 7), "brute L_local=7")
    ix.config(500, 500, force_brute=True)
    ix.set_deleted(deleted)
    assert_bitwise(ix.search(qs, k), ref_search(D, k, k, keep=alive), "deleted")
    assert_bitwise(ix.search(qs, k, filter_nodes=attr_lt(30)), ref_search(D, k, k, keep=alive & (attr < 30)),
                   "numeric filter")
    thr = float(np.nanmedian(D))
    assert_bitwise(ix.search(qs, k, filter_nodes=distance_lt(thr)),
                   ref_search(D, k, k, keep=alive, dyn=lambda d: d < thr), "@distance filter")
    ix.config(500, 500, prefilter=True)   # pre-filter: the filter sees distance 0
    assert_bitwise(ix.search(qs, 50, filter_nodes=attr_lt(10)), ref_search(D, 50, 50, keep=alive & (attr < 10)),
                   "prefilter")
    ix.close()


def test_sparse_scan_matches_reference_golden(vdb):
    """tests/golden/sparse.npz holds the reference's own VecSearchExecutor::Search answers (make_sparse_golden.py):
    brute force, the L_local cap, deleted rows, numeric / @distance / string filters and pre-filter, three metrics."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_sparse_golden import CASES, THR, crc, table
    from sparse_golden_check import GOLDEN, check_against_golden
    g = np.load(GOLDEN)
    for metric in (L2, COS, IP):
        n, vocab, rows, qs, attr, codes, dead = table(metric)
        assert crc(*rows, *qs) == int(g["m%d_table_crc32" % metric])
        ix = vdb.SparseIndex(metric, vocab)
        ix.append(rows)
        ix.set_attrs(attr.view(np.uint8), 4, n)
        ix.set_string_codes(0, 0, codes)   # dictionary: code c <-> the string "v<c>"
        deleted = np.zeros((n + 7) // 8, np.uint8)
        np.bitwise_or.at(deleted, dead >> 3, (1 << (dead & 7)).astype(np.uint8))
        for name, pre, ll, limit, _, use_del in CASES:
            ix.config(500, ll, prefilter=pre)
            ix.set_deleted(deleted if use_del else np.zeros(0, np.uint8))
            nodes = {"numeric": attr_lt(30), "prefilter": attr_lt(10), "distance": distance_lt(THR[metric]),
                     "string": np.array([[NT_STRING_ATTR, 0, -1, -1, 0, 0, 0, 0], [NT_STRING_CONST, 0, -1, -1, 3, 0, 0, -1],
                                         [NT_NE, 3, 0, 1, 0, 0, 0, -1]], np.int64)}.get(name)
            ids, ds, cnt, _ = ix.search(qs, limit, filter_nodes=nodes)
            check_against_golden(g, "m%d_%s" % (metric, name), ids, ds, cnt, metric)
        ix.close()


def test_sparse_appends_deleted_and_string_filter_20k(vdb):
    n, vocab, nq, k = 20000, 2000, 16, 20
    rows = sparse_rows(n, vocab, 21)
    qs = sparse_rows(nq, vocab, 22, max_nnz=35, empty_every=0, dup_every=0)
    D = ref_distances(densify(rows, vocab), densify(qs, vocab), IP)
    codes = (np.arange(n) % 5).astype(np.int32)
    ix = vdb.SparseIndex("ip", vocab)
    ix.append(csr_slice(rows, 0, 12345))
    ix.set_string_codes(0, 0, codes[:12345])
    ix.config(500, 500, force_brute=True)
    assert_bitwise(ix.search(qs, k), ref_search(D[:, :12345], k, k), "first append")
    ix.append(csr_slice(rows, 12345, n), first_row=12345)
    ix.set_string_codes(0, 12345, codes[12345:])
    deleted = np.zeros((n + 7) // 8, np.uint8)
    deleted[::13] = 0x21
    alive = ~np.unpackbits(deleted, bitorder="little")[:n].astype(bool)
    ix.set_deleted(deleted)
    eq3 = np.array([[NT_STRING_ATTR, 0, -1, -1, 0, 0, 0, 0], [NT_STRING_CONST, 0, -1, -1, 3, 0, 0, -1],
                    [NT_NE, 3, 0, 1, 0, 0, 0, -1]], np.int64)
    assert_bitwise(ix.search(qs, k, filter_nodes=eq3), ref_search(D, k, k, keep=alive & (codes != 3)),
                   "second append + deleted + string filter")
    ix.close()


def test_sparse_rejects_malformed_rows_and_dense_calls(vdb):
    ix = vdb.SparseIndex("l2", 100)
    ix.append((np.array([0, 2, 2]), np.array([1, 5]), np.array([1, 2], np.float32)))
    for bad in ((np.array([0, 2]), np.array([5, 1]), np.ones(2, np.float32)),     # unsorted
                (np.array([0, 2]), np.array([5, 5]), np.ones(2, np.float32)),     # repeated
                (np.array([0, 1]), np.array([100]), np.ones(1, np.float32)),      # >= dim
                (np.array([0, 1]), np.array([-1]), np.ones(1, np.float32))):      # negative
        with pytest.raises(vdb.EpsError) as e:
            ix.append(bad)
        assert e.value.code == 40005
    assert ix.rows == 2
    with pytest.raises(vdb.EpsError):
        ix.append((np.array([0, 1]), np.array([3]), np.ones(1, np.float32)), first_row=5)   # gap
    L = ix.L
    for call in (lambda: L.eps_index_sync_rows(ix.h, 2), lambda: L.eps_index_set_search_width(ix.h, 2),
                 lambda: L.eps_index_set_coarse(ix.h, 0), lambda: L.eps_index_set_graph_tuning(ix.h, 0, 0),
                 lambda: L.eps_index_set_graph(ix.h, 0, None, None, 0),
                 lambda: L.eps_search_batch(ix.h, np.zeros(100, np.float32).ctypes.data, 1, 1, None, 0,
                                            np.zeros(1, np.int64).ctypes.data, np.zeros(1).ctypes.data,
                                            np.zeros(1, np.int64).ctypes.data, None)):
        assert call() == 40005
    buf = np.zeros(64, np.int64)
    assert L.eps_index_adopt_device_rows(ix.h, buf.ctypes.data, 1) == 40005
    assert L.eps_search_batch_device(ix.h, buf.ctypes.data, 1, 1, None, 0, buf.ctypes.data, buf.ctypes.data,
                                     buf.ctypes.data, None, 1) == 40005
    from vectordb_b200.sharded import ShardGroup
    g = ShardGroup(ShardGroup.unique_id(), 0, 1, 0)
    assert L.eps_search_batch_sharded(g.h, ix.h, 0, buf.ctypes.data, 1, 1, None, 0, buf.ctypes.data, buf.ctypes.data,
                                      None, 1) == 40005
    g.close()
    assert L.eps_index_device_rows(ix.h) is None
    dense = vdb.Index("l2", 4, host_vectors=np.zeros((4, 4), np.float32))
    with pytest.raises(vdb.EpsError):
        vdb.SparseIndex.append(dense, (np.array([0, 1]), np.array([1]), np.ones(1, np.float32)), first_row=0)
    dense.close()
    ix.close()


def test_sparse_view_searches_concurrently(vdb):
    import threading
    n, vocab = 8000, 2000
    rows = sparse_rows(n, vocab, 31)
    qs = sparse_rows(64, vocab, 32, max_nnz=40, empty_every=0, dup_every=0)
    ix = vdb.SparseIndex("cosine", vocab)
    ix.append(rows)
    ix.config(500, 500, force_brute=True)
    want = ix.search(qs, 10)
    v = ix.view()
    assert isinstance(v, vdb.SparseIndex)   # searches take CSR queries through eps_search_sparse_batch
    out = {}
    def run(name, index):
        out[name] = [index.search(qs, 10) for _ in range(4)]
    ts = [threading.Thread(target=run, args=("base", ix)), threading.Thread(target=run, args=("view", v))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for res in out["base"] + out["view"]:
        assert np.array_equal(res[0], want[0]) and np.array_equal(res[2], want[2])
        assert np.array_equal(res[1].view(np.uint64), want[1].view(np.uint64))
    with pytest.raises(vdb.EpsError):
        ix.append(qs)   # a base with live views is frozen
    v.close()
    # a base destroyed before its view leaves an empty index behind, not a dangling one
    v2 = ix.view()
    ix.close()
    _, _, c2, _ = v2.search(qs, 10)
    assert (c2 == 0).all()
    v2.close()


def test_sparse_graph_build(vdb):
    """Lists = exact top-out_degree by (distance, id) without self; nav = exact L2 nearest row to the reference's
    sparse centre (last value per index / n); every row reachable from nav; the graph round-trips get_graph."""
    n, vocab, R_deg = 5000, 2000, 50
    rows = sparse_rows(n, vocab, 41)
    R = densify(rows, vocab)
    ix = vdb.SparseIndex("ip", vocab)
    ix.append(rows)
    ix.build(n)
    ni, off, nb, nav = ix.get_graph()
    assert ni == n and off[0] == 0 and off[-1] == nb.size
    # lists of a sample of vertices: their first out_degree entries are the exact kNN list
    sample = np.arange(0, n, 19)
    D = ref_distances(R, R[sample], IP)
    for i, v in enumerate(sample):
        d = D[i] + np.float32(0)
        d[v] = np.inf
        order = np.lexsort((np.arange(n), d))
        order = order[order != v][:R_deg]
        assert np.array_equal(nb[off[v]:off[v] + R_deg], order), "vertex %d: list is not the exact kNN list" % v
    # navigation point: exact L2 nearest row to the centre (std::map of the last value seen per index, / n)
    last = {}
    o, ii, vv = rows
    for j in range(ii.size):
        last[int(ii[j])] = vv[j]
    centre = np.zeros((1, vocab), np.float32)
    for key, val in last.items():
        centre[0, key] = np.float32(val) / np.float32(n)
    dc = ref_distances(R, centre, L2)[0] + np.float32(0)
    assert nav == int(np.lexsort((np.arange(n), dc))[0])
    # reachability from nav
    seen = np.zeros(n, bool)
    seen[nav] = True
    frontier = [nav]
    while frontier:
        nxt = []
        for u in frontier:
            for w in nb[off[u]:off[u + 1]]:
                if not seen[w]:
                    seen[w] = True
                    nxt.append(int(w))
        frontier = nxt
    assert seen.all()
    # searches still answer by exact scan with a graph installed
    ix.config(500, 500)
    qs = sparse_rows(8, vocab, 42, max_nnz=30, empty_every=0, dup_every=0)
    Dq = ref_distances(R, densify(qs, vocab), IP)
    assert_bitwise(ix.search(qs, 10), ref_search(Dq, 10, 10), "search with a graph installed")
    ix.close()


@pytest.mark.parametrize("metric", ["ip", "l2"])
def test_sparse_graph_build_ignores_deleted_rows(vdb, metric):
    """The sparse build indexes every row, deleted or not: a deleted bitset leaves the kNN lists and the L2 navigation
    point unchanged.  The bitset deletes the navigation point itself, so a scan that skipped deleted rows would pick
    another."""
    n, vocab = 3000, 2000
    rows = sparse_rows(n, vocab, 43)
    ix = vdb.SparseIndex(metric, vocab)
    ix.append(rows)
    ix.build(n)
    want = ix.get_graph()
    bits = np.full(n // 8 + 1, 0x5A, np.uint8)
    nav = want[3]
    bits[nav >> 3] |= 1 << (nav & 7)
    ix.set_deleted(bits)
    ix.build(n)
    got = ix.get_graph()
    for name, a, b in zip(("n_indexed", "offsets", "neighbours", "nav"), got, want):
        assert np.array_equal(a, b), name
    ix.close()
