"""Graph search of sparse-vector fields on the GPU (eps_index_set_sparse_search(ix, EPS_SPARSE_SEARCH_GRAPH)).

The expected answers come from sparse_graph_model.port_model: the oracle port run on the graph the device built, with
the distances of the numpy fp32 restatement of vector.cpp (test_gpu_sparse.ref_distances); test_sparse_graph_golden.py
pins that model to the reference's own sparse Search.  Ids, counts, n_dist and n_expand must be identical and distances
bitwise equal."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_sparse import (IP, L2, COS, NT_INT4_ATTR, NT_INT_CONST, NT_NE, NT_STRING_ATTR, NT_STRING_CONST,  # noqa: E402
                             assert_bitwise, attr_lt, csr_slice, densify, distance_lt, ref_distances, ref_search,
                             sparse_rows)
from sparse_graph_model import port_model  # noqa: E402

pytestmark = pytest.mark.gpu

GRAPH = "graph"


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200
    assert vectordb_b200.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    return vectordb_b200


def check(ix, port, qs, D, graph, L, limit, what, **kw):
    """Device search in graph mode == port model: ids, counts, bitwise distances, n_dist and n_expand."""
    ix.config(L, L)
    got = ix.search(qs, limit, filter_nodes=kw.get("nodes_dev", kw.get("nodes")))
    want = port_model(port, D, graph, L, limit, deleted=kw.get("deleted"), attrs=kw.get("attrs"),
                      stride=kw.get("stride", 0), nodes=kw.get("nodes"))
    assert_bitwise(got, want[:3], what)
    st = got[3]
    assert st["n_dist"] == want[3].sum(), "%s: n_dist %d != %d" % (what, st["n_dist"], want[3].sum())
    assert st["n_expand"] == want[4].sum(), "%s: n_expand %d != %d" % (what, st["n_expand"], want[4].sum())
    assert st["n_seed"] == D.shape[0] * min(L, graph[0])
    return got


def string_ne(code):
    """Device: string column 0 <> the literal whose dictionary code is `code`."""
    return np.array([[NT_STRING_ATTR, 0, -1, -1, 0, 0, 0, 0], [NT_STRING_CONST, 0, -1, -1, code, 0, 0, -1],
                     [NT_NE, 3, 0, 1, 0, 0, 0, -1]], np.int64)


def code_ne(code):
    """Port: the same predicate on the codes stored as an INT4 attribute at byte 4 of the row."""
    return np.array([[NT_INT4_ATTR, 1, -1, -1, 0, 0, 0, 4], [NT_INT_CONST, 1, -1, -1, code, 0, 0, -1],
                     [NT_NE, 3, 0, 1, 0, 0, 0, -1]], np.int64)


@pytest.mark.parametrize("metric", [L2, IP, COS])
def test_sparse_graph_matches_port(vdb, port, metric):
    n_graph, n, vocab, nq = 5000, 6000, 2000, 16
    # cosine: no empty rows or queries (0/0 = NaN, whose order the reference leaves unspecified)
    rows = sparse_rows(n, vocab, 51, empty_every=0 if metric == COS else 97)
    qs = sparse_rows(nq, vocab, 52, max_nnz=40, empty_every=0, dup_every=0)
    if metric != COS:
        qs = (np.concatenate([qs[0], [qs[0][-1]]]), qs[1], qs[2])  # + one empty query
    R, Qd = densify(rows, vocab), densify(qs, vocab)
    D = ref_distances(R, Qd, metric)
    a = (np.arange(n) * 7 % 100).astype(np.int32)
    codes = (np.arange(n) % 5).astype(np.int32)
    attrs = np.ascontiguousarray(np.stack([a, codes], 1)).view(np.uint8).ravel()

    ix = vdb.SparseIndex(metric, vocab)
    ix.append(csr_slice(rows, 0, n_graph))
    ix.build(n_graph)
    graph = ix.get_graph()
    assert graph[0] == n_graph
    ix.set_search_mode(GRAPH)
    check(ix, port, qs, D[:, :n_graph], graph, 100, 10, "no tail, L=100")

    ix.append(csr_slice(rows, n_graph, n), first_row=n_graph)
    ix.set_attrs(attrs, 8, n)
    ix.set_string_codes(0, 0, codes)
    for L in (16, 100, 500):
        for limit in (10, 50):  # L = 16, limit 50: L_local < limit
            check(ix, port, qs, D, graph, L, limit, "tail, L=%d limit=%d" % (L, limit))
    deleted = np.zeros((n + 7) // 8, np.uint8)
    dead = np.concatenate([np.arange(3, n, 41), [graph[3]]])  # + the navigation point
    np.bitwise_or.at(deleted, dead >> 3, (1 << (dead & 7)).astype(np.uint8))
    ix.set_deleted(deleted)
    kw = dict(deleted=deleted, attrs=attrs, stride=8)
    check(ix, port, qs, D, graph, 100, 10, "deleted", **kw)
    check(ix, port, qs, D, graph, 100, 10, "numeric filter", nodes=attr_lt(30), **kw)
    thr = float(np.median(D[np.isfinite(D)]))
    check(ix, port, qs, D, graph, 100, 10, "@distance filter", nodes=distance_lt(thr), **kw)
    check(ix, port, qs, D, graph, 500, 50, "string filter", nodes=code_ne(3), nodes_dev=string_ne(3), **kw)
    ix.close()


def clustered_rows(n_clusters, per, terms, pick, seed):
    """Clusters with disjoint vocabularies: cluster c uses terms [c * terms, (c + 1) * terms), each row `pick` of them
    with positive values, so that two rows of one cluster always share a term and rows of different clusters none."""
    rng = np.random.default_rng(seed)
    off, idx, val = [0], [], []
    for c in range(n_clusters):
        for _ in range(per):
            t = np.sort(rng.choice(terms, size=pick, replace=False)) + c * terms
            idx.append(t)
            val.append((rng.random(pick, dtype=np.float32) * 0.9 + 0.1).astype(np.float32))
            off.append(off[-1] + pick)
    return np.array(off, np.int64), np.concatenate(idx).astype(np.int64), np.concatenate(val).astype(np.float32)


def test_sparse_graph_long_navigation_row(vdb, port):
    """With out_degree 8 and clusters of 20 rows, the kNN lists stay inside the clusters: the build's repair makes every
    other cluster an entry of the navigation row, which is then longer than one 128-id chunk."""
    n_clusters, per, terms, vocab = 150, 20, 8, 150 * 8
    n = n_clusters * per
    rows = clustered_rows(n_clusters, per, terms, 5, 61)
    rng = np.random.default_rng(62)
    qrows = []
    for c in rng.choice(n_clusters, 12, replace=False):
        qrows.append((np.sort(rng.choice(terms, 4, replace=False)) + c * terms, rng.random(4, dtype=np.float32) + 0.1))
    qs = (np.concatenate([[0], np.cumsum([q[0].size for q in qrows])]).astype(np.int64),
          np.concatenate([q[0] for q in qrows]).astype(np.int64), np.concatenate([q[1] for q in qrows]).astype(np.float32))
    D = ref_distances(densify(rows, vocab), densify(qs, vocab), IP)
    ix = vdb.SparseIndex("ip", vocab)
    ix.append(rows)
    ix.build(n, out_degree=8)
    graph = ix.get_graph()
    _, off, _, nav = graph
    assert off[nav + 1] - off[nav] > 128, "navigation row has %d entries" % (off[nav + 1] - off[nav])
    ix.set_search_mode(GRAPH)
    for L in (100, 300):
        check(ix, port, qs, D, graph, L, 10, "clusters, L=%d" % L)
    ix.close()


def test_sparse_graph_bitmap_fallback(vdb, port):
    """L = 4096 on 20 000 rows: queries visit more ids than 3/4 of their 16384-entry hash set and move to the bitmap."""
    n, vocab, nq, L = 20000, 2000, 8, 4096
    rows = sparse_rows(n, vocab, 71)
    qs = sparse_rows(nq, vocab, 72, max_nnz=35, empty_every=0, dup_every=0)
    D = ref_distances(densify(rows, vocab), densify(qs, vocab), L2)
    ix = vdb.SparseIndex("l2", vocab)
    ix.append(rows)
    ix.build(n)
    graph = ix.get_graph()
    ix.set_search_mode(GRAPH)
    got = check(ix, port, qs, D, graph, L, 20, "bitmap fallback")
    assert got[3]["n_dist"] > nq * 12288, "queries did not outgrow their hash set"
    again = ix.search(qs, 20)
    assert np.array_equal(again[0], got[0]) and np.array_equal(again[1].view(np.uint64), got[1].view(np.uint64))
    ix.close()


def test_sparse_graph_bitmap_touched_words_clear(vdb, port):
    """L = 64 on 640 000 short rows: every query evaluates more rows than the 768 inserts its 1024-entry hash set
    allows, so it moves to the bitmap, and ten times its rows stay under the bitmap's 20 000 words, so the clean-up
    clears only the words it touched.  A word left dirty would change the second search."""
    n, vocab, nq, L = 640_000, 64, 4, 64
    rows = sparse_rows(n, vocab, 73, max_nnz=4)
    qs = sparse_rows(nq, vocab, 74, max_nnz=6, empty_every=0, dup_every=0)
    D = ref_distances(densify(rows, vocab), densify(qs, vocab), L2)
    ix = vdb.SparseIndex("l2", vocab)
    ix.append(rows)
    ix.build(n, out_degree=50)
    graph = ix.get_graph()
    ix.set_search_mode(GRAPH)
    n_dist = port_model(port, D, graph, L, 10)[3]  # per query; check() holds the device's total to their sum
    assert (n_dist > 768).all(), "n_dist per query %s: not every query moved to the bitmap" % n_dist
    assert (10 * n_dist < (n + 31) // 32).all(), "n_dist per query %s: the bitmap is cleared whole" % n_dist
    for run in (1, 2):
        check(ix, port, qs, D, graph, L, 10, "touched-words clear, search %d" % run)
    ix.close()


def test_sparse_graph_branch_rule(vdb):
    n, vocab, nq = 3000, 2000, 8
    rows = sparse_rows(n, vocab, 81)
    qs = sparse_rows(nq, vocab, 82, max_nnz=30, empty_every=0, dup_every=0)
    D = ref_distances(densify(rows, vocab), densify(qs, vocab), IP)
    attr = (np.arange(n) * 7 % 100).astype(np.int32)
    ix = vdb.SparseIndex("ip", vocab)
    ix.append(rows)
    ix.set_attrs(attr.view(np.uint8), 4, n)
    ix.build(n)
    ix.set_search_mode(GRAPH)
    ix.config(100, 100, force_brute=True)
    assert_bitwise(ix.search(qs, 10), ref_search(D, 10, 10), "graph mode, force_brute")
    ix.config(100, 100, prefilter=True)
    assert_bitwise(ix.search(qs, 20, filter_nodes=attr_lt(10)), ref_search(D, 20, 20, keep=attr < 10),
                   "graph mode, prefilter")
    ix.config(100, 100)
    st = ix.search(qs, 10)[3]
    assert st["n_expand"] > 0 and st["n_seed"] == nq * 100 and st["n_dist"] < nq * n
    ix.close()

    small = vdb.SparseIndex("ip", vocab)   # 400 indexed rows: below the reference's BruteforceThreshold (512)
    small.append(csr_slice(rows, 0, 1000))
    small.build(400)
    small.set_search_mode(GRAPH)
    small.config(100, 7)
    got = small.search(qs, 10)
    assert_bitwise(got, ref_search(D[:, :1000], 10, 7), "graph mode, 400 indexed rows")
    assert got[3]["n_expand"] == 0 and got[3]["n_dist"] == nq * 1000
    for bad in (2, -1):
        assert small.L.eps_index_set_sparse_search(small.h, bad) == 40005
    small.close()

    dense = vdb.Index("l2", 4, host_vectors=np.zeros((4, 4), np.float32))
    assert dense.L.eps_index_set_sparse_search(dense.h, 1) == 40005
    assert dense.L.eps_index_set_sparse_search(dense.h, 0) == 40005
    dense.close()


def test_sparse_graph_view_concurrent_and_repeated(vdb):
    import threading
    n, vocab = 8000, 2000
    rows = sparse_rows(n, vocab, 91)
    qs = sparse_rows(256, vocab, 92, max_nnz=40, empty_every=0, dup_every=0)
    ix = vdb.SparseIndex("l2", vocab)
    ix.append(csr_slice(rows, 0, 7000))
    ix.build(7000)
    ix.append(csr_slice(rows, 7000, n), first_row=7000)
    ix.config(200, 200)
    scan = ix.search(qs, 10)
    ix.set_search_mode(GRAPH)
    want = ix.search(qs, 10)
    v = ix.view()   # starts in its base's mode
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
        assert res[3]["n_dist"] == want[3]["n_dist"] and res[3]["n_expand"] == want[3]["n_expand"]
    v.set_search_mode("scan")   # a view's own mode
    got = v.search(qs, 10)
    assert np.array_equal(got[0], scan[0]) and np.array_equal(got[1].view(np.uint64), scan[1].view(np.uint64))
    again = ix.search(qs, 10)
    assert np.array_equal(again[0], want[0]) and again[3]["n_expand"] == want[3]["n_expand"]
    v.close()
    ix.close()
