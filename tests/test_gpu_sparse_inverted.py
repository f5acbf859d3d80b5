"""Inverted index of sparse IP / cosine fields on the GPU (eps_index_build_sparse_inverted).

The index changes no result: with posting lists built, every exact scan computes the covered rows' distances from them,
and ids, counts, n_dist (and n_expand in graph mode) must equal those of the same index without postings, with distances
bitwise equal; where the table is small enough they are also checked against the numpy restatement of vector.cpp
(test_gpu_sparse.ref_distances / ref_search)."""
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_sparse import (IP, COS, NT_NE, NT_STRING_ATTR, NT_STRING_CONST, assert_bitwise,  # noqa: E402
                             attr_lt, csr_slice, densify, distance_lt, ref_distances, ref_search, sparse_rows)

pytestmark = pytest.mark.gpu

STRING_NE3 = np.array([[NT_STRING_ATTR, 0, -1, -1, 0, 0, 0, 0], [NT_STRING_CONST, 0, -1, -1, 3, 0, 0, -1],
                       [NT_NE, 3, 0, 1, 0, 0, 0, -1]], np.int64)


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200
    assert vectordb_b200.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    return vectordb_b200


def with_empty_query(qs):
    return np.concatenate([qs[0], [qs[0][-1]]]), qs[1], qs[2]


def same(a, b, what, stats=("n_dist",)):
    """a (with postings) == b (without): ids, counts, bitwise distances and the named counters."""
    assert_bitwise(a, b[:3], what)
    for s in stats:
        assert a[3][s] == b[3][s], "%s: %s %d != %d" % (what, s, a[3][s], b[3][s])


def make_pair(vdb, metric, vocab, rows, n_attr=None):
    """The same table twice: one index with postings over every row, one without."""
    out = []
    for inverted in (True, False):
        ix = vdb.SparseIndex(metric, vocab)
        ix.append(rows)
        if n_attr is not None:
            attr, codes = n_attr
            ix.set_attrs(attr.view(np.uint8), 4, attr.size)
            ix.set_string_codes(0, 0, codes)
        if inverted:
            ix.build_inverted()
        out.append(ix)
    return out


@pytest.mark.parametrize("metric", [IP, COS])
def test_inverted_matches_model_and_scan(vdb, metric):
    n, vocab = 5000, 2000   # 5000 rows: the last 2048-row slice is partial
    rows = sparse_rows(n, vocab, 61)   # empty rows, duplicate rows, negative values
    qs = with_empty_query(sparse_rows(32, vocab, 62, max_nnz=40, empty_every=0, dup_every=0))   # 33 queries
    D = ref_distances(densify(rows, vocab), densify(qs, vocab), metric)
    attr = (np.arange(n) * 7 % 100).astype(np.int32)
    codes = (np.arange(n) % 5).astype(np.int32)
    inv, plain = make_pair(vdb, metric, vocab, rows, (attr, codes))
    info = inv.inverted_info()
    assert info["rows"] == n and info["postings"] == rows[0][-1]
    assert info["terms"] == np.unique(rows[1]).size
    assert plain.inverted_info() == dict(rows=0, terms=0, postings=0)

    def both(what, want, limit, **kw):
        got = inv.search(qs, limit, **kw)
        assert_bitwise(got, want, what)
        same(got, plain.search(qs, limit, **kw), what)
        return got

    for ix in (inv, plain):
        ix.config(500, 500, force_brute=True)
    for k in (1, 10, 500):
        got = both("force_brute k=%d" % k, ref_search(D, k, k), k)
        assert got[3]["n_dist"] == (qs[0].size - 1) * n
    one = csr_slice(qs, 3, 4)
    g1 = inv.search(one, 10)
    assert_bitwise(g1, ref_search(D[3:4], 10, 10), "nq = 1")
    same(g1, plain.search(one, 10), "nq = 1")
    for ix in (inv, plain):
        ix.config(500, 7)   # brute-force branch of an un-indexed table: min(limit, L_local)
    both("L_local cap", ref_search(D, 10, 7), 10)
    dead = np.arange(3, n, 41)
    deleted = np.zeros((n + 7) // 8, np.uint8)
    np.bitwise_or.at(deleted, dead >> 3, (1 << (dead & 7)).astype(np.uint8))
    alive = np.ones(n, bool)
    alive[dead] = False
    for ix in (inv, plain):
        ix.config(500, 500, force_brute=True)
        ix.set_deleted(deleted)
    both("deleted", ref_search(D, 10, 10, keep=alive), 10)
    both("numeric filter", ref_search(D, 10, 10, keep=alive & (attr < 30)), 10, filter_nodes=attr_lt(30))
    thr = float(np.nanmedian(D))
    both("@distance filter", ref_search(D, 10, 10, keep=alive, dyn=lambda d: d < thr), 10, filter_nodes=distance_lt(thr))
    both("string filter", ref_search(D, 10, 10, keep=alive & (codes != 3)), 10, filter_nodes=STRING_NE3)
    for ix in (inv, plain):
        ix.config(500, 500, prefilter=True)
    both("prefilter", ref_search(D, 50, 50, keep=alive & (attr < 10)), 50, filter_nodes=attr_lt(10))
    inv.close()
    plain.close()


def test_inverted_several_row_chunks(vdb):
    """4096 queries over 100 000 rows: the exact scan cuts the rows into chunks of 65 536, and with postings over the first
    70 000 rows the second chunk is read partly from postings and partly by the scan."""
    n, vocab, nq = 100_000, 3000, 4096
    rows = sparse_rows(n, vocab, 71, max_nnz=40)
    qs = sparse_rows(nq, vocab, 72, max_nnz=20, empty_every=0, dup_every=0)
    ix = vdb.SparseIndex("ip", vocab)
    ix.append(rows)
    ix.config(500, 500, force_brute=True)
    want = ix.search(qs, 10)
    for n_inv in (70_000, n):
        ix.build_inverted(n_inv)
        assert ix.inverted_info()["rows"] == n_inv
        same(ix.search(qs, 10), want, "4096 queries, postings over %d rows" % n_inv)
    ix.close()


def test_inverted_reference_golden(vdb):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_sparse_golden import CASES, THR, crc, table
    from sparse_golden_check import GOLDEN, check_against_golden
    g = np.load(GOLDEN)
    for metric in (COS, IP):
        n, vocab, rows, qs, attr, codes, dead = table(metric)
        assert crc(*rows, *qs) == int(g["m%d_table_crc32" % metric])
        ix = vdb.SparseIndex(metric, vocab)
        ix.append(rows)
        ix.set_attrs(attr.view(np.uint8), 4, n)
        ix.set_string_codes(0, 0, codes)
        ix.build_inverted()
        assert ix.inverted_info()["rows"] == n
        deleted = np.zeros((n + 7) // 8, np.uint8)
        np.bitwise_or.at(deleted, dead >> 3, (1 << (dead & 7)).astype(np.uint8))
        for name, pre, ll, limit, _, use_del in CASES:
            ix.config(500, ll, prefilter=pre)
            ix.set_deleted(deleted if use_del else np.zeros(0, np.uint8))
            nodes = {"numeric": attr_lt(30), "prefilter": attr_lt(10), "distance": distance_lt(THR[metric]),
                     "string": STRING_NE3}.get(name)
            ids, ds, cnt, _ = ix.search(qs, limit, filter_nodes=nodes)
            check_against_golden(g, "m%d_%s" % (metric, name), ids, ds, cnt, metric)
        ix.close()


@pytest.mark.parametrize("metric", ["ip", "cosine"])
def test_inverted_partial_coverage_and_appends(vdb, metric):
    n0, n1, n, vocab = 3000, 4500, 7000, 2000
    rows = sparse_rows(n, vocab, 81)
    qs = with_empty_query(sparse_rows(16, vocab, 82, max_nnz=40, empty_every=0, dup_every=0))
    m = {"ip": IP, "cosine": COS}[metric]
    D = ref_distances(densify(rows, vocab), densify(qs, vocab), m)
    ix = vdb.SparseIndex(metric, vocab)
    ix.append(csr_slice(rows, 0, n1))
    ix.config(500, 500, force_brute=True)
    ix.build_inverted(n0)
    assert ix.inverted_info() == dict(rows=n0, terms=np.unique(rows[1][:rows[0][n0]]).size, postings=int(rows[0][n0]))
    assert_bitwise(ix.search(qs, 20), ref_search(D[:, :n1], 20, 20), "postings over %d of %d rows" % (n0, n1))
    ix.append(csr_slice(rows, n1, n), first_row=n1)
    assert ix.inverted_info()["rows"] == n0   # appended rows are scanned until the next build
    got = ix.search(qs, 20)
    assert_bitwise(got, ref_search(D, 20, 20), "after the append")
    assert got[3]["n_dist"] == (qs[0].size - 1) * n
    ix.build_inverted()
    assert ix.inverted_info() == dict(rows=n, terms=np.unique(rows[1]).size, postings=int(rows[0][n]))
    assert_bitwise(ix.search(qs, 20), ref_search(D, 20, 20), "rebuilt over every row")
    ix.build_inverted(0)
    assert ix.inverted_info() == dict(rows=0, terms=0, postings=0)
    assert_bitwise(ix.search(qs, 20), ref_search(D, 20, 20), "dropped")
    ix.close()


@pytest.mark.parametrize("metric", ["ip", "cosine"])
def test_inverted_graph_mode(vdb, metric):
    """Graph mode with a tail: the graph search takes the raw queries and the tail scan reads postings; ids, distances,
    counts, n_dist, n_seed and n_expand are those without postings.  The brute-force branches (force_brute,
    prefilter) too."""
    n_graph, n, vocab = 5000, 6000, 2000
    rows = sparse_rows(n, vocab, 91, empty_every=0 if metric == "cosine" else 97)
    qs = sparse_rows(16, vocab, 92, max_nnz=40, empty_every=0, dup_every=0)
    ix = vdb.SparseIndex(metric, vocab)
    ix.append(csr_slice(rows, 0, n_graph))
    ix.build(n_graph)
    ix.append(csr_slice(rows, n_graph, n), first_row=n_graph)
    ix.set_attrs((np.arange(n) * 7 % 100).astype(np.int32).view(np.uint8), 4, n)
    ix.set_search_mode("graph")
    cases = [(dict(L_master=100), 10, None), (dict(L_master=500), 50, None), (dict(L_master=100), 10, attr_lt(30)),
             (dict(L_master=100, force_brute=True), 10, None), (dict(L_master=100, prefilter=True), 10, attr_lt(30))]
    want = []
    for cfg, limit, nodes in cases:
        ix.config(**cfg)
        want.append(ix.search(qs, limit, filter_nodes=nodes))
    for n_inv in (n, n_graph + 300, 2000):   # covering the tail, part of it, or part of the graph's rows only
        ix.build_inverted(n_inv)
        for (cfg, limit, nodes), w in zip(cases, want):
            ix.config(**cfg)
            same(ix.search(qs, limit, filter_nodes=nodes), w, "graph mode %s, postings over %d rows" % (cfg, n_inv),
                 stats=("n_dist", "n_seed", "n_expand", "n_edges"))
    ix.close()


def test_inverted_query_edges_and_largest_dim(vdb):
    """Empty queries, query terms no row has, indices up to 2^32 - 3 on an index of the largest legal dim, a query index
    of 2^32 - 2 (which no row can hold), and a query of 5 000 elements (more than one batch of term bounds)."""
    dim = 2 ** 32 - 2
    rng = np.random.default_rng(101)
    n, vocab = 3000, 8000
    small = sparse_rows(n, vocab, 102, max_nnz=50)
    small[1][small[0][2] - 1] = vocab - 1   # row 1 ends with the largest index
    # spread the indices over the whole 32-bit range, the largest one a row may hold (2^32 - 3) included
    spread = np.sort(rng.choice(2 ** 32 - 3, size=vocab - 1, replace=False)).astype(np.int64)
    spread = np.concatenate([spread, [2 ** 32 - 3]])
    rows = (small[0], spread[small[1]], small[2])
    q_small = sparse_rows(6, vocab, 103, max_nnz=40, empty_every=0, dup_every=0)
    big_idx = np.sort(rng.choice(vocab, size=5000, replace=False)).astype(np.int64)
    big_val = (rng.random(5000, dtype=np.float32) - 0.3).astype(np.float32)
    # queries: 6 ordinary ones, an empty one, one with absent terms and 2^32 - 2, and the 5000-element one
    parts = [(spread[q_small[1][q_small[0][i]:q_small[0][i + 1]]], q_small[2][q_small[0][i]:q_small[0][i + 1]])
             for i in range(6)]
    absent = np.setdiff1d(np.arange(1, 2 ** 20, 977), spread)[:5]
    parts += [(np.zeros(0, np.int64), np.zeros(0, np.float32)),
              (np.concatenate([np.sort(np.concatenate([absent, spread[1:2]])), [2 ** 32 - 2]]),
               np.full(absent.size + 2, 0.5, np.float32)),
              (spread[big_idx], big_val)]
    off = np.zeros(len(parts) + 1, np.int64)
    off[1:] = np.cumsum([p[0].size for p in parts])
    qs = (off, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]).astype(np.float32))
    # model on compacted columns: the order of the indices is all the sums depend on
    cols = np.unique(np.concatenate([rows[1], qs[1]]))
    compact = lambda csr: (csr[0], np.searchsorted(cols, csr[1]), csr[2])  # noqa: E731
    R, Qd = densify(compact(rows), cols.size), densify(compact(qs), cols.size)
    for metric in (IP, COS):
        D = ref_distances(R, Qd, metric)
        ix = vdb.SparseIndex(metric, dim)
        ix.append(rows)
        ix.config(500, 500, force_brute=True)
        plain = ix.search(qs, 10)
        ix.build_inverted()
        assert ix.inverted_info()["terms"] == np.unique(rows[1]).size
        got = ix.search(qs, 10)
        assert_bitwise(got, ref_search(D, 10, 10), "metric %d: model" % metric)
        same(got, plain, "metric %d: scan" % metric)
        ix.close()


def test_inverted_views(vdb):
    n, vocab = 8000, 2000
    rows = sparse_rows(n, vocab, 111)
    qs = sparse_rows(64, vocab, 112, max_nnz=40, empty_every=0, dup_every=0)
    ix = vdb.SparseIndex("cosine", vocab)
    ix.append(rows)
    ix.config(500, 500, force_brute=True)
    plain = ix.search(qs, 10)
    ix.build_inverted()
    v = ix.view()
    assert v.inverted_info() == ix.inverted_info()
    out = {}

    def run(name, index):
        out[name] = [index.search(qs, 10) for _ in range(4)]
    ts = [threading.Thread(target=run, args=("base", ix)), threading.Thread(target=run, args=("view", v))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for res in out["base"] + out["view"]:
        same(res, plain, "base and view side by side")
    for call in (lambda: v.build_inverted(), lambda: v.build_inverted(0), lambda: ix.build_inverted(),
                 lambda: ix.build_inverted(0)):
        with pytest.raises(vdb.EpsError) as e:
            call()
        assert e.value.code == 40005
    assert ix.inverted_info()["rows"] == n and v.inverted_info()["rows"] == n
    v.close()
    ix.build_inverted(0)   # no live views any more
    assert ix.inverted_info()["rows"] == 0
    ix.close()


def test_inverted_refusals_change_nothing(vdb):
    n, vocab = 4000, 2000
    rows = sparse_rows(n, vocab, 121)
    qs = sparse_rows(16, vocab, 122, max_nnz=40, empty_every=0, dup_every=0)
    l2 = vdb.SparseIndex("l2", vocab)
    l2.append(rows)
    l2.config(500, 500, force_brute=True)
    before = l2.search(qs, 10)
    with pytest.raises(vdb.EpsError) as e:
        l2.build_inverted()
    assert e.value.code == 40006 and "L2" in str(e.value)
    assert l2.inverted_info()["rows"] == 0
    same(l2.search(qs, 10), before, "L2 after the refusal")
    l2.close()

    ix = vdb.SparseIndex("ip", vocab)
    ix.append(rows)
    ix.config(500, 500, force_brute=True)
    ix.build_inverted(3000)
    info, before = ix.inverted_info(), ix.search(qs, 10)
    L = ix.L
    for n_bad in (-1, n + 1):
        assert L.eps_index_build_sparse_inverted(ix.h, n_bad) == 40005
    v = ix.view()
    assert L.eps_index_build_sparse_inverted(v.h, n) == 40005
    assert L.eps_index_build_sparse_inverted(ix.h, n) == 40005
    v.close()
    dense = vdb.Index("ip", 4, host_vectors=np.zeros((4, 4), np.float32))
    assert L.eps_index_build_sparse_inverted(dense.h, 0) == 40005
    assert L.eps_index_sparse_inverted_info(dense.h, None, None, None) == 40005
    dense.close()
    assert ix.inverted_info() == info
    same(ix.search(qs, 10), before, "after the refusals")
    ix.close()
