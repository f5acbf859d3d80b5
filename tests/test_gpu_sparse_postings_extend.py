"""Extending a sparse index's posting lists over appended rows (eps_index_extend_sparse_postings) on the GPU.

The extension must leave, byte for byte, the lists a full build over the same rows makes (the inverted index of an IP or
cosine index, the L2 screen of an L2 index): after every step of a chain of extensions the lists read back with
eps_index_get_sparse_postings equal a fresh build's on a second index with the same rows and the numpy model
(sparse_postings_model.postings_model).  Searches and graph builds then give what the freshly built index gives, and
what an index without lists gives: ids, bitwise distances, counts and the n_dist / n_seed / n_expand / n_edges
counters, and for L2 the same count of re-scored pairs as the freshly built screen."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sparse_l2_bound_model import to_csr  # noqa: E402
from sparse_postings_model import postings_model, same_postings  # noqa: E402
from test_gpu_sparse import assert_bitwise, attr_lt, csr_slice, sparse_rows  # noqa: E402

pytestmark = pytest.mark.gpu

VOCAB = 3000
N0, N = 12_000, 20_000
# indices no covered row holds: below the smallest covered index (0 included), between two covered ones, above the
# largest (VOCAB - 1 included)
NEW_ONLY = np.r_[0:10, 1000:1010, 2990:VOCAB]
EMPTY_RUN = (N0 + 1, N0 + 41)   # rows appended as a run of empty rows only
CHAIN = [N0 + 1, N0 + 1, EMPTY_RUN[1], N0 + 2000, N0 + 6000, N - 2000]   # a 1-row append, a no-op, the empty run, ...


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200
    assert vectordb_b200.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    return vectordb_b200


def table(seed):
    """N rows: the first N0 hold no index of NEW_ONLY; the rest are drawn over the whole vocabulary, with rows holding
    only NEW_ONLY indices (0 and VOCAB - 1 among them) and a run of empty rows.  Empty and duplicate rows throughout."""
    base = sparse_rows(N, VOCAB, seed, max_nnz=40)
    rng = np.random.default_rng(seed + 1)
    rows = []
    for r in range(N):
        idx, val = base[1][base[0][r]:base[0][r + 1]], base[2][base[0][r]:base[0][r + 1]]
        if r < N0:
            keep = ~np.isin(idx, NEW_ONLY)
            idx, val = idx[keep], val[keep]
        elif EMPTY_RUN[0] <= r < EMPTY_RUN[1]:
            idx, val = idx[:0], val[:0]
        elif r == N0 or r % 31 == 3:   # only indices no covered row holds
            idx = np.unique(np.r_[rng.choice(NEW_ONLY, 4, replace=False), 0, VOCAB - 1][: 2 + r % 5])
            val = (rng.random(idx.size, dtype=np.float32) + np.float32(0.25)).astype(np.float32)
        rows.append((idx, val))
    return to_csr(rows)


def queries(seed):
    qs = sparse_rows(24, VOCAB, seed, max_nnz=40, empty_every=0, dup_every=0)
    rows = [(qs[1][qs[0][q]:qs[0][q + 1]], qs[2][qs[0][q]:qs[0][q + 1]]) for q in range(24)]
    rows += [(np.array([0, 1003, VOCAB - 1]), np.float32([1.0, 0.5, 2.0])), (np.array([5, 2995]), np.float32([1.5, 1.0])),
             (np.zeros(0, np.int64), np.zeros(0, np.float32))]
    return to_csr(rows)


def build_lists(ix, metric, n=None):
    (ix.build_l2_screen if metric == "l2" else ix.build_inverted)(n)


def searched(ix, metric, qs, limit, **kw):
    """ix.search, and for L2 the pairs the search re-scored."""
    r0 = ix.l2_screen_info()["rescored"] if metric == "l2" else 0
    out = ix.search(qs, limit, **kw)
    return out, (ix.l2_screen_info()["rescored"] - r0 if metric == "l2" else 0)


STATS = ("n_dist", "n_seed", "n_expand", "n_edges")


def same_results(got, want, what):
    assert_bitwise(got, want[:3], what)
    for s in STATS:
        assert got[3][s] == want[3][s], "%s: %s %d != %d" % (what, s, got[3][s], want[3][s])


def check_searches(indexes, metric, qs, what, cases):
    """ext (extended), ref (built over the same rows) and plain (no lists) answer every case alike."""
    ext, ref, plain = indexes
    for cfg, limit, nodes in cases:
        for ix in indexes:
            ix.config(**cfg)
        w = "%s, %s, limit %d%s" % (what, cfg, limit, ", filtered" if nodes is not None else "")
        g, g_r = searched(ext, metric, qs, limit, filter_nodes=nodes)
        f, f_r = searched(ref, metric, qs, limit, filter_nodes=nodes)
        p, _ = searched(plain, metric, qs, limit, filter_nodes=nodes)
        same_results(g, f, w + ": extended vs built")
        same_results(g, p, w + ": extended vs no lists")
        assert g_r == f_r, "%s: re-scored %d != %d" % (w, g_r, f_r)


SCAN_CASES = [(dict(L_master=500), 10, None), (dict(L_master=500, force_brute=True), 50, None),
              (dict(L_master=500, prefilter=True), 10, attr_lt(40)), (dict(L_master=500, force_brute=True), 10, attr_lt(60))]


@pytest.mark.parametrize("metric", ["ip", "cosine", "l2"])
def test_extension_chain_equals_the_build(vdb, metric):
    rows = table({"ip": 11, "cosine": 12, "l2": 13}[metric])
    qs = queries(21)
    ext, ref, plain = (vdb.SparseIndex(metric, VOCAB) for _ in range(3))
    for ix in (ext, ref, plain):
        ix.append(csr_slice(rows, 0, N0))
    build_lists(ext, metric, N0)
    build_lists(ref, metric, N0)
    same_postings(ext.postings(), postings_model(rows, N0), "built over %d rows" % N0)
    r_ext = ext.l2_screen_info()["rescored"] if metric == "l2" else 0
    # appended a piece at a time, the lists extended over every mirrored row
    for n in CHAIN:
        if n > ext.rows:
            for ix in (ext, ref, plain):
                ix.append(csr_slice(rows, ix.rows, n), first_row=ix.rows)
        ext.extend_postings()
        build_lists(ref, metric, n)
        got = ext.postings()
        same_postings(got, postings_model(rows, n), "extended to %d rows: model" % n)
        same_postings(got, ref.postings(), "extended to %d rows: build" % n)
        assert ext.inverted_info() == ref.inverted_info() == dict(rows=n, terms=got["terms"].size,
                                                                  postings=got["post_rows"].size)
    if metric == "l2":
        assert ext.l2_screen_info()["rescored"] == r_ext   # extending re-scores nothing
    # a tail of 2000 appended rows: scanned by every index alike
    for ix in (ext, ref, plain):
        ix.append(csr_slice(rows, ix.rows, N), first_row=ix.rows)
        ix.set_attrs((np.arange(N) * 7 % 100).astype(np.int32).view(np.uint8), 4, N)
    check_searches((ext, ref, plain), metric, qs, "covered %d of %d rows" % (CHAIN[-1], N), SCAN_CASES)
    # deleted rows, then the lists over every row
    dead = np.arange(3, N, 37)
    deleted = np.zeros((N + 7) // 8, np.uint8)
    np.bitwise_or.at(deleted, dead >> 3, (1 << (dead & 7)).astype(np.uint8))
    for ix in (ext, ref, plain):
        ix.set_deleted(deleted)
    ext.extend_postings(N)
    build_lists(ref, metric, N)
    same_postings(ext.postings(), ref.postings(), "extended over every row, some deleted")
    same_postings(ext.postings(), postings_model(rows, N), "extended over every row: model")
    check_searches((ext, ref, plain), metric, qs, "covered every row, deleted rows", SCAN_CASES)
    # a view created after the extension shares the lists
    v = ext.view()
    same_postings(v.postings(), ref.postings(), "view")
    for limit in (10, 100):
        same_results(v.search(qs, limit), ref.search(qs, limit), "view, limit %d" % limit)
    v.close()
    # graph build after the extension, then graph mode with a tail of 3000 rows
    n_graph = N - 3000
    graphs = []
    for ix in (ext, ref, plain):
        ix.set_deleted(np.zeros(0, np.uint8))
        ix.build(n_graph, out_degree=24)
        graphs.append(ix.get_graph())
        ix.set_search_mode("graph")
    for other, name in ((graphs[1], "built"), (graphs[2], "no lists")):
        for part, a, b in zip(("n_indexed", "offsets", "neighbours", "nav"), graphs[0], other):
            assert np.array_equal(a, b), "graph build after the extension vs %s: %s differ" % (name, part)
    for ix in (ext, ref, plain):
        ix.set_deleted(deleted)
    check_searches((ext, ref, plain), metric, qs, "graph mode, %d rows indexed of %d" % (n_graph, N),
                   [(dict(L_master=100), 10, None), (dict(L_master=500), 50, None), (dict(L_master=100), 10, attr_lt(30)),
                    (dict(L_master=100, force_brute=True), 10, None),
                    (dict(L_master=100, prefilter=True), 10, attr_lt(30))])
    for ix in (ext, ref, plain):
        ix.close()


def test_refusals_leave_the_lists(vdb):
    rows = table(31)
    n1 = N0 + 500
    ix = vdb.SparseIndex("ip", VOCAB)
    ix.append(csr_slice(rows, 0, n1))
    L = ix.L
    assert L.eps_index_extend_sparse_postings(ix.h, n1) == 40005   # no lists yet
    assert ix.postings()["rows"] == 0 and ix.postings()["terms"].size == 0 and ix.postings()["ptr"].tolist() == [0]
    ix.build_inverted(N0)
    before = ix.postings()
    for n_bad in (-1, 0, N0 - 1, n1 + 1):   # below the covered rows, above the mirrored rows
        assert L.eps_index_extend_sparse_postings(ix.h, n_bad) == 40005, n_bad
        same_postings(ix.postings(), before, "after refusing n = %d" % n_bad)
    assert L.eps_index_extend_sparse_postings(ix.h, N0) == 0   # n == covered rows: nothing to do
    same_postings(ix.postings(), before, "after the no-op")
    v = ix.view()
    assert L.eps_index_extend_sparse_postings(v.h, n1) == 40005   # a view
    assert L.eps_index_extend_sparse_postings(ix.h, n1) == 40005  # an index with live views
    same_postings(v.postings(), before, "the view's lists")
    v.close()
    same_postings(ix.postings(), before, "after the view refusals")
    dense = vdb.Index("l2", 4, host_vectors=np.zeros((4, 4), np.float32))
    assert L.eps_index_extend_sparse_postings(dense.h, 0) == 40005
    assert L.eps_index_get_sparse_postings(dense.h, None, None, None, None, None, None, None) == 40005
    dense.close()
    ix.extend_postings()
    same_postings(ix.postings(), postings_model(rows, n1), "extended once the refusals are over")
    ix.build_inverted(0)   # dropped: nothing to extend
    assert L.eps_index_extend_sparse_postings(ix.h, n1) == 40005
    assert ix.inverted_info() == dict(rows=0, terms=0, postings=0)
    ix.close()
