"""L2 screen of sparse L2 fields on the GPU (eps_index_build_sparse_l2_screen).

The screen changes no result: with posting lists built on an L2 index, every exact scan bounds the covered rows,
re-scores the ones that can still be among the k best, and must give the ids, counts, n_dist (and n_seed / n_expand /
n_edges in graph mode) of the same index without the screen, with distances bitwise equal; where the table is small
enough they are also checked against the numpy restatement of vector.cpp (test_gpu_sparse.ref_distances /
ref_search) and against the reference's own answers (tests/golden/sparse.npz)."""
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sparse_l2_bound_model import adversarial, to_csr  # noqa: E402
from test_gpu_sparse import (L2, NT_NE, NT_STRING_ATTR, NT_STRING_CONST, assert_bitwise, attr_lt,  # noqa: E402
                             csr_slice, densify, distance_lt, ref_distances, ref_search, sparse_rows)

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


def with_negatives(csr, seed):
    """Values in [-1.5, 1.5): sparse_rows draws [-0.5, 1.5)."""
    rng = np.random.default_rng(seed)
    flip = rng.random(csr[2].size) < 0.3
    return csr[0], csr[1], np.where(flip, -csr[2], csr[2]).astype(np.float32)


def same(a, b, what, stats=("n_dist",)):
    """a (with the screen) == b (without): ids, counts, bitwise distances and the named counters."""
    assert_bitwise(a, b[:3], what)
    for s in stats:
        assert a[3][s] == b[3][s], "%s: %s %d != %d" % (what, s, a[3][s], b[3][s])


def make_pair(vdb, vocab, rows, n_attr=None):
    """The same L2 table twice: one index with the screen over every row, one without."""
    out = []
    for screened in (True, False):
        ix = vdb.SparseIndex("l2", vocab)
        ix.append(rows)
        if n_attr is not None:
            attr, codes = n_attr
            ix.set_attrs(attr.view(np.uint8), 4, attr.size)
            ix.set_string_codes(0, 0, codes)
        if screened:
            ix.build_l2_screen()
        out.append(ix)
    return out


def test_l2_screen_matches_model_and_scan(vdb):
    n, vocab = 5000, 2000
    rows = with_negatives(sparse_rows(n, vocab, 61), 60)   # empty rows, duplicate rows, negative values
    qs = with_empty_query(sparse_rows(32, vocab, 62, max_nnz=40, empty_every=0, dup_every=0))   # 33 queries
    nq = qs[0].size - 1
    D = ref_distances(densify(rows, vocab), densify(qs, vocab), L2)
    attr = (np.arange(n) * 7 % 100).astype(np.int32)
    codes = (np.arange(n) % 5).astype(np.int32)
    scr, plain = make_pair(vdb, vocab, rows, (attr, codes))
    assert scr.l2_screen_info() == dict(rows=n, rescored=0)
    info = scr.inverted_info()   # the same posting lists
    assert info["rows"] == n and info["postings"] == rows[0][-1] and info["terms"] == np.unique(rows[1]).size
    assert plain.l2_screen_info() == dict(rows=0, rescored=0)

    def both(what, want, limit, **kw):
        got = scr.search(qs, limit, **kw)
        assert_bitwise(got, want, what)
        same(got, plain.search(qs, limit, **kw), what)
        return got

    for ix in (scr, plain):
        ix.config(500, 500, force_brute=True)
    for k in (1, 10, 500):
        r0 = scr.l2_screen_info()["rescored"]
        got = both("force_brute k=%d" % k, ref_search(D, k, k), k)
        assert got[3]["n_dist"] == nq * n
        rescored = scr.l2_screen_info()["rescored"] - r0
        if k == 10:   # the screen screens: a few times k of the 5000 rows per query
            frac = rescored / (nq * n)
            print("force_brute k=10: re-scored %d of %d pairs (%.4f)" % (rescored, nq * n, frac))
            assert 0 < frac <= 0.05
    assert plain.l2_screen_info()["rescored"] == 0
    one = csr_slice(qs, 3, 4)
    g1 = scr.search(one, 10)
    assert_bitwise(g1, ref_search(D[3:4], 10, 10), "nq = 1")
    same(g1, plain.search(one, 10), "nq = 1")
    for ix in (scr, plain):
        ix.config(500, 7)   # brute-force branch of an un-indexed table: min(limit, L_local)
    both("L_local cap", ref_search(D, 10, 7), 10)
    dead = np.arange(3, n, 41)
    deleted = np.zeros((n + 7) // 8, np.uint8)
    np.bitwise_or.at(deleted, dead >> 3, (1 << (dead & 7)).astype(np.uint8))
    alive = np.ones(n, bool)
    alive[dead] = False
    for ix in (scr, plain):
        ix.config(500, 500, force_brute=True)
        ix.set_deleted(deleted)
    both("deleted", ref_search(D, 10, 10, keep=alive), 10)
    both("numeric filter", ref_search(D, 10, 10, keep=alive & (attr < 30)), 10, filter_nodes=attr_lt(30))
    both("string filter", ref_search(D, 10, 10, keep=alive & (codes != 3)), 10, filter_nodes=STRING_NE3)
    thr = float(np.nanmedian(D))
    r0 = scr.l2_screen_info()["rescored"]
    both("@distance filter", ref_search(D, 10, 10, keep=alive, dyn=lambda d: d < thr), 10, filter_nodes=distance_lt(thr))
    assert scr.l2_screen_info()["rescored"] == r0   # the merge tile for every row: nothing re-scored
    for ix in (scr, plain):
        ix.config(500, 500, prefilter=True)
    both("prefilter", ref_search(D, 50, 50, keep=alive & (attr < 10)), 50, filter_nodes=attr_lt(10))
    scr.close()
    plain.close()


def test_l2_screen_several_row_chunks(vdb):
    """4096 queries over 100 000 rows: the exact scan cuts the rows into chunks of 65 536, and with the screen over the
    first 70 000 rows the second chunk is partly bounded and partly merged."""
    n, vocab, nq = 100_000, 3000, 4096
    rows = sparse_rows(n, vocab, 71, max_nnz=40)
    qs = sparse_rows(nq, vocab, 72, max_nnz=20, empty_every=0, dup_every=0)
    ix = vdb.SparseIndex("l2", vocab)
    ix.append(rows)
    ix.config(500, 500, force_brute=True)
    want = ix.search(qs, 10)
    for n_scr in (70_000, n):
        ix.build_l2_screen(n_scr)
        assert ix.l2_screen_info()["rows"] == n_scr
        r0 = ix.l2_screen_info()["rescored"]
        same(ix.search(qs, 10), want, "4096 queries, screen over %d rows" % n_scr)
        print("screen over %d rows: re-scored %.5f of the covered pairs"
              % (n_scr, (ix.l2_screen_info()["rescored"] - r0) / (nq * n_scr)))
    ix.close()


def test_l2_screen_reference_golden(vdb):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_sparse_golden import CASES, THR, crc, table
    from sparse_golden_check import GOLDEN, check_against_golden
    g = np.load(GOLDEN)
    n, vocab, rows, qs, attr, codes, dead = table(L2)
    assert crc(*rows, *qs) == int(g["m%d_table_crc32" % L2])
    ix = vdb.SparseIndex(L2, vocab)
    ix.append(rows)
    ix.set_attrs(attr.view(np.uint8), 4, n)
    ix.set_string_codes(0, 0, codes)
    ix.build_l2_screen()
    assert ix.l2_screen_info()["rows"] == n
    deleted = np.zeros((n + 7) // 8, np.uint8)
    np.bitwise_or.at(deleted, dead >> 3, (1 << (dead & 7)).astype(np.uint8))
    for name, pre, ll, limit, _, use_del in CASES:
        ix.config(500, ll, prefilter=pre)
        ix.set_deleted(deleted if use_del else np.zeros(0, np.uint8))
        nodes = {"numeric": attr_lt(30), "prefilter": attr_lt(10), "distance": distance_lt(THR[L2]),
                 "string": STRING_NE3}.get(name)
        ids, ds, cnt, _ = ix.search(qs, limit, filter_nodes=nodes)
        check_against_golden(g, "m%d_%s" % (L2, name), ids, ds, cnt, L2)
    ix.close()


def test_l2_screen_partial_coverage_appends_rebuild_and_drop(vdb):
    n0, n1, n, vocab = 3000, 4500, 7000, 2000
    rows = with_negatives(sparse_rows(n, vocab, 81), 80)
    qs = with_empty_query(sparse_rows(16, vocab, 82, max_nnz=40, empty_every=0, dup_every=0))
    D = ref_distances(densify(rows, vocab), densify(qs, vocab), L2)
    ix = vdb.SparseIndex("l2", vocab)
    ix.append(csr_slice(rows, 0, n1))
    ix.config(500, 500, force_brute=True)
    ix.build_l2_screen(n0)
    assert ix.l2_screen_info()["rows"] == n0
    assert ix.inverted_info() == dict(rows=n0, terms=np.unique(rows[1][:rows[0][n0]]).size, postings=int(rows[0][n0]))
    assert_bitwise(ix.search(qs, 20), ref_search(D[:, :n1], 20, 20), "screen over %d of %d rows" % (n0, n1))
    ix.append(csr_slice(rows, n1, n), first_row=n1)
    assert ix.l2_screen_info()["rows"] == n0   # appended rows are merged until the next build
    got = ix.search(qs, 20)
    assert_bitwise(got, ref_search(D, 20, 20), "after the append")
    assert got[3]["n_dist"] == (qs[0].size - 1) * n
    ix.build_l2_screen()
    assert ix.l2_screen_info()["rows"] == n
    assert_bitwise(ix.search(qs, 20), ref_search(D, 20, 20), "rebuilt over every row")
    ix.build_l2_screen(0)
    assert ix.l2_screen_info()["rows"] == 0 and ix.inverted_info() == dict(rows=0, terms=0, postings=0)
    r0 = ix.l2_screen_info()["rescored"]
    assert_bitwise(ix.search(qs, 20), ref_search(D, 20, 20), "dropped")
    assert ix.l2_screen_info()["rescored"] == r0
    ix.close()


def test_l2_screen_graph_mode(vdb):
    """Graph mode with a tail: the graph search takes the raw queries and the tail scan is screened; ids, distances,
    counts, n_dist, n_seed, n_expand and n_edges are those without the screen.  The brute-force branches too."""
    n_graph, n, vocab = 5000, 6000, 2000
    rows = sparse_rows(n, vocab, 91)
    qs = sparse_rows(16, vocab, 92, max_nnz=40, empty_every=0, dup_every=0)
    ix = vdb.SparseIndex("l2", vocab)
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
    for n_scr in (n, n_graph + 300, 2000):   # covering the tail, part of it, or part of the graph's rows only
        ix.build_l2_screen(n_scr)
        for (cfg, limit, nodes), w in zip(cases, want):
            ix.config(**cfg)
            same(ix.search(qs, limit, filter_nodes=nodes), w, "graph mode %s, screen over %d rows" % (cfg, n_scr),
                 stats=("n_dist", "n_seed", "n_expand", "n_edges"))
    ix.close()


def test_l2_screen_view_beside_its_base(vdb):
    n, vocab = 8000, 2000
    rows = sparse_rows(n, vocab, 111)
    qs = sparse_rows(64, vocab, 112, max_nnz=40, empty_every=0, dup_every=0)
    ix = vdb.SparseIndex("l2", vocab)
    ix.append(rows)
    ix.config(500, 500, force_brute=True)
    plain = ix.search(qs, 10)
    ix.build_l2_screen()
    r_base = ix.l2_screen_info()["rescored"]
    v = ix.view()
    assert v.l2_screen_info() == dict(rows=n, rescored=0)   # the lists are shared, the count is the handle's
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
    assert v.l2_screen_info()["rescored"] > 0 and ix.l2_screen_info()["rescored"] > r_base
    for call in (lambda: v.build_l2_screen(), lambda: v.build_l2_screen(0), lambda: ix.build_l2_screen(),
                 lambda: ix.build_l2_screen(0)):
        with pytest.raises(vdb.EpsError) as e:
            call()
        assert e.value.code == 40005
    assert ix.l2_screen_info()["rows"] == n and v.l2_screen_info()["rows"] == n
    v.close()
    ix.build_l2_screen(0)   # no live views any more
    assert ix.l2_screen_info()["rows"] == 0
    ix.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_l2_screen_adversarial_rows_and_queries(vdb, seed):
    """Values near 1e19 whose squares overflow, near 1e-23 whose products underflow, NaN and +-inf, rows equal to a
    query or a query plus 1 ulp, 30 % empty rows: against the model and the plain scan, k = 10 and 500."""
    rows, qs, vocab = adversarial(seed, n_plain=700)
    n = rows[0].size - 1
    with np.errstate(all="ignore"):
        D = ref_distances(densify(rows, vocab), densify(qs, vocab), L2)
    scr, plain = make_pair(vdb, vocab, rows)
    for ix in (scr, plain):
        ix.config(500, 500, force_brute=True)
    for k in (10, 500):
        got = scr.search(qs, k)
        assert_bitwise(got, ref_search(D, k, k), "adversarial seed %d, k=%d: model" % (seed, k))
        same(got, plain.search(qs, k), "adversarial seed %d, k=%d: scan" % (seed, k))
    assert n > 500
    scr.close()
    plain.close()


@pytest.mark.parametrize("k", [10, 500])
def test_l2_screen_empty_rows_tie(vdb, k):
    """30 % empty rows: with queries of small norm every empty row ties at |q|^2 at the head of the list."""
    n, vocab = 3000, 1500
    base = sparse_rows(n, vocab, 131, empty_every=0, dup_every=0)
    rng = np.random.default_rng(132)
    empty = rng.random(n) < 0.3
    rows = to_csr([(np.zeros(0, np.int64), np.zeros(0, np.float32)) if empty[r] else
                   (base[1][base[0][r]:base[0][r + 1]], base[2][base[0][r]:base[0][r + 1]]) for r in range(n)])
    qs = sparse_rows(12, vocab, 133, max_nnz=30, empty_every=0, dup_every=0)
    qs = (qs[0], qs[1], (qs[2] * np.float32(0.05)).astype(np.float32))
    D = ref_distances(densify(rows, vocab), densify(qs, vocab), L2)
    scr, plain = make_pair(vdb, vocab, rows)
    for ix in (scr, plain):
        ix.config(500, 500, force_brute=True)
    got = scr.search(qs, k)
    assert_bitwise(got, ref_search(D, k, k), "empty-row ties, k=%d: model" % k)
    same(got, plain.search(qs, k), "empty-row ties, k=%d: scan" % k)
    assert np.isin(got[0][:, :min(k, int(empty.sum()))], np.nonzero(empty)[0]).all()
    scr.close()
    plain.close()


def test_l2_screen_refusals_change_nothing(vdb):
    n, vocab = 4000, 2000
    rows = sparse_rows(n, vocab, 121)
    qs = sparse_rows(16, vocab, 122, max_nnz=40, empty_every=0, dup_every=0)
    for metric in ("ip", "cosine"):
        ix = vdb.SparseIndex(metric, vocab)
        ix.append(rows)
        ix.config(500, 500, force_brute=True)
        ix.build_inverted(2000)
        info, before = ix.inverted_info(), ix.search(qs, 10)
        with pytest.raises(vdb.EpsError) as e:
            ix.build_l2_screen()
        assert e.value.code == 40005 and "eps_index_build_sparse_inverted" in str(e.value)
        assert ix.inverted_info() == info and ix.l2_screen_info() == dict(rows=0, rescored=0)
        same(ix.search(qs, 10), before, "%s after the refusal" % metric)
        ix.close()

    ix = vdb.SparseIndex("l2", vocab)
    ix.append(rows)
    ix.config(500, 500, force_brute=True)
    ix.build_l2_screen(3000)
    before = ix.search(qs, 10)
    info, inv = ix.l2_screen_info(), ix.inverted_info()
    L = ix.L
    for n_bad in (-1, n + 1):
        assert L.eps_index_build_sparse_l2_screen(ix.h, n_bad) == 40005
    v = ix.view()
    assert L.eps_index_build_sparse_l2_screen(v.h, n) == 40005
    assert L.eps_index_build_sparse_l2_screen(ix.h, n) == 40005
    v.close()
    dense = vdb.Index("l2", 4, host_vectors=np.zeros((4, 4), np.float32))
    assert L.eps_index_build_sparse_l2_screen(dense.h, 0) == 40005
    assert L.eps_index_sparse_l2_screen_info(dense.h, None, None) == 40005
    dense.close()
    assert ix.l2_screen_info() == info and ix.inverted_info() == inv
    same(ix.search(qs, 10), before, "after the refusals")
    ix.close()
