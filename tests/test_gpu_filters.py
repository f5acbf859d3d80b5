"""The device expression evaluator (filter.cuh prog_run, lowered by capi.cu) held to the reference's own answers and to
tests/expr_model.py at every kernel that calls it (run with -m gpu on an H100).

Direct evaluation: a facet batch of one-row result lists (one list per row and distance, `dists` set per list) exposes
single evaluations, bit for bit against tests/golden/exprs.npz: a BOOL key of a filter program is
LogicalEvaluate(root, row, d), a DOUBLE key and the MIN and MAX of a value expression are NumEvaluate(root, row, d).
The golden facet cases go through eps_facet_batch as they are.

Call sites: golden programs as search filters over integer-valued tables (graph_model.int_table; exact fp32
distances in any summation order) whose attribute rows are golden rows, so that each answer is exactly the model's
passing rows in (distance, id) order: the exact scan's row kernel, its fp32 path and each coarse mode, prefilter, the
graph branch with and without appended tail rows, deleted rows, a sparse index in scan and graph mode, and a view."""
import ctypes as C

import numpy as np
import pytest

import expr_model as em
import graph_model as gm
from test_gpu_graph_exact import Table, check

pytestmark = pytest.mark.gpu

BAD_ARG, UNSUPPORTED = 40005, 40006
ONE = np.array([[em.INT_CONST, em.VT_INT, -1, -1, 1, 0, 0, -1]], np.int64)   # the inner expression of COUNT(*)


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200
    assert vectordb_b200.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    return vectordb_b200


@pytest.fixture(scope="module")
def g():
    return em.Golden()


def mirror(ix, g, raw, codes):
    """Attribute rows `raw` [n x stride'], string codes [2 x n] and the golden dictionary on index ix."""
    ix.append_string_dictionary(0, g.words)
    ix.set_attrs(raw.ravel(), raw.shape[1], raw.shape[0])
    for c in range(codes.shape[0]):
        ix.set_string_codes(c, 0, codes[c])


def facet_one_row(ix, rows, dists, key_nodes, key_type, aggs):
    """eps_facet_batch over one-row lists: returns the key and the aggregate values of each list."""
    from vectordb_b200.index import filter_nodes_array
    from vectordb_b200.lib import FacetSpec, check as eps_check
    nl = rows.size
    ids = np.ascontiguousarray(rows, np.int64).reshape(nl, 1)
    d = np.ascontiguousarray(dists, np.float64).reshape(nl, 1)
    counts = np.ones(nl, np.int64)
    spec, keep = FacetSpec(), []
    karr, kn = filter_nodes_array(key_nodes)
    keep.append(karr)
    spec.key_nodes, spec.n_key_nodes, spec.key_type, spec.n_aggs = C.cast(karr, C.c_void_p), kn, key_type, len(aggs)
    for i, (t, nodes) in enumerate(aggs):
        arr, n = filter_nodes_array(nodes)
        keep.append(arr)
        spec.agg_nodes[i], spec.n_agg_nodes[i], spec.agg_types[i] = C.cast(arr, C.c_void_p), n, t
    ok = np.empty(nl, np.float64)
    ov = np.empty((nl, len(aggs)), np.float64)
    og = np.empty(nl, np.int64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    eps_check(ix.L.eps_facet_batch(ix.h, p(ids), p(d), p(counts), nl, 1, C.byref(spec), p(ok), p(ov), p(og)))
    assert (og == 1).all()
    return ok, ov


@pytest.fixture(scope="module")
def golden_ix(vdb, g):
    ix = vdb.Index("l2", 2, host_vectors=np.zeros((g.n, 2), np.float32))
    ix.sync_rows(g.n)
    mirror(ix, g, g.table.raw, g.str_codes)
    yield ix
    ix.close()


def test_filter_programs_bit_for_bit(vdb, g, golden_ix):
    D = g.filter_dists.size
    rows, dists = np.tile(np.arange(g.n), D), np.repeat(g.filter_dists, g.n)
    bad = []
    for i, nodes in enumerate(g.filters):
        key, _ = facet_one_row(golden_ix, rows, dists, nodes, em.VT_BOOL, [(em.COUNT, ONE)])
        if not np.array_equal(key.reshape(D, g.n) != 0, g.filter_bits[i]):
            bad.append(i)
    assert not bad, "%d of %d programs differ, first %r" % (len(bad), len(g.filters), g.filter_text[bad[0]])


def same_doubles(a, b):
    return (np.isnan(a) & np.isnan(b)) | (a.view(np.int64) == b.view(np.int64))


def test_value_expressions_bit_for_bit(vdb, g, golden_ix):
    D = g.value_dists.size
    rows, dists = np.tile(np.arange(g.n), D), np.repeat(g.value_dists, g.n)
    for i, nodes in enumerate(g.values):
        # the DOUBLE key, and MIN / MAX under a constant key (a NaN key is a group of its own that aggregates nothing:
        # the reference cannot group by NaN at all)
        key, _ = facet_one_row(golden_ix, rows, dists, nodes, em.VT_DOUBLE, [(em.COUNT, ONE)])
        _, vals = facet_one_row(golden_ix, rows, dists, ONE, em.VT_INT, [(em.MIN, nodes), (em.MAX, nodes)])
        want = g.value_num[i].ravel()
        for what, got in (("key", key), ("MIN", vals[:, 0]), ("MAX", vals[:, 1])):
            ok = same_doubles(got, want)
            assert ok.all(), "%r %s: %d differ, first row %d d=%r: %r vs %r" % (
                g.value_text[i], what, (~ok).sum(), np.flatnonzero(~ok)[0] % g.n, dists[~ok][0], got[~ok][0], want[~ok][0])


def test_golden_facets(vdb, g, golden_ix):
    """The reference's FacetExecutor answers: INT keys that are NaN, +-inf or beyond 2^63, BOOL keys that read
    "@distance", STRING keys, DOUBLE keys with -0.0 and 0.0, every aggregate type."""
    bad = []
    for case in g.facets:
        ids = case["ids"][None, :]
        aggs = list(zip(case["agg_types"], case["agg_nodes"]))
        got = golden_ix.facet(ids, [ids.shape[1]], case["key_nodes"], case["key_type"], aggs, dists=case["dists"][None, :])
        msg = em.facet_mismatch(case, got[0], g.words)
        if msg:
            bad.append("%s; device groups %s" % (msg, [(k, v[0]) for k, v in got[0]][:8]))
    assert not bad, "\n".join(bad)


# ---- call sites --------------------------------------------------------------------------------------------------
def pick_programs(g, reads_distance, count, seed, signed_zero=True):
    """`count` golden programs that read "@distance" (or not), the hand-written ones first.  signed_zero=False leaves
    out those that divide, where the sign of a zero distance (an inner product of 0 is -0.0) would decide."""
    uses = [bool(np.any(n[:, 7] == -2)) for n in g.filters]
    idx = [i for i in range(len(g.filters)) if uses[i] == reads_distance and
           (signed_zero or not np.any(g.filters[i][:, 0] == em.DIV))]
    head = [i for i in idx if i < 80]
    rest = np.random.default_rng(seed).permutation([i for i in idx if i >= 80])
    return (head[:count // 2] + list(rest))[:count]


def big_rows(g, n, seed):
    """Attribute rows and string codes of an n-row table: golden rows in a seeded order."""
    pick = np.random.default_rng(seed).integers(0, g.n, n)
    pick[:g.n] = np.arange(g.n)
    return g.table.raw[pick], g.str_codes[:, pick]


def keep_fn(g, raw, codes, nodes, prefilter=False):
    t = em.Table(raw.ravel(), raw.shape[1], raw.shape[0], codes, g.words)
    return lambda ids, ds: em.filter_rows(nodes, t.rows(ids), 0.0 if prefilter else ds.astype(np.float64))


def check_brute(g, ix, X, Q, raw, codes, progs, limit, what, prefilter=False, deleted=None):
    ix.config(limit, limit, prefilter=prefilter, force_brute=True)
    no_graph = (0, np.zeros(1, np.int64), np.zeros(0, np.int64), 0)
    for p in progs:
        nodes = g.filters[p]
        ids, ds, cnt, _ = ix.search(Q, limit, filter_nodes=nodes)
        m = gm.search(X, Q, ix_metric(ix), no_graph, limit, limit, deleted=deleted,
                      keep=keep_fn(g, raw, codes, nodes, prefilter))
        bad = np.flatnonzero((cnt != m.counts) | np.any(ids != m.ids, axis=1))
        assert bad.size == 0, "%s %r: %d queries differ, first q%d count %d vs model %d" % (
            what, g.filter_text[p], bad.size, bad[0], cnt[bad[0]], m.counts[bad[0]])
        v = ids >= 0
        assert np.array_equal(ds[v], m.dists[v]), "%s %r: distances" % (what, g.filter_text[p])


def ix_metric(ix):
    return {1: "l2", 2: "cosine", 3: "ip"}[ix.metric]


@pytest.mark.parametrize("metric", ["l2", "ip"])
def test_exact_scan_row_kernel(vdb, g, metric):
    """nq <= 16: the row kernel, with limit = n so that every passing row is listed.  k = 2048 is also a select list
    whose 48 KB of shared memory leaves no room for the kernel's static shared memory under the launch default."""
    n, d = 2048, 8
    X, Q = gm.int_table(n, d, 41), gm.int_table(9, d, 42, B=1)
    raw, codes = big_rows(g, n, 43)
    ix = vdb.Index(metric, d, host_vectors=X)
    ix.sync_rows(n)
    mirror(ix, g, raw, codes)
    progs = pick_programs(g, True, 16, 1, signed_zero=metric == "l2") + pick_programs(g, False, 16, 2)
    check_brute(g, ix, X, Q, raw, codes, progs, n, "row kernel " + metric)
    ix.close()


@pytest.mark.parametrize("coarse", ["fp32", "tf32", "bf16"])
def test_exact_scan_batch(vdb, g, coarse):
    """nq = 64, n = 8192: the fp32 scan, or the coarse pass whose boot select and fused epilogue read the pass bitmap
    (filters that read the distance take the fp32 select in every mode)."""
    n, d, limit = 8192, 32, 64
    X, Q = gm.int_table(n, d, 51), gm.int_table(64, d, 52)
    gm.assert_exact(X, Q)
    raw, codes = big_rows(g, n, 53)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.set_coarse(coarse)
    mirror(ix, g, raw, codes)
    progs = pick_programs(g, False, 12, 3) + pick_programs(g, True, 4, 4)
    check_brute(g, ix, X, Q, raw, codes, progs, limit, "batch " + coarse)
    ix.close()


def test_prefilter_and_deleted_rows(vdb, g):
    """Prefilter mode, where "@distance" reads 0, and deleted rows under filters in both modes."""
    n, d = 3000, 8
    X, Q = gm.int_table(n, d, 61), gm.int_table(7, d, 62, B=1)
    raw, codes = big_rows(g, n, 63)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    mirror(ix, g, raw, codes)
    progs = pick_programs(g, True, 10, 5) + pick_programs(g, False, 6, 6)
    check_brute(g, ix, X, Q, raw, codes, progs, n, "prefilter", prefilter=True)
    deleted = np.random.default_rng(64).random(n) < 0.3
    ix.set_deleted(np.packbits(deleted, bitorder="little"))
    check_brute(g, ix, X, Q, raw, codes, progs, n, "deleted", deleted=deleted)
    check_brute(g, ix, X, Q, raw, codes, progs[:6], n, "deleted prefilter", prefilter=True, deleted=deleted)
    ix.close()


@pytest.mark.parametrize("tail", [0, 300])
def test_graph_branch(vdb, g, tail):
    """L_master = L_local = limit = n_indexed: the seed set covers every indexed row, so the post-filter walk after the
    merge judges them all; with a tail, the hybrid merge brings in appended rows."""
    n_indexed, d = 512, 8
    n = n_indexed + tail
    X, Q = gm.int_table(n, d, 71), gm.int_table(6, d, 72, B=1)
    off, nb = gm.random_csr(n_indexed, 4, 16, 73)
    raw, codes = big_rows(g, n, 74)
    t = Table(vdb, X, (n_indexed, off, nb, 5), metrics=("l2",))
    mirror(t.ix["l2"], g, raw, codes)
    deleted = np.zeros(n, bool)
    for p in pick_programs(g, True, 10, 7) + pick_programs(g, False, 10, 8):
        check(t, "l2", Q, n_indexed, n_indexed, keep=keep_fn(g, raw, codes, g.filters[p]), nodes=g.filters[p],
              what="graph tail=%d %r" % (tail, g.filter_text[p]))
    deleted[::7] = True
    t.ix["l2"].set_deleted(np.packbits(deleted, bitorder="little"))
    p = pick_programs(g, True, 1, 9)[0]
    check(t, "l2", Q, n_indexed, n_indexed, deleted=deleted, keep=keep_fn(g, raw, codes, g.filters[p]),
          nodes=g.filters[p], what="graph deleted tail=%d %r" % (tail, g.filter_text[p]))
    t.close()


@pytest.mark.parametrize("mode", ["scan", "graph"])
def test_sparse_index(vdb, g, mode):
    """A sparse index: each distance-free program answers as the same search with an int32 flag column that marks the
    model's passing rows; a program that reads the distance lists only rows the model passes at their distance."""
    from test_gpu_sparse import sparse_rows
    n, vocab = 2000, 1500
    rows = sparse_rows(n, vocab, 81)
    qs = sparse_rows(8, vocab, 82, max_nnz=30, empty_every=0, dup_every=0)
    raw, codes = big_rows(g, n, 83)
    ix = vdb.SparseIndex("ip", vocab)
    ix.append(rows)
    if mode == "graph":
        ix.build(n)
        ix.set_search_mode("graph")
    ix.config(200, 200)
    ix.append_string_dictionary(0, g.words)
    for c in range(codes.shape[0]):
        ix.set_string_codes(c, 0, codes[c])
    table = em.Table(raw.ravel(), raw.shape[1], n, codes, g.words)
    progs = pick_programs(g, False, 10, 10)
    masks = np.stack([em.filter_rows(g.filters[p], table, 0.0) for p in progs], axis=1).astype(np.int32)
    ix.set_attrs(np.concatenate([raw, masks.view(np.uint8)], axis=1).ravel(), raw.shape[1] + 4 * len(progs), n)
    for j, p in enumerate(progs):   # flag column j: int32 at the end of the golden row
        flag = np.array([[em.INT4, em.VT_INT, -1, -1, 0, 0, 0, raw.shape[1] + 4 * j],
                         [em.INT_CONST, em.VT_INT, -1, -1, 1, 0, 0, -1], [em.EQ, em.VT_BOOL, 0, 1, 0, 0, 0, -1]], np.int64)
        got = ix.search(qs, 10, filter_nodes=g.filters[p])[:3]
        want = ix.search(qs, 10, filter_nodes=flag)[:3]
        for a, b in zip(got, want):
            assert np.array_equal(a, b), "sparse %s %r" % (mode, g.filter_text[p])
    for p in pick_programs(g, True, 6, 11, signed_zero=False):
        ids, ds, cnt = ix.search(qs, 50, filter_nodes=g.filters[p])[:3]
        for q in range(ids.shape[0]):
            r = ids[q, :cnt[q]]
            ok = em.filter_rows(g.filters[p], table.rows(r), ds[q, :cnt[q]].astype(np.float32).astype(np.float64))
            assert ok.all(), "sparse %s %r lists a row the filter rejects" % (mode, g.filter_text[p])
    ix.close()


def test_view(vdb, g):
    n, d = 2000, 8
    X, Q = gm.int_table(n, d, 91), gm.int_table(5, d, 92, B=1)
    raw, codes = big_rows(g, n, 93)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    mirror(ix, g, raw, codes)
    ix.config(n, n, force_brute=True)
    v = ix.view()
    p = pick_programs(g, True, 1, 12)[0]
    check_brute(g, v, X, Q, raw, codes, [p], n, "view")
    a, b = ix.search(Q, n, filter_nodes=g.filters[p])[:3], v.search(Q, n, filter_nodes=g.filters[p])[:3]
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    v.close()
    ix.close()


def test_refusals(vdb, g):
    n = g.n
    ix = vdb.Index("l2", 2, host_vectors=np.zeros((n + 44, 2), np.float32))
    ix.sync_rows(n)
    mirror(ix, g, g.table.raw, g.str_codes)
    Q = np.zeros((1, 2), np.float32)

    def code_of(nodes):
        with pytest.raises(vdb.EpsError) as e:
            ix.search(Q, 5, filter_nodes=nodes)
        return e.value.code

    p64 = next(nodes for nodes in g.filters if len(nodes) == 64)
    ix.search(Q, 5, filter_nodes=p64)   # 64 nodes: accepted
    p65 = np.vstack([p64, [[em.NOT, em.VT_BOOL, 63, -1, 0, 0, 0, -1]]])
    assert code_of(p65) == UNSUPPORTED
    in_node = np.array([[em.STRING_CONST, 0, -1, -1, 1, 0, 0, -1], [em.STRING_ATTR, 0, -1, -1, 0, 0, 0, 0],
                        [em.IN, em.VT_BOOL, 0, 0, 0, 0, 0, -1]], np.int64)
    assert code_of(in_node) == UNSUPPORTED
    for t, width in ((em.INT8, 8), (em.INT4, 4), (em.DOUBLE_ATTR, 8), (em.BOOL_ATTR, 1)):
        past = np.array([[t, 1, -1, -1, 0, 0, 0, g.stride - width + 1], [em.INT_CONST, 1, -1, -1, 0, 0, 0, -1],
                         [em.EQ, em.VT_BOOL, 0, 1, 0, 0, 0, -1]], np.int64)
        if t == em.BOOL_ATTR:
            past = past[:1]
        assert code_of(past) == BAD_ARG, t
    ix.sync_rows(n + 44)   # 300 vector rows, 256 attribute rows
    assert code_of(g.filters[0]) == BAD_ARG
    ix.set_attrs(np.concatenate([g.table.raw, g.table.raw[:44]]).ravel(), g.stride, n + 44)
    ix.set_string_codes(0, n, g.str_codes[0, :44])
    ix.set_string_codes(1, n, g.str_codes[1, :44])
    ix.search(Q, 5, filter_nodes=g.filters[0])
    ix.close()
