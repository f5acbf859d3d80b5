"""LIKE filters on the device (run with -m gpu on an H100), held to tests/like_model.py.

The match kernel's bits are read back through exact scans of a 1-d table whose row r sits at r, so a query at -1 lists
the admissible rows of a window in row order.  The search paths are checked with tests/exact_ref.check_exact and
tests/graph_model.py on the model's admissible rows, and bitwise against the same search with an integer column that
marks those rows."""
import numpy as np
import pytest

import exact_ref as er
import graph_model as gm
import like_model as lm
from test_gpu_graph_exact import Table, check
from test_gpu_sparse import sparse_rows

pytestmark = pytest.mark.gpu

S_CONST, INT4_ATTR, S_ATTR, INT_CONST, ADD, LT, EQ, GTE, AND, OR, NOT, LIKE = 2, 7, 9, 1, 14, 19, 21, 23, 25, 26, 27, 29
BAD_ARG, UNSUPPORTED = 40005, 40006
WINDOW = 8192


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200
    assert vectordb_b200.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    return vectordb_b200


class Expr:
    """Filter nodes in the parser's order; every builder returns the index of the node it appended."""

    def __init__(self):
        self.rows = []

    def add(self, t, vt, left=-1, right=-1, iv=0, fo=-1):
        self.rows.append([t, vt, left, right, iv, 0, 0, fo])
        return len(self.rows) - 1

    def col(self, c):
        return self.add(S_ATTR, 0, fo=c)

    def lit(self, code):
        return self.add(S_CONST, 0, iv=code)

    def like(self, a, b):
        return self.add(LIKE, 3, a, b)

    def int_cmp(self, op, offset, value):
        return self.add(op, 3, self.add(INT4_ATTR, 1, fo=offset), self.add(INT_CONST, 1, iv=value))

    def both(self, a, b):
        return self.add(AND, 3, a, b)

    def nodes(self):
        return np.array(self.rows, np.int64)

    def copy(self):
        e = Expr()
        e.rows = [r[:] for r in self.rows]
        return e


def like_expr(lhs, rhs):
    """lhs / rhs: ("col", column) or ("lit", code)."""
    e = Expr()
    a = e.col(lhs[1]) if lhs[0] == "col" else e.lit(lhs[1])
    b = e.col(rhs[1]) if rhs[0] == "col" else e.lit(rhs[1])
    e.like(a, b)
    return e


ALPHABET = np.frombuffer(b"aab\n\r%_.*\\[($^|?+{\xc3\xa9\xff\0", np.uint8)
WEIGHTS = np.array([8, 0, 6, 1, 1, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1], float)


def rand_strings(rng, n, max_len=300):
    out = []
    p = WEIGHTS / WEIGHTS.sum()
    for _ in range(n):
        m = int(rng.integers(0, max_len + 1)) if rng.random() < 0.5 else int(rng.integers(0, 12))
        out.append(ALPHABET[rng.choice(ALPHABET.size, m, p=p)].tobytes())
    return out


def derive(rng, s):
    """A pattern that matches s unless a line terminator fell under a wildcard: bytes become '_' and spans '%'."""
    b = bytearray(s)
    for _ in range(int(rng.integers(0, 4))):
        if b:
            b[int(rng.integers(0, len(b)))] = ord("_")
    for _ in range(int(rng.integers(0, 3))):
        i = int(rng.integers(0, len(b) + 1))
        j = min(len(b), i + int(rng.integers(0, 10)))
        b[i:j] = b"%"
    return bytes(b)


class Dict:
    """The caller's side of the string dictionary, mirrored to every index given to add()."""

    def __init__(self):
        self.strings = []

    def add(self, strings, *indexes):
        first = len(self.strings)
        self.strings += list(strings)
        for ix in indexes:
            ix.append_string_dictionary(first, strings)
        return np.arange(first, len(self.strings), dtype=np.int32)


def line_table(vdb, n, capacity=None):
    """Row r of a 1-d table sits at r; attribute row: int32 r."""
    X = np.arange(capacity or n, dtype=np.float32)[:, None]
    ix = vdb.Index("l2", 1, host_vectors=X)
    ix.sync_rows(n)
    ix.config(WINDOW, WINDOW, force_brute=True)
    ix.set_attrs(np.arange(capacity or n, dtype=np.int32).view(np.uint8), 4, n)
    return ix


def admitted(ix, expr, n):
    """The rows of [0, n) the filter admits, read through exact scans over windows of row ids."""
    out = np.zeros(n, bool)
    root = len(expr.rows) - 1
    for lo in range(0, n, WINDOW):
        e = expr.copy()
        e.both(e.both(root, e.int_cmp(GTE, 0, lo)), e.int_cmp(LT, 0, lo + WINDOW))
        ids, ds, cnt, _ = ix.search(np.array([[-1.0]], np.float32), WINDOW, filter_nodes=e.nodes())
        got = ids[0, :cnt[0]]
        assert np.all(np.diff(got) > 0) and np.all((got >= lo) & (got < lo + WINDOW))
        out[got] = True
    return out


def assert_bits(got, subjects, patterns, what, sample=None, rng=None, must=()):
    """Device bits against the model on every row, or on `sample` random rows plus the rows `must`."""
    idx = np.arange(got.size)
    if sample is not None and sample < got.size:
        idx = np.union1d(rng.choice(got.size, sample, replace=False), np.asarray(must, np.int64))
    want = lm.like_many([subjects[i] for i in idx], [patterns[i] for i in idx])
    bad = idx[got[idx] != want]
    assert bad.size == 0, "%s: %d of %d differ, first row %d: %r LIKE %r -> device %s" % (
        what, bad.size, idx.size, bad[0], subjects[bad[0]][:60], patterns[bad[0]][:60], got[bad[0]])
    return want


def test_bits_match_the_model_in_every_shape(vdb):
    rng = np.random.default_rng(1)
    n, extra = 20000, 1000
    base = rand_strings(rng, n // 2 - 100)
    for i in range(100):  # subjects past 1000 bytes, half of them on one line
        t = np.frombuffer(b"aab%_.", np.uint8)[rng.integers(0, 6, int(rng.integers(1000, 1500)))].tobytes()
        base.append(t if i % 2 else t[:500] + b"\n" + t[500:])
    longs = np.arange(n // 2 - 100, n // 2)
    derived = [derive(rng, s) for s in base]
    dic = Dict()
    ix = line_table(vdb, n, capacity=n + extra)
    dic.add(base + derived, ix)
    D = dic.strings
    col_s = np.array([r % (n // 2) for r in range(n)], np.int32)
    col_p = np.where(np.arange(n) % 2 == 0, n // 2 + col_s, rng.integers(0, n, n)).astype(np.int32)
    ix.set_string_codes(0, 0, np.arange(n, dtype=np.int32))
    ix.set_string_codes(1, 0, col_s)
    ix.set_string_codes(2, 0, col_p)

    # attr LIKE 'const': one bit per code
    pats = [b"%a%", b"%\n%", b"a%", b"%_%_%", b"%b", b"_", b"", b"%", b"%%", b"%a_b%", b"%\\%", b"\xc3\xa9%", b"%\0%"]
    long_pats = [derive(rng, base[-1]), derive(rng, base[-3]), b"%" + b"_" * 1000 + b"%", b"%" + b"a%" * 350 + b"_" * 350]
    codes = dic.add(pats + long_pats, ix)
    for p, c in zip(pats + long_pats, codes):
        got = admitted(ix, like_expr(("col", 0), ("lit", int(c))), n)
        want = assert_bits(got, D[:n], [p] * n, "attr LIKE %r" % p[:20], sample=300 if len(p) > 100 else None, rng=rng,
                           must=longs)
        assert len(p) < 1000 or want.any()
    # 'const' LIKE attr: one bit per code, the dictionary as patterns
    subjects = [b"", b"a\nb", b"ab", b"a_b%"] + [s for s in base if 5 < len(s) <= 40][:3]
    codes = dic.add(subjects, ix)
    for s, c in zip(subjects, codes):
        got = admitted(ix, like_expr(("lit", int(c)), ("col", 0)), n)
        assert_bits(got, [s] * n, D[:n], "%r LIKE attr" % s[:20], sample=2000, rng=rng, must=np.concatenate([longs, n // 2 + longs]))
    # attr LIKE attr: one bit per row
    got = admitted(ix, like_expr(("col", 1), ("col", 2)), n)
    want = assert_bits(got, [D[c] for c in col_s], [D[c] for c in col_p], "attr LIKE attr", sample=1000, rng=rng)
    assert 0.05 < want.mean() < 0.95
    # 'const' LIKE 'const': the same bit for every row
    a, b, c = dic.add([b"abc", b"a_c", b"a\nc"], ix)
    assert admitted(ix, like_expr(("lit", int(a)), ("lit", int(b))), n).all()
    assert not admitted(ix, like_expr(("lit", int(c)), ("lit", int(b))), n).any()
    # appends to the dictionary and to the rows between calls
    fresh = dic.add(rand_strings(rng, extra), ix)
    ix.sync_rows(n + extra)
    ix.set_attrs(np.arange(n + extra, dtype=np.int32).view(np.uint8), 4, n + extra)
    col0 = np.concatenate([np.arange(n, dtype=np.int32), fresh])
    ix.set_string_codes(0, n, fresh)
    ix.set_string_codes(1, n, fresh)
    ix.set_string_codes(2, n, fresh[::-1].copy())
    (pc,) = dic.add([b"%a%b%"], ix)
    got = admitted(ix, like_expr(("col", 0), ("lit", int(pc))), n + extra)
    assert_bits(got, [D[c] for c in col0], [b"%a%b%"] * (n + extra), "after appends")
    ix.close()


def dense_setup(vdb, n, d, seed, metric="l2"):
    """Rows with a string column (col 0) and its LIKE '%a_b%' mask mirrored as an int32 flag (offset 0)."""
    rng = np.random.default_rng(seed)
    strings = rand_strings(rng, 4000)
    codes = rng.integers(0, len(strings), n).astype(np.int32)
    X = rng.random((n, d), dtype=np.float32)
    pat = b"%a_b%"
    mask = lm.like_many([strings[c] for c in codes], [pat] * n)
    return X, strings, codes, mask, pat


def prepare(ix, strings, codes, mask, pat, n):
    dic = Dict()
    dic.add(strings, ix)
    (pc,) = dic.add([pat], ix)
    ix.set_string_codes(0, 0, codes)
    ix.set_attrs(mask.astype(np.int32).view(np.uint8), 4, n)
    e = Expr()
    e.int_cmp(EQ, 0, 1)
    return like_expr(("col", 0), ("lit", int(pc))).nodes(), e.nodes()


@pytest.mark.parametrize("nq,coarse,prefilter", [(7, "tf32", False), (40, "fp32", False), (256, "tf32", False),
                                                 (1024, "bf16", False), (7, "tf32", True)])
def test_exact_scan_paths(vdb, nq, coarse, prefilter):
    n, d = 20000, 36
    X, strings, codes, mask, pat = dense_setup(vdb, n, d, 5)
    Q = np.random.default_rng(6).random((nq, d), dtype=np.float32)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.config(500, 500, prefilter=prefilter, force_brute=True)
    ix.set_coarse(coarse)
    like, flag = prepare(ix, strings, codes, mask, pat, n)
    ids, ds, cnt, _ = ix.search(Q, 100, filter_nodes=like)
    er.check_exact(ids, ds, cnt, X, Q, "l2", 100, admissible=mask, what="LIKE nq=%d %s" % (nq, coarse))
    fids, fds, fcnt, _ = ix.search(Q, 100, filter_nodes=flag)
    assert np.array_equal(ids, fids) and np.array_equal(ds, fds) and np.array_equal(cnt, fcnt)
    ix.close()


@pytest.mark.parametrize("W", [1, 4])
def test_graph_branch_with_tail(vdb, W):
    n, n_indexed, d = 3000, 2500, 16
    rng = np.random.default_rng(7 + W)
    X = gm.int_table(n, d, 8)
    off, nb = gm.random_csr(n_indexed, 8, 40, 9)
    t = Table(vdb, X, (n_indexed, off, nb, 3), metrics=("l2",))
    strings = rand_strings(rng, 500)
    codes = rng.integers(0, len(strings), n).astype(np.int32)
    mask = lm.like_many([strings[c] for c in codes], [b"%a%"] * n)
    like, _ = prepare(t.ix["l2"], strings, codes, mask, b"%a%", n)
    Q = gm.int_table(33, d, 10 + W)
    check(t, "l2", Q, 64, 10, W=W, keep=lambda ids, ds: mask[ids], nodes=like, what="LIKE")
    t.close()


@pytest.mark.parametrize("mode", ["scan", "graph"])
def test_sparse_paths(vdb, mode):
    n, vocab = 3000, 2000
    rows = sparse_rows(n, vocab, 11, empty_every=0)
    qs = sparse_rows(12, vocab, 12, max_nnz=40, empty_every=0, dup_every=0)
    rng = np.random.default_rng(13)
    strings = rand_strings(rng, 600)
    codes = rng.integers(0, len(strings), n).astype(np.int32)
    mask = lm.like_many([strings[c] for c in codes], [b"%a_b%"] * n)
    ix = vdb.SparseIndex("ip", vocab)
    ix.append(rows)
    if mode == "graph":
        ix.build(n)
        ix.set_search_mode("graph")
    ix.config(200, 200)
    like, flag = prepare(ix, strings, codes, mask, b"%a_b%", n)
    got = ix.search(qs, 10, filter_nodes=like)[:3]
    want = ix.search(qs, 10, filter_nodes=flag)[:3]
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    assert np.all(mask[got[0][got[0] >= 0]])
    ix.close()


def test_view_beside_its_base(vdb):
    n, d = 5000, 16
    X, strings, codes, mask, pat = dense_setup(vdb, n, d, 14)
    Q = np.random.default_rng(15).random((20, d), dtype=np.float32)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.config(500, 500, force_brute=True)
    like, _ = prepare(ix, strings, codes, mask, pat, n)
    v = ix.view()
    a = ix.search(Q, 10, filter_nodes=like)[:3]
    b = v.search(Q, 10, filter_nodes=like)[:3]
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    er.check_exact(b[0], b[1], b[2], X, Q, "l2", 10, admissible=mask, what="view")
    with pytest.raises(vdb.EpsError) as e:
        ix.append_string_dictionary(len(strings) + 1, [b"x"])   # live view: the base is frozen
    assert e.value.code == BAD_ARG
    v.close()
    ix.close()


def test_facet_programs_share_the_like_scratch(vdb):
    """The key program holds three LIKE nodes (two per code, one per row); each aggregate program holds LIKE nodes of
    other patterns before its numeric root.  All of them are matched by one launch into one buffer, so a key bit
    overwritten by an aggregate's job would change the groups."""
    n, d = 5000, 16
    X, strings, codes, mask, pat = dense_setup(vdb, n, d, 16)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.config(500, 500, force_brute=True)
    prepare(ix, strings, codes, mask, pat, n)
    rng = np.random.default_rng(17)
    codes2 = rng.integers(0, len(strings), n).astype(np.int32)
    ix.set_string_codes(1, 0, codes2)
    dic = Dict()
    dic.strings = list(strings) + [pat]   # what prepare() mirrored
    c1, c2, c3, c4 = dic.add([b"%b", b"%a%", b"a%", b"_"], ix)
    S = [strings[c] for c in codes]
    T = [strings[c] for c in codes2]
    key_mask = (lm.like_many(S, [b"%b"] * n) & ~lm.like_many(S, [b"a%"] * n)) | lm.like_many(S, T)
    k = Expr()   # ((s LIKE '%b') AND NOT (s LIKE 'a%')) OR (s LIKE t)
    k.add(OR, 3, k.both(k.like(k.col(0), k.lit(int(c1))), k.add(NOT, 3, k.like(k.col(0), k.lit(int(c3))))),
          k.like(k.col(0), k.col(1)))
    aggs = []
    for t, lits in ((33, (c2, c4)), (30, (c4,)), (31, (c2,))):
        e = Expr()
        for c in lits:
            e.like(e.col(0), e.lit(int(c)))
        e.like(e.col(1), e.col(0))
        e.add(INT4_ATTR, 1, fo=0)   # the flag column: 1 on the rows of s LIKE '%a_b%'
        aggs.append((t, e.nodes()))
    ids = rng.integers(0, n, (6, 64)).astype(np.int64)
    counts = np.array([64, 0, 1, 30, 64, 17], np.int64)
    got = ix.facet(ids, counts, k.nodes(), 3, aggs)
    for q in range(ids.shape[0]):
        r = ids[q, :counts[q]]
        keys = key_mask[r].astype(float)
        want = []
        for key in dict.fromkeys(keys.tolist()):
            f = mask[r[keys == key]].astype(float)
            want.append((key, [float(f.size), float(f.sum()), float(f.min())]))
        assert [(float(kk), v) for kk, v in got[q]] == want, q
    ix.close()


def test_several_like_nodes_in_one_program(vdb):
    """Per-code, per-row and constant LIKE nodes in one program: one launch with several jobs, each node's words at
    its own offset."""
    rng = np.random.default_rng(21)
    n = 20000
    dic = Dict()
    ix = line_table(vdb, n)
    strings = rand_strings(rng, 6000)
    dic.add(strings, ix)
    ca, cb, cc = (rng.integers(0, len(strings), n).astype(np.int32) for _ in range(3))
    for col, c in enumerate((ca, cb, cc)):
        ix.set_string_codes(col, 0, c)
    A, B, C = ([strings[x] for x in c] for c in (ca, cb, cc))
    pa, pb, sx, sy = dic.add([b"%a%b%", b"%_", b"ab", b"a%"], ix)
    e = Expr()   # ((a LIKE '%a%b%') AND NOT (b LIKE '%_')) OR (b LIKE c) OR ((c LIKE a) AND ('ab' LIKE 'a%'))
    left = e.both(e.like(e.col(0), e.lit(int(pa))), e.add(NOT, 3, e.like(e.col(1), e.lit(int(pb)))))
    mid = e.add(OR, 3, left, e.like(e.col(1), e.col(2)))
    right = e.both(e.like(e.col(2), e.col(0)), e.like(e.lit(int(sx)), e.lit(int(sy))))
    e.add(OR, 3, mid, right)
    want = ((lm.like_many(A, [b"%a%b%"] * n) & ~lm.like_many(B, [b"%_"] * n)) | lm.like_many(B, C) | lm.like_many(C, A))
    got = admitted(ix, e, n)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (bad.size, bad[:5])
    assert 0.05 < want.mean() < 0.95
    # eps_stats.kernel_launches counts the one match-kernel launch
    q = np.array([[-1.0]], np.float32)
    plain = Expr()
    plain.int_cmp(GTE, 0, 0)
    with_like = ix.search(q, 10, filter_nodes=e.nodes())[3]["kernel_launches"]
    assert with_like == ix.search(q, 10, filter_nodes=plain.nodes())[3]["kernel_launches"] + 1
    ix.close()


def test_golden_searches_reproduce(vdb):
    """The reference's Search answers (tests/golden/like.npz) for LIKE filters parsed by its own parser: brute-force
    branch, prefilter, and the graph branch with a tail at width 1.  Ids identical, distances bitwise equal."""
    import os
    import sys
    import zlib
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.join(here, "golden"))
    import make_like_golden as mk
    g = np.load(os.path.join(here, "golden", "like.npz"), allow_pickle=False)
    X, Q, a, title, tag, off, nb = mk.search_table()
    assert zlib.crc32(X.tobytes() + Q.tobytes() + a.tobytes()) == int(g["search_table_crc32"])
    lits = [mk.unpack(g["search_lits_%d_off" % i], g["search_lits_%d_bytes" % i]) for i in range(len(mk.SEARCH_FILTERS))]
    cols = [[v.encode() for v in title], [v.encode() for v in tag]]
    assert cols[0] == mk.unpack(g["search_title_off"], g["search_title_bytes"])
    assert cols[1] == mk.unpack(g["search_tag_off"], g["search_tag_bytes"])
    words = sorted(set(cols[0]) | set(cols[1]) | {t for ls in lits for t in ls})
    code = {w: i for i, w in enumerate(words)}
    ix = vdb.Index("l2", mk.DIM, host_vectors=X)
    ix.sync_rows(mk.N_ROWS)
    ix.append_string_dictionary(0, words)
    ix.set_attrs(g["search_attrs"], int(g["search_stride"]), mk.N_ROWS)
    for col, vals in enumerate(cols):
        ix.set_string_codes(col, 0, np.array([code[v] for v in vals], np.int32))
    progs = []
    for i in range(len(mk.SEARCH_FILTERS)):
        nodes = g["search_nodes_%d" % i].copy()
        consts = np.flatnonzero(nodes[:, 0] == S_CONST)
        assert len(consts) == len(lits[i])
        nodes[consts, 4] = [code[t] for t in lits[i]]
        assert set(nodes[nodes[:, 0] == S_ATTR, 7]) <= {0, 1} and (nodes[nodes[:, 0] == LIKE, 1] == 3).all()
        progs.append(nodes)
    for name, pre in (("brute", False), ("prefilter", True), ("graph", False)):
        if name == "graph":
            ix.set_graph(mk.N_INDEXED, off, nb, 3)
            ix.config(mk.GRAPH_L, mk.GRAPH_L)
            ix.set_search_width(1)
        else:
            ix.config(500, 500, prefilter=pre)
        for i, nodes in enumerate(progs):
            ids, ds, cnt, _ = ix.search(Q, mk.LIMIT, filter_nodes=nodes)
            key = "search_%s_%d" % (name, i)
            what = "%s %r" % (name, mk.SEARCH_FILTERS[i])
            assert np.array_equal(cnt, g[key + "_counts"]), what
            assert np.array_equal(ids, g[key + "_ids"].astype(np.int64)), what
            v = ids >= 0
            assert np.array_equal(ds[v].astype(np.float32).view(np.uint32), g[key + "_dists"][v].view(np.uint32)), what
    ix.close()


def test_errors(vdb):
    n, d = 600, 8
    X, strings, codes, mask, pat = dense_setup(vdb, n, d, 18)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.config(500, 500, force_brute=True)
    like, _ = prepare(ix, strings, codes, mask, pat, n)
    size = len(strings) + 1
    Q = X[:2]

    def code_of(call):
        with pytest.raises(vdb.EpsError) as e:
            call()
        return e.value.code

    e = Expr()   # concatenation under LIKE
    e.like(e.add(ADD, 0, e.col(0), e.lit(0)), e.lit(1))
    assert code_of(lambda: ix.search(Q, 5, filter_nodes=e.nodes())) == UNSUPPORTED
    e = Expr()   # a numeric operand
    e.like(e.col(0), e.add(INT_CONST, 1, iv=3))
    assert code_of(lambda: ix.search(Q, 5, filter_nodes=e.nodes())) == UNSUPPORTED
    for c in (size, -1):   # a literal code outside the dictionary
        assert code_of(lambda: ix.search(Q, 5, filter_nodes=like_expr(("col", 0), ("lit", c)).nodes())) == BAD_ARG
    ix.set_string_codes(3, 0, np.full(n, size, np.int32))   # a column code outside the dictionary
    assert code_of(lambda: ix.search(Q, 5, filter_nodes=like_expr(("col", 3), ("lit", 0)).nodes())) == BAD_ARG
    ix.set_string_codes(4, 0, np.concatenate([[-1], np.zeros(n - 1, np.int32)]).astype(np.int32))
    assert code_of(lambda: ix.search(Q, 5, filter_nodes=like_expr(("lit", 0), ("col", 4)).nodes())) == BAD_ARG
    ix.set_string_codes(4, 0, np.zeros(n, np.int32))   # rewriting every row forgets the old range
    ix.search(Q, 5, filter_nodes=like_expr(("lit", 0), ("col", 4)).nodes())
    assert code_of(lambda: ix.append_string_dictionary(size + 1, [b"gap"])) == BAD_ARG
    assert code_of(lambda: ix.append_string_dictionary(size - 1, [b"overlap"])) == BAD_ARG
    L = vdb.load_library()
    off = np.zeros(2, np.int64)
    assert L.eps_index_append_string_dictionary(ix.h, size, -1, off.ctypes.data, off.ctypes.data) == BAD_ARG
    assert L.eps_index_append_string_dictionary(ix.h, size, 1, None, off.ctypes.data) == BAD_ARG
    back = np.array([3, 1], np.int64)
    assert L.eps_index_append_string_dictionary(ix.h, size, 1, back.ctypes.data, off.ctypes.data) == BAD_ARG
    bad = np.array([[LIKE, 3, 0, 0, 0, 0, 0, -1]], np.int64)   # children that do not precede the node
    assert code_of(lambda: ix.search(Q, 5, filter_nodes=bad)) == BAD_ARG
    # every failure above left the index usable, and the dictionary as it was
    ids, ds, cnt, _ = ix.search(Q, 5, filter_nodes=like)
    er.check_exact(ids, ds, cnt, X, Q, "l2", 5, admissible=mask, what="after errors")
    ix.append_string_dictionary(size, [b"next"])
    ix.close()
