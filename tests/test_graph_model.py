"""The width-W graph-search model (graph_model.py) on the CPU: integer tables give one distance in every arithmetic,
and at width 1 the model is the oracle port's SearchImpl, query by query, counters included."""
import numpy as np
import pytest

import graph_model as gm


def f32_sum_distance(metric, x, q):
    """fp32 arithmetic in numpy's own (pairwise) order, no float64 anywhere."""
    x, q = x.astype(np.float32), q.astype(np.float32)
    if metric == "l2":
        return np.float32(np.sum((x - q) * (x - q), dtype=np.float32))
    ip = np.float32(np.sum(x * q, dtype=np.float32))
    return np.float32(-ip) if metric == "ip" else np.float32(np.float32(1) - ip)


@pytest.mark.parametrize("metric", gm.METRICS)
@pytest.mark.parametrize("d", [1, 3, 17, 768, 8192])
def test_integer_distances_agree_bitwise(port, metric, d):
    X, Q = gm.int_table(40, d, 10 + d), gm.int_table(3, d, 20 + d)
    X[0] = 8; Q[0] = -8  # the extreme magnitudes
    gm.assert_exact(X, Q)
    for q in Q:
        want = gm.distances(metric, X, np.arange(X.shape[0]), q)
        for i in range(X.shape[0]):
            p = np.float32(port.distance(metric, X[i], q)) + np.float32(0)
            f = f32_sum_distance(metric, X[i], q) + np.float32(0)
            assert want[i].view(np.uint32) == p.view(np.uint32) == f.view(np.uint32), (metric, d, i, want[i], p, f)
            assert want[i] == np.round(want[i])


def test_exact_bound_is_enforced():
    gm.assert_exact(gm.int_table(2, 65535, 1), gm.int_table(1, 65535, 2))
    with pytest.raises(AssertionError):
        gm.assert_exact(gm.int_table(2, 65536, 1), gm.int_table(1, 65536, 2))
    with pytest.raises(AssertionError):
        gm.assert_exact(gm.int_table(2, 4, 1) + 0.5, gm.int_table(1, 4, 2))


def test_key_encoding_round_trips():
    d = np.array([-3.0, -0.0, 0.0, 1.0, 7.0, 1e30], np.float32)
    ids = np.array([5, 4, 3, 2, 1, 0])
    k = gm.keys_of(d, ids)
    assert np.array_equal(gm.key_ids(k), ids)
    assert np.array_equal(gm.key_dists(k), d + np.float32(0))
    assert gm.keys_of(np.float32([-0.0]), [1])[0] > gm.keys_of(np.float32([0.0]), [0])[0]  # -0 ties +0, id decides
    k0 = gm.keys_of(d, np.zeros(6, np.int64))[[0, 2, 3, 4, 5]]
    assert np.all(k0[1:] > k0[:-1])


def _graphs():
    """Device-independent graphs: (name, n_indexed, total, offsets, nbrs, nav, deleted, L list, filter)."""
    n = 3000
    out = []
    off, nb = gm.random_csr(n, 0, 300, 1)
    out.append(("deg0-300", n, n, off, nb, 7, None, [16, 100], None))
    off, nb = gm.random_csr(n, 2, 40, 2, self_loops=0.3, dup=0.2)
    out.append(("dup+selfloop", n, n, off, nb, 11, None, [1, 33], None))
    off2, nb2 = gm.with_rows(off, nb, {5: []})
    out.append(("empty-nav", n, n, off2, nb2, 5, None, [20], None))
    off3, nb3 = gm.with_rows(off, nb, {9: np.random.default_rng(3).integers(0, n, 250)})
    out.append(("long-nav", n, n, off3, nb3, 9, None, [64], None))
    out.append(("L=n_indexed", 600, 600, *gm.random_csr(600, 1, 12, 4), 0, None, [600], None))
    # tail rows, deleted rows (the navigation point and seeds among them) and a numeric filter
    off, nb = gm.random_csr(n, 4, 30, 5)
    total = n + 400
    dele = np.random.default_rng(6).random(total) < 0.1
    init = gm.prepare_init_ids(off, nb, 13, n, 48)
    dele[[13, *init[:5]]] = True
    out.append(("tail+deleted+filter", n, total, off, nb, 13, dele, [48], 30))
    return out


def _port_search(port, X, Q, metric, n_indexed, total, off, nb, nav, L, limit, deleted, attr, c):
    kw = {}
    if deleted is not None:
        kw["deleted"] = np.packbits(deleted, bitorder="little")
    if c is not None:
        kw.update(attrs=attr.view(np.uint8), attr_stride=4, filter_nodes=attr_lt(c))
    rows = []
    for i in range(Q.shape[0]):
        ids, ds, cnt, (nd, ne) = port.search_batch(metric=metric, vectors=X, queries=Q[i:i + 1], limit=limit,
                                                   total_rows=total, n_indexed=n_indexed, offsets=off, nbrs=nb, nav=nav,
                                                   L=L, **kw)
        rows.append((ids[0], ds[0], cnt[0], nd, ne))
    return rows


NT_INT_CONST, NT_INT4_ATTR, NT_LT = 1, 7, 19


def attr_lt(c):
    return np.array([[NT_INT4_ATTR, 1, -1, -1, 0, 0, 0, 0], [NT_INT_CONST, 1, -1, -1, c, 0, 0, -1],
                     [NT_LT, 3, 0, 1, 0, 0, 0, -1]], np.int64)


def _compare(m, rows, what):
    for i, (ids, ds, cnt, nd, ne) in enumerate(rows):
        assert m.counts[i] == cnt, "%s q%d: count %d != %d" % (what, i, m.counts[i], cnt)
        assert np.array_equal(m.ids[i], ids), "%s q%d: ids" % (what, i)
        assert np.array_equal(m.dists[i], ds), "%s q%d: distances" % (what, i)
        assert m.n_dist[i] == nd and m.n_expand[i] == ne, "%s q%d: n_dist %d/%d n_expand %d/%d" % (
            what, i, m.n_dist[i], nd, m.n_expand[i], ne)


@pytest.mark.parametrize("case", _graphs(), ids=lambda c: c[0])
def test_model_at_width_1_is_the_port(port, case):
    name, n_indexed, total, off, nb, nav, deleted, Ls, c = case
    d = 5
    for j, metric in enumerate(gm.METRICS):
        X, Q = gm.int_table(total, d, 100 + j), gm.int_table(6, d, 200 + j)
        gm.assert_exact(X, Q)
        attr = (np.arange(total) % 97).astype(np.int32)
        keep = None if c is None else (lambda ids, ds: attr[ids] < c)
        for L in Ls:
            for limit in (1, 10, L + 5):
                m = gm.search(X, Q, metric, (n_indexed, off, nb, nav), L, limit, W=1, total=total, deleted=deleted,
                              keep=keep)
                rows = _port_search(port, X, Q, metric, n_indexed, total, off, nb, nav, L, limit, deleted, attr, c)
                _compare(m, rows, "%s %s L=%d limit=%d" % (name, metric, L, limit))
                # n_edges: the ids of every expanded row
                assert np.all(m.n_edges >= 0) and np.all((m.n_expand > 0) | (m.n_edges == 0))


def test_model_below_the_brute_threshold_is_the_port(port):
    off, nb = gm.random_csr(511, 1, 20, 8)
    X, Q = gm.int_table(600, 7, 9), gm.int_table(4, 7, 10)
    for metric in gm.METRICS:
        m = gm.search(X, Q, metric, (511, off, nb, 3), 50, 20, W=4, total=600)
        _compare(m, _port_search(port, X, Q, metric, 511, 600, off, nb, 3, 50, 20, None, None, None), "brute " + metric)


@pytest.mark.parametrize("corrupt", ["tie", "skip", "second"])
def test_model_corruptions_are_caught(port, corrupt):
    n = 3000
    off, nb = gm.random_csr(n, 4, 40, 11)
    X, Q = gm.int_table(n, 3, 12, B=2), gm.int_table(24, 3, 13, B=2)  # few distinct distances: many ties
    m = gm.search(X, Q, "l2", (n, off, nb, 0), 40, 40, corrupt=corrupt)
    rows = _port_search(port, X, Q, "l2", n, n, off, nb, 0, 40, 40, None, None, None)
    with pytest.raises(AssertionError):
        _compare(m, rows, corrupt)


def test_wide_model_is_a_valid_search():
    """At W > 1 the queue is still sorted, unique and made of seeds and rows reachable from them, and every entry left
    in it is checked; W >= L expands the whole queue each step."""
    n = 2000
    off, nb = gm.random_csr(n, 0, 80, 14, dup=0.1)
    X, Q = gm.int_table(n, 6, 15), gm.int_table(5, 6, 16)
    for W in (1, 2, 3, 8, 64):
        for q in Q:
            r = gm.wide_search(X, q, "ip", (n, off, nb, 1), 64, W)
            assert np.all(r.keys[1:] > r.keys[:-1]) and r.checked.all()
            assert np.unique(gm.key_ids(r.keys)).size == 64
            assert r.n_dist == 64 + r.fresh


def test_vset_bucket_matches_the_device_rule():
    cap, shift, vmax = gm.vset_geometry(64)
    assert (cap, shift, vmax) == (1024, 25, 768)
    assert gm.vset_geometry(1024) == (16384, 21, 12288)
    ids = np.arange(1 << 16)
    b = gm.vset_bucket(ids, 64)
    assert b.min() == 0 and b.max() == cap - 8 and np.all(b % 8 == 0)
    assert b[1] == (((0x9e3779b1 * 1) & 0xffffffff) >> 25) << 3
