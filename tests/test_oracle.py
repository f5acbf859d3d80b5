"""CPU tests: the oracle restatement (oracle/oracle_port.c) against the reference's golden vectors
(tests/golden, generated from the compiled reference by tests/golden/make_golden.py), bit for bit."""
import os

import numpy as np
import pytest

from helpers import gen

METRICS = ("l2", "ip", "cosine")


@pytest.fixture(scope="module")
def refchecks():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refchecks.npz"), allow_pickle=False)


def test_dense_vector_known_answers(port, golden):
    """engine/test/engine/db/db_server.cpp:289-292 (DenseVector) and :1620-1627 (DenseVectorFilter)."""
    g = golden["dense_vector"]
    names = list(g["names"])
    expect = {"l2": ["Moscow", "Berlin", "Shanghai", "San Francisco", "London"],
              "ip": ["Moscow", "Berlin", "San Francisco", "London", "Shanghai"],
              "cosine": ["Moscow", "Shanghai", "Berlin", "San Francisco", "London"]}
    for m in METRICS:
        ids, ds, cnt, _ = port.search_batch(metric=m, vectors=g["stored_" + m], queries=g["query_" + m], limit=100)
        assert cnt[0] == 5
        assert [names[i] for i in ids[0, :5]] == expect[m]
        assert np.array_equal(ids[0, :5], g["order_" + m])
        assert np.array_equal(ds[0, :5], g["dist_" + m])  # bit-exact vs the reference
        ids, ds, cnt, _ = port.search_batch(metric=m, vectors=g["stored_" + m], queries=g["query_" + m], limit=100,
                                            attrs=g["attrs"], attr_stride=int(g["attr_stride"]),
                                            filter_nodes=g["filter_nodes"])
        assert cnt[0] == 2 and np.array_equal(ids[0, :2], g["filter_order_" + m])


def test_halfcircle_graph_golden(port, golden):
    """db_server.cpp:1085-1245: exact top-500 on the graph path, then graph + brute-force tail."""
    g = golden["halfcircle"]
    perm = g["perm"]
    kw = dict(metric="cosine", vectors=g["vectors"], queries=g["query"], limit=500, n_indexed=5000,
              offsets=g["offsets"], nbrs=g["nbrs"].astype(np.int64), nav=int(g["nav"]), L=500)
    ids, ds, cnt, _ = port.search_batch(total_rows=5000, **kw)
    assert cnt[0] == 500
    assert np.array_equal(ids[0], g["ids1"]) and np.array_equal(ds[0], g["d1"])
    assert np.array_equal(perm[ids[0]], np.sort(perm[:5000])[:500])
    ids, ds, cnt, _ = port.search_batch(total_rows=10000, **kw)
    assert np.array_equal(ids[0], g["ids2"]) and np.array_equal(ds[0], g["d2"])
    assert np.array_equal(perm[ids[0]], np.arange(500))


def _rand2k_case(port, g, m, tag, fi):
    n, tail = 2000, 300
    kw = dict(metric=m, vectors=g["stored_" + m], queries=g["queries_" + m], attrs=g["attrs"],
              attr_stride=int(g["attr_stride"]), filter_nodes=g["nodes_%d" % fi])
    limit = 100 if tag.endswith("100") else 10
    L = 64 if tag == "graphL64" else 500
    graph = dict(n_indexed=n, offsets=g["offsets_" + m], nbrs=g["nbrs_" + m].astype(np.int64), nav=int(g["nav_" + m]))
    if tag.startswith("graph"):
        kw.update(graph, total_rows=n)
    elif tag == "del10":
        kw.update(graph, total_rows=n, deleted=g["deleted"])
    elif tag.startswith("tail"):
        kw.update(graph, total_rows=n + tail, deleted=g["deleted"])
    elif tag == "pre10":
        kw.update(graph, total_rows=n + tail, deleted=g["deleted"], prefilter=True)
    elif tag == "brute10":
        kw.update(total_rows=400, n_indexed=0)
    return port.search_batch(limit=limit, L=L, **kw)


@pytest.mark.parametrize("m", METRICS)
def test_rand2k_port_matches_reference_outputs(port, golden, m):
    g = golden["rand2k"]
    tags = ["graph10", "brute10"] + (["graph100", "graphL64", "del10", "tail10", "tail100", "pre10"] if m == "l2" else [])
    for tag in tags:
        for fi in range(len(g["filters"])):
            ids, ds, cnt, st = _rand2k_case(port, g, m, tag, fi)
            key = "%s_%s_f%d_" % (m, tag, fi)
            assert np.array_equal(cnt, g[key + "counts"]), key
            assert np.array_equal(ids, g[key + "ids"]), key
            assert np.array_equal(ds, g[key + "dists"]), key
            assert st[0] == int(g[key + "ndist"].sum()), key  # same number of distance evaluations


def test_prepare_init_ids(port, golden):
    g = golden["rand2k"]
    off, nb, nav = g["offsets_l2"], g["nbrs_l2"].astype(np.int64), int(g["nav_l2"])
    ids = port.prepare_init_ids(off, nb, nav, 2000, 500)
    assert len(set(ids.tolist())) == 500
    row = nb[off[nav]:off[nav + 1]]
    assert np.array_equal(ids[:len(row)], row)
    rest = ids[len(row):]
    assert rest[0] == (nav + 1) % 2000 or (nav + 1) % 2000 in row


def test_distances_bitexact_vs_reference(port, refchecks):
    rng = np.random.default_rng(7)
    want = iter(refchecks["dist"])
    for d in list(range(1, 40)) + [127, 128, 130, 131, 768, 769, 770, 771, 1536]:
        for _ in range(4):
            a, b = rng.standard_normal(d).astype(np.float32), rng.random(d, dtype=np.float32)
            for m, x in zip(METRICS, next(want)):
                y = port.distance(m, a, b)
                assert np.float32(x).tobytes() == np.float32(y).tobytes(), (d, m, x, y)
    a = rng.random(333, dtype=np.float32)
    assert np.array_equal(refchecks["normalized"], port.normalize(a))


def test_port_matches_reference_search_live(port, refchecks):
    """Seeded table with the graph the reference built on it (fixture refchecks): port vs VecSearchExecutor (T=1)
    without filter, with an attribute filter and with a distance filter."""
    g = refchecks
    n, d = 3000, 24
    X, Q = gen(n, d, 5), gen(12, d, 6)
    graph = dict(n_indexed=int(g["live_n_indexed"]), offsets=g["live_offsets"], nbrs=g["live_nbrs"].astype(np.int64),
                 nav=int(g["live_nav"]))
    for fi in range(3):
        nodes = g["live_nodes_%d" % fi]
        for qi, q in enumerate(Q):
            n_want = int(g["live_counts_%d" % fi][qi])
            a, b = g["live_ids_%d" % fi][qi, :n_want], g["live_dists_%d" % fi][qi, :n_want]
            ids, ds, cnt, st = port.search_batch(metric="l2", vectors=X, queries=q, limit=20, attrs=g["live_attrs"],
                                                 attr_stride=int(g["live_stride"]), filter_nodes=nodes, **graph)
            assert cnt[0] == n_want and np.array_equal(ids[0, :n_want], a) and np.array_equal(ds[0, :n_want], b)
            assert st[0] == g["live_ndist_%d" % fi][qi]


def test_filter_eval_vs_reference(port, refchecks):
    """The port's evaluator on the node programs the reference's parser produced (fixture refchecks) against the
    reference's Expr evaluator on the same typed attribute table: every expression, row and distance."""
    g = refchecks
    attrs, stride = g["fe_attrs"], int(g["fe_stride"])
    for i, e in enumerate(g["fe_exprs"]):
        nodes = g["fe_nodes_%d" % i]
        for row in range(attrs.size // stride):
            for j, dist in enumerate((0.25, 0.75)):
                assert port.filter_eval(nodes, attrs, stride, row, dist) == g["fe_result"][i, row, j], (e, row)


def test_add_into_queue_properties(port):
    """AddIntoQueue (vec_search_executor.cpp:75-117): the bounded queue stays sorted by (distance,id), holds the
    best `cap` entries ever offered, never holds an id twice when the duplicate lands on its twin, and the
    returned position is where the entry went (cap = rejected / duplicate)."""
    import ctypes as C
    rng = np.random.default_rng(9)
    for cap in (1, 4, 16):
        ids = np.zeros(cap + 1, np.int64); ds = np.zeros(cap + 1, np.float32); ck = np.zeros(cap + 1, np.uint8)
        size = C.c_int64(0)
        offered = {}
        for step in range(200):
            i = int(rng.integers(0, 40)); d = float(np.float32(rng.integers(0, 12)) / 4)
            dup_of_existing = i in offered and offered[i] == d
            r = port.L.port_add_into_queue(ids.ctypes.data, ds.ctypes.data, ck.ctypes.data, C.byref(size), cap, i, C.c_float(d))
            n = size.value
            assert 0 <= n <= cap
            keys = list(zip(ds[:n].tolist(), ids[:n].tolist()))
            assert keys == sorted(keys), "queue must stay sorted by (distance, id)"
            if r < cap:
                assert ids[r] == i and ds[r] == np.float32(d)
                offered[i] = d
            elif dup_of_existing and (d, i) in keys:
                pass  # duplicate rejected (:91-95)
        best = sorted(keys)
        assert keys == best[:n]


def test_search_is_deterministic_and_L_monotone(port, golden):
    """The T=1 search is a pure function of its inputs, and a longer queue never evaluates fewer rows."""
    g = golden["rand2k"]
    kw = dict(metric="l2", vectors=g["stored_l2"][:2000], queries=g["queries_l2"][:4], limit=10, n_indexed=2000,
              offsets=g["offsets_l2"], nbrs=g["nbrs_l2"].astype(np.int64), nav=int(g["nav_l2"]), total_rows=2000)
    a = port.search_batch(L=128, **kw)
    b = port.search_batch(L=128, **kw)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[3] == b[3]
    c = port.search_batch(L=512, **kw)
    assert c[3][0] >= a[3][0]
    assert np.all(c[1][:, 0] <= a[1][:, 0] + 1e-12)  # the best distance can only improve with a longer queue


def test_port_matches_reference_on_its_own_20k_graph(port, golden_refgraph):
    """The C restatement on the graph the reference built over 20 000 x 128 rows (fixture refgraph20k, outputs of the
    reference at IntraQueryThreads = 1): identical ids, distances and distance-evaluation counts."""
    from helpers import assert_same_results, gen
    g = golden_refgraph
    n, d, nq = int(g["n"]), int(g["d"]), 32
    X, Q = gen(n, d, 901, "cluster"), gen(int(g["nq"]), d, 902, "cluster")[:nq]
    for L in (64, 200):
        ids, ds, cnt, (nd, _) = port.search_batch(metric="l2", vectors=X, queries=Q, limit=10, n_indexed=n,
                                                  offsets=g["offsets"].astype(np.int64), nbrs=g["nbrs"].astype(np.int64),
                                                  nav=int(g["nav"]), L=L)
        rate = assert_same_results(ids, ds, cnt, g["T1_L%d_ids" % L][:nq].astype(np.int64), g["T1_L%d_dists" % L][:nq],
                                   np.full(nq, 10), "port on refgraph L=%d" % L)
        assert rate == 1.0
        assert nd == int(g["T1_L%d_ndist" % L][:nq].sum())
