"""GPU test of the drop-in boundary: the reference engine's OWN classes (TableSegmentMVP, ANNGraphSegment,
VecSearchExecutor, Expr parser — compiled unmodified) with VecSearchExecutor::{ctor,Search} and
ANNGraphSegment::BuildFromVectorTable replaced at link time by integration/epsilla_b200_dropin.cpp, i.e.
the search and the build run on the GPU through the C ABI while the caller-facing surface is the
reference's.  Replays the reference's golden tests through that surface."""
import os

import numpy as np
import pytest

from helpers import assert_same_results, exact_topk, gen, recall

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROPIN = os.path.join(ROOT, "oracle", "_ref", "dropin", "libepsilla_ref_b200.so")


@pytest.fixture(scope="module")
def Drop():
    if not os.path.exists(DROPIN):
        pytest.skip("oracle/_ref/dropin/libepsilla_ref_b200.so was not built (needs a reference checkout at build time)")
    from oracle.oracle import Ref

    def make(metric, dim, cap, cols=()):
        return Ref(metric, dim, cap, cols, lib_path=DROPIN)
    return make


def test_dense_vector_through_reference_surface(Drop, golden):
    g = golden["dense_vector"]
    for m in ("l2", "ip", "cosine"):
        r = Drop(m, 4, 16, [("ID", "int4")])
        r.set_rows(g["stored_" + m])
        r.set_attr_column("ID", g["ids"])
        r.make_executors(2, 4, 500)  # TableMVP-style: several executors share one device mirror
        ids, ds, _ = r.search(g["query_" + m], 100)
        assert np.array_equal(ids, g["order_" + m])
        assert np.allclose(ds, g["dist_" + m], rtol=1e-4, atol=1e-7)
        ids, ds, _ = r.search(g["query_" + m], 100, "ID <= 2")  # string -> reference parser -> device filter
        assert np.array_equal(ids, g["filter_order_" + m])


def test_halfcircle_through_reference_surface(Drop, golden):
    g = golden["halfcircle"]
    perm = g["perm"]
    r = Drop("cosine", 2, 10000, [("ID", "int4")])
    r.set_rows(g["vectors"])
    r.set_attr_column("ID", perm)
    r.set_row_count(5000)
    r.set_graph(5000, g["offsets"], g["nbrs"].astype(np.int64), int(g["nav"]))
    r.make_executors(1, 4, 500)
    ids, ds, _ = r.search(g["query"], 500)
    assert np.array_equal(perm[ids], np.sort(perm[:5000])[:500])
    r.set_row_count(10000)  # rows appended after the executor was built: tail brute force + merge
    ids, ds, _ = r.search(g["query"], 500)
    assert np.array_equal(perm[ids], np.arange(500))
    r.set_deleted([int(np.nonzero(perm == 3)[0][0])])  # DeleteByPK: deleted rows vanish from results
    ids, ds, _ = r.search(g["query"], 500)
    assert 3 not in perm[ids].tolist() and len(ids) == 500 - 1


def test_gpu_build_through_reference_surface(Drop):
    """ANNGraphSegment::BuildFromVectorTable -> device build -> reference CSR members -> search."""
    n, d, nq = 5000, 32, 32
    X, Q = gen(n, d, 77), gen(nq, d, 78)
    r = Drop("l2", d, n, [("ID", "int4")])
    r.set_rows(X)
    r.set_attr_column("ID", np.arange(n))
    ni, off, nb, nav = r.build(threads=1)
    assert ni == n and off[-1] == len(nb) and nb.min() >= 0 and nb.max() < n
    r.make_executors(4, 1, 500)
    ids, ds, cnt = r.search_batch(Q, 10, "ID >= 100")
    assert np.all(cnt == 10) and np.all(ids >= 100)
    truth = exact_topk(X[100:], Q, 10) + 100
    assert recall(ids, truth, 10) >= 0.97


def test_concurrent_calls_are_coalesced_and_correct(Drop):
    """16 executors hammered by 16 threads (ExecutorPool-style concurrency): single-query Search calls are
    gathered into batched launches by the drop-in's batch former; every caller still gets its own answer."""
    n, d, nq = 20000, 48, 512
    X, Q = gen(n, d, 91), gen(nq, d, 92)
    r = Drop("l2", d, n, [("ID", "int4")])
    r.set_rows(X)
    import ctypes as C
    r.set_attr_column("ID", np.arange(n))
    r.make_executors(16, 4, 500)      # n_indexed = 0 -> exact-scan branch
    counters = lambda: (lambda c, l: (r.L.eps_dropin_counters(C.byref(c), C.byref(l)), (c.value, l.value))[1])(C.c_int64(), C.c_int64())
    c0, l0 = counters()
    ids, ds, cnt = r.search_batch(Q, 10)
    c1, l1 = counters()
    truth = exact_topk(X, Q, 10)
    assert np.all(cnt == 10) and recall(ids, truth, 10) > 0.999
    assert c1 - c0 == nq and l1 - l0 < nq, "coalescing: %d calls served by %d launches" % (c1 - c0, l1 - l0)
    ids5, _, cnt5 = r.search_batch(Q[:64], 5)   # a different limit goes into its own batch
    assert np.all(cnt5 == 5) and np.array_equal(ids5, ids[:64, :5])
    # filtered calls with the same program share launches too, and still answer per caller
    c2, l2 = counters()
    fids, _, fcnt = r.search_batch(Q, 10, "ID >= 1000")
    c3, l3 = counters()
    assert np.all(fcnt == 10) and fids.min() >= 1000
    assert recall(fids, exact_topk(X[1000:], Q, 10) + 1000, 10) > 0.999
    assert c3 - c2 == nq and l3 - l2 < nq


def test_deletes_and_appends_reach_the_device_incrementally(Drop):
    """f3: single-bit deletes and appended rows between calls (dirty-span bitset upload, append-only row / attribute
    upload) — results must track the segment exactly."""
    n, d = 6000, 24
    X, Q = gen(n, d, 95), gen(8, d, 96)
    r = Drop("l2", d, n, [("ID", "int4")])
    r.set_rows(X[:4000])
    r.set_attr_column("ID", np.arange(n))
    r.make_executors(1, 1, 500)
    live = np.ones(n, bool)
    live[4000:] = False
    for step in range(6):
        ids, _, cnt = r.search_batch(Q, 10, "ID >= 0")
        rows = np.nonzero(live)[0]
        want = rows[exact_topk(X[rows], Q, 10)]
        assert np.all(cnt == 10) and recall(ids, want, 10) == 1.0, step
        victims = ids[:, 0]                      # delete every query's nearest neighbour
        r.set_deleted(victims)
        live[victims] = False
        if step == 2:                            # rows appended while the executor lives
            r.vectors[4000:5000] = X[4000:5000]
            r.set_row_count(5000)
            live[4000:5000] = True


def test_graph_file_round_trip_through_reference_io(Drop, tmp_path):
    """GPU-built graph -> reference SaveANNGraph (ann_graph_<field>.bin) -> reference loader -> GPU search."""
    n, d, nq = 4000, 16, 16
    X, Q = gen(n, d, 61), gen(nq, d, 62)
    r = Drop("l2", d, n, [("ID", "int4")])
    r.set_rows(X)
    ni, off, nb, nav = r.build(threads=1)
    r.make_executors(1, 1, 500)
    before, bd, _ = r.search_batch(Q, 10)
    r.save_graph(str(tmp_path))
    path = tmp_path / "0" / "ann_graph_1.bin"
    raw = np.fromfile(path, dtype=np.int64)       # layout: n, first_id, offsets[n+1], nbrs[E], nav (:171-184)
    assert raw[0] == n and raw[1] == 0 and raw[-1] == nav and len(raw) == 2 + (n + 1) + off[-1] + 1
    assert np.array_equal(raw[2:2 + n + 1], off) and np.array_equal(raw[2 + n + 1:-1], nb)
    r2 = Drop("l2", d, n, [("ID", "int4")])
    r2.set_rows(X)
    r2.load_graph(str(tmp_path))
    r2.make_executors(1, 1, 500)
    after, ad, _ = r2.search_batch(Q, 10)
    assert np.array_equal(before, after) and np.allclose(bd, ad)


def test_string_filters_through_reference_surface(Drop):
    """f4: string EQ / NE / IN and column-to-column equality (expr_evaluator.cpp:110-125,:176-190) — the parser and
    the segment's string columns are the reference's, the drop-in dictionary-encodes them and the device compares
    codes; every result must equal the unmodified reference's on the same segment contents."""
    from oracle.oracle import Ref, have_ref
    if not have_ref():
        pytest.skip("oracle/_ref/libepsilla_ref.so did not travel")
    n, d, nq = 3000, 16, 24
    X, Q = gen(n, d, 71), gen(nq, d, 72)
    rng = np.random.default_rng(73)
    names = ["city%d" % v for v in rng.integers(0, 12, n)]
    tags = ["city%d" % v for v in rng.integers(0, 4, n)]
    cols = [("ID", "int4"), ("name", "string"), ("tag", "string")]
    filters = ["name = 'city3'", "name <> 'city3' AND ID < 1500", "name IN ('city1', 'nowhere', 'city7')",
               "NOT (name IN ('city1', 'city2')) AND ID >= 100", "name = tag", "name = 'nowhere'", "name <> 'nowhere'",
               "tag IN ('city0') OR @distance < 1.5"]

    def fill(r, rows):
        r.set_rows(X[:rows])
        r.set_attr_column("ID", np.arange(n))
        r.set_string_column("name", names)
        r.set_string_column("tag", tags)
        r.make_executors(2, 1, 500)

    ref, gpu = Ref("l2", d, n, cols), Drop("l2", d, n, cols)
    fill(ref, 2000)
    fill(gpu, 2000)
    for rows in (2000, n):                       # second round: rows (and their strings) appended afterwards
        ref.set_row_count(rows); ref.vectors[:rows] = X[:rows]
        gpu.set_row_count(rows); gpu.vectors[:rows] = X[:rows]
        for f in filters:
            wi, wd, wc = ref.search_batch(Q, 10, f)
            gi, gd, gc = gpu.search_batch(Q, 10, f)
            assert_same_results(gi, gd, gc, wi, wd, wc, "%s @%d" % (f, rows))
    with pytest.raises(Exception):
        gpu.search(Q[0], 10, "name LIKE 'city%'")  # regex work stays out of scope: reported, never computed on the CPU
