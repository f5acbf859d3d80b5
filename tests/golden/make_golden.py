"""Generate the committed golden fixtures from the REFERENCE ITSELF (oracle/_ref/libepsilla_ref.so =
epsilla-cloud/vectordb's own hot-path sources compiled unmodified, see oracle/Makefile).

Run where oracle.reference_dir() finds a checkout of the reference:   python tests/golden/make_golden.py
The tests read only the .npz files written here.

Fixtures
  dense_vector.npz  engine/test/engine/db/db_server.cpp:92-319  (DbServer.DenseVector) + :1407-1630 (DenseVectorFilter)
  halfcircle.npz    engine/test/engine/db/db_server.cpp:1085-1245 (QueryDenseVectorDuringRebuild, graph-path golden)
  rand2k.npz        seeded random table with a reference-built graph: search / filter / delete / tail / prefilter
                    outputs of VecSearchExecutor::Search at IntraQueryThreads = 1.
  refgraph20k.npz   20 000 x 128 clustered table (tests/helpers.gen seed 901): the graph the REFERENCE builds on it
                    (ANNGraphSegment::BuildFromVectorTable, 7 OpenMP threads) and what the reference's search
                    gets on that graph at IntraQueryThreads 1 and 4 (recall@10, distance evaluations, result ids) —
                    the yard-stick for the device build's quality and for the wide search mode.
"""
import os
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle.oracle import Ref  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def dense_vector():
    names = ["Berlin", "London", "Moscow", "San Francisco", "Shanghai"]
    rows = np.array([[0.05, 0.61, 0.76, 0.74], [0.19, 0.81, 0.75, 0.11], [0.36, 0.55, 0.47, 0.94],
                     [0.18, 0.01, 0.85, 0.8], [0.24, 0.18, 0.22, 0.44]], np.float32)
    ids = np.array([1, 2, 3, 4, 5], np.int32)
    q = np.array([0.35, 0.55, 0.47, 0.94], np.float32)
    expect = {"l2": ["Moscow", "Berlin", "Shanghai", "San Francisco", "London"],
              "ip": ["Moscow", "Berlin", "San Francisco", "London", "Shanghai"],
              "cosine": ["Moscow", "Shanghai", "Berlin", "San Francisco", "London"]}
    out = {"rows": rows, "ids": ids, "query": q, "names": np.array(names)}
    for m in ("l2", "ip", "cosine"):
        r = Ref(m, 4, 16, [("ID", "int4")])
        data, qq = rows.copy(), q.copy()
        if m == "cosine":  # insert normalises rows (table_segment_mvp.cpp:574-587), Search the query (table_mvp.cpp:337)
            data = np.stack([r.normalize(x) for x in data])
            qq = r.normalize(qq)
        r.set_rows(data)
        r.set_attr_column("ID", ids)
        r.make_executors(1, 1, 500)
        rid, rd, _ = r.search(qq, 100)
        assert [names[i] for i in rid] == expect[m], (m, rid)
        out["stored_" + m] = data
        out["query_" + m] = qq
        out["order_" + m] = rid
        out["dist_" + m] = rd
        fid, fd, _ = r.search(qq, 100, "ID <= 2")  # DenseVectorFilter: exactly 2 rows, all ID <= 2
        assert len(fid) == 2 and all(ids[i] <= 2 for i in fid)
        out["filter_nodes"] = r.filter_nodes("ID <= 2")
        out["filter_order_" + m] = fid
        out["attr_stride"] = np.int64(r.stride)
        out["attrs"] = r.attrs[: 5 * r.stride].copy()
    np.savez_compressed(os.path.join(OUT, "dense_vector.npz"), **out)


def halfcircle():
    n, limit = 10000, 500
    rng = np.random.default_rng(20240917)
    perm = rng.permutation(n)  # insertion order; row r holds ID perm[r]
    theta = np.pi / n * perm.astype(np.float64)
    vec = np.stack([np.cos(theta), np.sin(theta)], 1).astype(np.float32)
    r = Ref("cosine", 2, n, [("ID", "int4")])
    vec = np.stack([r.normalize(x) for x in vec])
    r.set_rows(vec)
    r.set_attr_column("ID", perm)
    q = r.normalize(np.array([1.0, 0.0], np.float32))
    # phase 1: first 5000 rows inserted and rebuilt -> pure graph path
    r.set_row_count(5000)
    n_idx, off, nb, nav = r.build(5000, threads=1)
    r.make_executors(1, 1, 500)
    ids1, d1, _ = r.search(q, limit)
    want1 = np.sort(perm[:5000])[:limit]
    assert np.array_equal(perm[ids1], want1), "phase 1 golden mismatch"
    # phase 2: 5000 indexed + 5000 unindexed rows -> graph + brute-force tail merge
    r.set_row_count(n)
    ids2, d2, _ = r.search(q, limit)
    assert np.array_equal(perm[ids2], np.arange(limit)), "phase 2 golden mismatch"
    np.savez_compressed(os.path.join(OUT, "halfcircle.npz"), vectors=vec, perm=perm.astype(np.int32), query=q,
                        offsets=off.astype(np.int64), nbrs=nb.astype(np.int32), nav=np.int64(nav), ids1=ids1, d1=d1,
                        ids2=ids2, d2=d2)


def rand2k():
    n, tail, d, nq = 2000, 300, 32, 16
    rng = np.random.default_rng(42)
    X = rng.random((n + tail, d), dtype=np.float32)
    Q = rng.random((nq, d), dtype=np.float32)
    cols = [("ID", "int4"), ("w", "double"), ("flag", "bool"), ("f", "float"), ("small", "int1")]
    out = {"X": X, "Q": Q}
    filters = ["", "ID < 500", "w > 0.5 AND ID >= 100", "NOT (flag = true) OR @distance < 3.0", "@distance < 3.2",
               "ID % 7 = 3", "f * 2 + small >= 1.5", "(ID + 1) * 2 <> 10 AND flag = true"]
    out["filters"] = np.array(filters)
    idv = np.arange(n + tail)
    wv = rng.random(n + tail)
    flagv = rng.integers(0, 2, n + tail)
    fv = rng.random(n + tail).astype(np.float32)
    sv = rng.integers(-3, 4, n + tail)
    deleted = np.zeros((n + tail + 7) // 8 + 8, np.uint8)
    del_ids = rng.choice(n + tail, 150, replace=False)
    for i in del_ids:
        deleted[i >> 3] |= 1 << (i & 7)
    out["deleted"] = deleted
    for m in ("l2", "ip", "cosine"):
        r = Ref(m, d, n + tail, cols)
        data, qq = X.copy(), Q.copy()
        if m == "cosine":
            data = np.stack([r.normalize(x) for x in data])
            qq = np.stack([r.normalize(x) for x in qq])
        r.set_rows(data)
        for nm, v in (("ID", idv), ("w", wv), ("flag", flagv), ("f", fv), ("small", sv)):
            r.set_attr_column(nm, v)
        r.set_row_count(n)
        n_idx, off, nb, nav = r.build(n, threads=1)
        out["stored_" + m] = data
        out["queries_" + m] = qq
        out["offsets_" + m] = off.astype(np.int64)
        out["nbrs_" + m] = nb.astype(np.int32)
        out["nav_" + m] = np.int64(nav)
        out["attrs"] = r.attrs.copy()
        out["attr_stride"] = np.int64(r.stride)
        for fi, f in enumerate(filters):
            out["nodes_%d" % fi] = r.filter_nodes(f)

        def run(tag, limit, L=500, prefilter=False):
            r.make_executors(1, 1, L, prefilter=prefilter, counting=True)
            for fi, f in enumerate(filters):
                ids = np.full((nq, limit), -1, np.int64)
                ds = np.full((nq, limit), np.inf, np.float64)
                cnt = np.zeros(nq, np.int64)
                nd = np.zeros(nq, np.int64)
                for qi in range(nq):
                    a, b, c = r.search(qq[qi], limit, f)
                    ids[qi, :len(a)] = a
                    ds[qi, :len(a)] = b
                    cnt[qi] = len(a)
                    nd[qi] = c
                out["%s_%s_f%d_ids" % (m, tag, fi)] = ids
                out["%s_%s_f%d_dists" % (m, tag, fi)] = ds
                out["%s_%s_f%d_counts" % (m, tag, fi)] = cnt
                out["%s_%s_f%d_ndist" % (m, tag, fi)] = nd

        run("graph10", 10)                      # pure graph path, n == n_indexed
        if m == "l2":
            run("graph100", 100)
            run("graphL64", 10, L=64)           # small queue
            for i in del_ids:
                r.set_deleted(int(i))
            run("del10", 10)                    # deleted bitmap in the post-filter
            r.set_row_count(n + tail)
            run("tail10", 10)                   # hybrid: graph + brute-force tail merge (Q3)
            run("tail100", 100)
            run("pre10", 10, prefilter=True)    # PreFilterBruteForceSearch over all rows
            for i in del_ids:
                r.set_deleted(int(i), False)
            r.set_row_count(n)
        # brute-force branch: no graph (n_indexed < 512)
        r.set_graph(0, np.zeros(1, np.int64), np.zeros(0, np.int64), 0)
        r.set_row_count(400)
        run("brute10", 10)
    # the l2 / ip table is X itself: stored as its CRC (tests/conftest.py redraws it) to keep the fixture small
    assert np.array_equal(out["stored_l2"], X) and np.array_equal(out["stored_ip"], X)
    for key in ("X", "stored_l2", "stored_ip"):
        del out[key]
    out["table_crc32"] = np.int64(zlib.crc32(X.tobytes()))
    np.savez_compressed(os.path.join(OUT, "rand2k.npz"), **out)


def refgraph20k():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from helpers import exact_topk, gen, recall
    n, d, nq = 20000, 128, 128
    X, Q = gen(n, d, 901, "cluster"), gen(nq, d, 902, "cluster")
    truth = exact_topk(X, Q, 10)
    r = Ref("l2", d, n, [("ID", "int4")])
    r.set_rows(X)
    n_idx, off, nb, nav = r.build(n, threads=7)
    out = {"offsets": off.astype(np.int32), "nbrs": nb.astype(np.int32), "nav": np.int64(nav), "truth": truth.astype(np.int32),
           "n": np.int64(n), "d": np.int64(d), "nq": np.int64(nq)}
    for T in (1, 4):
        for L in (64, 200, 500):
            r.make_executors(1, T, L, counting=True)
            ids = np.full((nq, 10), -1, np.int64)
            ds = np.full((nq, 10), np.inf, np.float64)
            nd = np.zeros(nq, np.int64)
            for qi in range(nq):
                a, b, c = r.search(Q[qi], 10)
                ids[qi, :len(a)] = a
                ds[qi, :len(a)] = b
                nd[qi] = c
            out["T%d_L%d_ids" % (T, L)] = ids.astype(np.int32)
            out["T%d_L%d_dists" % (T, L)] = ds
            out["T%d_L%d_ndist" % (T, L)] = nd
            out["T%d_L%d_recall" % (T, L)] = np.float64(recall(ids, truth, 10))
            print("refgraph20k T=%d L=%d recall %.4f n_dist %.0f" % (T, L, recall(ids, truth, 10), nd.mean()))
    np.savez_compressed(os.path.join(OUT, "refgraph20k.npz"), **out)


def refchecks():
    """What the reference itself answers for the CPU checks of tests/test_oracle.py: distance kernels and Normalize,
    the Expr evaluator on a typed attribute table, and VecSearchExecutor::Search (T = 1) on a graph it built."""
    from helpers import gen
    out = {}
    rng = np.random.default_rng(7)
    dims = list(range(1, 40)) + [127, 128, 130, 131, 768, 769, 770, 771, 1536]
    dist = []
    for d in dims:
        r = {m: Ref(m, d, 4) for m in ("l2", "ip", "cosine")}
        for _ in range(4):
            a, b = rng.standard_normal(d).astype(np.float32), rng.random(d, dtype=np.float32)
            dist.append([r[m].distance(a, b) for m in ("l2", "ip", "cosine")])
    out["dist"] = np.array(dist, np.float32)  # [len(dims) * 4, 3 metrics], drawn in that order
    a = rng.random(333, dtype=np.float32)
    out["normalized"] = r["l2"].normalize(a)

    rng = np.random.default_rng(3)
    n = 64
    r = Ref("l2", 4, n, [("a", "int1"), ("b", "int2"), ("c", "int4"), ("d", "int8"), ("x", "float"), ("y", "double"),
                         ("t", "bool")])
    r.set_rows(rng.random((n, 4), dtype=np.float32))
    r.set_attr_column("a", rng.integers(-100, 100, n)); r.set_attr_column("b", rng.integers(-1000, 1000, n))
    r.set_attr_column("c", rng.integers(-10**6, 10**6, n)); r.set_attr_column("d", rng.integers(-10**12, 10**12, n))
    r.set_attr_column("x", rng.standard_normal(n)); r.set_attr_column("y", rng.standard_normal(n))
    r.set_attr_column("t", rng.integers(0, 2, n))
    out["fe_attrs"], out["fe_stride"] = r.attrs.copy(), np.int64(r.stride)
    out["fe_exprs"] = np.array(FILTER_EVAL_EXPRS)
    res = np.zeros((len(FILTER_EVAL_EXPRS), n, 2), np.int8)
    for i, e in enumerate(FILTER_EVAL_EXPRS):
        out["fe_nodes_%d" % i] = r.filter_nodes(e)
        for row in range(n):
            for j, dd in enumerate((0.25, 0.75)):
                res[i, row, j] = r.filter_eval(e, row, dd)
    out["fe_result"] = res

    n, d = 3000, 24
    X, Q = gen(n, d, 5), gen(12, d, 6)
    r = Ref("l2", d, n, [("ID", "int4")])
    r.set_rows(X)
    r.set_attr_column("ID", np.arange(n))
    ni, off, nb, nav = r.build(threads=2)
    r.make_executors(1, 1, 500, counting=True)
    out.update(live_n_indexed=np.int64(ni), live_offsets=off.astype(np.int64), live_nbrs=nb.astype(np.int32),
               live_nav=np.int64(nav), live_attrs=r.attrs.copy(), live_stride=np.int64(r.stride))
    for fi, f in enumerate(LIVE_FILTERS):
        out["live_nodes_%d" % fi] = r.filter_nodes(f)
        ids = np.full((len(Q), 20), -1, np.int64)
        ds = np.full((len(Q), 20), np.inf, np.float64)
        cnt, nd = np.zeros(len(Q), np.int64), np.zeros(len(Q), np.int64)
        for qi, q in enumerate(Q):
            a, b, c = r.search(q, 20, f)
            ids[qi, :len(a)], ds[qi, :len(a)], cnt[qi], nd[qi] = a, b, len(a), c
        out["live_ids_%d" % fi], out["live_dists_%d" % fi], out["live_counts_%d" % fi], out["live_ndist_%d" % fi] = ids, ds, cnt, nd
    np.savez_compressed(os.path.join(OUT, "refchecks.npz"), **out)


def facets():
    """FacetExecutor::Aggregate + Project of the reference over exact top-64 result lists (tests/test_gpu_parity.py
    test_facets_match_reference): the attribute table, the parsed value expressions and the JSON the reference returns."""
    import json
    from helpers import gen
    from oracle.oracle import Port
    n, d, nq, k = 4000, 16, 12, 64
    X, Q = gen(n, d, 111), gen(nq, d, 112)
    rng = np.random.default_rng(113)
    r = Ref("l2", d, n, FACET_COLS)
    r.set_rows(X)
    idv, wv, fv = np.arange(n), rng.random(n), rng.integers(0, 2, n)
    names = ["n%d" % v for v in rng.integers(0, 9, n)]
    for nm, v in (("ID", idv), ("w", wv), ("flag", fv)):
        r.set_attr_column(nm, v)
    r.set_string_column("name", names)
    ids, ds, cnt, _ = Port().search_batch(metric="l2", vectors=X, queries=Q, limit=k, L=500, prefilter=True)
    out = {"attrs": r.attrs[: n * r.stride].copy(), "stride": np.int64(r.stride), "name_offset": np.int64(r.attr_offset("name")),
           "ids": ids, "dists": ds, "counts": cnt}
    for ci, (group, aggs) in enumerate(FACET_CASES):
        out["key_nodes_%d" % ci], kt = r.value_nodes(group if group else "1")
        out["key_type_%d" % ci] = np.int64(kt)
        for ai, a in enumerate(aggs):
            inner = "1" if a.upper().startswith("COUNT(") else a[a.index("(") + 1:-1]
            out["agg_nodes_%d_%d" % (ci, ai)] = r.value_nodes(inner)[0]
        out["want_%d" % ci] = np.array(json.dumps([r.facet(group, aggs, ids[q, :cnt[q]], ds[q, :cnt[q]]) for q in range(nq)]))
    np.savez_compressed(os.path.join(OUT, "facets.npz"), **out)


FILTER_EVAL_EXPRS = ["a < 0", "b >= 10 OR c < 0", "d / 1000 > a * b", "x + y < 0.5", "t = true", "NOT t = false", "t",
                     "NOT (a > 3 AND t = true)", "c % 5 = 2", "@distance < 0.5", "@distance < 0.5 AND a < 1000",
                     "x * @distance > y", "(a + b) * 2 - c / 3 <= d", "a = b OR x <> y", "true", "false OR t"]
LIVE_FILTERS = ["", "ID >= 1500", "@distance > 1.0"]
FACET_COLS = [("ID", "int4"), ("w", "double"), ("flag", "bool"), ("name", "string")]
FACET_CASES = [("ID % 7", ["SUM(w)", "COUNT(*)", "MIN(ID)", "MAX(w * 2 + @distance)"]), ("name", ["COUNT(*)", "SUM(ID)"]),
               ("flag", ["COUNT(*)", "MAX(@distance)"]), ("w * 2", ["COUNT(*)"]), ("", ["COUNT(*)", "SUM(w)", "MIN(@distance)"])]


if __name__ == "__main__":
    only = sys.argv[1:]
    for fn in (dense_vector, halfcircle, rand2k, refgraph20k, refchecks, facets):
        if not only or fn.__name__ in only:
            fn()
    for f in sorted(os.listdir(OUT)):
        if f.endswith(".npz"):
            print(f, os.path.getsize(os.path.join(OUT, f)))
