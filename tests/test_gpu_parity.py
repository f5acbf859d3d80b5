"""GPU parity tests (run with -m gpu on an H100).  Every call goes through the C ABI
(libepsilla_b200.so via vectordb_b200.Index); the checker is the oracle (oracle_port.c, and the compiled
reference oracle/_ref/libepsilla_ref.so when it travelled) and the committed golden fixtures."""
import numpy as np
import pytest

from helpers import assert_same_results, exact_topk, gen, recall

pytestmark = pytest.mark.gpu
METRICS = ("l2", "ip", "cosine")


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200
    L = vectordb_b200.load_library()
    assert L.eps_device_count() > 0, "GPU tests need a CUDA device"
    return vectordb_b200


# ---- A1-A3, A14: distances and Normalize ---------------------------------------------------------------
def test_pair_distances_match_oracle(vdb, port):
    from vectordb_b200.index import pair_distances
    rng = np.random.default_rng(11)
    for d in (1, 2, 3, 4, 7, 32, 100, 128, 130, 768, 1536):
        a = rng.standard_normal((64, d)).astype(np.float32)
        b = rng.random((64, d), dtype=np.float32)
        for m in METRICS:
            got = pair_distances(m, a, b)
            want = np.array([port.distance(m, a[i], b[i]) for i in range(64)], np.float32)
            assert np.allclose(got, want, rtol=1e-4, atol=1e-6), (d, m, np.abs(got - want).max())


def test_normalize_matches_oracle(vdb, port):
    from vectordb_b200.index import normalize
    rng = np.random.default_rng(12)
    for d in (2, 4, 33, 768):
        v = rng.standard_normal((8, d)).astype(np.float32)
        got = normalize(v)
        want = np.stack([port.normalize(x) for x in v])
        assert np.allclose(got, want, rtol=1e-5, atol=1e-7)


# ---- A9/A11 brute-force branch: reference known answers ---------------------------------------------------
def test_dense_vector_golden(vdb, golden):
    g = golden["dense_vector"]
    for m in METRICS:
        ix = vdb.Index(m, 4, host_vectors=g["stored_" + m])
        ix.sync_rows(5)
        ix.set_attrs(g["attrs"], int(g["attr_stride"]), 5)
        ids, ds, cnt, _ = ix.search(g["query_" + m], 100)
        assert cnt[0] == 5 and np.array_equal(ids[0, :5], g["order_" + m])
        assert np.allclose(ds[0, :5], g["dist_" + m], rtol=1e-4, atol=1e-7)
        assert np.all(ids[0, 5:] == -1)
        ids, ds, cnt, _ = ix.search(g["query_" + m], 100, filter_nodes=g["filter_nodes"])
        assert cnt[0] == 2 and np.array_equal(ids[0, :2], g["filter_order_" + m])
        ix.close()


# ---- A4-A8 + tail merge: the reference's graph-path golden test ------------------------------------------
def test_halfcircle_golden(vdb, golden):
    g = golden["halfcircle"]
    perm = g["perm"]
    ix = vdb.Index("cosine", 2, host_vectors=g["vectors"])
    ix.sync_rows(5000)
    ix.set_graph(5000, g["offsets"], g["nbrs"].astype(np.int64), int(g["nav"]))
    ix.config(500, 500)
    ids, ds, cnt, st = ix.search(g["query"], 500)
    assert cnt[0] == 500
    assert np.array_equal(perm[ids[0]], np.sort(perm[:5000])[:500]), "exact top-500 (db_server.cpp:1164-1181)"
    assert_same_results(ids, ds, cnt, g["ids1"][None], g["d1"][None], [500], "halfcircle phase 1")
    ix.sync_rows(10000)  # 5000 indexed + 5000 unindexed -> graph + brute-force tail merge
    ids, ds, cnt, st = ix.search(g["query"], 500)
    assert cnt[0] == 500
    assert np.array_equal(perm[ids[0]], np.arange(500)), "graph + tail (db_server.cpp:1185-1200)"
    assert_same_results(ids, ds, cnt, g["ids2"][None], g["d2"][None], [500], "halfcircle phase 2")
    ix.close()


# ---- every Search() mode against outputs of the reference itself ------------------------------------------
@pytest.mark.parametrize("m", METRICS)
def test_rand2k_all_modes(vdb, golden, m):
    g = golden["rand2k"]
    n, tail = 2000, 300
    ix = vdb.Index(m, 32, host_vectors=g["stored_" + m])
    ix.set_attrs(g["attrs"], int(g["attr_stride"]), n + tail)
    nf = len(g["filters"])
    rates = []

    def check(tag, limit):
        for fi in range(nf):
            ids, ds, cnt, st = ix.search(g["queries_" + m], limit, filter_nodes=g["nodes_%d" % fi])
            key = "%s_%s_f%d_" % (m, tag, fi)
            rates.append(assert_same_results(ids, ds, cnt, g[key + "ids"], g[key + "dists"], g[key + "counts"], key))
            if tag.startswith("graph"):
                assert st["n_dist"] == int(g[key + "ndist"].sum()) or abs(st["n_dist"] - int(g[key + "ndist"].sum())) < 0.02 * st["n_dist"], key

    # brute-force branch (no graph)
    ix.sync_rows(400)
    check("brute10", 10)
    ix.sync_rows(n)
    ix.set_graph(n, g["offsets_" + m], g["nbrs_" + m].astype(np.int64), int(g["nav_" + m]))
    ix.config(500, 500)
    check("graph10", 10)
    if m == "l2":
        check("graph100", 100)
        ix.config(64, 64)
        check("graphL64", 10)
        ix.config(500, 500)
        ix.set_deleted(g["deleted"])
        check("del10", 10)
        ix.sync_rows(n + tail)
        check("tail10", 10)
        check("tail100", 100)
        ix.config(500, 500, prefilter=True)
        check("pre10", 10)
    ix.close()
    assert np.mean(rates) > 0.9, "exact-match rate %.3f" % np.mean(rates)


# ---- same graph, GPU search vs oracle search, bigger table ------------------------------------------------
def test_graph_search_vs_port_same_graph(vdb, port):
    n, d, nq = 20000, 64, 48
    X, Q = gen(n, d, 101, "cluster"), gen(nq, d, 102, "cluster")
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.build(n)
    ni, off, nb, nav = ix.get_graph()
    assert ni == n and off[-1] == len(nb) and 0 <= nav < n
    deg = np.diff(off)
    assert deg.min() >= 1 and np.percentile(deg, 99) <= 64
    for L, limit in ((500, 10), (128, 100)):
        ix.config(L, L)
        ids, ds, cnt, st = ix.search(Q, limit)
        pids, pds, pcnt, pst = port.search_batch(metric="l2", vectors=X, queries=Q, limit=limit, n_indexed=n, offsets=off,
                                                 nbrs=nb, nav=nav, L=L)
        rate = assert_same_results(ids, ds, cnt, pids, pds, pcnt, "L=%d" % L)
        assert rate > 0.9
        assert abs(st["n_dist"] - pst[0]) <= 0.01 * pst[0]
        assert abs(st["n_expand"] - pst[1]) <= 0.01 * pst[1]
    truth = exact_topk(X, Q, 10)
    ix.config(500, 500)
    ids, _, _, _ = ix.search(Q, 10)
    assert recall(ids, truth, 10) >= 0.98
    # idempotence (visited bitmaps are left clean) and sortedness
    ids2, ds2, _, _ = ix.search(Q, 10)
    assert np.array_equal(ids, ids2)
    assert np.all(np.diff(ds2, axis=1) >= 0)
    ix.close()


def test_reference_executor_on_gpu_built_graph(vdb, have_ref):
    """The unmodified reference VecSearchExecutor searching the GPU-built CSR (BASELINE.md §3.2)."""
    if not have_ref:
        pytest.skip("oracle/_ref/libepsilla_ref.so did not travel")
    from oracle.oracle import Ref
    n, d, nq = 6000, 32, 24
    X, Q = gen(n, d, 7), gen(nq, d, 8)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.build(n)
    ni, off, nb, nav = ix.get_graph()
    ix.config(500, 500)
    ids, ds, cnt, _ = ix.search(Q, 10)
    r = Ref("l2", d, n, [("ID", "int4")])
    r.set_rows(X)
    r.set_graph(ni, off, nb, nav)
    r.make_executors(1, 1, 500)
    rids, rds, rcnt = r.search_batch(Q, 10)
    assert_same_results(ids, ds, cnt, rids, rds, rcnt, "reference executor")
    ix.close()


# ---- brute force: batched tile kernel and row kernel, all metrics, ragged dims ----------------------------
@pytest.mark.parametrize("m", METRICS)
def test_brute_force_batched(vdb, port, m):
    for n, d, nq, k in ((30000, 128, 64, 10), (5000, 33, 3, 100), (1000, 6, 40, 500), (513, 768, 17, 10)):
        X, Q = gen(n, d, n + d), gen(nq, d, n + d + 1)
        ix = vdb.Index(m, d, host_vectors=X)
        ix.sync_rows(n)
        ix.config(500, 500, force_brute=True)
        ids, ds, cnt, st = ix.search(Q, k)
        sub = slice(0, min(nq, 6))
        pids, pds, pcnt, _ = port.search_batch(metric=m, vectors=X, queries=Q[sub], limit=k, L=max(500, k), prefilter=True)
        assert_same_results(ids[sub], ds[sub], cnt[sub], pids, pds, pcnt, "bf %s %dx%d" % (m, n, d))
        assert st["n_dist"] == n * nq
        truth = exact_topk(X, Q, min(k, 10), m)
        assert recall(ids, truth, min(k, 10)) > 0.999
        ix.close()


def test_empty_and_edge_cases(vdb):
    X = gen(10, 8, 1)
    ix = vdb.Index("l2", 8, host_vectors=X, capacity=10)
    ids, ds, cnt, _ = ix.search(X[0], 5)  # zero rows mirrored
    assert cnt[0] == 0 and np.all(ids == -1) and np.all(np.isinf(ds))
    ix.sync_rows(3)
    ids, ds, cnt, _ = ix.search(X[:2], 5)  # fewer rows than limit
    assert list(cnt) == [3, 3] and ids[0, 0] == 0 and ids[1, 0] == 1 and np.all(ids[:, 3:] == -1)
    bits = np.zeros(2, np.uint8)
    bits[0] = 0b111
    ix.set_deleted(bits)  # everything deleted
    ids, ds, cnt, _ = ix.search(X[0], 5)
    assert cnt[0] == 0
    with pytest.raises(vdb.EpsError):
        ix.search(X[0], 5, filter_nodes=np.array([[29, 3, 0, 0, 0, 0, 0, -1]], np.int64))  # LIKE: out of scope (and malformed)
    ix.close()


# ---- build quality vs the reference-built graph on the same data -----------------------------------------
def test_build_quality_vs_reference_graph(vdb, golden):
    g = golden["rand2k"]
    X, Q = g["stored_l2"][:2000], g["queries_l2"]
    truth = exact_topk(X, Q, 10)
    ix = vdb.Index("l2", 32, host_vectors=X)
    ix.sync_rows(2000)
    out = {}
    for name in ("ref", "gpu"):
        if name == "ref":
            ix.set_graph(2000, g["offsets_l2"], g["nbrs_l2"].astype(np.int64), int(g["nav_l2"]))
        else:
            ix.build(2000)
        for L in (64, 500):
            ix.config(L, L)
            ids, _, _, st = ix.search(Q, 10)
            out[(name, L)] = (recall(ids, truth, 10), st["n_dist"] / len(Q))
    for L in (64, 500):
        assert out[("gpu", L)][0] >= out[("ref", L)][0] - 0.03, out
        assert out[("gpu", L)][1] <= 1.5 * out[("ref", L)][1], out
    ix.close()


# ---- device-pointer API and the shard merge (multi-GPU exchange step) -------------------------------------
def test_device_api_and_shard_merge(vdb):
    import torch
    from vectordb_b200.index import merge_shards_device
    n, d, nq, k, S = 9000, 48, 32, 10, 3
    X, Q = gen(n, d, 21), gen(nq, d, 22)
    tq = torch.from_numpy(Q).cuda()
    per = n // S
    all_ids = torch.empty((S, nq, k), dtype=torch.int64, device="cuda")
    all_d = torch.empty((S, nq, k), dtype=torch.float32, device="cuda")
    cnts = torch.empty((nq,), dtype=torch.int64, device="cuda")
    keep = []
    for s in range(S):
        ix = vdb.Index("l2", d, host_vectors=X[s * per:(s + 1) * per])
        ix.sync_rows(per)
        ix.config(500, 500, force_brute=True)
        ix.search_device(tq.data_ptr(), nq, k, all_ids[s].data_ptr(), all_d[s].data_ptr(), cnts.data_ptr())
        all_ids[s] += s * per
        keep.append(ix)
    out_i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_d = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    merge_shards_device(0, all_ids.data_ptr(), all_d.data_ptr(), S, nq, k, out_i.data_ptr(), out_d.data_ptr())
    truth = exact_topk(X, Q, k)
    assert recall(out_i.cpu().numpy(), truth, k) > 0.999
    assert torch.all(out_d[:, 1:] >= out_d[:, :-1])
    for ix in keep:
        ix.close()


# ---- exact scan on the tensor cores: coarse wgmma pass (tf32 / bf16 mirror) + fp32 re-score -------------------
def test_exact_scan_coarse_modes_match_oracle(vdb, port):
    n, d, nq, k = 60000, 96, 128, 10
    X, Q = gen(n, d, 301), gen(nq, d, 302)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.config(500, 500, force_brute=True)
    pids, pds, pcnt, _ = port.search_batch(metric="l2", vectors=X, queries=Q[:8], limit=k, L=500, prefilter=True)
    res = {}
    for mode in ("fp32", "tf32", "bf16"):
        ix.set_coarse(mode)
        ids, ds, cnt, st = ix.search(Q, k)
        assert_same_results(ids[:8], ds[:8], cnt[:8], pids, pds, pcnt, "coarse=" + mode)
        assert np.all(np.diff(ds, axis=1) >= 0)
        res[mode] = ids
    # re-scored results carry fp32-exact distances, so the three modes agree up to equal-distance swaps
    assert (res["tf32"] == res["fp32"]).mean() > 0.999 and (res["bf16"] == res["fp32"]).mean() > 0.999
    # deleted rows and a distance-free filter go through the pass bitmap inside the fused epilogue
    bits = np.zeros((n + 7) // 8, np.uint8)
    dead = res["fp32"][:, 0]
    for i in dead:
        bits[i >> 3] |= 1 << (i & 7)
    ix.set_deleted(bits)
    for mode in ("fp32", "bf16"):
        ix.set_coarse(mode)
        ids, ds, cnt, _ = ix.search(Q, k)
        assert not (set(ids.ravel().tolist()) & set(dead.tolist()))
        res["del_" + mode] = ids
    assert (res["del_bf16"] == res["del_fp32"]).mean() > 0.999
    ix.close()


def test_exact_scan_adversarial_row_order_falls_back(vdb):
    """Rows ordered so that EVERY later row beats the running thresholds: the fused candidate buffers overflow,
    which must be detected and answered by the fp32 path — never by dropping candidates."""
    n, d, nq, k = 200000, 32, 64, 10
    rng = np.random.default_rng(5)
    U = rng.standard_normal((n, d)).astype(np.float32)
    U /= np.linalg.norm(U, axis=1, keepdims=True)
    scale = np.linspace(8.0, 1.0, n, dtype=np.float32)[:, None]  # later rows are closer to the origin
    X = (U * scale).astype(np.float32)
    Q = (0.01 * rng.standard_normal((nq, d))).astype(np.float32)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.config(500, 500, force_brute=True)
    ix.set_coarse("fp32")
    want, wd, _, _ = ix.search(Q, k)
    ix.set_coarse("bf16")
    got, gd, _, _ = ix.search(Q, k)
    assert np.allclose(gd, wd, rtol=1e-5)
    assert (got == want).mean() > 0.99
    assert got.min() >= n - 5000  # the answers are the last rows
    ix.close()


def test_wide_expansion_matches_sequential_quality(vdb, port):
    """Search width 2/4/8 = the analogue of the reference's IntraQueryThreads > 1 (candidates expanded while the rows
    of earlier ones are in flight): not bit-identical to the sequential order, but the same recall, nearly the same
    answers and a bounded amount of extra work; width 1 stays deterministic."""
    n, d, nq = 20000, 64, 64
    X, Q = gen(n, d, 401, "cluster"), gen(nq, d, 402, "cluster")
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.build(n)
    ix.config(256, 256)
    truth = exact_topk(X, Q, 10)
    ix.set_search_width(1)
    base, bd, _, st1 = ix.search(Q, 10)
    r1 = recall(base, truth, 10)
    for w in (2, 4, 8):
        ix.set_search_width(w)
        ids, ds, cnt, st = ix.search(Q, 10)
        assert np.all(cnt == 10) and np.all(np.diff(ds, axis=1) >= 0)
        assert recall(ids, truth, 10) >= r1 - 0.01
        overlap = np.mean([len(set(ids[i]) & set(base[i])) / 10 for i in range(nq)])
        assert overlap > 0.9, (w, overlap)
        assert st["n_dist"] <= 1.3 * st1["n_dist"]
    ix.set_search_width(1)
    again, _, _, _ = ix.search(Q, 10)
    assert np.array_equal(again, base)
    ix.close()


def test_search_on_reference_built_graph_20k(vdb, golden_refgraph):
    """The reference's own graph (ANNGraphSegment::BuildFromVectorTable on 20 000 x 128, fixture refgraph20k) searched
    on the device: width 1 against the reference at IntraQueryThreads = 1 (ids, distances, distance-evaluation
    counts), width 4 against the reference at its default IntraQueryThreads = 4 (recall and work; that mode is racy
    in the reference itself, so ids are compared as quality)."""
    g = golden_refgraph
    n, d, nq = int(g["n"]), int(g["d"]), int(g["nq"])
    X, Q = gen(n, d, 901, "cluster"), gen(nq, d, 902, "cluster")
    truth = g["truth"]
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.set_graph(n, g["offsets"].astype(np.int64), g["nbrs"].astype(np.int64), int(g["nav"]))
    for L in (64, 200, 500):
        ix.config(L, L)
        ix.set_search_width(1)
        ids, ds, cnt, st = ix.search(Q, 10)
        want = g["T1_L%d_ids" % L].astype(np.int64)
        rate = assert_same_results(ids, ds, cnt, want, g["T1_L%d_dists" % L], np.full(nq, 10), "refgraph L=%d" % L)
        assert rate > 0.9
        ref_nd = int(g["T1_L%d_ndist" % L].sum())
        assert abs(st["n_dist"] - ref_nd) <= 0.02 * ref_nd, (L, st["n_dist"], ref_nd)
        ix.set_search_width(4)
        ids4, _, _, st4 = ix.search(Q, 10)
        assert recall(ids4, truth, 10) >= float(g["T4_L%d_recall" % L]) - 0.02
        assert st4["n_dist"] <= 1.3 * int(g["T4_L%d_ndist" % L].sum())
    ix.close()


@pytest.mark.parametrize("m", METRICS)
def test_nn_descent_build_quality(vdb, m):
    """B1: force the NN-descent branch (exact_knn_below far under n) and compare the searches on its graph with the
    searches on the exact-kNN graph of the same rows: recall within 0.05 at equal L, at most 1.5x the distance
    evaluations; the repair must not grow hubs."""
    n, d, nq = 60000, 64, 128
    X, Q = gen(n, d, 911, "cluster"), gen(nq, d, 912, "cluster")
    if m == "cosine":
        X /= np.linalg.norm(X, axis=1, keepdims=True)
        Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    truth = exact_topk(X, Q, 10, m)
    ix = vdb.Index(m, d, host_vectors=X)
    ix.sync_rows(n)
    res = {}
    for name, below in (("exact", 100000), ("nnd", 1000)):
        ix.build(n, exact_knn_below=below, knn_k=64)
        ni, off, nb, nav = ix.get_graph()
        deg = np.diff(off)
        others = np.delete(deg, nav)  # the navigation point also carries the entries of otherwise unreachable components
        assert ni == n and deg.min() >= 1 and others.max() <= 50 + 16, (name, others.max(), deg[nav])
        ix.config(200, 200)
        ix.set_search_width(1)
        ids, _, _, st = ix.search(Q, 10)
        res[name] = (recall(ids, truth, 10), st["n_dist"] / nq)
    assert res["nnd"][0] >= res["exact"][0] - 0.05, res
    assert res["nnd"][1] <= 1.5 * res["exact"][1], res
    ix.close()


def test_nn_descent_build_vs_reference_graph(vdb, golden_refgraph):
    """The device build (NN-descent forced) on the fixture's 20 000 x 128 rows against the graph the reference built
    on the same rows: recall at equal L within 0.05 of the reference's, distance evaluations at most 1.5x."""
    g = golden_refgraph
    n, d, nq = int(g["n"]), int(g["d"]), int(g["nq"])
    X, Q = gen(n, d, 901, "cluster"), gen(nq, d, 902, "cluster")
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.build(n, exact_knn_below=1000)
    ix.set_search_width(1)
    for L in (200, 500):
        ix.config(L, L)
        ids, _, _, st = ix.search(Q, 10)
        assert recall(ids, g["truth"], 10) >= float(g["T1_L%d_recall" % L]) - 0.05, L
        assert st["n_dist"] <= 1.5 * int(g["T1_L%d_ndist" % L].sum()), L
    ix.close()


def test_build_repair_does_not_grow_hubs(vdb):
    """B2 connectivity repair (nsg.cpp:734-775: nearest linked vertex of a search pool, else a random linked one) on
    the case that used to produce one vertex of degree O(n): an inner-product field over positive data."""
    n, d = 200000, 32
    X = gen(n, d, 921)
    ix = vdb.Index("ip", d, host_vectors=X)
    ix.sync_rows(n)
    ix.build(n, knn_k=64, nnd_iters=8)
    ni, off, nb, nav = ix.get_graph()
    deg = np.diff(off)
    assert np.delete(deg, nav).max() <= 50 + 16, (np.delete(deg, nav).max(), deg[nav])
    # every vertex reachable from the navigation point
    seen = np.zeros(n, bool)
    seen[nav] = True
    frontier = np.array([nav])
    while len(frontier):
        nxt = np.unique(np.concatenate([nb[off[v]:off[v + 1]] for v in frontier])) if len(frontier) < 50000 else \
            np.unique(nb[np.concatenate([np.arange(off[v], off[v + 1]) for v in frontier])])
        nxt = nxt[~seen[nxt]]
        seen[nxt] = True
        frontier = nxt
    assert seen.all()
    ix.close()


def test_large_batch_top100_with_filter(vdb, port):
    """Config C3 shape at test scale: batch > 1024 (grouped through the tensor-core pass), top-100, INT4 metadata
    filter 'attr < 10' (10 % selectivity) evaluated on device, both as exact scan and as graph post-filter."""
    n, d, nq, k = 50000, 64, 1536, 100
    X, Q = gen(n, d, 501), gen(nq, d, 502)
    attr = (np.arange(n) % 100).astype(np.int32)
    nodes = np.array([[7, 1, -1, -1, 0, 0, 0, 0],      # Int4Attr at offset 0
                      [1, 1, -1, -1, 10, 0, 0, -1],    # IntConst 10
                      [19, 3, 0, 1, 0, 0, 0, -1]],     # LT
                     np.int64)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.set_attrs(attr.view(np.uint8), 4, n)
    ix.config(500, 500, force_brute=True)
    ix.set_coarse("bf16")
    ids, ds, cnt, _ = ix.search(Q, k, filter_nodes=nodes)
    assert np.all(cnt == k) and np.all(attr[ids] < 10)
    sub = [0, 700, 1100, 1535]
    pids, pds, pcnt, _ = port.search_batch(metric="l2", vectors=X, queries=Q[sub], limit=k, L=500, prefilter=True,
                                           attrs=attr.view(np.uint8), attr_stride=4, filter_nodes=nodes)
    assert_same_results(ids[sub], ds[sub], cnt[sub], pids, pds, pcnt, "C3 exact scan + filter")
    ix.config(500, 500, force_brute=False)
    ix.build(n)
    gids, gds, gcnt, _ = ix.search(Q[:64], k, filter_nodes=nodes)  # post-filter: only the best L are considered
    assert np.all(gcnt <= k) and np.all(attr[gids[gids >= 0]] < 10)
    ix.close()


# ---- row shards with the exchange inside the library (NCCL bound at run time) -----------------------------------
def test_sharded_search_single_rank_group(vdb):
    """eps_search_batch_sharded with a world of one rank (all a 1-GPU box can form): local search -> global ids ->
    ncclAllGather -> merge kernel must equal the plain search shifted by id_base."""
    import torch
    from vectordb_b200.sharded import ShardGroup
    n, d, nq, k, base = 30000, 48, 64, 10, 1_000_000
    X, Q = gen(n, d, 31), gen(nq, d, 32)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.config(500, 500, force_brute=True)
    want, wd, _, _ = ix.search(Q, k)
    g = ShardGroup(ShardGroup.unique_id(), 0, 1, 0)
    tq = torch.from_numpy(Q).cuda()
    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    g.search(ix, base, tq.data_ptr(), nq, k, oi.data_ptr(), od.data_ptr())
    assert np.array_equal(oi.cpu().numpy(), want + base)
    assert np.allclose(od.cpu().numpy(), wd, rtol=1e-6)
    g.close()
    ix.close()


def _shard_worker(rank, world, uid_path, out_path):
    import os
    import time
    import numpy as np
    import torch
    import vectordb_b200
    from helpers import gen
    from vectordb_b200.sharded import ShardGroup, shard_range
    torch.cuda.set_device(rank)
    if rank == 0:
        with open(uid_path + ".tmp", "wb") as f:
            f.write(ShardGroup.unique_id())
        os.replace(uid_path + ".tmp", uid_path)
    while not os.path.exists(uid_path):
        time.sleep(0.05)
    uid = open(uid_path, "rb").read()
    n, d, nq, k = 40000, 48, 64, 10
    X, Q = gen(n, d, 41), gen(nq, d, 42)
    lo, hi = shard_range(n, rank, world)
    ix = vectordb_b200.Index("l2", d, host_vectors=X[lo:hi], device=rank)
    ix.sync_rows(hi - lo)
    ix.config(500, 500, force_brute=True)
    g = ShardGroup(uid, rank, world, rank)
    tq = torch.from_numpy(Q).cuda()
    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    g.search(ix, lo, tq.data_ptr(), nq, k, oi.data_ptr(), od.data_ptr())
    np.savez(out_path % rank, ids=oi.cpu().numpy(), dists=od.cpu().numpy())
    g.close()
    ix.close()


def test_sharded_search_two_ranks(vdb, tmp_path):
    """World of two ranks on two GPUs (skipped on a 1-GPU box): merged results on both ranks equal the exact top-k
    of the whole table."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    uid_path, out_path = str(tmp_path / "uid.bin"), str(tmp_path / "out%d.npz")
    mp.spawn(_shard_worker, args=(2, uid_path, out_path), nprocs=2, join=True)
    X, Q = gen(40000, 48, 41), gen(64, 48, 42)
    truth = exact_topk(X, Q, 10)
    for r in range(2):
        got = np.load(out_path % r)
        assert recall(got["ids"], truth, 10) > 0.999
        assert np.all(np.diff(got["dists"], axis=1) >= 0)
    assert np.array_equal(np.load(out_path % 0)["ids"], np.load(out_path % 1)["ids"])


def test_string_codes_filter_through_c_abi(vdb):
    """f4 at the C ABI: dictionary-coded string column + StringAttr / StringConst / EQ / NE / OR nodes."""
    n, d, nq, k = 20000, 32, 16, 10
    X, Q = gen(n, d, 81), gen(nq, d, 82)
    codes = (np.arange(n) % 7).astype(np.int32)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.config(500, 500, force_brute=True)
    ix.set_string_codes(0, 0, codes[:12000])
    ix.set_string_codes(0, 12000, codes[12000:])   # appended rows
    S_ATTR, S_CONST, EQ, NE, OR = 9, 2, 21, 24, 26
    def prog(op, lits):
        nodes = [[S_ATTR, 0, -1, -1, 0, 0, 0, 0]]
        acc = None
        for c in lits:
            nodes.append([S_CONST, 0, -1, -1, c, 0, 0, -1])
            nodes.append([op, 3, 0, len(nodes) - 1, 0, 0, 0, -1])
            if acc is not None:
                nodes.append([OR, 3, acc, len(nodes) - 1, 0, 0, 0, -1])
            acc = len(nodes) - 1
        return np.array(nodes, np.int64)
    for op, lits, keep in ((EQ, [3], codes == 3), (NE, [3], codes != 3), (EQ, [1, 5, -1], np.isin(codes, [1, 5]))):
        ids, ds, cnt, _ = ix.search(Q, k, filter_nodes=prog(op, lits))
        rows = np.nonzero(keep)[0]
        want = rows[exact_topk(X[rows], Q, k)]
        assert np.all(cnt == k) and recall(ids, want, k) == 1.0
    with pytest.raises(Exception):   # a column that is not mirrored for every row must be refused, not read out of bounds
        ix.search(Q, k, filter_nodes=np.array([[S_ATTR, 0, -1, -1, 0, 0, 0, 1], [S_CONST, 0, -1, -1, 0, 0, 0, -1], [EQ, 3, 0, 1, 0, 0, 0, -1]], np.int64))
    ix.close()


def test_facets_match_reference(vdb):
    """f4: FacetExecutor::Aggregate on the device (eps_facet_batch) against the reference's own FacetExecutor on the
    same result lists (fixture facets: the reference's attribute table, parsed expressions and JSON answers): int /
    double / bool / string keys, SUM / COUNT / MIN / MAX, '@distance' inside an aggregate."""
    import json
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "facets.npz"), allow_pickle=False)
    n, d, nq, k = 4000, 16, 12, 64
    X, Q = gen(n, d, 111), gen(nq, d, 112)
    rng = np.random.default_rng(113)
    rng.random(n), rng.integers(0, 2, n)  # the ID / w / flag columns, already in the fixture's attribute table
    names = ["n%d" % v for v in rng.integers(0, 9, n)]
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.set_attrs(g["attrs"], int(g["stride"]), n)
    dictionary = {s: i for i, s in enumerate(sorted(set(names)))}
    back = {i: s for s, i in dictionary.items()}
    ix.set_string_codes(int(g["name_offset"]), 0, np.array([dictionary[s] for s in names], np.int32))
    ix.config(500, 500, force_brute=True)
    sids, sds, scnt, _ = ix.search(Q, k)
    assert_same_results(sids, sds, scnt, g["ids"], g["dists"], g["counts"], "facet result lists")
    ids, ds, cnt = g["ids"], g["dists"].astype(np.float32), g["counts"]   # the lists the reference aggregated
    AGG = {"SUM": 30, "MIN": 31, "MAX": 32, "COUNT": 33}
    cases = [("ID % 7", ["SUM(w)", "COUNT(*)", "MIN(ID)", "MAX(w * 2 + @distance)"]), ("name", ["COUNT(*)", "SUM(ID)"]),
             ("flag", ["COUNT(*)", "MAX(@distance)"]), ("w * 2", ["COUNT(*)"]), ("", ["COUNT(*)", "SUM(w)", "MIN(@distance)"])]
    for ci, (group, aggs) in enumerate(cases):
        knodes, ktype = g["key_nodes_%d" % ci], int(g["key_type_%d" % ci])
        alist = [(AGG[a[:a.index("(")].upper()], g["agg_nodes_%d_%d" % (ci, ai)]) for ai, a in enumerate(aggs)]
        got = ix.facet(ids, cnt, knodes, ktype, alist, dists=ds)
        want_all = json.loads(str(g["want_%d" % ci]))
        for q in range(nq):
            want = want_all[q]
            assert len(got[q]) == len(want), (group, q)
            wmap = {}
            for obj in want:
                key = obj.get(group, 1) if group else 1
                wmap[key] = [obj[a] for a in aggs]
            for key, vals in got[q]:
                kk = back[int(key)] if ktype == 0 else (bool(key) if ktype == 3 else (int(key) if ktype == 1 else key))
                if ktype == 2:
                    kk = min(wmap, key=lambda x: abs(x - key))
                    assert abs(kk - key) <= 1e-12 * max(1.0, abs(key))
                ref_vals = wmap[kk]
                for v, w in zip(vals, ref_vals):
                    assert abs(v - w) <= 1e-9 * max(1.0, abs(w)) or (isinstance(w, int) and int(v) == w), (group, q, kk, vals, ref_vals)
    ix.close()


def test_exact_scan_guard_catches_a_coarse_pass_that_cannot_rank(vdb):
    """Weak point 1 of round 1: exactness of the tensor-core scan must be enforced, not hoped for.  300 rows of an
    ordinary table form a bundle around the queries whose members differ by far less than a bf16 rounding step: the
    coarse pass ranks the bundle ahead of everything else but cannot rank INSIDE it, so a 128-entry candidate list holds
    a random subset of it.  The guard (exact k-th best + 2 x the batch's largest observed coarse error must not exceed
    the coarse k'-th threshold) has to notice and the answer must be the fp32 scan's.  On ordinary data it stays silent."""
    n, d, nq, k = 100000, 64, 128, 10
    rng = np.random.default_rng(7)
    X = gen(n, d, 6)
    centre = rng.random(d, dtype=np.float32)
    where = rng.choice(n, 300, replace=False)
    X[where] = (centre[None, :] + 1e-3 * rng.standard_normal((300, d))).astype(np.float32)
    Q = (centre[None, :] + 1e-3 * rng.standard_normal((nq, d))).astype(np.float32)
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.config(500, 500, force_brute=True)
    ix.set_coarse("fp32")
    want, wd, _, _ = ix.search(Q, k)
    assert np.isin(want, where).all()
    for mode in ("bf16", "tf32"):
        ix.set_coarse(mode)
        got, gd, _, st = ix.search(Q, k)
        assert np.allclose(gd, wd, rtol=1e-5) and (got == want).mean() > 0.999, mode
        if mode == "bf16":
            assert st["n_redone"] > 0
    ix.set_coarse_guard(False)                    # the unguarded pass really is wrong here: the test has teeth
    ix.set_coarse("bf16")                         # (set_coarse to another mode and back resets the learnt k')
    raw, _, _, st0 = ix.search(Q, k)
    assert st0["n_redone"] == 0 and (raw == want).mean() < 0.9
    ix.close()
    X2, Q2 = gen(200000, d, 8), gen(nq, d, 9)
    ix = vdb.Index("l2", d, host_vectors=X2)
    ix.sync_rows(200000)
    ix.config(500, 500, force_brute=True)
    ix.set_coarse("fp32")
    want, _, _, _ = ix.search(Q2, k)
    ix.set_coarse("bf16")
    got, _, _, st = ix.search(Q2, k)
    assert st["n_redone"] == 0 and (got == want).mean() > 0.999
    ix.close()


def test_views_search_concurrently_and_freeze_the_base(vdb):
    """eps_index_create_view: a view answers exactly like its base (exact mode, width 1), batches issued to the base and
    to the view without synchronisation overlap and still give the same answers, and the base refuses modifications
    while the view lives."""
    import torch
    rng = np.random.default_rng(11)
    n, dim, nq, k = 6000, 64, 256, 10
    X = rng.standard_normal((n, dim)).astype(np.float32)
    Q = rng.standard_normal((nq, dim)).astype(np.float32)
    ix = vdb.Index("l2", dim, host_vectors=X)
    ix.sync_rows(n)
    ix.build(n, knn_k=32, out_degree=24)
    ix.config(64, 64)
    ix.set_search_width(1)
    want_ids, want_d, want_c, _ = ix.search(Q, k)
    v = ix.view()
    got_ids, got_d, got_c, _ = v.search(Q, k)
    assert np.array_equal(want_ids, got_ids) and np.array_equal(want_c, got_c) and np.allclose(want_d, got_d, rtol=1e-6)
    # asynchronous, interleaved batches on the two handles
    dev = torch.device("cuda", 0)
    dq = torch.from_numpy(Q).to(dev)
    outs = []
    for h in (ix, v, ix, v):
        oi = torch.empty((nq, k), dtype=torch.int64, device=dev); od = torch.empty((nq, k), dtype=torch.float32, device=dev)
        oc = torch.empty((nq,), dtype=torch.int64, device=dev)
        h.search_device(dq.data_ptr(), nq, k, oi.data_ptr(), od.data_ptr(), oc.data_ptr(), sync=False)
        outs.append((h, oi))
    for h, oi in outs:
        torch.cuda.ExternalStream(h.stream, device=dev).synchronize()
        assert np.array_equal(oi.cpu().numpy(), want_ids)
    # frozen base, read-only view
    for call in (lambda: ix.sync_rows(n), lambda: ix.build(n), lambda: ix.set_deleted(np.zeros(n // 8 + 1, np.uint8)),
                 lambda: v.set_deleted(np.zeros(n // 8 + 1, np.uint8)), lambda: v.build(n)):
        with pytest.raises(vdb.EpsError):
            call()
    v.close()
    ix.set_deleted(np.zeros(n // 8 + 1, np.uint8))  # thawed
    # a base destroyed before its view leaves an empty index behind, not a dangling one
    v2 = ix.view()
    ix.close()
    _, _, c2, _ = v2.search(Q[:4], k)
    assert (c2 == 0).all()
    v2.close()
