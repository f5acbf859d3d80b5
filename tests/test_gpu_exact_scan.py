"""Exactness of the exact scan on every dispatch path (run with -m gpu on an H100).

Every case searches through vectordb_b200.Index and is judged by tests/exact_ref.check_exact: float64 distances from
the fp32 inputs, a per-pair fp32 summation bound, no misses.  The shapes sit on the edges of the dispatch in
brute_force.cu / tc_dist.cu: the row kernel (nq <= 16), the SIMT tiles, row splits, SIMT chunks, the wgmma boot chunk
and fused launches (nq 64..1024, n >= 4096), the k' caps, 1024-query groups, the graph branch's tail scan, the
incremental mirrors and the filters of the fused epilogue.  Every table is drawn from a seed."""
import numpy as np
import pytest

import exact_ref as er

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200
    L = vectordb_b200.load_library()
    assert L.eps_device_count() > 0, "GPU tests need a CUDA device"
    return vectordb_b200


def _data(n, d, nq, seed, metric="l2", kind="uniform"):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        X, Q = rng.random((n, d), dtype=np.float32), rng.random((nq, d), dtype=np.float32)
    else:  # mixed signs
        X, Q = rng.standard_normal((n, d)).astype(np.float32), rng.standard_normal((nq, d)).astype(np.float32)
    if metric == "cosine":
        X /= np.linalg.norm(X, axis=1, keepdims=True)
        Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    return X, Q


def _index(vdb, metric, X, coarse="tf32", capacity=None):
    ix = vdb.Index(metric, X.shape[1], host_vectors=X, capacity=capacity)
    ix.sync_rows(X.shape[0])
    ix.config(500, 500, force_brute=True)
    ix.set_coarse(coarse)
    return ix


def _search(ix, X, Q, metric, k, admissible=None, what="", filter_nodes=None, n_rows=None):
    ids, ds, cnt, st = ix.search(Q, k, filter_nodes=filter_nodes)
    er.check_exact(ids, ds, cnt, X, Q, metric, k, admissible=admissible, what=what)
    assert st["n_dist"] == Q.shape[0] * (X.shape[0] if n_rows is None else n_rows), what
    return ids, ds, st


# ---- row kernel (nq <= 16) and SIMT tiles ---------------------------------------------------------------------------
@pytest.mark.parametrize("nq,d,n", [(1, 3, 5000), (7, 4, 5000), (16, 128, 5000), (7, 8192, 3000), (16, 8192, 1000)])
def test_row_kernel(vdb, nq, d, n):
    """d = 8192: at most 6 queries fit the kernel's shared memory (> 48 KB), so 16 queries take 3 launches."""
    X, Q = _data(n, d, nq, 10 + d)
    ix = _index(vdb, "l2", X)
    _search(ix, X, Q, "l2", 10, what="rows l2")
    ix.close()
    ix = _index(vdb, "ip", X)
    _search(ix, X, Q, "ip", 10, what="rows ip")
    ix.close()


@pytest.mark.parametrize("nq,d,n,metric", [(17, 1, 127, "l2"), (17, 15, 129, "ip"), (129, 17, 4095, "l2"),
                                           (129, 33, 129, "cosine"), (17, 768, 4095, "ip"), (129, 768, 4095, "l2")])
def test_simt_tiles(vdb, nq, d, n, metric):
    X, Q = _data(n, d, nq, 20 + d, metric)
    ix = _index(vdb, metric, X, coarse="fp32")
    _search(ix, X, Q, metric, 10, what="tiles")
    ix.close()


@pytest.mark.parametrize("nq,k", [(1, 1), (3, 100), (1, 8192), (3, 8192)])
def test_row_splits(vdb, nq, k):
    X, Q = _data(1_000_000, 32, nq, 30)
    ix = _index(vdb, "l2", X)
    ix.config(8192, 8192, force_brute=True)
    _search(ix, X, Q, "l2", k, what="splits k=%d" % k)
    ix.close()


def test_simt_chunks(vdb):
    """fp32 mode, nq * n > 2^28: two distance chunks, the second ragged."""
    X, Q = _data(270_000, 32, 1024, 40, "ip", kind="normal")
    ix = _index(vdb, "ip", X, coarse="fp32")
    _search(ix, X, Q, "ip", 10, what="chunks")
    ix.close()


# ---- wgmma coarse pass + re-score + guard ---------------------------------------------------------------------------
WGMMA = [("l2", "tf32", 32, 64, 4096), ("ip", "tf32", 36, 257, 4097), ("cosine", "bf16", 40, 256, 36865),
         ("l2", "bf16", 96, 255, 36865), ("ip", "tf32", 96, 1024, 36865), ("cosine", "tf32", 768, 64, 36865),
         ("l2", "bf16", 768, 256, 4097), ("ip", "bf16", 32, 256, 300_000)]


@pytest.mark.parametrize("metric,coarse,d,nq,n", WGMMA)
def test_wgmma(vdb, metric, coarse, d, nq, n):
    """n = 36865: the 4096-row boot chunk, one fused launch of 32768 rows, then a launch of one row.  d = 36 / 40 are
    not multiples of the 32 (tf32) / 64 (bf16) element k-block: TMA fills the missing columns with zeros."""
    X, Q = _data(n, d, nq, 50 + d + nq, metric, kind="normal" if metric == "ip" else "uniform")
    ix = _index(vdb, metric, X, coarse=coarse)
    _, _, st = _search(ix, X, Q, metric, 10, what="wgmma %s %s" % (metric, coarse))
    assert st["n_redone"] == 0, st  # ordinary data: the answer is the coarse pass's, not an fp32 redo
    ix.close()


@pytest.mark.parametrize("k", [1, 129, 1000, 4096, 8192])
def test_wgmma_k_edges(vdb, k):
    """k' = k + max(118, k), capped at 8192: at k = 4096 and 8192 the guard cannot pass and the per-query fp32 redo
    (gather / scatter of the unsafe queries) answers."""
    X, Q = _data(50_000, 32, 64, 60, "l2")
    ix = _index(vdb, "l2", X, coarse="bf16")
    ix.config(8192, 8192, force_brute=True)
    _, _, st = _search(ix, X, Q, "l2", k, what="k=%d" % k)
    if k == 8192:
        assert st["n_redone"] == 64
    ix.close()


def test_guard_boost_is_remembered_and_reset(vdb):
    """A bundle of 6000 rows closer together than a bf16 step, k = 1000 (k' = 2000): the guard flags most of the batch
    and the index learns a 4x larger k'; the next search with the learnt k' is exact too, and set_coarse away and back
    forgets it."""
    n, d, nq, k = 100_000, 64, 128, 1000
    rng = np.random.default_rng(7)
    X = rng.random((n, d), dtype=np.float32)
    centre = rng.random(d, dtype=np.float32)
    X[rng.choice(n, 6000, replace=False)] = centre[None, :] + 1e-3 * rng.standard_normal((6000, d)).astype(np.float32)
    Q = (centre[None, :] + 1e-3 * rng.standard_normal((nq, d))).astype(np.float32)
    ix = _index(vdb, "l2", X, coarse="bf16")
    ix.config(1000, 1000, force_brute=True)
    _, _, st = _search(ix, X, Q, "l2", k, what="boost 1")
    assert st["n_redone"] >= nq
    _search(ix, X, Q, "l2", k, what="boost learnt")
    ix.set_coarse("fp32")
    ix.set_coarse("bf16")
    _search(ix, X, Q, "l2", k, what="boost reset")
    ix.close()


@pytest.mark.parametrize("nq", [1025, 1088, 2100])
def test_query_groups(vdb, nq):
    """Batches above 1024 go through the wgmma pass in groups of 1024: a remainder of 1 (row kernel), 64 (wgmma) and
    52 (SIMT tiles)."""
    X, Q = _data(8192, 32, nq, 70 + nq)
    ix = _index(vdb, "l2", X, coarse="tf32")
    _search(ix, X, Q, "l2", 10, what="groups")
    ix.close()


# ---- graph branch: the tail rows are scanned with row_start > 0 ----------------------------------------------------
def test_graph_tail_on_wgmma_path(vdb):
    n0, nt, d, nq, k = 20_000, 8192, 32, 128, 10
    rng = np.random.default_rng(80)
    base = rng.random((n0, d), dtype=np.float32)
    centres = 3.0 + rng.random((nt // 16, d), dtype=np.float32)        # far from every indexed row
    tail = (np.repeat(centres, 16, axis=0) + 1e-2 * rng.standard_normal((nt, d))).astype(np.float32)
    X = np.concatenate([base, tail])
    Q = (centres[rng.choice(len(centres), nq, replace=False)] + 1e-2 * rng.standard_normal((nq, d))).astype(np.float32)
    ix = vdb.Index("l2", d, host_vectors=X, capacity=len(X))
    ix.sync_rows(n0)
    ix.build(n0)
    ix.sync_rows(len(X))
    ix.config(64, 64)
    out = {}
    for mode in ("tf32", "bf16", "fp32"):
        ix.set_coarse(mode)
        ids, ds, cnt, _ = ix.search(Q, k)
        er.check_exact(ids, ds, cnt, X, Q, "l2", k, what="tail " + mode)
        assert ids.min() >= n0
        out[mode] = (ids, ds)
    for mode in ("tf32", "bf16"):
        assert np.array_equal(out[mode][0], out["fp32"][0]), mode
    ix.close()


# ---- incremental mirrors (|x|^2, bf16 copy) ------------------------------------------------------------------------
@pytest.mark.parametrize("coarse", ["tf32", "bf16"])
def test_mirrors_follow_appends_adoption_and_views(vdb, coarse):
    import torch
    n, extra, d, nq, k = 40_000, 5000, 64, 128, 10
    rng = np.random.default_rng(90)
    X = rng.random((n + extra, d), dtype=np.float32)
    Q = rng.random((nq, d), dtype=np.float32)
    X[n:n + nq] = Q + 1e-3                                    # the appended rows hold the true neighbours
    ix = vdb.Index("l2", d, host_vectors=X, capacity=n + extra)
    ix.sync_rows(n)
    ix.config(500, 500, force_brute=True)
    ix.set_coarse(coarse)
    _search(ix, X[:n], Q, "l2", k, what="before append")
    ix.sync_rows(n + extra)
    ids, _, _ = _search(ix, X, Q, "l2", k, what="after append")
    assert np.array_equal(ids[:, 0], np.arange(n, n + nq))
    Y = np.ascontiguousarray(X[::-1])                            # a new device table: the mirrors must be rebuilt
    T = torch.from_numpy(Y).cuda()
    torch.cuda.synchronize()
    ix.adopt_device_rows(T.data_ptr(), len(Y))
    _search(ix, Y, Q, "l2", k, what="adopted")
    v = ix.view()
    _search(v, Y, Q, "l2", k, what="view")
    _search(ix, Y, Q, "l2", k, what="base beside view")
    v.close()
    ix.close()
    del T


# ---- filters inside the fused epilogue -----------------------------------------------------------------------------
LT = 19


def _attr_lt(limit):
    return np.array([[7, 1, -1, -1, 0, 0, 0, 0], [1, 1, -1, -1, limit, 0, 0, -1], [LT, 3, 0, 1, 0, 0, 0, -1]], np.int64)


def test_deleted_boot_chunk_overflows_to_fp32(vdb):
    """Rows [0, 4096) deleted: the boot chunk leaves every threshold at +inf, the fused launches overflow the candidate
    buffers and the whole batch is redone on the fp32 path."""
    X, Q = _data(60_000, 32, 64, 100)
    ix = _index(vdb, "l2", X, coarse="bf16")
    bits = np.zeros((len(X) + 7) // 8, np.uint8)
    bits[:4096 // 8] = 0xFF
    ix.set_deleted(bits)
    ok = np.ones(len(X), bool)
    ok[:4096] = False
    _, _, st = _search(ix, X, Q, "l2", 10, admissible=ok, what="deleted")
    assert st["n_redone"] == 64
    ix.close()


@pytest.mark.parametrize("prefilter", [False, True])
def test_sparse_static_filter(vdb, prefilter):
    """attr < 3 of 100: 3 % of the rows pass, so the boot chunk keeps fewer than k' of them (thresholds +inf) but the
    fused launches stay within the candidate buffers."""
    X, Q = _data(60_000, 32, 64, 110)
    attr = (np.arange(len(X)) % 100).astype(np.int32)
    ix = _index(vdb, "l2", X, coarse="tf32")
    ix.set_attrs(attr.view(np.uint8), 4, len(X))
    ix.config(500, 500, prefilter=prefilter, force_brute=True)
    _search(ix, X, Q, "l2", 10, admissible=attr < 3, filter_nodes=_attr_lt(3), what="filter")
    ix.close()


# ---- values ---------------------------------------------------------------------------------------------------------
def test_duplicates_tie_by_id_across_fused_launches(vdb):
    X, Q = _data(100_000, 32, 64, 120)
    rng = np.random.default_rng(121)
    where = np.sort(rng.choice(len(X), 500, replace=False))
    X[where] = X[where[0]]
    Q[:] = X[where[0]] + 1e-4 * rng.standard_normal((64, 32)).astype(np.float32)
    for coarse in ("tf32", "bf16"):
        ix = _index(vdb, "l2", X, coarse=coarse)
        ids, _, _ = _search(ix, X, Q, "l2", 10, what="duplicates")
        assert np.all(ids == where[:10][None, :])
        ix.close()


def test_zero_query_ip(vdb):
    """Every distance of an all-zero IP query is 0: the answer is ids 0..k-1."""
    X, Q = _data(20_000, 32, 64, 130, "ip", kind="normal")
    Q[5] = 0
    ix = _index(vdb, "ip", X, coarse="bf16")
    ids, ds, _ = _search(ix, X, Q, "ip", 10, what="zero query")
    assert np.array_equal(ids[5], np.arange(10)) and np.all(ds[5] == 0)
    ix.close()


@pytest.mark.parametrize("coarse", ["tf32", "bf16"])
def test_l2_large_offset_cancellation(vdb, coarse):
    rng = np.random.default_rng(140)
    X = (1000.0 + 1e-2 * rng.standard_normal((50_000, 32))).astype(np.float32)
    Q = (1000.0 + 1e-2 * rng.standard_normal((64, 32))).astype(np.float32)
    ix = _index(vdb, "l2", X, coarse=coarse)
    _search(ix, X, Q, "l2", 10, what="offset")
    ix.close()


# ---- the guard and large-norm rows ----------------------------------------------------------------------------------
@pytest.mark.parametrize("coarse", ["bf16", "tf32"])
def test_guard_catches_a_large_norm_row(vdb, coarse):
    """A row of norm ~10^4 among unit rows is the exact top-1 of the batch's query, but rounding its components to
    bf16 / tf32 drops its coarse dot far below the candidate list, and the errors sampled from the (unit-norm)
    re-scored rows cannot see it (tests/test_exact_ref.py shows both in a host model).  The guard scales the sampled
    error by the norm ratio, so the answer is exact; without the guard the row is missing."""
    X, Q, p = er.planted_ip_table()
    ix = _index(vdb, "ip", X, coarse=coarse)
    ids, _, st = _search(ix, X, Q, "ip", 10, what="planted " + coarse)
    assert np.all(ids[:, 0] == p) and st["n_redone"] > 0
    ix.set_coarse_guard(False)
    ix.set_coarse("fp32")                 # forget the k' the guard learnt on this table
    ix.set_coarse(coarse)
    raw, _, _, st0 = ix.search(Q, 10)
    assert st0["n_redone"] == 0 and not np.any(raw == p)
    ix.close()
