"""The graph kernel keeps each query's visited ids in a hash set of next_pow2(16 L) entries (clamped to
[1024, 16384]) and moves a query to a bitmap once the set would pass 3/4 full.  A case whose queries visit more ids
than that must give the oracle's results and leave both structures clean for the next search."""
import numpy as np
import pytest

from helpers import assert_same_results, gen

pytestmark = pytest.mark.gpu


def test_queries_that_outgrow_the_visited_hash_set(port):
    import vectordb_b200 as vdb
    assert vdb.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    n, d, nq = 20000, 64, 48
    X, Q = gen(n, d, 101), gen(nq, d, 102)  # iid uniform: a search visits many more rows per queue slot than on clusters
    ix = vdb.Index("l2", d, host_vectors=X)
    ix.sync_rows(n)
    ix.build(n)
    ni, off, nb, nav = ix.get_graph()
    L, limit = 64, 10
    cap = min(16384, max(1024, 1 << (16 * L - 1).bit_length()))
    ix.config(L, L)
    ids, ds, cnt, st = ix.search(Q, limit)
    # the mean query evaluates more rows than the set may hold: at least one query moved to the bitmap
    assert st["n_dist"] / nq > 0.75 * cap, "n_dist per query %.0f does not exceed 3/4 of %d" % (st["n_dist"] / nq, cap)
    pids, pds, pcnt, pst = port.search_batch(metric="l2", vectors=X, queries=Q, limit=limit, n_indexed=n, offsets=off,
                                             nbrs=nb, nav=nav, L=L)
    assert assert_same_results(ids, ds, cnt, pids, pds, pcnt, "L=%d" % L) > 0.9
    assert abs(st["n_dist"] - pst[0]) <= 0.01 * pst[0]
    assert abs(st["n_expand"] - pst[1]) <= 0.01 * pst[1]
    # a search left behind a stale hash entry or bitmap bit would skip that id now
    ids2, ds2, cnt2, st2 = ix.search(Q, limit)
    assert np.array_equal(ids, ids2) and np.array_equal(ds, ds2) and np.array_equal(cnt, cnt2)
    assert st2["n_dist"] == st["n_dist"] and st2["n_edges"] == st["n_edges"]
    ix.close()
