"""Bit-exact CPU model of the graph search of a sparse-vector field: the oracle port (oracle_port.c, the pinned
restatement of VecSearchExecutor::Search at IntraQueryThreads = 1) fed with a precomputed distance table.

The port only ever sees a distance through its dense distance function, so each query is given to it as a
1-dimensional inner-product table: row r holds -D[q, r] and the query is 1.0, and the port's -(0 + (-D[q, r]) * 1) is
D[q, r] exactly (a zero comes back as -0.0, which no comparison tells from +0.0).  Init ids, search, tail scan, merge,
post-filter and counters are the port's own.  The returned distances are looked up in D.  With D from the numpy fp32
restatement of vector.cpp (test_gpu_sparse.ref_distances) this reproduces the reference's sparse Search."""
import numpy as np


def port_model(port, D, graph, L, limit, deleted=None, attrs=None, stride=0, nodes=None):
    """Search of every query with distance table D [nq x total] over graph = (n_indexed, offsets, nbrs, nav) at queue
    length L (= L_local).  Returns ids [nq x limit] (-1 padded), dists float64 (inf padded), counts, and per query
    the distance evaluations and expansions."""
    n_indexed, off, nb, nav = graph
    nq, total = D.shape
    ids = np.full((nq, limit), -1, np.int64)
    ds = np.full((nq, limit), np.inf, np.float64)
    cnt = np.zeros(nq, np.int64)
    n_dist = np.zeros(nq, np.int64)
    n_expand = np.zeros(nq, np.int64)
    one = np.ones((1, 1), np.float32)
    for q in range(nq):
        table = np.ascontiguousarray(-D[q], np.float32)[:, None]
        i, _, c, (a, b) = port.search_batch(metric="ip", vectors=table, queries=one, limit=limit, total_rows=total,
                                            n_indexed=n_indexed, offsets=off, nbrs=nb, nav=nav, deleted=deleted,
                                            attrs=attrs, attr_stride=stride, filter_nodes=nodes, L=L)
        k = int(c[0])
        ids[q], cnt[q] = i[0], k
        ds[q, :k] = D[q, i[0, :k]]
        n_dist[q], n_expand[q] = a, b
    return ids, ds, cnt, n_dist, n_expand
