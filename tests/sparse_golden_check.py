"""Comparison of sparse search results with tests/golden/sparse.npz (the reference's own Search answers,
tests/golden/make_sparse_golden.py).  L2 and IP: ids identical and distances bitwise equal (+0 / -0 folded).
Cosine: the golden table has no empty rows, so only the empty query gives NaN (against every row); for it the
reference's std::sort order is unspecified (NaN breaks its strict weak ordering) and only the count is compared."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sparse.npz")


def check_against_golden(g, key, ids, dists, counts, metric):
    wi, wd, wc = g[key + "_ids"].astype(np.int64), g[key + "_dists"].astype(np.float32), g[key + "_counts"]
    gd = np.asarray(dists, np.float64).astype(np.float32)
    for q in range(wi.shape[0]):
        n = int(wc[q])
        assert int(counts[q]) == n, "%s query %d: count %d != %d" % (key, q, counts[q], n)
        if metric == 2 and np.isnan(wd[q, :n]).all():
            assert np.isnan(gd[q, :n]).all(), "%s query %d: expected NaN distances" % (key, q)
            continue
        a_i, a_d, b_i, b_d = ids[q, :n], gd[q, :n], wi[q, :n], wd[q, :n]
        assert np.array_equal(a_i, b_i), "%s query %d: ids %s != %s" % (key, q, a_i, b_i)
        assert np.array_equal((a_d + np.float32(0)).view(np.uint32), (b_d + np.float32(0)).view(np.uint32)), \
            "%s query %d: distances are not bitwise equal" % (key, q)
