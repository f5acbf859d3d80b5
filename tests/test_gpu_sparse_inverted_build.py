"""The sparse graph build reads its kNN distances from the posting lists when the index has them (IP / cosine).

The postings produce bitwise the exact scan's distance tile, so the graph (offsets, neighbours, navigation point) must be
identical to the one built without postings, whether the postings cover every row, part of the rows (the rest comes from
the merge) or more rows than the build indexes; and the build leaves the postings as they were."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_sparse import sparse_rows  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vdb():
    import vectordb_b200
    assert vectordb_b200.load_library().eps_device_count() > 0, "GPU tests need a CUDA device"
    return vectordb_b200


def same_graph(got, want, what):
    for name, a, b in zip(("n_indexed", "offsets", "neighbours", "nav"), got, want):
        assert np.array_equal(a, b), "%s: %s differ" % (what, name)


@pytest.mark.parametrize("metric", ["ip", "cosine"])
def test_build_through_postings_gives_the_same_graph(vdb, metric):
    # 20 000 rows: three 8192-row query chunks, the later ones planned from a non-zero element offset; every 97th row
    # is empty and every 53rd duplicates an earlier one
    n, vocab = 20_000, 3000
    rows = sparse_rows(n, vocab, 81, max_nnz=40)
    ix = vdb.SparseIndex(metric, vocab)
    ix.append(rows)
    want = {}
    for m in (n, n - 1000):
        ix.build(m, out_degree=24)
        want[m] = ix.get_graph()
    # postings over every row, over part of the rows (ending inside the second chunk), over fewer rows than one chunk
    for n_inv in (n, 11_000, 3000):
        ix.build_inverted(n_inv)
        info = ix.inverted_info()
        assert info["rows"] == n_inv
        for m in (n, n - 1000):   # n - 1000: with full postings, posting rows above the build's rows are left out
            ix.build(m, out_degree=24)
            assert ix.inverted_info() == info, "the build changed the postings"
            same_graph(ix.get_graph(), want[m], "%s, postings over %d rows, build of %d" % (metric, n_inv, m))
    ix.close()


def test_build_without_postings_leaves_none(vdb):
    """A build neither creates nor drops postings."""
    n, vocab = 3000, 1000
    rows = sparse_rows(n, vocab, 82)
    for metric in ("ip", "l2"):
        ix = vdb.SparseIndex(metric, vocab)
        ix.append(rows)
        ix.build(n)
        assert ix.inverted_info() == dict(rows=0, terms=0, postings=0)
        ix.close()
