"""The sparse graph build of an L2 index screens its kNN pass when the index has the L2 screen.

The screen re-scores every row that can still be among a row's out_degree nearest, with the merge's own distance, so
the graph (offsets, neighbours, navigation point) must be identical to the one built without it, whether the screen
covers every row, part of the rows (the rest comes from the merge) or more rows than the build indexes; and the build
leaves the screen's rows as they were."""
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


def test_build_through_the_l2_screen_gives_the_same_graph(vdb):
    # 20 000 rows: three 8192-row query chunks, the later ones planned from a non-zero element offset; every 97th row
    # is empty and every 53rd duplicates an earlier one
    n, vocab = 20_000, 3000
    rows = sparse_rows(n, vocab, 81, max_nnz=40)
    ix = vdb.SparseIndex("l2", vocab)
    ix.append(rows)
    want = {}
    for m in (n, n - 1000):
        ix.build(m, out_degree=24)
        want[m] = ix.get_graph()
    assert ix.l2_screen_info() == dict(rows=0, rescored=0)
    # the screen over every row, over part of the rows (ending inside the second chunk), over fewer rows than one chunk
    for n_scr in (n, 11_000, 3000):
        ix.build_l2_screen(n_scr)
        info = ix.inverted_info()
        assert info["rows"] == n_scr
        for m in (n, n - 1000):   # n - 1000: with the full screen, screened rows above the build's rows are left out
            r0 = ix.l2_screen_info()["rescored"]
            ix.build(m, out_degree=24)
            assert ix.inverted_info() == info and ix.l2_screen_info()["rows"] == n_scr, "the build changed the screen"
            same_graph(ix.get_graph(), want[m], "screen over %d rows, build of %d" % (n_scr, m))
            rescored = ix.l2_screen_info()["rescored"] - r0
            assert 0 < rescored < m * min(m, n_scr)
            print("screen over %d rows, build of %d: re-scored %.4f of the covered pairs"
                  % (n_scr, m, rescored / (m * min(m, n_scr))))
    ix.close()
