"""CPU tests of the L2 screen's entry points: declared in the header, exported, bound by lib.py, reachable from
SparseIndex, and refused without an index."""
import os
import re

from test_sparse_abi import ROOT, _lib

SCREEN = ("eps_index_build_sparse_l2_screen", "eps_index_sparse_l2_screen_info")


def test_l2_screen_declared_exported_and_bound():
    L = _lib()
    hdr = open(os.path.join(ROOT, "include", "epsilla_b200.h")).read()
    assert re.search(r"EPS_API int eps_index_build_sparse_l2_screen\(eps_index\* ix, int64_t n\);", hdr)
    assert re.search(r"EPS_API int eps_index_sparse_l2_screen_info\(eps_index\* ix, int64_t\* n_rows, "
                     r"uint64_t\* n_rescored\);", hdr)
    from vectordb_b200.lib import EXPORTS
    for name in SCREEN:
        assert name in EXPORTS
        assert getattr(L, name).argtypes, "%s has no ctypes signature" % name
    from vectordb_b200.index import SPARSE_SEARCH_MODES, SparseIndex
    assert callable(SparseIndex.build_l2_screen) and callable(SparseIndex.l2_screen_info)
    assert SPARSE_SEARCH_MODES == {"scan": 0, "graph": 1}   # the screen is not a search mode


def test_l2_screen_null_index_refused():
    L = _lib()
    for n in (-1, 0, 5):
        assert L.eps_index_build_sparse_l2_screen(None, n) == 40005   # EPS_ERR_INVALID_ARGUMENT: no index
    assert L.eps_index_sparse_l2_screen_info(None, None, None) == 40005
