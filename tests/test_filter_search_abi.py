"""CPU tests of the filter search mode's entry point: declared in the header with its two modes, exported, bound by
lib.py, reachable from Index, and refused without an index."""
import os
import re

from test_sparse_abi import ROOT, _lib


def test_filter_search_declared_exported_and_bound():
    L = _lib()
    hdr = open(os.path.join(ROOT, "include", "epsilla_b200.h")).read()
    assert re.search(r"EPS_API int eps_index_set_filter_search\(eps_index\* ix, int mode\);", hdr)
    assert re.search(r"#define EPS_FILTER_SEARCH_POST 0\b", hdr) and re.search(r"#define EPS_FILTER_SEARCH_COLLECT 1\b", hdr)
    from vectordb_b200.lib import EXPORTS
    assert "eps_index_set_filter_search" in EXPORTS
    assert L.eps_index_set_filter_search.argtypes
    from vectordb_b200.index import FILTER_SEARCH_MODES, Index
    assert FILTER_SEARCH_MODES == {"post": 0, "collect": 1}
    assert callable(Index.set_filter_search)


def test_filter_search_null_index_refused():
    L = _lib()
    for mode in (-1, 0, 1, 2):
        assert L.eps_index_set_filter_search(None, mode) == 40005   # EPS_ERR_INVALID_ARGUMENT: no index
