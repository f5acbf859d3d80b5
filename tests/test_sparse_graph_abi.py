"""CPU tests of eps_index_set_sparse_search: declared in the header, exported, bound by lib.py, refused without a GPU."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    import vectordb_b200
    if not os.path.exists(vectordb_b200.library_path()):
        from vectordb_b200.lib import build_library
        build_library()
    return vectordb_b200.load_library()


def test_sparse_search_mode_declared_exported_and_bound():
    L = _lib()
    hdr = open(os.path.join(ROOT, "include", "epsilla_b200.h")).read()
    assert re.search(r"EPS_API int eps_index_set_sparse_search\(eps_index\* ix, int mode\);", hdr)
    assert re.search(r"#define EPS_SPARSE_SEARCH_SCAN 0\b", hdr) and re.search(r"#define EPS_SPARSE_SEARCH_GRAPH 1\b", hdr)
    from vectordb_b200.lib import EXPORTS
    assert "eps_index_set_sparse_search" in EXPORTS
    assert L.eps_index_set_sparse_search.argtypes
    from vectordb_b200.index import SPARSE_SEARCH_MODES, SparseIndex
    assert SPARSE_SEARCH_MODES == {"scan": 0, "graph": 1}
    assert callable(SparseIndex.set_search_mode)


def test_sparse_search_mode_refused_without_index():
    L = _lib()
    for mode in (0, 1, 2):
        assert L.eps_index_set_sparse_search(None, mode) == 40005  # EPS_ERR_INVALID_ARGUMENT: no index
