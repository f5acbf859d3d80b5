"""CPU tests of the sparse inverted index's entry points: declared in the header, exported, bound by lib.py, reachable from
SparseIndex, and a null index refused before any device is needed."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("eps_index_build_sparse_inverted", "eps_index_sparse_inverted_info")


def _lib():
    import vectordb_b200
    if not os.path.exists(vectordb_b200.library_path()):
        from vectordb_b200.lib import build_library
        build_library()
    return vectordb_b200.load_library()


def test_sparse_inverted_declared_exported_and_bound():
    L = _lib()
    hdr = open(os.path.join(ROOT, "include", "epsilla_b200.h")).read()
    assert re.search(r"EPS_API int eps_index_build_sparse_inverted\(eps_index\* ix, int64_t n\);", hdr)
    assert re.search(r"EPS_API int eps_index_sparse_inverted_info\(eps_index\* ix, int64_t\* n_rows, int64_t\* n_terms, "
                     r"int64_t\* n_postings\);", hdr)
    from vectordb_b200.lib import EXPORTS
    for name in NAMES:
        assert name in EXPORTS
        assert getattr(L, name).argtypes, "%s has no ctypes signature" % name
    from vectordb_b200.index import SPARSE_SEARCH_MODES, SparseIndex
    assert callable(SparseIndex.build_inverted) and callable(SparseIndex.inverted_info)
    assert SPARSE_SEARCH_MODES == {"scan": 0, "graph": 1}   # the index is not a search mode


def test_sparse_inverted_null_index_refused():
    L = _lib()
    for n in (-1, 0, 5):
        assert L.eps_index_build_sparse_inverted(None, n) == 40005   # EPS_ERR_INVALID_ARGUMENT: no index
    assert L.eps_index_sparse_inverted_info(None, None, None, None) == 40005
