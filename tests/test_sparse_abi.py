"""CPU tests of the sparse-vector entry points (rows and search, the search mode, the inverted index): declared in the
header, exported, bound by lib.py, reachable from SparseIndex, and refused without a GPU or without an index."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPARSE = ("eps_index_create_sparse", "eps_index_append_sparse_rows", "eps_search_sparse_batch")
INVERTED = ("eps_index_build_sparse_inverted", "eps_index_sparse_inverted_info")


def _lib():
    import vectordb_b200
    if not os.path.exists(vectordb_b200.library_path()):
        from vectordb_b200.lib import build_library
        build_library()
    return vectordb_b200.load_library()


def test_sparse_entry_points_declared_and_bound():
    L = _lib()
    hdr = open(os.path.join(ROOT, "include", "epsilla_b200.h")).read()
    from vectordb_b200.lib import EXPORTS
    for name in SPARSE:
        assert re.search(r"EPS_API int %s\(" % name, hdr), name
        assert name in EXPORTS
        assert getattr(L, name).argtypes, "%s has no ctypes signature" % name


def test_sparse_calls_refused_without_gpu():
    import vectordb_b200
    L = _lib()
    if L.eps_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(vectordb_b200.EpsError) as e:
        vectordb_b200.SparseIndex("ip", 30522)
    assert e.value.code == 50001  # EPS_ERR_NO_DEVICE
    h = C.c_void_p()
    assert L.eps_index_create_sparse(C.byref(h), 3, 100, 10, 0) == 50001 and not h.value
    off = np.array([0, 1], np.int64)
    assert L.eps_index_append_sparse_rows(None, 0, 1, off.ctypes.data, off.ctypes.data, off.ctypes.data) != 0
    out = np.zeros(4, np.int64)
    assert L.eps_search_sparse_batch(None, 1, off.ctypes.data, off.ctypes.data, off.ctypes.data, 1, None, 0,
                                     out.ctypes.data, out.ctypes.data, out.ctypes.data, None) != 0


def test_as_csr_accepts_scipy_and_tuples():
    sp = pytest.importorskip("scipy.sparse")
    from vectordb_b200.index import as_csr
    m = sp.csr_matrix((np.array([1.0, 2.0, 3.0]), np.array([4, 1, 7]), np.array([0, 2, 3])), shape=(2, 10))
    off, idx, val = as_csr(m)
    assert off.dtype == np.int64 and idx.dtype == np.int64 and val.dtype == np.float32
    assert off.tolist() == [0, 2, 3] and idx.tolist() == [1, 4, 7] and val.tolist() == [2.0, 1.0, 3.0]
    off2, idx2, val2 = as_csr(([0, 2, 3], [1, 4, 7], [2.0, 1.0, 3.0]))
    assert np.array_equal(off, off2) and np.array_equal(idx, idx2) and np.array_equal(val, val2)


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


def test_sparse_inverted_declared_exported_and_bound():
    L = _lib()
    hdr = open(os.path.join(ROOT, "include", "epsilla_b200.h")).read()
    assert re.search(r"EPS_API int eps_index_build_sparse_inverted\(eps_index\* ix, int64_t n\);", hdr)
    assert re.search(r"EPS_API int eps_index_sparse_inverted_info\(eps_index\* ix, int64_t\* n_rows, int64_t\* n_terms, "
                     r"int64_t\* n_postings\);", hdr)
    from vectordb_b200.lib import EXPORTS
    for name in INVERTED:
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
