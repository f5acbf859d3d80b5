"""CPU test of eps_index_extend_graph's argument check: a null index is refused before any device work."""
import ctypes as C
import os


def _lib():
    import vectordb_b200
    if not os.path.exists(vectordb_b200.library_path()):
        from vectordb_b200.lib import build_library
        build_library()
    return vectordb_b200.load_library()


def test_extend_graph_null_index_is_refused_without_a_device():
    L = _lib()
    assert L.eps_index_extend_graph(None, 10, None) == 40005  # EPS_ERR_INVALID_ARGUMENT
    assert b"null index" in L.eps_last_error()
    from vectordb_b200.lib import BuildParams
    bp = BuildParams()
    assert L.eps_index_extend_graph(None, 10, C.byref(bp)) == 40005
