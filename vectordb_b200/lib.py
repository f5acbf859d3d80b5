"""ctypes loader for libepsilla_b200.so.  No fallback of any kind: a missing library is an error."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

EXPORTS = [
    "eps_index_create", "eps_index_destroy", "eps_index_create_view", "eps_index_sync_rows", "eps_index_adopt_device_rows", "eps_index_device_rows", "eps_index_rows",
    "eps_index_set_graph", "eps_index_build", "eps_index_get_graph", "eps_index_set_deleted", "eps_index_set_attrs", "eps_index_set_string_codes",
    "eps_index_config", "eps_index_set_coarse", "eps_index_set_coarse_guard", "eps_index_set_search_width", "eps_index_set_graph_tuning", "eps_search_batch", "eps_search_batch_device", "eps_merge_shards_device", "eps_facet_batch", "eps_shard_unique_id", "eps_shard_group_create", "eps_shard_group_destroy", "eps_search_batch_sharded", "eps_normalize",
    "eps_pair_distances", "eps_index_stream", "eps_last_error", "eps_version", "eps_device_count",
]


class EpsError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("epsilla_b200 error %d: %s" % (code, msg))
        self.code = code


class FilterNode(C.Structure):
    _fields_ = [("node_type", C.c_int64), ("value_type", C.c_int64), ("left", C.c_int64), ("right", C.c_int64),
                ("int_value", C.c_int64), ("double_value", C.c_double), ("bool_value", C.c_int64),
                ("field_offset", C.c_int64)]


class StatsStruct(C.Structure):
    _fields_ = [("n_dist", C.c_uint64), ("n_seed", C.c_uint64), ("n_expand", C.c_uint64), ("n_edges", C.c_uint64),
                ("n_queries", C.c_uint64), ("kernel_ms", C.c_double), ("total_ms", C.c_double),
                ("kernel_launches", C.c_uint64), ("n_redone", C.c_uint64)]


class FacetSpec(C.Structure):
    _fields_ = [("key_nodes", C.c_void_p), ("n_key_nodes", C.c_int64), ("key_type", C.c_int32), ("n_aggs", C.c_int32),
                ("agg_nodes", C.c_void_p * 8), ("n_agg_nodes", C.c_int64 * 8), ("agg_types", C.c_int32 * 8)]


class BuildParams(C.Structure):
    _fields_ = [("knn_k", C.c_int32), ("out_degree", C.c_int32), ("candidate_pool", C.c_int32),
                ("search_length", C.c_int32), ("nnd_iters", C.c_int32), ("nnd_sample", C.c_int32),
                ("exact_knn_below", C.c_int32), ("seed", C.c_int32), ("nnd_delta", C.c_float),
                ("min_degree", C.c_int32), ("alpha", C.c_float), ("reserved", C.c_int32)]


def library_path():
    # EPS_B200_LIB: developer override (e.g. the phase-timer build `make -C vectordb_b200/csrc prof`)
    return os.environ.get("EPS_B200_LIB") or os.path.join(HERE, "libepsilla_b200.so")


def build_library(verbose=False):
    """Compile csrc/ for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    out = None if verbose else subprocess.DEVNULL
    subprocess.check_call(["make", "-C", os.path.join(HERE, "csrc"), "-j8"], stdout=out)


def load_library():
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not os.path.exists(path):
        raise RuntimeError(
            "libepsilla_b200.so is missing (%s). Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C vectordb_b200/csrc`. There is no CPU fallback." % path)
    L = C.CDLL(path)
    vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int
    L.eps_index_create.argtypes = [C.POINTER(vp), i32, i64, vp, i64, i32]
    L.eps_index_destroy.argtypes = [vp]
    L.eps_index_create_view.argtypes = [vp, C.POINTER(vp)]
    L.eps_index_destroy.restype = None
    L.eps_index_sync_rows.argtypes = [vp, i64]
    L.eps_index_adopt_device_rows.argtypes = [vp, vp, i64]
    L.eps_index_device_rows.argtypes = [vp]
    L.eps_index_device_rows.restype = vp
    L.eps_index_rows.argtypes = [vp]
    L.eps_index_rows.restype = i64
    L.eps_index_set_graph.argtypes = [vp, i64, vp, vp, i64]
    L.eps_index_build.argtypes = [vp, i64, vp]
    L.eps_index_get_graph.argtypes = [vp, vp, vp, vp, vp, vp]
    L.eps_index_set_deleted.argtypes = [vp, vp, i64]
    L.eps_index_set_attrs.argtypes = [vp, vp, i64, i64]
    L.eps_index_set_string_codes.argtypes = [vp, i32, i64, vp, i64]
    L.eps_index_config.argtypes = [vp, i64, i64, i32, i32]
    L.eps_index_set_coarse.argtypes = [vp, i32]
    L.eps_index_set_coarse_guard.argtypes = [vp, i32]
    L.eps_index_set_search_width.argtypes = [vp, i32]
    L.eps_index_set_graph_tuning.argtypes = [vp, i32, i32]
    L.eps_search_batch.argtypes = [vp, vp, i64, i64, vp, i64, vp, vp, vp, vp]
    L.eps_search_batch_device.argtypes = [vp, vp, i64, i64, vp, i64, vp, vp, vp, vp, i32]
    L.eps_merge_shards_device.argtypes = [i32, vp, vp, i64, i64, i64, vp, vp]
    L.eps_normalize.argtypes = [i32, vp, i64, i64]
    L.eps_facet_batch.argtypes = [vp, vp, vp, vp, i64, i64, vp, vp, vp, vp]
    L.eps_shard_unique_id.argtypes = [vp]
    L.eps_shard_group_create.argtypes = [C.POINTER(vp), vp, i32, i32, i32]
    L.eps_shard_group_destroy.argtypes = [vp]
    L.eps_shard_group_destroy.restype = None
    L.eps_search_batch_sharded.argtypes = [vp, vp, i64, vp, i64, i64, vp, i64, vp, vp, vp, i32]
    L.eps_pair_distances.argtypes = [i32, i32, vp, vp, i64, i64, vp]
    L.eps_index_stream.argtypes = [vp]
    L.eps_index_stream.restype = vp
    L.eps_last_error.restype = C.c_char_p
    L.eps_version.restype = C.c_char_p
    L.eps_device_count.restype = i32
    _LIB = L
    return L


def check(rc):
    if rc != 0:
        raise EpsError(rc, load_library().eps_last_error().decode(errors="replace"))
