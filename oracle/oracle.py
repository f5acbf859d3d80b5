"""TEST INFRASTRUCTURE — ctypes bindings for the oracle.

``Port``  : oracle/_ref/libepsilla_port.so  (oracle_port.c, the plain-C restatement; always buildable)
``Ref``   : oracle/_ref/libepsilla_ref.so   (the reference's own sources compiled unmodified;
            built only where reference_dir() finds a checkout of the reference)

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / ``--impl reference`` legs import
this module.  The product package (vectordb_b200) never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
PORT_SO = os.path.join(OUT, "libepsilla_port.so")
REF_SO = os.path.join(OUT, "libepsilla_ref.so")

METRIC = {"l2": 1, "euclidean": 1, "cosine": 2, "cos": 2, "ip": 3, "dot": 3, "dot_product": 3}
# meta::FieldType (engine/db/catalog/meta_types.hpp:19-45)
FIELD_TYPE = {"int1": 1, "int2": 2, "int4": 3, "int8": 4, "float": 10, "double": 11, "string": 20, "bool": 30}
FIELD_NP = {"int1": np.int8, "int2": np.int16, "int4": np.int32, "int8": np.int64, "float": np.float32,
            "double": np.float64, "bool": np.uint8}


DEFAULT_REFERENCE = "/root/reference"


def reference_dir():
    """Checkout of epsilla-cloud/vectordb to compile the reference oracle from: $EPSILLA_REFERENCE, else
    DEFAULT_REFERENCE; None when neither holds the reference's engine/ sources."""
    d = os.environ.get("EPSILLA_REFERENCE") or DEFAULT_REFERENCE
    return d if os.path.isdir(os.path.join(d, "engine")) else None


def build(force=False):
    """Compile the port (always) and the reference library (when reference_dir() finds the reference)."""
    if force or not os.path.exists(PORT_SO) or os.path.getmtime(PORT_SO) < os.path.getmtime(
            os.path.join(HERE, "oracle_port.c")):
        subprocess.check_call(["make", "-C", HERE, "port"], stdout=subprocess.DEVNULL)
    if reference_dir() and (force or not os.path.exists(REF_SO)):
        subprocess.check_call(["make", "-C", HERE, "ref", "-j8", "REF=" + reference_dir()], stdout=subprocess.DEVNULL)


def have_ref():
    return os.path.exists(REF_SO)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class PortNode(C.Structure):
    _fields_ = [("node_type", C.c_int64), ("value_type", C.c_int64), ("left", C.c_int64), ("right", C.c_int64),
                ("int_value", C.c_int64), ("double_value", C.c_double), ("bool_value", C.c_int64),
                ("field_offset", C.c_int64)]


class PortIndex(C.Structure):
    _fields_ = [("metric", C.c_int32), ("prefilter", C.c_int32), ("dim", C.c_int64), ("vectors", C.c_void_p),
                ("total_rows", C.c_int64), ("n_indexed", C.c_int64), ("offsets", C.c_void_p), ("nbrs", C.c_void_p),
                ("nav", C.c_int64), ("deleted", C.c_void_p), ("attrs", C.c_void_p), ("attr_stride", C.c_int64),
                ("filter", C.c_void_p), ("n_filter", C.c_int64), ("L_master", C.c_int64), ("L_local", C.c_int64)]


class Port:
    """The C restatement (oracle_port.c)."""

    def __init__(self):
        build()
        L = C.CDLL(PORT_SO)
        for name in ("port_l2sqr", "port_inner_product"):
            getattr(L, name).restype = C.c_float
            getattr(L, name).argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.port_distance.restype = C.c_float
        L.port_distance.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
        L.port_normalize.argtypes = [C.c_void_p, C.c_int64]
        L.port_filter_eval.restype = C.c_int
        L.port_filter_eval.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_double]
        L.port_prepare_init_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p]
        L.port_search.restype = C.c_int64
        L.port_search.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.port_search_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p]
        L.port_add_into_queue.restype = C.c_int64
        L.port_add_into_queue.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                          C.c_float]
        self.L = L

    def distance(self, metric, a, b):
        a = np.ascontiguousarray(a, np.float32)
        b = np.ascontiguousarray(b, np.float32)
        return float(np.float32(self.L.port_distance(METRIC[metric], _p(a), _p(b), a.size)))

    def normalize(self, v):
        v = np.ascontiguousarray(v, np.float32).copy()
        self.L.port_normalize(_p(v), v.size)
        return v

    def filter_eval(self, nodes, attrs, stride, row, dist):
        nodes = np.ascontiguousarray(nodes, np.int64)
        return self.L.port_filter_eval(_p(nodes), nodes.size // 8, _p(attrs), stride, row, dist)

    def prepare_init_ids(self, offsets, nbrs, nav, n_indexed, L):
        out = np.zeros(L, np.int64)
        self.L.port_prepare_init_ids(_p(offsets), _p(nbrs), nav, n_indexed, L, _p(out))
        return out

    def search_batch(self, *, metric, vectors, queries, limit, total_rows=None, n_indexed=0, offsets=None,
                     nbrs=None, nav=0, deleted=None, attrs=None, attr_stride=0, filter_nodes=None, L=500,
                     prefilter=False):
        """Returns ids [nq,limit] int64 (-1 padded), dists float64 (inf padded), counts, (n_dist, n_expand)."""
        vectors = np.ascontiguousarray(vectors, np.float32)
        queries = np.ascontiguousarray(queries, np.float32)
        if queries.ndim == 1:
            queries = queries[None, :]
        nq, dim = queries.shape
        ix = PortIndex()
        ix.metric = METRIC[metric] if isinstance(metric, str) else metric
        ix.prefilter = 1 if prefilter else 0
        ix.dim = dim
        ix.vectors = vectors.ctypes.data
        ix.total_rows = vectors.shape[0] if total_rows is None else total_rows
        ix.n_indexed = n_indexed
        keep = [vectors, queries]
        if n_indexed > 0:
            offsets = np.ascontiguousarray(offsets, np.int64)
            nbrs = np.ascontiguousarray(nbrs, np.int64)
            keep += [offsets, nbrs]
            ix.offsets = offsets.ctypes.data
            ix.nbrs = nbrs.ctypes.data
        ix.nav = nav
        if deleted is not None:
            deleted = np.ascontiguousarray(deleted, np.uint8)
            keep.append(deleted)
            ix.deleted = deleted.ctypes.data
        if attrs is not None:
            keep.append(attrs)
            ix.attrs = attrs.ctypes.data
            ix.attr_stride = attr_stride
        if filter_nodes is not None and len(filter_nodes):
            fn = np.ascontiguousarray(filter_nodes, np.int64)
            keep.append(fn)
            ix.filter = fn.ctypes.data
            ix.n_filter = fn.size // 8
        ix.L_master = L
        ix.L_local = L
        ids = np.full((nq, limit), -1, np.int64)
        dists = np.full((nq, limit), np.inf, np.float64)
        counts = np.zeros(nq, np.int64)
        stats = np.zeros(2, np.uint64)
        self.L.port_search_batch(C.byref(ix), _p(queries), nq, limit, _p(ids), _p(dists), _p(counts), _p(stats))
        return ids, dists, counts, (int(stats[0]), int(stats[1]))


class Ref:
    """The reference itself (VecSearchExecutor / ANNGraphSegment / Expr), via oracle/ref_driver.cpp."""

    def __init__(self, metric, dim, capacity, attr_cols=(), lib_path=None):
        """attr_cols: sequence of (name, type) with type in FIELD_TYPE.  lib_path: an alternative build of the
        same driver (oracle/_ref/dropin/libepsilla_ref_b200.so = the reference engine with the GPU drop-in)."""
        if lib_path is None:
            if not have_ref():
                build()
            if not have_ref():
                raise RuntimeError("oracle/_ref/libepsilla_ref.so not available (no reference checkout found to build it from)")
        L = C.CDLL(lib_path or REF_SO)
        L.ref_create.restype = C.c_void_p
        L.ref_create.argtypes = [C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]
        L.ref_destroy.argtypes = [C.c_void_p]
        L.ref_vectors.restype = C.POINTER(C.c_float)
        L.ref_vectors.argtypes = [C.c_void_p]
        L.ref_attrs.restype = C.POINTER(C.c_char)
        L.ref_attrs.argtypes = [C.c_void_p]
        L.ref_attr_stride.restype = C.c_int64
        L.ref_attr_stride.argtypes = [C.c_void_p]
        L.ref_attr_offset.restype = C.c_int64
        L.ref_attr_offset.argtypes = [C.c_void_p, C.c_char_p]
        L.ref_set_rows.argtypes = [C.c_void_p, C.c_int64]
        L.ref_set_string.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_char_p]
        L.ref_set_deleted.argtypes = [C.c_void_p, C.c_int64, C.c_int]
        L.ref_build.argtypes = [C.c_void_p, C.c_int64, C.c_int]
        L.ref_set_graph.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64]
        L.ref_graph.restype = C.c_int64
        L.ref_graph.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ref_make_executors.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int,
                                         C.c_int]
        L.ref_search.restype = C.c_int64
        L.ref_search.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_char_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p]
        L.ref_search_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_char_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p]
        L.ref_save_graph.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_int64]
        L.ref_load_graph.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_int64]
        L.ref_distance.restype = C.c_float
        L.ref_distance.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
        L.ref_normalize.argtypes = [C.c_void_p, C.c_int64]
        L.ref_filter_eval.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_double]
        L.ref_value_nodes.restype = C.c_int64
        L.ref_value_nodes.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.ref_facet.restype = C.c_int64
        L.ref_facet.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int,
                                C.c_char_p, C.c_int64]
        L.ref_filter_nodes.restype = C.c_int64
        L.ref_filter_nodes.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]
        self.L = L
        self.metric = METRIC[metric] if isinstance(metric, str) else metric
        self.dim = dim
        self.capacity = capacity
        n = len(attr_cols)
        types = (C.c_int * max(n, 1))(*[FIELD_TYPE[t] for _, t in attr_cols])
        names = (C.c_char_p * max(n, 1))(*[nm.encode() for nm, _ in attr_cols])
        self.h = L.ref_create(self.metric, dim, capacity, n, types, names)
        self.attr_cols = list(attr_cols)
        self.stride = L.ref_attr_stride(self.h)
        self.rows = 0
        self.L_ = 500
        self.n_exec = 0

    def __del__(self):
        try:
            self.L.ref_destroy(self.h)
        except Exception:
            pass

    @property
    def vectors(self):
        return np.ctypeslib.as_array(self.L.ref_vectors(self.h), shape=(self.capacity, self.dim))

    @property
    def attrs(self):
        if self.stride == 0:
            return np.zeros(0, np.uint8)
        buf = C.cast(self.L.ref_attrs(self.h), C.POINTER(C.c_uint8))
        return np.ctypeslib.as_array(buf, shape=(self.capacity * self.stride,))

    def attr_offset(self, name):
        return self.L.ref_attr_offset(self.h, name.encode())

    def set_attr_column(self, name, values):
        typ = dict(self.attr_cols)[name]
        values = np.ascontiguousarray(values, FIELD_NP[typ])
        off = self.attr_offset(name)
        raw = self.attrs.reshape(self.capacity, self.stride)
        sz = values.dtype.itemsize
        raw[:values.shape[0], off:off + sz] = values.view(np.uint8).reshape(-1, sz)

    def set_string_column(self, name, values, first_row=0):
        """String attribute column (var_len_attr_table_): values[i] -> row first_row + i."""
        for i, v in enumerate(values):
            if self.L.ref_set_string(self.h, name.encode(), first_row + i, str(v).encode()) != 0:
                raise ValueError("no string field %r" % name)

    def set_rows(self, vectors):
        vectors = np.ascontiguousarray(vectors, np.float32)
        self.vectors[:vectors.shape[0]] = vectors
        self.rows = vectors.shape[0]
        self.L.ref_set_rows(self.h, self.rows)

    def set_row_count(self, n):
        self.rows = n
        self.L.ref_set_rows(self.h, n)

    def set_deleted(self, ids, flag=True):
        for i in np.atleast_1d(ids):
            self.L.ref_set_deleted(self.h, int(i), 1 if flag else 0)

    def build(self, n=None, threads=1):
        n = self.rows if n is None else n
        devnull = os.open(os.devnull, os.O_WRONLY)
        saved = os.dup(1)
        os.dup2(devnull, 1)  # the reference logs one DEBUG line per NN-descent iteration
        try:
            rc = self.L.ref_build(self.h, n, threads)
        finally:
            os.dup2(saved, 1)
            os.close(devnull)
            os.close(saved)
        if rc != 0:
            raise RuntimeError("reference build threw")
        return self.graph()

    def set_graph(self, n_indexed, offsets, nbrs, nav):
        offsets = np.ascontiguousarray(offsets, np.int64)
        nbrs = np.ascontiguousarray(nbrs, np.int64)
        self.L.ref_set_graph(self.h, n_indexed, _p(offsets), _p(nbrs), nav)

    def graph(self):
        po, pn, nav = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)(), C.c_int64()
        n = self.L.ref_graph(self.h, C.byref(po), C.byref(pn), C.byref(nav))
        if n == 0:
            return 0, np.zeros(1, np.int64), np.zeros(0, np.int64), 0
        off = np.ctypeslib.as_array(po, shape=(n + 1,)).copy()
        nb = np.ctypeslib.as_array(pn, shape=(int(off[n]),)).copy() if off[n] > 0 else np.zeros(0, np.int64)
        return n, off, nb, nav.value

    def save_graph(self, directory, table_id=0, field_id=1):
        if self.L.ref_save_graph(self.h, directory.encode(), table_id, field_id) != 0:
            raise RuntimeError("SaveANNGraph failed")

    def load_graph(self, directory, table_id=0, field_id=1):
        if self.L.ref_load_graph(self.h, directory.encode(), table_id, field_id) != 0:
            raise RuntimeError("ANNGraphSegment load failed")

    def make_executors(self, n_exec=1, T=1, L=500, iters=15, prefilter=False, counting=False):
        self.L_ = L
        self.n_exec = n_exec
        self.L.ref_make_executors(self.h, n_exec, T, L, L, iters, 1 if prefilter else 0, 1 if counting else 0)

    def search(self, query, limit, filter=""):
        """One VecSearchExecutor::Search.  Returns ids, dists(float64), n_dist."""
        q = np.ascontiguousarray(query, np.float32)
        cap = max(limit, self.L_) + 1
        ids = np.zeros(cap, np.int64)
        ds = np.zeros(cap, np.float64)
        nd = C.c_uint64(0)
        n = self.L.ref_search(self.h, 0, _p(q), limit, filter.encode(), _p(ids), _p(ds), C.byref(nd))
        if n == -2:
            raise RuntimeError("Search returned a non-OK status for filter %r" % filter)
        if n < 0:
            raise ValueError("filter failed to parse: %r" % filter)
        return ids[:n].copy(), ds[:n].copy(), nd.value

    def search_batch(self, queries, limit, filter=""):
        q = np.ascontiguousarray(queries, np.float32)
        nq = q.shape[0]
        ids = np.full((nq, limit), -1, np.int64)
        ds = np.full((nq, limit), np.inf, np.float64)
        counts = np.zeros(nq, np.int64)
        rc = self.L.ref_search_batch(self.h, _p(q), nq, limit, filter.encode(), _p(ids), _p(ds), _p(counts))
        if rc == -2:
            raise RuntimeError("Search returned a non-OK status for filter %r" % filter)
        if rc != 0:
            raise ValueError("filter failed to parse: %r" % filter)
        return ids, ds, counts

    def distance(self, a, b):
        a = np.ascontiguousarray(a, np.float32)
        b = np.ascontiguousarray(b, np.float32)
        return float(np.float32(self.L.ref_distance(self.metric, _p(a), _p(b), a.size)))

    def normalize(self, v):
        v = np.ascontiguousarray(v, np.float32).copy()
        self.L.ref_normalize(_p(v), v.size)
        return v

    def filter_eval(self, filter, row, dist=0.0):
        return self.L.ref_filter_eval(self.h, filter.encode(), row, dist)

    def value_nodes(self, expr):
        """Value expression (facet key / aggregate input) -> ([n,8] PODs, ValueType ordinal of the root)."""
        out = np.zeros((64, 8), np.int64)
        vt = C.c_int64(0)
        n = self.L.ref_value_nodes(self.h, expr.encode(), _p(out), 64, C.byref(vt))
        if n < 0:
            raise ValueError("expression failed to parse: %r" % expr)
        return out[:n].copy(), int(vt.value)

    def facet(self, group_expr, agg_exprs, ids, dists=None):
        """FacetExecutor::Aggregate + Project over one id list -> list of dicts (the reference's JSON array)."""
        import json
        ids = np.ascontiguousarray(ids, np.int64)
        d = None if dists is None else np.ascontiguousarray(dists, np.float64)
        arr = (C.c_char_p * len(agg_exprs))(*[e.encode() for e in agg_exprs])
        buf = C.create_string_buffer(1 << 20)
        n = self.L.ref_facet(self.h, group_expr.encode(), len(agg_exprs), arr, _p(ids), _p(d), ids.size, 0 if d is None else 1,
                             buf, len(buf))
        if n < 0:
            raise ValueError("facet failed (%d)" % n)
        return json.loads(buf.value.decode())

    def filter_nodes(self, filter):
        """Parsed node array as [n,8] int64 PODs (see oracle_port.c port_node)."""
        out = np.zeros((64, 8), np.int64)
        n = self.L.ref_filter_nodes(self.h, filter.encode(), _p(out), 64)
        if n < 0:
            raise ValueError("filter failed to parse: %r" % filter)
        return out[:n].copy()
