"""Python mirror of the C ABI (include/epsilla_b200.h).  One method per entry point."""
import ctypes as C

import numpy as np

from .lib import BuildParams, FacetSpec, FilterNode, StatsStruct, check, load_library

METRICS = {"l2": 1, "euclidean": 1, "cosine": 2, "cos": 2, "ip": 3, "dot": 3, "dot_product": 3}


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def filter_nodes_array(nodes):
    """[n,8] int64 node PODs (layout of eps_filter_node; double_value stored as raw bits) -> ctypes array."""
    if nodes is None:
        return None, 0
    nodes = np.ascontiguousarray(nodes, np.int64).reshape(-1, 8)
    n = nodes.shape[0]
    if n == 0:
        return None, 0
    arr = (FilterNode * n)()
    C.memmove(arr, nodes.ctypes.data, n * 64)
    return arr, n


class Stats(dict):
    @classmethod
    def from_struct(cls, s):
        return cls(n_dist=int(s.n_dist), n_seed=int(s.n_seed), n_expand=int(s.n_expand), n_edges=int(s.n_edges),
                   n_queries=int(s.n_queries), kernel_ms=float(s.kernel_ms), total_ms=float(s.total_ms),
                   kernel_launches=int(s.kernel_launches), n_redone=int(s.n_redone))


class Index:
    """Device mirror of one vector field of a TableSegmentMVP + its ANNGraphSegment + executor params."""

    def __init__(self, metric, dim, host_vectors=None, capacity=None, device=0):
        self.L = load_library()
        self.metric = METRICS[metric] if isinstance(metric, str) else int(metric)
        self.dim = int(dim)
        self.device = device
        self._host = None
        if host_vectors is not None:
            host_vectors = np.ascontiguousarray(host_vectors, np.float32)
            assert host_vectors.ndim == 2 and host_vectors.shape[1] == dim
            self._host = host_vectors
            capacity = host_vectors.shape[0] if capacity is None else capacity
        self.capacity = int(capacity or 0)
        h = C.c_void_p()
        check(self.L.eps_index_create(C.byref(h), self.metric, self.dim, _p(self._host), self.capacity, device))
        self.h = h
        self._keep = []

    def view(self):
        """Read-only view sharing this index's device data, with its own stream and scratch (eps_index_create_view):
        searches on the view overlap searches on the base.  Close the views before the base."""
        v = Index.__new__(Index)
        v.L, v.metric, v.dim, v.device, v._host, v.capacity, v._keep = self.L, self.metric, self.dim, self.device, None, self.capacity, []
        h = C.c_void_p()
        check(self.L.eps_index_create_view(self.h, C.byref(h)))
        v.h = h
        v._base = self  # keeps the base alive
        return v

    def close(self):
        if getattr(self, "h", None):
            self.L.eps_index_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- segment mirrors ---
    def sync_rows(self, n_rows):
        check(self.L.eps_index_sync_rows(self.h, int(n_rows)))

    def adopt_device_rows(self, ptr, n_rows):
        check(self.L.eps_index_adopt_device_rows(self.h, C.c_void_p(ptr), int(n_rows)))

    def set_graph(self, n_indexed, offsets, nbrs, nav):
        offsets = np.ascontiguousarray(offsets, np.int64)
        nbrs = np.ascontiguousarray(nbrs, np.int64)
        check(self.L.eps_index_set_graph(self.h, int(n_indexed), _p(offsets), _p(nbrs), int(nav)))

    def build(self, n, **params):
        bp = BuildParams()
        for k, v in params.items():
            setattr(bp, k, v)
        check(self.L.eps_index_build(self.h, int(n), C.byref(bp)))

    def get_graph(self):
        n, e, nav = C.c_int64(), C.c_int64(), C.c_int64()
        check(self.L.eps_index_get_graph(self.h, C.byref(n), C.byref(e), None, None, C.byref(nav)))
        off = np.zeros(n.value + 1, np.int64)
        nb = np.zeros(max(e.value, 1), np.int64)
        if n.value > 0:
            check(self.L.eps_index_get_graph(self.h, None, None, _p(off), _p(nb), None))
        return n.value, off, nb[:e.value], nav.value

    def set_deleted(self, bitset_bytes):
        b = np.ascontiguousarray(bitset_bytes, np.uint8)
        check(self.L.eps_index_set_deleted(self.h, _p(b), b.size))

    def set_attrs(self, table_bytes, stride, n_rows):
        t = np.ascontiguousarray(table_bytes, np.uint8)
        check(self.L.eps_index_set_attrs(self.h, _p(t), int(stride), int(n_rows)))

    def set_string_codes(self, column, first_row, codes):
        """Append the dictionary codes of rows [first_row, first_row + len(codes)) of string column `column`."""
        c = np.ascontiguousarray(codes, np.int32)
        check(self.L.eps_index_set_string_codes(self.h, int(column), int(first_row), _p(c), c.size))

    def config(self, L_master=500, L_local=None, prefilter=False, force_brute=False):
        L_local = L_master if L_local is None else L_local
        check(self.L.eps_index_config(self.h, int(L_master), int(L_local), int(bool(prefilter)), int(bool(force_brute))))

    def set_search_width(self, width):
        """1 = sequential expansion order of the reference (IntraQueryThreads=1); 2/4 = parallel expansion."""
        check(self.L.eps_index_set_search_width(self.h, int(width)))

    def set_graph_tuning(self, ring_slots=0, ctas_per_sm=0):
        """Launch geometry of the graph kernel (0 = auto): TMA row-ring slots per CTA, resident CTAs per SM."""
        check(self.L.eps_index_set_graph_tuning(self.h, int(ring_slots), int(ctas_per_sm)))

    def set_coarse(self, mode):
        """0 = fp32 SIMT only, 1 = wgmma TF32 (default), 2 = wgmma bf16 mirror (exact re-score in all modes)."""
        check(self.L.eps_index_set_coarse(self.h, {"fp32": 0, "tf32": 1, "bf16": 2}.get(mode, mode)))

    def set_coarse_guard(self, on=True):
        """Verify the coarse pass after the re-score and redo unsafe queries (on by default)."""
        check(self.L.eps_index_set_coarse_guard(self.h, int(bool(on))))

    # --- search ---
    def search(self, queries, limit, filter_nodes=None, want_stats=True):
        """HOST buffers in/out (eps_search_batch).  Returns ids [nq,limit], dists float64, counts, Stats."""
        q = np.ascontiguousarray(queries, np.float32)
        if q.ndim == 1:
            q = q[None, :]
        nq = q.shape[0]
        ids = np.empty((nq, limit), np.int64)
        dists = np.empty((nq, limit), np.float64)
        counts = np.empty(nq, np.int64)
        st = StatsStruct()
        arr, n = filter_nodes_array(filter_nodes)
        check(self.L.eps_search_batch(self.h, _p(q), nq, int(limit), arr, n, _p(ids), _p(dists), _p(counts),
                                      C.byref(st) if want_stats else None))
        return ids, dists, counts, Stats.from_struct(st)

    def search_device(self, d_queries_ptr, nq, limit, d_ids_ptr, d_dists_ptr, d_counts_ptr, filter_nodes=None,
                      want_stats=False, sync=True):
        """DEVICE pointers in/out (eps_search_batch_device)."""
        st = StatsStruct()
        arr, n = filter_nodes_array(filter_nodes)
        check(self.L.eps_search_batch_device(self.h, C.c_void_p(d_queries_ptr), int(nq), int(limit), arr, n,
                                             C.c_void_p(d_ids_ptr), C.c_void_p(d_dists_ptr), C.c_void_p(d_counts_ptr),
                                             C.byref(st) if want_stats else None, int(bool(sync))))
        return Stats.from_struct(st)

    def facet(self, ids, counts, key_nodes, key_type, aggs, dists=None):
        """FacetExecutor::Aggregate over result lists (eps_facet_batch).  key_nodes: [n,8] PODs of the group-by
        expression; key_type: 0 string (dictionary code), 1 int, 2 double, 3 bool; aggs: [(agg_type, nodes)] with
        agg_type 30 SUM / 31 MIN / 32 MAX / 33 COUNT.  Returns per query a list of (key, [values])."""
        ids = np.ascontiguousarray(ids, np.int64)
        nq, limit = ids.shape
        counts = np.ascontiguousarray(counts, np.int64)
        d = None if dists is None else np.ascontiguousarray(dists, np.float64)
        spec = FacetSpec()
        keep = []
        karr, kn = filter_nodes_array(key_nodes)
        keep.append(karr)
        spec.key_nodes, spec.n_key_nodes, spec.key_type, spec.n_aggs = C.cast(karr, C.c_void_p), kn, int(key_type), len(aggs)
        for i, (t, nodes) in enumerate(aggs):
            arr, n = filter_nodes_array(nodes)
            keep.append(arr)
            spec.agg_nodes[i], spec.n_agg_nodes[i], spec.agg_types[i] = C.cast(arr, C.c_void_p), n, int(t)
        ok = np.empty((nq, limit), np.float64)
        ov = np.empty((nq, limit, len(aggs)), np.float64)
        og = np.empty(nq, np.int64)
        check(self.L.eps_facet_batch(self.h, _p(ids), _p(d), _p(counts), nq, limit, C.byref(spec), _p(ok), _p(ov), _p(og)))
        return [[(ok[q, g], ov[q, g].tolist()) for g in range(og[q])] for q in range(nq)]

    @property
    def stream(self):
        return self.L.eps_index_stream(self.h)


def normalize(vectors, device=0):
    v = np.ascontiguousarray(vectors, np.float32).copy()
    if v.ndim == 1:
        v = v[None, :]
    check(load_library().eps_normalize(device, _p(v), v.shape[0], v.shape[1]))
    return v


def pair_distances(metric, a, b, device=0):
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    out = np.empty(a.shape[0], np.float32)
    m = METRICS[metric] if isinstance(metric, str) else metric
    check(load_library().eps_pair_distances(device, m, _p(a), _p(b), a.shape[0], a.shape[1], _p(out)))
    return out


def merge_shards_device(device, d_ids_ptr, d_dists_ptr, n_shards, nq, k, d_out_ids_ptr, d_out_dists_ptr):
    check(load_library().eps_merge_shards_device(device, C.c_void_p(d_ids_ptr), C.c_void_p(d_dists_ptr), n_shards, nq, k,
                                                 C.c_void_p(d_out_ids_ptr), C.c_void_p(d_out_dists_ptr)))
