"""Python mirror of the C ABI (include/epsilla_b200.h).  One method per entry point."""
import ctypes as C

import numpy as np

from .lib import BuildParams, FacetSpec, FilterNode, StatsStruct, check, load_library

FILTER_SEARCH_MODES = {"post": 0, "collect": 1}
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


def _build_params(params):
    """eps_build_params with the given fields set and the others 0."""
    bp = BuildParams()
    for k, v in params.items():
        setattr(bp, k, v)
    return bp


class Stats(dict):
    @classmethod
    def from_struct(cls, s):
        return cls(n_dist=int(s.n_dist), n_seed=int(s.n_seed), n_expand=int(s.n_expand), n_edges=int(s.n_edges),
                   n_queries=int(s.n_queries), kernel_ms=float(s.kernel_ms), total_ms=float(s.total_ms),
                   kernel_launches=int(s.kernel_launches), n_redone=int(s.n_redone))


class Index:
    """Device mirror of one vector field of a TableSegmentMVP + its ANNGraphSegment + executor params."""

    def __init__(self, metric, dim, host_vectors=None, capacity=None, device=0):
        if host_vectors is not None:
            host_vectors = np.ascontiguousarray(host_vectors, np.float32)
            assert host_vectors.ndim == 2 and host_vectors.shape[1] == dim
            capacity = host_vectors.shape[0] if capacity is None else capacity
        self._open(metric, dim, host_vectors, capacity, device,
                   lambda h: self.L.eps_index_create(h, self.metric, self.dim, _p(self._host), self.capacity, device))

    def _open(self, metric, dim, host, capacity, device, create):
        """Field set-up of every constructor and view; create(handle pointer) makes the C handle."""
        self.L = load_library()
        self.metric = METRICS[metric] if isinstance(metric, str) else int(metric)
        self.dim = int(dim)
        self.device = device
        self._host = host
        self.capacity = int(capacity or 0)
        self._keep = []
        h = C.c_void_p()
        check(create(C.byref(h)))
        self.h = h

    def view(self):
        """Read-only view sharing this index's device data, with its own stream and scratch (eps_index_create_view):
        searches on the view overlap searches on the base.  Close the views before the base."""
        v = type(self).__new__(type(self))
        v._open(self.metric, self.dim, None, self.capacity, self.device,
                lambda h: self.L.eps_index_create_view(self.h, h))
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
        check(self.L.eps_index_build(self.h, int(n), C.byref(_build_params(params))))

    def extend_graph(self, n, **params):
        """Link rows [n_indexed, n) into the installed graph without a full rebuild (eps_index_extend_graph); params are
        eps_build_params fields as for build (knn_k, out_degree, candidate_pool, search_length, min_degree, alpha,
        seed).  n == n_indexed does nothing."""
        check(self.L.eps_index_extend_graph(self.h, int(n), C.byref(_build_params(params))))

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

    def append_string_dictionary(self, first_code, strings):
        """Append the strings of dictionary codes [first_code, first_code + len(strings)) for LIKE filters
        (eps_index_append_string_dictionary); str is encoded as UTF-8, bytes are taken as they are."""
        enc = [s.encode("utf-8") if isinstance(s, str) else bytes(s) for s in strings]
        off = np.zeros(len(enc) + 1, np.int64)
        np.cumsum([len(b) for b in enc], out=off[1:])
        buf = np.frombuffer(b"".join(enc) + b"\0", np.uint8)  # never empty: a zero-length string list still has a buffer
        check(self.L.eps_index_append_string_dictionary(self.h, int(first_code), len(enc), _p(off), _p(buf)))

    def config(self, L_master=500, L_local=None, prefilter=False, force_brute=False):
        L_local = L_master if L_local is None else L_local
        check(self.L.eps_index_config(self.h, int(L_master), int(L_local), int(bool(prefilter)), int(bool(force_brute))))

    def set_search_width(self, width):
        """1 = sequential expansion order of the reference (IntraQueryThreads=1); 2/4 = parallel expansion."""
        check(self.L.eps_index_set_search_width(self.h, int(width)))

    def set_filter_search(self, mode):
        """Graph branch of a filtered search (eps_index_set_filter_search): "post" (default) = the reference's
        post-filter of the unfiltered queue, which can return fewer than `limit` rows; "collect" = min(limit, L_local,
        passing rows) rows per query, from the passing rows the graph search evaluates and an exact scan of the
        passing rows for the queries it leaves short."""
        check(self.L.eps_index_set_filter_search(self.h, FILTER_SEARCH_MODES.get(mode, mode)))

    def set_graph_tuning(self, ring_slots=0, ctas_per_sm=0):
        """Launch geometry of the graph kernel (0 = auto): TMA row-ring slots per CTA, resident CTAs per SM."""
        check(self.L.eps_index_set_graph_tuning(self.h, int(ring_slots), int(ctas_per_sm)))

    def set_graph_screen(self, mode):
        """Graph-search screen of fresh neighbours on their 32-float principal-subspace sketch (L2, inner product and
        cosine; never changes results): 0 = off, 1 = on, 2 = auto (on when the sketch's basis carries >= 90 % of the
        table's variance)."""
        check(self.L.eps_index_set_graph_screen(self.h, int(mode)))

    def graph_screen_info(self):
        """dict(active=bool, share=explained-variance share of the basis (any metric) or -1 when there is no basis,
        n_screened=ids dropped so far)."""
        act, share, n = C.c_int(0), C.c_double(0.0), C.c_uint64(0)
        check(self.L.eps_index_graph_screen_info(self.h, C.byref(act), C.byref(share), C.byref(n)))
        return dict(active=bool(act.value), share=float(share.value), n_screened=int(n.value))

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
        return self._search_host(self.L.eps_search_batch, (self.h, _p(q), nq), nq, limit, filter_nodes, want_stats)

    def _search_host(self, fn, head, nq, limit, filter_nodes, want_stats):
        """fn(*head, limit, filter, n_filter, ids, dists, counts, stats) into new host arrays: ids, dists, counts, Stats."""
        ids = np.empty((nq, limit), np.int64)
        dists = np.empty((nq, limit), np.float64)
        counts = np.empty(nq, np.int64)
        st = StatsStruct()
        arr, n = filter_nodes_array(filter_nodes)
        check(fn(*head, int(limit), arr, n, _p(ids), _p(dists), _p(counts), C.byref(st) if want_stats else None))
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


def as_csr(rows):
    """scipy CSR matrix or (offsets, indices, values) -> contiguous (int64 offsets, int64 indices, float32 values)."""
    if hasattr(rows, "indptr") and hasattr(rows, "indices") and hasattr(rows, "data"):
        m = rows.tocsr()
        if not m.has_sorted_indices:
            m = m.sorted_indices()
        offsets, indices, values = m.indptr, m.indices, m.data
    else:
        offsets, indices, values = rows
    return (np.ascontiguousarray(offsets, np.int64), np.ascontiguousarray(indices, np.int64),
            np.ascontiguousarray(values, np.float32))


SPARSE_SEARCH_MODES = {"scan": 0, "graph": 1}


class SparseIndex(Index):
    """Device mirror of one sparse-vector field (eps_index_create_sparse): rows are appended as CSR.  Searches are exact
    scans by default; set_search_mode("graph") searches the graph that build() installed where the reference would
    (n_indexed >= 512, no prefilter / force_brute), with the reference's results at IntraQueryThreads = 1.
    build_inverted() gives an IP or cosine index posting lists that the exact scans read, and build_l2_screen() gives an
    L2 index posting lists that screen the exact scans' rows with a proven lower bound, both with the same results;
    extend_postings() extends either over appended rows without a rebuild, and postings() copies them out.  Config,
    deleted bits, attributes, string codes and dictionary, facets, build and get_graph work as on Index."""

    def __init__(self, metric, dim, capacity=0, device=0):
        self._open(metric, dim, None, capacity, device,
                   lambda h: self.L.eps_index_create_sparse(h, self.metric, self.dim, self.capacity, device))

    @property
    def rows(self):
        return int(self.L.eps_index_rows(self.h))

    def set_search_mode(self, mode):
        """"scan" (default): exact scan always; "graph": the reference's branch rule (eps_index_set_sparse_search)."""
        check(self.L.eps_index_set_sparse_search(self.h, SPARSE_SEARCH_MODES.get(mode, mode)))

    def build_inverted(self, n=None):
        """Posting lists of rows [0, n) (None: every mirrored row; 0 drops them) for an IP or cosine index
        (eps_index_build_sparse_inverted).  Results do not change; the exact scans read the covered rows' distances
        from the postings.  Rows appended later are scanned until the next build or extend_postings()."""
        check(self.L.eps_index_build_sparse_inverted(self.h, self.rows if n is None else int(n)))

    def inverted_info(self):
        """dict(rows=rows covered (0: no index), terms=distinct indices, postings=posting entries)."""
        r, t, p = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        check(self.L.eps_index_sparse_inverted_info(self.h, C.byref(r), C.byref(t), C.byref(p)))
        return dict(rows=int(r.value), terms=int(t.value), postings=int(p.value))

    def build_l2_screen(self, n=None):
        """Posting lists of rows [0, n) (None: every mirrored row; 0 drops them) for an L2 index
        (eps_index_build_sparse_l2_screen).  Results do not change; the exact scans and the build's kNN pass re-score
        only the covered rows whose proven lower bound can still place them among the k best.  Rows appended later are
        merged until the next build or extend_postings()."""
        check(self.L.eps_index_build_sparse_l2_screen(self.h, self.rows if n is None else int(n)))

    def l2_screen_info(self):
        """dict(rows=rows covered (0: no screen), rescored=(query, row) pairs this handle has re-scored so far)."""
        r, c = C.c_int64(0), C.c_uint64(0)
        check(self.L.eps_index_sparse_l2_screen_info(self.h, C.byref(r), C.byref(c)))
        return dict(rows=int(r.value), rescored=int(c.value))

    def extend_postings(self, n=None):
        """Extend the posting lists (the inverted index or the L2 screen) over the rows appended since they were built,
        up to row n (None: every mirrored row), without rebuilding them (eps_index_extend_sparse_postings).  The lists
        are then those a build over [0, n) makes."""
        check(self.L.eps_index_extend_sparse_postings(self.h, self.rows if n is None else int(n)))

    def postings(self):
        """The posting lists (eps_index_get_sparse_postings): dict(rows=rows covered, terms=distinct indices ascending
        (uint32), ptr=their offsets (int64, terms + 1 of them), post_rows=rows (int32), ascending within a term,
        post_values=values (float32))."""
        r, t, p = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        check(self.L.eps_index_get_sparse_postings(self.h, C.byref(r), C.byref(t), C.byref(p), None, None, None, None))
        terms = np.zeros(t.value, np.uint32)
        ptr = np.zeros(t.value + 1, np.int64)
        rows = np.zeros(p.value, np.int32)
        values = np.zeros(p.value, np.float32)
        check(self.L.eps_index_get_sparse_postings(self.h, None, None, None, _p(terms), _p(ptr), _p(rows), _p(values)))
        return dict(rows=int(r.value), terms=terms, ptr=ptr, post_rows=rows, post_values=values)

    def append(self, rows, first_row=None):
        """Append CSR rows (scipy CSR or (offsets, indices, values)) after the rows already mirrored."""
        off, idx, val = as_csr(rows)
        first = self.rows if first_row is None else int(first_row)
        check(self.L.eps_index_append_sparse_rows(self.h, first, off.size - 1, _p(off), _p(idx), _p(val)))

    def search(self, queries, limit, filter_nodes=None, want_stats=True):
        """Search of CSR queries (eps_search_sparse_batch), by the mode of set_search_mode.  Returns ids [nq,limit], dists float64, counts, Stats."""
        off, idx, val = as_csr(queries)
        nq = off.size - 1
        return self._search_host(self.L.eps_search_sparse_batch, (self.h, nq, _p(off), _p(idx), _p(val)), nq, limit,
                                 filter_nodes, want_stats)


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
