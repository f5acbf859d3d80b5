/*
 * epsilla_b200.h — C ABI of libepsilla_b200.so, the H100-native (sm_90a) implementation of
 * Epsilla's vector-search hot path.  POD-only: plain pointers and sizes, no C++/torch types.
 *
 * Every entry point cites the reference interface it replaces (paths relative to
 * epsilla-cloud/vectordb `engine/`).  INTEGRATION.md shows the reference-side binding (the
 * VecSearchExecutor / ANNGraphSegment adapter a maintainer would compile in).
 *
 * All functions return 0 on success or a reference ErrorCode-compatible non-zero value
 * (utils/error.hpp:11-41; DB_UNEXPECTED_ERROR-class codes); eps_last_error() gives the message of
 * the calling thread's last failure.  There is NO CPU fallback: every compute entry point fails
 * with EPS_ERR_NO_DEVICE when no CUDA device is usable.
 */
#ifndef EPSILLA_B200_H_
#define EPSILLA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define EPS_API __attribute__((visibility("default")))
#else
#define EPS_API
#endif

#define EPS_OK 0
#define EPS_ERR_INVALID_ARGUMENT 40005 /* utils/error.hpp INVALID_* family */
#define EPS_ERR_UNSUPPORTED 40006
#define EPS_ERR_NO_DEVICE 50001 /* infra error: CUDA runtime/device unavailable */
#define EPS_ERR_CUDA 50002
#define EPS_ERR_OOM 50003

/* meta::MetricType, db/catalog/meta_types.hpp:47-52 */
#define EPS_METRIC_L2 1
#define EPS_METRIC_COSINE 2
#define EPS_METRIC_IP 3

typedef struct eps_index eps_index;

/* One filter-expression node: the fields of query::expr::ExprNode (query/expr/expr_types.hpp:77-90)
 * that numeric / bool predicates use, with field_name already resolved by the caller through
 * TableSegmentMVP::field_name_mem_offset_map_ to the byte offset inside an attribute row
 * (-1: no field, -2: the "@distance" pseudo-field, query/expr/expr_evaluator.cpp:143-145).
 * node_type / value_type carry the reference enum ordinals (expr_types.hpp:11-48, :67-74).
 * Nodes are in the parser's order: children before parents, root last
 * (db/execution/vec_search_executor.cpp:848).
 * Strings: a StringAttr node carries the string-column index in field_offset, a StringConst node the literal's
 * dictionary code in int_value (-1 if the literal is not in the dictionary); string EQ / NE compare codes; the
 * caller lowers `x IN (a, b, ..)` to `x = a OR x = b ..` (integration/epsilla_b200_dropin.cpp does).
 * LIKE (node_type 29, query/expr/expr_evaluator.cpp:229-241) takes two children, each a StringAttr or a StringConst
 * node (anything else: EPS_ERR_UNSUPPORTED); its value type is BOOL.  It matches byte for byte as the reference does:
 * an empty pattern matches only the empty string, the pattern "%" matches every string, otherwise '%' matches any run
 * of bytes and '_' one byte, neither across a '\n' or '\r', every other byte is a literal, case-sensitive, and the
 * pattern must cover the whole string.  The strings behind the codes come from eps_index_append_string_dictionary: a
 * LIKE literal's code must be a mirrored code, and a column a LIKE reads must hold mirrored codes only; otherwise the
 * search fails with EPS_ERR_INVALID_ARGUMENT before any launch.  Each call evaluates its LIKE nodes once, on the
 * device, before the search: per dictionary code when one side is a literal, per row when both are columns.  Strings
 * and patterns of any length are matched.  String concatenation and NEARBY nodes are rejected with
 * EPS_ERR_UNSUPPORTED. */
typedef struct eps_filter_node {
  int64_t node_type;
  int64_t value_type;
  int64_t left;  /* size_t index, -1 = none */
  int64_t right; /* size_t index, -1 = none */
  int64_t int_value;
  double double_value;
  int64_t bool_value;
  int64_t field_offset;
} eps_filter_node;

/* Counters the reference computes and discards (tmp_count_computation,
 * db/execution/vec_search_executor.cpp:409,441,479) plus kernel timing. */
typedef struct eps_stats {
  uint64_t n_dist;     /* (query,row) distance evaluations, seed set included */
  uint64_t n_seed;     /* of which seed-set evaluations (L per graph query) */
  uint64_t n_expand;   /* graph vertices expanded */
  uint64_t n_edges;    /* CSR entries read by expansions */
  uint64_t n_queries;
  double kernel_ms;    /* device time of the dominant kernel(s) of this call (CUDA events) */
  double total_ms;     /* device time of the whole call incl. copies (CUDA events) */
  uint64_t kernel_launches; /* launches of this call's search, the LIKE match pass included */
  uint64_t n_redone;   /* exact scan: queries the coarse-pass guard sent back (fp32 scan or a larger candidate list);
                          EPS_FILTER_SEARCH_COLLECT: queries answered by the scan over the passing rows */
} eps_stats;

/* Graph-build parameters.  Defaults (pass NULL) follow NSGConfig(45, 50, 300, 100) and the
 * NN-descent settings of the reference (db/ann_graph_segment.cpp:28-29, db/index/knn/knn.hpp:90-95). */
typedef struct eps_build_params {
  int32_t knn_k;           /* kNN-graph list length (reference K = 100) */
  int32_t out_degree;      /* max out-degree after pruning (reference 50) */
  int32_t candidate_pool;  /* pruning pool cap (reference 300) */
  int32_t search_length;   /* search-collect beam (reference 45) */
  int32_t nnd_iters;       /* max NN-descent iterations (reference 1000, stops at rate < 0.001) */
  int32_t nnd_sample;      /* per-vertex sample size S of the local join */
  int32_t exact_knn_below; /* use exact all-pairs kNN when n <= this (0 = library default) */
  int32_t seed;
  float nnd_delta;         /* NN-descent stop rate (reference 0.001) */
  int32_t min_degree;      /* degree floor: top up with nearest rejected candidates (0 = default 32) */
  float alpha;             /* occlusion slack: keep p unless alpha*d(r,p) < d(v,p) (0 = 1.0, the reference rule) */
  int32_t reserved;
} eps_build_params;

/* ---------------------------------------------------------------------------------------------
 * Index lifetime.  Replaces the state a VecSearchExecutor captures at construction
 * (db/execution/vec_search_executor.hpp:61-74, .cpp:29-73) plus the device mirror of the
 * TableSegmentMVP fields it reads (db/table_segment_mvp.hpp:65-88).
 * --------------------------------------------------------------------------------------------- */

/* host_vectors: TableSegmentMVP::vector_tables_[f] (row-major [capacity_rows x dim] float, never
 * reallocated — db/table_segment_mvp.cpp:106-111).  May be NULL when rows are supplied with
 * eps_index_adopt_device_rows().  device = CUDA ordinal. */
EPS_API int eps_index_create(eps_index** out, int metric, int64_t dim, const float* host_vectors, int64_t capacity_rows,
                     int device);
EPS_API void eps_index_destroy(eps_index* ix);

/* A read-only VIEW of an index for concurrent searches: the view shares the base's device table, graph, deleted bits
 * and attribute mirrors and has its own stream and scratch, so batches submitted to the base and to its views (from
 * different host threads, or with sync = 0) overlap on the device — the engine's analogue is the pool of
 * NumExecutorPerField executors over one field (db/execution/executor_pool.hpp, config.hpp:17).  The executor
 * parameters (eps_index_config, width, coarse mode) are copied at creation and may then be set per view.  While an
 * index has live views every call that would modify it (rows, graph, deleted bits, attributes, build) fails with
 * EPS_ERR_INVALID_ARGUMENT, and so does the same call on a view.  Destroy the views before the base. */
EPS_API int eps_index_create_view(eps_index* base, eps_index** out);

/* Mirror rows [uploaded, n_rows_now) to HBM; n_rows_now = record_number_ snapshot
 * (db/execution/vec_search_executor.cpp:839). */
EPS_API int eps_index_sync_rows(eps_index* ix, int64_t n_rows_now);

/* The device copy of the vector table ([rows x dim] float, row-major) and how many rows are mirrored; lets a second
 * index (the graph build that TableMVP::Rebuild runs beside the live executors, db/table_mvp.cpp:143-195) work on
 * the same HBM rows through eps_index_adopt_device_rows instead of uploading the table again. */
EPS_API const float* eps_index_device_rows(eps_index* ix);
EPS_API int64_t eps_index_rows(eps_index* ix);

/* Use an already device-resident [n_rows x dim] float table (not copied, not owned). */
EPS_API int eps_index_adopt_device_rows(eps_index* ix, const float* d_vectors, int64_t n_rows);

/* Install a reference CSR graph: ANNGraphSegment::{record_number_, offset_table_, neighbor_list_,
 * navigation_point_} (db/ann_graph_segment.hpp:45-49).  Host pointers; ids narrowed to int32 on
 * device.  n_indexed < 512 latches brute-force mode (vec_search_executor.hpp:28, .cpp:62). */
EPS_API int eps_index_set_graph(eps_index* ix, int64_t n_indexed, const int64_t* offset_table, const int64_t* neighbor_list,
                        int64_t navigation_point);

/* ANNGraphSegment::BuildFromVectorTable (db/ann_graph_segment.cpp:201-242) on device over rows
 * [0, n): kNN graph (db/index/knn) + NSG-style refinement (db/index/nsg), installed into the index. */
EPS_API int eps_index_build(eps_index* ix, int64_t n, const eps_build_params* params);

/* Link rows [n_indexed, n) of the mirrored table into the installed graph, so that afterwards n_indexed = n and searches
 * no longer scan those rows as the tail (vec_search_executor.cpp:885-900) — without the full rebuild that
 * TableMVP::Rebuild runs (db/table_mvp.cpp:94-203).  params as for eps_index_build (NULL = defaults); knn_k,
 * out_degree, candidate_pool, search_length, min_degree, alpha and seed are read.
 * Works on any installed dense graph: one built by eps_index_build or installed by eps_index_set_graph (a graph the
 * reference built included).  n == n_indexed does nothing and returns EPS_OK (the graph stays bitwise identical).
 * Errors: no graph installed, n < n_indexed, n above the mirrored rows, a view, an index with live views, or a sparse
 * index: EPS_ERR_INVALID_ARGUMENT; n >= 2^31: EPS_ERR_UNSUPPORTED; a failed argument check changes nothing.
 * Like the build, every row is indexed, deleted or not (ann_graph_segment.cpp:201).  The new rows are linked in
 * chunks of 65 536: each new row's candidates are the pool of a graph search over the graph as the previous chunks left
 * it (field metric, width 4, L = 128) merged with its exact kNN among the rows of its chunk (field metric), selected
 * with the build's L2 SelectEdge rule, and offered as reverse edges to their targets.  A new row gets at most
 * min(out_degree, 64) selected edges.  An old row changes only by being re-selected over its row and the new rows
 * offered to it, by having offered rows appended while it fits out_degree, or by repair edges appended at its end (the
 * build's repair: a vertex the navigation point does not reach is attached to the nearest reached vertex its own search
 * finds); a row already wider than out_degree (e.g. the navigation point with its component entries) is left as it is.  The navigation point does not change.  On return every row of [0, n) is
 * reachable from it.  The same table, graph, n and params give the same graph on every run.
 * The graph screen's basis, mean and share are kept, not re-sampled from the grown table; stored row sketches are
 * extended to the new rows.  The call's own searches are not screened and do not count in n_screened.
 * Device memory the call adds: a second CSR while the graph is spliced, [n x 64] int32 adjacency rows (which the search
 * keeps anyway), O(n) int32 / int64 arrays and per-chunk buffers (DESIGN.md §K4, B4). */
EPS_API int eps_index_extend_graph(eps_index* ix, int64_t n, const eps_build_params* params);

/* Copy the installed graph out as the reference's int64 CSR (the payload of ann_graph_<field>.bin,
 * db/ann_graph_segment.cpp:171-184).  Pass NULL buffers to query sizes. */
EPS_API int eps_index_get_graph(eps_index* ix, int64_t* n_indexed, int64_t* n_edges, int64_t* offset_table,
                        int64_t* neighbor_list, int64_t* navigation_point);

/* ConcurrentBitset bytes of TableSegmentMVP::deleted_ (utils/concurrent_bitset.cpp:9-19). */
EPS_API int eps_index_set_deleted(eps_index* ix, const uint8_t* bitset, int64_t nbytes);

/* TableSegmentMVP::attribute_table_ with row stride primitive_offset_
 * (db/table_segment_mvp.cpp:99, query/expr/expr_evaluator.cpp:61-102). */
EPS_API int eps_index_set_attrs(eps_index* ix, const char* attribute_table, int64_t row_stride, int64_t n_rows);

/* String columns (TableSegmentMVP::var_len_attr_table_[column], db/table_segment_mvp.hpp:82) are mirrored as
 * DICTIONARY CODES: the caller keeps one string -> int32 dictionary per table and appends the codes of new rows
 * [first_row, first_row + count) here; filter nodes then compare codes (query/expr/expr_evaluator.cpp:110-125,
 * :176-190: StrEvaluate / string EQ, NE / IN).  column = the field's index in var_len_attr_table_ (< 8).
 * Rows may be written again (first_row below the rows already mirrored).  For LIKE the call also records the range of
 * the column's codes on the host; that range only widens, unless a call rewrites every row from row 0.  So after a
 * partial rewrite that removes an out-of-range code, a LIKE on the column is still refused until the whole column is
 * written again. */
EPS_API int eps_index_set_string_codes(eps_index* ix, int column, int64_t first_row, const int32_t* codes, int64_t count);

/* The strings of dictionary codes [first_code, first_code + count), for LIKE: code first_code + i is
 * bytes[offsets[i] .. offsets[i+1]) (offsets[0] need not be 0; any byte, NUL included).  Append-only: first_code must
 * equal the number of codes already mirrored.  A LIKE literal gets a code like any other string (the caller adds it
 * to its dictionary and appends its bytes), so a row with the same text later gets the same code.  One dictionary per
 * index; views share it, and appending while the index has live views fails like every other mirror update.  A gap,
 * a negative count, null buffers or offsets that go backwards: EPS_ERR_INVALID_ARGUMENT; more than 2^31 - 1 codes in
 * all: EPS_ERR_UNSUPPORTED. */
EPS_API int eps_index_append_string_dictionary(eps_index* ix, int64_t first_code, int64_t count, const int64_t* offsets,
                                               const char* bytes);

/* Executor parameters snapshotted at construction (db/table_mvp.cpp:83-87): L_master, L_local
 * (config.hpp MasterQueueSize / LocalQueueSize), prefilter_enabled_.  force_brute != 0 makes every
 * search an exact scan (what the reference does for un-indexed tables). */
EPS_API int eps_index_config(eps_index* ix, int64_t L_master, int64_t L_local, int prefilter, int force_brute);

/* Graph-search expansion width: how many unchecked queue entries are expanded per iteration.  1 (default)
 * reproduces the reference at IntraQueryThreads = 1 exactly; 2 .. 8 are the device analogue of the reference's
 * IntraQueryThreads > 1 (config.hpp:18, default 4): candidates expanded in parallel against a slightly stale
 * bound — higher throughput, results not bit-identical to the sequential order (as in the reference) but the same on
 * every run. */
EPS_API int eps_index_set_search_width(eps_index* ix, int width);

/* How the graph branch of a filtered dense search answers (eps_search_batch, eps_search_batch_device and, through it,
 * eps_search_batch_sharded).  It applies only where the reference searches its graph (n_indexed >= 512, no prefilter,
 * no force_brute) and the filter is non-empty; every other call is unchanged.  A view copies the mode at creation and
 * may set its own.
 *   EPS_FILTER_SEARCH_POST (default): the reference's post-filter (vec_search_executor.cpp:906-927).  The page holds the
 *     passing rows of the unfiltered queue of L candidates, so a selective filter can return fewer than `limit` rows
 *     even when enough rows pass.
 *   EPS_FILTER_SEARCH_COLLECT: every query returns min(cap, P) rows, cap = min(n_indexed, limit, L_local, L) and P = the
 *     rows that are not deleted and pass the filter.  The graph search navigates as in POST and also keeps the best cap
 *     passing rows among all the rows it evaluates; the passing rows appended after the build are merged in exactly.
 *     A query left with fewer than min(cap, P) rows, or every query when P is small, is answered by an exact scan of
 *     the passing rows alone, with the distances of the prefilter scan under eps_index_set_coarse(0);
 *     eps_stats.n_redone counts those queries.  Results are ascending by (distance, id).  POST's rows of a query are
 *     the first rows of COLLECT's for the same query when every row is indexed and the query was not scanned.
 *     A filter whose root compares "@distance" fails with EPS_ERR_UNSUPPORTED before any launch.  The call
 *     synchronises the index's stream (to read P and the number of short queries), whatever `sync` says.
 * A sparse index, an unknown mode or a null index: EPS_ERR_INVALID_ARGUMENT. */
#define EPS_FILTER_SEARCH_POST 0
#define EPS_FILTER_SEARCH_COLLECT 1
EPS_API int eps_index_set_filter_search(eps_index* ix, int mode);

/* Launch geometry of the graph-search kernel (performance knob, never changes results): ring_slots = shared-memory row slots per CTA that TMA
 * bulk copies land in (0 = auto: ~48 KB of rows), ctas_per_sm = cap on resident CTAs, i.e. in-flight queries, per SM
 * (0 = whatever fits).  No reference counterpart (the CPU executor has no such geometry). */
EPS_API int eps_index_set_graph_tuning(eps_index* ix, int ring_slots, int ctas_per_sm);

/* Graph-search screen (L2, inner product and cosine; never changes results).  When a graph is installed (eps_index_build,
 * eps_index_set_graph), the index computes the top-32 principal subspace P~ of its rows (covariance of up to 2^20 rows,
 * subspace iteration in double) and, when the screen is on, a 32-float sketch fl(P~(x - mu)) of every indexed row with
 * a bound on its rounding error: 132 bytes per row next to the row's 4 * dim (140 for inner product and cosine, which
 * also keep the norm of the row's residual outside the subspace and its product with the mean).  The search then reads
 * the sketch of a fresh neighbour first and fetches its row only when a proven lower bound on its distance, taken from
 * the sketches, cannot reject it (DESIGN.md §K2; for inner product and cosine, from an upper bound on the fp32 dot
 * product); ids, distances and all eps_stats counters are those of the unscreened search.
 * mode: EPS_GRAPH_SCREEN_OFF, _ON, or _AUTO (default): on when the 32 components carry at least 90 % of the sampled
 * variance, i.e. when the rows lie close to a low-dimensional subspace.  Tables below 128 dimensions are not screened. */
#define EPS_GRAPH_SCREEN_OFF 0
#define EPS_GRAPH_SCREEN_ON 1
#define EPS_GRAPH_SCREEN_AUTO 2
EPS_API int eps_index_set_graph_screen(eps_index* ix, int mode);
/* State of the screen: active = whether the next graph search screens, share = share of the sampled variance the
 * basis carries (-1 when no basis was computed: no graph, below 128 dimensions, or mode off since the install),
 * n_screened = fresh neighbours dropped by the screen in all graph searches of this handle so far, with or without a
 * stats argument (waits for the handle's stream).  The count is kept here rather than in eps_stats so that eps_stats
 * keeps its size and layout.  The sketch is computed when a graph is installed and when this mode changes, never
 * inside a search: after eps_index_adopt_device_rows, which drops it, the screen stays off until the next install or
 * mode change.  If the sketch cannot be allocated, the index works on without the screen. */
EPS_API int eps_index_graph_screen_info(eps_index* ix, int* active, double* share, uint64_t* n_screened);

/* Precision of the COARSE pass of large-batch exact scans (nq >= 64): 0 = none (fp32 SIMT tiles only),
 * 1 = wgmma TF32 on the fp32 rows (default), 2 = wgmma BF16 on a bf16 mirror of the table
 * (+50 % HBM).  Whatever the mode, the k' = k + max(118, k) best coarse candidates of every query are re-evaluated
 * with the exact fp32 direct form, so returned distances are fp32-exact, and a GUARD checks that no row outside
 * the candidate list can belong to the answer: with T = the k'-th best coarse distance, e_k = the exact k-th best,
 * E = the largest |coarse - exact| over the batch's own k' x nq re-scored rows, M = the table's largest row norm and
 * M_s = the largest norm among those re-scored rows, a query is safe when e_k + 2 E max(1, M / M_s) <= T; unsafe
 * queries are redone on the fp32 path (or, when many are unsafe, the batch is redone with a 4x larger k' that the
 * index remembers).  eps_stats.n_redone counts them.  The guard is on by default.
 * What the guard assumes: a row's coarse error is at most the sampled E scaled by its norm relative to the sample's.
 * The rule rests on sampled errors, not on a worst-case bound: rows of the same norm whose products cancel in a way
 * none of the sampled rows does can still, in principle, escape it.  With the guard off the answer is the coarse
 * candidate list re-scored, with no check. */
EPS_API int eps_index_set_coarse(eps_index* ix, int mode);
EPS_API int eps_index_set_coarse_guard(eps_index* ix, int on);

/* ---------------------------------------------------------------------------------------------
 * Search.  Replaces VecSearchExecutor::Search (db/execution/vec_search_executor.cpp:833-935),
 * batched: query i's results are out_ids[i*limit .. i*limit+out_counts[i]) (internal row ids,
 * ascending (distance,id)), out_dists likewise (L2^2 / -IP / 1-cos, widened to double like
 * VecSearchExecutor::distance_, vec_search_executor.hpp:52).  Unused slots: id -1, dist +inf.
 * Cosine queries must already be normalised (db/table_mvp.cpp:337-349); see eps_normalize().
 * HOST buffers in and out; the call includes the H2D / D2H copies.
 * --------------------------------------------------------------------------------------------- */
EPS_API int eps_search_batch(eps_index* ix, const float* queries, int64_t nq, int64_t limit, const eps_filter_node* filter,
                     int64_t n_filter, int64_t* out_ids, double* out_dists, int64_t* out_counts, eps_stats* stats);

/* Same search with DEVICE-resident queries and outputs (ids int64, dists float, counts int64),
 * asynchronous on the index's stream unless sync != 0 (a filtered call in EPS_FILTER_SEARCH_COLLECT that takes the
 * graph branch synchronises the stream in any case).  For pipelines that keep queries in HBM and
 * for the multi-GPU exchange (the per-shard results feed an NCCL all-gather). */
EPS_API int eps_search_batch_device(eps_index* ix, const float* d_queries, int64_t nq, int64_t limit,
                            const eps_filter_node* filter, int64_t n_filter, int64_t* d_out_ids, float* d_out_dists,
                            int64_t* d_out_counts, eps_stats* stats, int sync);

/* k-way merge of per-shard results (the exchange step of a row-sharded table; the single-segment
 * reference has the same two-source merge between graph and tail results,
 * vec_search_executor.cpp:885-900).  d_ids/d_dists: [n_shards x nq x k] gathered results with
 * GLOBAL ids; output [nq x k] ascending (distance,id).  Runs on `device`. */
EPS_API int eps_merge_shards_device(int device, const int64_t* d_ids, const float* d_dists, int64_t n_shards, int64_t nq,
                            int64_t k, int64_t* d_out_ids, float* d_out_dists);

/* ---------------------------------------------------------------------------------------------
 * Facets.  Replaces FacetExecutor::Aggregate (db/execution/aggregation.hpp:232-300), batched over nq result
 * lists: one group-by expression (key_type = the ValueType ordinal of its root, query/expr/expr_types.hpp:67-74:
 * 0 STRING -> the key is the row's dictionary code, 1 INT -> truncated like the reference's (int64_t) cast, 2 DOUBLE,
 * 3 BOOL) and up to 8 aggregates, each an inner numeric expression with a type (NodeType ordinals 30 SUM, 31 MIN,
 * 32 MAX, 33 COUNT — db_server.cpp:362-382 parses "SUM(expr)" into exactly this pair; COUNT's inner expression is
 * "1").  Expressions are eps_filter_node arrays like the filters; "@distance" reads dists[i] (pass NULL when the
 * caller has no distances: has_distance = false).  Output per query q: out_groups[q] groups in order of first
 * appearance, keys out_keys[q*limit + g], values out_values[(q*limit + g)*n_aggs + a] (double, like the reference's
 * aggregators).  HOST buffers in and out.
 * INT keys follow the reference's (int64_t) cast as x86-64 computes it: a key that is NaN or lies outside
 * [-2^63, 2^63) (a division by zero, +-inf, an int64 product that overflows) becomes INT64_MIN, so with int4 columns
 * a = [0, 5, -5, 7, 0, 1, 2, 3] and b = [0, 0, 0, 2, 1, 1, 1, 1], "a / b" groups COUNT(*) as {0: 1, 1: 1, 2: 1, 3: 2,
 * INT64_MIN: 3} and "a % b" as {0: 4, 1: 1, INT64_MIN: 3}.  A NaN DOUBLE key makes the reference fail
 * (FacetExecutor::Project throws); the device's grouping of such keys is unspecified.
 * --------------------------------------------------------------------------------------------- */
typedef struct eps_facet {
  const eps_filter_node* key_nodes;
  int64_t n_key_nodes;
  int32_t key_type;
  int32_t n_aggs;
  const eps_filter_node* agg_nodes[8];
  int64_t n_agg_nodes[8];
  int32_t agg_types[8];
} eps_facet;
EPS_API int eps_facet_batch(eps_index* ix, const int64_t* ids, const double* dists, const int64_t* counts, int64_t nq,
                            int64_t limit, const eps_facet* spec, double* out_keys, double* out_values, int64_t* out_groups);

/* ---------------------------------------------------------------------------------------------
 * Row-sharded tables (one shard per GPU, one process or thread per GPU).  No reference counterpart: the reference
 * is single-segment (db/table_mvp.hpp:110); its own two-source merge of graph and tail results
 * (vec_search_executor.cpp:885-900) is the model.  The exchange (ONE ncclAllGather of nq*k*12 bytes per rank +
 * a k-way merge kernel) runs on the index's stream inside the library; NCCL is bound at run time (libnccl.so.2).
 * --------------------------------------------------------------------------------------------- */
typedef struct eps_shard_group eps_shard_group;

/* 128 bytes identifying a new group: call once (on any rank), hand the bytes to every rank by any host
 * transport (the reference engine would carry them in its cluster metadata), then create the group everywhere. */
EPS_API int eps_shard_unique_id(void* out128);
/* Collective over all ranks of the group (ncclCommInitRank).  device = the CUDA ordinal this rank's shard lives on. */
EPS_API int eps_shard_group_create(eps_shard_group** out, const void* unique_id128, int rank, int world, int device);
EPS_API void eps_shard_group_destroy(eps_shard_group* g);
/* VecSearchExecutor::Search over a row-sharded table.  Every rank passes the SAME device-resident query batch and
 * its own shard index; id_base = global id of the shard's row 0.  Output (device, on every rank): the merged global
 * top-k, ids int64 [nq x k] (-1 padded), dists float, ascending (distance, id).  Asynchronous on the index's stream
 * unless sync != 0 (stats != NULL also synchronises the local search to read its counters). */
EPS_API int eps_search_batch_sharded(eps_shard_group* g, eps_index* ix, int64_t id_base, const float* d_queries, int64_t nq,
                                     int64_t k, const eps_filter_node* filter, int64_t n_filter, int64_t* d_out_ids,
                                     float* d_out_dists, eps_stats* stats, int sync);

/* engine::Normalize (db/vector.cpp:60-69) for nq host vectors in place, on device. */
EPS_API int eps_normalize(int device, float* host_vectors, int64_t nq, int64_t dim);

/* Distances of nq query / row pairs (GetDistFunc(...)(a, b, &dim), db/index/index.cpp:10-35):
 * out[i] = dist(a[i], b[i]).  Host buffers.  Used by parity tests of rows A1-A3. */
EPS_API int eps_pair_distances(int device, int metric, const float* a, const float* b, int64_t n_pairs, int64_t dim,
                       float* out);

/* ---------------------------------------------------------------------------------------------
 * Sparse-vector fields (SPARSE_VECTOR_FLOAT / _DOUBLE, db/vector.hpp:13-20): TableSegmentMVP::var_len_attr_table_
 * rows of {index, value} pairs mirrored as a device CSR (int64 row offsets, interleaved {uint32 index, float value}
 * elements, one fp32 |row|^2 per row for cosine).
 *
 * These calls work on a sparse index as on a dense one: eps_index_set_deleted, eps_index_set_attrs,
 * eps_index_set_string_codes, eps_index_config, eps_index_create_view (the view shares the CSR), eps_index_build,
 * eps_index_get_graph, eps_index_rows, eps_facet_batch.  The dense-only calls (sync_rows, adopt_device_rows,
 * device_rows, set_graph, extend_graph, set_coarse, set_search_width, set_filter_search, set_graph_tuning, eps_search_batch*,
 * eps_search_batch_sharded) fail with EPS_ERR_INVALID_ARGUMENT (device_rows returns NULL).
 * --------------------------------------------------------------------------------------------- */

/* dim = the field's vector_dimension_ (< 2^32 - 1): every index of a row is < dim (table_segment_mvp.cpp:525-533).
 * capacity_rows is a hint; the mirror grows as rows are appended. */
EPS_API int eps_index_create_sparse(eps_index** out, int metric, int64_t dim, int64_t capacity_rows, int device);

/* Append rows [first_row, first_row + n_rows); first_row must equal the rows already mirrored.  Row r is
 * indices / values [offsets[r], offsets[r+1]) (offsets[0] need not be 0).  Rows with a negative index, an index
 * >= dim, or indices that are not strictly increasing are rejected with EPS_ERR_INVALID_ARGUMENT, as the reference's
 * insert rejects them (table_segment_mvp.cpp:539-550); nothing is appended then.  Empty rows are legal.  Values are
 * stored as given (the reference normalises cosine rows at insert, :556-562). */
EPS_API int eps_index_append_sparse_rows(eps_index* ix, int64_t first_row, int64_t n_rows, const int64_t* offsets,
                                         const int64_t* indices, const float* values);

/* VecSearchExecutor::Search of nq sparse queries (CSR like the rows; indices strictly increasing, < 2^32 - 1), with the
 * output contract of eps_search_batch.  Distances are bit-identical to GetL2DistSqr / GetInnerProductDist /
 * GetCosineDist (db/vector.cpp:7-100, row = v1, query = v2): the same sequential fp32 sums in the same order, no FMA.
 * Cosine queries must already be normalised (db/table_mvp.cpp:337-349), like dense ones.
 * In the default mode (EPS_SPARSE_SEARCH_SCAN) a sparse index ALWAYS answers by the exact scan over all mirrored rows,
 * with the reference's brute-force caps (prefilter / force_brute: limit results; otherwise min(limit, L_local)), even
 * when a graph is installed.  This is the one deliberate deviation from the reference: where it would search its graph
 * (n_indexed >= 512), the GPU returns the exact top-k.  eps_stats.n_dist counts nq x the rows scanned.
 * In EPS_SPARSE_SEARCH_GRAPH mode (eps_index_set_sparse_search) the index follows the reference's branch rule: prefilter,
 * force_brute or n_indexed < 512 select the same exact scan; otherwise the installed graph over rows [0, n_indexed) is
 * searched with queue length min(L_master, n_indexed) in the reference's sequential order (IntraQueryThreads = 1), rows
 * [n_indexed, total) are scanned, and the two are merged and post-filtered as Search does (:885-927).  The ids, the
 * distances (bitwise) and the distance-evaluation counts are then those of the reference at IntraQueryThreads = 1;
 * eps_stats.n_dist counts seeds, fresh neighbours and tail rows, n_seed the seeds, n_expand / n_edges the expansions
 * and the adjacency entries they read.
 * Cosine with an empty row or an empty query gives 0/0 = NaN (the reference's std::sort order of such entries is
 * unspecified): NaN distances sort after every number.
 * eps_index_build on a sparse index installs the exact out_degree-NN lists (field metric, self excluded), the L2
 * nearest row to the reference's sparse centre (nsg.cpp:120-135) as navigation point, and repair edges that make every
 * row reachable from it.  A build on an index with posting lists (eps_index_build_sparse_inverted) reads the covered
 * rows' kNN distances from them, bitwise the merge's, so the graph is the same; the build neither creates nor drops
 * posting lists.  HOST buffers in and out. */
EPS_API int eps_search_sparse_batch(eps_index* ix, int64_t nq, const int64_t* q_offsets, const int64_t* q_indices,
                                    const float* q_values, int64_t limit, const eps_filter_node* filter, int64_t n_filter,
                                    int64_t* out_ids, double* out_dists, int64_t* out_counts, eps_stats* stats);

/* How eps_search_sparse_batch answers on a sparse index (see there).  A view starts with its base's mode and may set
 * its own.  A dense index or an unknown mode: EPS_ERR_INVALID_ARGUMENT. */
#define EPS_SPARSE_SEARCH_SCAN 0   /* default: the exact scan always */
#define EPS_SPARSE_SEARCH_GRAPH 1  /* the reference's branch rule: graph search + tail scan where it searches its graph */
EPS_API int eps_index_set_sparse_search(eps_index* ix, int mode);

/* Inverted index of a sparse IP or cosine index: per-term posting lists of the rows [0, n).
 * What it does to results: nothing; it is not a search mode.  Every exact sparse scan a search call runs (the
 * EPS_SPARSE_SEARCH_SCAN default; the brute-force, prefilter and force_brute branches of graph mode; the tail scan of
 * graph mode) computes the distances of the covered rows from the postings and merges the uncovered rows [n, rows) as
 * before, into the same distance tile.  Each covered row's matched products row[i] * query[i] are added in increasing
 * index order from 0, in fp32 without FMA, as the merge adds them (db/vector.cpp:7-47), so the distances are bitwise
 * those of the scan: ids, distances, counts and the n_dist / n_seed / n_expand / n_edges counters are what they are
 * without the index.  Only kernel_launches and the timings change.
 * Appends: rows appended after the build are scanned until the caller builds again or extends the lists
 * (eps_index_extend_sparse_postings), the way the graph's tail is.
 * n = 0 drops the index.  A build replaces the previous index only once it has succeeded; a refused or failed call
 * leaves the previous index as it was.  Refusals: an L2 index, EPS_ERR_UNSUPPORTED (its merged order also adds the
 * row-only and query-only terms); a null or dense index, n < 0, n above the mirrored rows, a view, or an index with live
 * views, EPS_ERR_INVALID_ARGUMENT.  Views created after the build share the index; a detached view has none.
 * Device memory: 8 B per posting (one per element of the covered rows) plus 12 B per distinct index.  The build needs,
 * while it runs, 16 B more per posting (sort keys and a second value buffer) plus the sort's scratch, beside the
 * previous index, which is freed when the new one is installed.  A search call adds 16 B per query element; a graph
 * build (eps_index_build) 16 B per element of its largest 8192-row query chunk. */
EPS_API int eps_index_build_sparse_inverted(eps_index* ix, int64_t n);
/* Rows covered (0 = none), distinct terms, postings.  Any pointer may be NULL.  A null or dense index:
 * EPS_ERR_INVALID_ARGUMENT. */
EPS_API int eps_index_sparse_inverted_info(eps_index* ix, int64_t* n_rows, int64_t* n_terms, int64_t* n_postings);

/* L2 screen of a sparse L2 index: the posting lists of rows [0, n), with the same arrays, layout and build as
 * eps_index_build_sparse_inverted (whose info reports their rows, terms and postings on an L2 index too).
 * What it does to results: nothing; it is not a search mode.  Every exact sparse scan a search call runs (the places
 * listed for the inverted index) and the kNN pass of eps_index_build give each covered row a proven lower bound LB of
 * the reference's L2 distance D_ref from the postings, and compute D_ref itself (the merge of the scan) only for rows
 * that can still be among the K best: per chunk of rows, the K rows with the smallest bounds are re-scored, T = the
 * largest of their distances, and every row with LB <= T is re-scored; the others cannot beat those K rows.  Ids,
 * counts, bitwise distances and the n_dist / n_seed / n_expand / n_edges counters are what they are without the screen,
 * and eps_index_build installs the same graph.  Only kernel_launches and the timings change.  A search whose filter
 * compares "@distance" (outside prefilter mode) takes the merge for every row and re-scores nothing.
 * The bound: with m_r and m_q the row's and the query's element counts, m = m_r + m_q, u = 2^-24,
 * gamma_k = k u / (1 - k u), D the real distance, every term the reference adds is non-negative, so when nothing
 * overflows |D_ref - D| <= gamma_{m+2} D + m 2^-149 (the second term covers products that underflow).  D is bounded
 * below from the posting lists' fp32 dot of the matched elements, the stored fp32 |row|^2, the query's fp32 |q|^2
 * (each a sequential sum with a known error bound) and m_r, every step rounded toward -inf (sparse_inverted.cu
 * restates the derivation).  Rows with a non-finite |row|^2 (NaN or +-inf values, squares that overflow), pairs with
 * m + 2 > 2^20, and every row for a query with a non-finite |q|^2 are always re-scored.
 * Lifecycle as for the inverted index: rows appended after the build are merged until the caller builds again or
 * extends the lists (eps_index_extend_sparse_postings); n = 0 drops the
 * lists; a refused or failed call leaves the previous state; views created after the build share it.  Refusals, all
 * EPS_ERR_INVALID_ARGUMENT: a null or dense index, an inner-product or cosine index (eps_index_build_sparse_inverted
 * gives those exact distances from the same lists), n < 0, n above the mirrored rows, a view, or an index with live
 * views.  Device memory: as for the inverted index, plus 8 B x nq x k (x the scan's row splits) for the K best keys. */
EPS_API int eps_index_build_sparse_l2_screen(eps_index* ix, int64_t n);
/* Rows the L2 screen covers (0 = none, and 0 on an inner-product or cosine index) and the (query, row) pairs this
 * handle's searches and builds have re-scored through the merge so far; waits for the index's stream.  Any pointer may
 * be NULL.  A null or dense index: EPS_ERR_INVALID_ARGUMENT. */
EPS_API int eps_index_sparse_l2_screen_info(eps_index* ix, int64_t* n_rows, uint64_t* n_rescored);

/* Extend the posting lists of a sparse index (the inverted index of an IP or cosine index, the L2 screen of an L2 one)
 * over the rows [inv_rows, n) appended since they were built, without rebuilding them.  Afterwards the lists are,
 * byte for byte, those eps_index_build_sparse_inverted(ix, n) or eps_index_build_sparse_l2_screen(ix, n) would make
 * (deleted rows included, as the builds include them), so every search and graph build reads them as it would after
 * that build.  Only the appended rows' postings are sorted; the old postings keep their order and are copied once to
 * their place in the new arrays.  n == the covered rows does nothing and returns EPS_OK.  The call synchronises the
 * index's stream and does not touch the count of re-scored pairs.
 * Refusals, all EPS_ERR_INVALID_ARGUMENT and all leaving the lists as they were: a null or dense index, an index
 * without posting lists (build them first), n below the covered rows (a build with a smaller n shrinks them), n above
 * the mirrored rows, a view, or an index with live views.  A failed allocation or launch also leaves the previous lists
 * in place: the new ones are installed only once every step has succeeded.
 * Device memory while it runs, with P_old / T_old the postings / distinct indices of the lists, P_new / T_new those of
 * the appended rows and T the distinct indices after: the new lists, 8 B x (P_old + P_new) + 12 B x T + 8 B, beside the
 * old ones, which are freed when the new ones are installed; the appended rows' sort, 24 B x P_new plus the sort's
 * scratch, of which 8 B x P_new stay until the merge; and 28 B x T_new + 8 B x T_old of term bookkeeping plus a scan's
 * scratch.  A rebuild instead needs 24 B x (P_old + P_new) plus the sort's scratch beside the old lists. */
EPS_API int eps_index_extend_sparse_postings(eps_index* ix, int64_t n);
/* Copy the posting lists out, as eps_index_get_graph copies the graph: n_rows = the rows covered, then n_terms
 * distinct indices (terms, ascending), their n_terms + 1 offsets (ptr, from 0 to n_postings), and the postings split
 * into their rows and values (term terms[t] holds rows[ptr[t] .. ptr[t+1]), ascending, with their values).  Pass NULL
 * buffers to query the sizes.  An index without lists gives zeros and writes no buffer.  A null or dense index:
 * EPS_ERR_INVALID_ARGUMENT. */
EPS_API int eps_index_get_sparse_postings(eps_index* ix, int64_t* n_rows, int64_t* n_terms, int64_t* n_postings,
                                          uint32_t* terms, int64_t* ptr, int32_t* rows, float* values);

/* Raw stream handle (cudaStream_t) the index launches on, for callers that time with CUDA events. */
EPS_API void* eps_index_stream(eps_index* ix);

EPS_API const char* eps_last_error(void);
EPS_API const char* eps_version(void);
EPS_API int eps_device_count(void);

#ifdef __cplusplus
}
#endif
#endif /* EPSILLA_B200_H_ */
