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
 * caller lowers `x IN (a, b, ..)` to `x = a OR x = b ..` (integration/epsilla_b200_dropin.cpp does).  LIKE, string
 * concatenation and NEARBY nodes are rejected with EPS_ERR_UNSUPPORTED (regex / geo work, out of scope). */
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
  uint64_t kernel_launches;
  uint64_t n_redone;   /* exact scan: queries the coarse-pass guard sent back (fp32 scan or a larger candidate list) */
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
 * :176-190: StrEvaluate / string EQ, NE / IN).  column = the field's index in var_len_attr_table_ (< 8). */
EPS_API int eps_index_set_string_codes(eps_index* ix, int column, int64_t first_row, const int32_t* codes, int64_t count);

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

/* Launch geometry of the graph-search kernel (performance knob, never changes results): ring_slots = shared-memory row slots per CTA that TMA
 * bulk copies land in (0 = auto: ~48 KB of rows), ctas_per_sm = cap on resident CTAs, i.e. in-flight queries, per SM
 * (0 = whatever fits).  No reference counterpart (the CPU executor has no such geometry). */
EPS_API int eps_index_set_graph_tuning(eps_index* ix, int ring_slots, int ctas_per_sm);

/* Precision of the COARSE pass of large-batch exact scans (nq >= 64): 0 = none (fp32 SIMT tiles only),
 * 1 = wgmma TF32 on the fp32 rows (default), 2 = wgmma BF16 on a bf16 mirror of the table
 * (+50 % HBM).  Whatever the mode, the k' = k + max(118, k) best coarse candidates of every query are re-evaluated
 * with the exact fp32 direct form, so returned distances are fp32-exact, and a GUARD checks that no row outside
 * the candidate list can belong to the answer: with T = the k'-th best coarse distance, e_k = the exact k-th best
 * and E = the largest |coarse - exact| over the batch's own k' x nq re-scored rows, a query is safe when
 * e_k + 2 E <= T; unsafe queries are redone on the fp32 path (or, when many are unsafe, the batch is redone with a
 * 4x larger k' that the index remembers).  eps_stats.n_redone counts them.  The guard is on by default. */
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
 * asynchronous on the index's stream unless sync != 0.  For pipelines that keep queries in HBM and
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

/* Raw stream handle (cudaStream_t) the index launches on, for callers that time with CUDA events. */
EPS_API void* eps_index_stream(eps_index* ix);

EPS_API const char* eps_last_error(void);
EPS_API const char* eps_version(void);
EPS_API int eps_device_count(void);

#ifdef __cplusplus
}
#endif
#endif /* EPSILLA_B200_H_ */
