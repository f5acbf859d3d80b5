// Internal host-side declarations shared by the translation units of libepsilla_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "common.cuh"
#include "filter.cuh"

namespace eps {

// Device buffer that grows on demand (never shrinks); owned by an index / a call context.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }  // error paths (EPS_TRY / EPS_CUDA early returns) must not leak device memory
  int reserve(size_t bytes);
  void release();
  template <typename T>
  T* as() { return static_cast<T*>(p); }
};

// Device mirror of one string column as dictionary codes (filter.cuh).
struct StrCol {
  int32_t* d_codes = nullptr;
  int64_t rows = 0, cap = 0;
};

struct Index {
  int device = 0;
  int metric = EPS_METRIC_L2;
  int64_t dim = 0;
  int64_t capacity = 0;
  const float* host_vectors = nullptr;
  float* d_vectors = nullptr;   // [capacity x dim] (owned unless adopted)
  bool owns_vectors = false;
  Index* view_of = nullptr;     // read-only view (eps_index_create_view): table, graph, segment mirrors belong to this index
  int n_views = 0;              // live views of this index; mutating entry points refuse while > 0
  std::vector<Index*> views;    // the live views (detached when the base is destroyed first)
  bool detached_view = false;   // a view whose base has been destroyed: holds no data any more
  int64_t n_rows = 0;           // rows mirrored so far (record_number_ snapshot)
  bool vec4 = false;            // dim % 4 == 0 and 16-B aligned base

  // graph (ANNGraphSegment mirror)
  int64_t n_indexed = 0;
  int64_t n_edges = 0;
  int64_t nav = 0;
  int64_t* d_offsets = nullptr;  // [n_indexed + 1]
  int32_t* d_nbrs = nullptr;     // [n_edges]
  int32_t* d_init_ids = nullptr; // seed set for init_L
  int64_t init_L = 0;
  int32_t* d_ell = nullptr;      // fixed-stride adjacency [n_indexed x 64] (-1 padded), built lazily
  int64_t seed_rows_L = 0;       // L for which s_seed_rows holds the gathered seed rows

  // segment mirrors
  uint8_t* d_deleted = nullptr;
  int64_t deleted_bytes = 0;
  int64_t deleted_cap = 0;
  std::vector<uint8_t> h_deleted;  // host shadow of the uploaded bitset (dirty-span detection)
  bool any_deleted = false;
  char* d_attrs = nullptr;
  int64_t attr_stride = 0;
  int64_t attr_rows = 0;
  int64_t attr_cap_rows = 0;
  const char* attr_src = nullptr;  // host table the mirror was filled from (append detection)
  StrCol str_cols[kMaxStringCols];

  // executor parameters
  int64_t L_master = 500, L_local = 500;
  bool prefilter = false;
  bool force_brute = false;
  int search_width = 1;          // candidates expanded per iteration (1 = the reference's sequential order)
  int graph_ring_slots = 0;      // row-ring slots per CTA of the graph kernel (0 = auto)
  int graph_ctas_per_sm = 0;     // cap on resident CTAs (= in-flight queries) per SM (0 = occupancy limit)

  cudaStream_t stream = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  int num_sms = 132;

  // scratch
  DevBuf s_queries, s_dist, s_topk, s_topk2, s_pass, s_filter, s_visited, s_vlog, s_queue, s_tail, s_out_ids, s_out_dists,
      s_out_counts, s_stats, s_misc, s_seed_rows, s_seed_dist, s_xnorm, s_qnorm, s_coarse, s_thr, s_cand, s_cand_cnt, s_bf16, s_qbf16, s_flags;
  int coarse_mode = 1;           // exact-scan coarse pass: 0 = fp32 SIMT only, 1 = wgmma TF32, 2 = wgmma bf16 mirror
  int coarse_guard = 1;          // verify the coarse pass after the re-score and redo unsafe queries (brute_force.cu)
  int coarse_boost = 1;          // multiplier of k' learnt by the guard for this table (1, 4, 16, 64)
  int64_t bf16_rows = 0;
  const void* bf16_ptr = nullptr;
  int64_t xnorm_rows = 0;        // rows whose |x|^2 is current in s_xnorm
  const void* xnorm_ptr = nullptr;
  int64_t visited_slots = 0;
  const void* vis_clean_ptr = nullptr;  // geometry for which the visited bitmaps are known to be zero
  int64_t vis_clean_words = 0;
  size_t vis_clean_cap = 0;
  bool graph_counters_pending = false;
  int64_t prof_nq = 0;           // developer build (EPS_GS_PROFILE): queries of the last profiled launch
  void* h_out = nullptr;         // pinned host mirror of the packed result block (eps_search_batch)
  size_t h_out_cap = 0;
};

// ---- brute_force.cu ------------------------------------------------------------------------
// Exact top-k of rows [row_start,row_end) for nq device queries.  Writes per-query sorted keys
// (make_key(dist,row)) to d_topk [nq x k] (kKeyInf padded).  Applies deleted bits and, if
// prog != nullptr, the filter (prefilter=true evaluates it with distance 0).
int brute_force_topk(Index* ix, const float* d_queries, int64_t nq, int64_t row_start, int64_t row_end, int64_t k,
                     const FilterProg* d_prog, const FilterProg* h_prog, bool prefilter, unsigned long long* d_topk,
                     eps_stats* stats);

// Distances of rows [row_start,row_start+n) of A_base to nq device queries: D[q*ldd + i] (row kernel for
// nq <= 16, 128x128 tile kernel otherwise).
int launch_distances(Index* ix, const float* A_base, int64_t row_start, int64_t n, const float* d_queries, int64_t nq,
                     float* D, int64_t ldd, uint64_t* launches);

// tc_dist.cu: wgmma TF32 / BF16 coarse distances (same contract as launch_distances, values carry ~1e-3 rel. error)
bool tc_dist_usable(const Index* ix, int64_t nq);
struct TcFused {             // fused threshold selection in the epilogue (no distance tile written)
  const float* thr;          // [nq] running coarse k'-th best
  unsigned long long* cand;  // [nq x cand_cap]
  int* cand_cnt;             // [nq], zeroed by the caller
  const uint32_t* pass;      // may be null
  int64_t pass_base;
  int cand_cap;
};
int tc_launch_distances(Index* ix, int64_t row_start, int64_t n, const float* d_queries, int64_t nq, float* D, int64_t ldd,
                        uint64_t* launches, const TcFused* fused = nullptr);

// All-pairs variant used by the graph build: for queries = rows [q_start, q_start+nq) of the table.
int brute_force_knn_rows(Index* ix, int64_t q_start, int64_t nq, int64_t n_rows, int64_t k,
                         unsigned long long* d_topk, eps_stats* stats);

// ---- graph_search.cu -----------------------------------------------------------------------
// Best-first search of nq queries over the installed CSR graph with queue length L (<= n_indexed).
// Output: d_queue [nq x L] sorted keys.
int graph_search(Index* ix, const float* d_queries, int64_t nq, int64_t L, unsigned long long* d_queue,
                 eps_stats* stats);
int prepare_init_ids(Index* ix, int64_t L);
int ensure_ell(Index* ix, uint64_t* launches);  // fixed-stride adjacency of the installed graph (built once)
// out[i] = row d_ids[i] of the table (contiguous copy; used for seed rows and for the build's repair searches)
int gather_rows(Index* ix, const int32_t* d_ids, int64_t n, float* d_out);
int read_graph_counters(Index* ix, eps_stats* stats);

// ---- finalize.cu ---------------------------------------------------------------------------
// Post-filter walk / tail merge of VecSearchExecutor::Search (vec_search_executor.cpp:885-927).
int finalize_graph(Index* ix, unsigned long long* d_queue, int64_t nq, int64_t L, int64_t search_limit,
                   int64_t cand_num, const unsigned long long* d_tail, int64_t tail_k, int64_t limit,
                   const FilterProg* d_prog, const FilterProg* h_prog, int64_t* d_ids, float* d_dists,
                   int64_t* d_counts);
// Brute-force results: first min(valid, limit_cap) keys -> ids/dists/counts.
int finalize_keys(Index* ix, const unsigned long long* d_topk, int64_t nq, int64_t k, int64_t limit, int64_t cap,
                  int64_t* d_ids, float* d_dists, int64_t* d_counts);
// shard s reads ids + s*id_stride and dists + s*dist_stride (elements; <= 0: the dense [n_shards x nq x k] layout)
int merge_shards(int device, cudaStream_t stream, const int64_t* d_ids, const float* d_dists, int64_t n_shards,
                 int64_t nq, int64_t k, int64_t* d_out_ids, float* d_out_dists, int64_t id_stride = 0,
                 int64_t dist_stride = 0);

// ---- build.cu ------------------------------------------------------------------------------
int build_graph(Index* ix, int64_t n, const eps_build_params* params);

// ---- misc kernels (capi.cu) ----------------------------------------------------------------
int normalize_rows_device(cudaStream_t s, float* d, int64_t n, int64_t dim);

}  // namespace eps
