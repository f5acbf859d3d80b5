// Internal host-side declarations shared by the translation units of libepsilla_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "common.cuh"
#include "filter.cuh"

namespace eps {

// Device memory (pinned host memory when `host`) with its capacity in bytes.  This is the only code that allocates or
// frees; an alias refers to memory the object does not own and never frees it.
struct Mem {
  void* p = nullptr;
  size_t cap = 0;
  bool owns = false;
  bool host = false;
  uint64_t gen = 0;  // bumped whenever p takes new memory: contents filled under an older generation are gone
  Mem() = default;
  Mem(const Mem&) = delete;
  Mem& operator=(const Mem&) = delete;
  ~Mem() { release(); }  // error paths (EPS_TRY / EPS_CUDA early returns) must not leak device memory
  // Room for `bytes`; when that needs an allocation, the old memory is freed first and exactly `bytes` are allocated.
  int reserve(size_t bytes);
  // Room for `bytes`, keeping the first `keep` (a device-to-device copy on s); the old memory is freed last, so a
  // failure leaves the buffer as it was.
  int grow(size_t bytes, size_t keep, cudaStream_t s);
  // Exchange the memory of two buffers of the same kind (both device or both host).
  void swap(Mem& o);
  void release();
  void alias(void* q, size_t bytes);
  template <typename T>
  T* as() const { return static_cast<T*>(p); }
};

// Scratch buffer that grows on demand (never shrinks, at least 256 bytes); owned by an index / a call context.
struct DevBuf : Mem {
  int reserve(size_t bytes) { return Mem::reserve(bytes < 256 ? 256 : bytes); }
};

// Pinned host buffer.
struct HostBuf : Mem {
  HostBuf() { host = true; }
};

// Device array of T.  A copy is a non-owning alias of the same memory: a view assigned its base's Table frees nothing.
template <typename T>
struct DevArray : Mem {
  DevArray() = default;
  DevArray(const DevArray& o) : Mem() { alias(o.p, o.cap); }
  DevArray& operator=(const DevArray& o) {
    if (this != &o) alias(o.p, o.cap);
    return *this;
  }
  operator T*() const { return static_cast<T*>(p); }
  int64_t count() const { return static_cast<int64_t>(cap / sizeof(T)); }  // elements there is room for
};

// Device mirror of one string column as dictionary codes (filter.cuh).
struct StrCol {
  DevArray<int32_t> d_codes;
  int64_t rows = 0;
  bool any_negative = false;  // some mirrored code is < 0 (a LIKE cannot read the column then)
  int32_t max_code = -1;      // largest mirrored code
};

// Device mirror of the caller's string dictionary (like.cu): code c is bytes[off[c] .. off[c+1]).  Append-only,
// grown like StrCol; a view shares its base's.
struct StrDict {
  DevArray<int64_t> d_off;  // [n + 1], d_off[0] = 0
  DevArray<char> d_bytes;
  int64_t n = 0;            // codes mirrored
  int64_t bytes = 0;
};

// Device data a base owns and its views alias; only the base frees it.
struct Table {
  int64_t capacity = 0;
  DevArray<float> d_vectors;    // [capacity x dim] (an alias of the caller's rows once adopted)
  int64_t n_rows = 0;           // rows mirrored so far (record_number_ snapshot)
  bool vec4 = false;            // dim % 4 == 0 and 16-B aligned base

  // sparse column (eps_index_create_sparse): rows are a CSR of {uint32 index, float value} elements
  DevArray<int64_t> d_sp_ptr;   // [rows + 1] element offsets of the rows
  DevArray<uint2> d_sp_elems;   // {index, value bits}, indices strictly increasing within a row
  DevArray<float> d_sp_norm2;   // [rows] sequential fp32 sum of squares of each row (cosine); its room is the row room
  int64_t sp_nnz = 0;
  // posting lists of the sparse rows [0, inv_rows) (sparse_inverted.cu): the exact scan reads their distances from them
  // (IP / cosine: the inverted index), or screens them with a lower bound of their distance (L2: the L2 screen)
  DevArray<uint32_t> d_inv_terms;  // [inv_terms] the distinct indices, ascending
  DevArray<int64_t> d_inv_ptr;     // [inv_terms + 1] posting offsets of the terms
  DevArray<uint2> d_inv_post;      // [inv_postings] {int32 row, float value bits}, rows ascending within a term
  int64_t inv_rows = 0;            // rows covered (0: no index)
  int64_t inv_terms = 0;
  int64_t inv_postings = 0;

  // graph (ANNGraphSegment mirror)
  int64_t n_indexed = 0;
  int64_t n_edges = 0;
  int64_t nav = 0;
  DevArray<int64_t> d_offsets;  // [n_indexed + 1]
  DevArray<int32_t> d_nbrs;     // [n_edges]
  DevArray<int32_t> d_ell;      // fixed-stride adjacency [n_indexed x 64] (-1 padded), built lazily

  // segment mirrors
  DevArray<uint8_t> d_deleted;
  int64_t deleted_bytes = 0;
  bool any_deleted = false;
  DevArray<char> d_attrs;
  int64_t attr_stride = 0;
  int64_t attr_rows = 0;
  StrCol str_cols[kMaxStringCols];
  StrDict dict;

  // principal-subspace sketch of the indexed rows (sketch.cu), computed when a graph is installed; a view shares its
  // base's.  Dropped with the graph or the rows under it.
  int sk_m = 0;                  // floats per row sketch: kSketch, or 0 while there is no basis
  double sk_share = -1.0;        // share of the sampled variance the basis carries; -1 = no basis
  float sk_g = 0.f;              // 1 - gamma_{m+2}, rounded down
  float sk_scale = 0.f;          // (1 - 2 (dim + 2) 2^-24) / (1 + eps), rounded down
  double sk_eps = 0.0;           // sigma_max(P~)^2 <= 1 + sk_eps
  double sk_mu_norm = 0.0;       // |mu|, rounded up
  DevArray<float> d_sk_basis;    // [dim x sk_m] fp32 basis P~ (transposed), then [dim] mean
  // [n_indexed x sk_m] row sketches, then [n_indexed] their error bounds; inner product and cosine then add, from
  // float sk_terms_off(n_indexed) on, [n_indexed] float2 {|A y|, <mu, y>} rounded up (null: screen off)
  DevArray<float> d_sk;
};

// Executor and tuning parameters: a view starts with its base's and sets its own afterwards.
struct Config {
  int64_t L_master = 500, L_local = 500;
  bool prefilter = false;
  bool force_brute = false;
  int sparse_search = EPS_SPARSE_SEARCH_SCAN;  // sparse index: exact scan always, or the reference's graph branch
  int search_width = 1;          // candidates expanded per iteration (1 = the reference's sequential order)
  int graph_ring_slots = 0;      // row-ring slots per CTA of the graph kernel (0 = auto)
  int graph_ctas_per_sm = 0;     // cap on resident CTAs (= in-flight queries) per SM (0 = occupancy limit)
  int coarse_mode = 1;           // exact-scan coarse pass: 0 = fp32 SIMT only, 1 = wgmma TF32, 2 = wgmma bf16 mirror
  int coarse_guard = 1;          // verify the coarse pass after the re-score and redo unsafe queries (brute_force.cu)
  int coarse_boost = 1;          // multiplier of k' learnt by the guard for this table (1, 4, 16, 64)
  int graph_screen = EPS_GRAPH_SCREEN_AUTO;
  int filter_search = EPS_FILTER_SEARCH_POST;  // graph branch of a filtered dense search: post-filter or collect
};

// Deleted with its device current (eps_index_destroy): it frees what it owns, never its base's Table.
struct Index : Table, Config {
  int device = 0;
  int metric = EPS_METRIC_L2;
  int64_t dim = 0;
  bool sparse = false;
  int num_sms = 132;
  int smem_per_sm = 228 * 1024;   // shared memory an SM can give its CTAs (the largest carve-out)
  int smem_reserved_per_cta = 1024;  // shared memory the driver reserves per resident CTA
  int gs_static_smem = -1;        // static shared memory of the screened graph kernel (-1: not read yet)
  const float* host_vectors = nullptr;
  Index* view_of = nullptr;     // read-only view (eps_index_create_view): its Table belongs to this index
  int n_views = 0;              // live views of this index; mutating entry points refuse while > 0
  std::vector<Index*> views;    // the live views (detached when the base is destroyed first)
  bool detached_view = false;   // a view whose base has been destroyed: holds no data any more
  std::vector<uint8_t> h_deleted;  // host shadow of the uploaded deleted bitset (dirty-span detection)
  const char* attr_src = nullptr;  // host table the attribute mirror was filled from (append detection)

  DevArray<int32_t> d_init_ids;  // seed set for init_L
  int64_t init_L = 0;
  int64_t seed_rows_L = 0;       // L for which s_seed_rows holds the gathered seed rows

  cudaStream_t stream = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  ~Index() {
    for (auto& e : ev) if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
  }

  // scratch
  DevBuf s_queries, s_dist, s_topk, s_topk2, s_pass, s_filter, s_vset, s_visited, s_vlog, s_queue, s_tail, s_out_ids, s_out_dists,
      s_out_counts, s_stats, s_misc, s_seed_rows, s_seed_dist, s_xnorm, s_qnorm, s_coarse, s_thr, s_cand, s_cand_cnt, s_bf16, s_qbf16, s_flags,
      s_sparse_q, s_xnorm_max, s_like, s_like_jobs, s_inv_plan, s_l2_screen;
  // collect mode: the pass bitmap of [0, n_rows), its per-CTA counts and P, the passing ids, the lists of the passing
  // rows, the merged keys per query, the short queries, and the gathered rows of the scan over passing rows
  DevBuf s_cpass, s_ccount, s_cids, s_clist, s_ckeys, s_cshort, s_gather;
  int64_t bf16_rows = 0;         // rows converted into s_bf16 while it had generation bf16_gen
  uint64_t bf16_gen = 0;
  int64_t xnorm_rows = 0;        // rows whose |x|^2 is current in s_xnorm; s_xnorm_max holds the largest (float bits)
  uint64_t xnorm_gen = 0;
  int64_t visited_slots = 0;
  uint64_t visited_gen = 0;      // s_visited generation and bitmap words for which the bitmaps are known to be zero
  int64_t visited_words = 0;
  uint64_t vset_gen = 0;         // s_vset generation known to be all-ones (empty)
  bool graph_counters_pending = false;
  int64_t prof_nq = 0;           // developer build (EPS_GS_PROFILE): queries of the last graph-search launch
  DevBuf s_prof_qtimes;          // developer build: [prof_nq x 4] per-query timeline of the last dense launch
  bool prof_timeline = false;    // developer build: s_prof_qtimes belongs to the last launch
  DevBuf s_qsk;                  // [nq x sk_m] query sketches, then [nq] their error bounds (+ dot-product terms, sketch_queries)
  DevArray<unsigned long long> d_screened;  // device count of the fresh neighbours the screen dropped on this handle
  DevArray<unsigned long long> d_l2_rescored;  // device count of the (query, row) pairs the L2 screen re-scored here
  HostBuf h_out;                 // pinned host mirror of the packed result block (eps_search_batch)
};

// ---- brute_force.cu ------------------------------------------------------------------------
struct SparseL2Screen;
// Producer of the [nq x ldd] fp32 distance tile of rows [row_start, row_start + n) that the exact scan selects from,
// in place of launch_distances (the sparse scan, sparse.cu).
struct DistProducer {
  virtual ~DistProducer() = default;
  virtual int launch(Index* ix, int metric, int64_t row_start, int64_t n, float* D, int64_t ldd, uint64_t* launches) const = 0;
};

// One exact scan: everything it depends on besides the table itself.
struct ScanRequest {
  const float* queries = nullptr;      // dense queries [nq x dim] on the device, or
  const DistProducer* dist = nullptr;  // a producer of the fp32 distance tile (never the tensor-core pass)
  int64_t nq = 0, row_start = 0, row_end = 0, k = 0;
  int metric = EPS_METRIC_L2;          // the field's; L2 for the build's navigation point (nsg.cpp)
  const FilterProg* d_prog = nullptr;  // filter (device copy and host copy), or null
  const FilterProg* h_prog = nullptr;
  bool prefilter = false;              // evaluate the filter with distance 0
  bool skip_deleted = true;            // false: the build indexes every row, deleted or not (ann_graph_segment.cpp:201)
  int64_t self_base = -1;              // >= 0: row self_base + q is left out of query q's list (the build's kNN lists)
  // sparse L2 index with posting lists: fp32_scan bounds, thresholds and re-scores the covered rows before the select
  // (dist is then the plain SparseDist: a filter that reads the distance takes it for every row)
  const SparseL2Screen* l2_screen = nullptr;
};
// Exact top-k of rows [row_start, row_end): per-query sorted keys (make_key(dist,row)) in d_topk [nq x k], kKeyInf
// padded.
int exact_topk(Index* ix, const ScanRequest& r, unsigned long long* d_topk, eps_stats* stats);

// Distances of rows [row_start,row_start+n) of A_base to nq device queries: D[q*ldd + i] (row kernel for
// nq <= 16, 128x128 tile kernel otherwise).
// form_nq > 0 picks the kernel as for a batch of form_nq queries: the two kernels add a row's terms in different orders,
// so a subset of a batch takes the batch's kernel to get the batch's bits.
int launch_distances(Index* ix, int metric, const float* A_base, int64_t row_start, int64_t n, const float* d_queries,
                     int64_t nq, float* D, int64_t ldd, uint64_t* launches, int64_t form_nq = 0);

// Collect mode of a filtered graph search (capi.cu).  collect_pass: the pass bitmap of rows [0, r.row_end) into
// ix->s_cpass (not deleted, and passing r.d_prog at distance 0) and its popcount P; synchronises the stream to read P.
int collect_pass(Index* ix, const ScanRequest& r, int64_t* P, uint64_t* launches);
// passing_topk: the exact top-k over the P rows of that bitmap for the nb queries d_idx picks of the nq queries
// (d_idx null: all of them, nb = nq), written over their rows of d_topk [nq x k].  Rows are compacted into an ascending
// id list and scanned in chunks with the fp32 kernel of a batch of nq queries, so the keys are bitwise those of the
// exact scan of rows [0, n_rows) with the same filter, in prefilter mode with the coarse pass off.  Synchronises the
// stream when d_idx is set.
int passing_topk(Index* ix, const float* queries, int64_t nq, const int* d_idx, int64_t nb, int64_t k, int64_t P,
                 unsigned long long* d_topk, eps_stats* stats);

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
int tc_launch_distances(Index* ix, int metric, int64_t row_start, int64_t n, const float* d_queries, int64_t nq, float* D,
                        int64_t ldd, uint64_t* launches, const TcFused* fused = nullptr);

// ---- sparse.cu -----------------------------------------------------------------------------
// Queries of the sparse scan as a device CSR: ptr[q] .. ptr[q+1] index elems (absolute offsets), norm2[q] = the
// sequential fp32 sum of squares.
struct SparseQueries {
  const int64_t* ptr;
  const uint2* elems;
  const float* norm2;
};
struct SparseDist : DistProducer {
  SparseQueries q;
  int64_t nq;
  SparseDist(const SparseQueries& q_, int64_t nq_) : q(q_), nq(nq_) {}
  int launch(Index* ix, int metric, int64_t row_start, int64_t n, float* D, int64_t ldd, uint64_t* launches) const override;
};
// Validate and pack n rows of a caller CSR (offsets[0..n], indices, values) into ptr (n+1 entries, starting at
// ptr_base), elems and norm2.  Indices must be >= 0, < max_index and strictly increasing within a row.
int pack_sparse(int64_t n, const int64_t* offsets, const int64_t* indices, const float* values, int64_t max_index,
                int64_t ptr_base, std::vector<int64_t>* ptr, std::vector<uint2>* elems, std::vector<float>* norm2);
// Reserve buf for a query set packed by pack_sparse (ptr_base 0) and enqueue its upload on ix->stream as one block
// [ptr | norm2 | elems]; *q points into buf.
int upload_sparse_queries(Index* ix, const std::vector<int64_t>& ptr, const std::vector<uint2>& elems,
                          const std::vector<float>& norm2, DevBuf* buf, SparseQueries* q);
int sparse_append(Index* ix, int64_t first_row, int64_t n_rows, const int64_t* offsets, const int64_t* indices,
                  const float* values);
int build_graph_sparse(Index* ix, int64_t n, const eps_build_params* params);

// ---- sparse_inverted.cu --------------------------------------------------------------------
// Posting lists of rows [0, n) of a sparse index (n = 0 drops them); the caller has validated ix and n.
int build_sparse_inverted(Index* ix, int64_t n);
// The posting lists extended over rows [inv_rows, n), to the arrays build_sparse_inverted(ix, n) makes; the caller has
// validated ix and inv_rows < n <= n_rows.
int extend_sparse_inverted(Index* ix, int64_t n);
// The sparse scan's distance tile with the rows [0, inv_rows) read from the posting lists, bitwise the tile of
// SparseDist: each row's products are added in the query's index order, from 0, as sparse_dist_kernel adds them.
// Rows at or above inv_rows go to SparseDist.  The queries' elements are [elem_base, elem_base + n_elems) of q.elems
// (elem_base = q.ptr[0], n_elems = q.ptr[nq] - elem_base): 0 for an uploaded query set, the chunk's first element when
// the build's queries are rows of the mirror itself.  The plan holds those elements only.
struct InvertedDist : DistProducer {
  SparseDist scan;
  int64_t n_elems, elem_base;
  mutable bool planned = false;  // the query elements' posting ranges are in ix->s_inv_plan (one plan per call)
  InvertedDist(const SparseDist& s, int64_t n_elems_, int64_t elem_base_ = 0)
      : scan(s), n_elems(n_elems_), elem_base(elem_base_) {}
  int launch(Index* ix, int metric, int64_t row_start, int64_t n, float* D, int64_t ldd, uint64_t* launches) const override;
  int plan(Index* ix, uint64_t* launches) const;  // once per call, before the first score launch
};
// The L2 screen (eps_index_build_sparse_l2_screen): the posting lists of an L2 index give each covered row a proven
// lower bound LB <= D_ref of the reference's distance; fp32_scan (brute_force.cu) runs, per chunk of rows,
//   1. bounds():    the tile with LB for the covered rows (+inf for rows the bound does not cover) and the exact
//                   distances of the others (SparseDist);
//   2. the select of each query's K smallest tile keys (K = the scan's k), then threshold(): T[q] = the largest exact
//                   distance of those K rows (+inf when fewer than K finite keys came back or one is NaN);
//   3. rescore():   the exact distance of every covered row with LB <= T[q] or not covered by the bound, +inf for the
//                   others (the K rows of step 2 have D_ref <= T, so a row with LB > T is not among the K best);
//   4. the unchanged select over the tile.
struct SparseL2Screen {
  InvertedDist inv;
  explicit SparseL2Screen(const InvertedDist& i) : inv(i) {}
  int bounds(Index* ix, int64_t row_start, int64_t n, float* D, int64_t ldd, uint64_t* launches) const;
  // keys: [nq x k] sorted keys of the tile of step 1; T: [nq]
  int threshold(Index* ix, const unsigned long long* keys, int k, float* T, uint64_t* launches) const;
  // the covered rows of [row_start, row_start + n); pass (relative to pass_base, may be null) and self_base as in the
  // select: rows it drops are not re-scored
  int rescore(Index* ix, int64_t row_start, int64_t n, float* D, int64_t ldd, const float* T, const uint32_t* pass,
              int64_t pass_base, int64_t self_base, uint64_t* launches) const;
};

// ---- sparse_graph.cu -----------------------------------------------------------------------
// graph_search for sparse queries at width 1 (the reference's sequential order): d_queue [nq x L] sorted keys.
int sparse_graph_search(Index* ix, const SparseQueries& q, int64_t nq, int64_t L, unsigned long long* d_queue,
                        eps_stats* stats);

// ---- graph_search.cu -----------------------------------------------------------------------
// Best-first search of nq queries over the installed CSR graph with queue length L (<= n_indexed).
// Output: d_queue [nq x L] sorted keys.
// collect (a filtered search in EPS_FILTER_SEARCH_COLLECT): the same navigation, and per query the best `cap` keys of
// the rows it evaluates whose bit is set in `pass` (rows [0, n_indexed) at least), into out [nq x cap], ascending,
// kKeyInf padded.
struct GraphCollect {
  const uint32_t* pass;
  unsigned long long* out;
  int64_t cap;
};
int graph_search(Index* ix, const float* d_queries, int64_t nq, int64_t L, unsigned long long* d_queue,
                 eps_stats* stats, const GraphCollect* collect = nullptr);
int prepare_init_ids(Index* ix, int64_t L);
// Launch prologue shared by graph_search and sparse_graph_search: L in [1, n_indexed] (`who` names the caller in the
// error), the padded queue length Lp (a power of two >= 2, at most 16384) and the init ids.
int graph_launch_prologue(Index* ix, int64_t L, const char* who, int* Lp);
// Reserves and zeroes the counter block of a launch of nq queries (graph_search.cuh, GraphCounter).
int graph_counters(Index* ix, int64_t nq);
constexpr int kEll = 64;  // adjacency ids per fixed-stride (ELL) row
int ensure_ell(Index* ix, uint64_t* launches);  // fixed-stride adjacency of the installed graph (built once)
// out[i] = row d_ids[i] of the table (contiguous copy; used for seed rows and for the build's repair searches)
int gather_rows(Index* ix, const int32_t* d_ids, int64_t n, float* d_out);
int read_graph_counters(Index* ix, eps_stats* stats);
// Visited sets of `slots` concurrent graph queries at queue length L, shared by the dense and sparse kernels: per slot
// an open-addressing hash set (all-ones = empty, refilled by the kernel), a bitmap of n_indexed bits for queries that
// outgrow it (left zero by the kernel) and a log of the query's fresh ids.
struct VisitedSets {
  uint32_t* vset;
  int vset_cap, vset_shift, vset_max;  // entries per slot, bucket shift, inserts before a query moves to the bitmap
  uint32_t* visited;
  int64_t words;                        // bitmap words per slot
  int32_t* vlog;
  int vlog_cap;
};
int prepare_visited(Index* ix, int slots, int64_t L, VisitedSets* v);

// ---- sketch.cu -----------------------------------------------------------------------------
constexpr int kSketch = 32;       // floats per row sketch of the graph screen
// Top-m principal subspace of the first n_indexed rows: basis [m x dim] row-major with orthonormal rows (the first k
// rows span the top-k subspace), the sample mean [dim], and the share of the sample's variance the m rows carry.
int principal_subspace(Index* ix, int m, std::vector<float>* basis, std::vector<float>* mean, double* share);
// The graph search screens fresh neighbours with the sketch when the mode is on, or auto with the basis carrying at
// least kScreenShare of the variance.  L2 bounds the distance; inner product and cosine bound the dot product.
constexpr double kScreenShare = 0.9;
constexpr int kScreenNone = 0, kScreenL2 = 1, kScreenDot = 2;  // the graph kernel's screen kinds
// Basis (+ row sketches when the screen will run) of the installed graph's rows, at graph install and mode changes.
// Never fails: a sketch that cannot be set up leaves the screen off.  Row sketches are freed when the screen is off.
void ensure_sketch(Index* ix);
void free_sketch(Index* ix);
bool screen_on(const Index* ix);
int screen_kind(const Index* ix);  // the kind the next graph search runs (kScreenNone when the screen is off)
// float offset of the dot-product row terms in d_sk (8-byte aligned), and the floats d_sk takes, for n rows
__host__ __device__ inline int64_t sk_terms_off(int64_t n) { return (n * (kSketch + 1) + 1) & ~static_cast<int64_t>(1); }
int64_t sketch_floats(const Index* ix, int64_t n);
// sketches and error bounds of n rows at d_x (the table's layout) with the index's basis
int sketch_rows(Index* ix, const float* d_x, int64_t n, float* d_sk, float* d_ex);
// dot-product screen: {|A y|, <mu, y>} of n rows at d_x, rounded up
int dot_row_terms(Index* ix, const float* d_x, int64_t n, float2* d_terms);
// the per-query block of a graph search's screen in qsk: [nq x kSketch] sketches of q - mu, [nq] their error bounds,
// and for the dot-product kind, from float sk_qterms_off(nq) on (16-byte aligned for any nq), [nq x 4]
// {C0, C_ex, |A (q - mu)|, K} (sketch.cu); returns the launches it took
int sketch_queries(Index* ix, const float* d_q, int64_t nq, float* qsk, uint64_t* launches);
__host__ __device__ inline int64_t sk_qterms_off(int64_t nq) { return (nq * (kSketch + 1) + 3) & ~static_cast<int64_t>(3); }
inline int64_t sketch_query_floats(int kind, int64_t nq) { return kind == kScreenDot ? sk_qterms_off(nq) + 4 * nq : nq * (kSketch + 1); }

// ---- finalize.cu ---------------------------------------------------------------------------
// Post-filter walk / tail merge of VecSearchExecutor::Search (vec_search_executor.cpp:885-927).
int finalize_graph(Index* ix, unsigned long long* d_queue, int64_t nq, int64_t L, int64_t search_limit,
                   int64_t cand_num, const unsigned long long* d_tail, int64_t tail_k, int64_t limit,
                   const FilterProg* d_prog, const FilterProg* h_prog, int64_t* d_ids, float* d_dists,
                   int64_t* d_counts);
// Brute-force results: first min(valid, limit_cap) keys -> ids/dists/counts.
int finalize_keys(Index* ix, const unsigned long long* d_topk, int64_t nq, int64_t k, int64_t limit, int64_t cap,
                  int64_t* d_ids, float* d_dists, int64_t* d_counts);
// Collect mode: per query, the first cap keys of the merge of the graph search's passing-row list [nq x cap] and the
// tail scan's top keys [nq x tail_k] (disjoint rows; tail may be null) into out [nq x cap]; the queries left with fewer
// than min(cap, P) keys are listed on the device at *d_short_idx (in ix->s_cshort), and their number goes to *n_short
// (synchronises the stream).
int collect_merge(Index* ix, const unsigned long long* d_list, const unsigned long long* d_tail, int64_t nq, int64_t cap,
                  int64_t tail_k, int64_t P, unsigned long long* d_out, const int** d_short_idx, int64_t* n_short);
// shard s reads ids + s*id_stride and dists + s*dist_stride (elements; <= 0: the dense [n_shards x nq x k] layout)
int merge_shards(int device, cudaStream_t stream, const int64_t* d_ids, const float* d_dists, int64_t n_shards,
                 int64_t nq, int64_t k, int64_t* d_out_ids, float* d_out_dists, int64_t id_stride = 0,
                 int64_t dist_stride = 0);

// ---- build.cu ------------------------------------------------------------------------------
// The caller's build parameters with every unset (<= 0) field at its default.
eps_build_params build_defaults(const eps_build_params* params);
int build_graph(Index* ix, int64_t n, const eps_build_params* params);
// Install a host CSR (int64 offsets, int32 ids) as the index's graph, dropping everything derived from the old one.
int install_csr(Index* ix, int64_t n, const int64_t* off, const int32_t* nb, int64_t e, int64_t nav);
// Replace the installed CSR with a host CSR and drop the adjacency table and seed set; the sketch (basis and row
// sketches) is kept: the caller keeps the row sketches covering [0, n).
int upload_csr(Index* ix, int64_t n, const int64_t* off, const int32_t* nb, int64_t e, int64_t nav);
// graph_search with the metric and width given and the screen off, the handle's settings restored on every path
// (the build's pools: they must not depend on, or count in, the screen of the searches the caller runs).
int graph_search_as(Index* ix, int metric, int width, const float* d_queries, int64_t nq, int64_t L,
                    unsigned long long* d_queue, eps_stats* st);

// Connectivity repair of a build (CheckConnectivity, nsg.cpp:687-775) on host lists: the integer-only steps.
// lists: [n x stride] out-neighbours, cnt[v] of them valid; knn: [n x K] sorted keys (kKeyInf padded).
struct ConnRepair {
  int64_t n;
  const int32_t* lists;
  const int32_t* cnt;
  int stride;
  const int64_t* off = nullptr;  // set: lists is a CSR neighbour array and row u starts at off[u]
  const int32_t* row_of(int64_t u) const { return lists + (off ? off[u] : u * stride); }
  std::vector<uint8_t> seen;
  std::vector<int32_t> stack;
  int64_t linked = 0;
  std::vector<std::vector<int32_t>> extra;  // edges added by the repair
  std::vector<int32_t> entries;             // one per component that the kNN lists do not connect to the rest
  ConnRepair(int64_t n_, const int32_t* lists_, const int32_t* cnt_, int stride_);
  void flood(int32_t root);
  // steps 1 and 2: attach every unlinked vertex to its nearest linked kNN entry with room, or make it an entry
  void attach_from_knn(const unsigned long long* knn, int K);
  // step 4: attach u to a random linked vertex (rng: the build's LCG state)
  void attach_random(int32_t u, uint64_t* rng);
  // entries become out-neighbours of nav; flatten lists + extra edges to the reference CSR
  void flatten(int64_t nav, std::vector<int64_t>* off, std::vector<int32_t>* nb);
};
// Steps 3 and 4 of the repair over the installed graph (rng: the LCG state of step 4).
int repair_by_search(Index* ix, ConnRepair* rep, int64_t Ls, uint64_t* rng, eps_stats* st);

// ---- extend.cu -----------------------------------------------------------------------------
// Link rows [n_indexed, n) into the installed dense graph (eps_index_extend_graph); the caller has validated n.
int extend_graph(Index* ix, int64_t n, const eps_build_params* params);

// ---- like.cu -------------------------------------------------------------------------------
// Append codes [first_code, first_code + count) to the dictionary mirror (eps_index_append_string_dictionary).
int dict_append(Index* ix, int64_t first_code, int64_t count, const int64_t* offsets, const char* bytes);
// Validation of the LIKE nodes of a lowered program (constant codes and the columns they read); bind_program_columns
// calls it, so every failure comes before any launch.
int check_like(const Index* ix, const FilterProg& prog);
// One match-kernel launch on ix->stream for every LIKE node of progs[0 .. n): the bits go to ix->s_like, each
// program's like_bits points at its share and each LIKE node's pad at its words.  No launch without LIKE nodes;
// *launches (if given) counts the launch.
int bind_like(Index* ix, FilterProg* progs, int n, uint64_t* launches);

// ---- capi.cu -------------------------------------------------------------------------------
int normalize_rows_device(cudaStream_t s, float* d, int64_t n, int64_t dim);
int check_device(int device);
int bind_program_columns(Index* ix, FilterProg* prog);
void free_graph(Index* ix);  // the graph, its seed set and everything derived from them

}  // namespace eps
