// C ABI of libepsilla_b200 (include/epsilla_b200.h): index lifetime, segment mirrors, and the batched
// VecSearchExecutor::Search orchestration (engine/db/execution/vec_search_executor.cpp:833-935).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <memory>
#include <mutex>

#include "internal.h"

namespace eps {

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

int Mem::reserve(size_t bytes) {
  if (bytes <= cap && p) return EPS_OK;
  release();
  void* q = nullptr;
  const cudaError_t e = host ? cudaHostAlloc(&q, bytes, cudaHostAllocDefault) : cudaMalloc(&q, bytes);
  if (e != cudaSuccess)
    return fail(EPS_ERR_OOM, std::string(host ? "cudaHostAlloc(" : "cudaMalloc(") + std::to_string(bytes) + "): " +
                                 cudaGetErrorString(e));
  p = q;
  cap = bytes;
  owns = true;
  ++gen;
  return EPS_OK;
}

int Mem::grow(size_t bytes, size_t keep, cudaStream_t s) {
  if (bytes <= cap && p) return EPS_OK;
  Mem fresh;
  EPS_TRY(fresh.reserve(bytes));
  if (p && keep > 0) {
    EPS_CUDA(cudaMemcpyAsync(fresh.p, p, keep, cudaMemcpyDeviceToDevice, s));
    EPS_CUDA(cudaStreamSynchronize(s));
  }
  release();
  std::swap(p, fresh.p);
  std::swap(cap, fresh.cap);
  std::swap(owns, fresh.owns);
  ++gen;
  return EPS_OK;
}

void Mem::swap(Mem& o) {
  std::swap(p, o.p);
  std::swap(cap, o.cap);
  std::swap(owns, o.owns);
  ++gen;
  ++o.gen;
}

void Mem::release() {
  if (p && owns) {
    if (host) cudaFreeHost(p);
    else cudaFree(p);
  }
  p = nullptr;
  cap = 0;
  owns = false;
}

void Mem::alias(void* q, size_t bytes) {
  release();
  p = q;
  cap = bytes;
  ++gen;
}

int check_device(int device) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0)
    return fail(EPS_ERR_NO_DEVICE, std::string("no usable CUDA device (libepsilla_b200 has no CPU path): ") +
                                       (e != cudaSuccess ? cudaGetErrorString(e) : "device count 0"));
  if (device < 0 || device >= n) return fail(EPS_ERR_INVALID_ARGUMENT, "device ordinal out of range");
  EPS_CUDA(cudaSetDevice(device));
  return EPS_OK;
}

// Validate and lower the caller's node array (see filter.cuh).
int lower_filter(const eps_filter_node* nodes, int64_t n, FilterProg* out) {
  std::memset(out, 0, sizeof(*out));
  if (n <= 0 || nodes == nullptr) return EPS_OK;
  if (n > kMaxFilterNodes) return fail(EPS_ERR_UNSUPPORTED, "filter has more than 64 nodes");
  for (int64_t i = 0; i < n; ++i) {
    const eps_filter_node& s = nodes[i];
    FNode& d = out->nodes[i];
    const int t = static_cast<int>(s.node_type);
    switch (t) {
      case NT_IntConst: d.value = static_cast<double>(s.int_value); break;
      case NT_DoubleConst: d.value = s.double_value; break;
      case NT_BoolConst: d.value = s.bool_value ? 1.0 : 0.0; break;
      case NT_StringConst: d.value = static_cast<double>(s.int_value); break;  // dictionary code of the literal
      case NT_StringAttr:
        if (s.field_offset < 0 || s.field_offset >= kMaxStringCols)
          return fail(EPS_ERR_INVALID_ARGUMENT, "string attribute node needs a string-column index in [0, 8)");
        break;
      case NT_Int1Attr: case NT_Int2Attr: case NT_Int4Attr: case NT_Int8Attr: case NT_BoolAttr:
        if (s.field_offset < 0) return fail(EPS_ERR_INVALID_ARGUMENT, "filter attribute node without a field offset");
        break;
      case NT_DoubleAttr: case NT_FloatAttr:
        if (s.field_offset < 0 && s.field_offset != -2)
          return fail(EPS_ERR_INVALID_ARGUMENT, "filter attribute node without a field offset");
        if (s.field_offset == -2) out->uses_distance = 1;
        break;
      case NT_Add: case NT_Subtract: case NT_Multiply: case NT_Divide: case NT_Module: case NT_LT: case NT_LTE:
      case NT_EQ: case NT_GT: case NT_GTE: case NT_NE: case NT_AND: case NT_OR:
        if (s.left < 0 || s.left >= i || s.right < 0 || s.right >= i)
          return fail(EPS_ERR_INVALID_ARGUMENT, "filter node children must precede the node");
        break;
      case NT_NOT:
        if (s.left < 0 || s.left >= i) return fail(EPS_ERR_INVALID_ARGUMENT, "filter NOT child must precede the node");
        break;
      case NT_LIKE: {
        if (s.left < 0 || s.left >= i || s.right < 0 || s.right >= i)
          return fail(EPS_ERR_INVALID_ARGUMENT, "filter node children must precede the node");
        const int64_t lt = nodes[s.left].node_type, rt = nodes[s.right].node_type;
        if ((lt != NT_StringAttr && lt != NT_StringConst) || (rt != NT_StringAttr && rt != NT_StringConst))
          return fail(EPS_ERR_UNSUPPORTED, "LIKE operands must be string columns or literals (concatenation is out of scope)");
        break;
      }
      default:
        return fail(EPS_ERR_UNSUPPORTED,
                    "filter node type " + std::to_string(t) + " (IN not lowered to OR / geo / aggregation) is out of scope");
    }
    d.type = static_cast<int16_t>(t);
    d.vtype = static_cast<int16_t>(s.value_type);
    d.left = static_cast<int16_t>(s.left < 0 ? 0 : s.left);
    d.right = static_cast<int16_t>(s.right < 0 ? 0 : s.right);
    d.field_offset = static_cast<int32_t>(s.field_offset);
    if (t == NT_LIKE) {  // which bit prog_run reads (filter.cuh)
      const bool lc = nodes[s.left].node_type == NT_StringConst, rc = nodes[s.right].node_type == NT_StringConst;
      d.vtype = VT_BOOL;
      d.field_offset = lc && rc ? kLikeConst : (!lc && !rc ? kLikeByRow : (lc ? d.right : d.left));
    }
  }
  out->n = static_cast<int>(n);
  const FNode& r = out->nodes[n - 1];
  const bool cmp = r.type == NT_GT || r.type == NT_GTE || r.type == NT_LT || r.type == NT_LTE;
  const bool eq = (r.type == NT_EQ || r.type == NT_NE) && out->nodes[r.left].vtype != VT_BOOL &&
                  out->nodes[r.left].vtype != VT_STRING;  // string EQ goes through StrEvaluate: no distance
  out->root_uses_dist = (out->uses_distance && (cmp || eq)) ? 1 : 0;
  return EPS_OK;
}

__global__ void pair_distance_kernel(int metric, int vec4, const float* __restrict__ a, const float* __restrict__ b,
                                     int64_t n, int dim, float* __restrict__ out) {
  const int64_t w = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  float d = warp_distance(metric, vec4 != 0, a + w * dim, b + w * dim, dim, lane);
  if (lane == 0) out[w] = d;
}

// engine::Normalize (db/vector.cpp:60-69): v /= sqrt(sum v^2), fp32.
__global__ void normalize_kernel(float* __restrict__ v, int64_t n, int dim) {
  const int64_t w = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  float* p = v + w * dim;
  float s = 0.f;
  for (int i = lane; i < dim; i += 32) s = fmaf(p[i], p[i], s);
  s = sqrtf(warp_sum(s));
  for (int i = lane; i < dim; i += 32) p[i] = p[i] / s;
}

int normalize_rows_device(cudaStream_t s, float* d, int64_t n, int64_t dim) {
  normalize_kernel<<<static_cast<unsigned>((n * 32 + 127) / 128), 128, 0, s>>>(d, n, static_cast<int>(dim));
  EPS_CUDA(cudaGetLastError());
  return EPS_OK;
}

__global__ void narrow_ids_kernel(const int64_t* __restrict__ in, int64_t n, int64_t limit, int32_t* __restrict__ out,
                                  int* __restrict__ bad) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int64_t v = in[i];
  if (v < 0 || v >= limit) { *bad = 1; out[i] = 0; } else out[i] = static_cast<int32_t>(v);
}

void free_graph(Index* ix) {
  ix->d_offsets.release();
  ix->d_nbrs.release();
  ix->d_init_ids.release();
  ix->d_ell.release();
  free_sketch(ix);
  ix->seed_rows_L = 0;
  ix->init_L = 0;
  ix->n_indexed = 0;
  ix->n_edges = 0;
}

// Every attribute read of a lowered program must stay inside the mirrored row-major attribute table; string columns
// are bound to their device code arrays.
int bind_program_columns(Index* ix, FilterProg* prog) {
  for (int i = 0; i < prog->n; ++i) {
    const FNode& nd = prog->nodes[i];
    int width = 0;
    switch (nd.type) {
      case NT_Int1Attr: case NT_BoolAttr: width = 1; break;
      case NT_Int2Attr: width = 2; break;
      case NT_Int4Attr: case NT_FloatAttr: width = 4; break;
      case NT_Int8Attr: case NT_DoubleAttr: width = 8; break;
      default: break;
    }
    if (nd.type == NT_StringAttr) {
      const StrCol& sc = ix->str_cols[nd.field_offset];
      if (!sc.d_codes || sc.rows < ix->n_rows)
        return fail(EPS_ERR_INVALID_ARGUMENT, "expression reads a string column whose dictionary codes are not mirrored for every row");
      prog->str_col[nd.field_offset] = sc.d_codes;
      continue;
    }
    if (nd.type == NT_LIKE) continue;  // its field_offset selects a bit (check_like below)
    if (width == 0 || nd.field_offset < 0) continue;  // constants, operators, the @distance pseudo-field
    if (!ix->d_attrs) return fail(EPS_ERR_INVALID_ARGUMENT, "expression reads attributes but eps_index_set_attrs was not called");
    if (static_cast<int64_t>(nd.field_offset) + width > ix->attr_stride)
      return fail(EPS_ERR_INVALID_ARGUMENT, "field offset lies outside the attribute row");
    if (ix->attr_rows < ix->n_rows)
      return fail(EPS_ERR_INVALID_ARGUMENT, "attribute mirror has fewer rows than the vector mirror (call eps_index_set_attrs)");
  }
  return check_like(ix, *prog);
}

// A search call's queries, dense or sparse: their graph search over [0, n_indexed), and the exact scan's request
// with the queries filled in.
struct QueryBatch {
  ScanRequest scan;
  virtual ~QueryBatch() = default;
  virtual int graph(Index* ix, int64_t L, unsigned long long* d_queue, eps_stats* st) const = 0;
};

struct DenseBatch : QueryBatch {
  DenseBatch(const float* q, int64_t nq) { scan.queries = q; scan.nq = nq; }
  int graph(Index* ix, int64_t L, unsigned long long* d_queue, eps_stats* st) const override {
    return graph_search(ix, scan.queries, scan.nq, L, d_queue, st);
  }
};

struct SparseBatch : QueryBatch {
  const SparseDist& dist;  // the caller's: a copy of the batch still points at it
  // tile: the exact scan's producer, d itself or the inverted index's (the graph search always takes the raw queries);
  // l2_screen: the L2 screen's, or null
  SparseBatch(const SparseDist& d, const DistProducer& tile, const SparseL2Screen* l2_screen) : dist(d) {
    scan.dist = &tile;
    scan.nq = d.nq;
    scan.l2_screen = l2_screen;
  }
  int graph(Index* ix, int64_t L, unsigned long long* d_queue, eps_stats* st) const override {
    return sparse_graph_search(ix, dist.q, dist.nq, L, d_queue, st);
  }
};

// Below this many passing rows, a collect-mode call answers the whole batch by the scan over the passing rows, which
// costs nq x P distances; above it the graph search runs and only the queries it leaves short are scanned (DESIGN.md
// §K3).  EPS_COLLECT_SCAN_ROWS overrides it (developer knob: tools/filtered_check.py times both sides with it).
constexpr int64_t kCollectScanRows = 65536;
static int64_t collect_scan_rows() {
  const char* e = getenv("EPS_COLLECT_SCAN_ROWS");
  return e ? atoll(e) : kCollectScanRows;
}

// EPS_FILTER_SEARCH_COLLECT: the graph branch of a filtered dense search that returns min(cap, P) rows per query, P = the
// rows that are not deleted and pass the filter.  The keys go to ix->s_ckeys [nq x cap] for finalize_keys.
//   1. the pass bitmap of rows [0, total) and P;
//   2. P <= collect_scan_rows(): the exact scan over the passing rows answers every query;
//   3. otherwise the graph search keeps, per query, the best cap passing rows it evaluates, and
//   4. the filtered tail scan of rows [n_indexed, total) is merged in exactly;
//   5. queries left with fewer than min(cap, P) rows are answered by the scan over the passing rows.
// eps_stats.n_redone counts the queries answered in 2 or 5.
static int collect_search(Index* ix, ScanRequest scan, int64_t L, int64_t cap, eps_stats* local, eps_stats* stats) {
  if (cap > 8192) return fail(EPS_ERR_UNSUPPORTED, "collect filter search: more than 8192 results per query are not supported");
  const int64_t nq = scan.nq, total = ix->n_rows, n_indexed = ix->n_indexed;
  scan.row_start = 0; scan.row_end = total;
  int64_t P = 0;
  EPS_TRY(collect_pass(ix, scan, &P, &local->kernel_launches));
  EPS_TRY(ix->s_ckeys.reserve(static_cast<size_t>(nq) * cap * 8));
  unsigned long long* keys = ix->s_ckeys.as<unsigned long long>();
  if (P <= collect_scan_rows()) {
    EPS_TRY(passing_topk(ix, scan.queries, nq, nullptr, nq, cap, P, keys, local));
    local->n_redone += static_cast<uint64_t>(nq);
    if (stats) EPS_CUDA(cudaEventRecord(ix->ev[2], ix->stream));
    return EPS_OK;
  }
  EPS_TRY(ix->s_queue.reserve(static_cast<size_t>(nq) * L * 8));
  EPS_TRY(ix->s_clist.reserve(static_cast<size_t>(nq) * cap * 8));
  const GraphCollect gc{ix->s_cpass.as<uint32_t>(), ix->s_clist.as<unsigned long long>(), cap};
  EPS_TRY(graph_search(ix, scan.queries, nq, L, ix->s_queue.as<unsigned long long>(), local, &gc));
  ix->graph_counters_pending = true;
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[2], ix->stream));
  int64_t tail_k = 0;
  if (total > n_indexed) {
    tail_k = std::min<int64_t>(cap, total - n_indexed);
    EPS_TRY(ix->s_tail.reserve(static_cast<size_t>(nq) * tail_k * 8));
    scan.row_start = n_indexed; scan.k = tail_k;
    EPS_TRY(exact_topk(ix, scan, ix->s_tail.as<unsigned long long>(), local));
  }
  const int* d_short = nullptr;
  int64_t n_short = 0;
  EPS_TRY(collect_merge(ix, gc.out, ix->s_tail.as<unsigned long long>(), nq, cap, tail_k, P, keys, &d_short, &n_short));
  local->kernel_launches += 1;
  if (n_short > 0) {
    EPS_TRY(passing_topk(ix, scan.queries, nq, d_short, n_short, cap, P, keys, local));
    local->n_redone += static_cast<uint64_t>(n_short);
  }
  return EPS_OK;
}

// VecSearchExecutor::Search (:833-935) of nq queries into device ids / dists / counts.  ev[1] -> ev[2] brackets the
// search kernels when stats are wanted.
static int run_search(Index* ix, const QueryBatch& qb, int64_t nq, int64_t limit, const eps_filter_node* filter,
                      int64_t n_filter, int64_t* d_ids, float* d_dists, int64_t* d_counts, eps_stats* stats) {
  if (nq <= 0) return EPS_OK;
  if (limit < 1) return fail(EPS_ERR_INVALID_ARGUMENT, "limit must be >= 1");
  FilterProg h_prog;
  EPS_TRY(lower_filter(filter, n_filter, &h_prog));
  const int64_t total = ix->n_rows;
  const int64_t n_indexed = ix->n_indexed;
  // BruteforceThreshold (hpp:28); a sparse index in EPS_SPARSE_SEARCH_SCAN always scans, whatever graph is installed
  const bool graph = !ix->prefilter && !ix->force_brute && n_indexed >= 512 &&
                     (!ix->sparse || ix->sparse_search == EPS_SPARSE_SEARCH_GRAPH);
  const bool collect = graph && !ix->sparse && h_prog.n > 0 && ix->filter_search == EPS_FILTER_SEARCH_COLLECT;
  if (collect && h_prog.root_uses_dist)
    return fail(EPS_ERR_UNSUPPORTED, "collect filter search: a filter whose root compares @distance cannot be decided before "
                                     "the distance is known (use EPS_FILTER_SEARCH_POST)");
  const FilterProg* d_prog = nullptr;
  uint64_t like_launches = 0;
  if (h_prog.n > 0) {
    EPS_TRY(bind_program_columns(ix, &h_prog));
    EPS_TRY(bind_like(ix, &h_prog, 1, &like_launches));
    EPS_TRY(ix->s_filter.reserve(sizeof(FilterProg)));
    EPS_CUDA(cudaMemcpyAsync(ix->s_filter.p, &h_prog, sizeof(FilterProg), cudaMemcpyHostToDevice, ix->stream));
    // h_prog lives on this stack frame until the sync at the end of the caller's timing region; the copy
    // from pageable memory is staged synchronously by the runtime, so it is safe.
    d_prog = ix->s_filter.as<FilterProg>();
  }
  eps_stats local;
  std::memset(&local, 0, sizeof(local));
  local.kernel_launches = like_launches;  // the LIKE pass
  ScanRequest scan = qb.scan;
  scan.metric = ix->metric; scan.d_prog = d_prog; scan.h_prog = &h_prog;
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[1], ix->stream));
  if (collect) {
    const int64_t L = std::min<int64_t>(ix->L_master, n_indexed);
    const int64_t cap = std::min<int64_t>(std::min<int64_t>(std::min<int64_t>(n_indexed, limit), ix->L_local), L);
    EPS_TRY(collect_search(ix, scan, L, cap, &local, stats));
    EPS_TRY(finalize_keys(ix, ix->s_ckeys.as<unsigned long long>(), nq, cap, limit, cap, d_ids, d_dists, d_counts));
  } else if (graph) {
    // :869-933: graph search, exact scan of the rows appended after the build, merge of the two and post-filter walk
    const int64_t L = std::min<int64_t>(ix->L_master, n_indexed);  // Q1 clamp
    // :872 min(n_indexed, limit, L_local); the queue row holds L entries, so the merge window is clamped to it
    // (the reference ties L_local to L_master through setSearchQueueSize; the C ABI accepts them separately)
    const int64_t search_limit = std::min<int64_t>(std::min<int64_t>(std::min<int64_t>(n_indexed, limit), ix->L_local), L);
    EPS_TRY(ix->s_queue.reserve(static_cast<size_t>(nq) * L * 8));
    EPS_TRY(qb.graph(ix, L, ix->s_queue.as<unsigned long long>(), &local));
    ix->graph_counters_pending = true;
    if (stats) EPS_CUDA(cudaEventRecord(ix->ev[2], ix->stream));
    const unsigned long long* d_tail = nullptr;
    int64_t tail_k = 0;
    if (total > n_indexed) {  // :885-900
      // only the first search_limit slots can receive tail entries (:894-900)
      tail_k = std::min<int64_t>(std::min<int64_t>(limit, total - n_indexed), search_limit);
      if (tail_k > 8192) return fail(EPS_ERR_UNSUPPORTED, "more than 8192 tail results per query are not supported");
      EPS_TRY(ix->s_tail.reserve(static_cast<size_t>(nq) * tail_k * 8));
      scan.row_start = n_indexed; scan.row_end = total; scan.k = tail_k;
      EPS_TRY(exact_topk(ix, scan, ix->s_tail.as<unsigned long long>(), &local));
      d_tail = ix->s_tail.as<unsigned long long>();
    }
    EPS_TRY(finalize_graph(ix, ix->s_queue.as<unsigned long long>(), nq, L, search_limit, L, d_tail, tail_k, limit,
                           d_prog, &h_prog, d_ids, d_dists, d_counts));
  } else {
    // :857 prefilter: min(size, limit); :864 brute: min(size, limit, L_local).  Only that many entries are ever
    // emitted, so the exact top-k is taken for the EFFECTIVE k (a large `limit` on a small table is legal).
    const int64_t cap = (ix->prefilter || ix->force_brute) ? limit : std::min<int64_t>(limit, ix->L_local);
    const int64_t k = std::max<int64_t>(1, std::min<int64_t>(cap, total));
    if (k > 8192) return fail(EPS_ERR_UNSUPPORTED, "more than 8192 results per query from the exact scan are not supported");
    EPS_TRY(ix->s_topk.reserve(static_cast<size_t>(nq) * k * 8));
    scan.row_end = total; scan.k = k; scan.prefilter = ix->prefilter;
    EPS_TRY(exact_topk(ix, scan, ix->s_topk.as<unsigned long long>(), &local));
    if (stats) EPS_CUDA(cudaEventRecord(ix->ev[2], ix->stream));
    EPS_TRY(finalize_keys(ix, ix->s_topk.as<unsigned long long>(), nq, k, limit, cap, d_ids, d_dists, d_counts));
  }
  local.kernel_launches += 1;  // finalize_graph / finalize_keys
  if (stats) {
    stats->n_dist += local.n_dist;
    stats->n_seed += local.n_seed;
    stats->n_expand += local.n_expand;
    stats->n_edges += local.n_edges;
    stats->n_queries += static_cast<uint64_t>(nq);
    stats->kernel_launches += local.kernel_launches;
    stats->n_redone += local.n_redone;
  }
  return EPS_OK;
}

// The end of a call with stats, after the stream is synchronised: the graph search's counters if it ran, the kernel
// time ev[1] -> ev[2] and the call's time ev[0] -> ev[3].
static int finish_stats(Index* ix, eps_stats* stats) {
  if (ix->graph_counters_pending) {
    EPS_TRY(read_graph_counters(ix, stats));
    ix->graph_counters_pending = false;
  }
  float ms = 0.f;
  cudaEventElapsedTime(&ms, ix->ev[1], ix->ev[2]);
  stats->kernel_ms += ms;
  cudaEventElapsedTime(&ms, ix->ev[0], ix->ev[3]);
  stats->total_ms += ms;
  return EPS_OK;
}

// run_search of queries already on the device, returned to the caller's host arrays: one device block
// [ids | counts | dists] and one pinned host mirror of it, so a single D2H copy per call.
static int search_to_host(Index* ix, const QueryBatch& qb, int64_t nq, int64_t limit, const eps_filter_node* filter,
                          int64_t n_filter, int64_t* out_ids, double* out_dists, int64_t* out_counts, eps_stats* stats) {
  const size_t n_ids = static_cast<size_t>(nq) * limit;
  const size_t off_cnt = n_ids * 8, off_dist = off_cnt + static_cast<size_t>(nq) * 8, total = off_dist + n_ids * 4;
  EPS_TRY(ix->s_out_ids.reserve(total));
  EPS_TRY(ix->h_out.reserve(total));
  unsigned char* d_blk = ix->s_out_ids.as<unsigned char>();
  EPS_TRY(run_search(ix, qb, nq, limit, filter, n_filter, reinterpret_cast<int64_t*>(d_blk),
                     reinterpret_cast<float*>(d_blk + off_dist), reinterpret_cast<int64_t*>(d_blk + off_cnt), stats));
  EPS_CUDA(cudaMemcpyAsync(ix->h_out.p, d_blk, total, cudaMemcpyDeviceToHost, ix->stream));
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[3], ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  const unsigned char* hb = ix->h_out.as<const unsigned char>();
  std::memcpy(out_ids, hb, n_ids * 8);
  std::memcpy(out_counts, hb + off_cnt, static_cast<size_t>(nq) * 8);
  const float* hd = reinterpret_cast<const float*>(hb + off_dist);
  for (size_t i = 0; i < n_ids; ++i) out_dists[i] = static_cast<double>(hd[i]);  // distance_ is vector<double> (hpp:52)
  if (stats) EPS_TRY(finish_stats(ix, stats));
  ix->graph_counters_pending = false;
  return EPS_OK;
}

static int dense_only(const Index* ix) {
  if (ix->sparse) return fail(EPS_ERR_INVALID_ARGUMENT, "dense-vector call on a sparse index");
  return EPS_OK;
}

}  // namespace eps

using eps::Index;

extern "C" {

const char* eps_last_error(void) { return eps::g_err.c_str(); }
const char* eps_version(void) { return "epsilla_b200 0.1 (sm_90a)"; }
int eps_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

int eps_index_create(eps_index** out, int metric, int64_t dim, const float* host_vectors, int64_t capacity_rows,
                     int device) {
  if (!out) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "out is null");
  *out = nullptr;
  if (dim < 1 || capacity_rows < 0) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "bad dim / capacity");
  if (metric != EPS_METRIC_L2 && metric != EPS_METRIC_COSINE && metric != EPS_METRIC_IP)
    metric = EPS_METRIC_L2;  // GetDistFunc default branch (db/index/index.cpp:19-20)
  EPS_TRY(eps::check_device(device));
  std::unique_ptr<Index> ix(new Index());  // deleted on the error paths with its device current
  ix->device = device;
  ix->metric = metric;
  ix->dim = dim;
  ix->capacity = capacity_rows;
  ix->host_vectors = host_vectors;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) {
    ix->num_sms = prop.multiProcessorCount;
    ix->smem_per_sm = static_cast<int>(prop.sharedMemPerMultiprocessor);
    ix->smem_reserved_per_cta = static_cast<int>(prop.reservedSharedMemPerBlock);
  }
  cudaError_t e = cudaStreamCreateWithFlags(&ix->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) return eps::fail(EPS_ERR_CUDA, cudaGetErrorString(e));
  for (auto& ev : ix->ev) cudaEventCreate(&ev);
  if (capacity_rows > 0 && host_vectors) EPS_TRY(ix->d_vectors.reserve(static_cast<size_t>(capacity_rows) * dim * 4));
  ix->vec4 = (dim % 4 == 0);
  *out = reinterpret_cast<eps_index*>(ix.release());
  return EPS_OK;
}

int eps_index_create_sparse(eps_index** out, int metric, int64_t dim, int64_t capacity_rows, int device) {
  if (!out) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "out is null");
  *out = nullptr;
  if (dim < 1 || dim >= 0xffffffffll || capacity_rows < 0)
    return eps::fail(EPS_ERR_INVALID_ARGUMENT, "bad dim (must be in [1, 2^32 - 1)) / capacity");
  if (metric != EPS_METRIC_L2 && metric != EPS_METRIC_COSINE && metric != EPS_METRIC_IP) metric = EPS_METRIC_L2;
  EPS_TRY(eps::check_device(device));
  eps_index* h = nullptr;
  EPS_TRY(eps_index_create(&h, metric, dim, nullptr, 0, device));
  Index* ix = reinterpret_cast<Index*>(h);
  ix->sparse = true;
  ix->capacity = capacity_rows;
  const int64_t rows = std::max<int64_t>(capacity_rows, 1);
  auto row_table = [&]() -> int {
    EPS_TRY(ix->d_sp_ptr.reserve(static_cast<size_t>(rows + 1) * 8));
    EPS_TRY(ix->d_sp_norm2.reserve(static_cast<size_t>(rows) * 4));
    EPS_CUDA(cudaMemset(ix->d_sp_ptr, 0, 8));
    return EPS_OK;
  };
  if (const int rc = row_table(); rc != EPS_OK) {
    eps_index_destroy(h);
    return rc;
  }
  *out = h;
  return EPS_OK;
}

void eps_index_destroy(eps_index* h) {
  if (!h) return;
  Index* ix = reinterpret_cast<Index*>(h);
  cudaSetDevice(ix->device);
  cudaStreamSynchronize(ix->stream);
  if (Index* base = ix->view_of) {
    --base->n_views;
    base->views.erase(std::remove(base->views.begin(), base->views.end(), ix), base->views.end());
  }
  for (Index* v : ix->views) {  // base destroyed before its views: they become empty indexes instead of dangling
    cudaStreamSynchronize(v->stream);
    v->view_of = nullptr; v->detached_view = true;
    const int64_t nav = v->nav;  // eps_index_get_graph still reports it
    static_cast<eps::Table&>(*v) = eps::Table();
    v->nav = nav;
  }
  delete ix;
}

// A read-only view of an index: the same device table, graph and segment mirrors, its own stream and scratch.
// Searches on a view and on its base (or on several views) run concurrently — the tail of one batch, where a few
// long queries hold their SMs alone, overlaps the head of the next.  The base refuses to be modified while it has views.
int eps_index_create_view(eps_index* base_h, eps_index** out) {
  if (!out) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "out is null");
  *out = nullptr;
  Index* base = reinterpret_cast<Index*>(base_h);
  if (!base) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (base->view_of) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "a view cannot be the base of another view");
  EPS_TRY(eps::check_device(base->device));
  EPS_TRY(eps::ensure_ell(base, nullptr));
  EPS_CUDA(cudaStreamSynchronize(base->stream));  // uploads, graph install and the adjacency table are complete
  Index* ix = new Index();
  ix->view_of = base;
  ix->device = base->device; ix->metric = base->metric; ix->dim = base->dim; ix->sparse = base->sparse;
  ix->num_sms = base->num_sms; ix->smem_per_sm = base->smem_per_sm; ix->smem_reserved_per_cta = base->smem_reserved_per_cta;
  static_cast<eps::Table&>(*ix) = *base;
  static_cast<eps::Config&>(*ix) = *base;
  cudaError_t e = cudaStreamCreateWithFlags(&ix->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { delete ix; return eps::fail(EPS_ERR_CUDA, cudaGetErrorString(e)); }
  for (auto& ev : ix->ev) cudaEventCreate(&ev);
  ++base->n_views;
  base->views.push_back(ix);
  *out = reinterpret_cast<eps_index*>(ix);
  return EPS_OK;
}

// table, graph and segment mirrors of a view belong to its base; a base with live views is frozen
static int check_mutable(const Index* ix) {
  if (ix->view_of || ix->detached_view) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "a view is read-only");
  if (ix->n_views > 0) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "the index has live views: destroy them before modifying it");
  return EPS_OK;
}

int eps_index_sync_rows(eps_index* h, int64_t n_rows_now) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::check_device(ix->device));
  EPS_TRY(eps::dense_only(ix));
  EPS_TRY(check_mutable(ix));
  if (!ix->d_vectors.owns) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "index has no host vector table to mirror");
  if (n_rows_now < ix->n_rows || n_rows_now > ix->capacity)
    return eps::fail(EPS_ERR_INVALID_ARGUMENT, "n_rows_now outside [mirrored rows, capacity]");
  if (n_rows_now > ix->n_rows) {
    const size_t off = static_cast<size_t>(ix->n_rows) * ix->dim;
    const size_t cnt = static_cast<size_t>(n_rows_now - ix->n_rows) * ix->dim;
    EPS_CUDA(cudaMemcpyAsync(ix->d_vectors + off, ix->host_vectors + off, cnt * 4, cudaMemcpyHostToDevice, ix->stream));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
    ix->n_rows = n_rows_now;
  }
  return EPS_OK;
}

int eps_index_adopt_device_rows(eps_index* h, const float* d_vectors, int64_t n_rows) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix || !d_vectors) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null argument");
  EPS_TRY(eps::dense_only(ix));
  EPS_TRY(eps::check_device(ix->device));
  EPS_TRY(check_mutable(ix));
  if (n_rows < 0 || n_rows >= (1ll << 31)) return eps::fail(EPS_ERR_UNSUPPORTED, "row count must be in [0, 2^31): keys carry 31-bit ids");
  ix->d_vectors.alias(const_cast<float*>(d_vectors), static_cast<size_t>(n_rows) * ix->dim * 4);
  // state derived from the previous table: gathered seed rows always, the graph itself if it no longer fits
  ix->seed_rows_L = 0;
  eps::free_sketch(ix);  // computed from the rows this call replaces
  if (ix->n_indexed > n_rows) eps::free_graph(ix);
  ix->n_rows = n_rows;
  if (n_rows > ix->capacity) ix->capacity = n_rows;
  ix->vec4 = (ix->dim % 4 == 0) && ((reinterpret_cast<uintptr_t>(d_vectors) & 15) == 0);
  ix->xnorm_rows = 0;  // derived mirrors (row norms, bf16 copy) belong to the previous table
  ix->bf16_rows = 0;
  return EPS_OK;
}

int eps_index_set_graph(eps_index* h, int64_t n_indexed, const int64_t* offsets, const int64_t* nbrs, int64_t nav) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::dense_only(ix));
  EPS_TRY(eps::check_device(ix->device));
  EPS_TRY(check_mutable(ix));
  eps::free_graph(ix);
  if (n_indexed <= 0) return EPS_OK;
  if (!offsets) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null offset table");
  if (n_indexed > ix->n_rows) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "graph covers rows that are not mirrored yet");
  if (n_indexed >= (1ll << 31)) return eps::fail(EPS_ERR_UNSUPPORTED, "more than 2^31 indexed rows");
  if (nav < 0 || nav >= n_indexed) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "navigation point out of range");
  const int64_t e = offsets[n_indexed];
  if (offsets[0] != 0 || e < 0) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "offset table must start at 0 and end at the edge count");
  for (int64_t i = 0; i < n_indexed; ++i)
    if (offsets[i + 1] < offsets[i]) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "offset table is not monotonic");
  if (e > 0 && !nbrs) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null neighbor list");
  EPS_TRY(ix->d_offsets.reserve((static_cast<size_t>(n_indexed) + 1) * 8));
  EPS_TRY(ix->d_nbrs.reserve(static_cast<size_t>(e > 0 ? e : 1) * 4));
  EPS_CUDA(cudaMemcpyAsync(ix->d_offsets, offsets, (static_cast<size_t>(n_indexed) + 1) * 8, cudaMemcpyHostToDevice, ix->stream));
  // neighbour ids: int64 in the reference CSR, int32 on the device — narrowed and range-checked by a kernel over
  // 64M-edge chunks (a host loop over 4e8 edges costs seconds)
  {
    const int64_t chunk = 64ll << 20;
    eps::DevBuf stage, flag;
    EPS_TRY(stage.reserve(static_cast<size_t>(std::min<int64_t>(chunk, std::max<int64_t>(e, 1))) * 8));
    EPS_TRY(flag.reserve(4));
    EPS_CUDA(cudaMemsetAsync(flag.p, 0, 4, ix->stream));
    for (int64_t c0 = 0; c0 < e; c0 += chunk) {
      const int64_t cn = std::min(chunk, e - c0);
      EPS_CUDA(cudaMemcpyAsync(stage.p, nbrs + c0, static_cast<size_t>(cn) * 8, cudaMemcpyHostToDevice, ix->stream));
      eps::narrow_ids_kernel<<<static_cast<unsigned>((cn + 255) / 256), 256, 0, ix->stream>>>(stage.as<int64_t>(), cn, n_indexed,
                                                                                              ix->d_nbrs + c0, flag.as<int>());
      EPS_CUDA(cudaGetLastError());
      EPS_CUDA(cudaStreamSynchronize(ix->stream));  // the staging buffer is reused by the next chunk
    }
    int bad = 0;
    EPS_CUDA(cudaMemcpy(&bad, flag.p, 4, cudaMemcpyDeviceToHost));
    if (bad) { eps::free_graph(ix); return eps::fail(EPS_ERR_INVALID_ARGUMENT, "neighbor id out of range"); }
  }
  ix->n_indexed = n_indexed;
  ix->n_edges = e;
  ix->nav = nav;
  eps::ensure_sketch(ix);
  return EPS_OK;
}

int eps_index_build(eps_index* h, int64_t n, const eps_build_params* params) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::check_device(ix->device));
  EPS_TRY(check_mutable(ix));
  if (ix->sparse) return eps::build_graph_sparse(ix, n, params);
  EPS_TRY(eps::build_graph(ix, n, params));
  eps::ensure_sketch(ix);
  return EPS_OK;
}

int eps_index_extend_graph(eps_index* h, int64_t n, const eps_build_params* params) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::dense_only(ix));
  EPS_TRY(check_mutable(ix));
  if (ix->n_indexed == 0) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "extend_graph: no graph installed (build one with eps_index_build)");
  if (n < ix->n_indexed) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "extend_graph: n below the indexed rows");
  if (n >= (1ll << 31)) return eps::fail(EPS_ERR_UNSUPPORTED, "extend_graph: more than 2^31 rows per shard");
  if (n > ix->n_rows) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "extend_graph: n above the mirrored rows");
  if (n == ix->n_indexed) return EPS_OK;
  EPS_TRY(eps::check_device(ix->device));
  return eps::extend_graph(ix, n, params);
}

int eps_index_get_graph(eps_index* h, int64_t* n_indexed, int64_t* n_edges, int64_t* offsets, int64_t* nbrs,
                        int64_t* nav) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::check_device(ix->device));
  if (n_indexed) *n_indexed = ix->n_indexed;
  if (n_edges) *n_edges = ix->n_edges;
  if (nav) *nav = ix->nav;
  if (ix->n_indexed == 0) return EPS_OK;
  if (offsets) EPS_CUDA(cudaMemcpy(offsets, ix->d_offsets, (static_cast<size_t>(ix->n_indexed) + 1) * 8, cudaMemcpyDeviceToHost));
  if (nbrs && ix->n_edges > 0) {
    std::vector<int32_t> nb32(static_cast<size_t>(ix->n_edges));
    EPS_CUDA(cudaMemcpy(nb32.data(), ix->d_nbrs, nb32.size() * 4, cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < ix->n_edges; ++i) nbrs[i] = nb32[i];
  }
  return EPS_OK;
}

// The reference flips single bits of deleted_ (db/table_segment_mvp.cpp:429-449) and exposes no dirty tracking, so
// the mirror keeps a host shadow of what it uploaded and ships only the byte span that changed since the last
// call (nothing at all in the common case): a 64-bit-word compare of N/8 bytes instead of an N/8-byte H2D copy.
int eps_index_set_deleted(eps_index* h, const uint8_t* bitset, int64_t nbytes) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::check_device(ix->device));
  EPS_TRY(check_mutable(ix));
  if (!bitset || nbytes <= 0) { ix->any_deleted = false; ix->deleted_bytes = 0; ix->h_deleted.clear(); return EPS_OK; }
  int64_t lo = 0, hi = nbytes;  // dirty span [lo, hi)
  const bool same_geometry = ix->d_deleted && static_cast<int64_t>(ix->h_deleted.size()) == nbytes && nbytes <= ix->d_deleted.count();
  if (same_geometry) {
    const uint8_t* old = ix->h_deleted.data();
    int64_t w = 0;
    const int64_t nw = nbytes / 8;
    while (w < nw && reinterpret_cast<const uint64_t*>(old)[w] == reinterpret_cast<const uint64_t*>(bitset)[w]) ++w;
    lo = w * 8;
    while (lo < nbytes && old[lo] == bitset[lo]) ++lo;
    if (lo == nbytes) return EPS_OK;  // unchanged
    hi = nbytes;
    while (hi > lo && old[hi - 1] == bitset[hi - 1]) --hi;
  } else {
    // room for the whole table so that growth of record_number_ never reallocates; the old bitmap is freed only
    // once the new one is allocated, so a failure leaves the mirror as it was
    if (nbytes > ix->d_deleted.count())
      EPS_TRY(ix->d_deleted.grow(static_cast<size_t>(std::max<int64_t>(nbytes, (ix->capacity + 7) / 8 + 8)), 0, ix->stream));
    // nothing is known to be on the device until the whole bitset is
    ix->h_deleted.clear();
    ix->deleted_bytes = 0;
    ix->any_deleted = false;
  }
  EPS_CUDA(cudaMemcpyAsync(ix->d_deleted + lo, bitset + lo, static_cast<size_t>(hi - lo), cudaMemcpyHostToDevice, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  ix->h_deleted.resize(static_cast<size_t>(nbytes));
  std::memcpy(ix->h_deleted.data() + lo, bitset + lo, static_cast<size_t>(hi - lo));
  ix->deleted_bytes = nbytes;
  if (!ix->any_deleted) {
    bool any = false;
    for (int64_t i = lo; i < hi && !any; ++i) any = bitset[i] != 0;
    ix->any_deleted = any;  // sticky: un-deleting every row only costs a bitmap test per row
  }
  return EPS_OK;
}

// attribute_table_ is append-only for rows below record_number_ (an upsert deletes the old row and appends a new
// one, db/table_segment_mvp.cpp:564-587): the same table grown to more rows uploads only the new rows.
int eps_index_set_attrs(eps_index* h, const char* table, int64_t stride, int64_t n_rows) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::check_device(ix->device));
  EPS_TRY(check_mutable(ix));
  if (!table || stride <= 0 || n_rows <= 0) {
    ix->d_attrs.release();
    ix->attr_stride = stride; ix->attr_rows = 0; ix->attr_src = nullptr;
    return EPS_OK;
  }
  int64_t first = 0;
  if (ix->d_attrs && ix->attr_src == table && ix->attr_stride == stride && n_rows >= ix->attr_rows &&
      n_rows <= static_cast<int64_t>(ix->d_attrs.cap) / stride) {
    first = ix->attr_rows;  // append
  } else {
    ix->d_attrs.release();
    EPS_TRY(ix->d_attrs.reserve(static_cast<size_t>(stride) * std::max<int64_t>(n_rows, ix->capacity)));
  }
  ix->attr_stride = stride;
  ix->attr_src = table;
  if (n_rows > first) {
    EPS_CUDA(cudaMemcpyAsync(ix->d_attrs + first * stride, table + first * stride, static_cast<size_t>(stride) * (n_rows - first),
                             cudaMemcpyHostToDevice, ix->stream));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
  }
  ix->attr_rows = n_rows;
  return EPS_OK;
}

// Dictionary codes of rows [first_row, first_row + count) of string column `column` (TableSegmentMVP::
// var_len_attr_table_[column], db/table_segment_mvp.hpp:82).  Rows are append-only like the attribute table.
int eps_index_set_string_codes(eps_index* h, int column, int64_t first_row, const int32_t* codes, int64_t count) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (column < 0 || column >= eps::kMaxStringCols) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "string column index must be in [0, 8)");
  if (first_row < 0 || count < 0 || (count > 0 && !codes)) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "bad row range / null codes");
  EPS_TRY(eps::check_device(ix->device));
  EPS_TRY(check_mutable(ix));
  eps::StrCol& sc = ix->str_cols[column];
  if (first_row > sc.rows) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "string codes must be appended without gaps");
  const int64_t need = first_row + count;
  if (need > sc.d_codes.count()) {
    const int64_t cap = std::max<int64_t>(need, std::max<int64_t>(ix->capacity, 2 * sc.d_codes.count()));
    EPS_TRY(sc.d_codes.grow(static_cast<size_t>(cap) * 4, static_cast<size_t>(sc.rows) * 4, ix->stream));
  }
  if (count > 0) {
    EPS_CUDA(cudaMemcpyAsync(sc.d_codes + first_row, codes, static_cast<size_t>(count) * 4, cudaMemcpyHostToDevice, ix->stream));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
  }
  // code range of the mirror, for LIKE (check_like): a rewrite of every row starts afresh, otherwise it only widens
  if (first_row == 0 && need >= sc.rows) { sc.any_negative = false; sc.max_code = -1; }
  for (int64_t i = 0; i < count; ++i) {
    sc.any_negative |= codes[i] < 0;
    sc.max_code = std::max(sc.max_code, codes[i]);
  }
  sc.rows = std::max(sc.rows, need);
  return EPS_OK;
}

int eps_index_append_string_dictionary(eps_index* h, int64_t first_code, int64_t count, const int64_t* offsets,
                                       const char* bytes) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::check_device(ix->device));
  EPS_TRY(check_mutable(ix));
  return eps::dict_append(ix, first_code, count, offsets, bytes);
}

int eps_index_config(eps_index* h, int64_t L_master, int64_t L_local, int prefilter, int force_brute) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (L_master < 1 || L_local < 1) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "queue sizes must be >= 1");
  ix->L_master = L_master;
  ix->L_local = L_local;
  ix->prefilter = prefilter != 0;
  ix->force_brute = force_brute != 0;
  return EPS_OK;
}

int eps_search_batch_device(eps_index* h, const float* d_queries, int64_t nq, int64_t limit,
                            const eps_filter_node* filter, int64_t n_filter, int64_t* d_out_ids, float* d_out_dists,
                            int64_t* d_out_counts, eps_stats* stats, int sync) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix || !d_queries || !d_out_ids || !d_out_dists || !d_out_counts)
    return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null argument");
  EPS_TRY(eps::dense_only(ix));
  if (nq <= 0) return EPS_OK;  // nothing launched: no events to read back
  EPS_TRY(eps::check_device(ix->device));
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[0], ix->stream));
  EPS_TRY(eps::run_search(ix, eps::DenseBatch(d_queries, nq), nq, limit, filter, n_filter, d_out_ids, d_out_dists,
                          d_out_counts, stats));
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[3], ix->stream));
  else ix->graph_counters_pending = false;
  if (sync || stats) EPS_CUDA(cudaStreamSynchronize(ix->stream));
  if (stats) EPS_TRY(eps::finish_stats(ix, stats));
  return EPS_OK;
}

int eps_search_batch(eps_index* h, const float* queries, int64_t nq, int64_t limit, const eps_filter_node* filter,
                     int64_t n_filter, int64_t* out_ids, double* out_dists, int64_t* out_counts, eps_stats* stats) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix || !queries || !out_ids || !out_dists || !out_counts) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null argument");
  EPS_TRY(eps::dense_only(ix));
  if (nq <= 0) return EPS_OK;
  if (limit < 1) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "limit must be >= 1");
  EPS_TRY(eps::check_device(ix->device));
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[0], ix->stream));
  EPS_TRY(ix->s_queries.reserve(static_cast<size_t>(nq) * ix->dim * 4));
  EPS_CUDA(cudaMemcpyAsync(ix->s_queries.p, queries, static_cast<size_t>(nq) * ix->dim * 4, cudaMemcpyHostToDevice, ix->stream));
  return eps::search_to_host(ix, eps::DenseBatch(ix->s_queries.as<float>(), nq), nq, limit, filter, n_filter, out_ids,
                             out_dists, out_counts, stats);
}

int eps_index_append_sparse_rows(eps_index* h, int64_t first_row, int64_t n_rows, const int64_t* offsets,
                                 const int64_t* indices, const float* values) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (!ix->sparse) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "sparse rows appended to a dense index");
  EPS_TRY(eps::check_device(ix->device));
  EPS_TRY(check_mutable(ix));
  return eps::sparse_append(ix, first_row, n_rows, offsets, indices, values);
}

int eps_search_sparse_batch(eps_index* h, int64_t nq, const int64_t* q_offsets, const int64_t* q_indices, const float* q_values,
                            int64_t limit, const eps_filter_node* filter, int64_t n_filter, int64_t* out_ids, double* out_dists,
                            int64_t* out_counts, eps_stats* stats) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix || !out_ids || !out_dists || !out_counts) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null argument");
  if (!ix->sparse) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "sparse search on a dense index");
  if (nq <= 0) return EPS_OK;
  if (!q_offsets) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null query offsets");
  if (limit < 1) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "limit must be >= 1");
  EPS_TRY(eps::check_device(ix->device));
  // queries: any index the 32-bit element holds (the merge needs them strictly increasing)
  std::vector<int64_t> qp;
  std::vector<uint2> qe;
  std::vector<float> qn;
  EPS_TRY(eps::pack_sparse(nq, q_offsets, q_indices, q_values, 0xffffffffll, 0, &qp, &qe, &qn));
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[0], ix->stream));
  eps::SparseQueries q;
  EPS_TRY(eps::upload_sparse_queries(ix, qp, qe, qn, &ix->s_sparse_q, &q));
  const eps::SparseDist dist(q, nq);
  const eps::InvertedDist inv(dist, static_cast<int64_t>(qe.size()));
  const eps::SparseL2Screen screen(inv);
  // posting lists: the inverted index of an IP / cosine index, the L2 screen of an L2 one
  const bool lists = ix->inv_rows > 0, l2 = ix->metric == EPS_METRIC_L2;
  const eps::DistProducer& tile = lists && !l2 ? static_cast<const eps::DistProducer&>(inv) : dist;
  return eps::search_to_host(ix, eps::SparseBatch(dist, tile, lists && l2 ? &screen : nullptr), nq, limit, filter,
                             n_filter, out_ids, out_dists, out_counts, stats);
}

int eps_index_build_sparse_inverted(eps_index* h, int64_t n) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (!ix->sparse) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "inverted index on a dense index");
  if (ix->metric == EPS_METRIC_L2)
    return eps::fail(EPS_ERR_UNSUPPORTED, "inverted index on an L2 index: the L2 sum also adds the row-only and "
                                          "query-only terms in merged index order, which posting lists cannot reproduce "
                                          "(eps_index_build_sparse_l2_screen builds the L2 screen)");
  EPS_TRY(check_mutable(ix));
  if (n < 0 || n > ix->n_rows) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "inverted index: n outside [0, mirrored rows]");
  EPS_TRY(eps::check_device(ix->device));
  return eps::build_sparse_inverted(ix, n);
}

int eps_index_sparse_inverted_info(eps_index* h, int64_t* n_rows, int64_t* n_terms, int64_t* n_postings) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (!ix->sparse) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "inverted index info on a dense index");
  if (n_rows) *n_rows = ix->inv_rows;
  if (n_terms) *n_terms = ix->inv_terms;
  if (n_postings) *n_postings = ix->inv_postings;
  return EPS_OK;
}

int eps_index_build_sparse_l2_screen(eps_index* h, int64_t n) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (!ix->sparse) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "L2 screen on a dense index");
  if (ix->metric != EPS_METRIC_L2)
    return eps::fail(EPS_ERR_INVALID_ARGUMENT, "L2 screen on an inner-product or cosine index: its posting lists give "
                                               "the exact distances (eps_index_build_sparse_inverted)");
  EPS_TRY(check_mutable(ix));
  if (n < 0 || n > ix->n_rows) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "L2 screen: n outside [0, mirrored rows]");
  EPS_TRY(eps::check_device(ix->device));
  return eps::build_sparse_inverted(ix, n);
}

int eps_index_extend_sparse_postings(eps_index* h, int64_t n) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (!ix->sparse) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "posting lists on a dense index");
  EPS_TRY(check_mutable(ix));
  if (ix->inv_rows == 0)
    return eps::fail(EPS_ERR_INVALID_ARGUMENT, "extend_sparse_postings: no posting lists (build them first with "
                                               "eps_index_build_sparse_inverted or eps_index_build_sparse_l2_screen)");
  if (n < ix->inv_rows) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "extend_sparse_postings: n below the covered rows");
  if (n > ix->n_rows) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "extend_sparse_postings: n above the mirrored rows");
  if (n == ix->inv_rows) return EPS_OK;
  EPS_TRY(eps::check_device(ix->device));
  return eps::extend_sparse_inverted(ix, n);
}

int eps_index_get_sparse_postings(eps_index* h, int64_t* n_rows, int64_t* n_terms, int64_t* n_postings, uint32_t* terms,
                                  int64_t* ptr, int32_t* rows, float* values) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (!ix->sparse) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "posting lists of a dense index");
  if (n_rows) *n_rows = ix->inv_rows;
  if (n_terms) *n_terms = ix->inv_terms;
  if (n_postings) *n_postings = ix->inv_postings;
  if (ix->inv_rows == 0 || !(terms || ptr || rows || values)) return EPS_OK;
  EPS_TRY(eps::check_device(ix->device));
  if (terms && ix->inv_terms > 0)
    EPS_CUDA(cudaMemcpyAsync(terms, ix->d_inv_terms, static_cast<size_t>(ix->inv_terms) * 4, cudaMemcpyDeviceToHost, ix->stream));
  if (ptr)
    EPS_CUDA(cudaMemcpyAsync(ptr, ix->d_inv_ptr, static_cast<size_t>(ix->inv_terms + 1) * 8, cudaMemcpyDeviceToHost, ix->stream));
  std::vector<uint2> post;
  if ((rows || values) && ix->inv_postings > 0) {
    post.resize(static_cast<size_t>(ix->inv_postings));
    EPS_CUDA(cudaMemcpyAsync(post.data(), ix->d_inv_post, post.size() * 8, cudaMemcpyDeviceToHost, ix->stream));
  }
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  for (size_t i = 0; i < post.size(); ++i) {  // {row, value bits} pairs
    if (rows) rows[i] = static_cast<int32_t>(post[i].x);
    if (values) std::memcpy(&values[i], &post[i].y, 4);
  }
  return EPS_OK;
}

int eps_index_sparse_l2_screen_info(eps_index* h, int64_t* n_rows, uint64_t* n_rescored) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (!ix->sparse) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "L2 screen info on a dense index");
  if (n_rows) *n_rows = ix->metric == EPS_METRIC_L2 ? ix->inv_rows : 0;
  if (n_rescored) {
    *n_rescored = 0;
    if (ix->d_l2_rescored) {
      EPS_TRY(eps::check_device(ix->device));
      EPS_CUDA(cudaStreamSynchronize(ix->stream));
      unsigned long long v = 0;
      EPS_CUDA(cudaMemcpy(&v, ix->d_l2_rescored, 8, cudaMemcpyDeviceToHost));
      *n_rescored = v;
    }
  }
  return EPS_OK;
}

int eps_merge_shards_device(int device, const int64_t* d_ids, const float* d_dists, int64_t n_shards, int64_t nq,
                            int64_t k, int64_t* d_out_ids, float* d_out_dists) {
  EPS_TRY(eps::check_device(device));
  EPS_TRY(eps::merge_shards(device, nullptr, d_ids, d_dists, n_shards, nq, k, d_out_ids, d_out_dists));
  EPS_CUDA(cudaStreamSynchronize(nullptr));
  return EPS_OK;
}

int eps_normalize(int device, float* host_vectors, int64_t nq, int64_t dim) {
  EPS_TRY(eps::check_device(device));
  if (nq <= 0) return EPS_OK;
  if (!host_vectors || dim < 1) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null vectors / bad dim");
  const size_t bytes = static_cast<size_t>(nq) * dim * 4;
  eps::Mem d;
  EPS_TRY(d.reserve(bytes));
  EPS_CUDA(cudaMemcpy(d.p, host_vectors, bytes, cudaMemcpyHostToDevice));
  EPS_TRY(eps::normalize_rows_device(nullptr, d.as<float>(), nq, dim));
  EPS_CUDA(cudaMemcpy(host_vectors, d.p, bytes, cudaMemcpyDeviceToHost));
  return EPS_OK;
}

int eps_pair_distances(int device, int metric, const float* a, const float* b, int64_t n, int64_t dim, float* out) {
  EPS_TRY(eps::check_device(device));
  if (n <= 0) return EPS_OK;
  if (!a || !b || !out || dim < 1) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null argument / bad dim");
  const size_t bytes = static_cast<size_t>(n) * dim * 4;
  eps::Mem da, db, dout;
  EPS_TRY(da.reserve(bytes));
  EPS_TRY(db.reserve(bytes));
  EPS_TRY(dout.reserve(static_cast<size_t>(n) * 4));
  EPS_CUDA(cudaMemcpy(da.p, a, bytes, cudaMemcpyHostToDevice));
  EPS_CUDA(cudaMemcpy(db.p, b, bytes, cudaMemcpyHostToDevice));
  eps::pair_distance_kernel<<<static_cast<unsigned>((n * 32 + 127) / 128), 128>>>(metric, dim % 4 == 0 ? 1 : 0, da.as<float>(),
                                                                                 db.as<float>(), n, static_cast<int>(dim),
                                                                                 dout.as<float>());
  EPS_CUDA(cudaDeviceSynchronize());
  EPS_CUDA(cudaMemcpy(out, dout.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost));
  return EPS_OK;
}

int eps_index_set_search_width(eps_index* h, int width) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::dense_only(ix));
  if (width < 1 || width > 8) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "search width must be in [1, 8]");
  ix->search_width = width;
  return EPS_OK;
}

int eps_index_set_filter_search(eps_index* h, int mode) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (ix->sparse) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "filter search mode on a sparse index (its default search is exact)");
  if (mode != EPS_FILTER_SEARCH_POST && mode != EPS_FILTER_SEARCH_COLLECT)
    return eps::fail(EPS_ERR_INVALID_ARGUMENT, "filter search mode must be 0 (post) or 1 (collect)");
  ix->filter_search = mode;
  return EPS_OK;
}

int eps_index_set_sparse_search(eps_index* h, int mode) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (!ix->sparse) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "sparse search mode on a dense index");
  if (mode != EPS_SPARSE_SEARCH_SCAN && mode != EPS_SPARSE_SEARCH_GRAPH)
    return eps::fail(EPS_ERR_INVALID_ARGUMENT, "sparse search mode must be 0 (scan) or 1 (graph)");
  ix->sparse_search = mode;
  return EPS_OK;
}

int eps_index_set_graph_tuning(eps_index* h, int ring_slots, int ctas_per_sm) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::dense_only(ix));
  if (ring_slots < 0 || ring_slots > 24 || ctas_per_sm < 0 || ctas_per_sm > 32)
    return eps::fail(EPS_ERR_INVALID_ARGUMENT, "ring_slots must be in [0, 24] and ctas_per_sm in [0, 32] (0 = auto)");
  ix->graph_ring_slots = ring_slots;
  ix->graph_ctas_per_sm = ctas_per_sm;
  return EPS_OK;
}

int eps_index_set_graph_screen(eps_index* h, int mode) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::dense_only(ix));
  EPS_TRY(check_mutable(ix));
  if (mode != EPS_GRAPH_SCREEN_OFF && mode != EPS_GRAPH_SCREEN_ON && mode != EPS_GRAPH_SCREEN_AUTO)
    return eps::fail(EPS_ERR_INVALID_ARGUMENT, "graph screen mode must be 0 (off), 1 (on) or 2 (auto)");
  EPS_TRY(eps::check_device(ix->device));
  ix->graph_screen = mode;
  eps::ensure_sketch(ix);
  return EPS_OK;
}

int eps_index_graph_screen_info(eps_index* h, int* active, double* share, uint64_t* n_screened) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (active) *active = eps::screen_on(ix) ? 1 : 0;
  if (share) *share = ix->sk_share;
  if (n_screened) {
    *n_screened = 0;
    if (ix->d_screened) {
      EPS_TRY(eps::check_device(ix->device));
      EPS_CUDA(cudaStreamSynchronize(ix->stream));
      unsigned long long v = 0;
      EPS_CUDA(cudaMemcpy(&v, ix->d_screened, 8, cudaMemcpyDeviceToHost));
      *n_screened = v;
    }
  }
  return EPS_OK;
}

int eps_index_set_coarse(eps_index* h, int mode) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::dense_only(ix));
  if (mode < 0 || mode > 2) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "coarse mode must be 0 (fp32), 1 (tf32) or 2 (bf16)");
  if (mode != ix->coarse_mode) ix->coarse_boost = 1;  // the learnt k' multiplier belongs to one operand format
  ix->coarse_mode = mode;
  return EPS_OK;
}

int eps_index_set_coarse_guard(eps_index* h, int on) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  ix->coarse_guard = on ? 1 : 0;
  return EPS_OK;
}

const float* eps_index_device_rows(eps_index* h) {
  if (!h) return nullptr;
  if (eps::dense_only(reinterpret_cast<Index*>(h)) != EPS_OK) return nullptr;
  return reinterpret_cast<Index*>(h)->d_vectors;
}
int64_t eps_index_rows(eps_index* h) { return h ? reinterpret_cast<Index*>(h)->n_rows : 0; }

void* eps_index_stream(eps_index* h) { return h ? reinterpret_cast<Index*>(h)->stream : nullptr; }

}  // extern "C"
