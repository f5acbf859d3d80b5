// C ABI of libepsilla_b200 (include/epsilla_b200.h): index lifetime, segment mirrors, and the batched
// VecSearchExecutor::Search orchestration (engine/db/execution/vec_search_executor.cpp:833-935).
#include <cmath>
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <mutex>

#include "internal.h"

namespace eps {

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

int DevBuf::reserve(size_t bytes) {
  if (bytes <= cap && p) return EPS_OK;
  if (p) { cudaFree(p); p = nullptr; cap = 0; }
  size_t want = bytes < 256 ? 256 : bytes;
  cudaError_t e = cudaMalloc(&p, want);
  if (e != cudaSuccess) {
    p = nullptr;
    return fail(EPS_ERR_OOM, std::string("cudaMalloc(") + std::to_string(want) + "): " + cudaGetErrorString(e));
  }
  cap = want;
  return EPS_OK;
}
void DevBuf::release() {
  if (p) cudaFree(p);
  p = nullptr;
  cap = 0;
}

static int check_device(int device) {
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
      default:
        return fail(EPS_ERR_UNSUPPORTED,
                    "filter node type " + std::to_string(t) + " (LIKE / IN not lowered to OR / geo / aggregation) is out of scope");
    }
    d.type = static_cast<int16_t>(t);
    d.vtype = static_cast<int16_t>(s.value_type);
    d.left = static_cast<int16_t>(s.left < 0 ? 0 : s.left);
    d.right = static_cast<int16_t>(s.right < 0 ? 0 : s.right);
    d.field_offset = static_cast<int32_t>(s.field_offset);
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

static void free_graph(Index* ix) {
  if (ix->d_offsets) cudaFree(ix->d_offsets);
  if (ix->d_nbrs) cudaFree(ix->d_nbrs);
  if (ix->d_init_ids) cudaFree(ix->d_init_ids);
  if (ix->d_ell) cudaFree(ix->d_ell);
  ix->d_ell = nullptr;
  ix->seed_rows_L = 0;
  ix->d_offsets = nullptr;
  ix->d_nbrs = nullptr;
  ix->d_init_ids = nullptr;
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
    if (width == 0 || nd.field_offset < 0) continue;  // constants, operators, the @distance pseudo-field
    if (!ix->d_attrs) return fail(EPS_ERR_INVALID_ARGUMENT, "expression reads attributes but eps_index_set_attrs was not called");
    if (static_cast<int64_t>(nd.field_offset) + width > ix->attr_stride)
      return fail(EPS_ERR_INVALID_ARGUMENT, "field offset lies outside the attribute row");
    if (ix->attr_rows < ix->n_rows)
      return fail(EPS_ERR_INVALID_ARGUMENT, "attribute mirror has fewer rows than the vector mirror (call eps_index_set_attrs)");
  }
  return EPS_OK;
}

static int search_device(Index* ix, const float* d_queries, int64_t nq, int64_t limit, const eps_filter_node* filter,
                         int64_t n_filter, int64_t* d_ids, float* d_dists, int64_t* d_counts, eps_stats* stats) {
  if (nq <= 0) return EPS_OK;
  if (limit < 1) return fail(EPS_ERR_INVALID_ARGUMENT, "limit must be >= 1");
  FilterProg h_prog;
  EPS_TRY(lower_filter(filter, n_filter, &h_prog));
  const FilterProg* d_prog = nullptr;
  if (h_prog.n > 0) {
    EPS_TRY(bind_program_columns(ix, &h_prog));
    EPS_TRY(ix->s_filter.reserve(sizeof(FilterProg)));
    EPS_CUDA(cudaMemcpyAsync(ix->s_filter.p, &h_prog, sizeof(FilterProg), cudaMemcpyHostToDevice, ix->stream));
    // h_prog lives on this stack frame until the sync at the end of the caller's timing region; the copy
    // from pageable memory is staged synchronously by the runtime, so it is safe.
    d_prog = ix->s_filter.as<FilterProg>();
  }
  const int64_t total = ix->n_rows;
  const int64_t n_indexed = ix->n_indexed;
  const bool brute = ix->prefilter || ix->force_brute || n_indexed < 512;  // BruteforceThreshold (hpp:28)
  eps_stats local;
  std::memset(&local, 0, sizeof(local));
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[1], ix->stream));
  if (brute) {
    // :857 prefilter: min(size, limit); :864 brute: min(size, limit, L_local).  Only that many entries are ever
    // emitted, so the exact top-k is taken for the EFFECTIVE k (a large `limit` on a small table is legal).
    const int64_t cap = (ix->prefilter || ix->force_brute) ? limit : std::min<int64_t>(limit, ix->L_local);
    const int64_t k = std::max<int64_t>(1, std::min<int64_t>(cap, total));
    if (k > 8192) return fail(EPS_ERR_UNSUPPORTED, "more than 8192 results per query from the exact scan are not supported");
    EPS_TRY(ix->s_topk.reserve(static_cast<size_t>(nq) * k * 8));
    EPS_TRY(brute_force_topk(ix, d_queries, nq, 0, total, k, d_prog, &h_prog, ix->prefilter,
                             ix->s_topk.as<unsigned long long>(), &local));
    if (stats) EPS_CUDA(cudaEventRecord(ix->ev[2], ix->stream));
    EPS_TRY(finalize_keys(ix, ix->s_topk.as<unsigned long long>(), nq, k, limit, cap, d_ids, d_dists, d_counts));
    local.kernel_launches += 1;
  } else {
    const int64_t L = std::min<int64_t>(ix->L_master, n_indexed);  // Q1 clamp
    // :872 min(n_indexed, limit, L_local); the queue row holds L entries, so the merge window is clamped to it
    // (the reference ties L_local to L_master through setSearchQueueSize; the C ABI accepts them separately)
    const int64_t search_limit = std::min<int64_t>(std::min<int64_t>(std::min<int64_t>(n_indexed, limit), ix->L_local), L);
    EPS_TRY(ix->s_queue.reserve(static_cast<size_t>(nq) * L * 8));
    EPS_TRY(graph_search(ix, d_queries, nq, L, ix->s_queue.as<unsigned long long>(), &local));
    ix->graph_counters_pending = true;
    if (stats) EPS_CUDA(cudaEventRecord(ix->ev[2], ix->stream));
    const unsigned long long* d_tail = nullptr;
    int64_t tail_k = 0;
    if (total > n_indexed) {  // :885-900
      // only the first search_limit slots can receive tail entries (:894-900)
      tail_k = std::min<int64_t>(std::min<int64_t>(limit, total - n_indexed), search_limit);
      if (tail_k > 8192) return fail(EPS_ERR_UNSUPPORTED, "more than 8192 tail results per query are not supported");
      EPS_TRY(ix->s_tail.reserve(static_cast<size_t>(nq) * tail_k * 8));
      EPS_TRY(brute_force_topk(ix, d_queries, nq, n_indexed, total, tail_k, d_prog, &h_prog, false,
                               ix->s_tail.as<unsigned long long>(), &local));
      d_tail = ix->s_tail.as<unsigned long long>();
    }
    EPS_TRY(finalize_graph(ix, ix->s_queue.as<unsigned long long>(), nq, L, search_limit, L, d_tail, tail_k, limit,
                           d_prog, &h_prog, d_ids, d_dists, d_counts));
    local.kernel_launches += 1;
  }
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
  Index* ix = new Index();
  ix->device = device;
  ix->metric = metric;
  ix->dim = dim;
  ix->capacity = capacity_rows;
  ix->host_vectors = host_vectors;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ix->num_sms = prop.multiProcessorCount;
  cudaError_t e = cudaStreamCreateWithFlags(&ix->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { delete ix; return eps::fail(EPS_ERR_CUDA, cudaGetErrorString(e)); }
  for (auto& ev : ix->ev) cudaEventCreate(&ev);
  if (capacity_rows > 0 && host_vectors) {
    e = cudaMalloc(&ix->d_vectors, static_cast<size_t>(capacity_rows) * dim * 4);
    if (e != cudaSuccess) {
      cudaStreamDestroy(ix->stream);
      delete ix;
      return eps::fail(EPS_ERR_OOM, std::string("vector table: ") + cudaGetErrorString(e));
    }
    ix->owns_vectors = true;
  }
  ix->vec4 = (dim % 4 == 0);
  *out = reinterpret_cast<eps_index*>(ix);
  return EPS_OK;
}

void eps_index_destroy(eps_index* h) {
  if (!h) return;
  Index* ix = reinterpret_cast<Index*>(h);
  cudaSetDevice(ix->device);
  cudaStreamSynchronize(ix->stream);
  if (ix->view_of) {  // a view owns its seed set, stream and scratch only
    if (ix->d_init_ids) cudaFree(ix->d_init_ids);
    Index* base = ix->view_of;
    --base->n_views;
    base->views.erase(std::remove(base->views.begin(), base->views.end(), ix), base->views.end());
  } else if (ix->detached_view) {
    if (ix->d_init_ids) cudaFree(ix->d_init_ids);  // its base went first: nothing shared is left to release
  } else {
    for (Index* v : ix->views) {  // base destroyed before its views: they become empty indexes instead of dangling
      cudaStreamSynchronize(v->stream);
      v->view_of = nullptr; v->detached_view = true;
      v->d_vectors = nullptr; v->n_rows = 0; v->capacity = 0;
      v->d_offsets = nullptr; v->d_nbrs = nullptr; v->d_ell = nullptr; v->n_indexed = 0; v->n_edges = 0;
      v->d_deleted = nullptr; v->deleted_bytes = 0; v->any_deleted = false;
      v->d_attrs = nullptr; v->attr_rows = 0;
      for (auto& sc : v->str_cols) sc = eps::StrCol();
    }
    ix->views.clear();
    eps::free_graph(ix);
    if (ix->owns_vectors && ix->d_vectors) cudaFree(ix->d_vectors);
    if (ix->d_deleted) cudaFree(ix->d_deleted);
    if (ix->d_attrs) cudaFree(ix->d_attrs);
    for (auto& sc : ix->str_cols) if (sc.d_codes) cudaFree(sc.d_codes);
  }
  eps::DevBuf* bufs[] = {&ix->s_queries, &ix->s_dist, &ix->s_topk, &ix->s_topk2, &ix->s_pass, &ix->s_filter,
                         &ix->s_visited, &ix->s_vlog, &ix->s_queue, &ix->s_tail, &ix->s_out_ids, &ix->s_out_dists,
                         &ix->s_out_counts, &ix->s_stats, &ix->s_misc, &ix->s_seed_rows, &ix->s_seed_dist, &ix->s_xnorm, &ix->s_qnorm, &ix->s_coarse, &ix->s_thr, &ix->s_cand, &ix->s_cand_cnt, &ix->s_bf16, &ix->s_qbf16, &ix->s_flags};
  for (auto* b : bufs) b->release();
  if (ix->h_out) cudaFreeHost(ix->h_out);
  for (auto& ev : ix->ev) if (ev) cudaEventDestroy(ev);
  cudaStreamDestroy(ix->stream);
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
  ix->device = base->device; ix->metric = base->metric; ix->dim = base->dim; ix->capacity = base->capacity;
  ix->host_vectors = nullptr; ix->d_vectors = base->d_vectors; ix->owns_vectors = false; ix->n_rows = base->n_rows;
  ix->vec4 = base->vec4;
  ix->n_indexed = base->n_indexed; ix->n_edges = base->n_edges; ix->nav = base->nav;
  ix->d_offsets = base->d_offsets; ix->d_nbrs = base->d_nbrs; ix->d_ell = base->d_ell;
  ix->d_deleted = base->d_deleted; ix->deleted_bytes = base->deleted_bytes; ix->deleted_cap = base->deleted_cap;
  ix->any_deleted = base->any_deleted;
  ix->d_attrs = base->d_attrs; ix->attr_stride = base->attr_stride; ix->attr_rows = base->attr_rows;
  ix->attr_cap_rows = base->attr_cap_rows;
  for (int i = 0; i < eps::kMaxStringCols; ++i) ix->str_cols[i] = base->str_cols[i];
  ix->L_master = base->L_master; ix->L_local = base->L_local; ix->prefilter = base->prefilter; ix->force_brute = base->force_brute;
  ix->search_width = base->search_width; ix->graph_ring_slots = base->graph_ring_slots;
  ix->graph_ctas_per_sm = base->graph_ctas_per_sm; ix->num_sms = base->num_sms;
  ix->coarse_mode = base->coarse_mode; ix->coarse_guard = base->coarse_guard; ix->coarse_boost = base->coarse_boost;
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
  EPS_TRY(check_mutable(ix));
  if (!ix->owns_vectors) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "index has no host vector table to mirror");
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
  EPS_TRY(eps::check_device(ix->device));
  EPS_TRY(check_mutable(ix));
  if (n_rows < 0 || n_rows >= (1ll << 31)) return eps::fail(EPS_ERR_UNSUPPORTED, "row count must be in [0, 2^31): keys carry 31-bit ids");
  if (ix->owns_vectors && ix->d_vectors) cudaFree(ix->d_vectors);
  ix->owns_vectors = false;
  ix->d_vectors = const_cast<float*>(d_vectors);
  // state derived from the previous table: gathered seed rows always, the graph itself if it no longer fits
  ix->seed_rows_L = 0;
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
  EPS_CUDA(cudaMalloc(&ix->d_offsets, (static_cast<size_t>(n_indexed) + 1) * 8));
  EPS_CUDA(cudaMalloc(&ix->d_nbrs, static_cast<size_t>(e > 0 ? e : 1) * 4));
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
  return EPS_OK;
}

int eps_index_build(eps_index* h, int64_t n, const eps_build_params* params) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  EPS_TRY(eps::check_device(ix->device));
  EPS_TRY(check_mutable(ix));
  return eps::build_graph(ix, n, params);
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
  const bool same_geometry = ix->d_deleted && static_cast<int64_t>(ix->h_deleted.size()) == nbytes && nbytes <= ix->deleted_cap;
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
    if (nbytes > ix->deleted_cap) {
      if (ix->d_deleted) cudaFree(ix->d_deleted);
      ix->d_deleted = nullptr;
      // room for the whole table so that growth of record_number_ never reallocates
      const int64_t cap = std::max<int64_t>(nbytes, (ix->capacity + 7) / 8 + 8);
      EPS_CUDA(cudaMalloc(&ix->d_deleted, static_cast<size_t>(cap)));
      ix->deleted_cap = cap;
    }
    ix->h_deleted.assign(static_cast<size_t>(nbytes), 0);
    ix->any_deleted = false;
  }
  EPS_CUDA(cudaMemcpyAsync(ix->d_deleted + lo, bitset + lo, static_cast<size_t>(hi - lo), cudaMemcpyHostToDevice, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
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
    if (ix->d_attrs) { cudaFree(ix->d_attrs); ix->d_attrs = nullptr; }
    ix->attr_stride = stride; ix->attr_rows = 0; ix->attr_cap_rows = 0; ix->attr_src = nullptr;
    return EPS_OK;
  }
  int64_t first = 0;
  if (ix->d_attrs && ix->attr_src == table && ix->attr_stride == stride && n_rows >= ix->attr_rows && n_rows <= ix->attr_cap_rows) {
    first = ix->attr_rows;  // append
  } else {
    if (ix->d_attrs) { cudaFree(ix->d_attrs); ix->d_attrs = nullptr; }
    const int64_t cap = std::max<int64_t>(n_rows, ix->capacity);
    EPS_CUDA(cudaMalloc(&ix->d_attrs, static_cast<size_t>(stride) * cap));
    ix->attr_cap_rows = cap;
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
  if (need > sc.cap) {
    const int64_t cap = std::max<int64_t>(need, std::max<int64_t>(ix->capacity, 2 * sc.cap));
    int32_t* fresh = nullptr;
    EPS_CUDA(cudaMalloc(&fresh, static_cast<size_t>(cap) * 4));
    if (sc.d_codes && sc.rows > 0) {
      cudaError_t e = cudaMemcpyAsync(fresh, sc.d_codes, static_cast<size_t>(sc.rows) * 4, cudaMemcpyDeviceToDevice, ix->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(ix->stream);
      if (e != cudaSuccess) { cudaFree(fresh); return eps::fail(EPS_ERR_CUDA, cudaGetErrorString(e)); }
    }
    if (sc.d_codes) cudaFree(sc.d_codes);
    sc.d_codes = fresh;
    sc.cap = cap;
  }
  if (count > 0) {
    EPS_CUDA(cudaMemcpyAsync(sc.d_codes + first_row, codes, static_cast<size_t>(count) * 4, cudaMemcpyHostToDevice, ix->stream));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
  }
  sc.rows = std::max(sc.rows, need);
  return EPS_OK;
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
  if (nq <= 0) return EPS_OK;  // nothing launched: no events to read back
  EPS_TRY(eps::check_device(ix->device));
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[0], ix->stream));
  EPS_TRY(eps::search_device(ix, d_queries, nq, limit, filter, n_filter, d_out_ids, d_out_dists, d_out_counts, stats));
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[3], ix->stream));
  if (!stats) ix->graph_counters_pending = false;
  if (sync || stats) {
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
    if (stats) {
      if (ix->graph_counters_pending) { EPS_TRY(eps::read_graph_counters(ix, stats)); ix->graph_counters_pending = false; }
      float ms = 0.f;
      cudaEventElapsedTime(&ms, ix->ev[1], ix->ev[2]);
      stats->kernel_ms += ms;
      cudaEventElapsedTime(&ms, ix->ev[0], ix->ev[3]);
      stats->total_ms += ms;
    }
  }
  return EPS_OK;
}

int eps_search_batch(eps_index* h, const float* queries, int64_t nq, int64_t limit, const eps_filter_node* filter,
                     int64_t n_filter, int64_t* out_ids, double* out_dists, int64_t* out_counts, eps_stats* stats) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix || !queries || !out_ids || !out_dists || !out_counts) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null argument");
  if (nq <= 0) return EPS_OK;
  if (limit < 1) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "limit must be >= 1");
  EPS_TRY(eps::check_device(ix->device));
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[0], ix->stream));
  // one device block [ids | counts | dists] and one pinned host mirror of it: a single D2H copy per call
  const size_t n_ids = static_cast<size_t>(nq) * limit;
  const size_t off_cnt = n_ids * 8, off_dist = off_cnt + static_cast<size_t>(nq) * 8, total = off_dist + n_ids * 4;
  EPS_TRY(ix->s_queries.reserve(static_cast<size_t>(nq) * ix->dim * 4));
  EPS_TRY(ix->s_out_ids.reserve(total));
  if (ix->h_out_cap < total) {
    if (ix->h_out) cudaFreeHost(ix->h_out);
    ix->h_out = nullptr;
    ix->h_out_cap = 0;
    EPS_CUDA(cudaHostAlloc(&ix->h_out, total, cudaHostAllocDefault));
    ix->h_out_cap = total;
  }
  unsigned char* d_blk = ix->s_out_ids.as<unsigned char>();
  EPS_CUDA(cudaMemcpyAsync(ix->s_queries.p, queries, static_cast<size_t>(nq) * ix->dim * 4, cudaMemcpyHostToDevice, ix->stream));
  EPS_TRY(eps::search_device(ix, ix->s_queries.as<float>(), nq, limit, filter, n_filter, reinterpret_cast<int64_t*>(d_blk),
                             reinterpret_cast<float*>(d_blk + off_dist), reinterpret_cast<int64_t*>(d_blk + off_cnt), stats));
  EPS_CUDA(cudaMemcpyAsync(ix->h_out, d_blk, total, cudaMemcpyDeviceToHost, ix->stream));
  if (stats) EPS_CUDA(cudaEventRecord(ix->ev[3], ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  const unsigned char* hb = static_cast<const unsigned char*>(ix->h_out);
  std::memcpy(out_ids, hb, n_ids * 8);
  std::memcpy(out_counts, hb + off_cnt, static_cast<size_t>(nq) * 8);
  const float* hd = reinterpret_cast<const float*>(hb + off_dist);
  for (size_t i = 0; i < n_ids; ++i) out_dists[i] = static_cast<double>(hd[i]);  // distance_ is vector<double> (hpp:52)
  if (stats) {
    if (ix->graph_counters_pending) { EPS_TRY(eps::read_graph_counters(ix, stats)); ix->graph_counters_pending = false; }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ix->ev[1], ix->ev[2]);
    stats->kernel_ms += ms;
    cudaEventElapsedTime(&ms, ix->ev[0], ix->ev[3]);
    stats->total_ms += ms;
  }
  ix->graph_counters_pending = false;
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
  float* d = nullptr;
  EPS_CUDA(cudaMalloc(&d, bytes));
  cudaError_t e = cudaMemcpy(d, host_vectors, bytes, cudaMemcpyHostToDevice);
  int rc = EPS_OK;
  if (e == cudaSuccess) rc = eps::normalize_rows_device(nullptr, d, nq, dim);
  if (e == cudaSuccess && rc == EPS_OK) e = cudaMemcpy(host_vectors, d, bytes, cudaMemcpyDeviceToHost);
  cudaFree(d);
  if (e != cudaSuccess) return eps::fail(EPS_ERR_CUDA, cudaGetErrorString(e));
  return rc;
}

int eps_pair_distances(int device, int metric, const float* a, const float* b, int64_t n, int64_t dim, float* out) {
  EPS_TRY(eps::check_device(device));
  if (n <= 0) return EPS_OK;
  if (!a || !b || !out || dim < 1) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null argument / bad dim");
  float *da = nullptr, *db = nullptr, *dout = nullptr;
  const size_t bytes = static_cast<size_t>(n) * dim * 4;
  cudaError_t e = cudaMalloc(&da, bytes);
  if (e == cudaSuccess) e = cudaMalloc(&db, bytes);
  if (e == cudaSuccess) e = cudaMalloc(&dout, static_cast<size_t>(n) * 4);
  if (e == cudaSuccess) e = cudaMemcpy(da, a, bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(db, b, bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    eps::pair_distance_kernel<<<static_cast<unsigned>((n * 32 + 127) / 128), 128>>>(metric, dim % 4 == 0 ? 1 : 0, da, db, n,
                                                                                   static_cast<int>(dim), dout);
    e = cudaDeviceSynchronize();
  }
  if (e == cudaSuccess) e = cudaMemcpy(out, dout, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost);
  cudaFree(da); cudaFree(db); cudaFree(dout);
  if (e != cudaSuccess) return eps::fail(EPS_ERR_CUDA, cudaGetErrorString(e));
  return EPS_OK;
}

int eps_index_set_search_width(eps_index* h, int width) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (width < 1 || width > 8) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "search width must be in [1, 8]");
  ix->search_width = width;
  return EPS_OK;
}

int eps_index_set_graph_tuning(eps_index* h, int ring_slots, int ctas_per_sm) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
  if (ring_slots < 0 || ring_slots > 24 || ctas_per_sm < 0 || ctas_per_sm > 32)
    return eps::fail(EPS_ERR_INVALID_ARGUMENT, "ring_slots must be in [0, 24] and ctas_per_sm in [0, 32] (0 = auto)");
  ix->graph_ring_slots = ring_slots;
  ix->graph_ctas_per_sm = ctas_per_sm;
  return EPS_OK;
}

int eps_index_set_coarse(eps_index* h, int mode) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null index");
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

const float* eps_index_device_rows(eps_index* h) { return h ? reinterpret_cast<Index*>(h)->d_vectors : nullptr; }
int64_t eps_index_rows(eps_index* h) { return h ? reinterpret_cast<Index*>(h)->n_rows : 0; }

void* eps_index_stream(eps_index* h) { return h ? reinterpret_cast<Index*>(h)->stream : nullptr; }

}  // extern "C"
