// K5 — sparse-vector fields (SPARSE_VECTOR_FLOAT / _DOUBLE): device CSR mirror, query upload, exact scan, graph build.
//
// The reference's sparse distances (GetL2DistSqr / GetInnerProductDist / GetCosineDist) are reproduced bit for bit by
// SparseMerge and sparse_finish (common.cuh), which the sparse graph search (sparse_graph.cu) shares.
//
// sparse_dist_kernel writes the same [nq x chunk] fp32 tile as launch_distances; the exact scan's pass bitmap,
// bf_select_kernel and finalize_keys then run unchanged (exact_topk, brute_force.cu).
//   * one CTA = a tile of up to 32 queries (one per lane) x a slice of rows; the tile's elements are staged in shared
//     memory when they fit (kSpQCap), else lanes read their query from global memory;
//   * a warp walks one row at a time: 32 elements per coalesced 8-byte load, broadcast by shuffles, and every lane
//     feeds them to its own query's SparseMerge (a two-pointer merge: the only way to get the L2 order right);
//   * results of 32 rows are transposed through shared memory so the tile is written in 128-byte rows.
// Query tiles of the same row slice are adjacent in launch order, so a slice is read from HBM about once and from L2
// by the other tiles.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <unordered_map>

#include "internal.h"

namespace eps {

constexpr int kSpQ = 32;        // queries per CTA tile (one per lane)
constexpr int kSpWarps = 8;
constexpr int kSpQCap = 4096;   // query elements staged in shared memory per tile (32 KB)
constexpr size_t kSpSmem = static_cast<size_t>(kSpQCap) * 8 + static_cast<size_t>(kSpWarps) * 32 * 33 * 4;

template <int METRIC>
__global__ void __launch_bounds__(kSpWarps * 32) sparse_dist_kernel(
    const int64_t* __restrict__ row_ptr, const uint2* __restrict__ elems, const float* __restrict__ row_norm2,
    int64_t row_start, int64_t n, const int64_t* __restrict__ q_ptr, const uint2* __restrict__ q_elems,
    const float* __restrict__ q_norm2, int64_t nq, float* __restrict__ D, int64_t ldd) {
  extern __shared__ __align__(16) unsigned char sp_smem[];
  uint2* qs = reinterpret_cast<uint2*>(sp_smem);                 // [kSpQCap] the tile's query elements
  float* res = reinterpret_cast<float*>(qs + kSpQCap);           // [kSpWarps][32 rows][33]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t q0 = static_cast<int64_t>(blockIdx.x) * kSpQ;
  const int nt = static_cast<int>(min(static_cast<int64_t>(kSpQ), nq - q0));
  const int64_t t0 = q_ptr[q0], t1 = q_ptr[q0 + nt];
  const bool staged = t1 - t0 <= kSpQCap;
  if (staged)
    for (int64_t i = threadIdx.x; i < t1 - t0; i += blockDim.x) qs[i] = q_elems[t0 + i];
  __syncthreads();
  const uint2* qv = staged ? qs : q_elems + t0;  // generic pointer: shared or global
  const bool active = lane < nt;
  int64_t qb = 0, qe = 0;
  float qn = 0.f;
  if (active) {
    qb = q_ptr[q0 + lane] - t0;
    qe = q_ptr[q0 + lane + 1] - t0;
    if (METRIC == EPS_METRIC_COSINE) qn = q_norm2[q0 + lane];
  }
  float* my = res + warp * 32 * 33;
  const int64_t ngroups = (n + 31) >> 5;
  for (int64_t g = static_cast<int64_t>(blockIdx.y) * kSpWarps + warp; g < ngroups;
       g += static_cast<int64_t>(gridDim.y) * kSpWarps) {
    const int64_t base = g << 5;
    const int rows_here = static_cast<int>(min(static_cast<int64_t>(32), n - base));
    int64_t my_p0 = 0, my_p1 = 0;
    float my_rn = 0.f;
    if (lane < rows_here) {
      const int64_t r = row_start + base + lane;
      my_p0 = row_ptr[r];
      my_p1 = row_ptr[r + 1];
      if (METRIC == EPS_METRIC_COSINE) my_rn = row_norm2[r];
    }
    for (int j = 0; j < rows_here; ++j) {
      const int64_t p0 = __shfl_sync(kFull, my_p0, j), p1 = __shfl_sync(kFull, my_p1, j);
      SparseMerge<METRIC> mg(qv, qb, qe);
      for (int64_t c = p0; c < p1; c += 32) {
        uint2 e = make_uint2(0u, 0u);
        if (c + lane < p1) e = __ldg(elems + c + lane);
        const int m = static_cast<int>(min(static_cast<int64_t>(32), p1 - c));
        for (int t = 0; t < m; ++t) {
          const uint32_t idx = __shfl_sync(kFull, e.x, t);
          const float val = __uint_as_float(__shfl_sync(kFull, e.y, t));
          if (active) mg.add(idx, val);
        }
      }
      const float acc = mg.sum();
      float rn = 0.f;
      if (METRIC == EPS_METRIC_COSINE) rn = __shfl_sync(kFull, my_rn, j);
      my[j * 33 + lane] = sparse_finish<METRIC>(acc, rn, qn);
    }
    __syncwarp();
    if (lane < rows_here)
      for (int q = 0; q < nt; ++q) D[(q0 + q) * ldd + base + lane] = my[lane * 33 + q];
    __syncwarp();
  }
}

int SparseDist::launch(Index* ix, int metric, int64_t row_start, int64_t n, float* D, int64_t ldd, uint64_t* launches) const {
  if (n <= 0 || nq <= 0) return EPS_OK;
  const int64_t tiles = (nq + kSpQ - 1) / kSpQ;
  if (tiles > 0x7fffffffll) return fail(EPS_ERR_UNSUPPORTED, "sparse scan: too many queries in one launch");
  const int64_t groups = (n + 31) / 32;
  // about 4 CTAs per SM in all; each row slice is shared by the query tiles that run beside it
  const int64_t want = std::max<int64_t>(1, (4ll * ix->num_sms + tiles - 1) / tiles);
  const unsigned slices = static_cast<unsigned>(std::min<int64_t>(std::min<int64_t>(want, (groups + kSpWarps - 1) / kSpWarps), 65535));
  dim3 grid(static_cast<unsigned>(tiles), slices);
  const auto kernel = metric == EPS_METRIC_L2 ? sparse_dist_kernel<EPS_METRIC_L2>
                      : metric == EPS_METRIC_IP ? sparse_dist_kernel<EPS_METRIC_IP>
                                                : sparse_dist_kernel<EPS_METRIC_COSINE>;
  EPS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSpSmem)));
  kernel<<<grid, kSpWarps * 32, kSpSmem, ix->stream>>>(ix->d_sp_ptr, ix->d_sp_elems, ix->d_sp_norm2, row_start, n, q.ptr,
                                                       q.elems, q.norm2, nq, D, ldd);
  EPS_CUDA(cudaGetLastError());
  ++*launches;
  return EPS_OK;
}

int pack_sparse(int64_t n, const int64_t* offsets, const int64_t* indices, const float* values, int64_t max_index,
                int64_t ptr_base, std::vector<int64_t>* ptr, std::vector<uint2>* elems, std::vector<float>* norm2) {
  if (n < 0) return fail(EPS_ERR_INVALID_ARGUMENT, "negative row count");
  if (n > 0 && !offsets) return fail(EPS_ERR_INVALID_ARGUMENT, "null offsets");
  const int64_t e0 = n > 0 ? offsets[0] : 0, e1 = n > 0 ? offsets[n] : 0;
  if (e0 < 0 || e1 < e0) return fail(EPS_ERR_INVALID_ARGUMENT, "offsets must be non-negative and non-decreasing");
  if (e1 > e0 && (!indices || !values)) return fail(EPS_ERR_INVALID_ARGUMENT, "null indices / values");
  ptr->resize(static_cast<size_t>(n) + 1);
  elems->resize(static_cast<size_t>(e1 - e0));
  norm2->resize(static_cast<size_t>(n));
  (*ptr)[0] = ptr_base;
  for (int64_t r = 0; r < n; ++r) {
    const int64_t a = offsets[r], b = offsets[r + 1];
    if (b < a || b > e1) return fail(EPS_ERR_INVALID_ARGUMENT, "offsets must be non-decreasing");
    float s = 0.f;
    for (int64_t i = a; i < b; ++i) {
      const int64_t idx = indices[i];
      if (idx < 0) return fail(EPS_ERR_INVALID_ARGUMENT, "row " + std::to_string(r) + " has a negative index");
      if (idx >= max_index)
        return fail(EPS_ERR_INVALID_ARGUMENT, "row " + std::to_string(r) + " has an index >= the field's dimension");
      if (i > a && idx <= indices[i - 1])
        return fail(EPS_ERR_INVALID_ARGUMENT, "row " + std::to_string(r) + ": indices are not strictly increasing");
      const float v = values[i];
      // sequential fp32 sum of squares like the reference's cosine (vector.cpp:30-32); the host build is SSE2
      // without FMA contraction
      const float sq = v * v;
      s = s + sq;
      uint32_t bits;
      std::memcpy(&bits, &v, 4);
      (*elems)[static_cast<size_t>(i - e0)] = make_uint2(static_cast<uint32_t>(idx), bits);
    }
    (*norm2)[static_cast<size_t>(r)] = s;
    (*ptr)[static_cast<size_t>(r) + 1] = ptr_base + (b - e0);
  }
  return EPS_OK;
}

int upload_sparse_queries(Index* ix, const std::vector<int64_t>& ptr, const std::vector<uint2>& elems,
                          const std::vector<float>& norm2, DevBuf* buf, SparseQueries* q) {
  // one device block [ptr | norm2 | elems], the norms padded to 8 bytes
  const size_t nq = norm2.size(), ptr_bytes = ptr.size() * 8, nrm_off = ptr_bytes,
               el_off = nrm_off + ((nq * 4 + 7) & ~static_cast<size_t>(7));
  EPS_TRY(buf->reserve(el_off + elems.size() * 8));
  unsigned char* d = buf->as<unsigned char>();
  EPS_CUDA(cudaMemcpyAsync(d, ptr.data(), ptr_bytes, cudaMemcpyHostToDevice, ix->stream));
  EPS_CUDA(cudaMemcpyAsync(d + nrm_off, norm2.data(), nq * 4, cudaMemcpyHostToDevice, ix->stream));
  if (!elems.empty()) EPS_CUDA(cudaMemcpyAsync(d + el_off, elems.data(), elems.size() * 8, cudaMemcpyHostToDevice, ix->stream));
  *q = SparseQueries{reinterpret_cast<const int64_t*>(d), reinterpret_cast<const uint2*>(d + el_off),
                     reinterpret_cast<const float*>(d + nrm_off)};
  return EPS_OK;
}

int sparse_append(Index* ix, int64_t first_row, int64_t n_rows, const int64_t* offsets, const int64_t* indices,
                  const float* values) {
  if (first_row != ix->n_rows) return fail(EPS_ERR_INVALID_ARGUMENT, "rows must be appended after the mirrored ones (first_row != rows)");
  if (n_rows < 0) return fail(EPS_ERR_INVALID_ARGUMENT, "negative row count");
  if (n_rows == 0) return EPS_OK;
  if (ix->n_rows + n_rows >= (1ll << 31)) return fail(EPS_ERR_UNSUPPORTED, "row count must stay below 2^31: keys carry 31-bit ids");
  std::vector<int64_t> ptr;
  std::vector<uint2> el;
  std::vector<float> nrm;
  EPS_TRY(pack_sparse(n_rows, offsets, indices, values, ix->dim, ix->sp_nnz, &ptr, &el, &nrm));
  const int64_t rows = ix->n_rows + n_rows, nnz = ix->sp_nnz + static_cast<int64_t>(el.size());
  if (rows > ix->d_sp_norm2.count()) {
    const int64_t cap = std::max<int64_t>(rows, 2 * ix->d_sp_norm2.count());
    EPS_TRY(ix->d_sp_ptr.grow(static_cast<size_t>(cap + 1) * 8, static_cast<size_t>(ix->n_rows + 1) * 8, ix->stream));
    EPS_TRY(ix->d_sp_norm2.grow(static_cast<size_t>(cap) * 4, static_cast<size_t>(ix->n_rows) * 4, ix->stream));
    ix->capacity = std::max(ix->capacity, cap);
  }
  if (nnz > ix->d_sp_elems.count()) {
    const int64_t cap = std::max<int64_t>(nnz, 2 * ix->d_sp_elems.count());
    EPS_TRY(ix->d_sp_elems.grow(static_cast<size_t>(cap) * 8, static_cast<size_t>(ix->sp_nnz) * 8, ix->stream));
  }
  // ptr[0] (= the current nnz) is already on the device
  EPS_CUDA(cudaMemcpyAsync(ix->d_sp_ptr + ix->n_rows + 1, ptr.data() + 1, static_cast<size_t>(n_rows) * 8, cudaMemcpyHostToDevice, ix->stream));
  EPS_CUDA(cudaMemcpyAsync(ix->d_sp_norm2 + ix->n_rows, nrm.data(), static_cast<size_t>(n_rows) * 4, cudaMemcpyHostToDevice, ix->stream));
  if (!el.empty())
    EPS_CUDA(cudaMemcpyAsync(ix->d_sp_elems + ix->sp_nnz, el.data(), el.size() * 8, cudaMemcpyHostToDevice, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  ix->n_rows = rows;
  ix->sp_nnz = nnz;
  return EPS_OK;
}

// Graph build of a sparse column.  The graph exists so that SaveANNGraph writes a usable ann_graph_<field>.bin: its
// lists are the exact k-NN lists (field metric, self excluded, k = out_degree), the navigation point is the exact L2
// nearest row to the reference's sparse "centre" (nsg.cpp:120-135: the LAST value seen per index over the rows,
// divided by n — not a mean), and the integer steps of the dense build's connectivity repair (build.cu) make every
// row reachable from it.
int build_graph_sparse(Index* ix, int64_t n, const eps_build_params* params) {
  if (n < 2 || n > ix->n_rows) return fail(EPS_ERR_INVALID_ARGUMENT, "build: n out of range");
  const int out_degree = params && params->out_degree > 0 ? params->out_degree : 50;
  const int K = static_cast<int>(std::min<int64_t>(std::min(out_degree, 8192), n - 1));
  const int seed = params ? params->seed : 0;
  eps_stats st;
  std::memset(&st, 0, sizeof(st));
  std::vector<int64_t> ptr(static_cast<size_t>(n) + 1);  // the rows' element offsets (ptr[0] = 0)
  if (cudaMemcpy(ptr.data(), ix->d_sp_ptr, ptr.size() * 8, cudaMemcpyDeviceToHost) != cudaSuccess)
    return fail(EPS_ERR_CUDA, "build: row offsets download failed");
  // ---- kNN lists: the rows as queries of the exact scan; with posting lists, the covered rows' distances are read
  // from them (IP / cosine: bitwise the scan's tile) or screened and re-scored (L2: the same K best), so the lists do
  // not change ----
  const bool postings = ix->inv_rows > 0, l2 = ix->metric == EPS_METRIC_L2;
  std::vector<unsigned long long> h_knn(static_cast<size_t>(n) * K);
  {
    DevBuf knn;
    EPS_TRY(knn.reserve(static_cast<size_t>(n) * K * 8));
    const int64_t qc = 8192;  // queries per scan; with postings, also the rows one plan covers (16 B per element)
    for (int64_t q0 = 0; q0 < n; q0 += qc) {
      const int64_t nq = std::min(qc, n - q0);
      const SparseDist dist(SparseQueries{ix->d_sp_ptr + q0, ix->d_sp_elems, ix->d_sp_norm2 + q0}, nq);
      const InvertedDist inv(dist, ptr[q0 + nq] - ptr[q0], ptr[q0]);
      const SparseL2Screen screen(inv);
      ScanRequest r;
      r.dist = postings && !l2 ? static_cast<const DistProducer*>(&inv) : &dist;
      if (postings && l2) r.l2_screen = &screen;
      r.nq = nq; r.row_end = n; r.k = K; r.metric = ix->metric;
      r.skip_deleted = false; r.self_base = q0;
      EPS_TRY(exact_topk(ix, r, knn.as<unsigned long long>() + q0 * K, &st));
    }
    if (cudaMemcpyAsync(h_knn.data(), knn.p, h_knn.size() * 8, cudaMemcpyDeviceToHost, ix->stream) != cudaSuccess)
      return fail(EPS_ERR_CUDA, "build: kNN download failed");
    if (cudaStreamSynchronize(ix->stream) != cudaSuccess) return fail(EPS_ERR_CUDA, "build: kNN scan failed");
  }
  // ---- navigation point ----
  int64_t nav = 0;
  {
    std::vector<uint2> el(static_cast<size_t>(ptr[n]));
    if (!el.empty()) {
      const cudaError_t e = cudaMemcpy(el.data(), ix->d_sp_elems, el.size() * 8, cudaMemcpyDeviceToHost);
      if (e != cudaSuccess) return fail(EPS_ERR_CUDA, cudaGetErrorString(e));
    }
    std::unordered_map<uint32_t, float> last;
    for (const uint2& x : el) {
      float v;
      std::memcpy(&v, &x.y, 4);
      last[x.x] = v;  // tempCenterVec[index] = value: the last row wins
    }
    std::vector<uint32_t> idx;
    idx.reserve(last.size());
    for (const auto& kv : last) idx.push_back(kv.first);
    std::sort(idx.begin(), idx.end());  // std::map order
    std::vector<int64_t> c_off = {0, static_cast<int64_t>(idx.size())}, c_idx(idx.size());
    std::vector<float> c_val(idx.size());
    const float fn = static_cast<float>(n);
    for (size_t i = 0; i < idx.size(); ++i) { c_idx[i] = idx[i]; c_val[i] = last[idx[i]] / fn; }
    std::vector<int64_t> qp;
    std::vector<uint2> qe;
    std::vector<float> qn;
    DevBuf dq, top;
    SparseQueries centre;
    // the centre's indices are stored rows' indices, all below dim < 2^32 - 1
    EPS_TRY(pack_sparse(1, c_off.data(), c_idx.data(), c_val.data(), 0xffffffffll, 0, &qp, &qe, &qn));
    EPS_TRY(upload_sparse_queries(ix, qp, qe, qn, &dq, &centre));
    EPS_TRY(top.reserve(8));
    const SparseDist dist(centre, 1);
    ScanRequest r;
    r.dist = &dist; r.nq = 1; r.row_end = n; r.k = 1;
    r.skip_deleted = false; r.metric = EPS_METRIC_L2;  // the NSG stage always uses L2 (ann_graph_segment.cpp:216-218)
    EPS_TRY(exact_topk(ix, r, top.as<unsigned long long>(), &st));
    unsigned long long key = kKeyInf;
    if (cudaMemcpyAsync(&key, top.p, 8, cudaMemcpyDeviceToHost, ix->stream) != cudaSuccess ||
        cudaStreamSynchronize(ix->stream) != cudaSuccess)
      return fail(EPS_ERR_CUDA, "build: navigation point scan failed");
    nav = key_id(key);
  }

  // ---- lists, connectivity repair (steps 1, 2 and 4 of build.cu: no graph search on sparse rows) and CSR ----
  std::vector<int32_t> ids(static_cast<size_t>(n) * K), cnt(static_cast<size_t>(n));
  for (int64_t v = 0; v < n; ++v) {
    int c = 0;
    for (int j = 0; j < K; ++j) {
      const unsigned long long key = h_knn[static_cast<size_t>(v) * K + j];
      if ((key & kKeyMask) == kKeyInf) break;
      ids[static_cast<size_t>(v) * K + c++] = static_cast<int32_t>(key_id(key));
    }
    cnt[v] = c;
  }
  ConnRepair rep(n, ids.data(), cnt.data(), K);
  rep.flood(static_cast<int32_t>(nav));
  rep.attach_from_knn(h_knn.data(), K);
  uint64_t rng = 0x9E3779B97F4A7C15ull ^ static_cast<uint64_t>(seed);
  for (int64_t u = 0; u < n && rep.linked < n; ++u)
    if (!rep.seen[u]) rep.attach_random(static_cast<int32_t>(u), &rng);
  std::vector<int64_t> off;
  std::vector<int32_t> nb;
  rep.flatten(nav, &off, &nb);
  return install_csr(ix, n, off.data(), nb.data(), off[n], nav);
}

}  // namespace eps
