// K4 — graph build on device.  SURVEY.md §8a rows B1-B3.
//
// Reference pipeline (ANNGraphSegment::BuildFromVectorTable, engine/db/ann_graph_segment.cpp:201-242):
//   B1  kNN graph by NN-descent with the field metric (db/index/knn/nndescent.hpp, K = 100);
//   B2  NSG refinement, always with L2 (ann_graph_segment.cpp:216-218, SURVEY.md Q5):
//         navigation point = vertex nearest the centroid (nsg.cpp:101-155),
//         per vertex: candidate pool sorted by distance, MRNG-style selection — keep p unless a kept r
//         has d(r,p) < d(v,p) — at most out_degree edges (SyncPrune :540-580, SelectEdge :655-685),
//         reverse-edge insertion with re-selection on overflow (InterInsert :583-653),
//         connectivity repair from the navigation point (CheckConnectivity :687-775);
//   B3  flatten to the int64 CSR.
// The reference build is not reproducible (rand(), racy OpenMP), so parity for the build is graph QUALITY
// (recall / distance evaluations of searches on it), not edge identity (SURVEY.md §8c).  This build is reproducible:
// seeded choices, fixed-order sums, order-independent reverse lists (tile.cuh rev_push) and list updates.
//
// Device mapping:
//   * kNN lists: exact all-pairs tiles (brute_force.cu) when n <= exact_knn_below, NN-descent local joins
//     as batched gathered tiles otherwise (nn_descent.cu);
//   * selection: the pairwise distances among a vertex's <=127 candidates are one 128x128xd gathered
//     distance tile per vertex (pair_tile_kernel, fp32, direct (x-y)^2 form); the sequential MRNG scan then
//     runs one warp per vertex over that matrix (select_edges_kernel);
//   * reverse edges: atomic append into per-vertex slots, then the same tile + selection on the union;
//   * connectivity repair + CSR flatten: integer graph work, on the host over the copied-back lists.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <queue>

#include "internal.h"
#include "tile.cuh"

namespace eps {

int nn_descent(Index* ix, int64_t n, int K, const eps_build_params& bp, unsigned long long* d_knn, eps_stats* st);

// One warp per vertex.  cand[z][0] = the vertex, cand[z][1..] = its candidates (unsorted, -1 empty).
// Sorts candidates by (d(v,p), id), then SelectEdge: keep p unless some kept r has d(r,p) < d(v,p).
// keep_all: skip the selection when the candidate count already fits (InterInsert's append branch).
__global__ void select_edges_kernel(const int32_t* __restrict__ cand, const float* __restrict__ D, int batch,
                                    int out_degree, int pool_cap, int keep_all_if_fits, int min_degree, float alpha,
                                    int64_t v_base,
                                    int32_t* __restrict__ out_ids, float* __restrict__ out_dist,
                                    int32_t* __restrict__ out_cnt, int out_stride) {
  const int warp_in_block = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t z = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + warp_in_block;
  extern __shared__ __align__(16) unsigned char se_smem[];
  // per warp: order[kC] (slot indices sorted), kept[out_degree]
  int* order = reinterpret_cast<int*>(se_smem) + warp_in_block * (kC + 64);
  int* kept = order + kC;
  if (z >= batch) return;
  const int32_t* c = cand + z * kC;
  const float* M = D + z * kC * kC;
  // rank candidates 1..kC-1 by (distance to v, id); empty slots last
  int n_valid = 0;
  for (int s = 1 + lane; s < kC; s += 32) n_valid += (c[s] >= 0);
  n_valid = static_cast<int>(warp_sum(static_cast<float>(n_valid)));
  for (int s = 1 + lane; s < kC; s += 32) {
    const int id = c[s];
    if (id < 0) continue;
    const float d = M[s];  // row 0 = distances from v
    int r = 0;
    for (int t = 1; t < kC; ++t) {
      const int id2 = c[t];
      if (id2 < 0 || t == s) continue;
      const float d2 = M[t];
      r += (d2 < d) || (d2 == d && (id2 < id || (id2 == id && t < s)));  // total order: ranks are a permutation
    }
    order[r] = s;
  }
  __syncwarp();
  int64_t v = v_base + z;
  int32_t* oi = out_ids + v * out_stride;
  float* od = out_dist + v * out_stride;
  int nk = 0;
  if (keep_all_if_fits && n_valid <= out_degree) {
    for (int i = lane; i < n_valid; i += 32) { const int s = order[i]; oi[i] = c[s]; od[i] = M[s]; }
    nk = n_valid;
  } else {
    const int scan = min(n_valid, pool_cap);
    for (int i = 0; i < scan && nk < out_degree; ++i) {
      const int s = order[i];
      const float dvp = M[s];
      bool viol = false;
      for (int t = lane; t < nk; t += 32) viol |= (alpha * M[kept[t] * kC + s] < dvp);
      if (!__any_sync(kFull, viol)) {
        if (lane == 0) { kept[nk] = s; oi[nk] = c[s]; od[nk] = dvp; }
        ++nk;
        __syncwarp();
      }
    }
    // Degree floor: the reference's pool (every vertex its build-time search evaluated, up to 300 scanned)
    // is far more spread out than a kNN list, which the occlusion rule thins to a handful of edges on
    // concentrated data; top the list up with the nearest rejected candidates (DESIGN.md, build).
    if (nk < min_degree) {
      for (int i = 0; i < scan && nk < min_degree && nk < out_degree; ++i) {
        const int s = order[i];
        bool have = false;
        for (int t = lane; t < nk; t += 32) have |= (kept[t] == s);
        if (!__any_sync(kFull, have)) {
          if (lane == 0) { kept[nk] = s; oi[nk] = c[s]; od[nk] = M[s]; }
          ++nk;
          __syncwarp();
        }
      }
    }
  }
  if (lane == 0) out_cnt[v] = nk;
}

// cand row for pass 1: [v, knn ids...]
__global__ void fill_cand_from_knn_kernel(const unsigned long long* __restrict__ knn, int K, int64_t v0, int batch,
                                          int32_t* __restrict__ cand) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(batch) * kC) return;
  const int64_t z = i / kC;
  const int s = static_cast<int>(i % kC);
  int32_t id = -1;
  if (s == 0) id = static_cast<int32_t>(v0 + z);
  else if (s - 1 < K) {
    const unsigned long long key = knn[(v0 + z) * K + (s - 1)];
    if ((key & kKeyMask) != kKeyInf) id = static_cast<int32_t>(key_id(key));
  }
  cand[i] = id;
}

// reverse candidates: for edge v -> p push v to rev[p] (rev_cap of them, chosen independently of arrival order)
__global__ void append_reverse_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ cnt, int stride,
                                      int64_t n, int rev_cap, unsigned long long* __restrict__ rev, int32_t* __restrict__ rev_cnt,
                                      uint32_t salt) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t v = i / stride;
  const int j = static_cast<int>(i % stride);
  if (v >= n || j >= cnt[v]) return;
  const int p = ids[v * stride + j];
  rev_push(rev, rev_cap, rev_cnt, p, static_cast<int32_t>(v), salt);
}

// cand row for pass 2: [v, own list..., reverse candidates not already present...]
__global__ void fill_cand_union_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ cnt, int stride,
                                       const unsigned long long* __restrict__ rev, const int32_t* __restrict__ rev_cnt, int rev_cap,
                                       int64_t v0, int batch, int32_t* __restrict__ cand) {
  const int64_t z = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (z >= batch) return;
  const int64_t v = v0 + z;
  int32_t* c = cand + z * kC;
  int m = 0;
  c[m++] = static_cast<int32_t>(v);
  const int own = cnt[v];
  for (int j = 0; j < own && m < kC; ++j) c[m++] = ids[v * stride + j];
  const int nr = min(rev_cnt[v], rev_cap);
  for (int j = 0; j < nr && m < kC; ++j) {
    const int32_t u = rev_id(rev[v * rev_cap + j]);
    bool dup = (u == v);
    for (int t = 1; t <= own && !dup; ++t) dup = (c[t] == u);
    if (!dup) c[m++] = u;
  }
  for (; m < kC; ++m) c[m] = -1;
}

__global__ void column_sum_kernel(const float* __restrict__ vectors, int64_t n, int dim, float* __restrict__ part) {
  // grid.x covers columns, grid.y splits rows into slices; part[slice * dim + col] (fp32 sums like nsg.cpp:110-117)
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= dim) return;
  const int64_t per = (n + gridDim.y - 1) / gridDim.y;
  const int64_t r0 = blockIdx.y * per, r1 = min(n, r0 + per);
  float s = 0.f;
  for (int64_t r = r0; r < r1; ++r) s += vectors[r * dim + col];
  part[static_cast<int64_t>(blockIdx.y) * dim + col] = s;
}
// centroid = the slices' sums added in slice order (a fixed order: the navigation point is reproducible) / n
__global__ void centroid_kernel(const float* __restrict__ part, int slices, int dim, float inv_n, float* __restrict__ out) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= dim) return;
  float s = 0.f;
  for (int y = 0; y < slices; ++y) s += part[static_cast<int64_t>(y) * dim + col];
  out[col] = s * inv_n;
}

static int prune_pass(Index* ix, int64_t n, const unsigned long long* d_knn, int K, bool pass2, int out_degree,
                      int pool_cap, int min_degree, float alpha, int32_t* d_ids, float* d_dist, int32_t* d_cnt, int stride, const unsigned long long* d_rev,
                      const int32_t* d_rev_cnt, int rev_cap, int32_t* d_ids_out, float* d_dist_out, int32_t* d_cnt_out,
                      eps_stats* st) {
  const int64_t batch_max = 4096;
  DevBuf cand, D;
  EPS_TRY(cand.reserve(static_cast<size_t>(batch_max) * kC * 4));
  EPS_TRY(D.reserve(static_cast<size_t>(batch_max) * kC * kC * 4));
  const int warps = 4;
  const size_t smem = static_cast<size_t>(warps) * (kC + 64) * 4;
  for (int64_t v0 = 0; v0 < n; v0 += batch_max) {
    const int batch = static_cast<int>(std::min(batch_max, n - v0));
    if (!pass2) {
      const int64_t tot = static_cast<int64_t>(batch) * kC;
      fill_cand_from_knn_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, ix->stream>>>(d_knn, K, v0, batch,
                                                                                                cand.as<int32_t>());
    } else {
      fill_cand_union_kernel<<<(batch + 127) / 128, 128, 0, ix->stream>>>(d_ids, d_cnt, stride, d_rev, d_rev_cnt, rev_cap,
                                                                          v0, batch, cand.as<int32_t>());
    }
    EPS_TRY(launch_pair_tiles(ix, EPS_METRIC_L2, cand.as<int32_t>(), D.as<float>(), batch));
    if (getenv("EPS_DEBUG_SYNC")) EPS_CUDA(cudaStreamSynchronize(ix->stream));
    select_edges_kernel<<<(batch + warps - 1) / warps, warps * 32, smem, ix->stream>>>(
        cand.as<int32_t>(), D.as<float>(), batch, out_degree, pool_cap, pass2 ? 1 : 0, min_degree, alpha, v0, d_ids_out,
        d_dist_out, d_cnt_out, stride);
    EPS_CUDA(cudaGetLastError());
    if (st) st->kernel_launches += 3;
  }
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  cand.release();
  D.release();
  return EPS_OK;
}

// Install a host CSR (int64 offsets, int32 ids) as the index's graph, dropping everything derived from the old one.
static int install_csr(Index* ix, int64_t n, const int64_t* off, const int32_t* nb, int64_t e, int64_t nav) {
  if (ix->d_offsets) { cudaFree(ix->d_offsets); ix->d_offsets = nullptr; }
  if (ix->d_nbrs) { cudaFree(ix->d_nbrs); ix->d_nbrs = nullptr; }
  if (ix->d_init_ids) { cudaFree(ix->d_init_ids); ix->d_init_ids = nullptr; }
  if (ix->d_ell) { cudaFree(ix->d_ell); ix->d_ell = nullptr; }
  ix->seed_rows_L = 0;
  ix->init_L = 0;
  ix->n_indexed = 0;
  EPS_CUDA(cudaMalloc(&ix->d_offsets, (static_cast<size_t>(n) + 1) * 8));
  EPS_CUDA(cudaMalloc(&ix->d_nbrs, std::max<size_t>(static_cast<size_t>(e), 1) * 4));
  EPS_CUDA(cudaMemcpyAsync(ix->d_offsets, off, (static_cast<size_t>(n) + 1) * 8, cudaMemcpyHostToDevice, ix->stream));
  if (e > 0) EPS_CUDA(cudaMemcpyAsync(ix->d_nbrs, nb, static_cast<size_t>(e) * 4, cudaMemcpyHostToDevice, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  ix->n_indexed = n;
  ix->n_edges = e;
  ix->nav = nav;
  return EPS_OK;
}

int build_graph(Index* ix, int64_t n, const eps_build_params* params) {
  eps_build_params bp;
  std::memset(&bp, 0, sizeof(bp));
  if (params) bp = *params;
  if (bp.knn_k <= 0) bp.knn_k = 100;          // Default_NSG_Config.knng
  if (bp.out_degree <= 0) bp.out_degree = 50;  // .out_degree
  if (bp.candidate_pool <= 0) bp.candidate_pool = 300;
  if (bp.search_length <= 0) bp.search_length = 45;
  if (bp.nnd_iters <= 0) bp.nnd_iters = 30;
  if (bp.nnd_sample <= 0) bp.nnd_sample = 32;
  if (bp.nnd_delta <= 0.f) bp.nnd_delta = 0.001f;
  if (bp.exact_knn_below <= 0) bp.exact_knn_below = 60000;
  if (n < 2 || n > ix->n_rows) return fail(EPS_ERR_INVALID_ARGUMENT, "build: n out of range");
  if (n >= (1ll << 31)) return fail(EPS_ERR_UNSUPPORTED, "build: more than 2^31 rows per shard");
  const int R = std::min<int>(bp.out_degree, 64);
  const int min_deg = std::min<int>(bp.min_degree > 0 ? bp.min_degree : 32, R);
  const float alpha = bp.alpha > 0.f ? bp.alpha : 1.0f;
  const int K = static_cast<int>(std::min<int64_t>(std::min<int>(bp.knn_k, kC - 1), n - 1));
  eps_stats st;
  std::memset(&st, 0, sizeof(st));

  // ---- B1: kNN lists (field metric) -------------------------------------------------------
  DevBuf knn;
  EPS_TRY(knn.reserve(static_cast<size_t>(n) * K * 8));
  if (n <= bp.exact_knn_below) {
    const int64_t qc = 8192;
    for (int64_t q0 = 0; q0 < n; q0 += qc) {
      const int64_t nq = std::min(qc, n - q0);
      EPS_TRY(brute_force_knn_rows(ix, q0, nq, n, K, knn.as<unsigned long long>() + q0 * K, &st));
    }
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
  } else {
    EPS_TRY(nn_descent(ix, n, K, bp, knn.as<unsigned long long>(), &st));
  }

  // ---- B2a: navigation point = exact nearest row to the centroid (L2) ----------------------
  int64_t nav = 0;
  {
    DevBuf cen, part, top;
    const unsigned slices = static_cast<unsigned>(std::min<int64_t>(1024, (n + 255) / 256));
    EPS_TRY(cen.reserve(static_cast<size_t>(ix->dim) * 4));
    EPS_TRY(part.reserve(static_cast<size_t>(ix->dim) * slices * 4));
    EPS_TRY(top.reserve(8));
    dim3 g(static_cast<unsigned>((ix->dim + 127) / 128), slices);
    column_sum_kernel<<<g, 128, 0, ix->stream>>>(ix->d_vectors, n, static_cast<int>(ix->dim), part.as<float>());
    centroid_kernel<<<static_cast<unsigned>((ix->dim + 127) / 128), 128, 0, ix->stream>>>(
        part.as<float>(), static_cast<int>(slices), static_cast<int>(ix->dim), 1.0f / static_cast<float>(n), cen.as<float>());
    const int saved_metric = ix->metric;
    const bool saved_del = ix->any_deleted;
    ix->metric = EPS_METRIC_L2;
    ix->any_deleted = false;
    int rc = brute_force_topk(ix, cen.as<float>(), 1, 0, n, 1, nullptr, nullptr, false, top.as<unsigned long long>(), &st);
    ix->metric = saved_metric;
    ix->any_deleted = saved_del;
    EPS_TRY(rc);
    unsigned long long key;
    EPS_CUDA(cudaMemcpyAsync(&key, top.p, 8, cudaMemcpyDeviceToHost, ix->stream));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
    nav = key_id(key);
    cen.release();
    part.release();
    top.release();
  }

  // ---- B2b: selection pass 1 (SyncPrune / SelectEdge) --------------------------------------
  const int stride = 64;  // >= R
  DevBuf ids1, dist1, cnt1, ids2, dist2, cnt2, rev, rev_cnt;
  EPS_TRY(ids1.reserve(static_cast<size_t>(n) * stride * 4));
  EPS_TRY(dist1.reserve(static_cast<size_t>(n) * stride * 4));
  EPS_TRY(cnt1.reserve(static_cast<size_t>(n) * 4));
  EPS_TRY(prune_pass(ix, n, knn.as<unsigned long long>(), K, false, R, bp.candidate_pool, min_deg, alpha, nullptr, nullptr, nullptr, stride,
                     nullptr, nullptr, 0, ids1.as<int32_t>(), dist1.as<float>(), cnt1.as<int32_t>(), &st));

  // ---- B2c: reverse edges (InterInsert) ----------------------------------------------------
  const int rev_cap = kC - 1 - R;  // union always fits the candidate slots
  EPS_TRY(rev.reserve(static_cast<size_t>(n) * rev_cap * 8));
  EPS_TRY(rev_cnt.reserve(static_cast<size_t>(n) * 4));
  EPS_CUDA(cudaMemsetAsync(rev.p, 0xFF, static_cast<size_t>(n) * rev_cap * 8, ix->stream));
  EPS_CUDA(cudaMemsetAsync(rev_cnt.p, 0, static_cast<size_t>(n) * 4, ix->stream));
  {
    const int64_t tot = n * stride;
    append_reverse_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, ix->stream>>>(
        ids1.as<int32_t>(), cnt1.as<int32_t>(), stride, n, rev_cap, rev.as<unsigned long long>(), rev_cnt.as<int32_t>(),
        0x68E31DA4u + static_cast<uint32_t>(bp.seed));
    EPS_CUDA(cudaGetLastError());
  }
  EPS_TRY(ids2.reserve(static_cast<size_t>(n) * stride * 4));
  EPS_TRY(dist2.reserve(static_cast<size_t>(n) * stride * 4));
  EPS_TRY(cnt2.reserve(static_cast<size_t>(n) * 4));
  EPS_TRY(prune_pass(ix, n, nullptr, 0, true, R, kC, min_deg, alpha, ids1.as<int32_t>(), dist1.as<float>(), cnt1.as<int32_t>(), stride,
                     rev.as<unsigned long long>(), rev_cnt.as<int32_t>(), rev_cap, ids2.as<int32_t>(), dist2.as<float>(),
                     cnt2.as<int32_t>(), &st));

  // ---- B2d + B3: connectivity repair and CSR flatten (host, integer work) -------------------
  std::vector<int32_t> h_ids(static_cast<size_t>(n) * stride), h_cnt(static_cast<size_t>(n));
  EPS_CUDA(cudaMemcpyAsync(h_ids.data(), ids2.p, h_ids.size() * 4, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaMemcpyAsync(h_cnt.data(), cnt2.p, h_cnt.size() * 4, cudaMemcpyDeviceToHost, ix->stream));
  std::vector<unsigned long long> h_knn(static_cast<size_t>(n) * K);
  EPS_CUDA(cudaMemcpyAsync(h_knn.data(), knn.p, h_knn.size() * 8, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  ids1.release(); dist1.release(); cnt1.release(); ids2.release(); dist2.release(); cnt2.release();
  rev.release(); rev_cnt.release(); knn.release();

  // CheckConnectivity (nsg.cpp:687-775): flood from the navigation point; for the first unlinked vertex u, attach u
  // to the NEAREST ALREADY-LINKED vertex of a candidate pool, else to a RANDOM linked vertex; flood from u; repeat.
  // The reference's pool is what a graph search for u's own vector evaluated; its selection pools come from searches
  // that START at the navigation point, which is what makes its graph navigable from there.  Ours are kNN lists, so
  // on clustered data whole clusters are separate components; the repair has to give each of them an entry the search
  // can find.  In this order:
  //   1. u's own kNN list (exact near neighbours, already on hand): the nearest linked entry that has received fewer
  //      than kRepairCap repair edges so far (on inner-product tables the kNN lists of most vertices point at the same
  //      few large-norm rows; without the cap one of them collects O(n) repair edges);
  //   2. NO kNN entry of u is linked: u's neighbourhood is a component of its own and u becomes its ENTRY, an
  //      out-neighbour of the navigation point, i.e. part of every search's seed set (PrepareInitIds starts from the
  //      navigation point's out-neighbours) as long as the queue length covers the navigation point's degree.
  //      (A routing layer — 256 hub entries off the navigation point, every other entry off its nearest hub — was
  //      tried and dropped: with well-separated clusters in 768-d all hubs are about equally far from a query, best-
  //      first search cannot tell which hub leads to the query's component, recall fell from 0.99 to 0.89 at L = 2048.)
  //   3. the reference's own pool: the un-repaired graph is installed and the rows of the still unlinked vertices go
  //      through graph_search on the device (L2 like the rest of the refinement, beam = max(64, search_length));
  //   4. a random linked vertex (:767-774).
  // The attach / flood bookkeeping — integer work — runs on the host in the reference's order.
  constexpr size_t kRepairCap = 16;
  std::vector<int32_t> entries;  // one per component that the kNN lists do not connect to the rest
  std::vector<std::vector<int32_t>> extra(static_cast<size_t>(n));  // edges added by the repair
  {
    std::vector<uint8_t> seen(static_cast<size_t>(n), 0);
    std::vector<int32_t> stack;
    int64_t linked = 0;
    auto flood = [&](int32_t root) {
      if (seen[root]) return;
      seen[root] = 1; ++linked;
      stack.push_back(root);
      while (!stack.empty()) {
        const int32_t u = stack.back();
        stack.pop_back();
        const int32_t* row = &h_ids[static_cast<size_t>(u) * stride];
        for (int j = 0; j < h_cnt[u]; ++j) {
          const int32_t w = row[j];
          if (!seen[w]) { seen[w] = 1; ++linked; stack.push_back(w); }
        }
        for (int32_t w : extra[u]) if (!seen[w]) { seen[w] = 1; ++linked; stack.push_back(w); }
      }
    };
    flood(static_cast<int32_t>(nav));
    for (int64_t u = 0; u < n && linked < n; ++u) {
      if (seen[u]) continue;
      bool any_linked = false, done = false;
      for (int j = 0; j < K && !done; ++j) {  // 1. nearest linked kNN entry with room
        const unsigned long long key = h_knn[static_cast<size_t>(u) * K + j];
        if ((key & kKeyMask) == kKeyInf) break;
        const int32_t w = static_cast<int32_t>(key_id(key));
        if (!seen[w]) continue;
        any_linked = true;
        if (extra[w].size() < kRepairCap) {
          extra[w].push_back(static_cast<int32_t>(u));
          flood(static_cast<int32_t>(u));
          done = true;
        }
      }
      if (!done && !any_linked) {  // 2. a component of its own: u is its entry (wired up below)
        entries.push_back(static_cast<int32_t>(u));
        flood(static_cast<int32_t>(u));
      }
    }
    if (linked < n) {
      std::vector<int32_t> unl;
      for (int64_t v = 0; v < n; ++v) if (!seen[v]) unl.push_back(static_cast<int32_t>(v));
      // install the un-repaired graph for the batched searches
      {
        std::vector<int64_t> off0(static_cast<size_t>(n) + 1);
        int64_t e0 = 0;
        for (int64_t v = 0; v < n; ++v) { off0[v] = e0; e0 += h_cnt[v]; }
        off0[n] = e0;
        std::vector<int32_t> nb0(static_cast<size_t>(std::max<int64_t>(e0, 1)));
        for (int64_t v = 0; v < n; ++v) std::memcpy(&nb0[off0[v]], &h_ids[static_cast<size_t>(v) * stride], static_cast<size_t>(h_cnt[v]) * 4);
        EPS_TRY(install_csr(ix, n, off0.data(), nb0.data(), e0, nav));
      }
      const int64_t Ls = std::min<int64_t>(n, std::max<int>(64, bp.search_length));
      const int64_t chunk = 32768;
      DevBuf d_ids, d_q, d_queue;
      EPS_TRY(d_ids.reserve(static_cast<size_t>(chunk) * 4));
      EPS_TRY(d_q.reserve(static_cast<size_t>(chunk) * ix->dim * 4));
      EPS_TRY(d_queue.reserve(static_cast<size_t>(chunk) * Ls * 8));
      std::vector<unsigned long long> h_pool(static_cast<size_t>(chunk) * Ls);
      const int saved_metric = ix->metric, saved_width = ix->search_width;
      uint64_t rng = 0x9E3779B97F4A7C15ull ^ static_cast<uint64_t>(bp.seed);
      int rc = EPS_OK;
      for (size_t c0 = 0; c0 < unl.size() && rc == EPS_OK; c0 += static_cast<size_t>(chunk)) {
        const int64_t cn = static_cast<int64_t>(std::min<size_t>(static_cast<size_t>(chunk), unl.size() - c0));
        // many of this chunk's vertices may have been linked by earlier attachments: search only the rest
        std::vector<int32_t> todo;
        for (int64_t i = 0; i < cn; ++i) if (!seen[unl[c0 + i]]) todo.push_back(unl[c0 + i]);
        if (todo.empty()) continue;
        const int64_t tn = static_cast<int64_t>(todo.size());
        ix->metric = EPS_METRIC_L2;
        ix->search_width = 4;
        rc = cudaMemcpyAsync(d_ids.p, todo.data(), static_cast<size_t>(tn) * 4, cudaMemcpyHostToDevice, ix->stream) == cudaSuccess ? EPS_OK : fail(EPS_ERR_CUDA, "repair: id upload failed");
        if (rc == EPS_OK) rc = gather_rows(ix, d_ids.as<int32_t>(), tn, d_q.as<float>());
        if (rc == EPS_OK) rc = graph_search(ix, d_q.as<float>(), tn, Ls, d_queue.as<unsigned long long>(), &st);
        ix->metric = saved_metric;
        ix->search_width = saved_width;
        if (rc == EPS_OK && cudaMemcpyAsync(h_pool.data(), d_queue.p, static_cast<size_t>(tn) * Ls * 8, cudaMemcpyDeviceToHost, ix->stream) != cudaSuccess)
          rc = fail(EPS_ERR_CUDA, "repair: pool download failed");
        if (rc == EPS_OK && cudaStreamSynchronize(ix->stream) != cudaSuccess) rc = fail(EPS_ERR_CUDA, "repair: search failed");
        if (rc != EPS_OK) break;
        for (int64_t i = 0; i < tn; ++i) {
          const int32_t u = todo[i];
          if (seen[u]) continue;  // reached through an earlier attachment of this chunk
          int32_t root = -1;
          const unsigned long long* pool = &h_pool[static_cast<size_t>(i) * Ls];
          for (int64_t j = 0; j < Ls; ++j) {  // nearest linked vertex of the search pool (:757-766)
            if ((pool[j] & kKeyMask) == kKeyInf) break;
            const int32_t w = static_cast<int32_t>(key_id(pool[j]));
            if (w != u && seen[w]) { root = w; break; }
          }
          while (root < 0) {  // a random linked vertex (:767-774)
            rng = rng * 6364136223846793005ull + 1442695040888963407ull;
            const int32_t r = static_cast<int32_t>((rng >> 33) % static_cast<uint64_t>(n));
            if (seen[r]) root = r;
          }
          extra[root].push_back(u);  // nsg[root].push_back(id) (:774), may exceed out_degree (Q11)
          flood(u);
        }
      }
      ix->graph_counters_pending = false;
      if (rc != EPS_OK) return rc;
    }
  }
  // ---- entries of the separate components: out-neighbours of the navigation point ----
  for (int32_t u : entries) extra[nav].push_back(u);

  std::vector<int64_t> off(static_cast<size_t>(n) + 1);
  int64_t e = 0;
  for (int64_t v = 0; v < n; ++v) { off[v] = e; e += h_cnt[v] + static_cast<int64_t>(extra[v].size()); }
  off[n] = e;
  std::vector<int32_t> nb(static_cast<size_t>(e));
  for (int64_t v = 0; v < n; ++v) {
    int64_t o = off[v];
    for (int j = 0; j < h_cnt[v]; ++j) nb[o++] = h_ids[static_cast<size_t>(v) * stride + j];
    for (int32_t w : extra[v]) nb[o++] = w;
  }
  EPS_TRY(install_csr(ix, n, off.data(), nb.data(), e, nav));
  return EPS_OK;
}

}  // namespace eps
