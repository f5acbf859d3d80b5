// B4 — extend an installed dense graph with the rows appended after it (eps_index_extend_graph, DESIGN.md §K4 B4).
//
// The new rows [n_indexed, n) are linked in chunks of kExtendChunk rows; chunk [a, b) works on the graph the previous
// chunks left, over rows [0, a):
//   1. pools: a graph_search of each new row over [0, a) (field metric, width 4, L = min(128, a), unscreened) and its
//      exact kNN among the chunk's rows [a, b) (field metric, deleted rows included, as B1), merged by key into the
//      kC - 1 nearest — the scan is what links rows inserted together, e.g. a cluster the old rows do not have;
//   2. forward selection: SelectEdge (L2) over that pool, as the build's pass 1;
//   3. reverse edges: each new edge v -> p offers v to p (rev_push: the kept offers do not depend on arrival order).
//      Every new row and every old row that received an offer is re-selected over its row + offers (InterInsert: the
//      offers are appended while the row fits, otherwise SelectEdge).  Reverse slots are indexed by a compacted list
//      of the rows the chunk edits, not by vertex id.  An old row already wider than out_degree (the navigation point
//      with its component entries, repaired hubs) is left as it is and takes no offers;
//   4. splice, on the device: new offsets = exclusive scan of the new degrees, then one scatter of every row from the
//      old CSR or the chunk's edit table into a second CSR buffer, which becomes the graph; the ELL rows of the
//      edited vertices are rewritten in the same pass, so the next chunk's searches read the grown graph.
// After the last chunk the CSR is copied down once and flooded from the navigation point; vertices it does not reach
// are attached by the build's repair steps 3 and 4 (repair_by_search).  The sketch basis is kept and stored row
// sketches are extended to the new rows.
#include <cub/cub.cuh>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "internal.h"
#include "tile.cuh"

namespace eps {

namespace {

constexpr int64_t kExtendChunk = 65536;  // new rows per chunk
constexpr int kPoolL = 128;              // queue length of the pool searches
constexpr int kPoolWidth = 4;
constexpr int64_t kSelBatch = 4096;      // vertices per selection launch: 4096 x 64 KB distance tiles
constexpr int64_t kKnnQueries = 8192;    // queries per exact-scan call of the chunk kNN

// cand row z: [a + z, the kC - 1 nearest by key of its search pool (rows < a) and its chunk kNN list (rows >= a)]
__global__ void merge_pools_kernel(const unsigned long long* __restrict__ pool, int L,
                                   const unsigned long long* __restrict__ knn, int K, int64_t a, int cn,
                                   int32_t* __restrict__ cand) {
  const int z = blockIdx.x * blockDim.x + threadIdx.x;
  if (z >= cn) return;
  const unsigned long long* p = pool + static_cast<int64_t>(z) * L;
  const unsigned long long* q = knn + static_cast<int64_t>(z) * K;
  int32_t* c = cand + static_cast<int64_t>(z) * kC;
  c[0] = static_cast<int32_t>(a + z);
  int i = 0, j = 0, m = 1;
  while (m < kC) {
    const unsigned long long x = i < L ? (p[i] & kKeyMask) : kKeyInf;
    const unsigned long long y = j < K ? (q[j] & kKeyMask) : kKeyInf;
    if (x == kKeyInf && y == kKeyInf) break;
    if (x <= y) { c[m++] = static_cast<int32_t>(key_id(x)); ++i; }
    else { c[m++] = static_cast<int32_t>(key_id(y)); ++j; }
  }
  for (; m < kC; ++m) c[m] = -1;
}

// New row a + z owns edit slot z.
__global__ void own_new_slots_kernel(int64_t a, int cn, int32_t* __restrict__ slot_of, int32_t* __restrict__ vid) {
  const int z = blockIdx.x * blockDim.x + threadIdx.x;
  if (z >= cn) return;
  slot_of[a + z] = z;
  vid[z] = static_cast<int32_t>(a + z);
}

// An old target p of a new edge whose row fits (degree <= R) gets the next edit slot.  The slot numbers depend on
// the arrival order; nothing computed from a slot does.
__global__ void mark_targets_kernel(const int32_t* __restrict__ fwd_ids, const int32_t* __restrict__ fwd_cnt, int cn,
                                    int64_t a, const int64_t* __restrict__ off, int R, int32_t* __restrict__ slot_of,
                                    int32_t* __restrict__ vid, int32_t* __restrict__ n_slots) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t z = i / kEll;
  const int j = static_cast<int>(i % kEll);
  if (z >= cn || j >= fwd_cnt[z]) return;
  const int32_t p = fwd_ids[z * kEll + j];
  if (p >= a || off[p + 1] - off[p] > R) return;
  if (atomicCAS(&slot_of[p], -1, -2) == -1) {
    const int s = atomicAdd(n_slots, 1);
    vid[s] = p;
    slot_of[p] = s;
  }
}

// New edge a + z -> p offers a + z to the reverse list of p's edit slot (targets without one are skipped).
__global__ void push_reverse_kernel(const int32_t* __restrict__ fwd_ids, const int32_t* __restrict__ fwd_cnt, int cn,
                                    int64_t a, const int32_t* __restrict__ slot_of, int rev_cap,
                                    unsigned long long* __restrict__ rev, int32_t* __restrict__ rev_cnt, uint32_t salt) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t z = i / kEll;
  const int j = static_cast<int>(i % kEll);
  if (z >= cn || j >= fwd_cnt[z]) return;
  const int32_t s = slot_of[fwd_ids[z * kEll + j]];
  if (s >= 0) rev_push(rev, rev_cap, rev_cnt, s, static_cast<int32_t>(a + z), salt);
}

// Own row of each edit slot: a new row's forward selection, an old row's current neighbours (its ELL row: every
// edited old row has degree <= R <= kEll).
__global__ void gather_own_kernel(const int32_t* __restrict__ vid, int64_t T, int cn, const int32_t* __restrict__ fwd_ids,
                                  const int32_t* __restrict__ fwd_cnt, const int32_t* __restrict__ ell,
                                  const int64_t* __restrict__ off, int32_t* __restrict__ own_ids,
                                  int32_t* __restrict__ own_cnt) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t s = i / kEll;
  const int j = static_cast<int>(i % kEll);
  if (s >= T) return;
  int cnt;
  int32_t id = -1;
  if (s < cn) {
    cnt = fwd_cnt[s];
    if (j < cnt) id = fwd_ids[s * kEll + j];
  } else {
    const int64_t v = vid[s];
    cnt = static_cast<int>(off[v + 1] - off[v]);
    if (j < cnt) id = ell[v * kEll + j];
  }
  own_ids[i] = id;
  if (j == 0) own_cnt[s] = cnt;
}

// deg[v] = degree of v in the grown graph for v < b (edited rows: their selection; others: their old row), deg[b] = 0
__global__ void new_degrees_kernel(const int64_t* __restrict__ off, int64_t b, const int32_t* __restrict__ slot_of,
                                   const int32_t* __restrict__ sel_cnt, int64_t* __restrict__ deg) {
  const int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (v > b) return;
  if (v == b) { deg[v] = 0; return; }
  const int32_t s = slot_of[v];
  deg[v] = s >= 0 ? sel_cnt[s] : off[v + 1] - off[v];
}

// One warp per vertex of [0, b): its row of the grown CSR, from the edit table or the old CSR; an edited row is also
// written to its ELL row (-1 padded).
__global__ void splice_kernel(const int64_t* __restrict__ off, const int32_t* __restrict__ nbrs, int64_t b,
                              const int32_t* __restrict__ slot_of, const int32_t* __restrict__ sel_ids,
                              const int64_t* __restrict__ new_off, int32_t* __restrict__ new_nbrs, int32_t* __restrict__ ell) {
  const int64_t v = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (v >= b) return;
  const int32_t s = slot_of[v];
  int32_t* dst = new_nbrs + new_off[v];
  if (s < 0) {
    const int64_t o = off[v], d = off[v + 1] - o;
    for (int64_t j = lane; j < d; j += 32) dst[j] = nbrs[o + j];
    return;
  }
  const int d = static_cast<int>(new_off[v + 1] - new_off[v]);
  const int32_t* src = sel_ids + static_cast<int64_t>(s) * kEll;
  for (int j = lane; j < kEll; j += 32) {
    const int32_t id = j < d ? src[j] : -1;
    if (j < d) dst[j] = id;
    ell[v * kEll + j] = id;
  }
}

__global__ void clear_slots_kernel(const int32_t* __restrict__ vid, int64_t T, int32_t* __restrict__ slot_of) {
  const int64_t s = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (s < T) slot_of[vid[s]] = -1;
}

unsigned blocks(int64_t threads, int per) { return static_cast<unsigned>((threads + per - 1) / per); }

// Host wall time per phase when EPS_EXTEND_PHASES is set (one JSON line on stderr; the stream is synchronised at every
// phase boundary then, so the phases do not overlap).
struct Phases {
  enum { kSearch, kKnn, kSelect, kReverse, kSplice, kRepair, kN };
  bool on = getenv("EPS_EXTEND_PHASES") != nullptr;
  double ms[kN] = {};
  int64_t max_slots = 0;   // most edit slots of one chunk
  int64_t unreached = 0;   // vertices the flood after the last chunk did not reach
  std::chrono::steady_clock::time_point t = std::chrono::steady_clock::now();
  int mark(Index* ix, int phase) {
    if (!on) return EPS_OK;
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
    const auto now = std::chrono::steady_clock::now();
    ms[phase] += std::chrono::duration<double, std::milli>(now - t).count();
    t = now;
    return EPS_OK;
  }
  void print() const {
    if (!on) return;
    fprintf(stderr, "{\"extend_phases_ms\": {\"search\": %.1f, \"chunk_knn\": %.1f, \"select\": %.1f, \"reverse\": %.1f, "
                    "\"splice\": %.1f, \"repair\": %.1f}, \"max_edit_slots\": %lld, \"unreached\": %lld}\n", ms[kSearch], ms[kKnn],
            ms[kSelect], ms[kReverse], ms[kSplice], ms[kRepair], static_cast<long long>(max_slots), static_cast<long long>(unreached));
  }
};

// SelectEdge over cand rows [0, count) (pair tiles + selection in kSelBatch batches); fill(s0, batch) writes the
// batch's cand rows to cand when the rows are not all there already.
template <typename Fill>
int select_rows(Index* ix, int64_t count, int32_t* cand, int64_t cand_step, float* D, int R, int pool_cap, int keep_all,
                int min_deg, float alpha, int32_t* out_ids, float* out_dist, int32_t* out_cnt, Fill fill) {
  const int warps = 4;
  const size_t smem = static_cast<size_t>(warps) * (kC + 64) * 4;
  for (int64_t s0 = 0; s0 < count; s0 += kSelBatch) {
    const int batch = static_cast<int>(std::min(kSelBatch, count - s0));
    int32_t* c = cand + s0 * cand_step;
    fill(s0, batch, c);
    EPS_TRY(launch_pair_tiles(ix, EPS_METRIC_L2, c, D, batch));
    select_edges_kernel<<<blocks(batch, warps), warps * 32, smem, ix->stream>>>(c, D, batch, R, pool_cap, keep_all, min_deg,
                                                                               alpha, s0, out_ids, out_dist, out_cnt, kEll);
    EPS_CUDA(cudaGetLastError());
  }
  return EPS_OK;
}

int extend_chunks(Index* ix, int64_t n, const eps_build_params& bp, Phases* ph) {
  const int64_t n0 = ix->n_indexed, dim = ix->dim;
  const int R = std::min<int>(bp.out_degree, kEll);
  const int min_deg = std::min<int>(bp.min_degree, R);
  const int rev_cap = kC - 1 - R;  // own row + offers always fit the candidate slots
  const uint32_t salt = 0x2C1B3C6Du + static_cast<uint32_t>(bp.seed);
  const int64_t cmax = std::min(kExtendChunk, n - n0);
  eps_stats st;
  std::memset(&st, 0, sizeof(st));

  DevBuf slot_of, pool, knn, cand, D, fwd_ids, fwd_dist, fwd_cnt, vid, n_slots, rev, rev_cnt, own_ids, own_cnt, sel_ids,
      sel_dist, sel_cnt, deg, scan_tmp;
  DevArray<int64_t> off2;
  DevArray<int32_t> nbrs2;
  EPS_TRY(slot_of.reserve(static_cast<size_t>(n) * 4));
  EPS_CUDA(cudaMemsetAsync(slot_of.p, 0xFF, static_cast<size_t>(n) * 4, ix->stream));
  EPS_TRY(pool.reserve(static_cast<size_t>(cmax) * kPoolL * 8));
  EPS_TRY(knn.reserve(static_cast<size_t>(cmax) * (kC - 1) * 8));
  EPS_TRY(cand.reserve(static_cast<size_t>(std::max(cmax, kSelBatch)) * kC * 4));
  EPS_TRY(D.reserve(static_cast<size_t>(kSelBatch) * kC * kC * 4));
  EPS_TRY(fwd_ids.reserve(static_cast<size_t>(cmax) * kEll * 4));
  EPS_TRY(fwd_dist.reserve(static_cast<size_t>(cmax) * kEll * 4));
  EPS_TRY(fwd_cnt.reserve(static_cast<size_t>(cmax) * 4));
  EPS_TRY(vid.reserve(static_cast<size_t>(cmax) * (R + 1) * 4));
  EPS_TRY(n_slots.reserve(4));
  EPS_TRY(deg.reserve((static_cast<size_t>(n) + 1) * 8));
  // the adjacency table of the old rows, with room for the new ones
  EPS_TRY(ensure_ell(ix, nullptr));
  EPS_TRY(ix->d_ell.grow(static_cast<size_t>(n) * kEll * 4, static_cast<size_t>(n0) * kEll * 4, ix->stream));

  for (int64_t a = n0; a < n; a += kExtendChunk) {
    const int64_t b = std::min(n, a + kExtendChunk);
    const int cn = static_cast<int>(b - a);
    const float* rows = ix->d_vectors + a * dim;
    // ---- 1. pools: graph search over [0, a), exact kNN among [a, b) ----
    const int L = static_cast<int>(std::min<int64_t>(kPoolL, a));
    EPS_TRY(graph_search_as(ix, ix->metric, kPoolWidth, rows, cn, L, pool.as<unsigned long long>(), &st));
    ix->graph_counters_pending = false;
    EPS_TRY(ph->mark(ix, Phases::kSearch));
    const int K = std::min(std::min(bp.knn_k, kC - 1), cn - 1);
    if (K > 0) {
      ScanRequest r;
      r.row_start = a; r.row_end = b; r.k = K; r.metric = ix->metric; r.skip_deleted = false;
      for (int64_t q0 = a; q0 < b; q0 += kKnnQueries) {
        r.queries = ix->d_vectors + q0 * dim; r.nq = std::min(kKnnQueries, b - q0); r.self_base = q0;
        EPS_TRY(exact_topk(ix, r, knn.as<unsigned long long>() + (q0 - a) * K, &st));
      }
    }
    merge_pools_kernel<<<blocks(cn, 128), 128, 0, ix->stream>>>(pool.as<unsigned long long>(), L, knn.as<unsigned long long>(),
                                                                std::max(K, 0), a, cn, cand.as<int32_t>());
    EPS_CUDA(cudaGetLastError());
    EPS_TRY(ph->mark(ix, Phases::kKnn));
    // ---- 2. forward selection ----
    EPS_TRY(select_rows(ix, cn, cand.as<int32_t>(), kC, D.as<float>(), R, bp.candidate_pool, 0, min_deg, bp.alpha,
                        fwd_ids.as<int32_t>(), fwd_dist.as<float>(), fwd_cnt.as<int32_t>(), [](int64_t, int, int32_t*) {}));
    EPS_TRY(ph->mark(ix, Phases::kSelect));
    // ---- 3. reverse edges ----
    own_new_slots_kernel<<<blocks(cn, 256), 256, 0, ix->stream>>>(a, cn, slot_of.as<int32_t>(), vid.as<int32_t>());
    EPS_CUDA(cudaMemcpyAsync(n_slots.p, &cn, 4, cudaMemcpyHostToDevice, ix->stream));
    mark_targets_kernel<<<blocks(static_cast<int64_t>(cn) * kEll, 256), 256, 0, ix->stream>>>(
        fwd_ids.as<int32_t>(), fwd_cnt.as<int32_t>(), cn, a, ix->d_offsets, R, slot_of.as<int32_t>(), vid.as<int32_t>(),
        n_slots.as<int32_t>());
    EPS_CUDA(cudaGetLastError());
    int32_t T32 = 0;
    EPS_CUDA(cudaMemcpyAsync(&T32, n_slots.p, 4, cudaMemcpyDeviceToHost, ix->stream));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
    const int64_t T = T32;
    ph->max_slots = std::max(ph->max_slots, T);
    EPS_TRY(rev.reserve(static_cast<size_t>(T) * rev_cap * 8));
    EPS_TRY(rev_cnt.reserve(static_cast<size_t>(T) * 4));
    EPS_TRY(own_ids.reserve(static_cast<size_t>(T) * kEll * 4));
    EPS_TRY(own_cnt.reserve(static_cast<size_t>(T) * 4));
    EPS_TRY(sel_ids.reserve(static_cast<size_t>(T) * kEll * 4));
    EPS_TRY(sel_dist.reserve(static_cast<size_t>(T) * kEll * 4));
    EPS_TRY(sel_cnt.reserve(static_cast<size_t>(T) * 4));
    EPS_CUDA(cudaMemsetAsync(rev.p, 0xFF, static_cast<size_t>(T) * rev_cap * 8, ix->stream));
    EPS_CUDA(cudaMemsetAsync(rev_cnt.p, 0, static_cast<size_t>(T) * 4, ix->stream));
    push_reverse_kernel<<<blocks(static_cast<int64_t>(cn) * kEll, 256), 256, 0, ix->stream>>>(
        fwd_ids.as<int32_t>(), fwd_cnt.as<int32_t>(), cn, a, slot_of.as<int32_t>(), rev_cap, rev.as<unsigned long long>(),
        rev_cnt.as<int32_t>(), salt);
    gather_own_kernel<<<blocks(T * kEll, 256), 256, 0, ix->stream>>>(vid.as<int32_t>(), T, cn, fwd_ids.as<int32_t>(),
                                                                     fwd_cnt.as<int32_t>(), ix->d_ell, ix->d_offsets,
                                                                     own_ids.as<int32_t>(), own_cnt.as<int32_t>());
    EPS_CUDA(cudaGetLastError());
    auto fill_union = [&](int64_t s0, int batch, int32_t* c) {
      fill_cand_union_kernel<<<blocks(batch, 128), 128, 0, ix->stream>>>(own_ids.as<int32_t>(), own_cnt.as<int32_t>(), kEll,
                                                                         rev.as<unsigned long long>(), rev_cnt.as<int32_t>(),
                                                                         rev_cap, s0, batch, c, vid.as<int32_t>());
    };
    // cand_step 0: every batch fills the same kSelBatch cand rows
    EPS_TRY(select_rows(ix, T, cand.as<int32_t>(), 0, D.as<float>(), R, kC, 2, min_deg, bp.alpha, sel_ids.as<int32_t>(),
                        sel_dist.as<float>(), sel_cnt.as<int32_t>(), fill_union));
    EPS_TRY(ph->mark(ix, Phases::kReverse));
    // ---- 4. splice ----
    new_degrees_kernel<<<blocks(b + 1, 256), 256, 0, ix->stream>>>(ix->d_offsets, b, slot_of.as<int32_t>(),
                                                                   sel_cnt.as<int32_t>(), deg.as<int64_t>());
    EPS_CUDA(cudaGetLastError());
    EPS_TRY(off2.reserve((static_cast<size_t>(n) + 1) * 8));  // after the first swap: the previous offsets
    size_t tmp_bytes = 0;
    EPS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, deg.as<int64_t>(), off2.as<int64_t>(), b + 1, ix->stream));
    EPS_TRY(scan_tmp.reserve(tmp_bytes));
    EPS_CUDA(cub::DeviceScan::ExclusiveSum(scan_tmp.p, tmp_bytes, deg.as<int64_t>(), off2.as<int64_t>(), b + 1, ix->stream));
    int64_t e = 0;
    EPS_CUDA(cudaMemcpyAsync(&e, off2.as<int64_t>() + b, 8, cudaMemcpyDeviceToHost, ix->stream));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
    EPS_TRY(nbrs2.grow(std::max<size_t>(static_cast<size_t>(e), 1) * 4, 0, ix->stream));
    splice_kernel<<<blocks(b * 32, 256), 256, 0, ix->stream>>>(ix->d_offsets, ix->d_nbrs, b, slot_of.as<int32_t>(),
                                                               sel_ids.as<int32_t>(), off2, nbrs2, ix->d_ell);
    clear_slots_kernel<<<blocks(T, 256), 256, 0, ix->stream>>>(vid.as<int32_t>(), T, slot_of.as<int32_t>());
    EPS_CUDA(cudaGetLastError());
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
    ix->d_offsets.swap(off2);  // off2 / nbrs2 now hold the previous graph, and are reused for the next chunk
    ix->d_nbrs.swap(nbrs2);
    ix->n_indexed = b;
    ix->n_edges = e;
    ix->init_L = 0;  // the seed set (nav's row, then nav + 1, ... mod n_indexed) and its rows
    ix->seed_rows_L = 0;
    EPS_TRY(ph->mark(ix, Phases::kSplice));
  }
  return EPS_OK;
}

// Every row of [0, n) reachable from nav: flood over the copied-back CSR, then the build's repair steps 3 and 4.
int extend_repair(Index* ix, const eps_build_params& bp, Phases* ph) {
  const int64_t n = ix->n_indexed, e = ix->n_edges, nav = ix->nav;
  std::vector<int64_t> off(static_cast<size_t>(n) + 1);
  std::vector<int32_t> nb(static_cast<size_t>(std::max<int64_t>(e, 1)));
  EPS_CUDA(cudaMemcpyAsync(off.data(), ix->d_offsets, off.size() * 8, cudaMemcpyDeviceToHost, ix->stream));
  if (e > 0) EPS_CUDA(cudaMemcpyAsync(nb.data(), ix->d_nbrs, static_cast<size_t>(e) * 4, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  std::vector<int32_t> cnt(static_cast<size_t>(n));
  for (int64_t v = 0; v < n; ++v) cnt[v] = static_cast<int32_t>(off[v + 1] - off[v]);
  ConnRepair rep(n, nb.data(), cnt.data(), 0);
  rep.off = off.data();
  rep.flood(static_cast<int32_t>(nav));
  ph->unreached = n - rep.linked;
  if (rep.linked == n) return EPS_OK;
  const int64_t Ls = std::min<int64_t>(n, std::max<int>(64, bp.search_length));
  uint64_t rng = 0x9E3779B97F4A7C15ull ^ static_cast<uint64_t>(bp.seed);
  eps_stats st;
  std::memset(&st, 0, sizeof(st));
  EPS_TRY(repair_by_search(ix, &rep, Ls, &rng, &st));
  std::vector<int64_t> off2;
  std::vector<int32_t> nb2;
  rep.flatten(nav, &off2, &nb2);
  return upload_csr(ix, n, off2.data(), nb2.data(), off2[n], nav);
}

// Stored row sketches of [0, n0) extended to [0, n_indexed) with the kept basis: [n x m] sketches, then [n] bounds,
// then (inner product, cosine) [n] dot-product terms.
int extend_sketches(Index* ix, int64_t n0) {
  const int64_t n = ix->n_indexed, m = ix->sk_m;
  Mem fresh;
  EPS_TRY(fresh.reserve(static_cast<size_t>(sketch_floats(ix, n)) * 4));
  float* sk = fresh.as<float>();
  EPS_CUDA(cudaMemcpyAsync(sk, ix->d_sk, static_cast<size_t>(n0) * m * 4, cudaMemcpyDeviceToDevice, ix->stream));
  EPS_CUDA(cudaMemcpyAsync(sk + n * m, ix->d_sk + n0 * m, static_cast<size_t>(n0) * 4, cudaMemcpyDeviceToDevice, ix->stream));
  EPS_TRY(sketch_rows(ix, ix->d_vectors + n0 * ix->dim, n - n0, sk + n0 * m, sk + n * m + n0));
  if (ix->metric != EPS_METRIC_L2) {
    float2* terms = reinterpret_cast<float2*>(sk + sk_terms_off(n));
    EPS_CUDA(cudaMemcpyAsync(terms, ix->d_sk + sk_terms_off(n0), static_cast<size_t>(n0) * 8, cudaMemcpyDeviceToDevice, ix->stream));
    EPS_TRY(dot_row_terms(ix, ix->d_vectors + n0 * ix->dim, n - n0, terms + n0));
  }
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  ix->d_sk.swap(fresh);
  return EPS_OK;
}

}  // namespace

int extend_graph(Index* ix, int64_t n, const eps_build_params* params) {
  const eps_build_params bp = build_defaults(params);
  const int64_t n0 = ix->n_indexed;
  Phases ph;
  int rc = extend_chunks(ix, n, bp, &ph);
  if (rc == EPS_OK) rc = extend_repair(ix, bp, &ph);
  if (rc == EPS_OK) rc = ph.mark(ix, Phases::kRepair);
  ix->graph_counters_pending = false;
  if (rc != EPS_OK) {
    // The graph is a valid graph over the rows linked so far; what is derived from it is rebuilt on demand, and row
    // sketches that no longer cover the indexed rows are dropped (the screen is off until the next install or mode change).
    ix->d_ell.release();
    ix->init_L = 0;
    ix->seed_rows_L = 0;
    if (ix->n_indexed != n0) ix->d_sk.release();
    return rc;
  }
  if (ix->d_sk && extend_sketches(ix, n0) != EPS_OK) {  // the screen only saves time: without its sketches it is off
    cudaGetLastError();
    ix->d_sk.release();
  }
  ph.print();
  return EPS_OK;
}

}  // namespace eps
