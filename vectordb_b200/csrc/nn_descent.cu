// B1 — NN-descent kNN graph on device.  SURVEY.md §8a row B1.
//
// Reference: NNDescent<ORACLE>::iterate (engine/db/index/knn/nndescent.hpp:96-192) with KNN::update
// (nndescent_common.hpp:151-180), driven by KNNGraph (knn.hpp:88-110): random initial lists, then per
// iteration a LOCAL JOIN at every vertex over its sampled new/old neighbours and reverse neighbours
// (new x new, new x old — :101-134; old x old pairs were joined in an earlier iteration), each joined pair
// (p,q) offering q to p's list and p to q's list; entries inserted this iteration carry flag = true ("new"),
// sampled ones are cleared (:139-170); stop when updates / (K*N) < delta (knn.hpp:104-108).
//
// Device mapping (batched all-pairs tiles, north_star):
//   * one 128-slot candidate set per vertex: slots [0,64) = sampled NEW (forward + reverse), slots
//     [64,128) = sampled OLD (forward + reverse); the local join of a vertex is ONE gathered 128x128xd
//     distance tile (tile.cuh) in the field metric — O(S) operand reuse instead of S^2 independent pairs;
//   * updates are selective (the two closest join partners of every candidate), applied by a warp under a
//     per-list spin lock with a coalesced load / ballot-rank / shuffle-shift / store of the sorted list;
//   * sampling, reverse lists and flags are integer passes over the lists.
// Unlike the reference (rand(), random_shuffle, racy OpenMP) the result is reproducible: the initial lists are seeded,
// a list after a local-join launch is the best K of its old entries and every proposal whatever the insertion order,
// reverse lists keep a hash-chosen subset (rev_push), and the convergence test counts the entries a list gained over
// the iteration rather than racy insert successes.  Parity with the reference is graph quality (SURVEY.md §8c).
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "internal.h"
#include "tile.cuh"

namespace eps {

constexpr int kHalf = kC / 2;  // 64 new + 64 old slots

// Random initial lists (nndescent.hpp:76-91): K pseudo-random ids per vertex, distances evaluated, sorted,
// duplicates blanked.  One CTA (128 threads) per vertex.  All entries start "new" (flag bit clear).
__global__ void __launch_bounds__(128) nnd_init_kernel(const float* __restrict__ vectors, int64_t n, int dim, int metric,
                                                      int vec4, int K, uint32_t seed, unsigned long long* __restrict__ knn) {
  extern __shared__ __align__(16) unsigned char ni_smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(ni_smem);  // [128]
  float* qv = reinterpret_cast<float*>(keys + kC);
  const int64_t v = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < dim; i += blockDim.x) qv[i] = vectors[v * dim + i];
  keys[tid] = kKeyInf;
  __syncthreads();
  for (int j = warp; j < K; j += 4) {
    uint32_t h = mix32(static_cast<uint32_t>(v) * 0x9E3779B1u + static_cast<uint32_t>(j) * 0x85EBCA77u + seed);
    int64_t u = static_cast<int64_t>(h % static_cast<uint32_t>(n - 1));
    if (u >= v) ++u;  // never the vertex itself
    float d = warp_distance(metric, vec4 != 0, vectors + u * dim, qv, dim, lane);
    if (lane == 0) keys[j] = make_key(d, static_cast<uint32_t>(u));
  }
  __syncthreads();
  block_bitonic_sort(keys, kC);
  unsigned long long mine = keys[tid];
  bool dup = tid > 0 && mine != kKeyInf && key_id(keys[tid - 1]) == key_id(mine) && (keys[tid - 1] >> 32) == (mine >> 32);
  __syncthreads();
  if (dup) keys[tid] = kKeyInf;
  __syncthreads();
  block_bitonic_sort(keys, kC);
  if (tid < K) knn[v * K + tid] = keys[tid];
}

// Sampling (nndescent.hpp:139-170): up to S new entries (closest first) become this iteration's nn_new and
// lose their flag; up to S old entries become nn_old.  Also appends the vertex to the reverse lists of the
// sampled neighbours (:173-180), up to S each (rev_push).  Snapshots the ids of the list for the convergence
// count.  One thread per vertex.
__global__ void nnd_sample_kernel(unsigned long long* __restrict__ knn, int64_t n, int K, int S, uint32_t salt,
                                  int32_t* __restrict__ fnew, int32_t* __restrict__ fold, unsigned long long* __restrict__ rnew,
                                  unsigned long long* __restrict__ rold, int32_t* __restrict__ rnew_cnt,
                                  int32_t* __restrict__ rold_cnt, int32_t* __restrict__ snap) {
  const int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (v >= n) return;
  unsigned long long* list = knn + v * K;
  int nn = 0, no = 0;
  for (int j = 0; j < K; ++j) snap[v * K + j] = (list[j] & kKeyMask) == kKeyInf ? -1 : static_cast<int32_t>(key_id(list[j]));
  for (int j = 0; j < K; ++j) {
    const unsigned long long key = list[j];
    if ((key & kKeyMask) == kKeyInf) break;
    const int32_t u = static_cast<int32_t>(key_id(key));
    if (!(key & kCheckedBit)) {  // new
      if (nn < S) {
        fnew[v * S + nn++] = u;
        list[j] = key | kCheckedBit;
        rev_push(rnew, S, rnew_cnt, u, static_cast<int32_t>(v), salt);
      }
    } else if (no < S) {
      fold[v * S + no++] = u;
      rev_push(rold, S, rold_cnt, u, static_cast<int32_t>(v), salt ^ 0x5bd1e995u);
    }
  }
  for (; nn < S; ++nn) fnew[v * S + nn] = -1;
  for (; no < S; ++no) fold[v * S + no] = -1;
}

// Candidate rows of a batch of vertices: [new fwd | new rev | old fwd | old rev], duplicates blanked.
// One warp per vertex.
__global__ void nnd_fill_cand_kernel(const int32_t* __restrict__ fnew, const int32_t* __restrict__ fold,
                                     const unsigned long long* __restrict__ rnew, const unsigned long long* __restrict__ rold,
                                     const int32_t* __restrict__ rnew_cnt, const int32_t* __restrict__ rold_cnt, int S,
                                     int64_t v0, int batch, int32_t* __restrict__ cand) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= batch) return;
  const int64_t v = v0 + w;
  int32_t* c = cand + static_cast<int64_t>(w) * kC;
  const int nrn = min(rnew_cnt[v], S), nro = min(rold_cnt[v], S);
  for (int s = lane; s < kC; s += 32) {
    int32_t id = -1;
    if (s < kHalf) {
      if (s < S) id = fnew[v * S + s];
      else if (s - S < nrn && s - S < kHalf - S) id = rev_id(rnew[v * S + (s - S)]);
    } else {
      const int t = s - kHalf;
      if (t < S) id = fold[v * S + t];
      else if (t - S < nro && t - S < kHalf - S) id = rev_id(rold[v * S + (t - S)]);
    }
    if (id == v) id = -1;
    c[s] = id;
  }
  __syncwarp();
  // blank later duplicates (a vertex can be both a forward and a reverse neighbour, new and old)
  for (int s = lane; s < kC; s += 32) {
    const int32_t id = c[s];
    bool dup = false;
    if (id >= 0)
      for (int t = 0; t < s; ++t) dup |= (c[t] == id);
    __syncwarp();
    if (dup) c[s] = -2;
  }
  __syncwarp();
  for (int s = lane; s < kC; s += 32) if (c[s] == -2) c[s] = -1;
}

// Warp-cooperative insert of (key) into the sorted list of `target` (KNN::update,
// nndescent_common.hpp:151-180: reject if not better than the last entry or already present, else shift
// and place).  Returns 1 if inserted.  K <= 128.
__device__ int nnd_insert(unsigned long long* __restrict__ knn, int* __restrict__ locks, int K, int32_t target,
                          unsigned long long key, int lane) {
  unsigned long long* list = knn + static_cast<int64_t>(target) * K;
  // cheap unlocked reject (benign race: the worst entry only ever improves)
  unsigned long long worst = list[K - 1];
  if ((key & kKeyMask) >= (worst & kKeyMask)) return 0;
  if (lane == 0) { while (atomicCAS(&locks[target], 0, 1) != 0) {} }
  __syncwarp();
  __threadfence();
  unsigned long long a[4];
  const uint32_t id = key_id(key);
  bool dup = false;
  int less = 0;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int e = t * 32 + lane;
    a[t] = kKeyInf;
    if (e < K) a[t] = *reinterpret_cast<volatile unsigned long long*>(list + e);
    dup |= (e < K) && ((a[t] & kKeyMask) != kKeyInf) && key_id(a[t]) == id;
    less += __popc(__ballot_sync(kFull, (a[t] & kKeyMask) < (key & kKeyMask)));
  }
  const bool any_dup = __any_sync(kFull, dup);
  int done = 0;
  if (!any_dup && less < K) {
    const int pos = less;
    unsigned long long b[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      unsigned long long prev = __shfl_up_sync(kFull, a[t], 1);
      const unsigned long long tail = __shfl_sync(kFull, a[t > 0 ? t - 1 : 0], 31);
      if (lane == 0) prev = tail;
      const int e = t * 32 + lane;
      b[t] = e < pos ? a[t] : (e == pos ? key : prev);
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int e = t * 32 + lane;
      if (e < K && e >= pos) *reinterpret_cast<volatile unsigned long long*>(list + e) = b[t];
    }
    done = 1;
  }
  __threadfence();
  __syncwarp();
  if (lane == 0) atomicExch(&locks[target], 0);
  return done;
}

// Local join over the tile: row i (candidate cand[i]) looks at every partner j it is joined with
// (new x new and new x old: at least one of the two is in the new half) and offers itself its two closest
// partners.  One CTA of 128 threads per vertex; thread i scans row i, then the 4 warps apply the proposals.
__global__ void __launch_bounds__(128) nnd_join_kernel(const int32_t* __restrict__ cand, const float* __restrict__ D,
                                                      int batch, int K, unsigned long long* __restrict__ knn,
                                                      int* __restrict__ locks) {
  __shared__ int ids[kC];
  __shared__ int p_target[2 * kC];
  __shared__ unsigned long long p_key[2 * kC];
  __shared__ int n_prop;
  const int z = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  ids[tid] = cand[static_cast<int64_t>(z) * kC + tid];
  if (tid == 0) n_prop = 0;
  __syncthreads();
  const int me = ids[tid];
  if (me >= 0) {
    // the tile is symmetric: read COLUMN tid so consecutive threads touch consecutive addresses
    const float* col = D + static_cast<int64_t>(z) * kC * kC + tid;
    const bool i_new = tid < kHalf;
    unsigned long long b0 = kKeyInf, b1 = kKeyInf;
    const int jend = i_new ? kC : kHalf;  // an old row only joins with the new half
    for (int j = 0; j < jend; ++j) {
      const int other = ids[j];
      if (other < 0 || j == tid) continue;
      const unsigned long long key = make_key(col[j * kC], static_cast<uint32_t>(other));
      if (key < b0) { b1 = b0; b0 = key; } else if (key < b1) { b1 = key; }
    }
    const unsigned long long worst = knn[static_cast<int64_t>(me) * K + (K - 1)] & kKeyMask;
    if (b0 < worst) { const int s = atomicAdd(&n_prop, 1); p_target[s] = me; p_key[s] = b0; }
    if (b1 < worst) { const int s = atomicAdd(&n_prop, 1); p_target[s] = me; p_key[s] = b1; }
  }
  __syncthreads();
  const int np = n_prop;
  for (int p = warp; p < np; p += 4) nnd_insert(knn, locks, K, p_target[p], p_key[p], lane);
}

// Updates of an iteration (knn.hpp:104-108): entries of the lists that were not in them when it was sampled.  One warp
// per vertex, K <= 128.
__global__ void nnd_count_updates_kernel(const unsigned long long* __restrict__ knn, const int32_t* __restrict__ snap,
                                         int64_t n, int K, unsigned long long* __restrict__ n_updates) {
  const int64_t v = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (v >= n) return;
  int32_t f[4];
  bool seen[4] = {false, false, false, false};
  for (int h = 0; h < 4; ++h) {
    const int e = lane + 32 * h;
    const unsigned long long key = e < K ? knn[v * K + e] : kKeyInf;
    f[h] = (key & kKeyMask) == kKeyInf ? -1 : static_cast<int32_t>(key_id(key));
  }
  for (int t = 0; t < K; ++t) {
    const int32_t s = snap[v * K + t];
#pragma unroll
    for (int h = 0; h < 4; ++h) seen[h] |= f[h] == s;
  }
  int fresh = 0;
#pragma unroll
  for (int h = 0; h < 4; ++h) fresh += __popc(__ballot_sync(kFull, f[h] >= 0 && !seen[h]));
  if (lane == 0 && fresh) atomicAdd(n_updates, static_cast<unsigned long long>(fresh));
}

__global__ void nnd_clear_flags_kernel(unsigned long long* knn, int64_t total) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < total) knn[i] &= kKeyMask;
}

int nn_descent(Index* ix, int64_t n, int K, const eps_build_params& bp, unsigned long long* d_knn, eps_stats* st) {
  if (K > kC) return fail(EPS_ERR_UNSUPPORTED, "NN-descent supports K <= 128");
  const int S = std::max(4, std::min<int>(bp.nnd_sample, kHalf / 2));
  const int dim = static_cast<int>(ix->dim);
  const size_t init_smem = kC * 8 + static_cast<size_t>((dim + 3) & ~3) * 4;
  if (init_smem > 200 * 1024) return fail(EPS_ERR_UNSUPPORTED, "dimension too large for NN-descent init");
  if (init_smem > 48 * 1024)
    EPS_CUDA(cudaFuncSetAttribute(nnd_init_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(init_smem)));
  nnd_init_kernel<<<static_cast<unsigned>(n), 128, init_smem, ix->stream>>>(ix->d_vectors, n, dim, ix->metric,
                                                                           ix->vec4 ? 1 : 0, K, 0x1234567u + bp.seed, d_knn);
  EPS_CUDA(cudaGetLastError());

  DevBuf fnew, fold, rnew, rold, rnc, roc, locks, cand, D, counter, snap;
  EPS_TRY(fnew.reserve(static_cast<size_t>(n) * S * 4));
  EPS_TRY(fold.reserve(static_cast<size_t>(n) * S * 4));
  EPS_TRY(rnew.reserve(static_cast<size_t>(n) * S * 8));
  EPS_TRY(rold.reserve(static_cast<size_t>(n) * S * 8));
  EPS_TRY(snap.reserve(static_cast<size_t>(n) * K * 4));
  EPS_TRY(rnc.reserve(static_cast<size_t>(n) * 4));
  EPS_TRY(roc.reserve(static_cast<size_t>(n) * 4));
  EPS_TRY(locks.reserve(static_cast<size_t>(n) * 4));
  EPS_TRY(counter.reserve(8));
  EPS_CUDA(cudaMemsetAsync(locks.p, 0, static_cast<size_t>(n) * 4, ix->stream));
  const int64_t batch_max = 8192;
  EPS_TRY(cand.reserve(static_cast<size_t>(batch_max) * kC * 4));
  EPS_TRY(D.reserve(static_cast<size_t>(batch_max) * kC * kC * 4));

  int iters_done = 0;
  for (int it = 0; it < bp.nnd_iters; ++it) {
    EPS_CUDA(cudaMemsetAsync(rnc.p, 0, static_cast<size_t>(n) * 4, ix->stream));
    EPS_CUDA(cudaMemsetAsync(roc.p, 0, static_cast<size_t>(n) * 4, ix->stream));
    EPS_CUDA(cudaMemsetAsync(counter.p, 0, 8, ix->stream));
    EPS_CUDA(cudaMemsetAsync(rnew.p, 0xFF, static_cast<size_t>(n) * S * 8, ix->stream));
    EPS_CUDA(cudaMemsetAsync(rold.p, 0xFF, static_cast<size_t>(n) * S * 8, ix->stream));
    nnd_sample_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, ix->stream>>>(
        d_knn, n, K, S, 0x2545F491u * static_cast<uint32_t>(it + 1) + static_cast<uint32_t>(bp.seed), fnew.as<int32_t>(),
        fold.as<int32_t>(), rnew.as<unsigned long long>(), rold.as<unsigned long long>(), rnc.as<int32_t>(), roc.as<int32_t>(),
        snap.as<int32_t>());
    for (int64_t v0 = 0; v0 < n; v0 += batch_max) {
      const int batch = static_cast<int>(std::min(batch_max, n - v0));
      nnd_fill_cand_kernel<<<(batch * 32 + 127) / 128, 128, 0, ix->stream>>>(
          fnew.as<int32_t>(), fold.as<int32_t>(), rnew.as<unsigned long long>(), rold.as<unsigned long long>(), rnc.as<int32_t>(),
          roc.as<int32_t>(),
          S, v0, batch, cand.as<int32_t>());
      EPS_TRY(launch_pair_tiles(ix, ix->metric, cand.as<int32_t>(), D.as<float>(), batch));
      nnd_join_kernel<<<batch, 128, 0, ix->stream>>>(cand.as<int32_t>(), D.as<float>(), batch, K, d_knn, locks.as<int>());
      if (st) st->kernel_launches += 3;
    }
    nnd_count_updates_kernel<<<static_cast<unsigned>((n * 32 + 255) / 256), 256, 0, ix->stream>>>(
        d_knn, snap.as<int32_t>(), n, K, counter.as<unsigned long long>());
    EPS_CUDA(cudaGetLastError());
    unsigned long long upd = 0;
    EPS_CUDA(cudaMemcpyAsync(&upd, counter.p, 8, cudaMemcpyDeviceToHost, ix->stream));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
    ++iters_done;
    if (getenv("EPS_BUILD_VERBOSE")) fprintf(stderr, "[nn_descent] iter %d updates %llu (rate %.5f)\n", it, upd,
                                             static_cast<double>(upd) / (static_cast<double>(n) * K));
    if (static_cast<double>(upd) < static_cast<double>(bp.nnd_delta) * static_cast<double>(n) * K) break;
  }
  const int64_t total = n * K;
  nnd_clear_flags_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, ix->stream>>>(d_knn, total);
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  fnew.release(); fold.release(); rnew.release(); rold.release(); rnc.release(); roc.release();
  locks.release(); cand.release(); D.release(); counter.release(); snap.release();
  (void)iters_done;
  return EPS_OK;
}

}  // namespace eps
