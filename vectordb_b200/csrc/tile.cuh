// Gathered pairwise-distance tile shared by the NSG-style selection (build.cu) and the NN-descent local
// join (nn_descent.cu): one CTA computes the kC x kC distances among the <= kC rows listed in cand[z].
#pragma once
#include "internal.h"

namespace eps {

constexpr int kC = 128;  // candidate slots per vertex

__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}

// Bounded reverse lists that do not depend on arrival order: list p keeps the `cap` arrivals v with the smallest
// key (mix32 priority, v), in key order.  Each push runs an atomicMin cascade down the slots (a slot keeps the smaller
// of its key and the incoming one and passes the larger on), so slot i ends as the i-th smallest key pushed whatever
// the interleaving.  Slots start at kRevEmpty; cnt[p] counts every arrival.
constexpr unsigned long long kRevEmpty = ~0ull;
__device__ __forceinline__ void rev_push(unsigned long long* __restrict__ slots, int cap, int32_t* __restrict__ cnt,
                                         int32_t p, int32_t v, uint32_t salt) {
  atomicAdd(&cnt[p], 1);
  unsigned long long* s = slots + static_cast<int64_t>(p) * cap;
  unsigned long long x = (static_cast<unsigned long long>(mix32(static_cast<uint32_t>(v) * 0x9E3779B1u ^ salt)) << 32) |
                         static_cast<uint32_t>(v);
  if (*reinterpret_cast<volatile unsigned long long*>(s + cap - 1) <= x) return;  // the last kept key only ever drops
  for (int i = 0; i < cap; ++i) {
    const unsigned long long old = atomicMin(s + i, x);
    if (old == kRevEmpty) return;
    x = old > x ? old : x;
  }
}
__device__ __forceinline__ int32_t rev_id(unsigned long long key) { return static_cast<int32_t>(static_cast<uint32_t>(key)); }

// cand [batch x kC] row ids (-1 = empty).  D [batch x kC x kC] = L2^2 between candidate rows.
template <bool L2, bool VEC4>
__global__ void __launch_bounds__(256) pair_tile_kernel(const float* __restrict__ vectors, int dim, int metric,
                                                        const int32_t* __restrict__ cand, float* __restrict__ D) {
  constexpr int BK = 16, PAD = 4;
  __shared__ __align__(16) float As[2][BK][kC + PAD];
  __shared__ int ids[kC];
  const int tid = threadIdx.x;
  const int64_t z = blockIdx.x;
  if (tid < kC) ids[tid] = cand[z * kC + tid];
  __syncthreads();
  const int tx = tid & 15, ty = tid >> 4;
  const int lrow = tid >> 2, lk = (tid & 3) * 4;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  auto load = [&](int r, int k) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    const int id = ids[r];
    if (id >= 0) {
      const float* p = vectors + static_cast<int64_t>(id) * dim + k;
      if (VEC4) { if (k < dim) v = ldg_f4(p); }
      else {
        if (k < dim) v.x = __ldg(p);
        if (k + 1 < dim) v.y = __ldg(p + 1);
        if (k + 2 < dim) v.z = __ldg(p + 2);
        if (k + 3 < dim) v.w = __ldg(p + 3);
      }
    }
    return v;
  };
  float4 r0 = load(lrow, lk), r1 = load(lrow + 64, lk);
  auto stash = [&](int buf) {
    As[buf][lk + 0][lrow] = r0.x; As[buf][lk + 1][lrow] = r0.y; As[buf][lk + 2][lrow] = r0.z; As[buf][lk + 3][lrow] = r0.w;
    As[buf][lk + 0][lrow + 64] = r1.x; As[buf][lk + 1][lrow + 64] = r1.y; As[buf][lk + 2][lrow + 64] = r1.z; As[buf][lk + 3][lrow + 64] = r1.w;
  };
  stash(0);
  __syncthreads();
  const int nk = (dim + BK - 1) / BK;
  for (int kt = 0; kt < nk; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < nk) { r0 = load(lrow, (kt + 1) * BK + lk); r1 = load(lrow + 64, (kt + 1) * BK + lk); }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[8], b[8];
      *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[cur][k][ty * 8]);
      *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[cur][k][ty * 8 + 4]);
      *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&As[cur][k][tx * 8]);
      *reinterpret_cast<float4*>(&b[4]) = *reinterpret_cast<const float4*>(&As[cur][k][tx * 8 + 4]);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (L2) { float d = a[i] - b[j]; acc[i][j] = fmaf(d, d, acc[i][j]); }
          else { acc[i][j] = fmaf(a[i], b[j], acc[i][j]); }
        }
    }
    if (kt + 1 < nk) { stash(cur ^ 1); __syncthreads(); }
  }
  float* out = D + z * kC * kC;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float* dst = out + (ty * 8 + i) * kC + tx * 8;
    *reinterpret_cast<float4*>(dst) = make_float4(finish_metric(metric, acc[i][0]), finish_metric(metric, acc[i][1]),
                                                 finish_metric(metric, acc[i][2]), finish_metric(metric, acc[i][3]));
    *reinterpret_cast<float4*>(dst + 4) = make_float4(finish_metric(metric, acc[i][4]), finish_metric(metric, acc[i][5]),
                                                     finish_metric(metric, acc[i][6]), finish_metric(metric, acc[i][7]));
  }
}


// metric: EPS_METRIC_* of the distances wanted (L2 for the NSG selection, the field metric for NN-descent)
inline int launch_pair_tiles(Index* ix, int metric, const int32_t* d_cand, float* d_D, int batch) {
  const int dim = static_cast<int>(ix->dim);
  if (metric == EPS_METRIC_L2) {
    if (ix->vec4) pair_tile_kernel<true, true><<<batch, 256, 0, ix->stream>>>(ix->d_vectors, dim, metric, d_cand, d_D);
    else pair_tile_kernel<true, false><<<batch, 256, 0, ix->stream>>>(ix->d_vectors, dim, metric, d_cand, d_D);
  } else {
    if (ix->vec4) pair_tile_kernel<false, true><<<batch, 256, 0, ix->stream>>>(ix->d_vectors, dim, metric, d_cand, d_D);
    else pair_tile_kernel<false, false><<<batch, 256, 0, ix->stream>>>(ix->d_vectors, dim, metric, d_cand, d_D);
  }
  EPS_CUDA(cudaGetLastError());
  return EPS_OK;
}

// Selection kernels of the build (build.cu), also run by the extension (extend.cu).
__global__ void select_edges_kernel(const int32_t* __restrict__ cand, const float* __restrict__ D, int batch,
                                    int out_degree, int pool_cap, int keep_all_if_fits, int min_degree, float alpha,
                                    int64_t v_base,
                                    int32_t* __restrict__ out_ids, float* __restrict__ out_dist,
                                    int32_t* __restrict__ out_cnt, int out_stride);
__global__ void fill_cand_union_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ cnt, int stride,
                                       const unsigned long long* __restrict__ rev, const int32_t* __restrict__ rev_cnt, int rev_cap,
                                       int64_t v0, int batch, int32_t* __restrict__ cand, const int32_t* __restrict__ vids);

}  // namespace eps
