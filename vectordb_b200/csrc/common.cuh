// Shared device/host helpers for libepsilla_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/epsilla_b200.h"

namespace eps {

// ---------------------------------------------------------------------------------------------
// Error plumbing
// ---------------------------------------------------------------------------------------------
void set_error(const std::string& msg);
int fail(int code, const std::string& msg);

#define EPS_CUDA(expr)                                                                            \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      return ::eps::fail(_e == cudaErrorMemoryAllocation ? EPS_ERR_OOM : EPS_ERR_CUDA,            \
                         std::string(__FILE__) + ":" + std::to_string(__LINE__) + " " + #expr + ": " + cudaGetErrorString(_e));                    \
    }                                                                                             \
  } while (0)

#define EPS_TRY(expr)          \
  do {                         \
    int _rc = (expr);          \
    if (_rc != EPS_OK) return _rc; \
  } while (0)

constexpr int kWarp = 32;
constexpr unsigned kFull = 0xffffffffu;

// ---------------------------------------------------------------------------------------------
// Candidate keys.  The reference orders queue entries by (distance, id)
// (db/execution/candidate.hpp:16-22).  We pack one entry into 64 bits so that order is a single
// unsigned compare: [ordered-float bits : 32][checked flag : 1][id : 31].  The flag bit is masked
// out of every comparison (kKeyMask); ids are < 2^31 (NN-descent in the reference uses int ids too,
// db/index/knn/nndescent_common.hpp:118).
// ---------------------------------------------------------------------------------------------
constexpr unsigned long long kCheckedBit = 1ull << 31;
constexpr unsigned long long kKeyMask = ~kCheckedBit;
constexpr unsigned long long kKeyInf = 0xffffffffffffffffull & kKeyMask;  // sorts after everything

__host__ __device__ __forceinline__ uint32_t float_to_ordered(float f) {
#ifdef __CUDA_ARCH__
  uint32_t u = __float_as_uint(f + 0.0f);  // +0.0f folds -0 into +0 (reference compares floats)
#else
  float g = f + 0.0f;
  uint32_t u;
  memcpy(&u, &g, 4);
#endif
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ordered_to_float(uint32_t o) {
  uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}
__host__ __device__ __forceinline__ unsigned long long make_key(float dist, uint32_t id) {
  return (static_cast<unsigned long long>(float_to_ordered(dist)) << 32) | id;
}
__host__ __device__ __forceinline__ float key_dist(unsigned long long k) {
  return ordered_to_float(static_cast<uint32_t>(k >> 32));
}
__host__ __device__ __forceinline__ uint32_t key_id(unsigned long long k) {
  return static_cast<uint32_t>(k) & 0x7fffffffu;
}

// ---------------------------------------------------------------------------------------------
// Warp helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

__device__ __forceinline__ float4 ldg_f4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// Streaming 128-bit load that does not allocate in L1 (rows are touched once per query).
__device__ __forceinline__ float4 ldg_f4_stream(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

// Distance of the reference's three metrics from the raw accumulations
// (space_l2.hpp:8-26, space_cosine.hpp:13-16, space_ip.hpp:8-20).
__device__ __forceinline__ float finish_metric(int metric, float acc) {
  if (metric == EPS_METRIC_COSINE) return 1.0f - acc;
  if (metric == EPS_METRIC_IP) return -acc;
  return acc;
}

// Per-lane partial of one row against the query held in shared memory.
// VEC4 path: dim % 4 == 0 and 16-byte aligned rows; lane l covers float4 chunks l, l+32, ...
template <bool L2>
__device__ __forceinline__ float lane_partial_vec4(const float* __restrict__ row, const float* __restrict__ q_smem,
                                                   int dim4, int lane) {
  // All of a lane's 128-bit loads of the row are issued before the first use (up to 6 in flight = 3 KB per
  // warp), so a 768-d row costs ONE memory round trip instead of one per 64 floats.
  float a0 = 0.f, a1 = 0.f;
  for (int base = 0; base < dim4; base += 192) {
    float4 x[6];
#pragma unroll
    for (int u = 0; u < 6; ++u) {
      const int c = base + u * 32 + lane;
      if (c < dim4) x[u] = ldg_f4_stream(row + 4 * c);
    }
#pragma unroll
    for (int u = 0; u < 6; ++u) {
      const int c = base + u * 32 + lane;
      if (c < dim4) {
        const float4 q = *reinterpret_cast<const float4*>(q_smem + 4 * c);
        float& acc = (u & 1) ? a1 : a0;
        if (L2) {
          float d;
          d = x[u].x - q.x; acc = fmaf(d, d, acc);
          d = x[u].y - q.y; acc = fmaf(d, d, acc);
          d = x[u].z - q.z; acc = fmaf(d, d, acc);
          d = x[u].w - q.w; acc = fmaf(d, d, acc);
        } else {
          acc = fmaf(x[u].x, q.x, acc); acc = fmaf(x[u].y, q.y, acc);
          acc = fmaf(x[u].z, q.z, acc); acc = fmaf(x[u].w, q.w, acc);
        }
      }
    }
  }
  return a0 + a1;
}

// Generic path (any dim / alignment): lane-strided scalars.
template <bool L2>
__device__ __forceinline__ float lane_partial_scalar(const float* __restrict__ row, const float* __restrict__ q_smem,
                                                     int dim, int lane) {
  float a = 0.f;
  for (int i = lane; i < dim; i += 32) {
    float x = __ldg(row + i), q = q_smem[i];
    if (L2) { float d = x - q; a = fmaf(d, d, a); } else { a = fmaf(x, q, a); }
  }
  return a;
}

// Full warp-cooperative distance of one row to the smem query; every lane returns the value.
__device__ __forceinline__ float warp_distance(int metric, bool vec4, const float* __restrict__ row,
                                               const float* __restrict__ q_smem, int dim, int lane) {
  float p;
  if (metric == EPS_METRIC_L2) {
    p = vec4 ? lane_partial_vec4<true>(row, q_smem, dim >> 2, lane) : lane_partial_scalar<true>(row, q_smem, dim, lane);
  } else {
    p = vec4 ? lane_partial_vec4<false>(row, q_smem, dim >> 2, lane) : lane_partial_scalar<false>(row, q_smem, dim, lane);
  }
  return finish_metric(metric, warp_sum(p));
}

__host__ __device__ __forceinline__ int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

// Block-wide bitonic sort of n (power of two) 64-bit keys in shared memory, comparing under kKeyMask.
__device__ __forceinline__ void block_bitonic_sort(unsigned long long* keys, int n) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        int ixj = i ^ j;
        if (ixj > i) {
          unsigned long long a = keys[i], b = keys[ixj];
          bool up = (i & k) == 0;
          bool gt = (a & kKeyMask) > (b & kKeyMask);
          if (gt == up) { keys[i] = b; keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
}

}  // namespace eps
