// K1 — exact (brute-force) distance + top-k.  SURVEY.md §8a rows A9 / A10 (+ the tail of A11) and the
// all-pairs tiles of the graph build (B1).
//
// Reference behaviour restated (engine/db/execution/vec_search_executor.cpp):
//   BruteForceSearch (:717-768): distance for EVERY row of [start,end), drop deleted / filter-failing rows
//   (the filter sees the distance), sort ascending by (distance,id).
//   PreFilterBruteForceSearch (:770-831): deleted / filter (distance 0) first, distance for passing rows.
// A full sort is not needed: the caller only ever reads the first min(n, limit, L_local) entries, so we
// keep an exact top-k with the same (distance,id) order.
//
// Two distance kernels, both fp32 SIMT (this is exact-arithmetic work; the L2 form is the direct
// sum of squared differences like the reference, not the |x|^2-2xy+|y|^2 expansion):
//   * bf_dist_rows_kernel  — small batches (nq <= 16): one warp per row, coalesced float4 row loads, the
//     query tile in shared memory, warp-shuffle reduction.  HBM-bound: N*d*4 bytes per <=8 queries.
//   * bf_dist_tile_kernel  — large batches: 128x128x16 shared-memory tiles, 8x8 register micro-tiles.
//     FP32-pipe bound (2*N*d*B FMA-class ops, 3 for L2).
// followed by bf_select_kernel: threshold-filtered streaming top-k per (query, row-split).
#include <cstdlib>

#include "internal.h"

namespace eps {

// ------------------------------------------------------------------------------------------------
// pass bitmap: bit i set <=> row (row_start+i) is not deleted and passes the distance-free filter.
// ------------------------------------------------------------------------------------------------
__global__ void pass_bitmap_kernel(const uint8_t* __restrict__ deleted, int64_t deleted_bytes,
                                   const FilterProg* __restrict__ prog, const char* __restrict__ attrs,
                                   int64_t stride, int64_t row_start, int64_t n, uint32_t* __restrict__ pass) {
  int64_t w = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  int64_t nwords = (n + 31) >> 5;
  if (w >= nwords) return;
  uint32_t bits = 0;
  for (int b = 0; b < 32; ++b) {
    int64_t i = w * 32 + b;
    if (i >= n) break;
    int64_t r = row_start + i;
    bool ok = true;
    if (deleted && (r >> 3) < deleted_bytes) ok = !((deleted[r >> 3] >> (r & 7)) & 1);
    if (ok && prog) ok = filter_eval(*prog, attrs, stride, r, 0.f);
    if (ok) bits |= (1u << b);
  }
  pass[w] = bits;
}

// ------------------------------------------------------------------------------------------------
// Small-batch distances: warp per row.
// D[q * ldd + (r - row_start)] for q in [0,nq_tile), r in [row_start, row_start + n).
// ------------------------------------------------------------------------------------------------
constexpr int kRowsQT = 8;

template <bool L2, bool VEC4>
__global__ void __launch_bounds__(256) bf_dist_rows_kernel(const float* __restrict__ vectors, int dim, int metric,
                                                           int64_t row_start, int64_t n,
                                                           const float* __restrict__ queries, int nq_tile,
                                                           float* __restrict__ D, int64_t ldd) {
  extern __shared__ __align__(16) float q_smem[];  // [nq_tile][dim]
  for (int i = threadIdx.x; i < nq_tile * dim; i += blockDim.x) q_smem[i] = queries[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int64_t nwarps = (gridDim.x * static_cast<int64_t>(blockDim.x)) >> 5;
  const int64_t ngroups = (n + 31) >> 5;
  for (int64_t g = warp; g < ngroups; g += nwarps) {
    float keep[kRowsQT];
#pragma unroll
    for (int q = 0; q < kRowsQT; ++q) keep[q] = 0.f;
    const int64_t base = g << 5;
    const int rows_here = static_cast<int>(min(static_cast<int64_t>(32), n - base));
    for (int j = 0; j < rows_here; ++j) {
      const float* row = vectors + (row_start + base + j) * static_cast<int64_t>(dim);
      float acc[kRowsQT];
#pragma unroll
      for (int q = 0; q < kRowsQT; ++q) acc[q] = 0.f;
      if (VEC4) {
        const int dim4 = dim >> 2;
        for (int c = lane; c < dim4; c += 32) {
          float4 x = ldg_f4_stream(row + 4 * c);
#pragma unroll
          for (int q = 0; q < kRowsQT; ++q) {
            if (q < nq_tile) {
              float4 y = *reinterpret_cast<const float4*>(q_smem + q * dim + 4 * c);
              if (L2) {
                float d;
                d = x.x - y.x; acc[q] = fmaf(d, d, acc[q]);
                d = x.y - y.y; acc[q] = fmaf(d, d, acc[q]);
                d = x.z - y.z; acc[q] = fmaf(d, d, acc[q]);
                d = x.w - y.w; acc[q] = fmaf(d, d, acc[q]);
              } else {
                acc[q] = fmaf(x.x, y.x, acc[q]); acc[q] = fmaf(x.y, y.y, acc[q]);
                acc[q] = fmaf(x.z, y.z, acc[q]); acc[q] = fmaf(x.w, y.w, acc[q]);
              }
            }
          }
        }
      } else {
        for (int i = lane; i < dim; i += 32) {
          float x = __ldg(row + i);
#pragma unroll
          for (int q = 0; q < kRowsQT; ++q) {
            if (q < nq_tile) {
              float y = q_smem[q * dim + i];
              if (L2) { float d = x - y; acc[q] = fmaf(d, d, acc[q]); } else { acc[q] = fmaf(x, y, acc[q]); }
            }
          }
        }
      }
#pragma unroll
      for (int q = 0; q < kRowsQT; ++q) {
        if (q < nq_tile) {
          float s = warp_sum(acc[q]);
          if (lane == j) keep[q] = s;
        }
      }
    }
    if (lane < rows_here) {
#pragma unroll
      for (int q = 0; q < kRowsQT; ++q)
        if (q < nq_tile) D[q * ldd + base + lane] = finish_metric(metric, keep[q]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Large-batch distances: 128 (rows) x 128 (queries) x 16 tiles, 256 threads, 8x8 per thread.
// ------------------------------------------------------------------------------------------------
constexpr int kBM = 128, kBN = 128, kBK = 16, kPad = 4;

template <bool VEC4>
__device__ __forceinline__ float4 load_k4(const float* __restrict__ base, int64_t row, int64_t n_rows, int dim, int k) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (row < n_rows) {
    const float* p = base + row * static_cast<int64_t>(dim) + k;
    if (VEC4) {
      if (k < dim) v = ldg_f4(p);  // dim % 4 == 0 => k+3 < dim
    } else {
      if (k < dim) v.x = __ldg(p);
      if (k + 1 < dim) v.y = __ldg(p + 1);
      if (k + 2 < dim) v.z = __ldg(p + 2);
      if (k + 3 < dim) v.w = __ldg(p + 3);
    }
  }
  return v;
}

template <bool L2, bool VEC4>
__global__ void __launch_bounds__(256) bf_dist_tile_kernel(const float* __restrict__ A, int64_t a_rows,
                                                           const float* __restrict__ B, int64_t b_rows, int dim,
                                                           int metric, float* __restrict__ D, int64_t ldd) {
  __shared__ __align__(16) float As[2][kBK][kBM + kPad];
  __shared__ __align__(16) float Bs[2][kBK][kBN + kPad];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t a0 = static_cast<int64_t>(blockIdx.x) * kBM;
  const int64_t b0 = static_cast<int64_t>(blockIdx.y) * kBN;
  const int lrow = tid >> 2;       // 0..63
  const int lk = (tid & 3) * 4;    // 0,4,8,12

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra[2], rb[2];
  const int nk = (dim + kBK - 1) / kBK;
  // prologue
  ra[0] = load_k4<VEC4>(A, a0 + lrow, a_rows, dim, lk);
  ra[1] = load_k4<VEC4>(A, a0 + lrow + 64, a_rows, dim, lk);
  rb[0] = load_k4<VEC4>(B, b0 + lrow, b_rows, dim, lk);
  rb[1] = load_k4<VEC4>(B, b0 + lrow + 64, b_rows, dim, lk);
  auto stash = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int r = lrow + 64 * h;
      As[buf][lk + 0][r] = ra[h].x; As[buf][lk + 1][r] = ra[h].y; As[buf][lk + 2][r] = ra[h].z; As[buf][lk + 3][r] = ra[h].w;
      Bs[buf][lk + 0][r] = rb[h].x; Bs[buf][lk + 1][r] = rb[h].y; Bs[buf][lk + 2][r] = rb[h].z; Bs[buf][lk + 3][r] = rb[h].w;
    }
  };
  stash(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < nk) {
      const int k = (kt + 1) * kBK + lk;
      ra[0] = load_k4<VEC4>(A, a0 + lrow, a_rows, dim, k);
      ra[1] = load_k4<VEC4>(A, a0 + lrow + 64, a_rows, dim, k);
      rb[0] = load_k4<VEC4>(B, b0 + lrow, b_rows, dim, k);
      rb[1] = load_k4<VEC4>(B, b0 + lrow + 64, b_rows, dim, k);
    }
#pragma unroll
    for (int k = 0; k < kBK; ++k) {
      float a[8], b[8];
      *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[cur][k][ty * 8]);
      *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[cur][k][ty * 8 + 4]);
      *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 8]);
      *reinterpret_cast<float4*>(&b[4]) = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 8 + 4]);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (L2) { float d = a[i] - b[j]; acc[i][j] = fmaf(d, d, acc[i][j]); }
          else { acc[i][j] = fmaf(a[i], b[j], acc[i][j]); }
        }
    }
    if (kt + 1 < nk) {
      stash(cur ^ 1);
      __syncthreads();
    }
  }
  // epilogue: D[query][row]
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int64_t q = b0 + tx * 8 + j;
    if (q >= b_rows) continue;
    const int64_t r = a0 + ty * 8;
    float* dst = D + q * ldd + r;
    if (r + 7 < a_rows && ((ldd & 3) == 0)) {
      float4 v0 = make_float4(finish_metric(metric, acc[0][j]), finish_metric(metric, acc[1][j]),
                              finish_metric(metric, acc[2][j]), finish_metric(metric, acc[3][j]));
      float4 v1 = make_float4(finish_metric(metric, acc[4][j]), finish_metric(metric, acc[5][j]),
                              finish_metric(metric, acc[6][j]), finish_metric(metric, acc[7][j]));
      *reinterpret_cast<float4*>(dst) = v0;
      *reinterpret_cast<float4*>(dst + 4) = v1;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (r + i < a_rows) dst[i] = finish_metric(metric, acc[i][j]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Streaming top-k select.  One CTA per (query, split).
// ------------------------------------------------------------------------------------------------
constexpr int kSelThreads = 256;
constexpr int kSelItems = 4;
constexpr int kSelRound = kSelThreads * kSelItems;  // 1024
constexpr int kSelBuf = 2 * kSelRound;              // 2048

__device__ __forceinline__ int lower_bound_keys(const unsigned long long* a, int n, unsigned long long key) {
  int lo = 0, hi = n;
  key &= kKeyMask;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if ((a[mid] & kKeyMask) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Merge the nbuf unsorted keys of buf into the sorted top-k list; result (first k) back in topk.
__device__ void select_flush(unsigned long long* topk, unsigned long long* merged, unsigned long long* buf, int nbuf,
                             int k) {
  const int np = next_pow2(nbuf < 1 ? 1 : nbuf);
  for (int i = nbuf + threadIdx.x; i < np; i += blockDim.x) buf[i] = kKeyInf;
  __syncthreads();
  block_bitonic_sort(buf, np);
  for (int i = threadIdx.x; i < nbuf; i += blockDim.x) {
    unsigned long long key = buf[i];
    int dest = lower_bound_keys(topk, k, key) + i;
    if (dest < k) merged[dest] = key;
  }
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    unsigned long long key = topk[j];
    int dest = j + lower_bound_keys(buf, nbuf, key);
    if (dest < k) merged[dest] = key;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < k; j += blockDim.x) topk[j] = merged[j];
  __syncthreads();
}

struct SelectArgs {
  const float* D = nullptr;                     // [nq x ldd] distances of this chunk (KEYS_IN = false)
  const unsigned long long* keys_in = nullptr;  // [nq x n_in] candidate keys (KEYS_IN = true)
  int64_t ldd = 0;
  int64_t n = 0;                        // elements per query in this chunk
  int64_t row_base = 0;                 // global row id of element 0
  int nsplit = 1;
  int k = 0;
  unsigned long long* state = nullptr;  // [nq x nsplit x k]
  const uint32_t* pass = nullptr;       // bitmap relative to pass_base (may be null)
  int64_t pass_base = 0;
  const FilterProg* dyn = nullptr;      // per-candidate filter that needs the real distance (may be null)
  const char* attrs = nullptr;
  int64_t attr_stride = 0;
  int64_t self_base = -1;               // query q is row self_base + q and is excluded (-1: off)
  const int* counts = nullptr;          // KEYS_IN: valid keys per query (<= n), null = n
  float* thr_out = nullptr;             // if set: distance of the k-th entry after this pass (running threshold)
  int* overflow = nullptr;              // if set: raised when counts[q] > n (candidates were dropped)
};

template <bool KEYS_IN>
__global__ void __launch_bounds__(kSelThreads) bf_select_kernel(SelectArgs a) {
  extern __shared__ __align__(16) unsigned long long sel_smem[];
  unsigned long long* topk = sel_smem;
  unsigned long long* merged = topk + a.k;
  unsigned long long* buf = merged + a.k;
  __shared__ int nbuf;
  const int q = blockIdx.x;
  const int split = blockIdx.y;
  unsigned long long* st = a.state + (static_cast<int64_t>(q) * a.nsplit + split) * a.k;
  for (int j = threadIdx.x; j < a.k; j += blockDim.x) topk[j] = st[j];
  if (threadIdx.x == 0) nbuf = 0;
  __syncthreads();
  unsigned long long thr = topk[a.k - 1] & kKeyMask;
  int64_t n_here = a.n;
  if (KEYS_IN && a.counts) {
    const int c = a.counts[q];
    if (c > a.n) { if (a.overflow && threadIdx.x == 0) *a.overflow = 1; } else n_here = c;
  }
  const int64_t per = (n_here + a.nsplit - 1) / a.nsplit;
  const int64_t begin = split * per;
  const int64_t end = min(n_here, begin + per);
  for (int64_t base = begin; base < end; base += kSelRound) {
#pragma unroll
    for (int it = 0; it < kSelItems; ++it) {
      int64_t i = base + it * kSelThreads + threadIdx.x;
      if (i < end) {
        unsigned long long key;
        int64_t row;
        if (KEYS_IN) {
          key = a.keys_in[static_cast<int64_t>(q) * a.n + i] & kKeyMask;
          row = key_id(key);
        } else {
          row = a.row_base + i;
          key = make_key(a.D[static_cast<int64_t>(q) * a.ldd + i], static_cast<uint32_t>(row));
        }
        if (key < thr && key != kKeyInf) {
          bool ok = true;
          if (!KEYS_IN) {
            if (a.pass) {
              int64_t pi = row - a.pass_base;
              ok = (a.pass[pi >> 5] >> (pi & 31)) & 1u;
            }
            if (ok && a.self_base >= 0 && row == a.self_base + q) ok = false;
            if (ok && a.dyn) ok = filter_eval(*a.dyn, a.attrs, a.attr_stride, row, key_dist(key));
          }
          if (ok) {
            int slot = atomicAdd(&nbuf, 1);
            buf[slot] = key;
          }
        }
      }
    }
    __syncthreads();
    const int n_now = nbuf;
    __syncthreads();  // nobody may bump nbuf for the next round before everyone has read it
    if (n_now > kSelBuf - kSelRound) {
      int n = n_now;
      select_flush(topk, merged, buf, n, a.k);
      if (threadIdx.x == 0) nbuf = 0;
      thr = topk[a.k - 1] & kKeyMask;
      __syncthreads();
    }
  }
  {
    int n = nbuf;
    __syncthreads();
    if (n > 0) select_flush(topk, merged, buf, n, a.k);
  }
  for (int j = threadIdx.x; j < a.k; j += blockDim.x) st[j] = topk[j];
  if (a.thr_out && threadIdx.x == 0 && split == 0) {
    const unsigned long long w = topk[a.k - 1];
    a.thr_out[q] = ((w & kKeyMask) == kKeyInf) ? INFINITY : key_dist(w);
  }
}

__global__ void fill_keys_kernel(unsigned long long* p, int64_t n, unsigned long long v) {
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) p[i] = v;
}

// ------------------------------------------------------------------------------------------------
// Exact re-score of the coarse (tensor-core) candidates: one CTA per query, one warp per candidate, the fp32
// direct form of the reference; then the final (distance,id) sort.  coarse [nq x kc] -> out [nq x k].
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) rescore_kernel(const float* __restrict__ vectors, int dim, int metric, int vec4,
                                                     const float* __restrict__ queries,
                                                     const unsigned long long* __restrict__ coarse, int kc, int kcp, int k,
                                                     unsigned long long* __restrict__ out, unsigned* __restrict__ err_max_bits,
                                                     const float* __restrict__ xnorm, unsigned* __restrict__ xn_max_bits) {
  extern __shared__ __align__(16) unsigned char rs_smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(rs_smem);  // [kcp]
  float* qv = reinterpret_cast<float*>(keys + kcp);
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < dim; i += blockDim.x) qv[i] = queries[static_cast<int64_t>(q) * dim + i];
  for (int i = kc + tid; i < kcp; i += blockDim.x) keys[i] = kKeyInf;
  __syncthreads();
  for (int c = warp; c < kc; c += 4) {
    const unsigned long long ck = coarse[static_cast<int64_t>(q) * kc + c];
    unsigned long long key = kKeyInf;
    if ((ck & kKeyMask) != kKeyInf) {
      const uint32_t id = key_id(ck);
      const float d = warp_distance(metric, vec4 != 0, vectors + static_cast<int64_t>(id) * dim, qv, dim, lane);
      key = make_key(d, id);
      // calibration sample of the coarse pass: |coarse - exact| of a re-scored row (non-negative floats order as uints)
      if (lane == 0 && err_max_bits) {
        atomicMax(err_max_bits, __float_as_uint(fabsf(key_dist(ck) - d)));
        atomicMax(xn_max_bits, __float_as_uint(xnorm[id]));  // the sample's largest |x|^2
      }
    }
    if (lane == 0) keys[c] = key;
  }
  __syncthreads();
  block_bitonic_sort(keys, kcp);
  for (int i = tid; i < k; i += blockDim.x) out[static_cast<int64_t>(q) * k + i] = keys[i];
}

// ------------------------------------------------------------------------------------------------
// Exactness guard of the coarse pass.  A row outside the coarse top-k' has coarse distance >= T (the k'-th best
// coarse value); it can only belong to the exact top-k if its coarse error exceeds T - e_k (e_k = exact k-th best
// after the re-score).  The batch's own re-scored rows (k' x nq samples of |coarse - exact|, whatever the operand
// format or rounding mode did) calibrate the error E.  A coarse error grows with |x| |q|, and the sample only holds the
// re-scored rows, so E is scaled by max(1, M / M_s), M = the table's largest |x| and M_s = the sample's: a row whose
// norm is far above the candidates' cannot hide outside the list.  A query is SAFE when e_k + 2 * E_eff <= T, or when
// fewer than k' rows exist at all.  Unsafe queries are redone (exact fp32 scan, or the whole batch with a larger k').
// ------------------------------------------------------------------------------------------------
__global__ void verify_exact_kernel(const unsigned long long* __restrict__ final_keys, int k_final, const float* __restrict__ thr,
                                    const unsigned* __restrict__ err_max_bits, const unsigned* __restrict__ xn_table_bits,
                                    const unsigned* __restrict__ xn_sample_bits, int nq, int* __restrict__ flags,
                                    int* __restrict__ n_flagged) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  const unsigned long long kth = final_keys[static_cast<int64_t>(q) * k_final + (k_final - 1)];
  const float T = thr[q];
  const float m2 = __uint_as_float(*xn_table_bits), s2 = __uint_as_float(*xn_sample_bits);  // squared norms
  float err = __uint_as_float(*err_max_bits);
  // s2 == 0 < m2: every re-scored row is zero and says nothing about the others (+inf: every such query is unsafe)
  if (m2 > s2) err = s2 > 0.f ? err * sqrtf(m2 / s2) : INFINITY;
  const float eps = 2.0f * err;
  const bool unsafe = (kth & kKeyMask) != kKeyInf && !isinf(T) && !(key_dist(kth) + eps <= T);
  flags[q] = unsafe ? 1 : 0;
  if (unsafe) atomicAdd(n_flagged, 1);
}

__global__ void gather_queries_kernel(const float* __restrict__ queries, const int* __restrict__ idx, int n, int dim,
                                      float* __restrict__ out) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(n) * dim) return;
  out[i] = queries[static_cast<int64_t>(idx[i / dim]) * dim + (i % dim)];
}
__global__ void scatter_keys_kernel(const unsigned long long* __restrict__ in, const int* __restrict__ idx, int n, int k,
                                    unsigned long long* __restrict__ out) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(n) * k) return;
  out[static_cast<int64_t>(idx[i / k]) * k + (i % k)] = in[i];
}

// ------------------------------------------------------------------------------------------------
// Host driver
// ------------------------------------------------------------------------------------------------
// The instances of both SIMT distance kernels, [metric is L2][table is VEC4].
struct SimtKernels {
  decltype(&bf_dist_rows_kernel<true, true>) rows;
  decltype(&bf_dist_tile_kernel<true, true>) tile;
};
static const SimtKernels kSimt[2][2] = {{{bf_dist_rows_kernel<false, false>, bf_dist_tile_kernel<false, false>},
                                         {bf_dist_rows_kernel<false, true>, bf_dist_tile_kernel<false, true>}},
                                        {{bf_dist_rows_kernel<true, false>, bf_dist_tile_kernel<true, false>},
                                         {bf_dist_rows_kernel<true, true>, bf_dist_tile_kernel<true, true>}}};

int launch_distances(Index* ix, int metric, const float* A_base, int64_t row_start, int64_t n, const float* d_queries,
                     int64_t nq, float* D, int64_t ldd, uint64_t* launches, int64_t form_nq) {
  const int dim = static_cast<int>(ix->dim);
  const SimtKernels kern = kSimt[metric == EPS_METRIC_L2][ix->vec4];
  if ((form_nq > 0 ? form_nq : nq) <= 16) {
    int qt_cap = static_cast<int>(std::min<int64_t>(kRowsQT, (200 * 1024) / (ix->dim * 4)));
    if (qt_cap < 1) return fail(EPS_ERR_UNSUPPORTED, "dimension too large for the brute-force row kernel");
    for (int64_t q0 = 0; q0 < nq; q0 += qt_cap) {
      int nt = static_cast<int>(std::min<int64_t>(qt_cap, nq - q0));
      size_t smem = static_cast<size_t>(nt) * dim * 4;
      int64_t groups = (n + 31) / 32;
      int blocks = static_cast<int>(std::min<int64_t>((groups + 7) / 8, static_cast<int64_t>(ix->num_sms) * 8));
      if (blocks < 1) blocks = 1;
      if (smem > 48 * 1024)
        EPS_CUDA(cudaFuncSetAttribute(kern.rows, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
      kern.rows<<<blocks, 256, smem, ix->stream>>>(A_base, dim, metric, row_start, n, d_queries + q0 * dim, nt,
                                                   D + q0 * ldd, ldd);
      ++*launches;
    }
  } else {
    dim3 grid(static_cast<unsigned>((n + kBM - 1) / kBM), static_cast<unsigned>((nq + kBN - 1) / kBN));
    kern.tile<<<grid, 256, 0, ix->stream>>>(A_base + row_start * ix->dim, n, d_queries, nq, dim, metric, D, ldd);
    ++*launches;
  }
  EPS_CUDA(cudaGetLastError());
  return EPS_OK;
}

static void fill_inf(Index* ix, unsigned long long* p, int64_t n, uint64_t* launches) {
  fill_keys_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, ix->stream>>>(p, n, kKeyInf);
  ++*launches;
}

// A filter whose root compares "@distance" is evaluated per candidate inside the select kernel, on the real distance
// (not in prefilter mode, where the reference feeds it distance 0); any other filter goes into the pass bitmap.
static bool filter_reads_distance(const ScanRequest& r) {
  return r.h_prog && r.h_prog->n > 0 && !r.prefilter && r.h_prog->root_uses_dist;
}

// Pass bitmap of rows [row_start, row_end): bit i set <=> row row_start + i is not deleted (when the request skips
// deleted rows) and passes the distance-free filter.  *d_pass stays null when neither applies.
static int pass_bitmap(Index* ix, const ScanRequest& r, uint32_t** d_pass, uint64_t* launches) {
  const bool deleted = r.skip_deleted && ix->any_deleted;
  const bool filter = r.h_prog && r.h_prog->n > 0 && !filter_reads_distance(r);
  *d_pass = nullptr;
  if (!deleted && !filter) return EPS_OK;
  const int64_t n = r.row_end - r.row_start, words = (n + 31) / 32;
  EPS_TRY(ix->s_pass.reserve(static_cast<size_t>(words) * 4));
  *d_pass = ix->s_pass.as<uint32_t>();
  pass_bitmap_kernel<<<static_cast<unsigned>((words + 127) / 128), 128, 0, ix->stream>>>(
      deleted ? ix->d_deleted.as<const uint8_t>() : nullptr, ix->deleted_bytes, filter ? r.d_prog : nullptr, ix->d_attrs, ix->attr_stride,
      r.row_start, n, *d_pass);
  ++*launches;
  return EPS_OK;
}

// What both paths set up after filling their lists: the pass bitmap, the rows per materialised distance tile (the
// [nq x chunk] fp32 scratch D stays under ~1 GiB) and bf_select_kernel's shared memory for lists of k keys.
struct ScanSetup { uint32_t* pass; int64_t chunk; float* D; size_t smem; };
static int scan_setup(Index* ix, const ScanRequest& r, int64_t k, ScanSetup* s, uint64_t* launches) {
  const int64_t n = r.row_end - r.row_start;
  EPS_TRY(pass_bitmap(ix, r, &s->pass, launches));
  s->chunk = std::max<int64_t>(kBM, (256ll * 1024 * 1024 / r.nq / kBM) * kBM);
  if (s->chunk > n) s->chunk = ((n + 3) / 4) * 4;
  EPS_TRY(ix->s_dist.reserve(static_cast<size_t>(r.nq) * s->chunk * 4));
  s->D = ix->s_dist.as<float>();
  s->smem = (2 * static_cast<size_t>(k) + kSelBuf) * 8;
  // The 48 KB launch default bounds the dynamic AND the kernel's static shared memory (about 1 KB): a list of k = 1984 to
  // 2048 keys fits 48 KB alone but not with it.  Setting the limit on every call needs no guess at the static size.
  EPS_CUDA(cudaFuncSetAttribute(bf_select_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(s->smem)));
  EPS_CUDA(cudaFuncSetAttribute(bf_select_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(s->smem)));
  return EPS_OK;
}

template <bool KEYS_IN>
static int run_select(Index* ix, const SelectArgs& a, int64_t nq, size_t smem, uint64_t* launches) {
  bf_select_kernel<KEYS_IN><<<dim3(static_cast<unsigned>(nq), a.nsplit), kSelThreads, smem, ix->stream>>>(a);
  ++*launches;
  EPS_CUDA(cudaGetLastError());
  return EPS_OK;
}

// fp32 SIMT scan: per chunk of rows, the [nq x chunk] distance tile and a streaming select per (query, row split);
// then the merge of the splits' lists.
static int fp32_scan(Index* ix, const ScanRequest& r, unsigned long long* d_topk, eps_stats* stats) {
  uint64_t launches = 0;
  const int64_t nq = r.nq, k = r.k, n = r.row_end - r.row_start;
  fill_inf(ix, d_topk, nq * k, &launches);
  if (n <= 0 || nq <= 0) {
    if (stats) stats->kernel_launches += launches;
    return EPS_OK;
  }
  ScanSetup s;
  EPS_TRY(scan_setup(ix, r, k, &s, &launches));
  // splits: enough CTAs to fill the machine; a split must be worth its extra merge launch (>= 16384 elements)
  const int64_t want = (2ll * ix->num_sms + nq - 1) / nq, maxs = std::max<int64_t>(1, s.chunk / 16384);
  const int nsplit = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(want, maxs), 64)));
  unsigned long long* state = d_topk;
  if (nsplit > 1) {
    EPS_TRY(ix->s_topk2.reserve(static_cast<size_t>(nq) * nsplit * k * 8));
    state = ix->s_topk2.as<unsigned long long>();
    fill_inf(ix, state, nq * nsplit * k, &launches);
  }
  SelectArgs a;
  a.D = s.D; a.ldd = s.chunk; a.nsplit = nsplit; a.k = static_cast<int>(k); a.state = state;
  a.pass = s.pass; a.pass_base = r.row_start; a.self_base = r.self_base;
  if (filter_reads_distance(r)) { a.dyn = r.d_prog; a.attrs = ix->d_attrs; a.attr_stride = ix->attr_stride; }
  // The L2 screen (SparseL2Screen, sparse_inverted.cu) selects K = k keys of the bound tile first, into its own lists
  // [nq x nsplit x k] (then merged into [nq x k]), followed by T [nq].  A filter that reads the distance would select
  // them by bounds: such a call takes the merge tile for every row.
  const SparseL2Screen* screen = filter_reads_distance(r) ? nullptr : r.l2_screen;
  SelectArgs b = a, bm;
  unsigned long long* b_merged = nullptr;
  float* T = nullptr;
  if (screen) {
    const size_t lists = static_cast<size_t>(nq) * nsplit * k, merged = nsplit > 1 ? static_cast<size_t>(nq) * k : 0;
    EPS_TRY(ix->s_l2_screen.reserve((lists + merged) * 8 + static_cast<size_t>(nq) * 4));
    b.state = ix->s_l2_screen.as<unsigned long long>();
    b_merged = nsplit > 1 ? b.state + lists : b.state;
    T = reinterpret_cast<float*>(b.state + lists + merged);
    bm.keys_in = b.state; bm.n = static_cast<int64_t>(nsplit) * k; bm.k = static_cast<int>(k); bm.state = b_merged;
  }
  for (int64_t c0 = 0; c0 < n; c0 += s.chunk) {
    a.row_base = r.row_start + c0;
    a.n = std::min(s.chunk, n - c0);
    if (screen) {
      EPS_TRY(screen->bounds(ix, a.row_base, a.n, s.D, s.chunk, &launches));
      b.row_base = a.row_base; b.n = a.n;
      fill_inf(ix, b.state, nq * nsplit * k, &launches);
      if (nsplit > 1) fill_inf(ix, b_merged, nq * k, &launches);
      EPS_TRY(run_select<false>(ix, b, nq, s.smem, &launches));
      if (nsplit > 1) EPS_TRY(run_select<true>(ix, bm, nq, s.smem, &launches));
      EPS_TRY(screen->threshold(ix, b_merged, static_cast<int>(k), T, &launches));
      EPS_TRY(screen->rescore(ix, a.row_base, a.n, s.D, s.chunk, T, s.pass, r.row_start, r.self_base, &launches));
    } else if (r.dist) {
      EPS_TRY(r.dist->launch(ix, r.metric, a.row_base, a.n, s.D, s.chunk, &launches));
    } else {
      EPS_TRY(launch_distances(ix, r.metric, ix->d_vectors, a.row_base, a.n, r.queries, nq, s.D, s.chunk, &launches));
    }
    EPS_TRY(run_select<false>(ix, a, nq, s.smem, &launches));
  }
  if (nsplit > 1) {
    SelectArgs m;
    m.keys_in = state; m.n = static_cast<int64_t>(nsplit) * k; m.k = static_cast<int>(k); m.state = d_topk;
    EPS_TRY(run_select<true>(ix, m, nq, s.smem, &launches));
  }
  if (stats) stats->n_dist += static_cast<uint64_t>(nq) * static_cast<uint64_t>(n);
  if (stats) stats->kernel_launches += launches;
  return EPS_OK;
}

// Status of a coarse attempt, in s_cand_cnt after the nq candidate counts; the kernels get pointers to its fields.
struct CoarseStatus {
  int overflow;       // a fused launch had more survivors than its candidate buffer holds
  int n_unsafe;       // queries the guard could not prove exact
  unsigned err_bits;  // largest |coarse - exact| of the re-scored rows (float bits)
  unsigned xn_bits;   // largest |x|^2 of the re-scored rows (float bits)
};

enum class Coarse { ok, overflow, boost, redo };

// One attempt of the tensor-core coarse pass (tc_dist.cu) on a batch, into d_topk: a boot chunk that materialises its
// distance tile and seeds each query's running threshold of the k' coarse candidates, fused launches that keep only
// the rows under the thresholds (no distance tile leaves the SM), the exact re-score of the k' candidates and the
// guard, with ONE host round trip for their verdict.  *unsafe lists the queries to redo when it is Coarse::redo.
static int coarse_attempt(Index* ix, const ScanRequest& r, unsigned long long* d_topk, eps_stats* stats, Coarse* verdict,
                          std::vector<int>* unsafe) {
  // developer knobs, read once
  static const int64_t env_kmin = [] { const char* e = getenv("EPS_SCAN_KMIN"); return e ? atoll(e) : 118ll; }();
  static const int64_t env_boot = [] { const char* e = getenv("EPS_SCAN_BOOT"); return e ? atoll(e) : 4096ll; }();
  static const int64_t env_grow = [] { const char* e = getenv("EPS_SCAN_GROW"); return e ? atoll(e) : 8ll; }();
  uint64_t launches = 0;
  const int64_t nq = r.nq, n = r.row_end - r.row_start;
  // k' coarse candidates per query: k + max(118, k) (128 for top-10), times the boost the guard has learnt
  const int64_t k = std::min<int64_t>(8192, (r.k + std::max<int64_t>(env_kmin, r.k)) * std::max(1, ix->coarse_boost));
  EPS_TRY(ix->s_coarse.reserve(static_cast<size_t>(nq) * k * 8));
  unsigned long long* coarse = ix->s_coarse.as<unsigned long long>();
  fill_inf(ix, coarse, nq * k, &launches);
  ScanSetup s;
  EPS_TRY(scan_setup(ix, r, k, &s, &launches));
  const int cand_cap = static_cast<int>(std::max<int64_t>(4096, 16 * k));  // fused launches grow 8x: ~8 k' survivors each
#ifdef EPS_GS_PROFILE
  // developer build: event after every launch of the tensor-core scan, printed as a timeline at the end
  std::vector<std::pair<std::string, cudaEvent_t>> tl;
  auto mark = [&](const std::string& name) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, ix->stream);
    tl.push_back({name, e});
  };
#define TL_MARK(x) mark(x)
#else
#define TL_MARK(x) do { } while (0)
#endif
  TL_MARK("start");
  EPS_TRY(ix->s_thr.reserve(static_cast<size_t>(nq) * 4));
  EPS_TRY(ix->s_cand.reserve(static_cast<size_t>(nq) * cand_cap * 8));
  EPS_TRY(ix->s_cand_cnt.reserve(static_cast<size_t>(nq) * 4 + sizeof(CoarseStatus)));
  CoarseStatus* d_status = reinterpret_cast<CoarseStatus*>(ix->s_cand_cnt.as<int>() + nq);
  EPS_CUDA(cudaMemsetAsync(d_status, 0, sizeof(CoarseStatus), ix->stream));
  // boot chunk: only 4 K rows pay the distance-tile round trip (16 MB tile, 4 M keys to select from)
  SelectArgs a;
  a.D = s.D; a.ldd = s.chunk; a.row_base = r.row_start; a.n = std::min(std::min(s.chunk, env_boot), n);
  a.k = static_cast<int>(k); a.state = coarse; a.pass = s.pass; a.pass_base = r.row_start;
  a.thr_out = ix->s_thr.as<float>();
  EPS_TRY(tc_launch_distances(ix, r.metric, r.row_start, a.n, r.queries, nq, s.D, s.chunk, &launches));
  TL_MARK("dist tile " + std::to_string(a.n));
  EPS_TRY(run_select<false>(ix, a, nq, s.smem, &launches));
  TL_MARK("select");
  // fused launches grow 8x at a time as the thresholds tighten: expected survivors per query of a launch
  // ~ k' * rows_in_launch / rows_seen_so_far = 8 k' << candidate capacity
  TcFused f;
  f.thr = ix->s_thr.as<float>(); f.cand = ix->s_cand.as<unsigned long long>(); f.cand_cnt = ix->s_cand_cnt.as<int>();
  f.pass = s.pass; f.pass_base = r.row_start; f.cand_cap = cand_cap;
  SelectArgs m;
  m.keys_in = f.cand; m.n = cand_cap; m.k = static_cast<int>(k); m.state = coarse; m.counts = f.cand_cnt;
  m.thr_out = ix->s_thr.as<float>(); m.overflow = &d_status->overflow;
  for (int64_t c0 = a.n; c0 < n;) {
    const int64_t cn = std::min(std::min<int64_t>(env_grow * c0, 4 * 1024 * 1024), n - c0);
    EPS_CUDA(cudaMemsetAsync(f.cand_cnt, 0, static_cast<size_t>(nq) * 4, ix->stream));
    TL_MARK("memset");
    EPS_TRY(tc_launch_distances(ix, r.metric, r.row_start + c0, cn, r.queries, nq, nullptr, 0, &launches, &f));
    TL_MARK("fused " + std::to_string(cn));
    EPS_TRY(run_select<true>(ix, m, nq, s.smem, &launches));
    TL_MARK("merge");
    c0 += cn;
  }
  const int kc = static_cast<int>(k), kcp = next_pow2(kc);
  const size_t rs_smem = static_cast<size_t>(kcp) * 8 + static_cast<size_t>((ix->dim + 3) & ~3ll) * 4;
  if (rs_smem > 48 * 1024)
    EPS_CUDA(cudaFuncSetAttribute(rescore_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(rs_smem)));
  rescore_kernel<<<static_cast<unsigned>(nq), 128, rs_smem, ix->stream>>>(
      ix->d_vectors, static_cast<int>(ix->dim), r.metric, ix->vec4 ? 1 : 0, r.queries, coarse, kc, kcp,
      static_cast<int>(r.k), d_topk, &d_status->err_bits, ix->s_xnorm.as<float>(), &d_status->xn_bits);
  EPS_CUDA(cudaGetLastError());
  ++launches;
  std::vector<int> h_flags;
  const bool guard = ix->coarse_guard != 0;
  if (guard) {
    EPS_TRY(ix->s_flags.reserve(static_cast<size_t>(nq) * 4));
    verify_exact_kernel<<<static_cast<unsigned>((nq + 127) / 128), 128, 0, ix->stream>>>(
        d_topk, static_cast<int>(r.k), ix->s_thr.as<float>(), &d_status->err_bits, ix->s_xnorm_max.as<unsigned>(),
        &d_status->xn_bits, static_cast<int>(nq), ix->s_flags.as<int>(), &d_status->n_unsafe);
    EPS_CUDA(cudaGetLastError());
    ++launches;
    h_flags.resize(static_cast<size_t>(nq));
    EPS_CUDA(cudaMemcpyAsync(h_flags.data(), ix->s_flags.p, static_cast<size_t>(nq) * 4, cudaMemcpyDeviceToHost, ix->stream));
  }
  // candidate-buffer overflow (adversarial row order: the buffers are sized for the expected survivors) and the
  // guard's verdict
  TL_MARK("rescore+verify");
  CoarseStatus h_status;
  EPS_CUDA(cudaMemcpyAsync(&h_status, d_status, sizeof(h_status), cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
#ifdef EPS_GS_PROFILE
  if (tl.size() > 1 && n >= 1000000) {
    fprintf(stderr, "[scan-timeline]");
    for (size_t i = 1; i < tl.size(); ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, tl[i - 1].second, tl[i].second);
      fprintf(stderr, " %s %.3f |", tl[i].first.c_str(), ms);
    }
    float tot = 0.f;
    cudaEventElapsedTime(&tot, tl.front().second, tl.back().second);
    fprintf(stderr, " total %.3f ms\n", tot);
  }
  for (auto& t : tl) cudaEventDestroy(t.second);
#endif
  if (stats) stats->kernel_launches += launches;
  if (h_status.overflow) *verdict = Coarse::overflow;
  else if (!guard || h_status.n_unsafe == 0) *verdict = Coarse::ok;
  else if (h_status.n_unsafe > std::max<int64_t>(8, nq / 32) && k < 4096) *verdict = Coarse::boost;
  else *verdict = Coarse::redo;
  if (*verdict == Coarse::redo)
    for (int64_t q = 0; q < nq; ++q) if (h_flags[q]) unsafe->push_back(static_cast<int>(q));
  return EPS_OK;
}

// Exact fp32 scan of the queries idx of a coarse attempt, written over their rows of d_topk.  It reuses the fp32
// scan's scratch, none of the coarse pass's.  Its own launches are not counted; the gather and the scatter are.
static int redo_queries(Index* ix, const ScanRequest& r, const std::vector<int>& idx, unsigned long long* d_topk,
                        eps_stats* stats) {
  const int nb = static_cast<int>(idx.size());
  DevBuf d_idx, d_q, d_res;
  EPS_TRY(d_idx.reserve(idx.size() * 4));
  EPS_TRY(d_q.reserve(idx.size() * ix->dim * 4));
  EPS_TRY(d_res.reserve(idx.size() * r.k * 8));
  EPS_CUDA(cudaMemcpyAsync(d_idx.p, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, ix->stream));
  const int64_t tot = static_cast<int64_t>(nb) * ix->dim;
  gather_queries_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, ix->stream>>>(
      r.queries, d_idx.as<int>(), nb, static_cast<int>(ix->dim), d_q.as<float>());
  EPS_CUDA(cudaGetLastError());
  ScanRequest sub = r;
  sub.queries = d_q.as<float>();
  sub.nq = nb;
  EPS_TRY(fp32_scan(ix, sub, d_res.as<unsigned long long>(), nullptr));
  const int64_t tk = static_cast<int64_t>(nb) * r.k;
  scatter_keys_kernel<<<static_cast<unsigned>((tk + 255) / 256), 256, 0, ix->stream>>>(
      d_res.as<unsigned long long>(), d_idx.as<int>(), nb, static_cast<int>(r.k), d_topk);
  EPS_CUDA(cudaGetLastError());
  EPS_CUDA(cudaStreamSynchronize(ix->stream));  // the temporaries die with this frame
  if (stats) { stats->n_redone += static_cast<uint64_t>(nb); stats->kernel_launches += 2; }
  return EPS_OK;
}

// One batch: the tensor-core coarse pass and exact re-score where it applies, until its guard accepts; the fp32 scan
// otherwise.
static int scan_batch(Index* ix, const ScanRequest& r, unsigned long long* d_topk, eps_stats* stats) {
  if (r.k < 1 || r.k > 8192) return fail(EPS_ERR_UNSUPPORTED, "brute-force top-k supports 1 <= k <= 8192");
  const int64_t n = r.row_end - r.row_start;
  // The coarse pass takes large dense batches, except with a filter that reads the real distance (the select needs exact
  // values) and for queries that are rows of the table (the build's kNN lists, or a device batch that aliases it).
  const bool queries_alias_table = r.queries == ix->d_vectors;
  bool coarse = !r.dist && n >= 4096 && r.self_base < 0 && !filter_reads_distance(r) && tc_dist_usable(ix, r.nq) &&
                !queries_alias_table;
  while (coarse) {
    Coarse verdict;
    std::vector<int> unsafe;
    EPS_TRY(coarse_attempt(ix, r, d_topk, stats, &verdict, &unsafe));
    switch (verdict) {
      case Coarse::overflow:  // never silently truncated: the batch again on the fp32 path
        coarse = false;
        break;
      case Coarse::boost:  // too many unsafe queries for this table's distance spread: the batch again, with a 4x larger k'
        ix->coarse_boost = std::min(64, std::max(1, ix->coarse_boost) * 4);
        break;
      case Coarse::redo:  // a few unsafe queries: exact fp32 scan for those only
        EPS_TRY(redo_queries(ix, r, unsafe, d_topk, stats));
        [[fallthrough]];
      case Coarse::ok:
        if (stats) stats->n_dist += static_cast<uint64_t>(r.nq) * static_cast<uint64_t>(n);
        return EPS_OK;
    }
    if (stats) stats->n_redone += static_cast<uint64_t>(r.nq);
  }
  return fp32_scan(ix, r, d_topk, stats);
}

int exact_topk(Index* ix, const ScanRequest& r, unsigned long long* d_topk, eps_stats* stats) {
  // The tensor-core pass keeps its per-query constants in a 1024-entry shared-memory table: larger dense batches
  // (config C3: B = 4096) go through it in groups of 1024 queries.
  if (r.queries && r.self_base < 0 && r.nq > 1024 && r.row_end - r.row_start >= 4096 && tc_dist_usable(ix, 1024)) {
    ScanRequest g = r;
    for (int64_t q0 = 0; q0 < r.nq; q0 += 1024) {
      g.queries = r.queries + q0 * ix->dim;
      g.nq = std::min<int64_t>(1024, r.nq - q0);
      EPS_TRY(scan_batch(ix, g, d_topk + q0 * r.k, stats));
    }
    return EPS_OK;
  }
  return scan_batch(ix, r, d_topk, stats);
}

// ------------------------------------------------------------------------------------------------
// Collect mode of a filtered graph search (capi.cu): the pass bitmap of every row and its popcount P, then the exact
// top-k over the passing rows alone.  The bitmap is compacted into an ascending id list by two launches (counts per
// CTA span, then each CTA writes its ids after the counts of the spans before it).
// ------------------------------------------------------------------------------------------------
constexpr int kCompactThreads = 256, kCompactWords = 4;
constexpr int kCompactSpan = kCompactThreads * kCompactWords;  // bitmap words per CTA

__device__ __forceinline__ int span_count(const uint32_t* __restrict__ pass, int64_t words, int64_t w0) {
  int c = 0;
#pragma unroll
  for (int j = 0; j < kCompactWords; ++j)
    if (w0 + j < words) c += __popc(pass[w0 + j]);
  return c;
}

__global__ void __launch_bounds__(kCompactThreads) pass_count_kernel(const uint32_t* __restrict__ pass, int64_t words,
                                                                     int* __restrict__ counts, unsigned long long* __restrict__ total) {
  __shared__ int s_sum;
  if (threadIdx.x == 0) s_sum = 0;
  __syncthreads();
  const int c = span_count(pass, words, static_cast<int64_t>(blockIdx.x) * kCompactSpan + threadIdx.x * kCompactWords);
  if (c) atomicAdd(&s_sum, c);
  __syncthreads();
  if (threadIdx.x == 0) {
    counts[blockIdx.x] = s_sum;
    if (s_sum) atomicAdd(total, static_cast<unsigned long long>(s_sum));
  }
}

__global__ void __launch_bounds__(kCompactThreads) pass_compact_kernel(const uint32_t* __restrict__ pass, int64_t words,
                                                                       const int* __restrict__ counts, int32_t* __restrict__ ids) {
  __shared__ int s_base, s_warp[kCompactThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_base = 0;
  __syncthreads();
  int before = 0;
  for (unsigned b = tid; b < blockIdx.x; b += kCompactThreads) before += counts[b];
  if (before) atomicAdd(&s_base, before);
  const int64_t w0 = static_cast<int64_t>(blockIdx.x) * kCompactSpan + tid * kCompactWords;
  const int c = span_count(pass, words, w0);
  int x = c;  // inclusive scan of the thread counts: warp, then the warp totals
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(kFull, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  int o = s_base + x - c;
  for (int w = 0; w < warp; ++w) o += s_warp[w];
#pragma unroll
  for (int j = 0; j < kCompactWords; ++j) {
    if (w0 + j >= words) break;
    uint32_t bits = pass[w0 + j];
    while (bits) {
      ids[o++] = static_cast<int32_t>((w0 + j) * 32 + __ffs(bits) - 1);
      bits &= bits - 1;
    }
  }
}

// key (distance, list index) -> (distance, row id): the list is ascending, so the (distance, id) order is unchanged
__global__ void list_to_row_keys_kernel(unsigned long long* __restrict__ keys, int64_t n, const int32_t* __restrict__ ids) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  if ((k & kKeyMask) != kKeyInf) keys[i] = (k & 0xffffffff00000000ull) | static_cast<uint32_t>(ids[key_id(k)]);
}

int collect_pass(Index* ix, const ScanRequest& r, int64_t* P, uint64_t* launches) {
  const int64_t n = r.row_end, words = (n + 31) / 32, spans = std::max<int64_t>(1, (words + kCompactSpan - 1) / kCompactSpan);
  EPS_TRY(ix->s_cpass.reserve(static_cast<size_t>(words) * 4));
  EPS_TRY(ix->s_ccount.reserve(8 + static_cast<size_t>(spans) * 4));
  unsigned long long* d_total = ix->s_ccount.as<unsigned long long>();
  EPS_CUDA(cudaMemsetAsync(d_total, 0, 8, ix->stream));
  if (words > 0) {
    pass_bitmap_kernel<<<static_cast<unsigned>((words + 127) / 128), 128, 0, ix->stream>>>(
        ix->any_deleted ? ix->d_deleted.as<const uint8_t>() : nullptr, ix->deleted_bytes, r.d_prog, ix->d_attrs, ix->attr_stride, 0, n,
        ix->s_cpass.as<uint32_t>());
    pass_count_kernel<<<static_cast<unsigned>(spans), kCompactThreads, 0, ix->stream>>>(
        ix->s_cpass.as<uint32_t>(), words, reinterpret_cast<int*>(d_total + 1), d_total);
    EPS_CUDA(cudaGetLastError());
    *launches += 2;
  }
  unsigned long long h = 0;
  EPS_CUDA(cudaMemcpyAsync(&h, d_total, 8, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  *P = static_cast<int64_t>(h);
  return EPS_OK;
}

// The distance tile of list entries [row_start, row_start + n): the listed rows are gathered into ix->s_gather in
// pieces of at most 64 MB and scanned by the fp32 kernel that a batch of form_nq queries takes.
struct PassingRowsDist : DistProducer {
  const int32_t* ids;
  const float* queries;
  int64_t nq, form_nq;
  int launch(Index* ix, int metric, int64_t row_start, int64_t n, float* D, int64_t ldd, uint64_t* launches) const override {
    const int64_t piece = std::min(n, std::max<int64_t>(kBM, (64ll << 20) / (ix->dim * 4) / kBM * kBM));
    EPS_TRY(ix->s_gather.reserve(static_cast<size_t>(piece) * ix->dim * 4));
    for (int64_t s0 = 0; s0 < n; s0 += piece) {
      const int64_t sn = std::min(piece, n - s0);
      EPS_TRY(gather_rows(ix, ids + row_start + s0, sn, ix->s_gather.as<float>()));
      ++*launches;
      EPS_TRY(launch_distances(ix, metric, ix->s_gather.as<float>(), 0, sn, queries, nq, D + s0, ldd, launches, form_nq));
    }
    return EPS_OK;
  }
};

int passing_topk(Index* ix, const float* queries, int64_t nq, const int* d_idx, int64_t nb, int64_t k, int64_t P,
                 unsigned long long* d_topk, eps_stats* stats) {
  uint64_t launches = 0;
  const int64_t words = (ix->n_rows + 31) / 32, spans = (words + kCompactSpan - 1) / kCompactSpan;
  EPS_TRY(ix->s_cids.reserve(static_cast<size_t>(P) * 4));
  if (P > 0) {
    pass_compact_kernel<<<static_cast<unsigned>(spans), kCompactThreads, 0, ix->stream>>>(
        ix->s_cpass.as<uint32_t>(), words, reinterpret_cast<const int*>(ix->s_ccount.as<unsigned long long>() + 1), ix->s_cids.as<int32_t>());
    EPS_CUDA(cudaGetLastError());
    ++launches;
  }
  DevBuf d_q, d_res;
  const float* q = queries;
  unsigned long long* res = d_topk;
  if (d_idx) {  // the picked queries, and their lists scattered back below
    EPS_TRY(d_q.reserve(static_cast<size_t>(nb) * ix->dim * 4));
    EPS_TRY(d_res.reserve(static_cast<size_t>(nb) * k * 8));
    const int64_t tot = nb * ix->dim;
    gather_queries_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, ix->stream>>>(queries, d_idx, static_cast<int>(nb),
                                                                                          static_cast<int>(ix->dim), d_q.as<float>());
    EPS_CUDA(cudaGetLastError());
    ++launches;
    q = d_q.as<float>();
    res = d_res.as<unsigned long long>();
  }
  PassingRowsDist dist;
  dist.ids = ix->s_cids.as<int32_t>(); dist.queries = q; dist.nq = nb; dist.form_nq = nq;
  ScanRequest s;
  s.dist = &dist; s.nq = nb; s.row_start = 0; s.row_end = P; s.k = k; s.metric = ix->metric; s.skip_deleted = false;
  EPS_TRY(fp32_scan(ix, s, res, stats));
  const int64_t tk = nb * k;
  list_to_row_keys_kernel<<<static_cast<unsigned>((tk + 255) / 256), 256, 0, ix->stream>>>(res, tk, ix->s_cids.as<int32_t>());
  EPS_CUDA(cudaGetLastError());
  ++launches;
  if (d_idx) {
    scatter_keys_kernel<<<static_cast<unsigned>((tk + 255) / 256), 256, 0, ix->stream>>>(res, d_idx, static_cast<int>(nb),
                                                                                       static_cast<int>(k), d_topk);
    EPS_CUDA(cudaGetLastError());
    ++launches;
    EPS_CUDA(cudaStreamSynchronize(ix->stream));  // the temporaries die with this frame
  }
  if (stats) stats->kernel_launches += launches;
  return EPS_OK;
}

}  // namespace eps
