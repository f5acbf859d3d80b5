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
  const float* D;            // [nq x ldd] distances of this chunk (KEYS_IN = false)
  const unsigned long long* keys_in;  // [nq x n_in] candidate keys (KEYS_IN = true)
  int64_t ldd;
  int64_t n;                 // elements per query in this chunk
  int64_t row_base;          // global row id of element 0
  int nsplit;
  int k;
  unsigned long long* state; // [nq x nsplit x k]
  const uint32_t* pass;      // bitmap relative to pass_base (may be null)
  int64_t pass_base;
  const FilterProg* dyn;     // per-candidate filter that needs the real distance (may be null)
  const char* attrs;
  int64_t attr_stride;
  int64_t self_base;         // query q is row self_base + q and is excluded (-1: off)
  const int* counts;         // KEYS_IN: valid keys per query (<= n), null = n
  float* thr_out;            // if set: distance of the k-th entry after this pass (running threshold)
  int* overflow;             // if set: raised when counts[q] > n (candidates were dropped)
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
int launch_distances(Index* ix, const float* A_base, int64_t row_start, int64_t n, const float* d_queries,
                     int64_t nq, float* D, int64_t ldd, uint64_t* launches) {
  const int dim = static_cast<int>(ix->dim);
  const bool l2 = ix->metric == EPS_METRIC_L2;
  if (nq <= 16) {
    int qt_cap = static_cast<int>(std::min<int64_t>(kRowsQT, (200 * 1024) / (ix->dim * 4)));
    if (qt_cap < 1) return fail(EPS_ERR_UNSUPPORTED, "dimension too large for the brute-force row kernel");
    for (int64_t q0 = 0; q0 < nq; q0 += qt_cap) {
      int nt = static_cast<int>(std::min<int64_t>(qt_cap, nq - q0));
      size_t smem = static_cast<size_t>(nt) * dim * 4;
      int64_t groups = (n + 31) / 32;
      int blocks = static_cast<int>(std::min<int64_t>((groups + 7) / 8, static_cast<int64_t>(ix->num_sms) * 8));
      if (blocks < 1) blocks = 1;
#define LAUNCH_ROWS(L2_, V4_)                                                                                   \
  do {                                                                                                          \
    if (smem > 48 * 1024)                                                                                       \
      EPS_CUDA(cudaFuncSetAttribute(bf_dist_rows_kernel<L2_, V4_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                    static_cast<int>(smem)));                                                   \
    bf_dist_rows_kernel<L2_, V4_><<<blocks, 256, smem, ix->stream>>>(A_base, dim, ix->metric, row_start, n,     \
                                                                     d_queries + q0 * dim, nt, D + q0 * ldd, ldd); \
  } while (0)
      if (l2) { if (ix->vec4) LAUNCH_ROWS(true, true); else LAUNCH_ROWS(true, false); }
      else { if (ix->vec4) LAUNCH_ROWS(false, true); else LAUNCH_ROWS(false, false); }
#undef LAUNCH_ROWS
      ++*launches;
    }
  } else {
    dim3 grid(static_cast<unsigned>((n + kBM - 1) / kBM), static_cast<unsigned>((nq + kBN - 1) / kBN));
    const float* A = A_base + row_start * ix->dim;
    if (l2) {
      if (ix->vec4) bf_dist_tile_kernel<true, true><<<grid, 256, 0, ix->stream>>>(A, n, d_queries, nq, dim, ix->metric, D, ldd);
      else bf_dist_tile_kernel<true, false><<<grid, 256, 0, ix->stream>>>(A, n, d_queries, nq, dim, ix->metric, D, ldd);
    } else {
      if (ix->vec4) bf_dist_tile_kernel<false, true><<<grid, 256, 0, ix->stream>>>(A, n, d_queries, nq, dim, ix->metric, D, ldd);
      else bf_dist_tile_kernel<false, false><<<grid, 256, 0, ix->stream>>>(A, n, d_queries, nq, dim, ix->metric, D, ldd);
    }
    ++*launches;
  }
  EPS_CUDA(cudaGetLastError());
  return EPS_OK;
}

static int topk_impl(Index* ix, const float* d_queries, int64_t nq, int64_t row_start, int64_t row_end, int64_t k,
                     const FilterProg* d_prog, const FilterProg* h_prog, bool prefilter, int64_t self_base,
                     unsigned long long* d_topk, eps_stats* stats, bool allow_tc = true,
                     const DistProducer* producer = nullptr) {
  // never-shrinking scratch owned by the index would be overwritten by the nested fp32 redo of unsafe queries
  // (that redo never takes the tensor-core branch, so it uses none of the coarse-pass buffers)
  if (k < 1 || k > 8192) return fail(EPS_ERR_UNSUPPORTED, "brute-force top-k supports 1 <= k <= 8192");
  uint64_t launches = 0;
  const int64_t n = row_end - row_start;
  // Tensor-core coarse pass + exact re-score (tc_dist.cu) for large batches; a filter that reads the real
  // distance needs exact values inside the select and stays on the fp32 SIMT path.
  const bool dyn_filter = h_prog && h_prog->n > 0 && !prefilter && h_prog->root_uses_dist;
  const int64_t k_final = k;
  unsigned long long* d_final = d_topk;
  const bool use_tc = !producer && allow_tc && n >= 4096 && self_base < 0 && !dyn_filter && tc_dist_usable(ix, nq) && d_queries != ix->d_vectors;
  if (use_tc) {
    // k' coarse candidates per query: k + max(118, k) (128 for top-10), times the boost the guard has learnt
    static const int64_t env_kmin = [] { const char* e = getenv("EPS_SCAN_KMIN"); return e ? atoll(e) : 118ll; }();  // developer knob
    k = std::min<int64_t>(8192, (k_final + std::max<int64_t>(env_kmin, k_final)) * std::max(1, ix->coarse_boost));
    EPS_TRY(ix->s_coarse.reserve(static_cast<size_t>(nq) * k * 8));
    d_topk = ix->s_coarse.as<unsigned long long>();
  }
  {
    int64_t tot = nq * k;
    fill_keys_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, ix->stream>>>(d_topk, tot, kKeyInf);
    ++launches;
  }
  if (n <= 0 || nq <= 0) {
    if (stats) stats->kernel_launches += launches;
    return EPS_OK;
  }
  // static pass bitmap (deleted + distance-free filter); a filter whose root compares "@distance"
  // (and we are not in prefilter mode, where the reference feeds it distance 0) is evaluated per
  // candidate inside the select kernel instead.
  const bool has_prog = h_prog && h_prog->n > 0;
  const bool dynamic = has_prog && !prefilter && h_prog->root_uses_dist;
  const bool need_pass = ix->any_deleted || (has_prog && !dynamic);
  uint32_t* d_pass = nullptr;
  if (need_pass) {
    int64_t words = (n + 31) / 32;
    EPS_TRY(ix->s_pass.reserve(static_cast<size_t>(words) * 4));
    d_pass = ix->s_pass.as<uint32_t>();
    pass_bitmap_kernel<<<static_cast<unsigned>((words + 127) / 128), 128, 0, ix->stream>>>(
        ix->any_deleted ? ix->d_deleted : nullptr, ix->deleted_bytes, (has_prog && !dynamic) ? d_prog : nullptr,
        ix->d_attrs, ix->attr_stride, row_start, n, d_pass);
    ++launches;
  }
  // chunking: distance scratch <= ~1 GiB
  const int64_t scratch_floats = 256ll * 1024 * 1024;
  int64_t chunk = scratch_floats / nq;
  chunk = std::max<int64_t>(kBM, (chunk / kBM) * kBM);
  if (chunk > n) chunk = ((n + 3) / 4) * 4;
  EPS_TRY(ix->s_dist.reserve(static_cast<size_t>(nq) * chunk * 4));
  float* D = ix->s_dist.as<float>();
  // splits: enough CTAs to fill the machine, each >= 16384 elements
  int nsplit = 1;
  {
    int64_t want = (2ll * ix->num_sms + nq - 1) / nq;
    int64_t maxs = std::max<int64_t>(1, chunk / 16384);  // a split must be worth its extra merge launch
    nsplit = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(want, maxs), 64)));
    if (use_tc) nsplit = 1;  // the running threshold is read from the single per-query state
  }
  unsigned long long* state = d_topk;
  if (nsplit > 1) {
    EPS_TRY(ix->s_topk2.reserve(static_cast<size_t>(nq) * nsplit * k * 8));
    state = ix->s_topk2.as<unsigned long long>();
    int64_t tot = nq * nsplit * k;
    fill_keys_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, ix->stream>>>(state, tot, kKeyInf);
    ++launches;
  }
  const size_t sel_smem = (2 * static_cast<size_t>(k) + kSelBuf) * 8;
  if (sel_smem > 48 * 1024) {
    EPS_CUDA(cudaFuncSetAttribute(bf_select_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sel_smem)));
    EPS_CUDA(cudaFuncSetAttribute(bf_select_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sel_smem)));
  }
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
  int* d_overflow = nullptr;
  if (use_tc) {
    EPS_TRY(ix->s_thr.reserve(static_cast<size_t>(nq) * 4));
    EPS_TRY(ix->s_cand.reserve(static_cast<size_t>(nq) * cand_cap * 8));
    EPS_TRY(ix->s_cand_cnt.reserve(static_cast<size_t>(nq + 4) * 4));
    d_overflow = ix->s_cand_cnt.as<int>() + nq;  // [overflow, n_flagged, err_max bits, sample's max |x|^2 bits]
    EPS_CUDA(cudaMemsetAsync(d_overflow, 0, 16, ix->stream));
  }
  for (int64_t c0 = 0; c0 < n;) {
    // Chunk 0 (and every chunk of the SIMT path) materialises the [nq x chunk] distance tile and selects from
    // it; it also seeds the per-query running threshold.  Later tensor-core chunks filter against that
    // threshold inside the epilogue (no distance tile leaves the SM) and only the few survivors are merged.
    const bool fused = use_tc && c0 > 0;
    // tensor-core mode: a first chunk of only 4 K rows pays the distance-tile round trip (16 MB tile, 4 M keys to
    // select from), then fused launches grow 8x at a time as the thresholds tighten: expected survivors per query
    // of a launch ~ k' * rows_in_launch / rows_seen_so_far = 8 k' << candidate capacity
    int64_t want_rows = chunk;
    static const int64_t env_boot = [] { const char* e = getenv("EPS_SCAN_BOOT"); return e ? atoll(e) : 4096ll; }();   // developer knobs,
    static const int64_t env_grow = [] { const char* e = getenv("EPS_SCAN_GROW"); return e ? atoll(e) : 8ll; }();      // read once
    if (use_tc) want_rows = fused ? std::min<int64_t>(env_grow * c0, 4 * 1024 * 1024) : std::min<int64_t>(chunk, env_boot);
    const int64_t cn = std::min(want_rows, n - c0);
    SelectArgs a;
    a.ldd = chunk; a.row_base = row_start + c0; a.nsplit = nsplit; a.k = static_cast<int>(k); a.state = state;
    a.pass = d_pass; a.pass_base = row_start; a.dyn = dynamic ? d_prog : nullptr; a.attrs = ix->d_attrs;
    a.attr_stride = ix->attr_stride; a.self_base = self_base; a.counts = nullptr; a.overflow = nullptr;
    a.thr_out = use_tc ? ix->s_thr.as<float>() : nullptr;
    if (!fused) {
      if (use_tc) EPS_TRY(tc_launch_distances(ix, row_start + c0, cn, d_queries, nq, D, chunk, &launches));
      else if (producer) EPS_TRY(producer->launch(ix, row_start + c0, cn, D, chunk, &launches));
      else EPS_TRY(launch_distances(ix, ix->d_vectors, row_start + c0, cn, d_queries, nq, D, chunk, &launches));
      a.D = D; a.keys_in = nullptr; a.n = cn;
      TL_MARK("dist tile " + std::to_string(cn));
      bf_select_kernel<false><<<dim3(static_cast<unsigned>(nq), nsplit), kSelThreads, sel_smem, ix->stream>>>(a);
      TL_MARK("select");
    } else {
      EPS_CUDA(cudaMemsetAsync(ix->s_cand_cnt.p, 0, static_cast<size_t>(nq) * 4, ix->stream));
      TcFused f;
      f.thr = ix->s_thr.as<float>(); f.cand = ix->s_cand.as<unsigned long long>(); f.cand_cnt = ix->s_cand_cnt.as<int>();
      f.pass = d_pass; f.pass_base = row_start; f.cand_cap = cand_cap;
      TL_MARK("memset");
      EPS_TRY(tc_launch_distances(ix, row_start + c0, cn, d_queries, nq, nullptr, 0, &launches, &f));
      TL_MARK("fused " + std::to_string(cn));
      a.D = nullptr; a.keys_in = f.cand; a.n = cand_cap; a.counts = f.cand_cnt; a.overflow = d_overflow;
      a.pass = nullptr; a.dyn = nullptr;
      bf_select_kernel<true><<<dim3(static_cast<unsigned>(nq), 1), kSelThreads, sel_smem, ix->stream>>>(a);
      TL_MARK("merge");
    }
    ++launches;
    EPS_CUDA(cudaGetLastError());
    c0 += cn;
  }
  if (use_tc) {
    const int kc = static_cast<int>(k), kcp = next_pow2(kc);
    const size_t rs_smem = static_cast<size_t>(kcp) * 8 + static_cast<size_t>((ix->dim + 3) & ~3ll) * 4;
    if (rs_smem > 48 * 1024)
      EPS_CUDA(cudaFuncSetAttribute(rescore_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(rs_smem)));
    unsigned* d_err = reinterpret_cast<unsigned*>(d_overflow + 2);
    rescore_kernel<<<static_cast<unsigned>(nq), 128, rs_smem, ix->stream>>>(ix->d_vectors, static_cast<int>(ix->dim), ix->metric,
                                                                          ix->vec4 ? 1 : 0, d_queries, d_topk, kc, kcp,
                                                                          static_cast<int>(k_final), d_final, d_err,
                                                                          ix->s_xnorm.as<float>(), d_err + 1);
    EPS_CUDA(cudaGetLastError());
    ++launches;
    std::vector<int> h_flags;
    int h_state[2] = {0, 0};  // overflow, n_flagged
    const bool guard = ix->coarse_guard != 0;
    if (guard) {
      EPS_TRY(ix->s_flags.reserve(static_cast<size_t>(nq) * 4));
      verify_exact_kernel<<<static_cast<unsigned>((nq + 127) / 128), 128, 0, ix->stream>>>(
          d_final, static_cast<int>(k_final), ix->s_thr.as<float>(), d_err, ix->s_xnorm_max.as<unsigned>(), d_err + 1,
          static_cast<int>(nq), ix->s_flags.as<int>(), d_overflow + 1);
      EPS_CUDA(cudaGetLastError());
      ++launches;
      h_flags.resize(static_cast<size_t>(nq));
      EPS_CUDA(cudaMemcpyAsync(h_flags.data(), ix->s_flags.p, static_cast<size_t>(nq) * 4, cudaMemcpyDeviceToHost, ix->stream));
    }
    // ONE host round trip per tensor-core scan: candidate-buffer overflow (adversarial row order: the buffers are
    // sized for the expected survivors) and the guard's verdict
    TL_MARK("rescore+verify");
    EPS_CUDA(cudaMemcpyAsync(h_state, d_overflow, 8, cudaMemcpyDeviceToHost, ix->stream));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
#ifdef EPS_GS_PROFILE
    if (use_tc && tl.size() > 1 && n >= 1000000) {
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
    if (h_state[0]) {  // never silently truncated: the call is redone on the fp32 path
      if (stats) stats->n_redone += static_cast<uint64_t>(nq);
      return topk_impl(ix, d_queries, nq, row_start, row_end, k_final, d_prog, h_prog, prefilter, self_base, d_final, stats, false);
    }
    if (guard && h_state[1] > 0) {
      const int64_t n_bad = h_state[1];
      if (n_bad > std::max<int64_t>(8, nq / 32) && k < 4096) {
        // too many unsafe queries for this table's distance spread: remember a 4x larger k' and redo the batch
        ix->coarse_boost = std::min(64, std::max(1, ix->coarse_boost) * 4);
        if (stats) stats->n_redone += static_cast<uint64_t>(nq);
        return topk_impl(ix, d_queries, nq, row_start, row_end, k_final, d_prog, h_prog, prefilter, self_base, d_final, stats, true);
      }
      // a few unsafe queries: exact fp32 scan for those only
      std::vector<int> idx;
      for (int64_t q = 0; q < nq; ++q) if (h_flags[q]) idx.push_back(static_cast<int>(q));
      DevBuf d_idx, d_q, d_res;
      EPS_TRY(d_idx.reserve(idx.size() * 4));
      EPS_TRY(d_q.reserve(idx.size() * ix->dim * 4));
      EPS_TRY(d_res.reserve(idx.size() * k_final * 8));
      EPS_CUDA(cudaMemcpyAsync(d_idx.p, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, ix->stream));
      const int64_t tot = static_cast<int64_t>(idx.size()) * ix->dim;
      gather_queries_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, ix->stream>>>(d_queries, d_idx.as<int>(), static_cast<int>(idx.size()),
                                                                                             static_cast<int>(ix->dim), d_q.as<float>());
      EPS_CUDA(cudaGetLastError());
      EPS_TRY(topk_impl(ix, d_q.as<float>(), static_cast<int64_t>(idx.size()), row_start, row_end, k_final, d_prog, h_prog, prefilter, -1,
                        d_res.as<unsigned long long>(), nullptr, false));
      const int64_t tk = static_cast<int64_t>(idx.size()) * k_final;
      scatter_keys_kernel<<<static_cast<unsigned>((tk + 255) / 256), 256, 0, ix->stream>>>(d_res.as<unsigned long long>(), d_idx.as<int>(),
                                                                                           static_cast<int>(idx.size()), static_cast<int>(k_final), d_final);
      EPS_CUDA(cudaGetLastError());
      EPS_CUDA(cudaStreamSynchronize(ix->stream));  // the temporaries die with this frame
      if (stats) { stats->n_redone += static_cast<uint64_t>(idx.size()); stats->kernel_launches += 2; }
    }
    if (stats) stats->n_dist += static_cast<uint64_t>(nq) * static_cast<uint64_t>(n);
    return EPS_OK;
  }
  if (nsplit > 1) {
    SelectArgs a;
    a.D = nullptr; a.keys_in = state; a.ldd = 0; a.n = static_cast<int64_t>(nsplit) * k; a.row_base = 0; a.nsplit = 1;
    a.k = static_cast<int>(k); a.state = d_topk; a.pass = nullptr; a.pass_base = 0; a.dyn = nullptr;
    a.attrs = nullptr; a.attr_stride = 0; a.self_base = -1; a.counts = nullptr; a.thr_out = nullptr; a.overflow = nullptr;
    bf_select_kernel<true><<<dim3(static_cast<unsigned>(nq), 1), kSelThreads, sel_smem, ix->stream>>>(a);
    ++launches;
    EPS_CUDA(cudaGetLastError());
  }
  if (stats) {
    stats->n_dist += static_cast<uint64_t>(nq) * static_cast<uint64_t>(n);
    stats->kernel_launches += launches;
  }
  return EPS_OK;
}

int brute_force_topk(Index* ix, const float* d_queries, int64_t nq, int64_t row_start, int64_t row_end, int64_t k,
                     const FilterProg* d_prog, const FilterProg* h_prog, bool prefilter, unsigned long long* d_topk,
                     eps_stats* stats) {
  // The tensor-core pass keeps its per-query constants in a 1024-entry shared-memory table: larger batches
  // (config C3: B = 4096) go through it in groups of 1024 queries.
  if (nq > 1024 && row_end - row_start >= 4096 && tc_dist_usable(ix, 1024)) {
    for (int64_t q0 = 0; q0 < nq; q0 += 1024) {
      const int64_t g = std::min<int64_t>(1024, nq - q0);
      EPS_TRY(topk_impl(ix, d_queries + q0 * ix->dim, g, row_start, row_end, k, d_prog, h_prog, prefilter, -1, d_topk + q0 * k,
                        stats));
    }
    return EPS_OK;
  }
  return topk_impl(ix, d_queries, nq, row_start, row_end, k, d_prog, h_prog, prefilter, -1, d_topk, stats);
}

int scan_topk(Index* ix, const DistProducer& dist, int64_t nq, int64_t row_start, int64_t row_end, int64_t k,
              const FilterProg* d_prog, const FilterProg* h_prog, bool prefilter, int64_t self_base,
              unsigned long long* d_topk, eps_stats* stats) {
  return topk_impl(ix, nullptr, nq, row_start, row_end, k, d_prog, h_prog, prefilter, self_base, d_topk, stats, false, &dist);
}

int brute_force_knn_rows(Index* ix, int64_t q_start, int64_t nq, int64_t n_rows, int64_t k,
                         unsigned long long* d_topk, eps_stats* stats) {
  bool saved = ix->any_deleted;
  ix->any_deleted = false;  // the build indexes every row, deleted or not (ann_graph_segment.cpp:201)
  int rc = topk_impl(ix, ix->d_vectors + q_start * ix->dim, nq, 0, n_rows, k, nullptr, nullptr, false, q_start, d_topk,
                     stats);
  ix->any_deleted = saved;
  return rc;
}

}  // namespace eps
