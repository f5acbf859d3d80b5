// Principal-subspace sketch of a table (DESIGN.md §K2, "screen").
//
// For any matrix P with orthonormal rows, |P(x - q)|^2 <= |x - q|^2, so a projection of the rows onto the subspace that
// carries most of their variance gives a cheap lower bound on a distance.  The graph search reads the m-float sketch
// fl(P~(x - mu)) of a fresh neighbour and fetches its row only when that bound cannot reject it.  For inner product
// and cosine the bound is an upper bound on the dot product, which also needs |A y| and <mu, y> of each row
// (A = I - P~^T P~, y = x - mu) and a few numbers per query (dot_terms_kernel).
//
// Mean and covariance: two passes over up to 2^20 evenly spaced rows on the device, fp32 within a 512-row chunk and
// fp64 across chunks.  Basis: block subspace iteration with modified Gram-Schmidt on the host in double (the library
// links neither LAPACK nor cuSOLVER).  The columns are nested: the first k of them span the top-k subspace, so a
// prefix of the basis is the basis of a smaller sketch.
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <vector>

#include "internal.h"

namespace eps {

namespace {

constexpr int kCovTile = 32;
constexpr int kCovChunk = 512;  // sample rows per block: fp32 partial sums, then one fp64 atomic per entry

__device__ __forceinline__ int64_t sample_row(int64_t i, int64_t ns, int64_t n) { return i * n / ns; }

__global__ void sample_mean_kernel(const float* __restrict__ X, int64_t n, int64_t ns, int dim, double* __restrict__ sum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= dim) return;
  const int64_t i0 = static_cast<int64_t>(blockIdx.y) * kCovChunk, i1 = min(ns, i0 + kCovChunk);
  float s = 0.f;
  for (int64_t i = i0; i < i1; ++i) s += X[sample_row(i, ns, n) * dim + c];
  atomicAdd(sum + c, static_cast<double>(s));
}

// C[a][b] += sum over the block's sample rows of (x_a - mu_a)(x_b - mu_b), one 32 x 32 tile per block
__global__ void sample_cov_kernel(const float* __restrict__ X, int64_t n, int64_t ns, int dim, const float* __restrict__ mu,
                                  double* __restrict__ C) {
  __shared__ float xa[kCovTile][kCovTile + 1], xb[kCovTile][kCovTile + 1];
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  const int a0 = blockIdx.x * kCovTile, b0 = blockIdx.y * kCovTile;
  const int64_t i0 = static_cast<int64_t>(blockIdx.z) * kCovChunk, i1 = min(ns, i0 + kCovChunk);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int64_t r0 = i0; r0 < i1; r0 += kCovTile) {
    for (int k = ty; k < kCovTile; k += 8) {
      const int64_t i = r0 + k;
      float va = 0.f, vb = 0.f;
      if (i < i1) {
        const float* row = X + sample_row(i, ns, n) * dim;
        if (a0 + tx < dim) va = row[a0 + tx] - mu[a0 + tx];
        if (b0 + tx < dim) vb = row[b0 + tx] - mu[b0 + tx];
      }
      xa[k][tx] = va;
      xb[k][tx] = vb;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < kCovTile; ++k) {
      const float vb = xb[k][tx];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = fmaf(xa[k][ty + 8 * j], vb, acc[j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int ra = a0 + ty + 8 * j, cb = b0 + tx;
    if (ra < dim && cb < dim) atomicAdd(C + static_cast<int64_t>(ra) * dim + cb, static_cast<double>(acc[j]));
  }
}

double col_norm(const std::vector<double>& Q, int dim, int m, int j) {
  double s = 0;
  for (int i = 0; i < dim; ++i) s += Q[static_cast<size_t>(i) * m + j] * Q[static_cast<size_t>(i) * m + j];
  return std::sqrt(s);
}

// modified Gram-Schmidt, two passes, on the m <= dim columns of Q [dim x m] (column j at Q[i * m + j]); a column that
// (nearly) lies in the span of the earlier ones (a table of rank < m) is replaced by the next unit vector that does not
void mgs(std::vector<double>& Q, int dim, int m) {
  int unit = 0;
  for (int j = 0; j < m; ++j) {
    const double before = col_norm(Q, dim, m, j);
    for (int pass = 0; pass < 2; ++pass) {
      for (int k = 0; k < j; ++k) {
        double dot = 0;
        for (int i = 0; i < dim; ++i) dot += Q[static_cast<size_t>(i) * m + k] * Q[static_cast<size_t>(i) * m + j];
        for (int i = 0; i < dim; ++i) Q[static_cast<size_t>(i) * m + j] -= dot * Q[static_cast<size_t>(i) * m + k];
      }
    }
    const double nrm = col_norm(Q, dim, m, j);
    if (!(nrm > 1e-8 * before) || !(nrm > 0)) {
      for (int i = 0; i < dim; ++i) Q[static_cast<size_t>(i) * m + j] = (i == unit % dim) ? 1.0 : 0.0;
      ++unit;
      --j;  // orthogonalise the replacement
      continue;
    }
    for (int i = 0; i < dim; ++i) Q[static_cast<size_t>(i) * m + j] /= nrm;
  }
}

// Sketches of 32 rows per block of 256 threads: the rows, minus mu, are staged in shared memory once (fp32); thread
// (row r, group c) runs 4 fp32 fmaf chains over k = 0 .. dim-1 for components 4c .. 4c+3 of row r, reading P~^T as float4.
// Error of one component: v^_j = sum_k P~_jk fl(x_k - mu_k) (1 + theta_k), |theta_k| <= gamma_dim, so
// |v^_j - v_j| <= gamma_{dim+1} sum_k |P~_jk| |x_k - mu_k| <= gamma_{dim+1} |P~_j| |x - mu| <= gamma_{dim+1} sqrt(1 + eps) |x - mu|
// (Cauchy-Schwarz; |P~_j|^2 = (P~P~^T)_jj <= 1 + eps), plus dim 2^-149 for products that underflow.  ex bounds the
// norm over the m components: sqrt(m) (gamma_{dim+2} sqrt(1 + eps) |x - mu| + dim 2^-149), from |x - mu| summed in
// double from the exact differences, rounded up.
constexpr int kSkRows = 32;
__global__ void __launch_bounds__(256) sketch_rows_kernel(const float* __restrict__ X, int64_t n, int dim,
                                                          const float4* __restrict__ Pt4, const float* __restrict__ mu,
                                                          double err_per_norm, double err_abs, float* __restrict__ sk,
                                                          float* __restrict__ ex) {
  extern __shared__ float sx[];  // [kSkRows][dim + 1]
  __shared__ double s_n2[kSkRows];
  const int tid = threadIdx.x, ld = dim + 1;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * kSkRows;
  const int nr = n - r0 < kSkRows ? static_cast<int>(n - r0) : kSkRows;
  if (tid < kSkRows) s_n2[tid] = 0.0;
  __syncthreads();
  // stage: warp w takes rows w, w + 8, ...; its lanes stride the coordinates (coalesced), |x - mu|^2 in double
  for (int r = tid >> 5; r < nr; r += 8) {
    const float* x = X + (r0 + r) * dim;
    double n2 = 0.0;
    for (int k = tid & 31; k < dim; k += 32) {
      const float xv = x[k], mv = mu[k];
      sx[r * ld + k] = xv - mv;
      const double d = static_cast<double>(xv) - static_cast<double>(mv);
      n2 = fma(d, d, n2);
    }
    for (int o = 16; o > 0; o >>= 1) n2 += __shfl_xor_sync(kFull, n2, o);
    if ((tid & 31) == 0) s_n2[r] = n2;
  }
  __syncthreads();
  const int r = tid >> 3, c = tid & 7;
  if (r >= nr) return;
  const float* xr = sx + r * ld;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  for (int k = 0; k < dim; ++k) {
    const float d = xr[k];
    const float4 p = __ldg(Pt4 + k * (kSketch / 4) + c);
    a0 = fmaf(p.x, d, a0); a1 = fmaf(p.y, d, a1); a2 = fmaf(p.z, d, a2); a3 = fmaf(p.w, d, a3);
  }
  reinterpret_cast<float4*>(sk + (r0 + r) * kSketch)[c] = make_float4(a0, a1, a2, a3);
  if (c == 0) ex[r0 + r] = __double2float_ru((sqrt(s_n2[r]) * (1.0 + 0x1.0p-40) * err_per_norm + err_abs) * (1.0 + 0x1.0p-40));
}

float round_down(double x) {
  float f = static_cast<float>(x);
  if (static_cast<double>(f) > x) f = std::nextafter(f, 0.f);
  return f;
}

// Constants of the dot-product bound (graph_search.cu, screen_fresh), in double.
struct DotConsts {
  double ay_rel;    // |A y| <= (|r^| (1 + (d + 8) 2^-52) + |y^| ay_rel) (1 + 2^-50), see dot_terms_kernel
  double mu_norm;   // |mu|, rounded up
  double k;         // |y| <= k ex_x (ex_x = sqrt(m) (gamma_{d+2} sqrt(1 + eps) |y| + d 2^-149), rounded up)
  double s1;        // sqrt(1 + eps) k + 1: |s^_x| <= s1 ex_x
  double eps1;      // eps (1 + eps): |A - A^2| <= eps1
  double g_c;       // gamma_{n_c}, n_c = 4 ceil(d / 128) + 5: the consumer's fp32 dot product (lane chains + butterfly)
  double g7;        // gamma_7: the screen's 8-lane fp32 dot product of the sketches (4-step chains + 3-step butterfly)
  double tiny;      // (n_c + 8) 2^-149: products and sums of both that underflow
  double base;      // the metric's finish: distance = base - dot (IP: 0, cosine: 1)
};

// One warp per vector v, in double from the fp32 inputs: y = v - mu (each difference rounded once), w = P~ y (lane
// chains + butterfly), r = y - P~^T w (a chain of m fma from y_k), and |y|^2, |r|^2, <mu, y>.  |r - A y| is bounded by
// |y| (1 + eps) [gamma_m (1 + 1.01 sqrt(m)) + m gamma_{d+5}] (|P~|_F <= sqrt(m (1 + eps)), |w - P~ y| <= sqrt(m)
// gamma_{d+5} sqrt(1 + eps) |y|), and |A| <= max(1, eps) carries the rounding of y; ay_rel holds both with a factor 2.
// A row writes {|A y|, <mu, y>} rounded up.  A query (mu: the table's mean, v = q) writes {C0, C_ex, |A y|, K} from
// these, |q|, <q, mu> and its sketch's norm and bound E_q (qsk, written before by sketch_rows_kernel):
//   C0   = <q, mu> + g_c |q| |mu| + tiny - base,                     every quantity rounded up;
//   C_ex = |p^_q| + E_q + s1 (E_q + g7 |p^_q|) + k (eps1 |q - mu| + g_c |q|),
//   K    = |q| k, so that |q| |x| <= |q| |mu| + K ex_x;  +inf when |q| |mu| >= 2^125 (the screen keeps every id);
// a query whose norm is not finite gets C0 = NaN, which keeps every id too.
template <bool kQuery>
__global__ void __launch_bounds__(256) dot_terms_kernel(const float* __restrict__ X, int64_t n, int dim, const float4* __restrict__ Pt4,
                                                        const float* __restrict__ mu, DotConsts c, const float* __restrict__ qsk,
                                                        float2* __restrict__ row_out, float4* __restrict__ q_out) {
  const int lane = threadIdx.x & 31;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (i >= n) return;
  const float* x = X + i * dim;
  double w[kSketch];
#pragma unroll
  for (int j = 0; j < kSketch; ++j) w[j] = 0.0;
  double yy = 0.0, my = 0.0, qq = 0.0, qm = 0.0;
  for (int k = lane; k < dim; k += 32) {
    const double xv = x[k], mv = mu[k], y = xv - mv;
    yy = fma(y, y, yy);
    my = fma(mv, y, my);
    if (kQuery) { qq = fma(xv, xv, qq); qm = fma(xv, mv, qm); }
#pragma unroll
    for (int g = 0; g < kSketch / 4; ++g) {
      const float4 p = __ldg(Pt4 + k * (kSketch / 4) + g);
      w[4 * g] = fma(static_cast<double>(p.x), y, w[4 * g]);
      w[4 * g + 1] = fma(static_cast<double>(p.y), y, w[4 * g + 1]);
      w[4 * g + 2] = fma(static_cast<double>(p.z), y, w[4 * g + 2]);
      w[4 * g + 3] = fma(static_cast<double>(p.w), y, w[4 * g + 3]);
    }
  }
#pragma unroll
  for (int j = 0; j < kSketch; ++j)
    for (int o = 16; o > 0; o >>= 1) w[j] += __shfl_xor_sync(kFull, w[j], o);
  double rr = 0.0;
  for (int k = lane; k < dim; k += 32) {
    double r = static_cast<double>(x[k]) - static_cast<double>(mu[k]);
#pragma unroll
    for (int g = 0; g < kSketch / 4; ++g) {
      const float4 p = __ldg(Pt4 + k * (kSketch / 4) + g);
      r = fma(-static_cast<double>(p.x), w[4 * g], r);
      r = fma(-static_cast<double>(p.y), w[4 * g + 1], r);
      r = fma(-static_cast<double>(p.z), w[4 * g + 2], r);
      r = fma(-static_cast<double>(p.w), w[4 * g + 3], r);
    }
    rr = fma(r, r, rr);
  }
  double pp = 0.0;  // query: |p^_q|^2, one sketch component per lane
  if (kQuery) { const double p = qsk[i * kSketch + lane]; pp = p * p; }
  for (int o = 16; o > 0; o >>= 1) {
    yy += __shfl_xor_sync(kFull, yy, o);
    my += __shfl_xor_sync(kFull, my, o);
    rr += __shfl_xor_sync(kFull, rr, o);
    if (kQuery) {
      qq += __shfl_xor_sync(kFull, qq, o);
      qm += __shfl_xor_sync(kFull, qm, o);
      pp += __shfl_xor_sync(kFull, pp, o);
    }
  }
  if (lane != 0) return;
  const double up = 1.0 + (dim + 8) * 0x1.0p-52, yn = sqrt(yy) * up;
  const double ay = (sqrt(rr) * up + yn * c.ay_rel) * (1.0 + 0x1.0p-50);
  if (!kQuery) {
    const double muy = my + (dim + 6) * 0x1.0p-52 * c.mu_norm * yn;
    row_out[i] = make_float2(__double2float_ru(ay), __double2float_ru(muy + fabs(muy) * 0x1.0p-50));
    return;
  }
  const double qn = sqrt(qq) * up, q1n = yn * (1.0 + 0x1.0p-52), qmu = qm + (dim + 6) * 0x1.0p-52 * qn * c.mu_norm;
  const double pn = sqrt(pp) * (1.0 + 0x1.0p-45), eq = qsk[n * kSketch + i], qm_n = qn * c.mu_norm * (1.0 + 0x1.0p-50);
  double c0 = qmu + c.g_c * qm_n + c.tiny;
  c0 = c0 + fabs(c0) * 0x1.0p-50 - c.base;
  c0 += fabs(c0) * 0x1.0p-50;
  const double cex = (pn + eq + c.s1 * (eq + c.g7 * pn) + c.k * (c.eps1 * q1n + c.g_c * qn)) * (1.0 + 0x1.0p-40);
  double kq = qn * c.k * (1.0 + 0x1.0p-50);
  if (!(qm_n < 0x1.0p125)) kq = INFINITY;
  if (!(qn <= DBL_MAX)) c0 = NAN;
  q_out[i] = make_float4(__double2float_ru(c0), __double2float_ru(cex), __double2float_ru(ay), __double2float_ru(kq));
}

DotConsts dot_consts(const Index* ix) {
  const int dim = static_cast<int>(ix->dim), m = kSketch, nc = 4 * ((dim + 127) / 128) + 5;
  const double u = 0x1.0p-24, e = ix->sk_eps;
  const double epn = std::sqrt(static_cast<double>(m)) * ((dim + 2) * u / (1.0 - (dim + 2) * u)) * std::sqrt(1.0 + e);  // as sketch_rows
  DotConsts c;
  c.ay_rel = ((1.0 + e) * (m + 2) * (dim + m + 6) * 0x1.0p-52 + std::max(1.0, e) * 0x1.0p-52) * (1.0 + 0x1.0p-40);
  c.mu_norm = ix->sk_mu_norm;
  c.k = (1.0 / epn) * (1.0 + (dim + 8) * 0x1.0p-52) * (1.0 + 0x1.0p-40);
  c.s1 = (std::sqrt(1.0 + e) * c.k + 1.0) * (1.0 + 0x1.0p-40);
  c.eps1 = e * (1.0 + e) * (1.0 + 0x1.0p-40);
  c.g_c = nc * u / (1.0 - nc * u) * (1.0 + 0x1.0p-40);
  c.g7 = 7 * u / (1.0 - 7 * u) * (1.0 + 0x1.0p-40);
  c.tiny = (nc + 8) * 0x1.0p-149;
  c.base = ix->metric == EPS_METRIC_COSINE ? 1.0 : 0.0;
  return c;
}

template <bool kQuery>
int launch_dot_terms(Index* ix, const float* d_x, int64_t n, const float* qsk, float2* row_out, float4* q_out) {
  if (n <= 0) return EPS_OK;
  const int dim = static_cast<int>(ix->dim);
  dot_terms_kernel<kQuery><<<static_cast<unsigned>((n + 7) / 8), 256, 0, ix->stream>>>(
      d_x, n, dim, ix->d_sk_basis.as<const float4>(), ix->d_sk_basis + static_cast<int64_t>(dim) * kSketch, dot_consts(ix), qsk,
      row_out, q_out);
  EPS_CUDA(cudaGetLastError());
  return EPS_OK;
}

}  // namespace

void free_sketch(Index* ix) {
  ix->d_sk.release();
  ix->d_sk_basis.release();
  ix->sk_m = 0;
  ix->sk_share = -1.0;
}

int sketch_rows(Index* ix, const float* d_x, int64_t n, float* d_sk, float* d_ex) {
  if (n <= 0) return EPS_OK;
  const int dim = static_cast<int>(ix->dim);
  const double u = 0x1.0p-24, gam = (dim + 2) * u / (1.0 - (dim + 2) * u), sm = std::sqrt(static_cast<double>(kSketch));
  const size_t smem = static_cast<size_t>(kSkRows) * (dim + 1) * 4;
  EPS_CUDA(cudaFuncSetAttribute(sketch_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  sketch_rows_kernel<<<static_cast<unsigned>((n + kSkRows - 1) / kSkRows), 256, smem, ix->stream>>>(
      d_x, n, dim, ix->d_sk_basis.as<const float4>(), ix->d_sk_basis + static_cast<int64_t>(dim) * kSketch,
      sm * gam * std::sqrt(1.0 + ix->sk_eps), sm * dim * 0x1.0p-149, d_sk, d_ex);
  EPS_CUDA(cudaGetLastError());
  return EPS_OK;
}

int dot_row_terms(Index* ix, const float* d_x, int64_t n, float2* d_terms) {
  return launch_dot_terms<false>(ix, d_x, n, nullptr, d_terms, nullptr);
}

int sketch_queries(Index* ix, const float* d_q, int64_t nq, float* qsk, uint64_t* launches) {
  EPS_TRY(sketch_rows(ix, d_q, nq, qsk, qsk + nq * kSketch));
  ++*launches;
  if (ix->metric == EPS_METRIC_L2) return EPS_OK;
  EPS_TRY(launch_dot_terms<true>(ix, d_q, nq, qsk, nullptr, reinterpret_cast<float4*>(qsk + sk_qterms_off(nq))));
  ++*launches;
  return EPS_OK;
}

int64_t sketch_floats(const Index* ix, int64_t n) {
  return ix->metric == EPS_METRIC_L2 ? n * (kSketch + 1) : sk_terms_off(n) + 2 * n;
}

bool screen_on(const Index* ix) {
  return ix->d_sk &&
         (ix->graph_screen == EPS_GRAPH_SCREEN_ON || (ix->graph_screen == EPS_GRAPH_SCREEN_AUTO && ix->sk_share >= kScreenShare));
}

int screen_kind(const Index* ix) {
  if (!screen_on(ix)) return kScreenNone;
  return ix->metric == EPS_METRIC_L2 ? kScreenL2 : kScreenDot;
}

namespace {

int compute_sketch(Index* ix) {
  const int dim = static_cast<int>(ix->dim), m = kSketch;
  if (ix->sk_share < 0.0) {
    std::vector<float> basis, mean;
    double share = 0.0;
    EPS_TRY(principal_subspace(ix, m, &basis, &mean, &share));
    // eps = max row sum of |P~ P~^T - I| (+ the rounding of that sum), so that sigma_max(P~)^2 <= 1 + eps (Gershgorin)
    double eps = 0.0;
    for (int a = 0; a < m; ++a) {
      double row = 0.0;
      for (int b = 0; b < m; ++b) {
        double g = 0.0;
        for (int k = 0; k < dim; ++k)
          g += static_cast<double>(basis[static_cast<size_t>(a) * dim + k]) * static_cast<double>(basis[static_cast<size_t>(b) * dim + k]);
        row += std::fabs(g - (a == b ? 1.0 : 0.0));
      }
      eps = std::max(eps, row);
    }
    eps += static_cast<double>(m) * dim * 0x1.0p-52;
    const double u = 0x1.0p-24, gm = (m + 2) * u / (1.0 - (m + 2) * u);
    std::vector<float> up(static_cast<size_t>(dim) * m + dim);  // P~ transposed [dim x m], then mu
    for (int j = 0; j < m; ++j)
      for (int k = 0; k < dim; ++k) up[static_cast<size_t>(k) * m + j] = basis[static_cast<size_t>(j) * dim + k];
    for (int k = 0; k < dim; ++k) up[static_cast<size_t>(dim) * m + k] = mean[k];
    EPS_TRY(ix->d_sk_basis.reserve(up.size() * 4));
    EPS_CUDA(cudaMemcpyAsync(ix->d_sk_basis, up.data(), up.size() * 4, cudaMemcpyHostToDevice, ix->stream));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
    ix->sk_m = m;
    ix->sk_share = share;
    ix->sk_eps = eps;
    ix->sk_g = round_down(1.0 - gm);
    ix->sk_scale = round_down((1.0 - 2.0 * (dim + 2) * u) / (1.0 + eps));
    double mu2 = 0.0;
    for (int k = 0; k < dim; ++k) mu2 += static_cast<double>(mean[k]) * static_cast<double>(mean[k]);
    ix->sk_mu_norm = std::sqrt(mu2) * (1.0 + (dim + 8) * 0x1.0p-52);
  }
  const bool want = ix->graph_screen == EPS_GRAPH_SCREEN_ON || ix->sk_share >= kScreenShare;
  if (!want) ix->d_sk.release();

  if (want && !ix->d_sk) {
    const int64_t n = ix->n_indexed;
    EPS_TRY(ix->d_sk.reserve(static_cast<size_t>(sketch_floats(ix, n)) * 4));  // [n x m] sketches, [n] bounds (, [n] terms)
    EPS_TRY(sketch_rows(ix, ix->d_vectors, n, ix->d_sk, ix->d_sk + n * m));
    if (ix->metric != EPS_METRIC_L2)
      EPS_TRY(dot_row_terms(ix, ix->d_vectors, n, reinterpret_cast<float2*>(ix->d_sk + sk_terms_off(n))));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
  }
  return EPS_OK;
}

}  // namespace

void ensure_sketch(Index* ix) {
  if (ix->graph_screen == EPS_GRAPH_SCREEN_OFF || ix->dim < 128 || ix->n_indexed < 1 || !ix->d_vectors) {
    ix->d_sk.release();
    return;
  }
  // the screen only saves time: when it cannot be set up (out of device memory), the search runs without it
  if (compute_sketch(ix) != EPS_OK) {
    cudaGetLastError();  // a failed allocation must not surface in the next launch check
    free_sketch(ix);
  }
}

int principal_subspace(Index* ix, int m, std::vector<float>* basis, std::vector<float>* mean, double* share) {
  const int dim = static_cast<int>(ix->dim);
  const int64_t n = ix->n_indexed;
  if (m < 1 || m > dim || n < 1) return fail(EPS_ERR_INVALID_ARGUMENT, "principal_subspace: bad size");
  const int64_t ns = std::min<int64_t>(n, 1 << 20);
  const unsigned chunks = static_cast<unsigned>((ns + kCovChunk - 1) / kCovChunk);
  DevBuf d_sum, d_mu, d_cov;
  EPS_TRY(d_sum.reserve(static_cast<size_t>(dim) * 8));
  EPS_TRY(d_mu.reserve(static_cast<size_t>(dim) * 4));
  EPS_TRY(d_cov.reserve(static_cast<size_t>(dim) * dim * 8));
  EPS_CUDA(cudaMemsetAsync(d_sum.p, 0, static_cast<size_t>(dim) * 8, ix->stream));
  EPS_CUDA(cudaMemsetAsync(d_cov.p, 0, static_cast<size_t>(dim) * dim * 8, ix->stream));
  sample_mean_kernel<<<dim3((dim + 127) / 128, chunks), 128, 0, ix->stream>>>(ix->d_vectors, n, ns, dim, d_sum.as<double>());
  EPS_CUDA(cudaGetLastError());
  std::vector<double> sum(dim);
  EPS_CUDA(cudaMemcpyAsync(sum.data(), d_sum.p, static_cast<size_t>(dim) * 8, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  mean->assign(dim, 0.f);
  for (int c = 0; c < dim; ++c) (*mean)[c] = static_cast<float>(sum[c] / static_cast<double>(ns));
  EPS_CUDA(cudaMemcpyAsync(d_mu.p, mean->data(), static_cast<size_t>(dim) * 4, cudaMemcpyHostToDevice, ix->stream));
  const unsigned tiles = static_cast<unsigned>((dim + kCovTile - 1) / kCovTile);
  sample_cov_kernel<<<dim3(tiles, tiles, chunks), dim3(32, 8), 0, ix->stream>>>(ix->d_vectors, n, ns, dim, d_mu.as<float>(),
                                                                                d_cov.as<double>());
  EPS_CUDA(cudaGetLastError());
  std::vector<double> C(static_cast<size_t>(dim) * dim);
  EPS_CUDA(cudaMemcpyAsync(C.data(), d_cov.p, C.size() * 8, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  double trace = 0;
  for (int c = 0; c < dim; ++c) trace += C[static_cast<size_t>(c) * dim + c];

  // block subspace iteration from a seeded start
  std::vector<double> Q(static_cast<size_t>(dim) * m), Z(Q.size());
  uint64_t s = 0x9E3779B97F4A7C15ull;
  for (double& v : Q) {
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    v = static_cast<double>(s >> 11) * 0x1.0p-53 - 0.5;
  }
  mgs(Q, dim, m);
  for (int it = 0; it < 40; ++it) {
    std::fill(Z.begin(), Z.end(), 0.0);
    for (int i = 0; i < dim; ++i) {
      const double* ci = C.data() + static_cast<size_t>(i) * dim;
      double* zi = Z.data() + static_cast<size_t>(i) * m;
      for (int k = 0; k < dim; ++k) {
        const double c = ci[k];
        const double* qk = Q.data() + static_cast<size_t>(k) * m;
        for (int j = 0; j < m; ++j) zi[j] += c * qk[j];
      }
    }
    Q.swap(Z);
    mgs(Q, dim, m);
  }
  // explained share of the top m: trace(Q^T C Q) / trace(C)
  double expl = 0;
  for (int j = 0; j < m; ++j)
    for (int i = 0; i < dim; ++i) {
      double ci = 0;
      for (int k = 0; k < dim; ++k) ci += C[static_cast<size_t>(i) * dim + k] * Q[static_cast<size_t>(k) * m + j];
      expl += Q[static_cast<size_t>(i) * m + j] * ci;
    }
  *share = trace > 0 ? expl / trace : 0.0;
  basis->assign(static_cast<size_t>(m) * dim, 0.f);  // row-major [m x dim]
  for (int j = 0; j < m; ++j)
    for (int i = 0; i < dim; ++i) (*basis)[static_cast<size_t>(j) * dim + i] = static_cast<float>(Q[static_cast<size_t>(i) * m + j]);
  return EPS_OK;
}

}  // namespace eps
