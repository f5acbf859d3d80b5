// Posting lists of a sparse field (DESIGN.md §K5): per-term posting lists of rows [0, inv_rows).  On an IP / cosine
// field they are the inverted index (eps_index_build_sparse_inverted): the exact scan's distance tile is computed from
// them instead of merging every (query, row) pair.  On an L2 field they are the L2 screen
// (eps_index_build_sparse_l2_screen): the same score kernel writes a proven lower bound of each covered row's distance
// (sparse_l2_lower_bound), and only the rows whose bound can still place them among the k best are merged
// (l2_threshold_kernel, l2_rescore_kernel; the steps are driven by fp32_scan, brute_force.cu).
//
// Why the tile is bitwise the scan's: for IP and cosine the reference adds the matched products row[i] * query[i] in
// increasing index order, from 0 (engine/db/vector.cpp:7-47).  inverted_score_kernel walks a query's elements in their
// (increasing) index order and adds each term's posting value times the query value into a per-row fp32 accumulator
// that starts at 0, with __fmul_rn / __fadd_rn: every row sees the same operations in the same order as in SparseMerge
// (common.cuh), and the tile finishes through sparse_finish like every other sparse distance.  A row that matches
// nothing keeps 0, as in the merge.  L2 cannot be served that way: its merged order also adds the row-only and
// query-only terms; the screen bounds it instead and takes the exact value from SparseMerge.
//
// Build: expand the CSR elements of rows [0, n) to (index, {row, value}) pairs, sort them by index with a stable radix
// sort (rows stay ascending within a term), flag the first posting of each term and take the int64 exclusive sum of the
// flags (term slots), then scatter the terms and their offsets.  The new arrays replace the old ones only when every
// step has succeeded.
//
// Extension (eps_index_extend_sparse_postings): rows [inv_rows, n) are sorted the same way on their own, and the two
// lists are merged term by term: each old term's block moves, unchanged, to its place in the union, and the new rows'
// postings follow it.  Old postings are copied once and never sorted again; the arrays are the full build's, bit for
// bit (extend_sparse_inverted).
//
// Search: once per call, inverted_plan_kernel maps every query element to its posting range (binary search on the
// terms; an index no covered row has gets an empty range).  inverted_score_kernel: one CTA = one query x a slice of
// kInvSlice rows with their accumulators in shared memory.  Per batch of up to kInvThreads terms, one thread per term
// finds the term's postings inside the slice (binary search on rows); then the terms are applied in query order, the
// threads striding over a term's postings (its rows are distinct, so no two threads touch one accumulator), with a
// barrier after each term that has postings in the slice.  The queries of one slice are adjacent in launch order, so
// the slice's postings are read from HBM about once and from L2 by the other queries.
//
// The sparse graph build (sparse.cu) uses the same producer for its kNN pass: its queries are chunks of the mirror's own
// rows, whose elements start at the chunk's element offset (InvertedDist::elem_base) rather than at 0.
#include <cub/cub.cuh>

#include <algorithm>

#include "internal.h"

namespace eps {

namespace {

constexpr int kInvSlice = 2048;   // rows per CTA: 8 KB of accumulators; 1M rows give one query 489 CTAs
constexpr int kInvThreads = 256;  // threads per CTA = terms whose bounds one pass finds

// One warp per row of [row_base, n): element p of row r becomes the pair (index, {r, value bits}) at position
// p - elem_base (elem_base = row_ptr[row_base]).
__global__ void inverted_expand_kernel(const int64_t* __restrict__ row_ptr, const uint2* __restrict__ elems,
                                       int64_t row_base, int64_t elem_base, int64_t n, uint32_t* __restrict__ keys,
                                       uint2* __restrict__ vals) {
  const int64_t r = row_base + ((blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const int64_t p1 = row_ptr[r + 1];
  for (int64_t p = row_ptr[r] + lane; p < p1; p += 32) {
    const uint2 e = elems[p];
    keys[p - elem_base] = e.x;
    vals[p - elem_base] = make_uint2(static_cast<uint32_t>(r), e.y);
  }
}

__device__ __forceinline__ bool term_starts(const uint32_t* keys, int64_t i, int64_t P) {
  return i < P && (i == 0 || keys[i] != keys[i - 1]);
}

// flags[i] = 1 where posting i starts a term (i < P), flags[P] = 0: their exclusive sum is each term's slot and, at P,
// the number of terms.
__global__ void inverted_flag_kernel(const uint32_t* __restrict__ keys, int64_t P, int64_t* __restrict__ flags) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i <= P) flags[i] = term_starts(keys, i, P) ? 1 : 0;
}

__global__ void inverted_scatter_kernel(const uint32_t* __restrict__ keys, int64_t P, const int64_t* __restrict__ slot,
                                        uint32_t* __restrict__ terms, int64_t* __restrict__ ptr) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i > P) return;
  if (i == P) {
    ptr[slot[P]] = P;
  } else if (term_starts(keys, i, P)) {
    terms[slot[i]] = keys[i];
    ptr[slot[i]] = i;
  }
}

// First i of [0, len) with a[i] >= x (a ascending).
__device__ __forceinline__ int64_t terms_lower_bound(const uint32_t* a, int64_t len, uint32_t x) {
  int64_t lo = 0, hi = len;
  while (lo < hi) {
    const int64_t m = lo + ((hi - lo) >> 1);
    if (a[m] < x) lo = m + 1;
    else hi = m;
  }
  return lo;
}

__device__ __forceinline__ bool has_term(const uint32_t* a, int64_t len, int64_t i, uint32_t x) {
  return i < len && a[i] == x;
}

// Extension, step 1 (one thread per term j of the appended rows, plus one): only[j] = 1 when no old term equals new
// term j, only[t_new] = 0.  Their exclusive sum is, at j, the new-only terms below new term j and, at t_new, their number.
__global__ void extend_probe_kernel(const uint32_t* __restrict__ old_terms, int64_t t_old,
                                    const uint32_t* __restrict__ new_terms, int64_t t_new, int64_t* __restrict__ only) {
  const int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (j > t_new) return;
  only[j] = j < t_new && !has_term(old_terms, t_old, terms_lower_bound(old_terms, t_old, new_terms[j]), new_terms[j]);
}

// Step 2 (one thread per old term, then one per new term, plus one): the union's terms, ascending, and each one's
// posting count in count[0, t), count[t] = 0.  Old term i goes to slot i + (new-only terms below it); new term j to slot
// (old terms below it) + below[j], where an old term with the same index is.  A shared term is counted by its new term.
__global__ void extend_union_kernel(const uint32_t* __restrict__ old_terms, const int64_t* __restrict__ old_ptr,
                                    int64_t t_old, const uint32_t* __restrict__ new_terms,
                                    const int64_t* __restrict__ new_ptr, int64_t t_new, const int64_t* __restrict__ below,
                                    int64_t* __restrict__ old_slot, int64_t* __restrict__ new_slot,
                                    uint32_t* __restrict__ terms, int64_t* __restrict__ count, int64_t t) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < t_old) {
    const uint32_t x = old_terms[i];
    const int64_t j = terms_lower_bound(new_terms, t_new, x);
    const int64_t s = i + below[j];
    old_slot[i] = s;
    terms[s] = x;
    if (!has_term(new_terms, t_new, j, x)) count[s] = old_ptr[i + 1] - old_ptr[i];
  } else if (i < t_old + t_new) {
    const int64_t j = i - t_old;
    const uint32_t x = new_terms[j];
    const int64_t o = terms_lower_bound(old_terms, t_old, x);
    const int64_t s = o + below[j];
    new_slot[j] = s;
    int64_t c = new_ptr[j + 1] - new_ptr[j];
    if (has_term(old_terms, t_old, o, x)) c += old_ptr[o + 1] - old_ptr[o];
    else terms[s] = x;
    count[s] = c;
  } else if (i == t_old + t_new) {
    count[t] = 0;
  }
}

// Step 3 (one thread per posting p of one source: the old lists, or the appended rows' sorted postings): p's term i is
// the last one whose offset is <= p (every term has a posting, so src_ptr ascends strictly).  The old postings open
// their union term's block, in their order; the new ones close it, in theirs.
__global__ void extend_place_kernel(const uint2* __restrict__ src, const int64_t* __restrict__ src_ptr, int64_t t_src,
                                    int64_t p_src, const int64_t* __restrict__ slot, bool at_end,
                                    const int64_t* __restrict__ ptr, uint2* __restrict__ post) {
  const int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (p >= p_src) return;
  int64_t lo = 0, hi = t_src - 1;
  while (lo < hi) {
    const int64_t m = hi - ((hi - lo) >> 1);
    if (src_ptr[m] <= p) lo = m;
    else hi = m - 1;
  }
  const int64_t d = at_end ? ptr[slot[lo] + 1] - src_ptr[lo + 1] : ptr[slot[lo]] - src_ptr[lo];
  post[p + d] = src[p];
}

// plan[e] = the posting range of query element e's index, or an empty range when no covered row has it.
__global__ void inverted_plan_kernel(const uint32_t* __restrict__ terms, int64_t n_terms, const int64_t* __restrict__ ptr,
                                     const uint2* __restrict__ q_elems, int64_t n_elems, longlong2* __restrict__ plan) {
  const int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (e >= n_elems) return;
  const uint32_t idx = q_elems[e].x;
  int64_t lo = 0, hi = n_terms;
  while (lo < hi) {
    const int64_t m = lo + ((hi - lo) >> 1);
    if (terms[m] < idx) lo = m + 1;
    else hi = m;
  }
  plan[e] = lo < n_terms && terms[lo] == idx ? make_longlong2(ptr[lo], ptr[lo + 1]) : make_longlong2(0, 0);
}

// First posting of [b, e) whose row is >= row.
__device__ __forceinline__ int64_t rows_lower_bound(const uint2* post, int64_t b, int64_t e, int32_t row) {
  while (b < e) {
    const int64_t m = b + ((e - b) >> 1);
    if (static_cast<int32_t>(__ldg(&post[m].x)) < row) b = m + 1;
    else e = m;
  }
  return b;
}

// Lower bound of the reference's L2 distance D_ref of a (row, query) pair from the fp32 dot of their matched elements
// (the score kernel's accumulator), the fp32 squared norms rn = d_sp_norm2[row] and qn, and the element counts m_r and
// m_q; +inf when the bound does not cover the pair.  Derivation (u = 2^-24, eta = 2^-149, gamma_k = k u / (1 - k u),
// m = m_r + m_q, R2 / Q2 / P the real |row|^2, |query|^2 and <row, query>, D = R2 + Q2 - 2 P):
//   * rn is a sequential sum of m_r non-negative fl(v * v): |rn - R2| <= gamma_{m_r} R2 + m_r eta (a product that
//     underflows is off by at most 2^-150; a sum with a subnormal result is exact), so
//     R2 >= max(0, (1 - gamma_{m_r}) (rn - m_r eta)); the same for Q2 with qn and m_q;
//   * dot sums c <= m products fl(r_i q_i): |dot - P| <= gamma_m sum |r_i q_i| + m eta, and sum |r_i q_i| <= (R2 + Q2) / 2,
//     so D >= (1 - gamma_m) (R2 + Q2) - 2 dot - 2 m eta, and D >= 0;
//   * D_ref adds m' <= m non-negative terms fl(fl(a - b)^2) or fl(v * v), each within m + 2 roundings of its real value:
//     D_ref >= (1 - gamma_{m+2}) D - m eta (when D_ref is finite; +inf bounds itself).
// Every step is rounded toward -inf in fp64.  m + 2 <= 2^20 keeps k u <= 2^-4, where gamma_k <= (9/8) k u and
// 1 - (9/8) k u is exact.  Pairs with a non-finite input or more elements get +inf: they are always re-scored.
constexpr int64_t kL2BoundTerms = 1 << 20;

__device__ __forceinline__ float sparse_l2_lower_bound(float dot, float rn, float qn, int64_t m_r, int64_t m_q) {
  const int64_t m = m_r + m_q;
  if (!isfinite(dot) || !isfinite(rn) || !isfinite(qn) || m + 2 > kL2BoundTerms) return INFINITY;
  const double eta = 0x1p-149;
  const auto one_minus_gamma = [](int64_t k) { return 1.0 - static_cast<double>(k) * (1.125 * 0x1p-24); };  // exact
  // k * eta and 2 * dot are exact in fp64
  const double r2 = fmax(0.0, __dmul_rd(one_minus_gamma(m_r), __dadd_rd(rn, -static_cast<double>(m_r) * eta)));
  const double q2 = fmax(0.0, __dmul_rd(one_minus_gamma(m_q), __dadd_rd(qn, -static_cast<double>(m_q) * eta)));
  double d = __dmul_rd(one_minus_gamma(m), __dadd_rd(r2, q2));
  d = __dadd_rd(__dadd_rd(d, -2.0 * static_cast<double>(dot)), -2.0 * static_cast<double>(m) * eta);
  const double lb = __dadd_rd(__dmul_rd(one_minus_gamma(m + 2), fmax(d, 0.0)), -static_cast<double>(m) * eta);
  return __double2float_rd(lb);
}

// IP / cosine: the distance tile.  L2: the lower-bound tile of the L2 screen (row_ptr gives each row's element count).
template <int METRIC>
__global__ void __launch_bounds__(kInvThreads) inverted_score_kernel(
    const uint2* __restrict__ post, const longlong2* __restrict__ plan, const int64_t* __restrict__ q_ptr,
    const uint2* __restrict__ q_elems, int64_t elem_base, const float* __restrict__ q_norm2,
    const float* __restrict__ row_norm2, const int64_t* __restrict__ row_ptr, int64_t nq, int64_t row_start, int64_t n,
    float* __restrict__ D, int64_t ldd) {
  __shared__ float acc[kInvSlice];
  __shared__ int64_t lo_s[kInvThreads], hi_s[kInvThreads];
  __shared__ float qv_s[kInvThreads];
  const int64_t q = blockIdx.x % nq, s = blockIdx.x / nq;
  const int64_t r0 = row_start + s * kInvSlice;
  const int rows = static_cast<int>(min(static_cast<int64_t>(kInvSlice), row_start + n - r0));
  const int32_t row_lo = static_cast<int32_t>(r0), row_hi = static_cast<int32_t>(r0 + rows);
  for (int i = threadIdx.x; i < kInvSlice; i += kInvThreads) acc[i] = 0.f;
  // element offsets relative to the plan's first element (q_elems points at it)
  const int64_t e0 = q_ptr[q] - elem_base, e1 = q_ptr[q + 1] - elem_base;
  for (int64_t t0 = e0; t0 < e1; t0 += kInvThreads) {
    const int nt = static_cast<int>(min(static_cast<int64_t>(kInvThreads), e1 - t0));
    __syncthreads();  // the accumulators are zeroed and the previous batch's bounds are read
    if (threadIdx.x < nt) {
      const longlong2 r = plan[t0 + threadIdx.x];
      const int64_t lo = rows_lower_bound(post, r.x, r.y, row_lo);
      lo_s[threadIdx.x] = lo;
      hi_s[threadIdx.x] = rows_lower_bound(post, lo, r.y, row_hi);
      qv_s[threadIdx.x] = __uint_as_float(q_elems[t0 + threadIdx.x].y);
    }
    __syncthreads();
    for (int j = 0; j < nt; ++j) {
      const int64_t a = lo_s[j], b = hi_s[j];
      if (a == b) continue;  // the same for every thread: the barrier below is reached by all or none
      const float y = qv_s[j];
      for (int64_t p = a + threadIdx.x; p < b; p += kInvThreads) {
        const uint2 e = __ldg(post + p);
        const int r = static_cast<int>(e.x) - row_lo;
        acc[r] = __fadd_rn(acc[r], __fmul_rn(__uint_as_float(e.y), y));
      }
      __syncthreads();  // the next term adds to these rows after this one, in the query's index order
    }
  }
  __syncthreads();
  float qn = 0.f;
  if (METRIC != EPS_METRIC_IP) qn = q_norm2[q];
  float* out = D + q * ldd + (r0 - row_start);
  for (int i = threadIdx.x; i < rows; i += kInvThreads) {
    float rn = 0.f;
    if (METRIC != EPS_METRIC_IP) rn = row_norm2[r0 + i];
    if (METRIC == EPS_METRIC_L2)
      out[i] = sparse_l2_lower_bound(acc[i], rn, qn, row_ptr[r0 + i + 1] - row_ptr[r0 + i], e1 - e0);
    else
      out[i] = sparse_finish<METRIC>(acc[i], rn, qn);
  }
}

// Step 2 of the L2 screen: T[q] = the largest exact distance of the K rows of keys[q] (+inf when one is missing, has an
// unbounded key or a NaN distance).  Rows at or above inv_rows carry their exact distance in the key already.
constexpr int kL2Threads = 256;
__global__ void __launch_bounds__(kL2Threads) l2_threshold_kernel(
    const int64_t* __restrict__ row_ptr, const uint2* __restrict__ elems, int64_t inv_rows, const int64_t* __restrict__ q_ptr,
    const uint2* __restrict__ q_elems, const unsigned long long* __restrict__ keys, int k, float* __restrict__ T,
    unsigned long long* __restrict__ n_rescored) {
  __shared__ unsigned t_bits;  // exact distances are >= +0 and order as their bits
  __shared__ unsigned long long cnt;
  const int64_t q = blockIdx.x;
  if (threadIdx.x == 0) { t_bits = 0u; cnt = 0ull; }
  __syncthreads();
  const uint2* qv = q_elems + q_ptr[q];
  const int64_t qn_el = q_ptr[q + 1] - q_ptr[q];
  unsigned my = 0u, mine = 0u;
  for (int j = threadIdx.x; j < k; j += kL2Threads) {
    const unsigned long long key = keys[q * k + j] & kKeyMask;
    float d = key_dist(key);
    if (key == kKeyInf || isinf(d)) {
      d = INFINITY;
    } else if (key_id(key) < inv_rows) {
      d = sparse_row_dist<EPS_METRIC_L2>(row_ptr, elems, nullptr, key_id(key), qv, qn_el, 0.f);
      ++mine;
    }
    if (d != d) d = INFINITY;
    my = max(my, __float_as_uint(d));
  }
  atomicMax(&t_bits, my);
  if (mine) atomicAdd(&cnt, static_cast<unsigned long long>(mine));
  __syncthreads();
  if (threadIdx.x == 0) {
    T[q] = __uint_as_float(t_bits);
    if (cnt) atomicAdd(n_rescored, cnt);
  }
}

// Step 3: one CTA = one query x kInvSlice rows of the tile.  A row the select will keep (pass bit set, not the query's
// own row) whose bound is <= T[q] or +inf gets its exact distance; every other row gets +inf.
__global__ void __launch_bounds__(kL2Threads) l2_rescore_kernel(
    const int64_t* __restrict__ row_ptr, const uint2* __restrict__ elems, const int64_t* __restrict__ q_ptr,
    const uint2* __restrict__ q_elems, const float* __restrict__ T, const uint32_t* __restrict__ pass, int64_t pass_base,
    int64_t self_base, int64_t nq, int64_t row_start, int64_t n, float* __restrict__ D, int64_t ldd,
    unsigned long long* __restrict__ n_rescored) {
  __shared__ unsigned cnt;
  const int64_t q = blockIdx.x % nq, s = blockIdx.x / nq;
  const int64_t i0 = s * kInvSlice;
  const int rows = static_cast<int>(min(static_cast<int64_t>(kInvSlice), n - i0));
  if (threadIdx.x == 0) cnt = 0u;
  __syncthreads();
  const float t = T[q];
  const uint2* qv = q_elems + q_ptr[q];
  const int64_t qn_el = q_ptr[q + 1] - q_ptr[q];
  float* out = D + q * ldd + i0;
  unsigned mine = 0u;
  for (int i = threadIdx.x; i < rows; i += kL2Threads) {
    const int64_t r = row_start + i0 + i;
    const float lb = out[i];
    bool ok = lb <= t || lb == INFINITY;
    if (ok && pass) {
      const int64_t pi = r - pass_base;
      ok = (pass[pi >> 5] >> (pi & 31)) & 1u;
    }
    if (ok && self_base >= 0 && r == self_base + q) ok = false;
    float d = INFINITY;
    if (ok) {
      d = sparse_row_dist<EPS_METRIC_L2>(row_ptr, elems, nullptr, static_cast<uint32_t>(r), qv, qn_el, 0.f);
      ++mine;
    }
    out[i] = d;
  }
  if (mine) atomicAdd(&cnt, mine);
  __syncthreads();
  if (threadIdx.x == 0 && cnt) atomicAdd(n_rescored, static_cast<unsigned long long>(cnt));
}

unsigned blocks_for(int64_t threads, int per_block) { return static_cast<unsigned>((threads + per_block - 1) / per_block); }

// Posting lists of some rows, laid out as the index's: terms ascending, offsets, postings with rows ascending per term.
struct Postings {
  DevArray<uint32_t> terms;  // [T]
  DevArray<int64_t> ptr;     // [T + 1]
  DevArray<uint2> post;      // [P]
  int64_t T = 0, P = 0;
};

// The posting lists of rows [r0, n): expand them to (index, {row, value}) pairs, sort the pairs by index with a stable
// radix sort (rows stay ascending within a term), flag the first posting of each term, take the int64 exclusive sum of
// the flags (term slots), then scatter the terms and their offsets.  Offsets count from the first posting of row r0.
int sort_postings(Index* ix, int64_t r0, int64_t n, Postings* out) {
  int64_t e[2] = {0, 0};  // element offsets of rows r0 and n
  EPS_CUDA(cudaMemcpyAsync(&e[0], ix->d_sp_ptr + r0, 8, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaMemcpyAsync(&e[1], ix->d_sp_ptr + n, 8, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  const int64_t P = e[1] - e[0];
  // indices are < dim: the sort looks at the bits of dim - 1 only
  int bits = 1;
  while (bits < 32 && ((static_cast<uint64_t>(ix->dim) - 1) >> bits) != 0) ++bits;
  DevArray<uint32_t> keys_a, keys_b, terms;
  DevArray<uint2> vals_a, vals_b;  // P + 1 entries: the spare one holds the term flags, an int64 per posting + 1
  DevArray<int64_t> ptr;
  DevBuf tmp;
  const size_t P1 = static_cast<size_t>(P) + 1;
  EPS_TRY(keys_a.reserve(std::max<size_t>(P, 1) * 4));
  EPS_TRY(keys_b.reserve(std::max<size_t>(P, 1) * 4));
  EPS_TRY(vals_a.reserve(P1 * 8));
  EPS_TRY(vals_b.reserve(P1 * 8));
  inverted_expand_kernel<<<blocks_for((n - r0) * 32, 256), 256, 0, ix->stream>>>(ix->d_sp_ptr, ix->d_sp_elems, r0, e[0], n,
                                                                                 keys_a, vals_a);
  EPS_CUDA(cudaGetLastError());
  cub::DoubleBuffer<uint32_t> kb(keys_a, keys_b);
  cub::DoubleBuffer<uint64_t> vb(reinterpret_cast<uint64_t*>(vals_a.p), reinterpret_cast<uint64_t*>(vals_b.p));
  size_t sort_bytes = 0, scan_bytes = 0;
  EPS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, kb, vb, P, 0, bits, ix->stream));
  EPS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, reinterpret_cast<int64_t*>(vals_b.p), static_cast<int64_t>(P1),
                                         ix->stream));
  EPS_TRY(tmp.reserve(std::max(sort_bytes, scan_bytes)));
  if (P > 0) EPS_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, sort_bytes, kb, vb, P, 0, bits, ix->stream));
  // the sorted postings are in vb.Current(); the other value buffer takes the flags and, in place, their sum
  const bool in_a = vb.Current() == reinterpret_cast<uint64_t*>(vals_a.p);
  DevArray<uint2>& post = in_a ? vals_a : vals_b;
  int64_t* flags = reinterpret_cast<int64_t*>((in_a ? vals_b : vals_a).p);
  inverted_flag_kernel<<<blocks_for(P + 1, 256), 256, 0, ix->stream>>>(kb.Current(), P, flags);
  EPS_CUDA(cudaGetLastError());
  EPS_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, scan_bytes, flags, static_cast<int64_t>(P1), ix->stream));
  int64_t T = 0;
  EPS_CUDA(cudaMemcpyAsync(&T, flags + P, 8, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  EPS_TRY(terms.reserve(static_cast<size_t>(std::max<int64_t>(T, 1)) * 4));
  EPS_TRY(ptr.reserve(static_cast<size_t>(T + 1) * 8));
  inverted_scatter_kernel<<<blocks_for(P + 1, 256), 256, 0, ix->stream>>>(kb.Current(), P, flags, terms, ptr);
  EPS_CUDA(cudaGetLastError());
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  out->terms.swap(terms);
  out->ptr.swap(ptr);
  out->post.swap(post);
  out->T = T;
  out->P = P;
  return EPS_OK;
}

// Every step succeeded: the lists replace the index's (whose arrays go out with `l`).
void install(Index* ix, Postings* l, int64_t n) {
  ix->d_inv_terms.swap(l->terms);
  ix->d_inv_ptr.swap(l->ptr);
  ix->d_inv_post.swap(l->post);
  ix->inv_rows = n;
  ix->inv_terms = l->T;
  ix->inv_postings = l->P;
}

}  // namespace

int build_sparse_inverted(Index* ix, int64_t n) {
  if (n == 0) {
    ix->d_inv_terms.release();
    ix->d_inv_ptr.release();
    ix->d_inv_post.release();
    ix->inv_rows = ix->inv_terms = ix->inv_postings = 0;
    return EPS_OK;
  }
  Postings l;
  EPS_TRY(sort_postings(ix, 0, n, &l));
  install(ix, &l, n);
  return EPS_OK;
}

// The lists of rows [inv_rows, n) are sorted on their own and merged into the index's: the union of the two term sets
// (extend_probe_kernel, its exclusive sum, extend_union_kernel), the union's offsets (the exclusive sum of its counts),
// then every old posting and every new one copied to its place (extend_place_kernel).  The new rows are numbered above
// every covered row, so appending them to their terms' blocks gives each block the order a stable sort of [0, n) gives
// it: the arrays are those build_sparse_inverted(ix, n) makes.
int extend_sparse_inverted(Index* ix, int64_t n) {
  Postings add;
  EPS_TRY(sort_postings(ix, ix->inv_rows, n, &add));
  if (add.P == 0) {  // empty rows only: the lists do not change
    ix->inv_rows = n;
    return EPS_OK;
  }
  const int64_t t_old = ix->inv_terms, p_old = ix->inv_postings;
  DevArray<int64_t> below, old_slot, new_slot;
  DevBuf tmp;
  EPS_TRY(below.reserve(static_cast<size_t>(add.T + 1) * 8));
  EPS_TRY(old_slot.reserve(static_cast<size_t>(std::max<int64_t>(t_old, 1)) * 8));
  EPS_TRY(new_slot.reserve(static_cast<size_t>(add.T) * 8));
  extend_probe_kernel<<<blocks_for(add.T + 1, 256), 256, 0, ix->stream>>>(ix->d_inv_terms, t_old, add.terms, add.T, below);
  EPS_CUDA(cudaGetLastError());
  size_t scan_bytes = 0;
  EPS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, below.as<int64_t>(), add.T + 1, ix->stream));
  EPS_TRY(tmp.reserve(scan_bytes));
  EPS_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, scan_bytes, below.as<int64_t>(), add.T + 1, ix->stream));
  int64_t only = 0;
  EPS_CUDA(cudaMemcpyAsync(&only, below + add.T, 8, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  Postings all;
  all.T = t_old + only;
  all.P = p_old + add.P;
  EPS_TRY(all.terms.reserve(static_cast<size_t>(all.T) * 4));
  EPS_TRY(all.ptr.reserve(static_cast<size_t>(all.T + 1) * 8));
  EPS_TRY(all.post.reserve(static_cast<size_t>(all.P) * 8));
  extend_union_kernel<<<blocks_for(t_old + add.T + 1, 256), 256, 0, ix->stream>>>(
      ix->d_inv_terms, ix->d_inv_ptr, t_old, add.terms, add.ptr, add.T, below, old_slot, new_slot, all.terms, all.ptr,
      all.T);
  EPS_CUDA(cudaGetLastError());
  EPS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, all.ptr.as<int64_t>(), all.T + 1, ix->stream));
  EPS_TRY(tmp.reserve(scan_bytes));
  EPS_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, scan_bytes, all.ptr.as<int64_t>(), all.T + 1, ix->stream));
  if (p_old > 0) {
    extend_place_kernel<<<blocks_for(p_old, 256), 256, 0, ix->stream>>>(ix->d_inv_post, ix->d_inv_ptr, t_old, p_old,
                                                                         old_slot, false, all.ptr, all.post);
    EPS_CUDA(cudaGetLastError());
  }
  extend_place_kernel<<<blocks_for(add.P, 256), 256, 0, ix->stream>>>(add.post, add.ptr, add.T, add.P, new_slot, true,
                                                                       all.ptr, all.post);
  EPS_CUDA(cudaGetLastError());
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  install(ix, &all, n);
  return EPS_OK;
}

int InvertedDist::plan(Index* ix, uint64_t* launches) const {
  if (planned) return EPS_OK;
  EPS_TRY(ix->s_inv_plan.reserve(static_cast<size_t>(n_elems) * sizeof(longlong2)));
  if (n_elems > 0) {
    inverted_plan_kernel<<<blocks_for(n_elems, 256), 256, 0, ix->stream>>>(
        ix->d_inv_terms, ix->inv_terms, ix->d_inv_ptr, scan.q.elems + elem_base, n_elems, ix->s_inv_plan.as<longlong2>());
    EPS_CUDA(cudaGetLastError());
    ++*launches;
  }
  planned = true;
  return EPS_OK;
}

namespace {

// Rows of [row_start, row_start + n) the posting lists cover: the first ones.
int64_t covered_rows(const Index* ix, int64_t row_start, int64_t n) {
  return std::max<int64_t>(0, std::min(row_start + n, ix->inv_rows) - row_start);
}

// One CTA per (query, slice of kInvSlice of the n rows), the queries of a slice adjacent.
int slice_blocks(int64_t nq, int64_t n, unsigned* blocks) {
  const int64_t b = nq * ((n + kInvSlice - 1) / kInvSlice);
  if (b > 0x7fffffffll) return fail(EPS_ERR_UNSUPPORTED, "posting lists: too many queries in one launch");
  *blocks = static_cast<unsigned>(b);
  return EPS_OK;
}

// The score kernel over the covered rows [row_start, row_start + covered).
int score(Index* ix, const InvertedDist& inv, int metric, int64_t row_start, int64_t covered, float* D, int64_t ldd,
          uint64_t* launches) {
  unsigned blocks = 0;
  EPS_TRY(slice_blocks(inv.scan.nq, covered, &blocks));
  EPS_TRY(inv.plan(ix, launches));
  const auto kernel = metric == EPS_METRIC_IP       ? inverted_score_kernel<EPS_METRIC_IP>
                      : metric == EPS_METRIC_COSINE ? inverted_score_kernel<EPS_METRIC_COSINE>
                                                    : inverted_score_kernel<EPS_METRIC_L2>;
  const SparseQueries& q = inv.scan.q;
  kernel<<<blocks, kInvThreads, 0, ix->stream>>>(ix->d_inv_post, ix->s_inv_plan.as<longlong2>(), q.ptr,
                                                 q.elems + inv.elem_base, inv.elem_base, q.norm2, ix->d_sp_norm2,
                                                 ix->d_sp_ptr, inv.scan.nq, row_start, covered, D, ldd);
  EPS_CUDA(cudaGetLastError());
  ++*launches;
  return EPS_OK;
}

// The handle's count of re-scored pairs, created at its first use.
int rescored_counter(Index* ix, unsigned long long** p) {
  if (!ix->d_l2_rescored) {
    EPS_TRY(ix->d_l2_rescored.reserve(8));
    EPS_CUDA(cudaMemsetAsync(ix->d_l2_rescored, 0, 8, ix->stream));
  }
  *p = ix->d_l2_rescored;
  return EPS_OK;
}

}  // namespace

int InvertedDist::launch(Index* ix, int metric, int64_t row_start, int64_t n, float* D, int64_t ldd,
                         uint64_t* launches) const {
  if (n <= 0 || scan.nq <= 0) return EPS_OK;
  const int64_t covered = covered_rows(ix, row_start, n);
  if (covered > 0) {
    if (metric != EPS_METRIC_IP && metric != EPS_METRIC_COSINE)
      return fail(EPS_ERR_UNSUPPORTED, "inverted index: only inner-product and cosine distances are read from postings");
    EPS_TRY(score(ix, *this, metric, row_start, covered, D, ldd, launches));
  }
  if (covered < n) return scan.launch(ix, metric, row_start + covered, n - covered, D + covered, ldd, launches);
  return EPS_OK;
}

int SparseL2Screen::bounds(Index* ix, int64_t row_start, int64_t n, float* D, int64_t ldd, uint64_t* launches) const {
  if (n <= 0 || inv.scan.nq <= 0) return EPS_OK;
  const int64_t covered = covered_rows(ix, row_start, n);
  if (covered > 0) EPS_TRY(score(ix, inv, EPS_METRIC_L2, row_start, covered, D, ldd, launches));
  if (covered < n)
    return inv.scan.launch(ix, EPS_METRIC_L2, row_start + covered, n - covered, D + covered, ldd, launches);
  return EPS_OK;
}

int SparseL2Screen::threshold(Index* ix, const unsigned long long* keys, int k, float* T, uint64_t* launches) const {
  const SparseQueries& q = inv.scan.q;
  if (inv.scan.nq <= 0) return EPS_OK;
  if (inv.scan.nq > 0x7fffffffll) return fail(EPS_ERR_UNSUPPORTED, "L2 screen: too many queries in one launch");
  unsigned long long* cnt = nullptr;
  EPS_TRY(rescored_counter(ix, &cnt));
  l2_threshold_kernel<<<static_cast<unsigned>(inv.scan.nq), kL2Threads, 0, ix->stream>>>(
      ix->d_sp_ptr, ix->d_sp_elems, ix->inv_rows, q.ptr, q.elems, keys, k, T, cnt);
  EPS_CUDA(cudaGetLastError());
  ++*launches;
  return EPS_OK;
}

int SparseL2Screen::rescore(Index* ix, int64_t row_start, int64_t n, float* D, int64_t ldd, const float* T,
                            const uint32_t* pass, int64_t pass_base, int64_t self_base, uint64_t* launches) const {
  const int64_t covered = n > 0 ? covered_rows(ix, row_start, n) : 0;
  if (covered <= 0 || inv.scan.nq <= 0) return EPS_OK;
  unsigned blocks = 0;
  EPS_TRY(slice_blocks(inv.scan.nq, covered, &blocks));
  unsigned long long* cnt = nullptr;
  EPS_TRY(rescored_counter(ix, &cnt));
  const SparseQueries& q = inv.scan.q;
  l2_rescore_kernel<<<blocks, kL2Threads, 0, ix->stream>>>(ix->d_sp_ptr, ix->d_sp_elems, q.ptr, q.elems, T, pass,
                                                           pass_base, self_base, inv.scan.nq, row_start, covered, D,
                                                           ldd, cnt);
  EPS_CUDA(cudaGetLastError());
  ++*launches;
  return EPS_OK;
}

}  // namespace eps
