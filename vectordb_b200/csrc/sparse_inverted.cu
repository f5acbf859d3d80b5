// Inverted index of a sparse IP / cosine field (eps_index_build_sparse_inverted, DESIGN.md §K5): per-term posting lists
// of rows [0, inv_rows), from which the exact scan's distance tile is computed instead of merging every (query, row)
// pair.
//
// Why the tile is bitwise the scan's: for IP and cosine the reference adds the matched products row[i] * query[i] in
// increasing index order, from 0 (engine/db/vector.cpp:7-47).  inverted_score_kernel walks a query's elements in their
// (increasing) index order and adds each term's posting value times the query value into a per-row fp32 accumulator
// that starts at 0, with __fmul_rn / __fadd_rn: every row sees the same operations in the same order as in SparseMerge
// (common.cuh), and the tile finishes through sparse_finish like every other sparse distance.  A row that matches
// nothing keeps 0, as in the merge.  L2 cannot be served: its merged order also adds the row-only and query-only terms.
//
// Build: expand the CSR elements of rows [0, n) to (index, {row, value}) pairs, sort them by index with a stable radix
// sort (rows stay ascending within a term), flag the first posting of each term and take the int64 exclusive sum of the
// flags (term slots), then scatter the terms and their offsets.  The new arrays replace the old ones only when every
// step has succeeded.
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

// One warp per row: element p of row r becomes the pair (index, {r, value bits}) at position p (row_ptr[0] = 0).
__global__ void inverted_expand_kernel(const int64_t* __restrict__ row_ptr, const uint2* __restrict__ elems, int64_t n,
                                       uint32_t* __restrict__ keys, uint2* __restrict__ vals) {
  const int64_t r = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const int64_t p1 = row_ptr[r + 1];
  for (int64_t p = row_ptr[r] + lane; p < p1; p += 32) {
    const uint2 e = elems[p];
    keys[p] = e.x;
    vals[p] = make_uint2(static_cast<uint32_t>(r), e.y);
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

template <int METRIC>
__global__ void __launch_bounds__(kInvThreads) inverted_score_kernel(
    const uint2* __restrict__ post, const longlong2* __restrict__ plan, const int64_t* __restrict__ q_ptr,
    const uint2* __restrict__ q_elems, int64_t elem_base, const float* __restrict__ q_norm2,
    const float* __restrict__ row_norm2, int64_t nq, int64_t row_start, int64_t n, float* __restrict__ D, int64_t ldd) {
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
  if (METRIC == EPS_METRIC_COSINE) qn = q_norm2[q];
  float* out = D + q * ldd + (r0 - row_start);
  for (int i = threadIdx.x; i < rows; i += kInvThreads) {
    float rn = 0.f;
    if (METRIC == EPS_METRIC_COSINE) rn = row_norm2[r0 + i];
    out[i] = sparse_finish<METRIC>(acc[i], rn, qn);
  }
}

unsigned blocks_for(int64_t threads, int per_block) { return static_cast<unsigned>((threads + per_block - 1) / per_block); }

}  // namespace

int build_sparse_inverted(Index* ix, int64_t n) {
  if (n == 0) {
    ix->d_inv_terms.release();
    ix->d_inv_ptr.release();
    ix->d_inv_post.release();
    ix->inv_rows = ix->inv_terms = ix->inv_postings = 0;
    return EPS_OK;
  }
  int64_t P = 0;
  EPS_CUDA(cudaMemcpyAsync(&P, ix->d_sp_ptr + n, 8, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
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
  inverted_expand_kernel<<<blocks_for(n * 32, 256), 256, 0, ix->stream>>>(ix->d_sp_ptr, ix->d_sp_elems, n, keys_a, vals_a);
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
  // every step succeeded: install (the previous arrays go out with the temporaries)
  ix->d_inv_terms.swap(terms);
  ix->d_inv_ptr.swap(ptr);
  ix->d_inv_post.swap(post);
  ix->inv_rows = n;
  ix->inv_terms = T;
  ix->inv_postings = P;
  return EPS_OK;
}

int InvertedDist::launch(Index* ix, int metric, int64_t row_start, int64_t n, float* D, int64_t ldd,
                         uint64_t* launches) const {
  if (n <= 0 || scan.nq <= 0) return EPS_OK;
  const int64_t nq = scan.nq;
  const int64_t covered = std::max<int64_t>(0, std::min(row_start + n, ix->inv_rows) - row_start);
  if (covered > 0) {
    if (metric != EPS_METRIC_IP && metric != EPS_METRIC_COSINE)
      return fail(EPS_ERR_UNSUPPORTED, "inverted index: only inner-product and cosine distances are read from postings");
    const int64_t blocks = nq * ((covered + kInvSlice - 1) / kInvSlice);
    if (blocks > 0x7fffffffll) return fail(EPS_ERR_UNSUPPORTED, "inverted index: too many queries in one launch");
    if (!planned) {
      EPS_TRY(ix->s_inv_plan.reserve(static_cast<size_t>(n_elems) * sizeof(longlong2)));
      if (n_elems > 0) {
        inverted_plan_kernel<<<blocks_for(n_elems, 256), 256, 0, ix->stream>>>(
            ix->d_inv_terms, ix->inv_terms, ix->d_inv_ptr, scan.q.elems + elem_base, n_elems, ix->s_inv_plan.as<longlong2>());
        EPS_CUDA(cudaGetLastError());
        ++*launches;
      }
      planned = true;
    }
    const auto kernel = metric == EPS_METRIC_IP ? inverted_score_kernel<EPS_METRIC_IP> : inverted_score_kernel<EPS_METRIC_COSINE>;
    kernel<<<static_cast<unsigned>(blocks), kInvThreads, 0, ix->stream>>>(ix->d_inv_post, ix->s_inv_plan.as<longlong2>(),
                                                                         scan.q.ptr, scan.q.elems + elem_base, elem_base,
                                                                         scan.q.norm2, ix->d_sp_norm2, nq, row_start,
                                                                         covered, D, ldd);
    EPS_CUDA(cudaGetLastError());
    ++*launches;
  }
  if (covered < n) return scan.launch(ix, metric, row_start + covered, n - covered, D + covered, ldd, launches);
  return EPS_OK;
}

}  // namespace eps
