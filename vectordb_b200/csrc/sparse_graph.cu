// K5 — graph search of sparse-vector queries (EPS_SPARSE_SEARCH_GRAPH).
//
// What the reference computes is SearchImpl at IntraQueryThreads = 1 (vec_search_executor.cpp:446-715, see
// graph_search.cu) with SparseVecDistFunc as the distance (:417-421, :473-475): seed the queue with the L init ids,
// expand the first unchecked entry, reject neighbours with dist > worst-in-queue, insert the rest, k = (r <= k) ? r : k+1.
// The distances come from the exact scan's SparseMerge and sparse_finish (common.cuh), which are bit-exact, so this
// kernel gives the reference's ids, distances and distance-evaluation counts exactly.  As in the dense kernel,
// inserting the fresh neighbours of a chunk of one adjacency row at once is equivalent to inserting them one by one:
// the queue after the merge is the top-L by (distance, id) of the queue and the chunk, and the lowest insert position
// is the merge's p0.
//
// Mapping:
//   * persistent grid, one CTA (128 threads) per in-flight query, queries claimed from an atomic counter;
//   * the sorted queue (L 64-bit keys, [ordered dist][checked][id]) and the query's {index, value} elements (up to
//     kSgQCap; a longer query is read from global memory) live in shared memory;
//   * adjacency: straight from the CSR in chunks of 128 ids (sparse graphs have long navigation rows: the build's
//     repair adds its component entries there), one id per thread;
//   * visited: the per-slot visited set of graph_search.cuh, shared with the dense kernel (its rules are written
//     there); fresh ids are compacted in adjacency order and logged;
//   * distances: one thread per fresh row feeds the row to a SparseMerge against the staged query (a row's fp32 sum is
//     a serial chain whichever way the work is split; 128 chains run side by side); keys below the worst queue entry
//     go to the pending buffer;
//   * merge: the dense kernel's block merge (merge_pending) after every chunk, which also lowers the cursor to the
//     lowest insert position.
#include <algorithm>
#include <climits>

#include "graph_search.cuh"
#include "internal.h"

namespace eps {

constexpr int kSgQCap = 2048;  // query elements staged in shared memory (16 KB)

struct SGArgs {
  const int64_t* row_ptr;         // table CSR: rows' element offsets, {index, value} elements, fp32 |row|^2
  const uint2* elems;
  const float* row_norm2;
  const int64_t* offsets;         // graph CSR
  const int32_t* nbrs;
  const int32_t* init_ids;        // [L] PrepareInitIds
  const int64_t* q_ptr;           // queries (SparseQueries)
  const uint2* q_elems;
  const float* q_norm2;
  uint32_t* vset;                 // visited sets (VisitedSets)
  int vset_cap, vset_shift, vset_max;
  uint32_t* visited;
  int64_t visited_words;
  int32_t* vlog;
  int vlog_cap;
  unsigned long long* out_queue;  // [nq x L]
  int* work_counter;
  unsigned long long* stats;      // counter block (GraphCounter slots)
  int L, Lp, nq;
};

template <int METRIC>
__global__ void __launch_bounds__(kGsThreads) sparse_graph_search_kernel(SGArgs a) {
  extern __shared__ __align__(16) unsigned char sg_smem[];
  unsigned long long* qa = reinterpret_cast<unsigned long long*>(sg_smem);  // [Lp]
  unsigned long long* pend = qa + a.Lp;                                     // [kPC]
  unsigned long long* cs = pend + kPC;                                      // [kPC]
  uint2* qs = reinterpret_cast<uint2*>(cs + kPC);                           // [kSgQCap] the query's elements
  int* pos = reinterpret_cast<int*>(qs + kSgQCap);                          // [kPC]
  int* fresh = pos + kPC;                                                   // [kGsThreads] fresh ids of one chunk
  unsigned* ubits = reinterpret_cast<unsigned*>(fresh + kGsThreads);        // [(Lp + 31) / 32] unchecked-entry bitmap
  __shared__ int s_q, s_npend, s_cursor, s_cid;
  __shared__ int s_wcnt[kGsThreads / 32];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned lane_lt = (1u << lane) - 1u;
  const int L = a.L;
  uint32_t* vset = a.vset + static_cast<int64_t>(blockIdx.x) * a.vset_cap;
  const uint32_t vmask = static_cast<uint32_t>(a.vset_cap) - 1u;
  uint32_t* visited = a.visited + static_cast<int64_t>(blockIdx.x) * a.visited_words;
  int32_t* vlog = a.vlog + static_cast<int64_t>(blockIdx.x) * a.vlog_cap;
  unsigned long long vacc = 0;  // developer build: hash-set accesses
  unsigned long long st_ndist = 0, st_nexp = 0, st_nedge = 0;

  for (;;) {
    __syncthreads();
    if (tid == 0) s_q = atomicAdd(a.work_counter, 1);
    __syncthreads();
    const int q = s_q;
    if (q >= a.nq) break;
    const int64_t qb = a.q_ptr[q], qn_el = a.q_ptr[q + 1] - qb;
    const bool qstaged = qn_el <= kSgQCap;
    if (qstaged)
      for (int64_t i = tid; i < qn_el; i += kGsThreads) qs[i] = a.q_elems[qb + i];
    const uint2* qv = qstaged ? qs : a.q_elems + qb;  // generic pointer: shared or global
    const float qn = METRIC == EPS_METRIC_COSINE ? a.q_norm2[q] : 0.f;
    bool hashed = L <= a.vset_max;  // false: the query has moved to the bitmap
    __syncthreads();

    // ---- seed (InitializeSetLPara): visited, distances, sort ----
    for (int i = tid; i < a.Lp; i += kGsThreads) {
      unsigned long long key = kKeyInf;
      if (i < L) {
        const uint32_t id = static_cast<uint32_t>(a.init_ids[i]);
        visit_seed(vset, vmask, a.vset_shift, visited, hashed, id, vacc);
        key = make_key(sparse_row_dist<METRIC>(a.row_ptr, a.elems, a.row_norm2, id, qv, qn_el, qn), id);
      }
      qa[i] = key;
    }
    if (tid == 0) { s_npend = 0; s_cursor = 0; }
    __syncthreads();
    block_bitonic_sort(qa, a.Lp);
    init_unchecked(ubits, L);
    if (tid == 0) st_ndist += static_cast<unsigned long long>(L);
    uint32_t n_fresh = 0;  // fresh ids of this query so far (block-uniform)

    // ---- best-first loop (SearchImpl) ----
    for (;;) {
      __syncthreads();  // the previous expansion is merged; every thread has read s_cid
      // pick: the first unchecked entry at or after the cursor (warp 0)
      if (warp == 0) {
        const int qpos = first_unchecked(ubits, L, s_cursor, lane);
        if (lane == 0) {
          if (qpos >= 0) {
            qa[qpos] |= kCheckedBit;
            ubits[qpos >> 5] &= ~(1u << (qpos & 31));
            s_cid = static_cast<int>(key_id(qa[qpos]));
            s_cursor = qpos + 1;  // k + 1, lowered by the merges to the lowest insert position (:648-652)
          } else {
            s_cid = -1;
          }
        }
      }
      __syncthreads();
      const int c = s_cid;
      if (c < 0) break;  // no unchecked entry left
      if (tid == 0) ++st_nexp;
      const int64_t e1 = a.offsets[c + 1];
      for (int64_t e = a.offsets[c]; e < e1; e += kGsThreads) {
        const int nslots = static_cast<int>(min(static_cast<int64_t>(kGsThreads), e1 - e));
        // a chunk inserts at most nslots ids (visited-set rules: graph_search.cuh).  Block-uniform.
        if (hashed && static_cast<uint32_t>(L) + n_fresh + static_cast<uint32_t>(nslots) > static_cast<uint32_t>(a.vset_max)) {
          move_to_bitmap(a.init_ids, L, vlog, n_fresh, visited);
          hashed = false;
        }
        // test-and-insert (ExpandOneCandidate :403-406); of two slots racing on one id exactly one finds it fresh
        const int nb = tid < nslots ? __ldg(a.nbrs + e + tid) : -1;
        bool fr = false;
        if (nb >= 0) {
          if (hashed) {
            const uint32_t id = static_cast<uint32_t>(nb), at = vset_probe(vset, vmask, a.vset_shift, id);
            fr = at != kVsetEmpty && vset_settle(vset, vmask, at, atomicCAS(vset + at, kVsetEmpty, id), id, vacc);
          } else {
            const uint32_t bit = 1u << (nb & 31);
            fr = !(atomicOr(&visited[nb >> 5], bit) & bit);
          }
        }
        const unsigned bal = __ballot_sync(kFull, fr);
        if (lane == 0) s_wcnt[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kGsThreads / 32; ++w) {
          if (w == warp) before = total;
          total += s_wcnt[w];
        }
        if (fr) {  // ordered compaction: fresh ids in adjacency order
          const int at = before + __popc(bal & lane_lt);
          fresh[at] = nb;
          if (n_fresh + static_cast<uint32_t>(at) < static_cast<uint32_t>(a.vlog_cap)) vlog[n_fresh + at] = nb;
        }
        __syncthreads();
        // distances, one fresh row per thread; dist > worst-in-queue is rejected (:424), ties by id
        if (tid < total) {
          const uint32_t id = static_cast<uint32_t>(fresh[tid]);
          const float d = sparse_row_dist<METRIC>(a.row_ptr, a.elems, a.row_norm2, id, qv, qn_el, qn);
          const unsigned long long key = make_key(d, id);
          if (key < (qa[L - 1] & kKeyMask)) pend[atomicAdd(&s_npend, 1)] = key;
        }
        n_fresh += static_cast<uint32_t>(total);
        if (tid == 0) {
          st_ndist += static_cast<unsigned long long>(total);
          st_nedge += static_cast<unsigned long long>(nslots);
        }
        __syncthreads();
        const int m = s_npend;
        if (m > 0) merge_pending(qa, pend, cs, pos, m, L, &s_npend, &s_cursor, ubits);  // ends with a block barrier
      }
    }

    // ---- results + visited reset (:711-714) ----
    unsigned long long* out = a.out_queue + static_cast<int64_t>(q) * L;
    for (int i = tid; i < L; i += kGsThreads) out[i] = qa[i];
    reset_visited(vset, a.vset_cap, hashed, visited, a.visited_words, a.init_ids, L, vlog, n_fresh);
  }
#ifdef EPS_GS_PROFILE
  if (vacc) atomicAdd(&a.stats[kGcVsetAccesses], vacc);
#endif
  if (st_ndist) atomicAdd(&a.stats[kGcDist], st_ndist);
  if (st_nexp) atomicAdd(&a.stats[kGcExpand], st_nexp);
  if (st_nedge) atomicAdd(&a.stats[kGcEdges], st_nedge);
}

int sparse_graph_search(Index* ix, const SparseQueries& q, int64_t nq, int64_t L, unsigned long long* d_queue,
                        eps_stats* stats) {
  int Lp = 0;
  EPS_TRY(graph_launch_prologue(ix, L, "sparse_graph_search", &Lp));
  if (nq > INT_MAX) return fail(EPS_ERR_UNSUPPORTED, "sparse graph search: too many queries in one launch");
  const size_t smem = static_cast<size_t>(Lp) * 8 + 2 * kPC * 8 + static_cast<size_t>(kSgQCap) * 8 + kPC * 4 + kGsThreads * 4 +
                      static_cast<size_t>((Lp + 31) / 32) * 4;
  void (*kernel)(SGArgs) = ix->metric == EPS_METRIC_L2 ? sparse_graph_search_kernel<EPS_METRIC_L2>
                           : ix->metric == EPS_METRIC_IP ? sparse_graph_search_kernel<EPS_METRIC_IP>
                                                         : sparse_graph_search_kernel<EPS_METRIC_COSINE>;
  EPS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  int per_sm = 0;
  EPS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kGsThreads, smem));
  if (per_sm < 1) return fail(EPS_ERR_UNSUPPORTED, "sparse graph search: queue does not fit in shared memory");
  const int slots = static_cast<int>(std::min<int64_t>(nq, static_cast<int64_t>(per_sm) * ix->num_sms));
  VisitedSets vis;
  EPS_TRY(prepare_visited(ix, slots, L, &vis));
  EPS_TRY(graph_counters(ix, nq));
  SGArgs a;
  a.row_ptr = ix->d_sp_ptr; a.elems = ix->d_sp_elems; a.row_norm2 = ix->d_sp_norm2;
  a.offsets = ix->d_offsets; a.nbrs = ix->d_nbrs; a.init_ids = ix->d_init_ids;
  a.q_ptr = q.ptr; a.q_elems = q.elems; a.q_norm2 = q.norm2;
  a.vset = vis.vset; a.vset_cap = vis.vset_cap; a.vset_shift = vis.vset_shift; a.vset_max = vis.vset_max;
  a.visited = vis.visited; a.visited_words = vis.words; a.vlog = vis.vlog; a.vlog_cap = vis.vlog_cap;
  a.out_queue = d_queue;
  a.work_counter = reinterpret_cast<int*>(ix->s_misc.as<unsigned long long>() + kGcWork);
  a.stats = ix->s_misc.as<unsigned long long>();
  a.L = static_cast<int>(L); a.Lp = Lp; a.nq = static_cast<int>(nq);
  kernel<<<slots, kGsThreads, smem, ix->stream>>>(a);
  EPS_CUDA(cudaGetLastError());
  if (stats) {
    stats->n_seed += static_cast<uint64_t>(nq) * static_cast<uint64_t>(L);
    stats->kernel_launches += 1;
  }
  return EPS_OK;
}

}  // namespace eps
