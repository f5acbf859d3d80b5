// K2 — batched best-first graph search.  SURVEY.md §8a rows A4-A8.
//
// What the reference computes (engine/db/execution/vec_search_executor.cpp):
//   InitializeSetLPara (:446-485)  seed the queue with the L query-independent init ids, mark them
//                                  visited, sort by (distance,id);
//   SearchImpl (:518-715)          repeatedly expand the first unchecked queue entry;
//   ExpandOneCandidate (:384-444)  for each CSR neighbour: skip if visited, mark, distance, reject if
//                                  dist > worst-in-queue, else AddIntoQueue (:75-117, sorted insert with
//                                  eviction); return the lowest insert position r;
//   k = (r <= k) ? r : k+1 (:648-652); stop when no unchecked entry is left.
//   IntraQueryThreads > 1 (:601-698): the master deals unchecked candidates to workers, which expand them
//   concurrently against a slightly stale bound and merge back — not a pure function of the inputs.
// The queue after one expansion is the top-L by (distance,id) of {queue ∪ unvisited neighbours}, whatever
// the insertion order, and r is the final position of the smallest inserted entry; so evaluating all
// neighbour distances of a vertex in parallel and merging them at once is equivalent (DESIGN.md §K2).
//
// Mapping (ONE kernel, two modes):
//   * persistent grid, one CTA (128 threads) per in-flight query, queries claimed from an atomic counter;
//   * the sorted queue (L 64-bit keys), the query vector, a FIFO of fresh neighbour ids and a RING of row
//     slots live in shared memory;
//   * a neighbour row is brought HBM -> shared memory by ONE 1-D bulk async copy (TMA engine,
//     cp.async.bulk + mbarrier complete_tx) issued by a single lane: no registers are held across the wait,
//     every free ring slot is in flight at once, and the adjacency reads + visited-bitmap atomics of the NEXT
//     candidates run while the rows of the previous ones land;
//   * distances: warps 1-3 own the ring slots (slot s <-> warp 1 + s % 3); a warp waits on the mbarriers of its
//     occupied slots, evaluates up to 8 landed rows with all 32 lanes on every row (float4 from shared memory, the
//     lane's query chunk loaded once, 5 shuffle steps per row), refills its slots from the FIFO and keeps streaming
//     while the FIFO has a backlog; accepted keys (key < worst-in-queue) go to a small pending buffer that is merged
//     into the sorted queue by a block-parallel rank-and-shift, at the latest when the expansion is consumed;
//   * adjacency: fixed-stride rows of 64 int32 ids (one 256-byte read from the vertex id; longer rows
//     continue in the CSR); visited: one bitmap per in-flight query in global memory, atomicOr test-and-set,
//     cleared by the CTA after the query like the reference clears its vector<bool> (:711-714) — on large tables
//     only the words the query touched, from a log of its fresh ids.
// every iteration picks up to W (the search width) unchecked candidates, and the next pick waits until all their rows
//   are consumed and merged.  Width 1 has the visit order, results and distance-evaluation counts of the reference
//   at IntraQueryThreads = 1; widths 2..8 expand W candidates together — the device analogue of IntraQueryThreads > 1,
//   not bit-identical to the sequential order but, unlike that racy mode, the same on every run: the queue after a
//   merge is the best L of the queue and all fresh rows, whatever order the rows land in.
#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "async.cuh"
#include "internal.h"

namespace eps {

constexpr int kEll = 64;        // adjacency ids per fixed-stride row
constexpr int kGsThreads = 128;
constexpr int kMaxW = 8;        // candidates picked per iteration (upper bound)
constexpr int kPC = 128;        // accepted keys pending their merge (= one key per thread in the merge)
constexpr int kMaxS = 8;        // ring slots per consumer warp (upper bound)
constexpr int kMaxR = 24;       // ring slots (upper bound: 3 consumer warps x kMaxS)
constexpr int kRounds = kMaxW * kEll / kGsThreads;  // adjacency slots per thread

// Developer build only (make EXTRA=-DEPS_GS_PROFILE): per-phase cycle counters of warp 0 (pick / adjacency / merge /
// barrier waits) and of warp 1 (row wait / row math), summed over CTAs into stats[8..15].  Compiled out otherwise.
#ifdef EPS_GS_PROFILE
#define GS_T(var) const long long var = clock64()
#define GS_ACC(slot, t0, t1) do { if (lane == 0) prof[slot] += (t1) - (t0); } while (0)
#else
#define GS_T(var) do {} while (0)
#define GS_ACC(slot, t0, t1) do {} while (0)
#endif

struct GSArgs {
  const float* vectors;
  const int64_t* offsets;
  const int32_t* nbrs;
  const int32_t* ell;             // [n x kEll], -1 padded
  const int32_t* init_ids;
  const float* seed_dist;         // [nq x seed_ld] distances of the seed set (dense tile product)
  const float* queries;
  uint32_t* visited;              // [slots x visited_words]
  int32_t* vlog;                  // [slots x vlog_cap] ids whose bit the running query has set, in FIFO order (visited reset)
  int vlog_cap;
  unsigned long long* out_queue;  // [nq x L]
  int* work_counter;
  unsigned long long* stats;      // n_dist, n_expand, n_edges
  int64_t visited_words;
  int64_t seed_ld;
  int dim, metric, vec4;
  int L, Lp;
  int nq;
  int W;                          // candidates per iteration (the search width)
  int R;                          // ring slots (slot s is owned by consumer warp s % 3)
  int fc;                         // fresh-id FIFO capacity (power of two)
  unsigned long long* qtimes;     // developer build: [nq x 2] globaltimer at query start / end (null otherwise)
  int slot_bytes;                 // ring slot pitch (row bytes, multiple of 16); 0 when rows are not staged
};

__device__ __forceinline__ int lb_masked(const unsigned long long* a, int n, unsigned long long key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if ((a[mid] & kKeyMask) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

template <bool L2>
__device__ __forceinline__ void acc4(const float4& x, const float4& y, float& a) {
  if (L2) {
    float d;
    d = x.x - y.x; a = fmaf(d, d, a); d = x.y - y.y; a = fmaf(d, d, a);
    d = x.z - y.z; a = fmaf(d, d, a); d = x.w - y.w; a = fmaf(d, d, a);
  } else {
    a = fmaf(x.x, y.x, a); a = fmaf(x.y, y.y, a); a = fmaf(x.z, y.z, a); a = fmaf(x.w, y.w, a);
  }
}
// Distances of up to S landed rows (ring slots of ONE consumer warp) to the query, all 32 lanes on every row: lane l
// covers float4 chunks l, l + 32, ...; a query chunk is loaded once per trip and used against all S rows, so shared-
// memory traffic per row is (1 + 1/S) chunks instead of 2.  `mask` bit s = row s is occupied; row s lives at first + s * step.
template <bool L2, int S>
__device__ __forceinline__ void warp_rows_vec4(const unsigned char* first, uint32_t step, unsigned mask, const float4* __restrict__ q,
                                               int dim4, int lane, float (&out)[S]) {
  float acc[S];
#pragma unroll
  for (int s = 0; s < S; ++s) acc[s] = 0.f;
  for (int c = lane; c < dim4; c += 32) {
    const float4 y = q[c];
#pragma unroll
    for (int s = 0; s < S; ++s)
      if ((mask >> s) & 1u) acc4<L2>(reinterpret_cast<const float4*>(first + s * step)[c], y, acc[s]);
  }
#pragma unroll
  for (int s = 0; s < S; ++s) out[s] = warp_sum(acc[s]);
}
// rows not staged (dim % 4 != 0 or a misaligned table): lanes stride the scalars of the global rows
template <bool L2, int S>
__device__ __forceinline__ void warp_rows_scalar(const float* const (&rows)[S], unsigned mask, const float* __restrict__ q, int dim,
                                                 int lane, float (&out)[S]) {
  float acc[S];
#pragma unroll
  for (int s = 0; s < S; ++s) acc[s] = 0.f;
  for (int i = lane; i < dim; i += 32) {
    const float y = q[i];
#pragma unroll
    for (int s = 0; s < S; ++s) {
      if ((mask >> s) & 1u) {
        const float x = __ldg(rows[s] + i);
        if (L2) { const float d = x - y; acc[s] = fmaf(d, d, acc[s]); } else { acc[s] = fmaf(x, y, acc[s]); }
      }
    }
  }
#pragma unroll
  for (int s = 0; s < S; ++s) out[s] = warp_sum(acc[s]);
}

// Consumer step of one warp over its S slots (slot of local index s = cw + 3 s): wait for the landed rows, distances,
// accepted keys to the pending buffer.  Returns nothing; the caller refills the slots.
template <int S>
__device__ __forceinline__ void consume_slots(const GSArgs& a, unsigned occ_mask, unsigned par_mask, int cw, int lane, bool staged,
                                              const unsigned char* ring, uint32_t bar0, const float* qv, const int* slot_id,
                                              unsigned long long bound, unsigned long long* pend, int* s_npend) {
  float d[S];
  if (staged) {
#pragma unroll
    for (int s = 0; s < S; ++s)
      if ((occ_mask >> s) & 1u) mbar_wait(bar0 + 8 * (cw + 3 * s), (par_mask >> s) & 1u);
    const unsigned char* first = ring + static_cast<size_t>(cw) * a.slot_bytes;
    const uint32_t step = 3u * static_cast<uint32_t>(a.slot_bytes);
    if (a.metric == EPS_METRIC_L2) warp_rows_vec4<true, S>(first, step, occ_mask, reinterpret_cast<const float4*>(qv), a.dim >> 2, lane, d);
    else warp_rows_vec4<false, S>(first, step, occ_mask, reinterpret_cast<const float4*>(qv), a.dim >> 2, lane, d);
  } else {
    const float* rows[S];
#pragma unroll
    for (int s = 0; s < S; ++s) rows[s] = a.vectors + static_cast<int64_t>(((occ_mask >> s) & 1u) ? slot_id[cw + 3 * s] : 0) * a.dim;
    if (a.metric == EPS_METRIC_L2) warp_rows_scalar<true, S>(rows, occ_mask, qv, a.dim, lane, d);
    else warp_rows_scalar<false, S>(rows, occ_mask, qv, a.dim, lane, d);
  }
  // lane s publishes row s
  float mine = 0.f;
#pragma unroll
  for (int s = 0; s < S; ++s) if (lane == s) mine = d[s];
  if (lane < S && ((occ_mask >> lane) & 1u)) {
    const unsigned long long key = make_key(finish_metric(a.metric, mine), static_cast<uint32_t>(slot_id[cw + 3 * lane]));
    if (key < bound) pend[atomicAdd(s_npend, 1)] = key;  // dist > bound rejected (:424); ties by id
  }
}

// Block-wide merge of the m (<= kPC) pending keys into the sorted queue qa[0..L): sort by counting, binary-search
// the insertion points, shift the tail in place in super-tiles of 8 keys per thread (each key moves right by the
// number of pending keys that precede it), drop the keys into the holes.  Entries pushed past L are evicted
// (AddIntoQueue's drop-worst, :104-108).  Returns the lowest insert position through *s_cursor (min).
__device__ __forceinline__ void merge_pending(unsigned long long* qa, unsigned long long* pend, unsigned long long* cs, int* pos,
                                              int m, int L, int* s_npend, int* s_cursor, unsigned* ubits) {
  const int tid = threadIdx.x;
  if (tid < m) {
    const unsigned long long key = pend[tid];
    int r = 0;
    for (int j = 0; j < m; ++j) r += ((pend[j] & kKeyMask) < (key & kKeyMask));
    cs[r] = key;
  }
  __syncthreads();
  if (tid < m) pos[tid] = lb_masked(qa, L, cs[tid] & kKeyMask);
  __syncthreads();
  const int p0 = pos[0];
  for (int hi = L; hi > p0; hi -= 8 * kGsThreads) {
    unsigned long long kreg[8];
    int dreg[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int j = hi - 1 - (u * kGsThreads + tid);
      dreg[u] = L;
      if (j >= p0) {
        kreg[u] = qa[j];
        int sft = 0;
        if (m <= 8) { for (int i = 0; i < m; ++i) sft += (pos[i] <= j); }
        else { int lo = 0, up = m; while (lo < up) { const int mid = (lo + up) >> 1; if (pos[mid] <= j) lo = mid + 1; else up = mid; } sft = lo; }
        dreg[u] = j + sft;
      }
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < 8; ++u) if (dreg[u] < L) qa[dreg[u]] = kreg[u];
    __syncthreads();
  }
  if (tid < m) {
    const int f = pos[tid] + tid;
    if (f < L) qa[f] = cs[tid];
  }
  if (tid == 0) {
    *s_npend = 0;
    if (p0 < *s_cursor) *s_cursor = p0;
  }
  __syncthreads();
  // the unchecked-entry bitmap (one bit per queue slot, what the pick scans) from the first changed word on
  if (p0 < L) {
    const int nwords = (L + 31) >> 5, lane = tid & 31;
    for (int w = (p0 >> 5) + (tid >> 5); w < nwords; w += kGsThreads / 32) {
      const int idx = w * 32 + lane;
      const unsigned b = __ballot_sync(kFull, idx < L && !(qa[idx] & kCheckedBit));
      if (lane == 0) ubits[w] = b;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kGsThreads, 7) graph_search_kernel(GSArgs a) {
  extern __shared__ __align__(128) unsigned char gs_smem[];
  const int dim4p = (a.dim + 3) & ~3;
  unsigned char* ring = gs_smem;                                                                   // [R][slot_bytes]
  unsigned long long* qa = reinterpret_cast<unsigned long long*>(ring + static_cast<size_t>(a.R) * a.slot_bytes);  // [Lp]
  unsigned long long* pend = qa + a.Lp;                                                            // [kPC]
  unsigned long long* cs = pend + kPC;                                                             // [kPC]
  unsigned long long* bars = cs + kPC;                                                             // [kMaxR]
  float* qv = reinterpret_cast<float*>(bars + kMaxR);                                              // [dim4p]
  int* pos = reinterpret_cast<int*>(qv + dim4p);                                                   // [kPC]
  int* fifo = pos + kPC;                                                                           // [fc]
  int* slot_id = fifo + a.fc;                                                                      // [kMaxR] row id in each ring slot
  unsigned* ubits = reinterpret_cast<unsigned*>(slot_id + kMaxR);                                  // [(Lp + 31) / 32] unchecked-entry bitmap
  __shared__ int s_q, s_ncur, s_cursor, s_npend, s_ncont;
  __shared__ unsigned s_head;                      // FIFO entries [s_head, fifo_tail) are not yet issued to the ring
  __shared__ int s_cid[kMaxW];
  __shared__ int s_wcnt[kRounds][kGsThreads / 32];
  __shared__ long long s_cont_e[kMaxW], s_cont_end[kMaxW];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // warp 0 picks candidates and leads the adjacency step; warps 1-3 are the row consumers: ring slot s belongs to
  // consumer warp s % 3 for the whole kernel (local index s / 3, at most kMaxS per warp)
  const int cw = warp - 1;
  const unsigned lane_lt = (1u << lane) - 1u;
  const int L = a.L, R = a.R, W = a.W;
  const unsigned fmask = static_cast<unsigned>(a.fc) - 1u;
  const bool staged = a.slot_bytes > 0;
  const uint32_t ring0 = smem_u32(ring), bar0 = smem_u32(bars);
  const uint32_t row_bytes = static_cast<uint32_t>(a.dim) * 4u;
  uint32_t* visited = a.visited + static_cast<int64_t>(blockIdx.x) * a.visited_words;
  int32_t* vlog = a.vlog + static_cast<int64_t>(blockIdx.x) * a.vlog_cap;

  if (tid == 0) {
    for (int s = 0; s < R; ++s) mbar_init(bar0 + 8 * s, 1);
    mbar_fence_init();
  }
  // The owning warp issues the bulk copy into a slot, waits on its mbarrier, reads it and refills it — no block
  // barrier guards a slot.  Per-slot state (occupied, mbarrier phase parity) is a pair of warp-uniform bit masks.
  unsigned occ_mask = 0u, par_mask = 0u;
  const int n_own = cw >= 0 ? (R - cw + 2) / 3 : 0;  // slots cw, cw + 3, ... < R
  unsigned long long st_ndist = 0, st_nexp = 0, st_nedge = 0;
#ifdef EPS_GS_PROFILE
  long long prof[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // 0 barrier X, 1 merge, 2 row wait, 3 row math, 4 pick, 5 barrier 1, 6 adjacency+visited, 7 barrier 2 + FIFO
  const long long t_kernel0 = clock64();
#endif

  for (;;) {
    __syncthreads();
    if (tid == 0) s_q = atomicAdd(a.work_counter, 1);
    __syncthreads();
    const int q = s_q;
    if (q >= a.nq) break;
#ifdef EPS_GS_PROFILE
    if (tid == 0 && a.qtimes) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); a.qtimes[4 * q] = t; }
    const unsigned long long prof_nd0 = st_ndist;
    unsigned long long prof_iters = 0;
#endif

    // ---- seed (InitializeSetLPara): precomputed distances of the query-independent seed set ----
    for (int i = tid; i < a.dim; i += kGsThreads) qv[i] = a.queries[static_cast<int64_t>(q) * a.dim + i];
    for (int i = a.dim + tid; i < dim4p; i += kGsThreads) qv[i] = 0.f;
    for (int i = tid; i < a.Lp; i += kGsThreads) {
      unsigned long long key = kKeyInf;
      if (i < L) {
        const uint32_t id = static_cast<uint32_t>(a.init_ids[i]);
        atomicOr(&visited[id >> 5], 1u << (id & 31));
        key = make_key(a.seed_dist[static_cast<int64_t>(q) * a.seed_ld + i], id);
      }
      qa[i] = key;
    }
    if (tid == 0) { s_npend = 0; s_ncont = 0; s_cursor = 0; s_ncur = 0; s_head = 0u; }
    __syncthreads();
    block_bitonic_sort(qa, a.Lp);
    for (int w = tid; w < ((L + 31) >> 5); w += kGsThreads)  // every seed starts unchecked
      ubits[w] = (w * 32 + 32 <= L) ? 0xffffffffu : ((1u << (L & 31)) - 1u);
    if (tid == 0) st_ndist += static_cast<unsigned long long>(L);
    uint32_t fifo_tail = 0;

    // ---- best-first loop (SearchImpl) ----
    for (;;) {
#ifdef EPS_GS_PROFILE
      ++prof_iters;
#endif
      // barrier X: pending appends, FIFO writes and slot states of the previous iteration are settled;
      // the count is the number of ring slots with a row in flight
      GS_T(tx0);
      const int inflight = __syncthreads_count(lane < kMaxS && ((occ_mask >> lane) & 1u));
      GS_T(tx1);
      GS_ACC(0, tx0, tx1);
      const int m = s_npend;
      const uint32_t head = s_head;
      const int ncont = s_ncont;
      // -- D: merge the pending keys --
      const bool merged = m > 0;
      // s_npend / s_head are bumped by the consumer phase below: no thread may get there before EVERY thread has taken
      // the snapshot above (the merge's own barriers do that when there is a merge)
      if (merged) merge_pending(qa, pend, cs, pos, m, L, &s_npend, &s_cursor, ubits);
      else __syncthreads();
      GS_T(tm1);
      GS_ACC(1, tx1, tm1);
      const bool idle = inflight == 0 && head == fifo_tail;
      // A runs when the previous expansion has been consumed and merged
      const bool want = idle;

      // -- C/B, per consumer warp: distances of the landed rows of its slots, then refill every slot from the FIFO.
      // The warp keeps streaming (consume, refill, consume ...) without coming back to the block barrier while the FIFO
      // has a backlog and the pending buffer has room: its slots stay in flight for the whole backlog instead of one ring
      // pass per block iteration.  It leaves with its last refills in flight, so that the pick / adjacency / visited
      // phases below overlap them.  Accepting against the bound of the last merge only lets more keys into the pending
      // buffer (the bound never grows); the merge evicts them, so the queue after the merge is the same.
      if (n_own > 0) {
        const unsigned long long bound = qa[L - 1] & kKeyMask;  // worst entry as of the last merge (:546)
        for (;;) {
          if (occ_mask) {
            GS_T(tw0);
            if (n_own <= 1) consume_slots<1>(a, occ_mask, par_mask, cw, lane, staged, ring, bar0, qv, slot_id, bound, pend, &s_npend);
            else if (n_own <= 2) consume_slots<2>(a, occ_mask, par_mask, cw, lane, staged, ring, bar0, qv, slot_id, bound, pend, &s_npend);
            else if (n_own <= 4) consume_slots<4>(a, occ_mask, par_mask, cw, lane, staged, ring, bar0, qv, slot_id, bound, pend, &s_npend);
            else consume_slots<8>(a, occ_mask, par_mask, cw, lane, staged, ring, bar0, qv, slot_id, bound, pend, &s_npend);
            par_mask ^= occ_mask;
            GS_T(tw1);
            GS_ACC(3, tw0, tw1);
          }
          __syncwarp();  // every lane has finished reading the slots
          bool got = false;
          if (lane < n_own) {
            const unsigned idx = atomicAdd(&s_head, 1u);
            if (idx >= fifo_tail) atomicSub(&s_head, 1u);  // nothing left: hand the index back
            else {
              const int slot = cw + 3 * lane;
              const int id = fifo[idx & fmask];
              slot_id[slot] = id;
              got = true;
              if (staged) {
                const uint32_t bar = bar0 + 8 * slot;
                mbar_expect_tx(bar, row_bytes);
                bulk_load_1d(ring0 + slot * static_cast<uint32_t>(a.slot_bytes), a.vectors + static_cast<int64_t>(id) * a.dim, row_bytes, bar);
              }
            }
          }
          occ_mask = __ballot_sync(kFull, got);
          // go round again only with a full set of refills (the FIFO had at least n_own entries for this warp), a
          // backlog behind them, and room for every slot of the ring in the pending buffer
          if (__popc(occ_mask) < n_own) break;
          const unsigned head_now = *reinterpret_cast<volatile unsigned*>(&s_head);
          const int npend_now = *reinterpret_cast<volatile int*>(&s_npend);
          if (head_now >= fifo_tail || npend_now + R > kPC) break;
        }
      }
      if (!want) continue;
      GS_T(tp0);

      // -- A0: pick up to W unchecked candidates, smallest first, from queue ∪ pending (warp 0) --
      if (warp == 0) {
        int cnt = 0;
        if (ncont == 0) {
          const int np = merged ? 0 : m;  // entries appended during this iteration's consumer phase are picked next time
          int sp = s_cursor;
          unsigned long long pk[kPC / 32];
#pragma unroll
          for (int u = 0; u < kPC / 32; ++u) {
            const int i = u * 32 + lane;
            pk[u] = ~0ull;
            if (i < np) { const unsigned long long k = pend[i]; if (!(k & kCheckedBit)) pk[u] = k; }
          }
          unsigned long long pmin = ~0ull;  // smallest unchecked pending key
          bool pscan = np > 0;
          while (cnt < W) {
            int qpos = -1;
            {
              const int nwords = (L + 31) >> 5;
              for (int w0 = sp >> 5; w0 < nwords; w0 += 32) {
                const int wi = w0 + lane;
                unsigned word = wi < nwords ? ubits[wi] : 0u;
                if (wi == (sp >> 5)) word &= ~((1u << (sp & 31)) - 1u);  // entries before the cursor are checked
                const unsigned b = __ballot_sync(kFull, word != 0u);
                if (b) {
                  const int src = __ffs(b) - 1;
                  const unsigned wsel = __shfl_sync(kFull, word, src);
                  qpos = (w0 + src) * 32 + __ffs(wsel) - 1;
                  break;
                }
              }
            }
            if (qpos < 0) sp = L;  // queue exhausted: later picks of this iteration do not rescan it
            const unsigned long long qkey = qpos >= 0 ? (qa[qpos] & kKeyMask) : ~0ull;
            if (pscan) {
              unsigned long long mn = pk[0];
#pragma unroll
              for (int u = 1; u < kPC / 32; ++u) mn = pk[u] < mn ? pk[u] : mn;
#pragma unroll
              for (int o = 16; o > 0; o >>= 1) {
                const unsigned long long other = __shfl_xor_sync(kFull, mn, o);
                mn = other < mn ? other : mn;
              }
              pmin = mn;
              pscan = false;
            }
            if (qpos < 0 && pmin == ~0ull) break;
            if (qkey <= pmin) {
              if (lane == 0) {
                qa[qpos] |= kCheckedBit;
                ubits[qpos >> 5] &= ~(1u << (qpos & 31));
                s_cid[cnt] = static_cast<int>(key_id(qkey));
              }
              sp = qpos + 1;
            } else {
              // keys are distinct: exactly one lane owns the pending minimum and marks it
#pragma unroll
              for (int u = 0; u < kPC / 32; ++u) {
                if (pk[u] == pmin) {
                  pk[u] = ~0ull;
                  pend[u * 32 + lane] = pmin | kCheckedBit;
                  s_cid[cnt] = static_cast<int>(key_id(pmin));
                }
              }
              pscan = true;
            }
            ++cnt;
            __syncwarp();
          }
          if (lane == 0) s_cursor = sp;
        }
        if (lane == 0) s_ncur = cnt;
      }
      GS_T(tp1);
      GS_ACC(4, tp0, tp1);
      __syncthreads();  // (1)
      GS_T(tb1);
      GS_ACC(5, tp1, tb1);
      const int ncur = s_ncur;
      if (ncur == 0 && ncont == 0) {
        if (idle) break;  // nothing unchecked in queue ∪ pending, nothing in flight, nothing queued: done
        continue;         // candidates may still come out of the rows in flight
      }

      // -- A1: adjacency ids -> visited test-and-set -> ordered compaction of the fresh ids into the FIFO --
      const bool cont_mode = ncur == 0;  // draining the CSR continuation of a row longer than kEll
      long long e0 = 0;
      int nslots = ncur * kEll;
      if (cont_mode) {
        e0 = s_cont_e[ncont - 1];
        nslots = static_cast<int>(min(static_cast<long long>(kGsThreads), s_cont_end[ncont - 1] - e0));
      }
      int nb[kRounds];
      unsigned bal[kRounds];
      bool fr[kRounds];
#pragma unroll
      for (int r = 0; r < kRounds; ++r) {
        const int s = r * kGsThreads + tid;
        nb[r] = -1;
        if (s < nslots)
          nb[r] = cont_mode ? a.nbrs[e0 + s] : __ldg(a.ell + static_cast<int64_t>(s_cid[s >> 6]) * kEll + (s & (kEll - 1)));
      }
#pragma unroll
      for (int r = 0; r < kRounds; ++r) {
        fr[r] = false;
        if (nb[r] >= 0) {
          const uint32_t bit = 1u << (nb[r] & 31);
          fr[r] = !(atomicOr(&visited[nb[r] >> 5], bit) & bit);  // ExpandOneCandidate :403-406
        }
      }
#pragma unroll
      for (int r = 0; r < kRounds; ++r) {
        bal[r] = __ballot_sync(kFull, fr[r]);
        const unsigned vb = __ballot_sync(kFull, nb[r] >= 0);
        if (lane == 0) { s_wcnt[r][warp] = __popc(bal[r]); st_nedge += static_cast<unsigned long long>(__popc(vb)); }
      }
      GS_T(ta1);
      GS_ACC(6, tb1, ta1);
      __syncthreads();  // (2)
      int total = 0;
#pragma unroll
      for (int r = 0; r < kRounds; ++r) {
        int mine = 0;
#pragma unroll
        for (int w = 0; w < kGsThreads / 32; ++w) {
          if (w == warp) mine = total;
          total += s_wcnt[r][w];
        }
        if (fr[r]) {
          const uint32_t at = fifo_tail + static_cast<uint32_t>(mine + __popc(bal[r] & lane_lt));
          fifo[at & fmask] = nb[r];
          if (at < static_cast<uint32_t>(a.vlog_cap)) vlog[at] = nb[r];
        }
      }
      fifo_tail += static_cast<uint32_t>(total);
      if (cont_mode) {
        if (tid == 0) {
          s_cont_e[ncont - 1] = e0 + nslots;
          if (e0 + nslots >= s_cont_end[ncont - 1]) s_ncont = ncont - 1;
        }
      } else {
        // a full fixed-stride row may continue in the CSR (rare: repair hubs, reference graphs above 64)
#pragma unroll
        for (int r = 0; r < kRounds; ++r) {
          const int s = r * kGsThreads + tid;
          if (s < nslots && (s & (kEll - 1)) == kEll - 1 && nb[r] >= 0) {
            const int c = s_cid[s >> 6];
            const long long eb = a.offsets[c] + kEll, ee = a.offsets[c + 1];
            if (ee > eb) {
              const int i = atomicAdd(&s_ncont, 1);
              s_cont_e[i] = eb;
              s_cont_end[i] = ee;
            }
          }
        }
        if (tid == 0) st_nexp += static_cast<unsigned long long>(ncur);
      }
      if (tid == 0) st_ndist += static_cast<unsigned long long>(total);
      GS_T(tf1);
      GS_ACC(7, ta1, tf1);
    }

    // ---- results + visited reset (:711-714) ----
    {
      const int m = s_npend;  // only checked entries can be left (the last pick found nothing unchecked)
      if (m > 0) merge_pending(qa, pend, cs, pos, m, L, &s_npend, &s_cursor, ubits);
    }
    unsigned long long* out = a.out_queue + static_cast<int64_t>(q) * L;
    for (int i = tid; i < L; i += kGsThreads) out[i] = qa[i];
#ifdef EPS_GS_PROFILE
    if (tid == 0 && a.qtimes) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      a.qtimes[4 * q + 1] = t; a.qtimes[4 * q + 2] = st_ndist - prof_nd0; a.qtimes[4 * q + 3] = prof_iters;
    }
#endif
    if (fifo_tail <= static_cast<uint32_t>(a.vlog_cap) && 10ll * (fifo_tail + L) < a.visited_words) {
      // large table: clear only the words this query touched (the seeds and the logged fresh ids) instead of
      // streaming zeros over the whole bitmap (1.25 MB per query at 10M rows)
      for (int i = tid; i < L; i += kGsThreads) visited[static_cast<uint32_t>(a.init_ids[i]) >> 5] = 0u;
      for (uint32_t i = tid; i < fifo_tail; i += kGsThreads) visited[static_cast<uint32_t>(vlog[i]) >> 5] = 0u;
    } else {
      uint4* v4 = reinterpret_cast<uint4*>(visited);
      const int64_t n4 = a.visited_words >> 2;
      const uint4 z = make_uint4(0, 0, 0, 0);
      for (int64_t i = tid; i < n4; i += kGsThreads) v4[i] = z;
    }
  }
#ifdef EPS_GS_PROFILE
  if (lane == 0 && warp < 2) {
    for (int i = 0; i < 8; ++i) atomicAdd(&a.stats[8 + warp * 8 + i], static_cast<unsigned long long>(prof[i]));
    if (warp == 0) atomicAdd(&a.stats[24], static_cast<unsigned long long>(clock64() - t_kernel0));
  }
#endif
  if (st_ndist) atomicAdd(&a.stats[0], st_ndist);
  if (st_nexp) atomicAdd(&a.stats[1], st_nexp);
  if (st_nedge) atomicAdd(&a.stats[2], st_nedge);
}

__global__ void csr_to_ell_kernel(const int64_t* __restrict__ offsets, const int32_t* __restrict__ nbrs, int64_t n,
                                  int32_t* __restrict__ ell) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n * kEll) return;
  const int64_t v = i / kEll;
  const int s = static_cast<int>(i % kEll);
  const int64_t e = offsets[v] + s;
  ell[i] = e < offsets[v + 1] ? nbrs[e] : -1;
}

__global__ void gather_rows_kernel(const float* __restrict__ vectors, const int32_t* __restrict__ ids, int n, int dim,
                                   float* __restrict__ out) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(n) * dim) return;
  const int r = static_cast<int>(i / dim), c = static_cast<int>(i % dim);
  out[i] = vectors[static_cast<int64_t>(ids[r]) * dim + c];
}

int gather_rows(Index* ix, const int32_t* d_ids, int64_t n, float* d_out) {
  const int64_t tot = n * ix->dim;
  if (tot <= 0) return EPS_OK;
  gather_rows_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, ix->stream>>>(ix->d_vectors, d_ids, static_cast<int>(n),
                                                                                      static_cast<int>(ix->dim), d_out);
  EPS_CUDA(cudaGetLastError());
  return EPS_OK;
}

// PrepareInitIds (vec_search_executor.cpp:487-516): dedup'd out-neighbours of the navigation point, then
// ids nav+1, nav+2, ... (mod n) until L entries.  Pure index logic on <= L + deg entries; runs on the host
// over the navigation row copied back from the device.  L is clamped to n_indexed by the caller (the
// reference loops forever when L > n_indexed, SURVEY.md Q1).
int prepare_init_ids(Index* ix, int64_t L) {
  if (ix->init_L == L && ix->d_init_ids) return EPS_OK;
  int64_t e[2];
  EPS_CUDA(cudaMemcpyAsync(e, ix->d_offsets + ix->nav, 16, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  std::vector<int32_t> row(static_cast<size_t>(e[1] - e[0]));
  if (!row.empty()) {
    EPS_CUDA(cudaMemcpyAsync(row.data(), ix->d_nbrs + e[0], row.size() * 4, cudaMemcpyDeviceToHost, ix->stream));
    EPS_CUDA(cudaStreamSynchronize(ix->stream));
  }
  std::vector<int32_t> ids;
  ids.reserve(static_cast<size_t>(L));
  std::vector<bool> sel(static_cast<size_t>(ix->n_indexed), false);
  for (size_t i = 0; i < row.size() && static_cast<int64_t>(ids.size()) < L; ++i) {
    int32_t v = row[i];
    if (sel[v]) continue;
    sel[v] = true;
    ids.push_back(v);
  }
  int64_t tmp = ix->nav + 1;
  while (static_cast<int64_t>(ids.size()) < L) {
    if (tmp == ix->n_indexed) tmp = 0;
    int64_t v = tmp++;
    if (sel[v]) continue;
    sel[v] = true;
    ids.push_back(static_cast<int32_t>(v));
  }
  if (ix->d_init_ids) { cudaFree(ix->d_init_ids); ix->d_init_ids = nullptr; }
  EPS_CUDA(cudaMalloc(&ix->d_init_ids, static_cast<size_t>(L) * 4));
  EPS_CUDA(cudaMemcpyAsync(ix->d_init_ids, ids.data(), static_cast<size_t>(L) * 4, cudaMemcpyHostToDevice, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  ix->init_L = L;
  return EPS_OK;
}


// Ring geometry: ~48 KB of row slots per CTA (16 rows at d = 768) unless the index carries a tuning override
// (eps_index_set_graph_tuning); at least 2, at most kMaxR slots.
static int ring_slots_for(const Index* ix, int slot_bytes) {
  if (slot_bytes <= 0) return 16;
  int r = ix->graph_ring_slots > 0 ? ix->graph_ring_slots : (48 * 1024) / slot_bytes;
  return std::max(2, std::min(r, kMaxR));
}

int ensure_ell(Index* ix, uint64_t* launches) {
  if (ix->d_ell || !ix->d_offsets) return EPS_OK;
  EPS_CUDA(cudaMalloc(&ix->d_ell, static_cast<size_t>(ix->n_indexed) * kEll * 4));
  const int64_t tot = ix->n_indexed * kEll;
  csr_to_ell_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, ix->stream>>>(ix->d_offsets, ix->d_nbrs, ix->n_indexed, ix->d_ell);
  EPS_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return EPS_OK;
}

int graph_search(Index* ix, const float* d_queries, int64_t nq, int64_t L, unsigned long long* d_queue,
                 eps_stats* stats) {
  if (L < 1 || L > ix->n_indexed) return fail(EPS_ERR_INVALID_ARGUMENT, "graph_search: L out of range");
  const int Lp = std::max(2, next_pow2(static_cast<int>(L)));
  if (Lp > 16384) return fail(EPS_ERR_UNSUPPORTED, "SearchQueueSize above 16384 is not supported by the graph kernel");
  EPS_TRY(prepare_init_ids(ix, L));
  const int dim = static_cast<int>(ix->dim);
  const int dimp = (dim + 3) & ~3;
  const int width = std::max(1, std::min(ix->search_width, kMaxW));
  const bool staged = ix->vec4;  // 16-byte aligned rows of a multiple of 16 bytes: eligible for bulk async copies
  const int slot_bytes = staged ? dim * 4 : 0;
  int R = ring_slots_for(ix, slot_bytes);
  // FIFO: a backlog below R entries + the ids one A step appends (W adjacency rows or one 128-id continuation chunk)
  const int fc = next_pow2(std::max(width * kEll, kGsThreads) + kMaxR);
  auto smem_for = [&](int r) {
    return static_cast<size_t>(r) * slot_bytes + static_cast<size_t>(Lp) * 8 + 2 * kPC * 8 + kMaxR * 8 +
           static_cast<size_t>(dimp) * 4 + kPC * 4 + static_cast<size_t>(fc) * 4 + kMaxR * 4 + static_cast<size_t>((Lp + 31) / 32) * 4;
  };
  while (R > 2 && smem_for(R) > 200 * 1024) --R;
  if (smem_for(R) > 226 * 1024) return fail(EPS_ERR_UNSUPPORTED, "queue + query + row ring do not fit in shared memory");
  EPS_CUDA(cudaFuncSetAttribute(graph_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_for(R))));
  auto resident = [&](int r, int* out) {
    EPS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(out, graph_search_kernel, kGsThreads, smem_for(r)));
    if (*out < 1) *out = 1;
    if (ix->graph_ctas_per_sm > 0) *out = std::min(*out, ix->graph_ctas_per_sm);
    return EPS_OK;
  };
  int per_sm = 0;
  EPS_TRY(resident(R, &per_sm));
  // Auto geometry.  A batch of nq queries runs in rounds = ceil(nq / resident CTAs) waves of whole queries, and a
  // partly filled last wave is pure loss while the kernel is latency-bound; so among ring sizes >= 4 take the one
  // with the fewest rounds (a smaller ring = more resident queries), the largest ring on ties, and launch exactly
  // ceil(nq / rounds) CTAs so that every CTA serves the same number of queries (profiles/r02_graph_geometry_*).
  auto rounds_of = [&](int p) { return (nq + static_cast<int64_t>(p) * ix->num_sms - 1) / (static_cast<int64_t>(p) * ix->num_sms); };
  if (staged && ix->graph_ring_slots == 0 && rounds_of(per_sm) > 1) {
    int best_r = R, best_p = per_sm;
    for (int r = R - 1; r >= 4; --r) {
      int p = 0;
      EPS_TRY(resident(r, &p));
      if (rounds_of(p) < rounds_of(best_p)) { best_r = r; best_p = p; }
    }
    R = best_r;
    per_sm = best_p;
  }
  const size_t smem = smem_for(R);
  const int64_t rounds = rounds_of(per_sm);
  int slots = static_cast<int>(std::min<int64_t>((nq + rounds - 1) / rounds, static_cast<int64_t>(per_sm) * ix->num_sms));
  if (ix->graph_ring_slots > 0 || ix->graph_ctas_per_sm > 0)  // tuning override: every resident slot, queries claimed dynamically
    slots = static_cast<int>(std::min<int64_t>(nq, static_cast<int64_t>(per_sm) * ix->num_sms));
  const int64_t words = ((ix->n_indexed + 31) / 32 + 3) & ~3ll;
  if (ix->visited_slots < slots || ix->s_visited.cap < static_cast<size_t>(slots) * words * 4) {
    EPS_TRY(ix->s_visited.reserve(static_cast<size_t>(slots) * words * 4));
    ix->visited_slots = slots;
  }
  // bitmaps must start clean; the kernel leaves them clean.  (Re)zero when the geometry changed.
  // (a re-grown buffer may come back at the old address: the capacity is part of the geometry)
  if (ix->vis_clean_ptr != ix->s_visited.p || ix->vis_clean_words != words || ix->vis_clean_cap != ix->s_visited.cap) {
    EPS_CUDA(cudaMemsetAsync(ix->s_visited.p, 0, ix->s_visited.cap, ix->stream));
    ix->vis_clean_ptr = ix->s_visited.p;
    ix->vis_clean_words = words;
    ix->vis_clean_cap = ix->s_visited.cap;
  }
  EPS_TRY(ix->s_misc.reserve(256));  // [0..3] counters, [+32 B] work counter, [8..24] developer phase timers
  EPS_CUDA(cudaMemsetAsync(ix->s_misc.p, 0, 256, ix->stream));
  uint64_t launches = 1;
  EPS_TRY(ensure_ell(ix, &launches));
  if (ix->seed_rows_L != L) {  // contiguous copy of the query-independent seed rows
    EPS_TRY(ix->s_seed_rows.reserve(static_cast<size_t>(L) * ix->dim * 4));
    const int64_t tot = L * ix->dim;
    gather_rows_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, ix->stream>>>(
        ix->d_vectors, ix->d_init_ids, static_cast<int>(L), dim, ix->s_seed_rows.as<float>());
    EPS_CUDA(cudaGetLastError());
    ix->seed_rows_L = L;
    ++launches;
  }
  const int64_t seed_ld = (L + 3) & ~3ll;
  EPS_TRY(ix->s_seed_dist.reserve(static_cast<size_t>(nq) * seed_ld * 4));
  EPS_TRY(launch_distances(ix, ix->s_seed_rows.as<float>(), 0, L, d_queries, nq, ix->s_seed_dist.as<float>(), seed_ld,
                           &launches));
  GSArgs a;
  a.vectors = ix->d_vectors; a.offsets = ix->d_offsets; a.nbrs = ix->d_nbrs; a.ell = ix->d_ell;
  a.init_ids = ix->d_init_ids; a.seed_dist = ix->s_seed_dist.as<float>(); a.queries = d_queries;
  constexpr int kVlogCap = 32768;
  EPS_TRY(ix->s_vlog.reserve(static_cast<size_t>(slots) * kVlogCap * 4));
  a.vlog = ix->s_vlog.as<int32_t>(); a.vlog_cap = kVlogCap;
  a.visited = ix->s_visited.as<uint32_t>(); a.out_queue = d_queue;
  a.work_counter = reinterpret_cast<int*>(ix->s_misc.as<unsigned char>() + 32);
  a.stats = ix->s_misc.as<unsigned long long>();
  a.visited_words = words; a.seed_ld = seed_ld; a.dim = dim; a.metric = ix->metric;
  a.vec4 = ix->vec4 ? 1 : 0; a.L = static_cast<int>(L); a.Lp = Lp; a.nq = static_cast<int>(nq);
  a.W = width; a.R = R; a.slot_bytes = slot_bytes; a.fc = fc;
  a.qtimes = nullptr;
#ifdef EPS_GS_PROFILE
  EPS_TRY(ix->s_tail.reserve(static_cast<size_t>(nq) * 32));  // borrowed scratch (the hybrid tail buffer is filled after the search)
  a.qtimes = ix->s_tail.as<unsigned long long>();
  ix->prof_nq = nq;
#endif
  graph_search_kernel<<<slots, kGsThreads, smem, ix->stream>>>(a);
  EPS_CUDA(cudaGetLastError());
  if (stats) {
    stats->n_seed += static_cast<uint64_t>(nq) * static_cast<uint64_t>(L);
    stats->kernel_launches += launches;
  }
  return EPS_OK;
}

// Device counters of the last graph_search launch (call after the stream has been synchronised).
int read_graph_counters(Index* ix, eps_stats* stats) {
  if (!stats || !ix->s_misc.p) return EPS_OK;
  unsigned long long h[4];
  EPS_CUDA(cudaMemcpy(h, ix->s_misc.p, 32, cudaMemcpyDeviceToHost));
  stats->n_dist += h[0];
  stats->n_expand += h[1];
  stats->n_edges += h[2];
#ifdef EPS_GS_PROFILE
  unsigned long long pr[32];
  EPS_CUDA(cudaMemcpy(pr, ix->s_misc.p, 256, cudaMemcpyDeviceToHost));
  const char* names[8] = {"barrierX", "merge", "row_wait", "team_phase", "pick", "barrier1", "adj+visited", "barrier2+fifo"};
  const double tot = static_cast<double>(pr[24]) + 1.0;
  fprintf(stderr, "[gs-profile] kernel cycles summed over CTAs %.3e;", tot);
  for (int w = 0; w < 2; ++w)
    for (int i = 0; i < 8; ++i) fprintf(stderr, " w%d.%s=%.1f%%", w, names[i], 100.0 * static_cast<double>(pr[8 + w * 8 + i]) / tot);
  fprintf(stderr, "\n");
  if (ix->prof_nq > 0 && ix->s_tail.p) {
    std::vector<unsigned long long> t(static_cast<size_t>(ix->prof_nq) * 4);
    EPS_CUDA(cudaMemcpy(t.data(), ix->s_tail.p, t.size() * 8, cudaMemcpyDeviceToHost));
    unsigned long long t0 = ~0ull, t1 = 0;
    for (int64_t q = 0; q < ix->prof_nq; ++q) { t0 = std::min(t0, t[4 * q]); t1 = std::max(t1, t[4 * q + 1]); }
    std::vector<double> end, dur;
    std::vector<std::pair<double, int64_t>> by_dur;
    double nd_sum = 0, it_sum = 0;
    for (int64_t q = 0; q < ix->prof_nq; ++q) {
      end.push_back((t[4 * q + 1] - t0) * 1e-3);
      dur.push_back((t[4 * q + 1] - t[4 * q]) * 1e-3);
      by_dur.push_back({dur.back(), q});
      nd_sum += static_cast<double>(t[4 * q + 2]); it_sum += static_cast<double>(t[4 * q + 3]);
    }
    std::sort(end.begin(), end.end());
    std::sort(dur.begin(), dur.end());
    std::sort(by_dur.begin(), by_dur.end());
    const size_t n = end.size();
    fprintf(stderr, "[gs-profile] span %.0f us; query END times (us) p10 %.0f p50 %.0f p90 %.0f p99 %.0f max %.0f; query DURATION (us) p10 %.0f p50 %.0f p90 %.0f max %.0f\n",
            (t1 - t0) * 1e-3, end[n / 10], end[n / 2], end[n * 9 / 10], end[n * 99 / 100], end[n - 1], dur[n / 10], dur[n / 2], dur[n * 9 / 10], dur[n - 1]);
    fprintf(stderr, "[gs-profile] per query: mean n_dist %.0f, mean iterations %.0f; slowest:", nd_sum / n, it_sum / n);
    for (size_t i = 0; i < 6 && i < n; ++i) {
      const int64_t q = by_dur[n - 1 - i].second;
      fprintf(stderr, " [q%lld %.0f us n_dist %llu it %llu]", static_cast<long long>(q), by_dur[n - 1 - i].first, t[4 * q + 2], t[4 * q + 3]);
    }
    fprintf(stderr, "; median:");
    for (size_t i = 0; i < 3 && i < n; ++i) {
      const int64_t q = by_dur[n / 2 + i].second;
      fprintf(stderr, " [q%lld %.0f us n_dist %llu it %llu]", static_cast<long long>(q), by_dur[n / 2 + i].first, t[4 * q + 2], t[4 * q + 3]);
    }
    fprintf(stderr, "\n");
  }
#endif
  return EPS_OK;
}

}  // namespace eps
