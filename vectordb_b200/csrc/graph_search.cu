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
//     cp.async.bulk + mbarrier complete_tx, L2 evict_first) issued by a single lane: no registers are held across the wait,
//     every free ring slot is in flight at once, and the adjacency reads + visited tests of the NEXT
//     candidates run while the rows of the previous ones land;
//   * distances: warps 1-3 own the ring slots (slot s <-> warp 1 + s % 3); a warp waits on the mbarriers of its
//     occupied slots, evaluates up to 8 landed rows with all 32 lanes on every row (float4 from shared memory, the
//     lane's query chunk loaded once, 5 shuffle steps per row), refills its slots from the FIFO and keeps streaming
//     while the FIFO has a backlog; accepted keys (key < worst-in-queue) go to a small pending buffer that is merged
//     into the sorted queue by a block-parallel rank-and-shift, at the latest when the expansion is consumed;
//   * adjacency: fixed-stride rows of 64 int32 ids (one 256-byte read from the vertex id; longer rows
//     continue in the CSR); visited: a per-slot open-addressing hash set of int32 ids in global memory (16 L entries,
//     at most 64 KB: the tables of all resident queries fit in L2), one 32-byte bucket read + atomicCAS per
//     test-and-insert, refilled with 0xFF after the query like the reference clears its vector<bool> (:711-714).  A
//     query that would fill the set beyond 3/4 moves to a bitmap of n bits (atomicOr test-and-set) for the rest of
//     its run; that bitmap is cleared after the query — on large tables only the words the query touched, from a log
//     of its fresh ids.
//   * screen (sketch.cu; L2, and inner product / cosine through a bound on the dot product): once the queue holds L
//     entries, the fresh ids of a step are checked against a proven lower bound from 32-float principal-subspace
//     sketches of the row and the query, and only those it cannot reject enter
//     the FIFO and have their rows fetched (screen_fresh; DESIGN.md §K2);
// every iteration picks up to W (the search width) unchecked candidates, and the next pick waits until all their rows
//   are consumed and merged.  The result at any width W is that of this rule: each step takes the first
//   min(W, #unchecked) unchecked queue entries and marks them checked, tests-and-sets every id of their full CSR rows
//   against one visited set, evaluates the fresh ids, and keeps the best L by (distance, id) of the queue and the fresh
//   rows, checked flags kept; the search stops when nothing is unchecked.  It holds because at a pick the pending buffer
//   is empty, continuation chunks are drained before the next pick, and keys accepted against a stale bound are evicted
//   by the merge, so neither the landing order of rows nor the launch geometry can change it.  Width 1 is the reference
//   at IntraQueryThreads = 1 (visit order, results, distance-evaluation counts); widths 2..8 are the device analogue of
//   IntraQueryThreads > 1, deterministic where that mode races.  tests/graph_model.py restates the rule and
//   tests/test_gpu_graph_exact.py holds the kernel to it bit for bit.
#include <algorithm>
#include <cfloat>
#include <cstdio>
#include <cstdlib>

#include "async.cuh"
#include "graph_search.cuh"
#include "internal.h"

namespace eps {

constexpr int kMaxW = 8;        // candidates picked per iteration (upper bound)
constexpr int kMaxS = 8;        // ring slots per consumer warp (upper bound)
constexpr int kMaxR = 24;       // ring slots (upper bound: 3 consumer warps x kMaxS)
constexpr int kRounds = kMaxW * kEll / kGsThreads;  // adjacency slots per thread

// Developer build only (make EXTRA=-DEPS_GS_PROFILE): per-phase cycle counters of warp 0 (pick / adjacency / screen /
// merge / barrier waits) and of warp 1 (row wait + math), summed over CTAs into the kGcPhase slots of the counter block,
// the visited-set counts and a per-query timeline.  Compiled out otherwise.
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
  uint32_t* vset;                 // [slots x vset_cap] hash set of the ids the running query has visited (kVsetEmpty = free)
  int vset_cap;                   // entries per slot: a power of two >= 1024
  int vset_shift;                 // bucket of an id = (id * kVsetMul) >> vset_shift, 8 entries per bucket
  int vset_max;                   // entries a query may insert before it moves to the bitmap (3/4 of vset_cap)
  uint32_t* visited;              // [slots x visited_words] bitmaps of the queries that outgrew their hash set
  int32_t* vlog;                  // [slots x vlog_cap] the running query's fresh ids in FIFO order (migration, bitmap reset)
  int vlog_cap;
  unsigned long long* out_queue;  // [nq x L]
  int* work_counter;
  unsigned long long* stats;      // counter block (GraphCounter slots)
  int64_t visited_words;
  int64_t seed_ld;
  int dim, metric, vec4;  // vec4: not read; removing it, or moving qtimes, grows the spills of the 72- and 128-register instances
  int L, Lp;
  int nq;
  int W;                          // candidates per iteration (the search width)
  int R;                          // ring slots (slot s is owned by consumer warp s % 3)
  int fc;                         // fresh-id FIFO capacity (power of two)
  unsigned long long* qtimes;     // developer build: [nq x 4] globaltimer at query start and end, n_dist, iterations
  int slot_bytes;                 // ring slot pitch (row bytes, multiple of 16); 0 when rows are not staged
  // screen (sketch.cu; sk == null: off): fresh neighbours whose sketch bound fails the bound never enter the FIFO
  const float* sk;                // [n x kSketch] row sketches, then [n] their error bounds
  const float* qsk;               // [nq x kSketch] query sketches, then [nq] their error bounds
  int64_t n_sk;                   // rows sketched (n_indexed)
  float sk_g, sk_scale;           // rounded-down factors of the bound (see screen_fresh)
  unsigned long long* n_screened; // ids the screen dropped, summed over every search of the handle
  // collect mode (kCollect): besides the queue, each query keeps the best `cap` keys of the passing rows it evaluates
  const uint32_t* pass;           // bit i: row i is not deleted and passes the filter
  unsigned long long* out_r;      // [nq x cap] those keys, ascending, kKeyInf padded
  int cap;
};

__device__ __forceinline__ bool row_passes(const uint32_t* pass, uint32_t id) { return (pass[id >> 5] >> (id & 31)) & 1u; }

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

// Screen of the fresh ids fifo[tail .. tail + total) of one expansion step (all 128 threads).  Eight lanes per id read its
// sketch s_x (one float4 each) and its error bound ex_x; the loads of up to kScreenIds ids are issued before any is
// used.  With p_q, E_q the query's sketch and bound (shared memory) and l^ = the fp32 sum of (s_x - p_q)^2:
//   LB = [(sqrt(l^ (1 - gamma_{m+2})) - ex_x - E_q)+]^2 (1 - 2 (d + 2) 2^-24) / (1 + eps),   every step rounded down.
// |s_x - p_q| - ex_x - E_q <= |P~(x - q)| <= sqrt(1 + eps) |x - q|, and the kernel's fp32 L2 sum of the row is at least
// (1 - 2 (d + 2) 2^-24) |x - q|^2, so LB never exceeds the distance the consumer would compute.  An id is dropped iff
// make_key(LB, id) >= bound; the consumer's bound is at most this one, so it would have dropped the id too.  Bit i of
// keep is set for every id i that stays.  In collect mode the id must also stay out of the passing rows' list: it is
// dropped only when it fails the filter or make_key(LB, id) >= rbound, the list's worst key (kKeyInf until it is full).
//
// Inner product and cosine (kScreenDot): the consumer computes acc = the fp32 dot product of q and x (lane fmaf chains
// of at most 4 ceil(d / 128) terms, then the 5-step butterfly: n_c = 4 ceil(d / 128) + 5 roundings, which also covers
// the scalar path's ceil(d / 32) + 5) and the distance base - acc (IP: -acc, base = 0; cosine: fl(1 - acc)).  With
// y = x - mu, q' = q - mu and A = I - P~^T P~ (symmetric, A - A^2 = P~^T (I - P~ P~^T) P~, so |A - A^2| <= eps (1 + eps)):
//   <q, x> = <q, mu> + <mu, y> + <P~ q', P~ y> + <A q', A y> + q'^T (A - A^2) y
//   acc    <= <q, x> + gamma_{n_c} |q| |x| + n_c 2^-149                         (n_c 2^-149: products that underflow)
// and, with the sketches s^_x (bound ex_x) and p^_q (bound E_q) and s^ = the 8-lane fp32 sum of their products (lane
// chains of 4, 3-step butterfly: error <= gamma_7 |p^_q| |s^_x| + 7 2^-149),
//   <P~ q', P~ y> <= s^ + gamma_7 |p^_q| |s^_x| + E_q |s^_x| + |p^_q| ex_x + E_q ex_x + 7 2^-149.
// Each row's ex_x bounds its |y| (|y| <= k ex_x, k = 1 / (sqrt(m) gamma_{d+2} sqrt(1 + eps)), see sketch_rows_kernel),
// and so |s^_x| <= (sqrt(1 + eps) k + 1) ex_x and |x| <= |mu| + k ex_x.  That folds every query-only factor into four
// numbers per query, computed in double and rounded up by dot_terms_kernel (sketch.cu), psk[kSketch ..]:
//   UB = s^ + (C0 - base) + <mu, y> + |A q'| |A y| + C_ex ex_x,   every step rounded up (__fadd_ru, __fmul_ru);
//   LB = -0 - UB rounded down  (= round_down(base - UB): IP -UB, cosine round_down(1 - UB); -0 for a zero)
// with <mu, y> and |A y| stored per row (float2, rounded up).  acc <= UB, and base - acc and fl(1 - acc) are
// non-increasing in acc, so LB never exceeds the consumer's distance.  The consumer's products and partial sums stay
// below FLT_MAX when |q| |x| < 2^126: an id is dropped only when K ex_x < 2^125 (K = |q| k; +inf when |q| |mu| >= 2^125),
// UB is finite (NaN or inf from any term, a row that overflows, a query whose norm is not finite: kept), and
// make_key(LB, id) >= bound, with the same collect-mode condition as L2.
constexpr int kScreenIds = 64;  // ids whose loads are in flight together (4 per 8-lane group)
template <int kScreen, bool kCollect>
__device__ __forceinline__ void screen_fresh(const GSArgs& a, const int* fifo, unsigned fmask, uint32_t tail, int total, const float* psk,
                                             unsigned long long bound, unsigned long long rbound, int tid, unsigned* keep) {
  constexpr bool kDot = kScreen == kScreenDot;
  const int g = tid >> 3, j = tid & 7;
  constexpr int kPer = kScreenIds / (kGsThreads / 8);
  const float4* sk4 = reinterpret_cast<const float4*>(a.sk);
  const float* skex = a.sk + a.n_sk * kSketch;
  const float2* skt = kDot ? reinterpret_cast<const float2*>(a.sk + sk_terms_off(a.n_sk)) : nullptr;
  const float4 p0 = reinterpret_cast<const float4*>(psk)[j];
  const float eq = psk[kSketch];
  const float4 qc = kDot ? reinterpret_cast<const float4*>(psk + kSketch)[0] : make_float4(0.f, 0.f, 0.f, 0.f);  // C0 - base, C_ex, |A q'|, K
  for (int i0 = 0; i0 < total; i0 += kScreenIds) {
    int id[kPer];
    float4 x0[kPer];
    float xe[kPer];
    float2 xt[kPer];
#pragma unroll
    for (int b = 0; b < kPer; ++b) {
      const int i = i0 + b * (kGsThreads / 8) + g;
      id[b] = i < total ? fifo[(tail + static_cast<uint32_t>(i)) & fmask] : -1;
      x0[b] = p0;
      xe[b] = 0.f;
      if (kDot) xt[b] = make_float2(0.f, 0.f);
      if (id[b] >= 0) {
        x0[b] = __ldg(sk4 + static_cast<int64_t>(id[b]) * (kSketch / 4) + j);
        if (j == 0) xe[b] = __ldg(skex + id[b]);
        if (kDot && j == 0) xt[b] = __ldg(skt + id[b]);
      }
    }
#pragma unroll
    for (int b = 0; b < kPer; ++b) {
      float acc = 0.f, d;
      if (kDot) {
        acc = fmaf(x0[b].x, p0.x, acc); acc = fmaf(x0[b].y, p0.y, acc); acc = fmaf(x0[b].z, p0.z, acc); acc = fmaf(x0[b].w, p0.w, acc);
      } else {
        d = x0[b].x - p0.x; acc = fmaf(d, d, acc); d = x0[b].y - p0.y; acc = fmaf(d, d, acc);
        d = x0[b].z - p0.z; acc = fmaf(d, d, acc); d = x0[b].w - p0.w; acc = fmaf(d, d, acc);
      }
      acc += __shfl_xor_sync(kFull, acc, 1);
      acc += __shfl_xor_sync(kFull, acc, 2);
      acc += __shfl_xor_sync(kFull, acc, 4);
      if (j == 0 && id[b] >= 0) {
        const int i = i0 + b * (kGsThreads / 8) + g;
        bool drop = false;
        if (kDot) {
          float ub = __fadd_ru(__fadd_ru(acc, qc.x), xt[b].y);
          ub = __fadd_ru(ub, __fmul_ru(qc.z, xt[b].x));
          ub = __fadd_ru(ub, __fmul_ru(qc.y, xe[b]));
          const float lb = __fsub_rd(-0.f, ub);
          drop = __fmul_ru(qc.w, xe[b]) < 0x1.0p125f && fabsf(ub) <= FLT_MAX && make_key(lb, static_cast<uint32_t>(id[b])) >= bound;
          if (kCollect && drop)
            drop = !row_passes(a.pass, static_cast<uint32_t>(id[b])) || make_key(lb, static_cast<uint32_t>(id[b])) >= rbound;
        } else {
          float r = __fsqrt_rd(__fmul_rd(acc, a.sk_g));
          r = __fsub_rd(__fsub_rd(r, xe[b]), eq);
          if (r > 0.f) {  // false for NaN as well
            const float lb = __fmul_rd(__fmul_rd(r, r), a.sk_scale);
            drop = lb <= FLT_MAX && make_key(lb, static_cast<uint32_t>(id[b])) >= bound;
            if (kCollect && drop)
              drop = !row_passes(a.pass, static_cast<uint32_t>(id[b])) || make_key(lb, static_cast<uint32_t>(id[b])) >= rbound;
          }
        }
        if (!drop) atomicOr(keep + (i >> 5), 1u << (i & 31));
      }
    }
  }
}

// Consumer step of one warp over its S slots (slot of local index s = cw + 3 s): wait for the landed rows, distances,
// accepted keys to the pending buffer; in collect mode, the keys of passing rows under rbound to the list's pending buffer
// rpend.  Returns nothing; the caller refills the slots.
template <int S, bool kCollect>
__device__ __forceinline__ void consume_slots(const GSArgs& a, unsigned occ_mask, unsigned par_mask, int cw, int lane, bool staged,
                                              const unsigned char* ring, uint32_t bar0, const float* qv, const int* slot_id,
                                              unsigned long long bound, unsigned long long* pend, int* s_npend,
                                              unsigned long long rbound, unsigned long long* rpend, int* s_nrpend) {
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
    if (kCollect && key < rbound && row_passes(a.pass, key_id(key))) rpend[atomicAdd(s_nrpend, 1)] = key;
  }
}

// Two register budgets of the same kernel: 72 registers per thread allow 7 resident CTAs per SM but spill 376 B per
// thread to local memory (348 B of spill loads); 128 registers allow 4 and spill 12 B (16 B of loads).  graph_search
// picks the instance from the geometry it launches.  kScreen: the screen kind (kScreenNone, kScreenL2, kScreenDot for
// inner product and cosine) is compiled in only where it runs, so that a search without it (tables it cannot pay on)
// keeps the registers of the kernel without it, and the L2 instances carry no metric branch.  kCollect: the
// collect mode of a filtered search (DESIGN.md §K2), which navigates as the other instances do and also keeps each
// query's list of the best a.cap keys of the passing rows it evaluates, merged like the queue.
template <int kMinCtas, int kScreen, bool kCollect = false>
__global__ void __launch_bounds__(kGsThreads, kMinCtas) graph_search_kernel(GSArgs a) {
  extern __shared__ __align__(128) unsigned char gs_smem[];
  const int dim4p = (a.dim + 3) & ~3;
  unsigned char* ring = gs_smem;                                                                   // [R][slot_bytes]
  unsigned long long* qa = reinterpret_cast<unsigned long long*>(ring + static_cast<size_t>(a.R) * a.slot_bytes);  // [Lp]
  unsigned long long* pend = qa + a.Lp;                                                            // [kPC]
  unsigned long long* cs = pend + kPC;                                                             // [kPC]
  unsigned long long* bars = cs + kPC;                                                             // [kMaxR]
  float* qv = reinterpret_cast<float*>(bars + kMaxR);                                              // [dim4p]
  float* psk = qv + dim4p;                                                                         // [kSketch + 4] query sketch, bound (screen)
  int* pos = reinterpret_cast<int*>(psk + (kScreen ? kSketch + 4 : 0));                            // [kPC]
  int* fifo = pos + kPC;                                                                           // [fc]
  int* slot_id = fifo + a.fc;                                                                      // [kMaxR] row id in each ring slot
  unsigned* ubits = reinterpret_cast<unsigned*>(slot_id + kMaxR);                                  // [(Lp + 31) / 32] unchecked-entry bitmap
  // collect: [cap] the passing rows' list, [kPC] its pending keys (8-byte aligned after an even number of bitmap words)
  unsigned long long* rq = reinterpret_cast<unsigned long long*>(ubits + (((a.Lp + 31) / 32 + 1) & ~1));
  unsigned long long* rpend = rq + a.cap;
  __shared__ int s_nrpend;
  __shared__ int s_q, s_ncur, s_cursor, s_npend, s_ncont;
  __shared__ unsigned s_head;                      // FIFO entries [s_head, fifo_tail) are not yet issued to the ring
  __shared__ int s_cid[kMaxW];
  __shared__ int s_wcnt[kRounds][kGsThreads / 32];
  __shared__ long long s_cont_e[kMaxW], s_cont_end[kMaxW];
  __shared__ unsigned s_keep[kMaxW * kEll / 32];  // screen: bit i = fresh id i of the step stays

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
  uint32_t* vset = a.vset + static_cast<int64_t>(blockIdx.x) * a.vset_cap;
  const uint32_t vmask = static_cast<uint32_t>(a.vset_cap) - 1u;
  uint32_t* visited = a.visited + static_cast<int64_t>(blockIdx.x) * a.visited_words;
  int32_t* vlog = a.vlog + static_cast<int64_t>(blockIdx.x) * a.vlog_cap;
  unsigned long long vacc = 0;  // developer build: hash-set accesses (bucket reads + CAS) of this thread

  if (tid == 0) {
    for (int s = 0; s < R; ++s) mbar_init(bar0 + 8 * s, 1);
    mbar_fence_init();
  }
  // The owning warp issues the bulk copy into a slot, waits on its mbarrier, reads it and refills it — no block
  // barrier guards a slot.  Per-slot state (occupied, mbarrier phase parity) is a pair of warp-uniform bit masks.
  unsigned occ_mask = 0u, par_mask = 0u;
  const int n_own = cw >= 0 ? (R - cw + 2) / 3 : 0;  // slots cw, cw + 3, ... < R
  unsigned long long st_ndist = 0, st_nexp = 0, st_nedge = 0, st_nscr = 0;
#ifdef EPS_GS_PROFILE
  long long prof[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // 0 barrier X, 1 merge, 2 screen, 3 row wait + math, 4 pick, 5 barrier 1, 6 adjacency+visited, 7 barrier 2 + FIFO
  const long long t_kernel0 = clock64();
  unsigned long long prof_vtest = 0, prof_migrated = 0;  // hash-set test-and-inserts of this thread; queries moved to the bitmap
#endif

  for (;;) {
    __syncthreads();
    if (tid == 0) s_q = atomicAdd(a.work_counter, 1);
    __syncthreads();
    const int q = s_q;
    if (q >= a.nq) break;
#ifdef EPS_GS_PROFILE
    if (tid == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); a.qtimes[4 * q] = t; }
    const unsigned long long prof_nd0 = st_ndist;
    unsigned long long prof_iters = 0;
#endif

    // ---- seed (InitializeSetLPara): precomputed distances of the query-independent seed set ----
    for (int i = tid; i < a.dim; i += kGsThreads) qv[i] = a.queries[static_cast<int64_t>(q) * a.dim + i];
    for (int i = a.dim + tid; i < dim4p; i += kGsThreads) qv[i] = 0.f;
    if (kScreen == kScreenL2 && tid <= kSketch)
      psk[tid] = tid < kSketch ? a.qsk[static_cast<int64_t>(q) * kSketch + tid] : a.qsk[static_cast<int64_t>(a.nq) * kSketch + q];
    if (kScreen == kScreenDot && tid < kSketch + 4)  // the sketch, then C0 - base, C_ex, |A q'|, K
      psk[tid] = tid < kSketch ? a.qsk[static_cast<int64_t>(q) * kSketch + tid]
                               : a.qsk[sk_qterms_off(a.nq) + 4 * static_cast<int64_t>(q) + tid - kSketch];
    bool hashed = L <= a.vset_max;  // the visited set is the hash set (false: the query has moved to the bitmap)
    for (int i = tid; i < a.Lp; i += kGsThreads) {
      unsigned long long key = kKeyInf;
      if (i < L) {
        const uint32_t id = static_cast<uint32_t>(a.init_ids[i]);
        if (hashed) {
          vset_claim(vset, vmask, vset_bucket(id, a.vset_shift), id, vacc);
#ifdef EPS_GS_PROFILE
          ++prof_vtest;
#endif
        } else {
          atomicOr(&visited[id >> 5], 1u << (id & 31));
        }
        key = make_key(a.seed_dist[static_cast<int64_t>(q) * a.seed_ld + i], id);
      }
      qa[i] = key;
    }
    if (tid == 0) { s_npend = 0; s_ncont = 0; s_cursor = 0; s_ncur = 0; s_head = 0u; }
    __syncthreads();
    block_bitonic_sort(qa, a.Lp);
    for (int w = tid; w < ((L + 31) >> 5); w += kGsThreads)  // every seed starts unchecked
      ubits[w] = (w * 32 + 32 <= L) ? 0xffffffffu : ((1u << (L & 31)) - 1u);
    if (kCollect) {  // the list starts with the first cap passing seeds of the sorted queue
      if (warp == 0) {
        int n = 0;
        for (int base = 0; base < L && n < a.cap; base += 32) {
          const int i = base + lane;
          const unsigned long long key = i < L ? qa[i] : kKeyInf;
          const bool ok = i < L && row_passes(a.pass, key_id(key));
          const unsigned b = __ballot_sync(kFull, ok);
          const int o = n + __popc(b & lane_lt);
          if (ok && o < a.cap) rq[o] = key;
          n += __popc(b);
        }
        for (int i = min(n, a.cap) + lane; i < a.cap; i += 32) rq[i] = kKeyInf;
      }
      if (tid == 0) s_nrpend = 0;
    }
    if (tid == 0) st_ndist += static_cast<unsigned long long>(L);
    uint32_t fifo_tail = 0;   // ids appended to the FIFO
    uint32_t fresh_n = 0;  // fresh ids of the query (= fifo_tail unless the screen dropped some); the log holds them
    auto fresh_tail = [&]() { return kScreen ? fresh_n : fifo_tail; };

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
      const int rm = kCollect ? s_nrpend : 0;
      const uint32_t head = s_head;
      const int ncont = s_ncont;
      // -- D: merge the pending keys --
      const bool merged = m > 0;
      // s_npend / s_head are bumped by the consumer phase below: no thread may get there before EVERY thread has taken
      // the snapshot above (the merge's own barriers do that when there is a merge)
      if (merged) merge_pending(qa, pend, cs, pos, m, L, &s_npend, &s_cursor, ubits);
      else __syncthreads();
      if (kCollect && rm > 0) merge_pending<false>(rq, rpend, cs, pos, rm, a.cap, &s_nrpend, nullptr, nullptr);
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
        const unsigned long long rbound = kCollect ? rq[a.cap - 1] : kKeyInf;
        for (;;) {
          if (occ_mask) {
            GS_T(tw0);
#define GS_CONSUME(S) consume_slots<S, kCollect>(a, occ_mask, par_mask, cw, lane, staged, ring, bar0, qv, slot_id, bound, pend, &s_npend, \
                                                 rbound, rpend, &s_nrpend)
            if (n_own <= 1) GS_CONSUME(1);
            else if (n_own <= 2) GS_CONSUME(2);
            else if (n_own <= 4) GS_CONSUME(4);
            else GS_CONSUME(8);
#undef GS_CONSUME
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
                // rows are mostly read once: L2 evicts them first, so that they do not push out the visited tables
                bulk_load_1d(ring0 + slot * static_cast<uint32_t>(a.slot_bytes), a.vectors + static_cast<int64_t>(id) * a.dim, row_bytes, bar,
                             l2_policy_evict_first());
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
          if (kCollect && *reinterpret_cast<volatile int*>(&s_nrpend) + R > kPC) break;
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
      // a step inserts at most nslots ids: move to the bitmap before the hash set could pass 3/4 full.  Every id the
      // query has visited is a seed or in the log (fifo_tail <= vset_max < vlog_cap).  Block-uniform.
      if (hashed && L + fresh_tail() + static_cast<uint32_t>(nslots) > static_cast<uint32_t>(a.vset_max)) {
        for (int i = tid; i < L; i += kGsThreads) {
          const uint32_t id = static_cast<uint32_t>(a.init_ids[i]);
          atomicOr(&visited[id >> 5], 1u << (id & 31));
        }
        for (uint32_t i = tid; i < fresh_tail(); i += kGsThreads) {
          const uint32_t id = static_cast<uint32_t>(vlog[i]);
          atomicOr(&visited[id >> 5], 1u << (id & 31));
        }
        hashed = false;
        __syncthreads();  // every bit is set before any thread tests one
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
      // test-and-insert (ExpandOneCandidate :403-406); of two slots racing on one id exactly one finds it fresh
      if (hashed) {
        // one bucket read per id: an entry equal to it = visited; else a CAS on the first free entry of the bucket (the
        // next bucket's first entry when it is full), and a CAS lost to another id goes on probing entry by entry
        uint32_t at[kRounds], old[kRounds];
#pragma unroll
        for (int r = 0; r < kRounds; ++r) {
          at[r] = kVsetEmpty;
          if (nb[r] >= 0) {
            const uint32_t id = static_cast<uint32_t>(nb[r]), b = vset_bucket(id, a.vset_shift);
            const uint4 lo = __ldcg(reinterpret_cast<const uint4*>(vset + b)), hi = __ldcg(reinterpret_cast<const uint4*>(vset + b) + 1);
            const uint32_t e[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
            bool hit = false;
            uint32_t fe = 8;
#pragma unroll
            for (int j = 7; j >= 0; --j) {
              hit |= e[j] == id;
              if (e[j] == kVsetEmpty) fe = j;
            }
            if (!hit) at[r] = (b + fe) & vmask;
#ifdef EPS_GS_PROFILE
            ++prof_vtest; ++vacc;
#endif
          }
        }
#pragma unroll
        for (int r = 0; r < kRounds; ++r) old[r] = at[r] != kVsetEmpty ? atomicCAS(vset + at[r], kVsetEmpty, static_cast<uint32_t>(nb[r])) : 0u;
#pragma unroll
        for (int r = 0; r < kRounds; ++r) {
          fr[r] = false;
          if (at[r] != kVsetEmpty) {
#ifdef EPS_GS_PROFILE
            ++vacc;
#endif
            const uint32_t id = static_cast<uint32_t>(nb[r]);
            fr[r] = old[r] == kVsetEmpty || (old[r] != id && vset_claim(vset, vmask, (at[r] + 1) & vmask, id, vacc));
          }
        }
      } else {
#pragma unroll
        for (int r = 0; r < kRounds; ++r) {
          fr[r] = false;
          if (nb[r] >= 0) {
            const uint32_t bit = 1u << (nb[r] & 31);
            fr[r] = !(atomicOr(&visited[nb[r] >> 5], bit) & bit);
          }
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
      if (kScreen && tid < kMaxW * kEll / 32) s_keep[tid] = 0u;
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
          const uint32_t rank = static_cast<uint32_t>(mine + __popc(bal[r] & lane_lt));
          fifo[(fifo_tail + rank) & fmask] = nb[r];
          if (fresh_tail() + rank < static_cast<uint32_t>(a.vlog_cap)) vlog[fresh_tail() + rank] = nb[r];
        }
      }
      if (kScreen) fresh_n += static_cast<uint32_t>(total);
      GS_T(ts0);
      // -- A2: screen the fresh ids on their sketches once the queue holds L entries (block-uniform) --
      const unsigned long long sbound = kScreen ? qa[L - 1] & kKeyMask : kKeyInf;
      if (kScreen && total > 0 && sbound != kKeyInf) {
        __syncthreads();  // (3) the fresh ids are in the FIFO, s_keep is clear
        screen_fresh<kScreen, kCollect>(a, fifo, fmask, fifo_tail, total, psk, sbound, kCollect ? rq[a.cap - 1] : kKeyInf, tid, s_keep);
        int mine[kMaxW * kEll / kGsThreads];
#pragma unroll
        for (int r = 0; r < kMaxW * kEll / kGsThreads; ++r) {
          const int i = r * kGsThreads + tid;
          mine[r] = i < total ? fifo[(fifo_tail + static_cast<uint32_t>(i)) & fmask] : -1;
        }
        __syncthreads();  // (4) every keep bit is set and every id read: compact the survivors in order
        int kept = 0;
        for (int w = 0; w < (total + 31) >> 5; ++w) kept += __popc(s_keep[w]);
#pragma unroll
        for (int r = 0; r < kMaxW * kEll / kGsThreads; ++r) {
          const int i = r * kGsThreads + tid;
          if (i < total && ((s_keep[i >> 5] >> (i & 31)) & 1u)) {
            int rank = __popc(s_keep[i >> 5] & ((1u << (i & 31)) - 1u));
            for (int w = 0; w < (i >> 5); ++w) rank += __popc(s_keep[w]);
            fifo[(fifo_tail + static_cast<uint32_t>(rank)) & fmask] = mine[r];
          }
        }
        if (tid == 0) st_nscr += static_cast<unsigned long long>(total - kept);
        fifo_tail += static_cast<uint32_t>(kept);
      } else {
        fifo_tail += static_cast<uint32_t>(total);
      }
      GS_T(ts1);
      GS_ACC(2, ts0, ts1);
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
      GS_ACC(7, ts1, ts0);  // less the screen, which is its own phase
    }

    // ---- results + visited reset (:711-714) ----
    {
      const int m = s_npend;  // only checked entries can be left (the last pick found nothing unchecked)
      if (m > 0) merge_pending(qa, pend, cs, pos, m, L, &s_npend, &s_cursor, ubits);
      const int rm = kCollect ? s_nrpend : 0;
      if (rm > 0) merge_pending<false>(rq, rpend, cs, pos, rm, a.cap, &s_nrpend, nullptr, nullptr);
    }
    unsigned long long* out = a.out_queue + static_cast<int64_t>(q) * L;
    for (int i = tid; i < L; i += kGsThreads) out[i] = qa[i];
    if (kCollect)
      for (int i = tid; i < a.cap; i += kGsThreads) a.out_r[static_cast<int64_t>(q) * a.cap + i] = rq[i];
#ifdef EPS_GS_PROFILE
    if (tid == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      a.qtimes[4 * q + 1] = t; a.qtimes[4 * q + 2] = st_ndist - prof_nd0; a.qtimes[4 * q + 3] = prof_iters;
    }
#endif
    // the hash set: 16-byte stores over the whole table (at most 64 KB, in L2); the bitmap only if the query moved to it
    {
      uint4* t4 = reinterpret_cast<uint4*>(vset);
      const uint4 e = make_uint4(kVsetEmpty, kVsetEmpty, kVsetEmpty, kVsetEmpty);
      for (int i = tid; i < (a.vset_cap >> 2); i += kGsThreads) t4[i] = e;
    }
#ifdef EPS_GS_PROFILE
    if (tid == 0 && !hashed) ++prof_migrated;
#endif
    if (hashed) continue;
    if (fresh_tail() <= static_cast<uint32_t>(a.vlog_cap) && 10ll * (fresh_tail() + L) < a.visited_words) {
      // large table: clear only the words this query touched (the seeds and the logged fresh ids) instead of
      // streaming zeros over the whole bitmap (1.25 MB per query at 10M rows)
      for (int i = tid; i < L; i += kGsThreads) visited[static_cast<uint32_t>(a.init_ids[i]) >> 5] = 0u;
      for (uint32_t i = tid; i < fresh_tail(); i += kGsThreads) visited[static_cast<uint32_t>(vlog[i]) >> 5] = 0u;
    } else {
      uint4* v4 = reinterpret_cast<uint4*>(visited);
      const int64_t n4 = a.visited_words >> 2;
      const uint4 z = make_uint4(0, 0, 0, 0);
      for (int64_t i = tid; i < n4; i += kGsThreads) v4[i] = z;
    }
  }
#ifdef EPS_GS_PROFILE
  if (lane == 0 && warp < 2) {
    for (int i = 0; i < 8; ++i) atomicAdd(&a.stats[kGcPhase + warp * 8 + i], static_cast<unsigned long long>(prof[i]));
    if (warp == 0) atomicAdd(&a.stats[kGcCycles], static_cast<unsigned long long>(clock64() - t_kernel0));
  }
  if (prof_vtest) atomicAdd(&a.stats[kGcVsetTests], prof_vtest);
  if (prof_migrated) atomicAdd(&a.stats[kGcMigrated], prof_migrated);
  if (vacc) atomicAdd(&a.stats[kGcVsetAccesses], vacc);
#endif
  if (st_ndist) atomicAdd(&a.stats[kGcDist], st_ndist);
  if (st_nexp) atomicAdd(&a.stats[kGcExpand], st_nexp);
  if (st_nedge) atomicAdd(&a.stats[kGcEdges], st_nedge);
  if (st_nscr) atomicAdd(a.n_screened, st_nscr);
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
  ix->d_init_ids.release();
  EPS_TRY(ix->d_init_ids.reserve(static_cast<size_t>(L) * 4));
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
  EPS_TRY(ix->d_ell.reserve(static_cast<size_t>(ix->n_indexed) * kEll * 4));
  const int64_t tot = ix->n_indexed * kEll;
  csr_to_ell_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, ix->stream>>>(ix->d_offsets, ix->d_nbrs, ix->n_indexed, ix->d_ell);
  EPS_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return EPS_OK;
}

int graph_search(Index* ix, const float* d_queries, int64_t nq, int64_t L, unsigned long long* d_queue,
                 eps_stats* stats, const GraphCollect* collect) {
  int Lp = 0;
  EPS_TRY(graph_launch_prologue(ix, L, "graph_search", &Lp));
  const int dim = static_cast<int>(ix->dim);
  const int dimp = (dim + 3) & ~3;
  const int width = std::max(1, std::min(ix->search_width, kMaxW));
  const bool staged = ix->vec4;  // 16-byte aligned rows of a multiple of 16 bytes: eligible for bulk async copies
  const int slot_bytes = staged ? dim * 4 : 0;
  int R = ring_slots_for(ix, slot_bytes);
  // FIFO: a backlog below R entries + the ids one A step appends (W adjacency rows or one 128-id continuation chunk)
  const int fc = next_pow2(std::max(width * kEll, kGsThreads) + kMaxR);
  const int screen = screen_kind(ix);  // the query sketch takes shared memory only when the screen runs
  // collect: the passing rows' list and its pending keys after the bitmap words (padded to an even count)
  const size_t collect_bytes = collect ? 4 + static_cast<size_t>(collect->cap + kPC) * 8 : 0;
  auto smem_for = [&](int r) {
    return static_cast<size_t>(r) * slot_bytes + static_cast<size_t>(Lp) * 8 + 2 * kPC * 8 + kMaxR * 8 +
           static_cast<size_t>(dimp) * 4 + (screen ? (kSketch + 4) * 4 : 0) + kPC * 4 + static_cast<size_t>(fc) * 4 + kMaxR * 4 + static_cast<size_t>((Lp + 31) / 32) * 4 +
           collect_bytes;
  };
  while (R > 2 && smem_for(R) > 200 * 1024) --R;
  if (smem_for(R) > 226 * 1024) return fail(EPS_ERR_UNSUPPORTED, "queue + query + row ring do not fit in shared memory");
  using Kernel = void (*)(GSArgs);
  // [collect][per_sm <= 4][screen kind]
  const Kernel kernels[2][2][3] = {
      {{graph_search_kernel<7, kScreenNone>, graph_search_kernel<7, kScreenL2>, graph_search_kernel<7, kScreenDot>},
       {graph_search_kernel<4, kScreenNone>, graph_search_kernel<4, kScreenL2>, graph_search_kernel<4, kScreenDot>}},
      {{graph_search_kernel<7, kScreenNone, true>, graph_search_kernel<7, kScreenL2, true>, graph_search_kernel<7, kScreenDot, true>},
       {graph_search_kernel<4, kScreenNone, true>, graph_search_kernel<4, kScreenL2, true>, graph_search_kernel<4, kScreenDot, true>}}};
  const int ci = collect ? 1 : 0;
  for (int p = 0; p < 2; ++p)
    for (int s = 0; s < 3; ++s)
      EPS_CUDA(cudaFuncSetAttribute(kernels[ci][p][s], cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_for(R))));
  auto resident = [&](int r, int* out) {
    EPS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(out, kernels[ci][0][0], kGsThreads, smem_for(r)));
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
  // With the screen, between two rings with the same rounds and the same CTAs per SM (so the same kernel instance), one
  // whose resident CTAs fit the 196 KB shared-memory carve-out wins over a larger one that needs the 228 KB carve-out,
  // and the launch asks for that carve-out: it leaves the L1 60 KB of the SM's 256 KB instead of 28.  The screen's
  // sketch loads keep up to 64 lines of 128 B in flight per CTA, 32 KB at 4 CTAs per SM.  On one H100 at 10M x 768,
  // L = 768, 3 batches in flight, ring 10 at 4 CTAs per SM is 3 % faster than ring 12, and no faster with the carve-out
  // pinned at 228 KB.  Without the screen (the clustered table, L = 1536) the smaller L1 costs nothing and a smaller
  // ring does (ring 7 instead of 10: 1.5 %), so there the largest ring still wins.
  constexpr size_t kL1Carveout = 196 * 1024;  // H100: the largest carve-out below the 228 KB maximum
  if (screen && ix->gs_static_smem < 0) {
    cudaFuncAttributes fa;
    EPS_CUDA(cudaFuncGetAttributes(&fa, kernels[ci][1][screen]));
    ix->gs_static_smem = static_cast<int>(fa.sharedSizeBytes);
  }
  auto sm_smem = [&](int r, int p) { return static_cast<size_t>(p) * (smem_for(r) + ix->gs_static_smem + ix->smem_reserved_per_cta); };
  auto l1_kept = [&](int r, int p) { return screen && sm_smem(r, p) <= kL1Carveout; };
  auto rounds_of = [&](int p) { return (nq + static_cast<int64_t>(p) * ix->num_sms - 1) / (static_cast<int64_t>(p) * ix->num_sms); };
  bool keep_l1 = false;
  if (staged && ix->graph_ring_slots == 0 && rounds_of(per_sm) > 1) {
    int best_r = R, best_p = per_sm;
    for (int r = R - 1; r >= 4; --r) {
      int p = 0;
      EPS_TRY(resident(r, &p));
      if (rounds_of(p) < rounds_of(best_p) || (p == best_p && l1_kept(r, p) && !l1_kept(best_r, best_p))) { best_r = r; best_p = p; }
    }
    R = best_r;
    per_sm = best_p;
    keep_l1 = l1_kept(R, per_sm);
  }
  const size_t smem = smem_for(R);
  const int64_t rounds = rounds_of(per_sm);
  int slots = static_cast<int>(std::min<int64_t>((nq + rounds - 1) / rounds, static_cast<int64_t>(per_sm) * ix->num_sms));
  if (ix->graph_ring_slots > 0 || ix->graph_ctas_per_sm > 0)  // tuning override: every resident slot, queries claimed dynamically
    slots = static_cast<int>(std::min<int64_t>(nq, static_cast<int64_t>(per_sm) * ix->num_sms));
  VisitedSets vis;
  EPS_TRY(prepare_visited(ix, slots, L, &vis));
  EPS_TRY(graph_counters(ix, nq));
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
  EPS_TRY(launch_distances(ix, ix->metric, ix->s_seed_rows.as<float>(), 0, L, d_queries, nq, ix->s_seed_dist.as<float>(),
                           seed_ld, &launches));
  GSArgs a;
  a.vectors = ix->d_vectors; a.offsets = ix->d_offsets; a.nbrs = ix->d_nbrs; a.ell = ix->d_ell;
  a.init_ids = ix->d_init_ids; a.seed_dist = ix->s_seed_dist.as<float>(); a.queries = d_queries;
  a.vlog = vis.vlog; a.vlog_cap = vis.vlog_cap;
  a.vset = vis.vset; a.vset_cap = vis.vset_cap; a.vset_max = vis.vset_max; a.vset_shift = vis.vset_shift;
  a.visited = vis.visited; a.out_queue = d_queue;
  a.work_counter = reinterpret_cast<int*>(ix->s_misc.as<unsigned long long>() + kGcWork);
  a.stats = ix->s_misc.as<unsigned long long>();
  a.visited_words = vis.words; a.seed_ld = seed_ld; a.dim = dim; a.metric = ix->metric;
  a.vec4 = ix->vec4 ? 1 : 0; a.L = static_cast<int>(L); a.Lp = Lp; a.nq = static_cast<int>(nq);
  a.W = width; a.R = R; a.slot_bytes = slot_bytes; a.fc = fc;
  a.qtimes = nullptr;
  a.sk = nullptr; a.qsk = nullptr; a.n_sk = 0; a.sk_g = 0.f; a.sk_scale = 0.f; a.n_screened = nullptr;
  a.pass = collect ? collect->pass : nullptr;
  a.out_r = collect ? collect->out : nullptr;
  a.cap = collect ? static_cast<int>(collect->cap) : 0;
  if (screen) {
    if (!ix->d_screened) {
      EPS_TRY(ix->d_screened.reserve(8));
      EPS_CUDA(cudaMemsetAsync(ix->d_screened, 0, 8, ix->stream));
    }
    EPS_TRY(ix->s_qsk.reserve(static_cast<size_t>(sketch_query_floats(screen, nq)) * 4));
    float* qsk = ix->s_qsk.as<float>();
    EPS_TRY(sketch_queries(ix, d_queries, nq, qsk, &launches));
    a.sk = ix->d_sk; a.qsk = qsk; a.n_sk = ix->n_indexed; a.sk_g = ix->sk_g; a.sk_scale = ix->sk_scale;
    a.n_screened = ix->d_screened;
  }

#ifdef EPS_GS_PROFILE
  EPS_TRY(ix->s_prof_qtimes.reserve(static_cast<size_t>(nq) * 32));
  a.qtimes = ix->s_prof_qtimes.as<unsigned long long>();
  ix->prof_timeline = true;
#endif
  // at most 4 resident CTAs per SM (what the auto rule picks for batches above one wave at 7 per SM, e.g. 1024 queries
  // at L = 768): the register file has room for 128 registers per thread, so the instance that hardly spills runs;
  // smaller batches keep 7 resident queries per SM
  const Kernel kernel = kernels[ci][per_sm <= 4 ? 1 : 0][screen];
  // the smallest carve-out that holds the resident CTAs (the driver rounds the percentage up to one it supports), or
  // the driver's own choice
  const int carveout = keep_l1 ? static_cast<int>((100 * sm_smem(R, per_sm) + ix->smem_per_sm - 1) / ix->smem_per_sm)
                               : static_cast<int>(cudaSharedmemCarveoutDefault);
  EPS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
  kernel<<<slots, kGsThreads, smem, ix->stream>>>(a);
  EPS_CUDA(cudaGetLastError());
  if (stats) {
    stats->n_seed += static_cast<uint64_t>(nq) * static_cast<uint64_t>(L);
    stats->kernel_launches += launches;
  }
  return EPS_OK;
}

int graph_launch_prologue(Index* ix, int64_t L, const char* who, int* Lp) {
  if (L < 1 || L > ix->n_indexed) return fail(EPS_ERR_INVALID_ARGUMENT, std::string(who) + ": L out of range");
  *Lp = std::max(2, next_pow2(static_cast<int>(L)));
  if (*Lp > 16384) return fail(EPS_ERR_UNSUPPORTED, "SearchQueueSize above 16384 is not supported by the graph kernel");
  return prepare_init_ids(ix, L);
}

int graph_counters(Index* ix, int64_t nq) {
  EPS_TRY(ix->s_misc.reserve(kGcSlots * 8));
  EPS_CUDA(cudaMemsetAsync(ix->s_misc.p, 0, kGcSlots * 8, ix->stream));
#ifdef EPS_GS_PROFILE
  ix->prof_nq = nq;
  ix->prof_timeline = false;  // graph_search sets up a per-query timeline
#endif
  return EPS_OK;
}

int prepare_visited(Index* ix, int slots, int64_t L, VisitedSets* v) {
  const int64_t words = ((ix->n_indexed + 31) / 32 + 3) & ~3ll;
  if (ix->visited_slots < slots || ix->s_visited.cap < static_cast<size_t>(slots) * words * 4) {
    EPS_TRY(ix->s_visited.reserve(static_cast<size_t>(slots) * words * 4));
    ix->visited_slots = slots;
  }
  // bitmaps must start clean; the kernel leaves them clean.  (Re)zero when the buffer or the geometry changed.
  if (ix->visited_gen != ix->s_visited.gen || ix->visited_words != words) {
    EPS_CUDA(cudaMemsetAsync(ix->s_visited.p, 0, ix->s_visited.cap, ix->stream));
    ix->visited_gen = ix->s_visited.gen;
    ix->visited_words = words;
  }
  // Visited hash sets: 16 entries per queue slot, so that the ~10 L ids a query visits load its table about 2/3 (a
  // query that needs more moves to its bitmap), and at most 16384 entries = 64 KB per slot: the tables of the 528
  // queries resident at the benchmark's geometry take 34 MB of the 50 MB L2.  The kernel refills every table it
  // touched, so the whole buffer is all-ones between launches whatever the table size; fill it when it is (re)allocated.
  const int vset_cap = std::min(16384, std::max(1024, next_pow2(16 * static_cast<int>(L))));
  EPS_TRY(ix->s_vset.reserve(static_cast<size_t>(slots) * vset_cap * 4));
  if (ix->vset_gen != ix->s_vset.gen) {
    EPS_CUDA(cudaMemsetAsync(ix->s_vset.p, 0xff, ix->s_vset.cap, ix->stream));
    ix->vset_gen = ix->s_vset.gen;
  }
  // fresh ids of the running query in FIFO order: the migration to the bitmap and the bitmap reset read them
  constexpr int kVlogCap = 32768;
  EPS_TRY(ix->s_vlog.reserve(static_cast<size_t>(slots) * kVlogCap * 4));
  v->vset = ix->s_vset.as<uint32_t>(); v->vset_cap = vset_cap; v->vset_max = vset_cap / 4 * 3;
  v->vset_shift = 32 - (__builtin_ctz(static_cast<unsigned>(vset_cap)) - 3);
  v->visited = ix->s_visited.as<uint32_t>(); v->words = words;
  v->vlog = ix->s_vlog.as<int32_t>(); v->vlog_cap = kVlogCap;
  return EPS_OK;
}

// Device counters of the last graph_search launch (call after the stream has been synchronised).
int read_graph_counters(Index* ix, eps_stats* stats) {
  if (!stats || !ix->s_misc.p) return EPS_OK;
  unsigned long long h[kGcSlots];
  EPS_CUDA(cudaMemcpy(h, ix->s_misc.p, sizeof(h), cudaMemcpyDeviceToHost));
  stats->n_dist += h[kGcDist];
  stats->n_expand += h[kGcExpand];
  stats->n_edges += h[kGcEdges];
#ifdef EPS_GS_PROFILE
  const unsigned long long* pr = h;
  const char* names[8] = {"barrierX", "merge", "screen", "rows", "pick", "barrier1", "adj+visited", "barrier2+fifo"};
  const double tot = static_cast<double>(pr[kGcCycles]) + 1.0;
  fprintf(stderr, "[gs-profile] kernel cycles summed over CTAs %.3e;", tot);
  for (int w = 0; w < 2; ++w)
    for (int i = 0; i < 8; ++i) fprintf(stderr, " w%d.%s=%.1f%%", w, names[i], 100.0 * static_cast<double>(pr[kGcPhase + w * 8 + i]) / tot);
  fprintf(stderr, "\n");
  fprintf(stderr, "[gs-profile] visited hash set: %llu test-and-inserts, %.3f table accesses (bucket reads + CAS) each; "
                  "%llu queries moved to the bitmap (%.2f%%)\n",
          pr[kGcVsetTests], static_cast<double>(pr[kGcVsetAccesses]) / (static_cast<double>(pr[kGcVsetTests]) + 1e-9), pr[kGcMigrated],
          ix->prof_nq > 0 ? 100.0 * static_cast<double>(pr[kGcMigrated]) / static_cast<double>(ix->prof_nq) : 0.0);
  if (ix->prof_timeline && ix->prof_nq > 0) {
    std::vector<unsigned long long> t(static_cast<size_t>(ix->prof_nq) * 4);
    EPS_CUDA(cudaMemcpy(t.data(), ix->s_prof_qtimes.p, t.size() * 8, cudaMemcpyDeviceToHost));
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
