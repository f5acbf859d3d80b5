// Device code shared by the graph-search kernels (graph_search.cu: dense rows, sparse_graph.cu: sparse rows): the slots
// of their counter block, the visited set (its sizes, rules, seeding, test-and-insert, move to the bitmap and clean-up),
// the pick's scan of unchecked queue entries and the block merge of accepted keys into the sorted queue.
#pragma once
#include <algorithm>

#include "common.cuh"

namespace eps {

constexpr int kGsThreads = 128;
constexpr int kPC = 128;        // accepted keys pending their merge (= one key per thread in the merge)

// Counter block of one launch of either kernel (Index::s_misc, zeroed by graph_counters): 64-bit slots summed over CTAs.
// read_graph_counters adds the first three to eps_stats; the developer build (EPS_GS_PROFILE) prints the others.
enum GraphCounter {
  kGcDist, kGcExpand, kGcEdges,  // n_dist, n_expand, n_edges
  kGcWork,                       // work counter: the next query to claim (an int)
  kGcVsetTests,                  // developer: hash-set test-and-inserts (dense kernel)
  kGcVsetAccesses,               // developer: hash-set accesses (bucket reads + CAS)
  kGcMigrated,                   // developer: queries moved to the bitmap (dense kernel)
  kGcCycles,                     // developer: kernel cycles of warp 0 (dense kernel)
  kGcPhase,                      // developer: 16 phase timers of the dense kernel, warp 0 then warp 1
  kGcSlots = kGcPhase + 16
};

__device__ __forceinline__ int lb_masked(const unsigned long long* a, int n, unsigned long long key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if ((a[mid] & kKeyMask) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// ---- Visited set of one query, used by both kernels on their CTA's slot (prepare_visited allocates the slots) ----
// Each slot has a hash set in global memory, a bitmap of n_indexed bits and a log of the query's fresh ids.
//  * The hash set has vset_cap_for(L) entries, 16 per queue slot clamped to [kVsetMinCap, kVsetMaxCap].  The ~10 L ids
//    a query typically visits then fill about 2/3 of it.  At most 64 KB per slot keeps the tables of all resident
//    queries in L2: 34 MB for the 528 queries resident at the benchmark's geometry, of the H100's 50 MB.
//  * A query inserts at most vset_max_for(cap) = 3/4 of the entries.  Linear probing then always finds a free entry
//    (vset_claim terminates) after a short run.  Before a step that could insert past that, the query moves to its
//    bitmap for the rest of its run (move_to_bitmap); from then on a test-and-set is one atomicOr.
//  * The seeds and the log are every id the query has visited.  The set starts empty, the seeds are inserted first,
//    and every id a step finds fresh is appended to the log in order.  The log holds kVlogCap > 3/4 of the largest
//    set, so at the move nothing has been dropped from it.
//  * After the query the slot is left clean for the next one (reset_visited).  The hash set is refilled whole (at most
//    64 KB, in L2).  The bitmap is dirty only if the query moved to it.  Then, if the log holds every fresh id and the
//    seeds plus the log are under 1 / kClearRatio of the bitmap's words, only the words they touched are cleared;
//    otherwise the whole bitmap is.  A scattered 4-byte store still writes a 32-byte sector (8 words), so it moves
//    fewer bytes than the streamed clear only below 1/8 of the words; 1/10 keeps a margin.  At 10M rows the bitmap is
//    1.25 MB per query.
constexpr int kVsetMinCap = 1024, kVsetMaxCap = 16384;  // hash-set entries per slot
constexpr int kVlogCap = 32768;                         // fresh ids logged per query
constexpr int kClearRatio = 10;
inline int vset_cap_for(int64_t L) { return std::min(kVsetMaxCap, std::max(kVsetMinCap, next_pow2(16 * static_cast<int>(L)))); }
constexpr int vset_max_for(int cap) { return cap / 4 * 3; }
static_assert(vset_max_for(kVsetMaxCap) < kVlogCap, "the log must hold every fresh id of a query that moves to the bitmap");

// Hash set: linear probing over the entries of a slot's table from the first entry of the id's bucket of 8
// (multiplicative hash).  Entries go from kVsetEmpty to an id once and stay until the table is refilled after the
// query, so an id found anywhere is visited, and an entry seen holding another id stays so.  Of two threads racing on
// one id exactly one finds it fresh.  Reads bypass L1 (__ldcg): the entries are written by L2 atomics.
constexpr uint32_t kVsetEmpty = 0xffffffffu;  // ids are < 2^31
constexpr uint32_t kVsetMul = 0x9e3779b1u;
__device__ __forceinline__ uint32_t vset_bucket(uint32_t id, int shift) { return ((id * kVsetMul) >> shift) << 3; }
// Test-and-insert from entry p on, one atomicCAS per entry: true when the id was absent (this thread inserted it).
// Terminates because a query never fills its table beyond 3/4.  `acc` counts table accesses (developer build).
__device__ __forceinline__ bool vset_claim(uint32_t* t, uint32_t mask, uint32_t p, uint32_t id, unsigned long long& acc) {
  for (;;) {
    const uint32_t old = atomicCAS(t + p, kVsetEmpty, id);
#ifdef EPS_GS_PROFILE
    ++acc;
#endif
    if (old == kVsetEmpty) return true;
    if (old == id) return false;
    p = (p + 1) & mask;
  }
}
// Test-and-insert in three steps, so that a thread can issue the bucket reads of several ids, then their CASes:
//   at = vset_probe(...)                          one 32-byte bucket read; kVsetEmpty: the id is there (visited), else
//                                                 the entry to CAS (the bucket's first free one, or the next bucket's
//                                                 first when it is full)
//   old = atomicCAS(vset + at, kVsetEmpty, id)
//   fresh = vset_settle(...)                      true when this thread inserted the id; a CAS lost to another id
//                                                 probes on entry by entry
__device__ __forceinline__ uint32_t vset_probe(const uint32_t* vset, uint32_t vmask, int shift, uint32_t id) {
  const uint32_t b = vset_bucket(id, shift);
  const uint4 lo = __ldcg(reinterpret_cast<const uint4*>(vset + b)), hi = __ldcg(reinterpret_cast<const uint4*>(vset + b) + 1);
  const uint32_t e[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
  bool hit = false;
  uint32_t fe = 8;
#pragma unroll
  for (int j = 7; j >= 0; --j) {
    hit |= e[j] == id;
    if (e[j] == kVsetEmpty) fe = j;
  }
  return hit ? kVsetEmpty : (b + fe) & vmask;
}
__device__ __forceinline__ bool vset_settle(uint32_t* vset, uint32_t vmask, uint32_t at, uint32_t old, uint32_t id,
                                            unsigned long long& acc) {
  return old == kVsetEmpty || (old != id && vset_claim(vset, vmask, (at + 1) & vmask, id, acc));
}

// Marks one seed visited: in the hash set, or in the bitmap when the query starts there (L > vset_max).
__device__ __forceinline__ void visit_seed(uint32_t* vset, uint32_t vmask, int shift, uint32_t* visited, bool hashed, uint32_t id,
                                           unsigned long long& acc) {
  if (hashed) vset_claim(vset, vmask, vset_bucket(id, shift), id, acc);
  else atomicOr(&visited[id >> 5], 1u << (id & 31));
}

// Moves the query to its bitmap: sets the bits of the L seeds and the n logged fresh ids (all 128 threads).  Ends with
// the block barrier, so that every bit is set before any thread tests one.
__device__ __forceinline__ void move_to_bitmap(const int32_t* init_ids, int L, const int32_t* vlog, uint32_t n, uint32_t* visited) {
  for (int i = threadIdx.x; i < L; i += kGsThreads) {
    const uint32_t id = static_cast<uint32_t>(init_ids[i]);
    atomicOr(&visited[id >> 5], 1u << (id & 31));
  }
  for (uint32_t i = threadIdx.x; i < n; i += kGsThreads) {
    const uint32_t id = static_cast<uint32_t>(vlog[i]);
    atomicOr(&visited[id >> 5], 1u << (id & 31));
  }
  __syncthreads();
}

// Leaves the slot clean after a query with n_fresh fresh ids (all 128 threads): the hash set refilled with 16-byte
// stores, and the bitmap cleared if the query moved to it (hashed = false).
__device__ __forceinline__ void reset_visited(uint32_t* vset, int vset_cap, bool hashed, uint32_t* visited, int64_t words,
                                              const int32_t* init_ids, int L, const int32_t* vlog, uint32_t n_fresh) {
  const int tid = threadIdx.x;
  uint4* t4 = reinterpret_cast<uint4*>(vset);
  const uint4 e = make_uint4(kVsetEmpty, kVsetEmpty, kVsetEmpty, kVsetEmpty);
  for (int i = tid; i < (vset_cap >> 2); i += kGsThreads) t4[i] = e;
  if (hashed) return;
  if (n_fresh <= static_cast<uint32_t>(kVlogCap) && static_cast<long long>(kClearRatio) * (n_fresh + L) < words) {
    for (int i = tid; i < L; i += kGsThreads) visited[static_cast<uint32_t>(init_ids[i]) >> 5] = 0u;
    for (uint32_t i = tid; i < n_fresh; i += kGsThreads) visited[static_cast<uint32_t>(vlog[i]) >> 5] = 0u;
  } else {
    uint4* v4 = reinterpret_cast<uint4*>(visited);
    const int64_t n4 = words >> 2;
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (int64_t i = tid; i < n4; i += kGsThreads) v4[i] = z;
  }
}

// Every seed starts unchecked: bits [0, L) of the unchecked-entry bitmap (one bit per queue slot).
__device__ __forceinline__ void init_unchecked(unsigned* ubits, int L) {
  for (int w = threadIdx.x; w < ((L + 31) >> 5); w += kGsThreads) ubits[w] = (w * 32 + 32 <= L) ? 0xffffffffu : ((1u << (L & 31)) - 1u);
}

// Warp scan of the unchecked-entry bitmap (all 32 lanes, same answer): the first unchecked queue entry at or after the
// cursor sp, -1 when there is none.
__device__ __forceinline__ int first_unchecked(const unsigned* ubits, int L, int sp, int lane) {
  const int nwords = (L + 31) >> 5;
  for (int w0 = sp >> 5; w0 < nwords; w0 += 32) {
    const int wi = w0 + lane;
    unsigned word = wi < nwords ? ubits[wi] : 0u;
    if (wi == (sp >> 5)) word &= ~((1u << (sp & 31)) - 1u);  // entries before the cursor are not looked at
    const unsigned b = __ballot_sync(kFull, word != 0u);
    if (b) {
      const int src = __ffs(b) - 1;
      const unsigned wsel = __shfl_sync(kFull, word, src);
      return (w0 + src) * 32 + __ffs(wsel) - 1;
    }
  }
  return -1;
}

// Block-wide merge of the m (<= kPC) pending keys into the sorted queue qa[0..L): sort by counting, binary-search
// the insertion points, shift the tail in place in super-tiles of 8 keys per thread (each key moves right by the
// number of pending keys that precede it), drop the keys into the holes.  Entries pushed past L are evicted
// (AddIntoQueue's drop-worst, :104-108).  Returns the lowest insert position through *s_cursor (min).  kQueue = false:
// a plain sorted list of L keys (the collect mode's passing rows), with no cursor and no unchecked-entry bitmap.
template <bool kQueue = true>
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
    if (kQueue && p0 < *s_cursor) *s_cursor = p0;
  }
  __syncthreads();
  // the unchecked-entry bitmap (one bit per queue slot, what the pick scans) from the first changed word on
  if (kQueue && p0 < L) {
    const int nwords = (L + 31) >> 5, lane = tid & 31;
    for (int w = (p0 >> 5) + (tid >> 5); w < nwords; w += kGsThreads / 32) {
      const int idx = w * 32 + lane;
      const unsigned b = __ballot_sync(kFull, idx < L && !(qa[idx] & kCheckedBit));
      if (lane == 0) ubits[w] = b;
    }
    __syncthreads();
  }
}

}  // namespace eps
