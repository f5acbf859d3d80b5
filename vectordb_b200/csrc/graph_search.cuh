// Device code shared by the graph-search kernels (graph_search.cu: dense rows, sparse_graph.cu: sparse rows): the slots
// of their counter block, the visited hash set and the block merge of accepted keys into the sorted queue.
#pragma once
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

// Visited hash set: linear probing over the entries of a slot's table from the first entry of the id's bucket
// (multiplicative hash).  Entries go from kVsetEmpty to an id once and stay until the table is refilled after the
// query, so an id found anywhere is visited, and an entry seen holding another id stays so.  Reads bypass L1
// (__ldcg): the entries are written by L2 atomics.
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
