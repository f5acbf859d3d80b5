// Result finalisation: the tail of VecSearchExecutor::Search (engine/db/execution/vec_search_executor.cpp
// :857-861, :864-868, :885-927) — hybrid tail merge, post-filter walk, id/distance emission — and the
// k-way shard merge used when a table is row-sharded across GPUs.
#include "internal.h"

namespace eps {

// One warp per query.
//  1. Hybrid mode (rows [n_indexed,total) not in the graph): the brute-forced tail (already deleted-/filter-
//     checked, sorted, <= min(#tail, limit) entries) is merged into the FIRST search_limit slots of the
//     master queue with the reference's fixed-length sequential merge
//     (MergeTwoQueuesInto1stQueueSeqFixed, :150-217, called at :894-900) — including its quirks: an
//     insertion at the last slot overwrites it, displaced entries are dropped, slots >= search_limit keep
//     un-merged graph candidates (SURVEY.md Q3).  Graph ids and tail ids are disjoint, so the duplicate
//     branch can never fire.  Done by lane 0 (<= limit sequential steps on <= limit entries).
//  2. Post-filter walk (:906-914 / :919-927): scan the first cand_num entries in order, skip deleted rows
//     and rows failing LogicalEvaluate(root, id, distance), emit up to search_limit.
__global__ void finalize_graph_kernel(unsigned long long* __restrict__ queues, int nq, int L, int search_limit,
                                      int cand_num, const unsigned long long* __restrict__ tail, int tail_k,
                                      int limit, const uint8_t* __restrict__ deleted, int64_t deleted_bytes,
                                      const FilterProg* __restrict__ prog, const char* __restrict__ attrs,
                                      int64_t stride, int64_t* __restrict__ out_ids, float* __restrict__ out_dists,
                                      int64_t* __restrict__ out_counts) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= nq) return;
  unsigned long long* q1 = queues + static_cast<int64_t>(warp) * L;
  if (tail && lane == 0) {
    const unsigned long long* q2 = tail + static_cast<int64_t>(warp) * tail_k;
    int n2 = 0;
    while (n2 < tail_k && n2 < limit && (q2[n2] & kKeyMask) != kKeyInf) ++n2;  // bruteForceQueueSize (:890)
    const int n1 = search_limit;
    if (n2 > 0 && n1 > 0) {
      auto lt = [](unsigned long long x, unsigned long long y) { return (x & kKeyMask) < (y & kKeyMask); };
      auto insert_at = [&](unsigned long long c, int idx) {  // InsertOneElementAt (:137-148)
        for (int t = n1 - 1; t > idx; --t) q1[t] = q1[t - 1];
        q1[idx] = c;
      };
      int ins = 0;
      {
        int lo = 0, hi = n1;
        while (lo < hi) { int mid = (lo + hi) >> 1; if (lt(q1[mid], q2[0])) lo = mid + 1; else hi = mid; }
        ins = lo;
      }
      if (ins == n1) {
        // nothing from the tail is better than the first search_limit entries
      } else if (ins == n1 - 1) {
        q1[ins] = q2[0];
      } else {
        insert_at(q2[0], ins);
        int i1 = ins + 1, i2 = 1;
        for (int at = ins + 1; at < n1; ++at) {
          if (i1 >= n1 || i2 >= n2) break;
          if (lt(q1[i1], q2[i2])) { ++i1; }
          else { insert_at(q2[i2++], at); ++i1; }
        }
      }
    }
  }
  __syncwarp();
  int result = 0;
  for (int base = 0; base < cand_num && result < search_limit; base += 32) {
    const int idx = base + lane;
    bool ok = false;
    unsigned long long key = 0;
    if (idx < cand_num) {
      key = q1[idx];
      const int64_t id = key_id(key);
      ok = (key & kKeyMask) != kKeyInf;
      if (ok && deleted && (id >> 3) < deleted_bytes) ok = !((deleted[id >> 3] >> (id & 7)) & 1);
      if (ok && prog) ok = filter_eval(*prog, attrs, stride, id, key_dist(key));
    }
    const unsigned b = __ballot_sync(kFull, ok);
    const int o = result + __popc(b & ((1u << lane) - 1));
    if (ok && o < search_limit) {
      out_ids[static_cast<int64_t>(warp) * limit + o] = key_id(key);
      out_dists[static_cast<int64_t>(warp) * limit + o] = key_dist(key);
    }
    result += __popc(b);
  }
  if (result > search_limit) result = search_limit;
  for (int i = result + lane; i < limit; i += 32) {
    out_ids[static_cast<int64_t>(warp) * limit + i] = -1;
    out_dists[static_cast<int64_t>(warp) * limit + i] = INFINITY;
  }
  if (lane == 0) out_counts[warp] = result;
}

// Brute-force modes: the sorted exact top-k is the brute_force_queue_; emit min(size, cap) entries
// (:857-861 prefilter: cap = limit; :864-868: cap = min(limit, L_local)).
__global__ void finalize_keys_kernel(const unsigned long long* __restrict__ topk, int nq, int k, int limit, int cap,
                                     int64_t* __restrict__ out_ids, float* __restrict__ out_dists,
                                     int64_t* __restrict__ out_counts) {
  const int q = blockIdx.x;
  if (q >= nq) return;
  __shared__ int cnt;
  if (threadIdx.x == 0) cnt = 0;
  __syncthreads();
  const unsigned long long* t = topk + static_cast<int64_t>(q) * k;
  for (int i = threadIdx.x; i < limit; i += blockDim.x) {
    bool valid = i < k && i < cap && (t[i] & kKeyMask) != kKeyInf;
    out_ids[static_cast<int64_t>(q) * limit + i] = valid ? static_cast<int64_t>(key_id(t[i])) : -1;
    out_dists[static_cast<int64_t>(q) * limit + i] = valid ? key_dist(t[i]) : INFINITY;
    if (valid) atomicAdd(&cnt, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) out_counts[q] = cnt;
}

// Collect mode (capi.cu): one thread per query merges the graph search's list of passing rows with the tail scan's top
// keys.  Both are ascending and kKeyInf padded, and their rows are disjoint (graph rows < n_indexed <= tail rows), so
// the first cap keys of the merge are the best cap of the union: no slot quirk of the post-filter merge applies.  A
// query left with fewer than min(cap, P) keys is listed in short_idx.
__global__ void collect_merge_kernel(const unsigned long long* __restrict__ list, const unsigned long long* __restrict__ tail,
                                     int nq, int cap, int tail_k, int64_t P, unsigned long long* __restrict__ out,
                                     int* __restrict__ short_idx, int* __restrict__ n_short) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  const unsigned long long* a = list + static_cast<int64_t>(q) * cap;
  const unsigned long long* b = tail ? tail + static_cast<int64_t>(q) * tail_k : nullptr;
  unsigned long long* o = out + static_cast<int64_t>(q) * cap;
  int i = 0, j = 0, n = 0;
  for (int t = 0; t < cap; ++t) {
    const unsigned long long x = i < cap ? a[i] & kKeyMask : kKeyInf;
    const unsigned long long y = j < tail_k ? b[j] & kKeyMask : kKeyInf;
    unsigned long long z;
    if (x <= y) { z = x; ++i; } else { z = y; ++j; }
    o[t] = z;
    n += z != kKeyInf;
  }
  if (n < min(static_cast<int64_t>(cap), P)) short_idx[atomicAdd(n_short, 1)] = q;
}

// k-way merge of n_shards sorted lists per query (ids are GLOBAL int64).  One CTA per query, bitonic
// sort of the (ordered-distance, id) pairs in shared memory.
__global__ void merge_shards_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dists, int n_shards,
                                    int nq, int k, int np, int64_t id_stride, int64_t dist_stride,
                                    int64_t* __restrict__ out_ids, float* __restrict__ out_dists) {
  extern __shared__ __align__(16) unsigned char ms_smem[];
  int64_t* sid = reinterpret_cast<int64_t*>(ms_smem);
  uint32_t* sod = reinterpret_cast<uint32_t*>(sid + np);
  const int q = blockIdx.x;
  const int n = n_shards * k;
  for (int i = threadIdx.x; i < np; i += blockDim.x) {
    int64_t id = -1;
    uint32_t od = 0xffffffffu;
    if (i < n) {
      const int s = i / k, j = i % k;
      const int64_t within = static_cast<int64_t>(q) * k + j;  // shard s: ids + s*id_stride, dists + s*dist_stride
      id = ids[static_cast<int64_t>(s) * id_stride + within];
      od = id >= 0 ? float_to_ordered(dists[static_cast<int64_t>(s) * dist_stride + within]) : 0xffffffffu;
      if (id < 0) id = INT64_MAX;
    } else {
      id = INT64_MAX;
    }
    sid[i] = id;
    sod[i] = od;
  }
  __syncthreads();
  for (int kk = 2; kk <= np; kk <<= 1) {
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < np; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const bool up = (i & kk) == 0;
          const bool gt = sod[i] > sod[ixj] || (sod[i] == sod[ixj] && sid[i] > sid[ixj]);
          if (gt == up) {
            uint32_t to = sod[i]; sod[i] = sod[ixj]; sod[ixj] = to;
            int64_t ti = sid[i]; sid[i] = sid[ixj]; sid[ixj] = ti;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    const bool valid = sid[i] != INT64_MAX;
    out_ids[static_cast<int64_t>(q) * k + i] = valid ? sid[i] : -1;
    out_dists[static_cast<int64_t>(q) * k + i] = valid ? ordered_to_float(sod[i]) : INFINITY;
  }
}

int finalize_graph(Index* ix, unsigned long long* d_queue, int64_t nq, int64_t L, int64_t search_limit,
                   int64_t cand_num, const unsigned long long* d_tail, int64_t tail_k, int64_t limit,
                   const FilterProg* d_prog, const FilterProg* h_prog, int64_t* d_ids, float* d_dists,
                   int64_t* d_counts) {
  const bool has_prog = h_prog && h_prog->n > 0;
  const int threads = 128;
  const int blocks = static_cast<int>((nq * 32 + threads - 1) / threads);
  finalize_graph_kernel<<<blocks, threads, 0, ix->stream>>>(
      d_queue, static_cast<int>(nq), static_cast<int>(L), static_cast<int>(search_limit), static_cast<int>(cand_num),
      d_tail, static_cast<int>(tail_k), static_cast<int>(limit), ix->any_deleted ? ix->d_deleted.as<const uint8_t>() : nullptr,
      ix->deleted_bytes, has_prog ? d_prog : nullptr, ix->d_attrs, ix->attr_stride, d_ids, d_dists, d_counts);
  EPS_CUDA(cudaGetLastError());
  return EPS_OK;
}

int finalize_keys(Index* ix, const unsigned long long* d_topk, int64_t nq, int64_t k, int64_t limit, int64_t cap,
                  int64_t* d_ids, float* d_dists, int64_t* d_counts) {
  finalize_keys_kernel<<<static_cast<unsigned>(nq), 128, 0, ix->stream>>>(d_topk, static_cast<int>(nq), static_cast<int>(k),
                                                                        static_cast<int>(limit), static_cast<int>(cap),
                                                                        d_ids, d_dists, d_counts);
  EPS_CUDA(cudaGetLastError());
  return EPS_OK;
}

int collect_merge(Index* ix, const unsigned long long* d_list, const unsigned long long* d_tail, int64_t nq, int64_t cap,
                  int64_t tail_k, int64_t P, unsigned long long* d_out, const int** d_short_idx, int64_t* n_short) {
  EPS_TRY(ix->s_cshort.reserve(static_cast<size_t>(nq + 1) * 4));  // [count | query indices]
  int* d_n = ix->s_cshort.as<int>();
  *d_short_idx = d_n + 1;
  EPS_CUDA(cudaMemsetAsync(d_n, 0, 4, ix->stream));
  collect_merge_kernel<<<static_cast<unsigned>((nq + 127) / 128), 128, 0, ix->stream>>>(
      d_list, tail_k > 0 ? d_tail : nullptr, static_cast<int>(nq), static_cast<int>(cap), static_cast<int>(tail_k), P, d_out,
      d_n + 1, d_n);
  EPS_CUDA(cudaGetLastError());
  int h = 0;
  EPS_CUDA(cudaMemcpyAsync(&h, d_n, 4, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  *n_short = h;
  return EPS_OK;
}

int merge_shards(int device, cudaStream_t stream, const int64_t* d_ids, const float* d_dists, int64_t n_shards,
                 int64_t nq, int64_t k, int64_t* d_out_ids, float* d_out_dists, int64_t id_stride, int64_t dist_stride) {
  if (id_stride <= 0) id_stride = nq * k;      // dense [n_shards x nq x k] layout
  if (dist_stride <= 0) dist_stride = nq * k;
  EPS_CUDA(cudaSetDevice(device));
  const int np = next_pow2(static_cast<int>(n_shards * k));
  const size_t smem = static_cast<size_t>(np) * 12;
  if (smem > 200 * 1024) return fail(EPS_ERR_UNSUPPORTED, "merge_shards: n_shards * k too large");
  if (smem > 48 * 1024)
    EPS_CUDA(cudaFuncSetAttribute(merge_shards_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  merge_shards_kernel<<<static_cast<unsigned>(nq), 256, smem, stream>>>(d_ids, d_dists, static_cast<int>(n_shards),
                                                                        static_cast<int>(nq), static_cast<int>(k), np,
                                                                        id_stride, dist_stride, d_out_ids, d_out_dists);
  EPS_CUDA(cudaGetLastError());
  return EPS_OK;
}

}  // namespace eps
