// K1-TC — coarse distance tiles of the exact scan on the Hopper tensor cores (wgmma, sm_90a).
//
// The large-batch exact scan (BruteForceSearch / PreFilter branch, engine/db/execution/vec_search_executor.cpp
// :717-831, at batch B) is a dense contraction D[q,r] = <Q[q,:], X[r,:]> with 2*B*N*d flops against N*d*4 bytes
// (512 flop/B at B = 1024), far more arithmetic per byte than the fp32 SIMT tile kernel in brute_force.cu can
// issue.  This kernel produces the same [B x chunk] distance tile with warpgroup MMAs (wgmma, TF32 or BF16 inputs,
// fp32 accumulate):
//   * operands stay the reference's fp32 rows — TMA (cp.async.bulk.tensor, 128-byte swizzle) stages 128-row x 32-
//     float blocks of the table and 256-query x 32-float blocks of the query batch into a 4-stage shared-memory
//     ring; the tensor cores read them as TF32 (no converted copy of the table is kept);
//   * warpgroup 0 is the producer (one thread issues the TMA loads); warpgroups 1 and 2 each own 64 rows of the
//     128-row tile and issue 4 wgmma m64n256k8 per 128-byte block straight from shared-memory descriptors into a
//     64 x 256 fp32 register accumulator (128 registers per thread), releasing each stage as its MMAs retire;
//   * the consumer warpgroups turn dot products into the metric in registers (|x|^2 + |q|^2 - 2 dot | 1 - dot |
//     -dot) and store the tile query-major, or filter it against the running thresholds; meanwhile the producer
//     keeps filling the ring for the next tile.
// TF32 products carry ~1e-3 relative error, so this is a COARSE pass: bf_select_kernel keeps k' > k candidates
// per query and rescore_kernel re-evaluates them with the exact fp32 direct form before the final (distance,id)
// sort — returned ids/distances are those of the fp32 path (SURVEY.md §7 step 3: "TF32 MMA with fp32 re-score of
// survivors").  Bound: tensor pipe / L2 operand traffic (DESIGN.md §3).
#include <cuda.h>
#include <cuda_bf16.h>

#include <cstdlib>

#include "async.cuh"
#include "internal.h"

namespace eps {

constexpr int kTcBM = 128;      // table rows per tile  (two consumer warpgroups x wgmma M = 64)
constexpr int kTcBN = 256;      // queries per tile     (wgmma N)
constexpr int kTcBK = 32;       // floats per k-block = one 128-byte swizzle atom
constexpr int kTcStages = 4;
constexpr int kTcABytes = kTcBM * kTcBK * 4;   // 16 KB
constexpr int kTcBBytes = kTcBN * kTcBK * 4;   // 32 KB
constexpr int kTcStageBytes = kTcABytes + kTcBBytes;
constexpr int kTcThreads = 384;  // warpgroup 0 TMA, warpgroups 1-2 MMA + epilogue
constexpr int kTcEpiWarps = 8;
constexpr int kTcStgCap = 256;   // staged survivors per consumer warp (8-byte key + 2-byte query index each)
constexpr int kTcStgBytes = kTcEpiWarps * kTcStgCap * 10 + 4 * kTcEpiWarps;
constexpr int kTcSmem = kTcStages * kTcStageBytes + 1024 /*align*/ + 8192 /*qnorm + thresholds*/ + 256 /*barriers*/ + kTcStgBytes;
static_assert(kTcSmem <= 227 * 1024, "tc_dist_kernel must fit the 227 KB of shared memory a block may use");

struct TcArgs {
  int64_t row_start;   // absolute first row of this chunk
  int64_t n;           // rows in this chunk
  int64_t nq;
  int64_t ldd;
  const float* xnorm;  // |x|^2 per absolute row (L2 only)
  const float* qnorm;  // |q|^2 per query (L2 only)
  float* D;            // [nq x ldd]
  int dim;
  int metric;
  int n_row_tiles;
  int n_q_tiles;
  int kb_elems;        // elements per 128-byte k-block: 32 (fp32 read as TF32) or 64 (bf16 mirror)
  // fused selection (D == nullptr): only entries below the query's running threshold leave the SM
  const float* thr;             // [nq] coarse k'-th best so far
  unsigned long long* cand;     // [nq x cand_cap] keys
  int* cand_cnt;                // [nq]
  const uint32_t* pass;         // deleted / static-filter bitmap relative to pass_base (may be null)
  int64_t pass_base;
  int cand_cap;
};

// Survivors of the fused selection are staged per consumer warp in shared memory.  A push straight to the per-query
// list needs the value its global atomicAdd returns (a long round trip under contention) before the warp can go on,
// and while the running thresholds are still loose — the first fused launches of a scan, or a clustered table where
// whole blobs pass — those round trips, serialised per warp, would dominate the launch.  The stage is checked every
// 8 queries of a thread's accumulator, flushed when half full and at the end of the CTA's tiles, four independent
// global atomics per lane at a time.
struct TcStage {
  unsigned long long* key;  // [kTcStgCap]
  unsigned short* q;        // [kTcStgCap]
  int* cnt;
  const float* qn;          // |q|^2 per query of the batch (shared memory)
};

__device__ __forceinline__ void cand_push_global(const TcArgs& a, int q, unsigned long long key) {
  const int slot = atomicAdd(&a.cand_cnt[q], 1);
  if (slot < a.cand_cap) a.cand[static_cast<int64_t>(q) * a.cand_cap + slot] = key;
}

__device__ __forceinline__ void cand_flush(const TcArgs& a, const TcStage& st, int lane) {
  __syncwarp();
  const int n = min(*st.cnt, kTcStgCap);
  for (int base = 0; base < n; base += 128) {
    int q[4], slot[4];
    unsigned long long key[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int idx = base + 32 * u + lane;
      q[u] = idx < n ? st.q[idx] : -1;
      key[u] = idx < n ? st.key[idx] : 0ull;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) slot[u] = q[u] >= 0 ? atomicAdd(&a.cand_cnt[q[u]], 1) : a.cand_cap;
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (slot[u] < a.cand_cap) a.cand[static_cast<int64_t>(q[u]) * a.cand_cap + slot[u]] = key[u];
  }
  __syncwarp();
  if (lane == 0) *st.cnt = 0;
  __syncwarp();
}

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
// K-major, 128-byte-swizzled operand tile: rows of 128 bytes, 8-row groups 1024 bytes apart (stride byte offset),
// layout type 1 = SWIZZLE_128B (wgmma matrix descriptor, PTX ISA "Matrix Descriptor Format").  Every operand base is
// 1024-byte aligned, so the base-offset field stays 0.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFF) >> 4);        // start address, 16-byte units
  d |= static_cast<uint64_t>(1) << 16;                        // leading byte offset (unused for swizzled K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;                // stride byte offset = 8 rows * 128 B
  d |= static_cast<uint64_t>(1) << 62;                        // SWIZZLE_128B
  return d;
}
// D[64 x 256] (+)= A[64 x K] * B[256 x K]^T, both K-major in shared memory; K = 8 (tf32) or 16 (bf16).
__device__ __forceinline__ void wgmma_tf32(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1;\n"
      "}\n"
      :
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_bf16(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, 0, 0;\n"
      "}\n"
      :
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads or writes across the asynchronous MMAs
__device__ __forceinline__ void acc_fence(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// One fused-mode survivor (t = m*dot + |x|^2 passed the query's threshold): the coarse distance goes to the warp's stage.
__device__ __forceinline__ void stage_push(const TcArgs& a, const TcStage& st, int q, float t, int64_t row_abs) {
  float d = t;
  if (a.metric == EPS_METRIC_L2) d = fmaxf(d + st.qn[q], 0.f);
  else if (a.metric == EPS_METRIC_COSINE) d = 1.0f + d;
  const unsigned long long key = make_key(d, static_cast<uint32_t>(row_abs));
  const int pos = atomicAdd(st.cnt, 1);  // shared memory
  if (pos < kTcStgCap) { st.key[pos] = key; st.q[pos] = static_cast<unsigned short>(q); }
  else cand_push_global(a, q, key);      // stage full (flushed at the next check)
}

// Epilogue of one 64 x 256 accumulator.  This thread holds rows r[h] (h = 0, 1: acc[4j + 2h + c]) and queries
// qc + 8j + c (j < 32, c = 0, 1) — the wgmma fp32 accumulator fragment.
__device__ __forceinline__ void epilogue(const TcArgs& a, const float (&acc)[128], int qc, const bool (&row_ok)[2],
                                         const float (&xn)[2], const int64_t (&i)[2], const int64_t (&row_abs)[2],
                                         const float* thr_s, const float* qn_s, const TcStage& st, int lane) {
  if (a.D == nullptr) {
    // ---- fused selection: 2 instructions per element (FFMA + compare), survivors are rare ----
    const float m = a.metric == EPS_METRIC_L2 ? -2.0f : -1.0f;
#pragma unroll
    for (int g = 0; g < 8; ++g) {
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = 4 * g + jj;
        const float2 ct = *reinterpret_cast<const float2*>(thr_s + qc + 8 * j);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float t0 = fmaf(m, acc[4 * j + 2 * h], xn[h]), t1 = fmaf(m, acc[4 * j + 2 * h + 1], xn[h]);
          if (row_ok[h] && ((t0 < ct.x) | (t1 < ct.y))) {
            if (t0 < ct.x) stage_push(a, st, qc + 8 * j, t0, row_abs[h]);
            if (t1 < ct.y) stage_push(a, st, qc + 8 * j + 1, t1, row_abs[h]);
          }
        }
      }
      __syncwarp();
      if (*st.cnt >= kTcStgCap / 2) cand_flush(a, st, lane);
    }
  } else {
    // ---- distance tile to global memory (first chunk: seeds the running thresholds) ----
#pragma unroll
    for (int j = 0; j < 32; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int q = qc + 8 * j + c;
          if (row_ok[h] && q < a.nq) {
            const float dot = acc[4 * j + 2 * h + c];
            float d;
            if (a.metric == EPS_METRIC_L2) d = fmaxf(xn[h] + qn_s[q] - 2.0f * dot, 0.f);
            else if (a.metric == EPS_METRIC_COSINE) d = 1.0f - dot;
            else d = -dot;
            a.D[static_cast<int64_t>(q) * a.ldd + i[h]] = d;
          }
        }
      }
    }
  }
}

template <bool BF16>
__global__ void __launch_bounds__(kTcThreads, 1) tc_dist_kernel(const __grid_constant__ CUtensorMap tmA,
                                                              const __grid_constant__ CUtensorMap tmB, TcArgs a) {
  extern __shared__ unsigned char tc_smem_raw[];
  // 1024-byte alignment for the 128-byte swizzle pattern
  unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~uintptr_t(1023));
  float* qn_s = reinterpret_cast<float*>(base + kTcStages * kTcStageBytes);  // [<=1024]
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + kTcStages * kTcStageBytes + 8192);  // [0..3] full, [4..7] empty
  unsigned char* stg = base + kTcStages * kTcStageBytes + 8192 + 256;  // [8 x keys][8 x query indices][8 counters]
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + kTcStages);
  const uint32_t stage0 = smem_u32(base);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkb = (a.dim + a.kb_elems - 1) / a.kb_elems;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kTcStages; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, kTcEpiWarps); }
    mbar_fence_init();
  }
  float* thr_s = qn_s + 1024;  // [<=1024] thresholds (fused mode)
  // fused mode compares t = m*dot + xn (m = -2 for L2, -1 otherwise) with a per-query constant:
  //   L2: d = t + |q|^2 < thr  <=>  t < thr - |q|^2;   cosine: d = 1 + t < thr  <=>  t < thr - 1;   IP: d = t < thr.
  // Queries beyond nq get -inf, so they never pass and need no bounds test in the inner loop.
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) {
    const float qn = (a.metric == EPS_METRIC_L2 && i < a.nq) ? a.qnorm[i] : 0.f;
    qn_s[i] = qn;
    float c = -INFINITY;
    if (a.D == nullptr && i < a.nq) {
      const float th = a.thr[i];
      c = a.metric == EPS_METRIC_L2 ? th - qn : (a.metric == EPS_METRIC_COSINE ? th - 1.0f : th);
    }
    thr_s[i] = c;
  }
  __syncthreads();

  const int tiles_per_row = a.n_q_tiles;
  if (warp < 4) {
    // ===== TMA producer (warpgroup 0; gives its registers to the consumers) =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (threadIdx.x == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
      uint32_t it = 0;
      for (int rt = blockIdx.x; rt < a.n_row_tiles; rt += gridDim.x) {
        const int row0 = static_cast<int>(a.row_start) + rt * kTcBM;
        for (int qt = 0; qt < tiles_per_row; ++qt) {
          for (int kb = 0; kb < nkb; ++kb, ++it) {
            const uint32_t s = it % kTcStages, ph = (it / kTcStages) & 1;
            mbar_wait(empty0 + 8 * s, ph ^ 1);
            mbar_expect_tx(full0 + 8 * s, kTcStageBytes);
            const uint32_t sa = stage0 + s * kTcStageBytes;
            tma_load_2d(sa, &tmA, kb * a.kb_elems, row0, full0 + 8 * s);
            tma_load_2d(sa + kTcABytes, &tmB, kb * a.kb_elems, qt * kTcBN, full0 + 8 * s);
          }
        }
      }
    }
  } else {
    // ===== consumers: warpgroup 1 + cw owns rows 64*cw .. +63 of every tile, warp (warp & 3) 16 of them =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int cw = (warp >> 2) - 1, ew = warp - 4;
    TcStage st;
    st.key = reinterpret_cast<unsigned long long*>(stg) + ew * kTcStgCap;
    st.q = reinterpret_cast<unsigned short*>(stg + kTcEpiWarps * kTcStgCap * 8) + ew * kTcStgCap;
    st.cnt = reinterpret_cast<int*>(stg + kTcEpiWarps * kTcStgCap * 10) + ew;
    st.qn = qn_s;
    if (lane == 0) *st.cnt = 0;
    __syncwarp();
    const int r_lo = 64 * cw + 16 * (warp & 3) + (lane >> 2);  // tile row of acc[4j + 0..1]; acc[4j + 2..3]: r_lo + 8
    float acc[128];
#pragma unroll
    for (int v = 0; v < 128; ++v) acc[v] = 0.f;
    uint32_t it = 0;
    for (int rt = blockIdx.x; rt < a.n_row_tiles; rt += gridDim.x) {
      bool row_ok[2];
      float xn[2];
      int64_t i[2], row_abs[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        i[h] = static_cast<int64_t>(rt) * kTcBM + r_lo + 8 * h;  // row index inside the chunk
        row_ok[h] = i[h] < a.n;
        xn[h] = (a.metric == EPS_METRIC_L2 && row_ok[h]) ? a.xnorm[a.row_start + i[h]] : 0.f;
        row_abs[h] = a.row_start + i[h];
        if (a.D == nullptr && a.pass && row_ok[h]) {
          const int64_t pi = row_abs[h] - a.pass_base;
          row_ok[h] = (a.pass[pi >> 5] >> (pi & 31)) & 1u;
        }
      }
      for (int qt = 0; qt < tiles_per_row; ++qt) {
        uint32_t prev = 0;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const uint32_t s = it % kTcStages, ph = (it / kTcStages) & 1;
          mbar_wait(full0 + 8 * s, ph);
          const uint32_t sa = stage0 + s * kTcStageBytes;
          const uint64_t ad = gmma_desc(sa + cw * (kTcABytes / 2)), bd = gmma_desc(sa + kTcABytes);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) {  // 4 MMAs per 128-byte block: K = 8 tf32 / 16 bf16 = 32 bytes = +2 (16-B units)
            if (BF16) wgmma_bf16(acc, ad + 2 * k, bd + 2 * k, (kb | k) ? 1u : 0u);
            else wgmma_tf32(acc, ad + 2 * k, bd + 2 * k, (kb | k) ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<1>();  // the previous block's MMAs have retired: its stage can be refilled
          if (kb > 0 && lane == 0) mbar_arrive(empty0 + 8 * prev);
          prev = s;
        }
        wgmma_wait<0>();
        acc_fence(acc);
        if (lane == 0) mbar_arrive(empty0 + 8 * prev);
        epilogue(a, acc, qt * kTcBN + 2 * (lane & 3), row_ok, xn, i, row_abs, thr_s, qn_s, st, lane);
        acc_fence(acc);
      }
    }
    if (a.D == nullptr) cand_flush(a, st, lane);  // what is left in the stage (it is also flushed whenever half full)
  }
}

// |x|^2 per row (fp32, warp per row) for the L2 expansion of the coarse pass.
__global__ void row_norm_kernel(const float* __restrict__ v, int64_t row0, int64_t n, int dim, float* __restrict__ out) {
  const int64_t w = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const float* p = v + (row0 + w) * dim;
  float s = 0.f;
  for (int i = lane; i < dim; i += 32) s = fmaf(p[i], p[i], s);
  s = warp_sum(s);
  if (lane == 0) out[row0 + w] = s;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static int make_map(CUtensorMap* tm, const void* base, int64_t rows, int dim, int box_rows, bool bf16) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(EPS_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  const int esz = bf16 ? 2 : 4;
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(dim), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstride[1] = {static_cast<cuuint64_t>(dim) * esz};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(128 / esz), static_cast<cuuint32_t>(box_rows)};  // 128-byte rows
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base),
                   gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(EPS_ERR_CUDA, "cuTensorMapEncodeTiled failed: " + std::to_string(static_cast<int>(r)));
  return EPS_OK;
}

__global__ void to_bf16_kernel(const float* __restrict__ in, int64_t n, unsigned short* __restrict__ out) {
  const int64_t i = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) * 4;
  if (i + 3 < n) {
    const float4 v = *reinterpret_cast<const float4*>(in + i);
    const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<const uint32_t*>(&a);
    o.y = *reinterpret_cast<const uint32_t*>(&b);
    *reinterpret_cast<uint2*>(out + i) = o;
  } else {
    for (int64_t j = i; j < n; ++j) {
      const __nv_bfloat16 h = __float2bfloat16_rn(in[j]);
      out[j] = *reinterpret_cast<const unsigned short*>(&h);
    }
  }
}

bool tc_dist_usable(const Index* ix, int64_t nq) {
  static const bool env_off = getenv("EPS_NO_TC") != nullptr;  // read once
  if (env_off || ix->coarse_mode == 0) return false;
  if (nq < 64 || nq > 1024) return false;            // per-query constants live in a 4 KB shared-memory table
  const int align = ix->coarse_mode == 2 ? 8 : 4;    // TMA: 16-byte row pitch
  if (ix->dim % align != 0 || ix->dim < 32) return false;
  if ((reinterpret_cast<uintptr_t>(ix->d_vectors) & 15) != 0) return false;
  return get_encode() != nullptr;
}

// Same contract as launch_distances() (D[q*ldd + i] for rows [row_start, row_start+n)), coarse values; with
// `fused` the tile is filtered against the running thresholds in the epilogue instead of being written.
int tc_launch_distances(Index* ix, int64_t row_start, int64_t n, const float* d_queries, int64_t nq, float* D,
                        int64_t ldd, uint64_t* launches, const TcFused* fused) {
  const int dim = static_cast<int>(ix->dim);
  const bool bf16 = ix->coarse_mode == 2;
  if (ix->metric == EPS_METRIC_L2) {
    if (ix->xnorm_rows < ix->n_rows) {  // row norms for rows appended since the last call
      EPS_TRY(ix->s_xnorm.reserve(static_cast<size_t>(ix->capacity > ix->n_rows ? ix->capacity : ix->n_rows) * 4));
      if (ix->s_xnorm.p != ix->xnorm_ptr) { ix->xnorm_rows = 0; ix->xnorm_ptr = ix->s_xnorm.p; }
      const int64_t cnt = ix->n_rows - ix->xnorm_rows;
      row_norm_kernel<<<static_cast<unsigned>((cnt * 32 + 255) / 256), 256, 0, ix->stream>>>(ix->d_vectors, ix->xnorm_rows, cnt,
                                                                                            dim, ix->s_xnorm.as<float>());
      ix->xnorm_rows = ix->n_rows;
      ++*launches;
    }
    EPS_TRY(ix->s_qnorm.reserve(static_cast<size_t>(nq) * 4));
    row_norm_kernel<<<static_cast<unsigned>((nq * 32 + 255) / 256), 256, 0, ix->stream>>>(d_queries, 0, nq, dim,
                                                                                         ix->s_qnorm.as<float>());
    ++*launches;
  }
  const void* a_base = ix->d_vectors;
  const void* b_base = d_queries;
  if (bf16) {
    // bf16 mirror of the table (coarse pass only; the re-score reads the fp32 rows), kept current incrementally
    if (ix->bf16_rows < ix->n_rows) {
      EPS_TRY(ix->s_bf16.reserve(static_cast<size_t>(ix->capacity > ix->n_rows ? ix->capacity : ix->n_rows) * dim * 2));
      if (ix->s_bf16.p != ix->bf16_ptr) { ix->bf16_rows = 0; ix->bf16_ptr = ix->s_bf16.p; }
      const int64_t cnt = (ix->n_rows - ix->bf16_rows) * dim;
      to_bf16_kernel<<<static_cast<unsigned>((cnt / 4 + 256) / 256), 256, 0, ix->stream>>>(
          ix->d_vectors + ix->bf16_rows * dim, cnt, ix->s_bf16.as<unsigned short>() + ix->bf16_rows * dim);
      ix->bf16_rows = ix->n_rows;
      ++*launches;
    }
    EPS_TRY(ix->s_qbf16.reserve(static_cast<size_t>(nq) * dim * 2));
    const int64_t cnt = nq * dim;
    to_bf16_kernel<<<static_cast<unsigned>((cnt / 4 + 256) / 256), 256, 0, ix->stream>>>(d_queries, cnt, ix->s_qbf16.as<unsigned short>());
    ++*launches;
    a_base = ix->s_bf16.p;
    b_base = ix->s_qbf16.p;
  }
  CUtensorMap tmA, tmB;
  EPS_TRY(make_map(&tmA, a_base, ix->n_rows, dim, kTcBM, bf16));
  EPS_TRY(make_map(&tmB, b_base, nq, dim, kTcBN, bf16));
  TcArgs a;
  a.row_start = row_start; a.n = n; a.nq = nq; a.ldd = ldd;
  a.xnorm = ix->s_xnorm.as<float>(); a.qnorm = ix->s_qnorm.as<float>(); a.D = D; a.dim = dim; a.metric = ix->metric;
  a.kb_elems = bf16 ? 64 : 32;
  a.thr = nullptr; a.cand = nullptr; a.cand_cnt = nullptr; a.pass = nullptr; a.pass_base = 0; a.cand_cap = 0;
  if (fused) {
    a.D = nullptr;
    a.thr = fused->thr; a.cand = fused->cand; a.cand_cnt = fused->cand_cnt; a.pass = fused->pass;
    a.pass_base = fused->pass_base; a.cand_cap = fused->cand_cap;
  }
  a.n_row_tiles = static_cast<int>((n + kTcBM - 1) / kTcBM);
  a.n_q_tiles = static_cast<int>((nq + kTcBN - 1) / kTcBN);
  static bool attr_set = false;
  if (!attr_set) {
    EPS_CUDA(cudaFuncSetAttribute(tc_dist_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmem));
    EPS_CUDA(cudaFuncSetAttribute(tc_dist_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmem));
    attr_set = true;
  }
  const int grid = std::min(a.n_row_tiles, ix->num_sms);
  if (bf16) tc_dist_kernel<true><<<grid, kTcThreads, kTcSmem, ix->stream>>>(tmA, tmB, a);
  else tc_dist_kernel<false><<<grid, kTcThreads, kTcSmem, ix->stream>>>(tmA, tmB, a);
  EPS_CUDA(cudaGetLastError());
  ++*launches;
  return EPS_OK;
}

}  // namespace eps
