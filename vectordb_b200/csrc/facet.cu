// Facets over result lists (SURVEY.md §8f-4).  Reference: FacetExecutor::Aggregate
// (engine/db/execution/aggregation.hpp:232-300): for every id of a query's result list evaluate ONE group-by
// expression (int / double / bool / string key) and the inner expressions of the aggregates with NumEvaluate (the
// candidate's distance reaches "@distance"), then SUM / COUNT / MIN / MAX per key in double precision
// (SumAggregator / CountAggregator / MinAggregator / MaxAggregator, :47-120).
//
// Device mapping, batched over nq result lists:
//   facet_eval_kernel   one thread per (query, result): key and aggregate inputs through the same program evaluator
//                       as the filters (filter.cuh); an INT key is truncated like the reference's (int64_t) cast
//                       (int_key: NaN and out-of-range keys become INT64_MIN), a
//                       BOOL key is LogicalEvaluate, a STRING key is the row's dictionary code;
//   facet_group_kernel  one warp per query: a result is a group leader if no earlier result has its key; leaders
//                       reduce their group sequentially in result order (the same order the reference adds values
//                       in, so SUMs round identically); groups come out in order of first appearance.
#include "internal.h"

namespace eps {

constexpr int kMaxAggs = 8;

struct FacetArgs {
  const int64_t* ids;      // [nq x limit]
  const double* dists;     // [nq x limit] or null
  const int64_t* counts;   // [nq]
  const FilterProg* progs; // [1 + n_aggs]: key, aggregate inputs
  const char* attrs;
  int64_t attr_stride;
  int nq, limit, n_aggs, key_type;
  int agg_types[kMaxAggs];
  double* keys;            // [nq x limit] scratch
  double* vals;            // [nq x limit x n_aggs] scratch
  double* out_keys;        // [nq x limit]
  double* out_vals;        // [nq x limit x n_aggs]
  int64_t* out_groups;     // [nq]
};

// (int64_t)(NumEvaluate(..)) of an INT key (:272) as the reference computes it on x86-64 (cvttsd2si): NaN and every value
// outside [-2^63, 2^63) become INT64_MIN.  The device's own conversion (cvt.rzi.s64.f64) saturates +inf and values of
// 2^63 and above to INT64_MAX instead.
__device__ __forceinline__ double int_key(double v) {
  constexpr double kTwo63 = 9223372036854775808.0;
  if (!(v >= -kTwo63 && v < kTwo63)) return -kTwo63;
  return static_cast<double>(static_cast<long long>(v));
}

__global__ void facet_eval_kernel(FacetArgs a) {
  const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= static_cast<int64_t>(a.nq) * a.limit) return;
  const int q = static_cast<int>(t / a.limit), i = static_cast<int>(t % a.limit);
  if (i >= a.counts[q]) return;
  const int64_t row = a.ids[t];
  const double dist = a.dists ? a.dists[t] : 0.0;
  double key;
  if (a.key_type == VT_BOOL) {
    double nv; bool bv;
    // LogicalEvaluate(root, id, distance): the filter rule for where the distance is visible applies (:170-258)
    prog_run(a.progs[0], a.attrs, a.attr_stride, row, a.progs[0].root_uses_dist ? dist : 0.0, &nv, &bv);
    key = bv ? 1.0 : 0.0;
  } else {
    key = value_eval(a.progs[0], a.attrs, a.attr_stride, row, dist);
    if (a.key_type == VT_INT) key = int_key(key);
  }
  a.keys[t] = key;
  for (int g = 0; g < a.n_aggs; ++g) a.vals[t * a.n_aggs + g] = value_eval(a.progs[1 + g], a.attrs, a.attr_stride, row, dist);
}

__global__ void facet_group_kernel(FacetArgs a) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (q >= a.nq) return;
  const int n = static_cast<int>(a.counts[q]);
  const double* keys = a.keys + static_cast<int64_t>(q) * a.limit;
  const double* vals = a.vals + static_cast<int64_t>(q) * a.limit * a.n_aggs;
  int ngroups = 0;
  for (int base = 0; base < n; base += 32) {
    const int i = base + lane;
    bool leader = i < n;
    double key = 0.0;
    if (leader) {
      key = keys[i];
      for (int j = 0; j < i && leader; ++j) leader = !(keys[j] == key);
    }
    const unsigned b = __ballot_sync(kFull, leader);
    if (leader) {
      const int slot = ngroups + __popc(b & ((1u << lane) - 1u));
      a.out_keys[static_cast<int64_t>(q) * a.limit + slot] = key;
      for (int g = 0; g < a.n_aggs; ++g) {
        double acc = 0.0;
        bool first = true;
        for (int j = i; j < n; ++j) {
          if (!(keys[j] == key)) continue;
          const double v = vals[static_cast<int64_t>(j) * a.n_aggs + g];
          switch (a.agg_types[g]) {
            case NT_SumAgg: acc += v; break;
            case NT_CountAgg: acc += 1.0; break;
            case NT_MinAgg: if (first || v < acc) acc = v; break;
            case NT_MaxAgg: if (first || v > acc) acc = v; break;
            default: break;
          }
          first = false;
        }
        a.out_vals[(static_cast<int64_t>(q) * a.limit + slot) * a.n_aggs + g] = acc;
      }
    }
    ngroups += __popc(b);
  }
  if (lane == 0) a.out_groups[q] = ngroups;
}

}  // namespace eps

using eps::Index;

extern "C" int eps_facet_batch(eps_index* h, const int64_t* ids, const double* dists, const int64_t* counts, int64_t nq,
                               int64_t limit, const eps_facet* spec, double* out_keys, double* out_values, int64_t* out_groups) {
  Index* ix = reinterpret_cast<Index*>(h);
  if (!ix || !ids || !counts || !spec || !out_keys || !out_values || !out_groups)
    return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null argument");
  if (nq <= 0) return EPS_OK;
  if (limit < 1 || limit > 8192) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "limit must be in [1, 8192]");
  if (spec->n_aggs < 1 || spec->n_aggs > eps::kMaxAggs) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "1 to 8 aggregates per facet");
  if (spec->key_type < 0 || spec->key_type > eps::VT_BOOL) return eps::fail(EPS_ERR_UNSUPPORTED, "group-by key must be string, int, double or bool");
  for (int64_t q = 0; q < nq; ++q)
    if (counts[q] < 0 || counts[q] > limit) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "result count outside [0, limit]");
  EPS_TRY(eps::check_device(ix->device));
  const int n_aggs = spec->n_aggs;
  std::vector<eps::FilterProg> progs(static_cast<size_t>(1 + n_aggs));
  EPS_TRY(eps::lower_filter(spec->key_nodes, spec->n_key_nodes, &progs[0]));
  if (progs[0].n == 0) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "empty group-by expression");
  for (int g = 0; g < n_aggs; ++g) {
    const int t = spec->agg_types[g];
    if (t != eps::NT_SumAgg && t != eps::NT_MinAgg && t != eps::NT_MaxAgg && t != eps::NT_CountAgg)
      return eps::fail(EPS_ERR_INVALID_ARGUMENT, "aggregate type must be SUM / MIN / MAX / COUNT (NodeType ordinals 30-33)");
    EPS_TRY(eps::lower_filter(spec->agg_nodes[g], spec->n_agg_nodes[g], &progs[1 + g]));
    if (progs[1 + g].n == 0) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "empty aggregate expression");
  }
  for (auto& p : progs) EPS_TRY(eps::bind_program_columns(ix, &p));
  for (int64_t i = 0, tot = nq * limit; i < tot; ++i) {
    const int64_t q = i / limit;
    if (i % limit < counts[q] && (ids[i] < 0 || ids[i] >= ix->n_rows)) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "result id outside the mirrored rows");
  }
  EPS_TRY(eps::bind_like(ix, progs.data(), static_cast<int>(progs.size()), nullptr));  // the programs' bitmaps share ix->s_like
  const size_t nl = static_cast<size_t>(nq) * limit;
  eps::DevBuf d_ids, d_dists, d_counts, d_progs, d_keys, d_vals, d_okeys, d_ovals, d_groups;
  EPS_TRY(d_ids.reserve(nl * 8));
  EPS_TRY(d_counts.reserve(static_cast<size_t>(nq) * 8));
  EPS_TRY(d_progs.reserve(progs.size() * sizeof(eps::FilterProg)));
  EPS_TRY(d_keys.reserve(nl * 8));
  EPS_TRY(d_vals.reserve(nl * 8 * n_aggs));
  EPS_TRY(d_okeys.reserve(nl * 8));
  EPS_TRY(d_ovals.reserve(nl * 8 * n_aggs));
  EPS_TRY(d_groups.reserve(static_cast<size_t>(nq) * 8));
  EPS_CUDA(cudaMemcpyAsync(d_ids.p, ids, nl * 8, cudaMemcpyHostToDevice, ix->stream));
  EPS_CUDA(cudaMemcpyAsync(d_counts.p, counts, static_cast<size_t>(nq) * 8, cudaMemcpyHostToDevice, ix->stream));
  EPS_CUDA(cudaMemcpyAsync(d_progs.p, progs.data(), progs.size() * sizeof(eps::FilterProg), cudaMemcpyHostToDevice, ix->stream));
  if (dists) {
    EPS_TRY(d_dists.reserve(nl * 8));
    EPS_CUDA(cudaMemcpyAsync(d_dists.p, dists, nl * 8, cudaMemcpyHostToDevice, ix->stream));
  }
  eps::FacetArgs a;
  a.ids = d_ids.as<int64_t>(); a.dists = dists ? d_dists.as<double>() : nullptr; a.counts = d_counts.as<int64_t>();
  a.progs = d_progs.as<eps::FilterProg>(); a.attrs = ix->d_attrs; a.attr_stride = ix->attr_stride;
  a.nq = static_cast<int>(nq); a.limit = static_cast<int>(limit); a.n_aggs = n_aggs; a.key_type = spec->key_type;
  for (int g = 0; g < eps::kMaxAggs; ++g) a.agg_types[g] = g < n_aggs ? spec->agg_types[g] : 0;
  a.keys = d_keys.as<double>(); a.vals = d_vals.as<double>(); a.out_keys = d_okeys.as<double>(); a.out_vals = d_ovals.as<double>();
  a.out_groups = d_groups.as<int64_t>();
  eps::facet_eval_kernel<<<static_cast<unsigned>((nl + 127) / 128), 128, 0, ix->stream>>>(a);
  EPS_CUDA(cudaGetLastError());
  eps::facet_group_kernel<<<static_cast<unsigned>((nq * 32 + 127) / 128), 128, 0, ix->stream>>>(a);
  EPS_CUDA(cudaGetLastError());
  EPS_CUDA(cudaMemcpyAsync(out_keys, d_okeys.p, nl * 8, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaMemcpyAsync(out_values, d_ovals.p, nl * 8 * n_aggs, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaMemcpyAsync(out_groups, d_groups.p, static_cast<size_t>(nq) * 8, cudaMemcpyDeviceToHost, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  return EPS_OK;
}
