// Row-sharded search across GPUs (SURVEY.md §8e): the exchange step lives INSIDE the library so that a C++ host
// (the reference engine with the drop-in) can shard a table that exceeds one GPU's HBM.
//
// One process (or thread) per GPU holds one shard: rows [base, base + n) with its own graph over LOCAL ids.  The
// query batch is replicated; every rank searches its shard, converts the ids to GLOBAL ids, packs (ids | distances)
// into one block, and ONE ncclAllGather of nq*k*12 bytes per rank brings all blocks to every rank, where a k-way merge
// kernel keeps the best k by (distance, id) — exact as long as every shard returns its own top-k.  The single-segment
// reference has the same two-source merge between graph and tail results (vec_search_executor.cpp:885-900).
// Everything is enqueued on the index's stream: no host synchronisation between the search, the collective and the
// merge.
//
// NCCL is bound at run time (dlopen "libnccl.so.2"): a process that already carries NCCL (PyTorch) shares that copy,
// a plain C++ host gets the system one, and libepsilla_b200.so itself has no link-time dependency on it.
#include <dlfcn.h>

#include <cstring>
#include <mutex>

#include "internal.h"

namespace eps {

namespace {

struct NcclUid { char internal[128]; };  // ncclUniqueId (nccl.h: NCCL_UNIQUE_ID_BYTES = 128)
typedef void* NcclComm;
typedef int (*FnGetUniqueId)(NcclUid*);
typedef int (*FnCommInitRank)(NcclComm*, int, NcclUid, int);
typedef int (*FnCommDestroy)(NcclComm);
typedef int (*FnAllGather)(const void*, void*, size_t, int /*ncclDataType_t*/, NcclComm, cudaStream_t);
typedef const char* (*FnGetErrorString)(int);
constexpr int kNcclInt8 = 0;  // ncclDataType_t ncclInt8 / ncclChar

struct NcclApi {
  void* handle = nullptr;
  FnGetUniqueId get_unique_id = nullptr;
  FnCommInitRank comm_init_rank = nullptr;
  FnCommDestroy comm_destroy = nullptr;
  FnAllGather all_gather = nullptr;
  FnGetErrorString error_string = nullptr;
  std::string why;
};

NcclApi* nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (api.handle) break;
    }
    if (!api.handle) { api.why = std::string("dlopen(libnccl.so.2) failed: ") + dlerror(); return; }
    api.get_unique_id = reinterpret_cast<FnGetUniqueId>(dlsym(api.handle, "ncclGetUniqueId"));
    api.comm_init_rank = reinterpret_cast<FnCommInitRank>(dlsym(api.handle, "ncclCommInitRank"));
    api.comm_destroy = reinterpret_cast<FnCommDestroy>(dlsym(api.handle, "ncclCommDestroy"));
    api.all_gather = reinterpret_cast<FnAllGather>(dlsym(api.handle, "ncclAllGather"));
    api.error_string = reinterpret_cast<FnGetErrorString>(dlsym(api.handle, "ncclGetErrorString"));
    if (!api.get_unique_id || !api.comm_init_rank || !api.comm_destroy || !api.all_gather) {
      api.why = "libnccl.so.2 lacks a required symbol";
      api.handle = nullptr;
    }
  });
  return &api;
}

int nccl_fail(const NcclApi* api, int rc, const char* what) {
  return fail(EPS_ERR_CUDA, std::string(what) + ": " + (api->error_string ? api->error_string(rc) : "NCCL error") + " (" +
                                std::to_string(rc) + ")");
}

}  // namespace

struct ShardGroup {
  int rank = 0, world = 1, device = 0;
  NcclComm comm = nullptr;
  DevBuf send, recv;
};

// local ids -> global ids (empty slots stay -1), packed as [ids int64 x nk | dists float x nk], 16-byte aligned parts
__global__ void pack_shard_block_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dists, int64_t nk, int64_t base,
                                        int64_t* __restrict__ out_ids, float* __restrict__ out_dists) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= nk) return;
  const int64_t id = ids[i];
  out_ids[i] = id >= 0 ? id + base : -1;
  out_dists[i] = dists[i];
}

}  // namespace eps

using eps::Index;
using eps::ShardGroup;

extern "C" {

int eps_shard_unique_id(void* out128) {
  if (!out128) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null unique-id buffer");
  eps::NcclApi* api = eps::nccl_api();
  if (!api->handle) return eps::fail(EPS_ERR_UNSUPPORTED, "NCCL unavailable: " + api->why);
  eps::NcclUid id;
  const int rc = api->get_unique_id(&id);
  if (rc != 0) return eps::nccl_fail(api, rc, "ncclGetUniqueId");
  std::memcpy(out128, &id, sizeof(id));
  return EPS_OK;
}

int eps_shard_group_create(eps_shard_group** out, const void* unique_id128, int rank, int world, int device) {
  if (!out) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "out is null");
  *out = nullptr;
  if (!unique_id128 || world < 1 || rank < 0 || rank >= world) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "bad rank / world / id");
  eps::NcclApi* api = eps::nccl_api();
  if (!api->handle) return eps::fail(EPS_ERR_UNSUPPORTED, "NCCL unavailable: " + api->why);
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) return eps::fail(EPS_ERR_NO_DEVICE, "no usable CUDA device");
  if (device < 0 || device >= n) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "device ordinal out of range");
  EPS_CUDA(cudaSetDevice(device));
  ShardGroup* g = new ShardGroup();
  g->rank = rank; g->world = world; g->device = device;
  eps::NcclUid id;
  std::memcpy(&id, unique_id128, sizeof(id));
  const int rc = api->comm_init_rank(&g->comm, world, id, rank);
  if (rc != 0) { delete g; return eps::nccl_fail(api, rc, "ncclCommInitRank"); }
  *out = reinterpret_cast<eps_shard_group*>(g);
  return EPS_OK;
}

void eps_shard_group_destroy(eps_shard_group* h) {
  if (!h) return;
  ShardGroup* g = reinterpret_cast<ShardGroup*>(h);
  cudaSetDevice(g->device);
  if (g->comm) eps::nccl_api()->comm_destroy(g->comm);
  delete g;
}

int eps_search_batch_sharded(eps_shard_group* gh, eps_index* h, int64_t id_base, const float* d_queries, int64_t nq, int64_t k,
                             const eps_filter_node* filter, int64_t n_filter, int64_t* d_out_ids, float* d_out_dists,
                             eps_stats* stats, int sync) {
  ShardGroup* g = reinterpret_cast<ShardGroup*>(gh);
  Index* ix = reinterpret_cast<Index*>(h);
  if (!g || !ix || !d_queries || !d_out_ids || !d_out_dists) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "null argument");
  if (ix->sparse) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "sharded search of a sparse index is not supported");
  if (nq <= 0) return EPS_OK;
  if (k < 1) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "k must be >= 1");
  if (ix->device != g->device) return eps::fail(EPS_ERR_INVALID_ARGUMENT, "index and shard group live on different devices");
  eps::NcclApi* api = eps::nccl_api();
  const int64_t nk = nq * k;
  const size_t ids_bytes = (static_cast<size_t>(nk) * 8 + 15) & ~size_t(15), dist_bytes = (static_cast<size_t>(nk) * 4 + 15) & ~size_t(15);
  const size_t block = ids_bytes + dist_bytes;
  // local search into scratch owned by the index (ids | counts | dists), asynchronous on the index stream
  EPS_TRY(ix->s_out_ids.reserve(static_cast<size_t>(nk) * 8));
  EPS_TRY(ix->s_out_dists.reserve(static_cast<size_t>(nk) * 4));
  EPS_TRY(ix->s_out_counts.reserve(static_cast<size_t>(nq) * 8));
  EPS_TRY(g->send.reserve(block));
  EPS_TRY(g->recv.reserve(block * static_cast<size_t>(g->world)));
  int rc = eps_search_batch_device(h, d_queries, nq, k, filter, n_filter, ix->s_out_ids.as<int64_t>(), ix->s_out_dists.as<float>(),
                                   ix->s_out_counts.as<int64_t>(), stats, 0);
  if (rc != EPS_OK) return rc;
  unsigned char* sb = g->send.as<unsigned char>();
  eps::pack_shard_block_kernel<<<static_cast<unsigned>((nk + 255) / 256), 256, 0, ix->stream>>>(
      ix->s_out_ids.as<int64_t>(), ix->s_out_dists.as<float>(), nk, id_base, reinterpret_cast<int64_t*>(sb),
      reinterpret_cast<float*>(sb + ids_bytes));
  EPS_CUDA(cudaGetLastError());
  const int nrc = api->all_gather(sb, g->recv.p, block, eps::kNcclInt8, g->comm, ix->stream);
  if (nrc != 0) return eps::nccl_fail(api, nrc, "ncclAllGather");
  const unsigned char* rb = g->recv.as<unsigned char>();
  EPS_TRY(eps::merge_shards(g->device, ix->stream, reinterpret_cast<const int64_t*>(rb), reinterpret_cast<const float*>(rb + ids_bytes),
                            g->world, nq, k, d_out_ids, d_out_dists, static_cast<int64_t>(block / 8), static_cast<int64_t>(block / 4)));
  if (stats) stats->kernel_launches += 3;
  if (sync) EPS_CUDA(cudaStreamSynchronize(ix->stream));
  return EPS_OK;
}

}  // extern "C"
