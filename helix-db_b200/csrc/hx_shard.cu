// hx_shard.cu — the sharded path behind the C ABI (SURVEY §8e; north_star: "shards by id-range across the 8 GPUs of one
// box with a single NCCL all-gather of per-shard top-k over NVLink on the sharded path only").
//
// One rank per device: each rank owns an hx_index holding a contiguous id range (its own vectors, its own HNSW graph or
// just the rows for the exhaustive paths).  Every rank answers every query on its shard, the per-shard top-k BLOCKS —
// ids | scores | counts, written by the search kernels straight into the send block — cross NVLink in ONE ncclAllGather,
// and every rank selects the k smallest by (score, id) from the gathered blocks with the merge kernel (no pack / unpack
// passes).  The (score, id) rule is the reference's Candidate order (model.rs:41-61), so the merged answer of exact
// per-shard scans is independent of the number of shards.  No exchange inside the traversal; n_shards == 1 never touches
// NCCL.  The reference itself has no distributed vector search: this row exists because the north_star names it.
//
// NCCL is resolved at run time (dlopen of libnccl.so.2: the copy PyTorch already loaded in a torch process, the system
// one in a Rust host), so libhelix_b200.so carries no link-time dependency on it.
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstring>

#include "hx_index.hpp"
#include "k_util.cuh"

struct HxNccl {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
};

static HxNccl* hx_nccl() {
  static HxNccl api;
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  if (api.lib) return &api;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) {
    hx_set_error("NCCL is not available (dlopen libnccl.so.2: %s)", dlerror());
    return nullptr;
  }
  api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(h, "ncclGetUniqueId");
  api.CommInitRank = (decltype(api.CommInitRank))dlsym(h, "ncclCommInitRank");
  api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
  api.AllGather = (decltype(api.AllGather))dlsym(h, "ncclAllGather");
  api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
  api.GetVersion = (decltype(api.GetVersion))dlsym(h, "ncclGetVersion");
  if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllGather || !api.GetErrorString) {
    hx_set_error("libnccl.so.2 lacks a required symbol");
    dlclose(h);
    return nullptr;
  }
  api.lib = h;
  return &api;
}

#define HX_NCCL(call)                                                                     \
  do {                                                                                    \
    ncclResult_t _r = (call);                                                             \
    if (_r != ncclSuccess) {                                                              \
      hx_set_error("%s failed: %s", #call, nccl->GetErrorString(_r));                     \
      return HX_ERR_CUDA;                                                                 \
    }                                                                                     \
  } while (0)

struct hx_shard_group {
  hx_index* ix = nullptr;
  uint32_t n_shards = 1, rank = 0;
  ncclComm_t comm = nullptr;
  HxScratch scr;                 // dense path + restricted path scratch, timing events
  DevBuf<uint8_t> send, recv;    // per-rank block / gathered blocks
  DevBuf<float> d_q;             // host-buffer entry points
  DevBuf<uint64_t> d_cand;
  DevBuf<uint32_t> d_slots;
  DevBuf<uint64_t> o_ids;
  DevBuf<float> o_sc;
  DevBuf<uint32_t> o_cnt;
  cudaStream_t stream = nullptr; // host-buffer entry points
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, evc0 = nullptr, evc1 = nullptr, evk0 = nullptr, evk1 = nullptr;
  bool kernel_timed = false;
  std::mutex mu;                 // one sharded call at a time per group (a collective is an ordered operation)
  float last_local_ms = 0.f, last_collective_ms = 0.f;
};

static inline size_t al8(size_t x) { return (x + 7) & ~(size_t)7; }

extern "C" hx_status hx_shard_unique_id(uint8_t* out, size_t cap) {
  if (!out || cap < sizeof(ncclUniqueId)) {
    hx_set_error("hx_shard_unique_id: %zu bytes are required", sizeof(ncclUniqueId));
    return HX_ERR_INVALID_PARAMETER;
  }
  HxNccl* nccl = hx_nccl();
  if (!nccl) return HX_ERR_UNSUPPORTED;
  ncclUniqueId id;
  HX_NCCL(nccl->GetUniqueId(&id));
  memcpy(out, &id, sizeof(id));
  return HX_OK;
}

extern "C" hx_status hx_shard_group_create(hx_index* shard, uint32_t n_shards, uint32_t rank, const uint8_t* unique_id,
                                           hx_shard_group** out) {
  if (!shard) {
    hx_set_error("null index handle");
    return HX_ERR_INDEX_NOT_FOUND;
  }
  if (!out || n_shards == 0 || n_shards > 128 || rank >= n_shards || (n_shards > 1 && !unique_id)) {
    hx_set_error("hx_shard_group_create: 1 <= n_shards <= 128, rank < n_shards, a unique id for n_shards > 1");
    return HX_ERR_INVALID_PARAMETER;
  }
  *out = nullptr;
  HX_CUDA(cudaSetDevice(shard->device));
  hx_shard_group* g = new hx_shard_group();
  g->ix = shard;
  g->n_shards = n_shards;
  g->rank = rank;
  cudaError_t e = cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreate(&g->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&g->ev1);
  if (e == cudaSuccess) e = cudaEventCreate(&g->evc0);
  if (e == cudaSuccess) e = cudaEventCreate(&g->evc1);
  if (e == cudaSuccess) e = cudaEventCreate(&g->evk0);
  if (e == cudaSuccess) e = cudaEventCreate(&g->evk1);
  if (e != cudaSuccess) {
    hx_set_error("shard group creation failed: %s", cudaGetErrorString(e));
    delete g;
    return HX_ERR_CUDA;
  }
  if (n_shards > 1) {
    HxNccl* nccl = hx_nccl();
    if (!nccl) {
      delete g;
      return HX_ERR_UNSUPPORTED;
    }
    ncclUniqueId id;
    memcpy(&id, unique_id, sizeof(id));
    ncclResult_t r = nccl->CommInitRank(&g->comm, (int)n_shards, id, (int)rank);   // collective: every rank calls it
    if (r != ncclSuccess) {
      hx_set_error("ncclCommInitRank failed: %s", nccl->GetErrorString(r));
      delete g;
      return HX_ERR_CUDA;
    }
  }
  *out = g;
  return HX_OK;
}

extern "C" void hx_shard_group_destroy(hx_shard_group* g) {
  if (!g) return;
  cudaSetDevice(g->ix->device);
  cudaDeviceSynchronize();
  if (g->comm) {
    HxNccl* nccl = hx_nccl();
    if (nccl) nccl->CommDestroy(g->comm);
  }
  g->send.release(); g->recv.release(); g->d_q.release(); g->d_cand.release(); g->d_slots.release();
  g->o_ids.release(); g->o_sc.release(); g->o_cnt.release();
  g->scr.destroy();
  if (g->stream) cudaStreamDestroy(g->stream);
  for (cudaEvent_t ev : {g->ev0, g->ev1, g->evc0, g->evc1, g->evk0, g->evk1})
    if (ev) cudaEventDestroy(ev);
  delete g;
}

struct HxBlock {   // one rank's block of per-shard results for B queries, k_loc entries each
  size_t off_sc, off_cnt, bytes;
};
static HxBlock block_layout(size_t B, uint32_t k_loc) {
  HxBlock b;
  b.off_sc = al8(B * (size_t)k_loc * 8);
  b.off_cnt = b.off_sc + al8(B * (size_t)k_loc * 4);
  b.bytes = b.off_cnt + al8(B * 4);
  return b;
}

// gather + merge of a filled send block (stream-ordered)
static hx_status gather_and_merge(hx_shard_group* g, size_t B, uint32_t k_loc, uint32_t k_out, uint64_t* d_out_ids,
                                  float* d_out_scores, uint32_t* d_out_counts, cudaStream_t stream) {
  const HxBlock bl = block_layout(B, k_loc);
  const unsigned char* base = g->send.p;
  size_t stride = 0;
  HX_CUDA(cudaEventRecord(g->evc0, stream));
  if (g->n_shards > 1) {
    HxNccl* nccl = hx_nccl();
    if (!nccl) return HX_ERR_UNSUPPORTED;
    HX_NCCL(nccl->AllGather(g->send.p, g->recv.p, bl.bytes, ncclUint8, g->comm, stream));
    base = g->recv.p;
    stride = bl.bytes;
  }
  k_merge_topk<<<(unsigned)((B + 7) / 8), 256, 0, stream>>>(base, base + bl.off_sc, base + bl.off_cnt, stride, stride, stride,
                                                           g->n_shards, B, k_loc, k_out, d_out_ids, d_out_scores, d_out_counts);
  HX_CUDA(cudaGetLastError());
  HX_CUDA(cudaEventRecord(g->evc1, stream));
  return HX_OK;
}

static hx_status reserve_blocks(hx_shard_group* g, size_t B, uint32_t k_loc) {
  const HxBlock bl = block_layout(B, k_loc);
  hx_status rc;
  if ((rc = g->send.reserve(bl.bytes))) return rc;
  if (g->n_shards > 1 && (rc = g->recv.reserve(bl.bytes * g->n_shards))) return rc;
  return HX_OK;
}

static hx_status sharded_device_locked(hx_shard_group* g, int32_t path, const float* d_queries, size_t B,
                                       const hx_search_params* local, uint32_t k_out, uint64_t* d_out_ids,
                                       float* d_out_scores, uint32_t* d_out_counts, cudaStream_t stream) {
  if (!local || local->k == 0 || k_out == 0) {
    hx_set_error("result count must be non-zero");
    return HX_ERR_INVALID_PARAMETER;
  }
  if (B == 0) return HX_OK;
  if (!d_queries || !d_out_ids || !d_out_scores || !d_out_counts) return HX_ERR_INVALID_PARAMETER;
  HX_CUDA(cudaSetDevice(g->ix->device));
  const uint32_t k_loc = local->k;
  hx_status rc = reserve_blocks(g, B, k_loc);
  if (rc) return rc;
  const HxBlock bl = block_layout(B, k_loc);
  uint64_t* s_ids = reinterpret_cast<uint64_t*>(g->send.p);
  float* s_sc = reinterpret_cast<float*>(g->send.p + bl.off_sc);
  uint32_t* s_cnt = reinterpret_cast<uint32_t*>(g->send.p + bl.off_cnt);
  HX_CUDA(cudaEventRecord(g->ev0, stream));
  if (path == HX_SHARD_DENSE) {
    if ((rc = hx_dense_device(g->ix, &g->scr, d_queries, B, local, s_ids, s_sc, s_cnt, stream, g->evk0, g->evk1)))
      return rc;
    g->kernel_timed = true;
  } else if (path == HX_SHARD_HNSW) {
    if ((rc = hx_search_device(g->ix, d_queries, B, local, s_ids, s_sc, s_cnt, stream, nullptr))) return rc;
  } else {
    hx_set_error("unknown sharded path %d", path);
    return HX_ERR_INVALID_PARAMETER;
  }
  HX_CUDA(cudaEventRecord(g->ev1, stream));
  return gather_and_merge(g, B, k_loc, k_out, d_out_ids, d_out_scores, d_out_counts, stream);
}

extern "C" hx_status hx_search_sharded_device(hx_shard_group* g, int32_t path, const float* d_queries, size_t B,
                                              const hx_search_params* local, uint32_t k_out, uint64_t* d_out_ids,
                                              float* d_out_scores, uint32_t* d_out_counts, void* cuda_stream) {
  if (!g) {
    hx_set_error("null shard group");
    return HX_ERR_INDEX_NOT_FOUND;
  }
  std::lock_guard<std::mutex> lk(g->mu);
  return sharded_device_locked(g, path, d_queries, B, local, k_out, d_out_ids, d_out_scores, d_out_counts,
                               (cudaStream_t)cuda_stream);
}

static hx_status download(hx_shard_group* g, size_t B, uint32_t k_out, uint64_t* out_ids, float* out_scores,
                          uint32_t* out_counts) {
  HX_CUDA(cudaMemcpyAsync(out_ids, g->o_ids.p, B * (size_t)k_out * 8, cudaMemcpyDeviceToHost, g->stream));
  HX_CUDA(cudaMemcpyAsync(out_scores, g->o_sc.p, B * (size_t)k_out * 4, cudaMemcpyDeviceToHost, g->stream));
  HX_CUDA(cudaMemcpyAsync(out_counts, g->o_cnt.p, B * 4, cudaMemcpyDeviceToHost, g->stream));
  HX_CUDA(cudaStreamSynchronize(g->stream));
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, g->ev0, g->ev1) == cudaSuccess) g->last_local_ms = ms;
  if (cudaEventElapsedTime(&ms, g->evc0, g->evc1) == cudaSuccess) g->last_collective_ms = ms;
  if (g->kernel_timed && cudaEventElapsedTime(&ms, g->evk0, g->evk1) == cudaSuccess) {   // k_dense_scores alone
    g->ix->last_kernel_ms = ms;
    g->ix->last_kernel_launches = 1;
  }
  g->kernel_timed = false;
  return HX_OK;
}

extern "C" hx_status hx_search_sharded(hx_shard_group* g, int32_t path, const float* queries, size_t B,
                                       const hx_search_params* local, uint32_t k_out, uint64_t* out_ids, float* out_scores,
                                       uint32_t* out_counts) {
  if (!g) {
    hx_set_error("null shard group");
    return HX_ERR_INDEX_NOT_FOUND;
  }
  if (B == 0) return HX_OK;
  if (!queries || !out_ids || !out_scores || !out_counts || k_out == 0) return HX_ERR_INVALID_PARAMETER;
  std::lock_guard<std::mutex> lk(g->mu);
  HX_CUDA(cudaSetDevice(g->ix->device));
  const uint32_t dim = g->ix->cfg.dimension;
  hx_status rc;
  if ((rc = g->d_q.reserve(B * (size_t)dim)) || (rc = g->o_ids.reserve(B * (size_t)k_out)) ||
      (rc = g->o_sc.reserve(B * (size_t)k_out)) || (rc = g->o_cnt.reserve(B)))
    return rc;
  HX_CUDA(cudaMemcpyAsync(g->d_q.p, queries, B * (size_t)dim * 4, cudaMemcpyHostToDevice, g->stream));
  if ((rc = sharded_device_locked(g, path, g->d_q.p, B, local, k_out, g->o_ids.p, g->o_sc.p, g->o_cnt.p, g->stream)))
    return rc;
  if ((rc = download(g, B, k_out, out_ids, out_scores, out_counts))) return rc;
  // the local search's device flags (tie / visited overflow, invalid score) and, for the dense path, query validation
  if (path == HX_SHARD_HNSW) {
    uint32_t flags = 0;
    hx_status st = HX_OK;
    if ((rc = hx_device_flags(g->ix, g->stream, &flags, &st))) return rc;
    if (st) return st;
  }
  return HX_OK;
}

// Restricted search across shards: every rank passes the SAME ascending candidate list; a shard scores the slice that
// falls into its id range (an empty slice is RestrictedVectorCandidates::Empty for that shard: zero results), then the
// same gather + merge.  Exact, so the answer does not depend on the number of shards.
extern "C" hx_status hx_search_restricted_sharded(hx_shard_group* g, const float* queries, size_t B,
                                                  const hx_search_params* p, const uint64_t* cand_ids, size_t n_cand,
                                                  uint64_t* out_ids, float* out_scores, uint32_t* out_counts) {
  if (!g) {
    hx_set_error("null shard group");
    return HX_ERR_INDEX_NOT_FOUND;
  }
  if (!p || p->k == 0) {
    hx_set_error("result count must be non-zero");
    return HX_ERR_INVALID_PARAMETER;
  }
  if (B == 0) return HX_OK;
  if (!queries || !out_ids || !out_scores || !out_counts || (n_cand && !cand_ids)) return HX_ERR_INVALID_PARAMETER;
  if (n_cand > 1000000ull) {
    hx_set_error("restricted vector search accepts at most 1000000 unique candidates");
    return HX_ERR_QUERY;
  }
  if (std::min<uint64_t>(p->k, n_cand) > 800) {
    hx_set_error("restricted vector search result count must be at most 800");
    return HX_ERR_QUERY;
  }
  for (size_t i = 1; i < n_cand; ++i)
    if (cand_ids[i] <= cand_ids[i - 1]) {
      hx_set_error("candidate ids must be ascending and unique (RoaringTreemap iteration order)");
      return HX_ERR_INVALID_PARAMETER;
    }
  std::lock_guard<std::mutex> lk(g->mu);
  hx_index* ix = g->ix;
  HX_CUDA(cudaSetDevice(ix->device));
  const uint32_t dim = ix->cfg.dimension, k = p->k;
  // this shard's slice of the candidate list
  size_t i0 = 0, i1 = 0;
  if (ix->n) {
    const uint64_t lo = ix->ids_sorted.front(), hi = ix->ids_sorted.back();
    i0 = (size_t)(std::lower_bound(cand_ids, cand_ids + n_cand, lo) - cand_ids);
    i1 = (size_t)(std::upper_bound(cand_ids, cand_ids + n_cand, hi) - cand_ids);
  }
  const size_t mine = i1 - i0;
  hx_status rc;
  if ((rc = reserve_blocks(g, B, k))) return rc;
  if ((rc = g->d_q.reserve(B * (size_t)dim)) || (rc = g->o_ids.reserve(B * (size_t)k)) || (rc = g->o_sc.reserve(B * (size_t)k)) ||
      (rc = g->o_cnt.reserve(B)) || (rc = g->d_cand.reserve(std::max<size_t>(mine, 1))) ||
      (rc = g->d_slots.reserve(std::max<size_t>(mine, 1))))
    return rc;
  const HxBlock bl = block_layout(B, k);
  uint64_t* s_ids = reinterpret_cast<uint64_t*>(g->send.p);
  float* s_sc = reinterpret_cast<float*>(g->send.p + bl.off_sc);
  uint32_t* s_cnt = reinterpret_cast<uint32_t*>(g->send.p + bl.off_cnt);
  HX_CUDA(cudaMemcpyAsync(g->d_q.p, queries, B * (size_t)dim * 4, cudaMemcpyHostToDevice, g->stream));
  HX_CUDA(cudaEventRecord(g->ev0, g->stream));
  if (mine) {
    HX_CUDA(cudaMemcpyAsync(g->d_cand.p, cand_ids + i0, mine * 8, cudaMemcpyHostToDevice, g->stream));
    if ((rc = hx_map_candidates_device(ix, g->d_cand.p, mine, g->d_slots.p, nullptr, g->stream))) return rc;
    if ((rc = hx_search_restricted_device(ix, g->d_q.p, B, p, g->d_slots.p, nullptr, mine, mine, s_ids, s_sc, s_cnt, g->stream)))
      return rc;
  } else {
    HX_CUDA(cudaMemsetAsync(s_cnt, 0, B * 4, g->stream));
  }
  HX_CUDA(cudaEventRecord(g->ev1, g->stream));
  if ((rc = gather_and_merge(g, B, k, k, g->o_ids.p, g->o_sc.p, g->o_cnt.p, g->stream))) return rc;
  return download(g, B, k, out_ids, out_scores, out_counts);
}

extern "C" hx_status hx_shard_group_last_ms(hx_shard_group* g, float* local_ms, float* collective_ms) {
  if (!g) return HX_ERR_INDEX_NOT_FOUND;
  if (local_ms) *local_ms = g->last_local_ms;
  if (collective_ms) *collective_ms = g->last_collective_ms;
  return HX_OK;
}
