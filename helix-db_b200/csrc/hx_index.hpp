// hx_index.hpp — host-side state of one device-resident index shard (opaque `hx_index` of the C ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <condition_variable>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/helix_b200.h"
#include "hx_common.cuh"

// thread-local error text (hx_last_error)
void hx_set_error(const char* fmt, ...);
void hx_set_error_index(uint32_t idx);

#define HX_CUDA(call)                                                                              \
  do {                                                                                             \
    cudaError_t _e = (call);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      hx_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__);    \
      return _e == cudaErrorMemoryAllocation ? HX_ERR_OUT_OF_MEMORY : HX_ERR_CUDA;                 \
    }                                                                                              \
  } while (0)

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;   // elements
  hx_status reserve(size_t n) {
    if (n <= cap) return HX_OK;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = n + n / 4 + 16;
    cudaError_t e = cudaMalloc((void**)&p, want * sizeof(T));
    if (e != cudaSuccess) {
      hx_set_error("cudaMalloc(%zu bytes) failed: %s", want * sizeof(T), cudaGetErrorString(e));
      return HX_ERR_OUT_OF_MEMORY;
    }
    cap = want;
    return HX_OK;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

template <typename T>
struct PinBuf {
  T* p = nullptr;
  size_t cap = 0;
  hx_status reserve(size_t n) {
    if (n <= cap) return HX_OK;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    size_t want = n + n / 4 + 16;
    cudaError_t e = cudaMallocHost((void**)&p, want * sizeof(T));
    if (e != cudaSuccess) {
      hx_set_error("cudaMallocHost(%zu bytes) failed: %s", want * sizeof(T), cudaGetErrorString(e));
      return HX_ERR_OUT_OF_MEMORY;
    }
    cap = want;
    return HX_OK;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
};

// dense path state cached across calls on one scratch set: encoded tensor maps, the shape they were built for
struct HxDenseCache {
  alignas(64) unsigned char map_q[128];
  alignas(64) unsigned char map_x[128];
  size_t B = 0;
  uint32_t kprime = 0, ldb = 0;
  const void* map_x_base = nullptr;
  size_t map_x_rows = 0;
};

// One scratch set per in-flight host call (the handle is Send+Sync like the reference's index:
// concurrent searches each take a private stream + buffers; SURVEY §8b "Threading").
struct HxScratch {
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;   // host->device query chunks of the pipelined hx_search (created on first use)
  cudaEvent_t ev_copy = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  DevBuf<float> d_queries, d_qhdr, d_out_scores;
  DevBuf<uint32_t> d_qstatus, d_out_counts, d_qstats, d_err, d_cand_slots;
  DevBuf<uint64_t> d_out_ids, d_cand_ids, d_cand_offsets, d_keys;
  DevBuf<uint32_t> d_vtab, d_vpool, d_vbusy;   // ring build: visited hash sets, overflow pool, pool busy flags
  uint32_t vpool_n = 0xffffffffu, vpool_cap = 0;
  DevBuf<uint64_t> d_tiepool;                  // overflow regions of the tie stack (HxRingArgs::tie_pool)
  DevBuf<uint32_t> d_tiebusy;
  bool tiepool_init = false;
  DevBuf<uint64_t> d_partial;                  // fused scan + top-k: per-CTA lists
  DevBuf<uint32_t> d_tickets;                  // ... and the per-query CTA tickets (self-resetting)
  size_t tickets_zeroed = 0;
  // filtered (ACORN) walk: per-CTA stamp arrays [grid][n] + epochs, bridge frontiers, eligible lists, candidate bitmap, seeds
  DevBuf<uint32_t> d_fg_stamps, d_fg_epochs, d_fg_elig, d_fg_bits, d_fg_seed;
  DevBuf<uint64_t> d_fg_bridge;
  size_t fg_stamp_rows = 0;
  uint32_t fg_stamp_grid = 0;
  DevBuf<uint32_t> d_qerr;                     // per-query error flags
  PinBuf<uint32_t> h_qerr;
  DevBuf<unsigned long long> d_prof;   // HX_PHASE_PROF diagnostics
  DevBuf<unsigned long long> d_pstats; // policy counters
  DevBuf<uint64_t> d_qsim;             // query fingerprints
  bool prof_init = false;
  DevBuf<uint8_t> misc[16];   // dense path buffers (kept across calls)
  HxDenseCache dense;
  // exact dense entries: certificate flags + compaction + the view word, how, and the gathered rescan queries and results
  DevBuf<uint32_t> x_flag, x_status, x_counts;
  DevBuf<uint8_t> x_how;
  DevBuf<float> x_queries, x_hdr, x_scores;
  DevBuf<uint64_t> x_ids;
  PinBuf<uint32_t> h_x;
  DevBuf<uint8_t> d_block;    // small calls: results packed into one block -> one device-to-host copy
  PinBuf<uint8_t> h_block;
  PinBuf<uint64_t> h_ids, h_cand_offsets;
  PinBuf<float> h_scores, h_queries, h_qhdr;
  PinBuf<uint32_t> h_counts, h_qstats, h_status, h_err, h_avail;
  bool busy = false;
  // ring of event pairs for the device-buffer path (timed without host synchronisation)
  std::vector<cudaEvent_t> ring0, ring1;
  size_t ring_pos = 0, ring_pending = 0;
  hx_status ring_next(cudaEvent_t* e0, cudaEvent_t* e1);
  void destroy();
};

struct HxLayerRows {   // host staging of one mirrored HNSW layer (slot space)
  std::vector<uint32_t> node;      // slot owning the row
  std::vector<uint32_t> offsets;   // CSR into nbr
  std::vector<uint32_t> nbr;       // neighbour slots (ascending); neighbours without a vector removed
  std::vector<uint32_t> raw_len;   // row length as stored by the reference (for neighbors_examined)
};

struct hx_index {
  hx_index_config cfg{};
  hx_tuning tune{};   // launch-shape knobs: environment at hx_index_create, hx_index_set_tuning afterwards
  int device = 0;
  int sm_count = 132;
  uint32_t lim0 = 32;   // MutationDegreeLimits.layer0 = max(m0, 2m)  (mutation.rs:179-199)
  // vectors
  size_t n = 0;
  uint32_t ld = 0;
  std::vector<uint64_t> ids_sorted;   // host copy: slot -> id
  bool contiguous = false;
  uint64_t first_id = 0;
  uint64_t vector_generation = 0;     // bumped whenever the slot numbering changes (hx_candidates are tied to it)
  // incremental maintenance (hx_mirror.inl): allocated capacity of the per-row / upper-row arrays (0 = exactly n / rows),
  // tombstones of deleted nodes
  size_t cap_rows = 0, cap_upper = 0;
  uint8_t* d_deleted = nullptr;
  std::vector<uint8_t> host_deleted;
  size_t n_deleted = 0;
  std::atomic<uint64_t> mirror_patches{0};
  float* d_vec = nullptr;
  float* d_hdr = nullptr;
  uint64_t* d_ids = nullptr;
  // graph (device)
  uint32_t* d_nbr0 = nullptr;
  uint16_t* d_deg0 = nullptr;
  uint16_t* d_raw0 = nullptr;
  uint32_t* d_upper_off = nullptr;
  uint32_t* d_upper_nbr = nullptr;
  uint16_t* d_upper_deg = nullptr;
  uint8_t* d_level = nullptr;
  uint32_t stride0 = 0, stride_u = 0;
  size_t n_upper_rows = 0;
  // graph (host staging until finalize)
  std::vector<HxLayerRows> staged;   // index = layer
  std::atomic<bool> graph_dirty{false};   // set by the load calls, cleared by hx_finalize_graph (under fin_mu)
  std::mutex fin_mu;
  bool populated = false;
  uint64_t entry_id = 0;
  uint32_t entry_slot = 0;
  int max_layer = 0;
  // SimHash policy state (production-default search mode)
  hx_simhash_config simcfg{43u, 0.8f, 1u, 0.1f};
  uint64_t* d_simhash = nullptr;       // [n] slot order
  uint8_t* d_has_simhash = nullptr;    // [n]
  float* d_planes_t = nullptr;         // [dim][64] (transposed for coalesced projection)
  size_t simhash_count = 0;
  // dense path state (k_dense.cu), built on first use after every mirror write and published under dense_mu only once
  // complete: the ascending slots of the live (not deleted) rows, and the bf16 copy of those rows compacted in that order
  std::mutex dense_mu;
  uint32_t* d_live_slots = nullptr;
  size_t n_live = 0;
  void* d_vec_bf16 = nullptr;
  float* d_sqnorm = nullptr;
  // row contents: bumped wherever the whole-corpus bf16 copy is dropped and wherever vector_generation moves, so a resident
  // candidate view (HxResident) knows that its gathered tile no longer holds the rows' current values
  std::atomic<uint64_t> content_epoch{0};
  // scratch pool
  std::mutex mu;
  std::condition_variable cv;
  std::vector<HxScratch*> pool;
  // device-buffer calls are ordered by the caller's stream: one scratch set PER STREAM (calls on different streams may
  // run concurrently and must not share the error word, the query counter or the visited tables)
  std::map<cudaStream_t, HxScratch*> dev_scratch;
  HxScratch* last_dev_scratch = nullptr;   // the stream hx_last_kernel_ms reports (most recent device-buffer call)
  // last dominant-kernel timing
  std::atomic<float> last_kernel_ms{0.f};
  std::atomic<uint32_t> last_kernel_launches{0};
  // mirror version (SURVEY §8b snapshot semantics): the host stamps the (generation, visible sequence) the image was
  // hydrated at; the Rust guard (read_index.rs:53-65) compares it with the request's snapshot before dispatching here
  std::atomic<uint64_t> mirror_generation{0}, mirror_visible_seq{0};

  HxDev dev() const;
  void free_vectors();
  void free_graph();
};

#define HX_SCRATCH_POOL_MAX 64   // concurrent host-buffer calls per handle before a caller has to wait
hx_status hx_acquire_scratch(hx_index* ix, HxScratch** out);
void hx_release_scratch(hx_index* ix, HxScratch* s);
hx_status hx_finalize_graph(hx_index* ix);

// CTA-per-query ring build (k_hnsw_ring.cuh): launch configuration shared by hx_search's small-batch path and hx_service
struct HxCtaRingCfg {
  uint32_t qch, warps, RC, vt_cap, fr_cap, ef;
  size_t smem;
};
struct HxHnswArgs;
struct HxRingArgs;
bool hx_cta_ring_config(const hx_index* ix, uint32_t ef, uint32_t want_warps, uint32_t want_rc, uint32_t want_vt_log2,
                        size_t budget, HxCtaRingCfg* c);
hx_status hx_launch_cta_ring(hx_index* ix, const HxCtaRingCfg& c, const HxHnswArgs& a, const HxRingArgs& rg, uint32_t grid,
                             cudaStream_t stream, int* ctas_per_sm);
bool hx_slot_of(const hx_index* ix, uint64_t id, uint32_t* slot);

// The certificate of the exact dense entries (k_dense.cu: k_dense_certify), left on the call's stream for the rescan
struct HxDenseCert {
  bool small = false;                   // the view is below hx_dense_min_rows(k): the exact scan answered every query
  const uint32_t* flagged = nullptr;    // [B] the indices of the queries the certificate could not clear, ascending
  const uint32_t* n_flagged = nullptr;  // device word: how many
  const uint8_t* how = nullptr;         // [B] 0 certified, 1 flagged
};

// implemented in k_build.cu / k_dense.cu
hx_status hx_build_impl(hx_index* ix, const uint16_t* levels, uint64_t seed, int sequential);
// exact = false: hx_search_dense; true: hx_search_dense_exact (out_how may be null)
hx_status hx_dense_impl(hx_index* ix, const float* queries, size_t B, const hx_search_params* p, uint64_t* out_ids,
                        float* out_scores, uint32_t* out_counts, hx_stats* stats, bool exact = false,
                        uint8_t* out_how = nullptr);
// cert != null: the certificate runs after the re-rank (or cert->small is set)
hx_status hx_dense_device(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, const hx_search_params* p,
                          uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt, cudaStream_t stream,
                          cudaEvent_t e0, cudaEvent_t e1, uint32_t* launches_out, HxDenseCert* cert = nullptr);
// hx_api.cu: the exact scan of the flagged queries over the view's ascending slot list, results scattered into the output
// rows.  Synchronises the stream once to read the flagged count; *err_before receives the device error word as it was
// before the scan reset it.
hx_status hx_dense_rescan(hx_index* ix, HxScratch* s, const float* d_q, uint32_t k, const uint32_t* slots,
                          size_t n_view, const HxDenseCert& cert, uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt,
                          cudaStream_t stream, cudaEvent_t e0, cudaEvent_t e1, uint32_t* launches, size_t* n_flagged,
                          uint32_t* err_before);
// rows below which the dense paths answer with the exact scan (the tensor-core pass could not fill its nominee lists)
size_t hx_dense_min_rows(uint32_t k);
hx_status hx_dense_compact(hx_index* ix, HxScratch* scr, const uint32_t* d_slots, size_t n, cudaStream_t stream,
                           const uint32_t** d_present, size_t* n_present, uint32_t* launches);
hx_status hx_dense_restricted_device(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, uint32_t k,
                                     const uint32_t* d_present, size_t n_present, uint64_t* d_out_ids, float* d_out_sc,
                                     uint32_t* d_out_cnt, cudaStream_t stream, cudaEvent_t e0, cudaEvent_t e1,
                                     uint32_t* launches, HxDenseCert* cert = nullptr);

// The resident tensor-core view of a device candidate set (hx_candidates_make_resident): what
// hx_search_dense_restricted_set otherwise rebuilds on every call, built once and kept by the set.  The present list never
// changes while the set is valid (deletes and reloads move vector_generation, which refuses the set; upserts do not touch
// the set's slots), so only the row values can go stale: `epoch` is the index's content_epoch the tile was gathered at.
struct HxResident {
  std::mutex mu;                     // held by a refresh; a new epoch is published under it once the tile is complete
  std::atomic<uint64_t> epoch{0};
  cudaStream_t stream = nullptr;     // builds and refreshes run here, never on a caller's stream
  uint32_t* slots = nullptr;         // [n] the set's present slots, ascending (hx_dense_compact)
  size_t n = 0;
  void* rows = nullptr;              // [n rounded up to 256][ldb] bf16, tile placement over candidate rank (k_to_bf16)
  float* aux = nullptr;              // row terms by position, then (at the end) k_dense_view_bound's word
  uint32_t* word = nullptr;
  uint64_t bytes = 0;                // device memory held
};
// hx_candidates_make_resident: compaction of the set's slot list, gather, view word; blocking.  *out is set on success.
hx_status hx_resident_build(hx_index* ix, const uint32_t* d_slots, size_t n_slots, HxResident** out);
// the first call after a row write re-gathers the tile and the view word in place (same present list); otherwise nothing
hx_status hx_resident_current(hx_index* ix, HxResident* r);
void hx_resident_free(HxResident* r);
// hx_dense_restricted_device over a resident view (r.n >= hx_dense_min_rows(k)): no compaction, no gather, and the
// certificate reads the view word the view holds
hx_status hx_dense_resident_device(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, uint32_t k, const HxResident& r,
                                   uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt, cudaStream_t stream,
                                   cudaEvent_t e0, cudaEvent_t e1, uint32_t* launches, HxDenseCert* cert = nullptr);
