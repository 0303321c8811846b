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

// Tile shape of the dense path (k_dense.cu) that its host code sizes buffers by
#define HXD_BN 256          // corpus rows per placement tile (the unit of the row interleave and of the column quarters)
#define HXD_BK 64           // bf16 elements per k-block = 128 bytes = one swizzle atom
// bf16 elements per row of a dense view or query tile: dim rounded up to a whole k-block
inline uint32_t hx_dense_ldb(uint32_t dim) { return (dim + HXD_BK - 1) / HXD_BK * HXD_BK; }
// rows of a dense view rounded up to a whole placement tile
inline size_t hx_dense_rows_pad(size_t n) { return (n + HXD_BN - 1) / HXD_BN * HXD_BN; }

// Dense path buffers of one scratch set, kept across calls
struct HxDenseScratch {
  // the tensor-core pass (k_dense.cu: dense_pass); each sized with 256 bytes of slack
  DevBuf<uint16_t> q_tile;          // [B_pad][ldb] the queries in bf16
  DevBuf<float> q_aux;              // [B_pad] their query terms
  DevBuf<uint64_t> bucket_keys;     // [B][n_split][HXD_PARTS][HXD_T] k_dense_scores' buckets
  DevBuf<uint64_t> sel_ids;         // [B][k'] the nominees ...
  DevBuf<float> sel_sc;             // ... their approximate scores
  DevBuf<uint32_t> sel_cnt;         // ... and how many per query
  DevBuf<uint32_t> nominee_slots;   // [B][k'] ascending corpus slots of the nominees
  DevBuf<uint64_t> nominee_offs;    // [B + 1] b * k'
  DevBuf<uint64_t> rerank_keys;     // [B][k'] the exact re-rank's keys
  // q_tile's pad rows and columns, q_aux's pad entries, nominee_offs and map_q are written once per (these three
  // buffers, B, k', ldb) and re-initialised when any of them changes
  const void* init_q_tile = nullptr;
  const void* init_q_aux = nullptr;
  const void* init_offs = nullptr;
  size_t init_B = 0;
  uint32_t init_kprime = 0, init_ldb = 0;
  alignas(64) unsigned char map_q[128];
  alignas(64) unsigned char map_x[128];   // keyed on the view's (rows, padded row count)
  const void* map_x_base = nullptr;
  size_t map_x_rows = 0;
  // a candidate view gathered per call (hx_dense_gather): the compacted present slots, the bf16 tile, its row terms
  DevBuf<uint32_t> present, present_counts;
  DevBuf<uint16_t> view_rows;
  DevBuf<float> view_aux;
  // the certificate (dense_certify): per-query flags, their compaction, the view word, how
  DevBuf<uint32_t> flag, flagged, flag_counts, view_word;
  DevBuf<uint8_t> how;
  // the rescan of the flagged queries (hx_dense.inl): gathered queries, headers, status words, their answers
  DevBuf<float> rescan_q, rescan_hdr, rescan_sc;
  DevBuf<uint32_t> rescan_status, rescan_cnt;
  DevBuf<uint64_t> rescan_ids;
  PinBuf<uint32_t> h_rescan;        // the flagged count and the error word before the rescan
  void release() {
    q_tile.release(); q_aux.release(); bucket_keys.release(); sel_ids.release(); sel_sc.release(); sel_cnt.release();
    nominee_slots.release(); nominee_offs.release(); rerank_keys.release();
    init_q_tile = init_q_aux = init_offs = nullptr;
    map_x_base = nullptr;
    present.release(); present_counts.release(); view_rows.release(); view_aux.release();
    flag.release(); flagged.release(); flag_counts.release(); view_word.release(); how.release();
    rescan_q.release(); rescan_hdr.release(); rescan_sc.release(); rescan_status.release(); rescan_cnt.release();
    rescan_ids.release(); h_rescan.release();
  }
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
  HxDenseScratch dense;
  DevBuf<uint8_t> d_block;   // small calls: results packed into one block -> one device-to-host copy
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

// implemented in k_build.cu
hx_status hx_build_impl(hx_index* ix, const uint16_t* levels, uint64_t seed, int sequential);

// ---- the dense path: k_dense.cu (kernels, views, pass, certificate), hx_dense.inl (entry points) ----
// The corpus a tensor-core pass runs over: `n` bf16 rows in tile placement (k_to_bf16 with tiled = 1), their row terms
// (indexed by position), and the ascending slot table that maps row w of the view to its corpus slot.  `word`: the view's
// k_dense_view_bound word when the view holds one (null: the certificate reduces it per call).
struct HxDenseView {
  const void* rows = nullptr;
  const float* aux = nullptr;
  const uint32_t* slots = nullptr;
  size_t n = 0;
  const uint32_t* word = nullptr;
};

// The certificate of the exact dense entries (k_dense_certify), left on the call's stream for the rescan
struct HxDenseCert {
  const uint32_t* flagged = nullptr;    // [B] the indices of the queries the certificate could not clear, ascending
  const uint32_t* n_flagged = nullptr;  // device word: how many
  const uint8_t* how = nullptr;         // [B] 0 certified, 1 flagged
};

// rows below which the dense paths answer with the exact scan (the tensor-core pass could not fill its nominee lists)
size_t hx_dense_min_rows(uint32_t k);
// The whole-corpus view: the ascending live slots and, when `rows`, the bf16 copy of the live rows.  Built on first use
// after every mirror write (blocking on `stream`) and published under ix->dense_mu only once complete.
hx_status hx_dense_corpus_view(hx_index* ix, bool rows, cudaStream_t stream, HxDenseView* v);
// A per-call view over the ascending slot list `d_slots` (n entries, HX_ABSENT for ids without a row and deleted rows): the
// present slots compacted in order (one synchronisation reads their count) and, when there are at least
// hx_dense_min_rows(k), their rows gathered into a bf16 tile of the scratch set (v->rows stays null otherwise).
hx_status hx_dense_gather(hx_index* ix, HxScratch* scr, const uint32_t* d_slots, size_t n, uint32_t k, cudaStream_t stream,
                          HxDenseView* v, uint32_t* launches);
// The tensor-core pass over a view (v.n >= hx_dense_min_rows(k), k <= 800) and the exact re-rank, then (cert != null)
// the certificate.  The queries' exact headers and status words must be in scr->d_qhdr / d_qstatus.  Enqueued on `stream`,
// no synchronisation; adds the launches it issues to *launches.
hx_status hx_dense_search(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, uint32_t k, const HxDenseView& v,
                          uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt, cudaStream_t stream, cudaEvent_t e0,
                          cudaEvent_t e1, uint32_t* launches, HxDenseCert* cert = nullptr);
// hx_search_dense over every live row on device buffers (the sharded path): everything on `stream`, no synchronisation
// once the whole-corpus view exists
hx_status hx_dense_device(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, const hx_search_params* p,
                          uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt, cudaStream_t stream,
                          cudaEvent_t e0, cudaEvent_t e1);

// The resident tensor-core view of a device candidate set (hx_candidates_make_resident): what
// hx_search_dense_restricted_set otherwise rebuilds on every call, built once and kept by the set.  The present list never
// changes while the set is valid (deletes and reloads move vector_generation, which refuses the set; upserts do not touch
// the set's slots), so only the row values can go stale: `epoch` is the index's content_epoch the tile was gathered at.
struct HxResident {
  std::mutex mu;                     // held by a refresh; a new epoch is published under it once the tile is complete
  std::atomic<uint64_t> epoch{0};
  cudaStream_t stream = nullptr;     // builds and refreshes run here, never on a caller's stream
  uint32_t* slots = nullptr;         // [n] the set's present slots, ascending
  size_t n = 0;
  void* rows = nullptr;              // [n rounded up to 256][ldb] bf16, tile placement over candidate rank (k_to_bf16)
  float* aux = nullptr;              // row terms by position, then (at the end) k_dense_view_bound's word
  uint32_t* word = nullptr;
  uint64_t bytes = 0;                // device memory held
  HxDenseView view() const { return HxDenseView{rows, aux, slots, n, word}; }
};
// hx_candidates_make_resident: compaction of the set's slot list, gather, view word; blocking.  *out is set on success.
hx_status hx_resident_build(hx_index* ix, const uint32_t* d_slots, size_t n_slots, HxResident** out);
// the first call after a row write re-gathers the tile and the view word in place (same present list); otherwise nothing
hx_status hx_resident_current(hx_index* ix, HxResident* r);
void hx_resident_free(HxResident* r);
