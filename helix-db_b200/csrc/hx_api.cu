// hx_api.cu — C ABI of libhelix_b200 (include/helix_b200.h): index mirror management and the
// search entry points that stand in for VectorIndex::search / search_restricted
// (crates/db/src/search/vector/index.rs:1578-1587, restricted.rs:466-613).
//
// There is deliberately NO CPU fallback in this file: every search runs the CUDA kernels or fails.
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <numeric>

#include "hx_index.hpp"
#include "k_hnsw.cuh"
#include "k_hnsw_ring.cuh"
#include "k_hnsw_policy.cuh"
#include "k_scan.cuh"
#include "k_filtered.cuh"
#include "k_util.cuh"

// ------------------------------------------------------------------------------------------------
// diagnostics
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static thread_local uint32_t g_err_index = 0;

void hx_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void hx_set_error_index(uint32_t idx) { g_err_index = idx; }

extern "C" const char* hx_last_error(void) { return g_err; }
extern "C" uint32_t hx_last_error_index(void) { return g_err_index; }
extern "C" const char* hx_version(void) { return "helix_b200 0.1 (sm_90a)"; }

// ------------------------------------------------------------------------------------------------
// helpers
// ------------------------------------------------------------------------------------------------
static inline uint32_t round_up(uint32_t x, uint32_t m) { return (x + m - 1) / m * m; }

// VectorComponentLimit::try_new (domain.rs:24-79)
static bool component_limit(int metric, uint32_t dim, float* limit) {
  if (metric == HX_METRIC_COSINE) return false;
  const double factor = metric == HX_METRIC_EUCLIDEAN ? 8.0 : 4.0;
  const double divisor = (double)dim * factor;
  const double exact =
      metric == HX_METRIC_EUCLIDEAN ? std::sqrt((double)FLT_MAX / divisor) : (double)FLT_MAX / divisor;
  float rounded = (float)exact;
  if ((double)rounded > exact) {
    uint32_t bits;
    memcpy(&bits, &rounded, 4);
    bits -= 1;
    memcpy(&rounded, &bits, 4);
  }
  *limit = rounded;
  return true;
}

// scaled_l2_norm / norm_no_header on the host (cosine.rs:12-36,120-122) for the small-batch path.
static float host_cosine_norm(const float* v, uint32_t d) {
  double scale = 0.0, scaled_sum = 1.0;
  for (uint32_t i = 0; i < d; ++i) {
    double magnitude = (double)std::fabs(v[i]);
    if (magnitude == 0.0) continue;
    if (scale < magnitude) {
      double ratio = scale / magnitude;
      double t = scaled_sum * ratio;
      t = t * ratio;
      scaled_sum = 1.0 + t;
      scale = magnitude;
    } else {
      double ratio = magnitude / scale;
      double t = ratio * ratio;
      scaled_sum = scaled_sum + t;
    }
  }
  double n = scale == 0.0 ? 0.0 : scale * std::sqrt(scaled_sum);
  if (n > (double)FLT_MAX) n = (double)FLT_MAX;
  return (float)n;
}

// ValidatedMetricVector::try_new on the host; returns status word like k_validate_and_header
static uint32_t host_validate(const float* v, uint32_t dim, int metric, bool has_limit, float limit) {
  for (uint32_t i = 0; i < dim; ++i)
    if (!std::isfinite(v[i])) return (HX_ST_COMPONENT << 24) | (i & 0xffffffu);
  if (metric == HX_METRIC_COSINE) {
    bool nz = false;
    for (uint32_t i = 0; i < dim; ++i)
      if (!(v[i] == 0.0f)) { nz = true; break; }
    if (!nz) return HX_ST_ZERO_NORM << 24;
  }
  if (has_limit)
    for (uint32_t i = 0; i < dim; ++i)
      if (std::fabs(v[i]) > limit) return (HX_ST_MAGNITUDE << 24) | (i & 0xffffffu);
  return HX_ST_OK;
}

static hx_status status_from_word(uint32_t w, size_t which, const char* what);

// Empty / unpopulated index: the reference validates the query first (search.rs:1101-1128, restricted.rs:539-566) and only
// then answers Ok(vec![]).  No device work: every query is validated on the host.
static hx_status answer_empty_index(const hx_index* ix, const float* queries, size_t B, uint32_t* out_counts,
                                    hx_status* out_status) {
  float limit = 0.f;
  const uint32_t dim = ix->cfg.dimension;
  const bool has_limit = component_limit(ix->cfg.metric, dim, &limit);
  for (size_t b = 0; b < B; ++b) {
    const uint32_t w = host_validate(queries + b * (size_t)dim, dim, ix->cfg.metric, has_limit, limit);
    const hx_status st = w == 0u ? HX_OK : status_from_word(w, b, "query");
    out_counts[b] = 0;
    if (out_status) out_status[b] = st;
    else if (st) return st;
  }
  return HX_OK;
}

static hx_status status_from_word(uint32_t w, size_t which, const char* what) {
  const uint32_t code = w >> 24, idx = w & 0xffffffu;
  hx_set_error_index(idx);
  switch (code) {
    case HX_ST_COMPONENT:
      hx_set_error("%s %zu: component %u is not finite", what, which, idx);
      return HX_ERR_INVALID_VECTOR_COMPONENT;
    case HX_ST_ZERO_NORM:
      hx_set_error("%s %zu: zero-norm vector under the cosine metric", what, which);
      return HX_ERR_ZERO_NORM_COSINE;
    case HX_ST_MAGNITUDE:
      hx_set_error("%s %zu: component %u exceeds the metric magnitude limit", what, which, idx);
      return HX_ERR_MAGNITUDE_EXCEEDED;
    default:
      return HX_OK;
  }
}

HxDev hx_index::dev() const {
  HxDev d{};
  d.vec = d_vec;
  d.hdr = d_hdr;
  d.ids = d_ids;
  d.nbr0 = d_nbr0;
  d.deg0 = d_deg0;
  d.raw0 = d_raw0;
  d.upper_off = d_upper_off;
  d.upper_nbr = d_upper_nbr;
  d.upper_deg = d_upper_deg;
  d.level = d_level;
  d.n = (uint32_t)n;
  d.dim = cfg.dimension;
  d.ld = ld;
  d.stride0 = stride0;
  d.stride_u = stride_u;
  d.metric = cfg.metric;
  d.entry_slot = entry_slot;
  d.max_layer = max_layer;
  d.populated = populated ? 1 : 0;
  return d;
}

void hx_index::free_vectors() {
  if (d_vec) cudaFree(d_vec);
  if (d_hdr) cudaFree(d_hdr);
  if (d_ids) cudaFree(d_ids);
  if (d_vec_bf16) cudaFree(d_vec_bf16);
  if (d_sqnorm) cudaFree(d_sqnorm);
  if (d_simhash) cudaFree(d_simhash);
  if (d_has_simhash) cudaFree(d_has_simhash);
  d_simhash = nullptr; d_has_simhash = nullptr; simhash_count = 0;
  if (d_live_slots) cudaFree(d_live_slots);
  d_vec = nullptr; d_hdr = nullptr; d_ids = nullptr; d_vec_bf16 = nullptr; d_sqnorm = nullptr; d_live_slots = nullptr;
  n_live = 0;
  if (d_deleted) cudaFree(d_deleted);
  d_deleted = nullptr;
  host_deleted.clear();
  n_deleted = 0;
  cap_rows = 0;
  n = 0;
  ids_sorted.clear();
}

void hx_index::free_graph() {
  if (d_nbr0) cudaFree(d_nbr0);
  if (d_deg0) cudaFree(d_deg0);
  if (d_raw0) cudaFree(d_raw0);
  if (d_upper_off) cudaFree(d_upper_off);
  if (d_upper_nbr) cudaFree(d_upper_nbr);
  if (d_upper_deg) cudaFree(d_upper_deg);
  if (d_level) cudaFree(d_level);
  d_nbr0 = nullptr; d_deg0 = nullptr; d_raw0 = nullptr; d_upper_off = nullptr;
  d_upper_nbr = nullptr; d_upper_deg = nullptr; d_level = nullptr;
  stride0 = 0; stride_u = 0; n_upper_rows = 0;
  cap_upper = 0;
  staged.clear();
  populated = false;
  // graph_dirty is NOT touched here: hx_finalize_graph calls this while it holds fin_mu with the flag still set — clearing
  // it would let a concurrent search skip the lock and launch on a half-uploaded graph.  Callers that really reset the
  // graph clear the flag themselves.
}

hx_status HxScratch::ring_next(cudaEvent_t* e0, cudaEvent_t* e1) {
  const size_t cap = 512;
  if (ring0.size() < cap) {
    cudaEvent_t a, b;
    HX_CUDA(cudaEventCreate(&a));
    HX_CUDA(cudaEventCreate(&b));
    ring0.push_back(a);
    ring1.push_back(b);
    *e0 = a;
    *e1 = b;
    ring_pos = ring0.size() % cap;
  } else {
    *e0 = ring0[ring_pos];
    *e1 = ring1[ring_pos];
    ring_pos = (ring_pos + 1) % cap;
  }
  if (ring_pending < cap) ring_pending++;
  return HX_OK;
}

void HxScratch::destroy() {
  for (cudaEvent_t e : ring0) cudaEventDestroy(e);
  for (cudaEvent_t e : ring1) cudaEventDestroy(e);
  ring0.clear();
  ring1.clear();
  if (stream) cudaStreamDestroy(stream);
  if (copy_stream) cudaStreamDestroy(copy_stream);
  if (ev_copy) cudaEventDestroy(ev_copy);
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  d_queries.release(); d_qhdr.release(); d_out_scores.release();
  d_qstatus.release(); d_out_counts.release(); d_qstats.release(); d_err.release();
  d_cand_slots.release(); d_out_ids.release(); d_cand_ids.release(); d_cand_offsets.release(); d_keys.release();
  d_tiepool.release(); d_tiebusy.release(); d_qerr.release(); h_qerr.release(); d_partial.release(); d_tickets.release();
  d_fg_stamps.release(); d_fg_epochs.release(); d_fg_bridge.release(); d_fg_elig.release(); d_fg_bits.release(); d_fg_seed.release();
  d_vtab.release(); d_vpool.release(); d_vbusy.release(); d_prof.release(); d_pstats.release(); d_qsim.release();
  for (auto& m : misc) m.release();
  x_flag.release(); x_status.release(); x_counts.release(); x_how.release(); x_queries.release(); x_hdr.release();
  x_scores.release(); x_ids.release(); h_x.release();
  h_ids.release(); h_cand_offsets.release(); h_scores.release(); h_queries.release(); h_qhdr.release();
  h_counts.release(); h_qstats.release(); h_status.release(); h_err.release(); h_avail.release();
  d_block.release(); h_block.release();
}

hx_status hx_acquire_scratch(hx_index* ix, HxScratch** out) {
  std::unique_lock<std::mutex> lk(ix->mu);
  for (;;) {
    for (HxScratch* s : ix->pool)
      if (!s->busy) {
        s->busy = true;
        *out = s;
        return HX_OK;
      }
    if (ix->pool.size() < HX_SCRATCH_POOL_MAX) {
      HxScratch* s = new HxScratch();
      cudaError_t e = cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking);
      if (e == cudaSuccess) e = cudaEventCreate(&s->ev0);
      if (e == cudaSuccess) e = cudaEventCreate(&s->ev1);
      if (e != cudaSuccess) {
        hx_set_error("scratch creation failed: %s", cudaGetErrorString(e));
        s->destroy();
        delete s;
        return HX_ERR_CUDA;
      }
      s->busy = true;
      ix->pool.push_back(s);
      *out = s;
      return HX_OK;
    }
    ix->cv.wait(lk);
  }
}

void hx_release_scratch(hx_index* ix, HxScratch* s) {
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    s->busy = false;
  }
  ix->cv.notify_one();
}

// Device-buffer calls are ordered by the caller's stream: one dedicated scratch set per stream, so calls issued on
// different streams (from different threads) never share the error word, the query counter or the visited tables.
static hx_status dev_scratch(hx_index* ix, cudaStream_t stream, HxScratch** out) {
  std::lock_guard<std::mutex> lk(ix->mu);
  HxScratch*& s = ix->dev_scratch[stream];
  if (!s) s = new HxScratch();
  ix->last_dev_scratch = s;
  *out = s;
  return HX_OK;
}

struct ScratchGuard {
  hx_index* ix;
  HxScratch* s;
  ~ScratchGuard() {
    if (s) hx_release_scratch(ix, s);
  }
};

bool hx_slot_of(const hx_index* ix, uint64_t id, uint32_t* slot) {
  if (ix->n == 0) return false;
  uint32_t s;
  if (ix->contiguous) {
    if (id < ix->first_id || id - ix->first_id >= ix->n) return false;
    s = (uint32_t)(id - ix->first_id);
  } else {
    auto it = std::lower_bound(ix->ids_sorted.begin(), ix->ids_sorted.end(), id);
    if (it == ix->ids_sorted.end() || *it != id) return false;
    s = (uint32_t)(it - ix->ids_sorted.begin());
  }
  if (!ix->host_deleted.empty() && ix->host_deleted[s]) return false;   // deleted by hx_index_delete_vectors
  *slot = s;
  return true;
}

// ------------------------------------------------------------------------------------------------
// launch-shape knobs (hx_tuning): seeded from the environment ONCE per handle, never read on the search path
// ------------------------------------------------------------------------------------------------
static int32_t env_knob(const char* name, long lo, long hi) {
  const char* e = getenv(name);
  if (!e || !*e) return -1;
  const long v = atol(e);
  return v >= lo && v <= hi ? (int32_t)v : -1;
}
static void tuning_from_env(hx_tuning* t) {
  t->ring_warps = env_knob("HX_RING_WARPS", 1, 16);
  t->ring_rows = env_knob("HX_RING_R", 1, 32);
  t->visited_log2 = env_knob("HX_VT_CAP_LOG2", 6, 24);
  t->visited_pool = env_knob("HX_VT_POOL", 0, 1024);
  t->l2_hint = env_knob("HX_L2_HINT", 0, 1);
  t->prefetch_below = env_knob("HX_PREFETCH_BELOW", 0, 1 << 20);
  t->lat_warps = env_knob("HX_LAT_WARPS", 1, 12);
  const char* adm = getenv("HX_LAT_ADMIT");
  t->lat_admit_seq = adm ? (strcmp(adm, "seq") == 0 ? 1 : 0) : -1;
  t->lat_spec = env_knob("HX_LAT_SPEC", 0, 1);
  t->phase_prof = env_knob("HX_PHASE_PROF", 0, 1);
  t->pipeline = env_knob("HX_PIPELINE", 0, 1);
  t->scan_fused = env_knob("HX_SCAN_FUSED", 0, 1);
  t->pol_warps = env_knob("HX_POL_WARPS", 1, 16);
  t->pol_min_rows = env_knob("HX_POL_MINR", 1, 32);
  t->pol_cta = env_knob("HX_POL_CTA", 0, 1);
  t->pol_early_sim = env_knob("HX_POL_EARLY_SIM", 0, 1);
  t->build_max_batch = env_knob("HX_BUILD_MAX_BATCH", 1, 65536);
}
static inline uint32_t knob(int32_t v, uint32_t dflt) { return v < 0 ? dflt : (uint32_t)v; }

extern "C" hx_status hx_index_get_tuning(const hx_index* ix, hx_tuning* out) {
  if (!ix || !out) {
    hx_set_error("hx_index_get_tuning: null argument");
    return HX_ERR_INVALID_PARAMETER;
  }
  *out = ix->tune;
  return HX_OK;
}
extern "C" hx_status hx_index_set_tuning(hx_index* ix, const hx_tuning* t) {
  if (!ix) {
    hx_set_error("hx_index_set_tuning: null handle");
    return HX_ERR_INVALID_PARAMETER;
  }
  if (t) ix->tune = *t;
  else tuning_from_env(&ix->tune);   // NULL: back to the environment's values
  return HX_OK;
}

// ------------------------------------------------------------------------------------------------
// lifecycle
// ------------------------------------------------------------------------------------------------
extern "C" hx_status hx_index_create(const hx_index_config* cfg, hx_index** out) {
  if (!cfg || !out) {
    hx_set_error("hx_index_create: null argument");
    return HX_ERR_INVALID_PARAMETER;
  }
  *out = nullptr;
  if (cfg->dimension == 0 || cfg->m == 0 || cfg->metric < 0 || cfg->metric > 2) {
    hx_set_error("invalid vector index config: dimension=%u m=%u metric=%d", cfg->dimension, cfg->m, cfg->metric);
    return HX_ERR_INVALID_VECTOR_CONFIG;
  }
  // Layer0Connections / ConstructionBeamWidth (parameters.rs:54-100, config/indexes.rs:413-417): both must cover m
  if (cfg->m0 < cfg->m || cfg->ef_construction < cfg->m) {
    hx_set_error("invalid vector index config: m0=%u and ef_construction=%u must be at least m=%u", cfg->m0,
                 cfg->ef_construction, cfg->m);
    return HX_ERR_INVALID_VECTOR_CONFIG;
  }
  if (cfg->dimension > 65536) {
    hx_set_error("dimension %u above the supported maximum 65536", cfg->dimension);
    return HX_ERR_INVALID_VECTOR_CONFIG;
  }
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    hx_set_error("no CUDA device available (%s): libhelix_b200 has no CPU fallback", cudaGetErrorString(e));
    return HX_ERR_CUDA;
  }
  if (cfg->device < 0 || cfg->device >= ndev) {
    hx_set_error("device ordinal %d out of range (%d devices)", cfg->device, ndev);
    return HX_ERR_INVALID_PARAMETER;
  }
  HX_CUDA(cudaSetDevice(cfg->device));
  hx_index* ix = new hx_index();
  ix->cfg = *cfg;
  ix->device = cfg->device;
  tuning_from_env(&ix->tune);
  ix->lim0 = std::max(cfg->m0, 2 * cfg->m);
  ix->ld = round_up(cfg->dimension, 32);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, cfg->device) == cudaSuccess) ix->sm_count = prop.multiProcessorCount;
  *out = ix;
  return HX_OK;
}

extern "C" void hx_index_destroy(hx_index* ix) {
  if (!ix) return;
  cudaSetDevice(ix->device);
  cudaDeviceSynchronize();
  for (HxScratch* s : ix->pool) {
    s->destroy();
    delete s;
  }
  for (auto& kv : ix->dev_scratch) {
    kv.second->destroy();
    delete kv.second;
  }
  ix->dev_scratch.clear();
  ix->free_graph();
  ix->free_vectors();
  if (ix->d_planes_t) cudaFree(ix->d_planes_t);
  delete ix;
}

static hx_status alloc_vectors(hx_index* ix, size_t n) {
  ix->free_graph();
  ix->graph_dirty.store(false, std::memory_order_release);   // no staged rows, no device graph: nothing to finalise
  ix->free_vectors();
  if (n >= (1ull << 31)) {
    hx_set_error("a shard holds at most 2^31-1 rows (got %zu)", n);
    return HX_ERR_INVALID_PARAMETER;
  }
  if (n == 0) return HX_OK;
  HX_CUDA(cudaMalloc((void**)&ix->d_vec, n * (size_t)ix->ld * sizeof(float)));
  HX_CUDA(cudaMalloc((void**)&ix->d_hdr, n * sizeof(float)));
  HX_CUDA(cudaMalloc((void**)&ix->d_ids, n * sizeof(uint64_t)));
  ix->n = n;
  ix->vector_generation++;
  ix->content_epoch.fetch_add(1, std::memory_order_release);
  return HX_OK;
}

// validate rows on the device like decode_item_borrowed (mod.rs:889-949) and compute row headers
static hx_status validate_rows_device(hx_index* ix) {
  const size_t n = ix->n;
  uint32_t* d_status = nullptr;
  HX_CUDA(cudaMalloc((void**)&d_status, n * sizeof(uint32_t)));
  float limit = 0.f;
  const bool has_limit = component_limit(ix->cfg.metric, ix->cfg.dimension, &limit);
  const size_t threads = 256, warps_per_block = threads / 32;
  const size_t blocks = (n + warps_per_block - 1) / warps_per_block;
  k_validate_and_header<<<(unsigned)blocks, (unsigned)threads>>>(ix->d_vec, n, ix->cfg.dimension, ix->ld,
                                                               ix->cfg.metric, limit, has_limit ? 1 : 0, ix->d_hdr,
                                                               d_status);
  cudaError_t e = cudaGetLastError();
  std::vector<uint32_t> st(n);
  if (e == cudaSuccess) e = cudaMemcpy(st.data(), d_status, n * sizeof(uint32_t), cudaMemcpyDeviceToHost);
  cudaFree(d_status);
  if (e != cudaSuccess) {
    hx_set_error("row validation failed: %s", cudaGetErrorString(e));
    return HX_ERR_CUDA;
  }
  for (size_t i = 0; i < n; ++i)
    if (st[i] != HX_ST_OK) return status_from_word(st[i], i, "row (slot)");
  return HX_OK;
}

extern "C" hx_status hx_index_load_vectors(hx_index* ix, const uint64_t* ids, const float* rows, size_t n) {
  if (!ix) {
    hx_set_error("null index handle");
    return HX_ERR_INDEX_NOT_FOUND;
  }
  if (n && (!ids || !rows)) {
    hx_set_error("hx_index_load_vectors: null pointer");
    return HX_ERR_INVALID_PARAMETER;
  }
  HX_CUDA(cudaSetDevice(ix->device));
  hx_status rc = alloc_vectors(ix, n);
  if (rc) return rc;
  if (n == 0) return HX_OK;
  const uint32_t dim = ix->cfg.dimension;
  // slot order = ascending id
  std::vector<uint32_t> order(n);
  std::iota(order.begin(), order.end(), 0u);
  bool sorted = true;
  for (size_t i = 1; i < n; ++i)
    if (ids[i - 1] >= ids[i]) { sorted = false; break; }
  if (!sorted) {
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return ids[a] < ids[b]; });
    for (size_t i = 1; i < n; ++i)
      if (ids[order[i - 1]] == ids[order[i]]) {
        hx_set_error("duplicate node id %llu", (unsigned long long)ids[order[i]]);
        ix->free_vectors();
        return HX_ERR_INVARIANT_VIOLATION;
      }
  }
  ix->ids_sorted.resize(n);
  for (size_t i = 0; i < n; ++i) ix->ids_sorted[i] = ids[order[i]];
  ix->first_id = ix->ids_sorted[0];
  ix->contiguous = (ix->ids_sorted[n - 1] - ix->ids_sorted[0] == (uint64_t)(n - 1));
  HX_CUDA(cudaMemcpy(ix->d_ids, ix->ids_sorted.data(), n * sizeof(uint64_t), cudaMemcpyHostToDevice));
  if (sorted && ix->ld == dim) {
    HX_CUDA(cudaMemcpy(ix->d_vec, rows, n * (size_t)dim * sizeof(float), cudaMemcpyHostToDevice));
  } else if (sorted) {
    HX_CUDA(cudaMemset(ix->d_vec, 0, n * (size_t)ix->ld * sizeof(float)));
    HX_CUDA(cudaMemcpy2D(ix->d_vec, (size_t)ix->ld * sizeof(float), rows, (size_t)dim * sizeof(float),
                         (size_t)dim * sizeof(float), n, cudaMemcpyHostToDevice));
  } else {
    const size_t chunk = std::max<size_t>(1, (64u << 20) / ((size_t)ix->ld * sizeof(float)));
    std::vector<float> stage(chunk * (size_t)ix->ld, 0.f);
    for (size_t b = 0; b < n; b += chunk) {
      const size_t c = std::min(chunk, n - b);
      for (size_t i = 0; i < c; ++i)
        memcpy(stage.data() + i * (size_t)ix->ld, rows + (size_t)order[b + i] * dim, dim * sizeof(float));
      HX_CUDA(cudaMemcpy(ix->d_vec + b * (size_t)ix->ld, stage.data(), c * (size_t)ix->ld * sizeof(float),
                         cudaMemcpyHostToDevice));
    }
  }
  rc = validate_rows_device(ix);
  if (rc) {
    ix->free_vectors();
    return rc;
  }
  return HX_OK;
}

// kind 0: isolated isotropic clusters in full dimension (SURVEY §8d recipe); kind r in 2..64: rank-r latent mixture
static hx_status launch_generator(hx_index* ix, float* d_out, size_t count, size_t ld, uint64_t seed,
                                  uint32_t n_centroids, float sigma, uint64_t first_index, uint64_t tag, uint32_t kind) {
  const uint32_t dim = ix->cfg.dimension;
  if (kind == 0) {
    k_generate_mixture<<<(unsigned)((count + 7) / 8), 256>>>(d_out, count, dim, ld, seed, n_centroids, sigma,
                                                           first_index, tag);
    HX_CUDA(cudaGetLastError());
    return HX_OK;
  }
  if (kind < 2 || kind > 64) {
    hx_set_error("generator kind must be 0 or a latent rank in 2..64");
    return HX_ERR_INVALID_PARAMETER;
  }
  float* d_A = nullptr;
  HX_CUDA(cudaMalloc((void**)&d_A, (size_t)dim * kind * sizeof(float)));
  k_generate_proj<<<(dim * kind + 255) / 256, 256>>>(d_A, dim, kind, seed);
  k_generate_latent<<<(unsigned)((count + 7) / 8), 256>>>(d_out, count, dim, ld, seed, n_centroids, sigma, first_index,
                                                         tag, d_A, kind, 0.02f);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaFree(d_A);
  if (e != cudaSuccess) {
    hx_set_error("generator failed: %s", cudaGetErrorString(e));
    return HX_ERR_CUDA;
  }
  return HX_OK;
}

extern "C" hx_status hx_index_generate_vectors(hx_index* ix, uint64_t first_id, size_t n, uint64_t seed,
                                               uint32_t n_centroids, float sigma, uint32_t kind) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (n_centroids == 0) return HX_ERR_INVALID_PARAMETER;
  HX_CUDA(cudaSetDevice(ix->device));
  hx_status rc = alloc_vectors(ix, n);
  if (rc || n == 0) return rc;
  // the global id (not the slot) keys the generator, so id-range shards reproduce the unsharded corpus
  if ((rc = launch_generator(ix, ix->d_vec, n, ix->ld, seed, n_centroids, sigma, first_id, 0x1111ull, kind))) {
    ix->free_vectors();
    return rc;
  }
  k_iota_ids<<<(unsigned)((n + 255) / 256), 256>>>(ix->d_ids, n, first_id);
  HX_CUDA(cudaGetLastError());
  ix->ids_sorted.resize(n);
  for (size_t i = 0; i < n; ++i) ix->ids_sorted[i] = first_id + i;
  ix->first_id = first_id;
  ix->contiguous = true;
  rc = validate_rows_device(ix);
  if (rc) ix->free_vectors();
  return rc;
}

extern "C" hx_status hx_generate_queries(hx_index* ix, uint64_t seed, uint32_t n_centroids, float sigma,
                                         uint64_t first_query, size_t n_queries, float* out_host, uint32_t kind) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (!out_host || n_centroids == 0) return HX_ERR_INVALID_PARAMETER;
  if (n_queries == 0) return HX_OK;
  HX_CUDA(cudaSetDevice(ix->device));
  float* d = nullptr;
  const uint32_t dim = ix->cfg.dimension;
  HX_CUDA(cudaMalloc((void**)&d, n_queries * (size_t)ix->ld * sizeof(float)));
  hx_status grc = launch_generator(ix, d, n_queries, ix->ld, seed, n_centroids, sigma, first_query, 0x2222ull, kind);
  if (grc) {
    cudaFree(d);
    return grc;
  }
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess)
    e = cudaMemcpy2D(out_host, (size_t)dim * sizeof(float), d, (size_t)ix->ld * sizeof(float),
                     (size_t)dim * sizeof(float), n_queries, cudaMemcpyDeviceToHost);
  cudaFree(d);
  if (e != cudaSuccess) {
    hx_set_error("query generation failed: %s", cudaGetErrorString(e));
    return HX_ERR_CUDA;
  }
  return HX_OK;
}

extern "C" hx_status hx_index_download_vectors(hx_index* ix, size_t first_slot, size_t n, float* out_rows,
                                               uint64_t* out_ids) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (first_slot + n > ix->n) {
    hx_set_error("slot range [%zu,%zu) outside the index (%zu rows)", first_slot, first_slot + n, ix->n);
    return HX_ERR_INVALID_PARAMETER;
  }
  if (n == 0) return HX_OK;
  HX_CUDA(cudaSetDevice(ix->device));
  const uint32_t dim = ix->cfg.dimension;
  if (out_rows)
    HX_CUDA(cudaMemcpy2D(out_rows, (size_t)dim * sizeof(float), ix->d_vec + first_slot * (size_t)ix->ld,
                         (size_t)ix->ld * sizeof(float), (size_t)dim * sizeof(float), n, cudaMemcpyDeviceToHost));
  if (out_ids) memcpy(out_ids, ix->ids_sorted.data() + first_slot, n * sizeof(uint64_t));
  return HX_OK;
}

// ------------------------------------------------------------------------------------------------
// graph mirror
// ------------------------------------------------------------------------------------------------
extern "C" hx_status hx_index_load_graph(hx_index* ix, uint16_t layer, const uint64_t* node_ids,
                                         const uint32_t* offsets, const uint64_t* neighbors, size_t n_nodes) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (n_nodes && (!node_ids || !offsets)) return HX_ERR_INVALID_PARAMETER;
  if (layer > 63) {   // MAX_SELECTED_LAYER (mod.rs:772)
    hx_set_error("layer %u above the maximum 63", layer);
    return HX_ERR_INVALID_PARAMETER;
  }
  if (ix->staged.size() <= layer) ix->staged.resize((size_t)layer + 1);
  HxLayerRows& L = ix->staged[layer];
  L = HxLayerRows();
  L.offsets.push_back(0);
  for (size_t i = 0; i < n_nodes; ++i) {
    uint32_t slot;
    if (!hx_slot_of(ix, node_ids[i], &slot)) continue;   // a row whose owner has no vector is unreachable
    const uint32_t b = offsets[i], e = offsets[i + 1];
    uint32_t kept = 0;
    uint64_t prev = 0;
    for (uint32_t j = b; j < e; ++j) {
      if (j > b && neighbors[j] <= prev) {
        hx_set_error("layer %u row of node %llu is not strictly ascending", layer, (unsigned long long)node_ids[i]);
        return HX_ERR_INVARIANT_VIOLATION;   // canonical rows are ascending & unique (values/vectors.rs:67-110)
      }
      prev = neighbors[j];
      uint32_t ns;
      if (neighbors[j] == node_ids[i]) {
        hx_set_error("layer %u row of node %llu links to itself", layer, (unsigned long long)node_ids[i]);
        return HX_ERR_INVARIANT_VIOLATION;
      }
      if (hx_slot_of(ix, neighbors[j], &ns)) {
        L.nbr.push_back(ns);
        kept++;
      }
    }
    (void)kept;
    L.node.push_back(slot);
    L.offsets.push_back((uint32_t)L.nbr.size());
    L.raw_len.push_back(e - b);
  }
  ix->graph_dirty = true;
  return HX_OK;
}

// ------------------------------------------------------------------------------------------------
// row-image import / export (SURVEY §8(f).2)
// ------------------------------------------------------------------------------------------------
static inline uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
static inline uint64_t be64(const uint8_t* p) { return ((uint64_t)be32(p) << 32) | be32(p + 4); }
static inline void put_be32(uint8_t* p, uint32_t v) { p[0] = v >> 24; p[1] = v >> 16; p[2] = v >> 8; p[3] = v; }
static inline void put_be64(uint8_t* p, uint64_t v) { put_be32(p, (uint32_t)(v >> 32)); put_be32(p + 4, (uint32_t)v); }

extern "C" hx_status hx_decode_neighbor_row(uint16_t layer, const uint8_t* row, size_t len, uint64_t* out_ids, size_t cap,
                                            size_t* out_count, uint64_t* out_simhash, int32_t* out_has_simhash) {
  if (out_count) *out_count = 0;
  if (out_has_simhash) *out_has_simhash = 0;
  if (len && !row) return HX_ERR_INVALID_PARAMETER;
  size_t off = 0, count = 0;
  if (layer == 0) {
    if (len == 0) return HX_OK;   // missing row == the deployed empty-neighbour state (values/vectors.rs:181-183)
    const uint8_t type = row[0];
    if (type == 0x12) {           // ENCODING_TYPE_LAYER0_NEIGHBORS
      if (len < 5) { hx_set_error("layer-0 row too short: %zu bytes", len); return HX_ERR_INVARIANT_VIOLATION; }
      count = be32(row + 1);
      off = 5;
    } else if (type == 0x13) {    // ENCODING_TYPE_LAYER0_RECORD
      if (len < 6) { hx_set_error("layer-0 record too short: %zu bytes", len); return HX_ERR_INVARIANT_VIOLATION; }
      const uint8_t flags = row[1];
      if (flags & ~0x01u) { hx_set_error("invalid layer-0 record flags: %#04x", flags); return HX_ERR_INVARIANT_VIOLATION; }
      count = be32(row + 2);
      off = 6;
      if (flags & 1) {
        if (len < off + 8) { hx_set_error("layer-0 record too short for its SimHash"); return HX_ERR_INVARIANT_VIOLATION; }
        uint64_t bits = 0;
        for (int i = 0; i < 8; ++i) bits |= (uint64_t)row[off + i] << (8 * i);   // little endian
        if (out_simhash) *out_simhash = bits;
        if (out_has_simhash) *out_has_simhash = 1;
        off += 8;
      }
    } else {
      hx_set_error("invalid layer-0 encoding type %#04x", type);
      return HX_ERR_INVARIANT_VIOLATION;
    }
  } else {
    if (len < 4) { hx_set_error("upper-layer row too short: %zu bytes", len); return HX_ERR_INVARIANT_VIOLATION; }
    count = be32(row);
    off = 4;
  }
  if (len != off + count * 8) {
    hx_set_error("neighbour row length %zu does not match its count %zu (expected %zu)", len, count, off + count * 8);
    return HX_ERR_INVARIANT_VIOLATION;
  }
  if (out_count) *out_count = count;
  if (count > cap) {
    hx_set_error("neighbour row holds %zu ids, caller capacity %zu", count, cap);
    return HX_ERR_INVALID_PARAMETER;
  }
  for (size_t i = 0; i < count; ++i) out_ids[i] = be64(row + off + 8 * i);
  return HX_OK;
}

extern "C" hx_status hx_encode_neighbor_row(uint16_t layer, const uint64_t* ids, size_t n, uint8_t* out, size_t cap,
                                            size_t* out_len) {
  if (n && !ids) return HX_ERR_INVALID_PARAMETER;
  // layer 0 canonicalises to sorted unique ids (encode_layer0_neighbors, values/vectors.rs:97-110)
  std::vector<uint64_t> canon(ids, ids + n);
  if (layer == 0) {
    bool sorted = true;
    for (size_t i = 1; i < n; ++i)
      if (!(canon[i - 1] < canon[i])) { sorted = false; break; }
    if (!sorted) {
      std::sort(canon.begin(), canon.end());
      canon.erase(std::unique(canon.begin(), canon.end()), canon.end());
    }
  }
  const size_t hdr = layer == 0 ? 5 : 4, need = hdr + canon.size() * 8;
  if (out_len) *out_len = need;
  if (!out || cap < need) {
    hx_set_error("encoded neighbour row needs %zu bytes, capacity %zu", need, cap);
    return HX_ERR_INVALID_PARAMETER;
  }
  size_t off = 0;
  if (layer == 0) out[off++] = 0x12;
  put_be32(out + off, (uint32_t)canon.size());
  off += 4;
  for (uint64_t id : canon) { put_be64(out + off, id); off += 8; }
  return HX_OK;
}

// ---- row keys (encoding/v1/keys/vectors.rs) -----------------------------------------------------------------------
extern "C" hx_status hx_parse_vector_key(const uint8_t* key, size_t len, hx_vector_key* out) {
  if (!out || (len && !key)) return HX_ERR_INVALID_PARAMETER;
  memset(out, 0, sizeof(*out));
  if (len == 0) { hx_set_error("empty key"); return HX_ERR_INVARIANT_VIOLATION; }
  const uint8_t lane = key[0];
  if (lane == 0x03) {                       // KEY_SPACE_INDEX / INDEX_TYPE_VECTOR: metadata + txn guard (keys/vectors.rs:321-361)
    if (len < 2 || key[1] != 0x03) { hx_set_error("not a vector-index key"); return HX_ERR_INVARIANT_VIOLATION; }
    if (len != 10 && len != 11) { hx_set_error("invalid vector default key length %zu", len); return HX_ERR_INVARIANT_VIOLATION; }
    out->index_id = be64(key + 2);
    if (len == 11) {
      if (key[10] == 0x01) out->kind = HX_KEY_METADATA;
      else if (key[10] != 0x09) { hx_set_error("invalid vector default key kind %#04x", key[10]); return HX_ERR_INVARIANT_VIOLATION; }
    }
    return HX_OK;
  }
  if (lane != 0xF0 && lane != 0xF1) { hx_set_error("invalid key prefix %#04x", lane); return HX_ERR_INVARIANT_VIOLATION; }
  if (len < 9) { hx_set_error("vector key too short: %zu bytes", len); return HX_ERR_INVARIANT_VIOLATION; }
  out->index_id = be64(key + 1);
  if (len == 9) return HX_OK;               // lane prefix key
  const uint8_t kind = key[9];
  const size_t NODE = 18, LAYER_NODE = 20, ORDERED = 26, KINDPFX = 10, REVERSE = 28;
  auto bad_len = [&]() { hx_set_error("invalid vector key length %zu for kind %#04x", len, kind); return HX_ERR_INVARIANT_VIOLATION; };
  if (lane == 0xF0) {                       // vector-hot lane (:363-404)
    switch (kind) {
      case 0x16: if (len != NODE) return bad_len(); out->kind = HX_KEY_LAYER0_NEIGHBORS; out->node_id = be64(key + 10); return HX_OK;
      case 0x11: if (len != LAYER_NODE) return bad_len(); out->kind = HX_KEY_UPPER_NEIGHBORS;
                 out->layer = (uint16_t)((key[10] << 8) | key[11]); out->node_id = be64(key + 12); return HX_OK;
      case 0x12: if (len != NODE) return bad_len(); out->kind = HX_KEY_SIMHASH; out->node_id = be64(key + 10); return HX_OK;
      case 0x13: if (len != NODE) return bad_len(); out->kind = HX_KEY_UPPER_VECTOR; out->node_id = be64(key + 10); return HX_OK;
      default: hx_set_error("invalid vector-hot key kind %#04x", kind); return HX_ERR_INVARIANT_VIOLATION;
    }
  }
  switch (kind) {                           // layer-0 lane (:406-467)
    case 0x02:
      if (len == KINDPFX) return HX_OK;
      if (len != ORDERED) return bad_len();
      out->kind = HX_KEY_VECTOR; out->order_code = be64(key + 10); out->node_id = be64(key + 18); return HX_OK;
    case 0x17: if (len != KINDPFX && len != ORDERED) return bad_len(); return HX_OK;
    case 0x04: if (len != KINDPFX && len != LAYER_NODE) return bad_len(); return HX_OK;
    case 0x05: if (len != NODE) return bad_len(); return HX_OK;
    case 0x15: if (len != NODE && len != REVERSE) return bad_len(); return HX_OK;
    default: hx_set_error("invalid vector-l0 key kind %#04x", kind); return HX_ERR_INVARIANT_VIOLATION;
  }
}

extern "C" hx_status hx_encode_vector_key(const hx_vector_key* k, uint8_t* out, size_t cap, size_t* out_len) {
  if (!k) return HX_ERR_INVALID_PARAMETER;
  size_t need = 0;
  switch (k->kind) {
    case HX_KEY_VECTOR: need = 26; break;
    case HX_KEY_LAYER0_NEIGHBORS: case HX_KEY_SIMHASH: case HX_KEY_UPPER_VECTOR: need = 18; break;
    case HX_KEY_UPPER_NEIGHBORS: need = 20; break;
    case HX_KEY_METADATA: need = 11; break;
    default: hx_set_error("key kind %d cannot be encoded", k->kind); return HX_ERR_INVALID_PARAMETER;
  }
  if (out_len) *out_len = need;
  if (!out || cap < need) { hx_set_error("encoded key needs %zu bytes, capacity %zu", need, cap); return HX_ERR_INVALID_PARAMETER; }
  size_t off = 0;
  if (k->kind == HX_KEY_METADATA) {
    out[off++] = 0x03; out[off++] = 0x03; put_be64(out + off, k->index_id); off += 8; out[off++] = 0x01;
    return HX_OK;
  }
  out[off++] = k->kind == HX_KEY_VECTOR ? 0xF1 : 0xF0;
  put_be64(out + off, k->index_id); off += 8;
  switch (k->kind) {
    case HX_KEY_VECTOR: out[off++] = 0x02; put_be64(out + off, k->order_code); off += 8; break;
    case HX_KEY_LAYER0_NEIGHBORS: out[off++] = 0x16; break;
    case HX_KEY_UPPER_NEIGHBORS: out[off++] = 0x11; out[off++] = (uint8_t)(k->layer >> 8); out[off++] = (uint8_t)k->layer; break;
    case HX_KEY_SIMHASH: out[off++] = 0x12; break;
    default: out[off++] = 0x13; break;
  }
  put_be64(out + off, k->node_id);
  return HX_OK;
}

extern "C" hx_status hx_index_load_vector_rows(hx_index* ix, const uint64_t* ids, const uint8_t* rows, size_t n) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (n && (!ids || !rows)) return HX_ERR_INVALID_PARAMETER;
  const uint32_t dim = ix->cfg.dimension;
  const size_t rb = 4 + 4 * (size_t)dim;
  std::vector<float> vecs(n * (size_t)dim);
  std::vector<uint32_t> hdr_bits(n);
  for (size_t i = 0; i < n; ++i) {
    memcpy(&hdr_bits[i], rows + i * rb, 4);
    memcpy(vecs.data() + i * (size_t)dim, rows + i * rb + 4, 4 * (size_t)dim);
  }
  hx_status rc = hx_index_load_vectors(ix, ids, vecs.data(), n);
  if (rc || n == 0) return rc;
  // decode_item_borrowed: `bytes_of(&header) != bytes_of(&expected_header)` => HeaderMismatch (mod.rs:942-945)
  std::vector<float> dev_hdr(n);
  HX_CUDA(cudaMemcpy(dev_hdr.data(), ix->d_hdr, n * sizeof(float), cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < n; ++i) {
    uint32_t slot;
    if (!hx_slot_of(ix, ids[i], &slot)) continue;
    uint32_t expect;
    memcpy(&expect, &dev_hdr[slot], 4);
    if (expect != hdr_bits[i]) {
      hx_set_error("vector item row of node %llu: stored header does not match the recomputed header",
                   (unsigned long long)ids[i]);
      ix->free_vectors();
      return HX_ERR_INVARIANT_VIOLATION;
    }
  }
  return HX_OK;
}

extern "C" hx_status hx_index_load_neighbor_rows(hx_index* ix, uint16_t layer, const uint64_t* node_ids,
                                                 const uint8_t* blob, const uint64_t* row_offsets, size_t n) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (n && (!node_ids || !row_offsets)) return HX_ERR_INVALID_PARAMETER;
  std::vector<uint32_t> offs(n + 1, 0);
  std::vector<uint64_t> nbrs;
  std::vector<uint64_t> tmp(4096);
  for (size_t i = 0; i < n; ++i) {
    const size_t len = (size_t)(row_offsets[i + 1] - row_offsets[i]);
    size_t count = 0;
    hx_status rc = hx_decode_neighbor_row(layer, blob + row_offsets[i], len, tmp.data(), tmp.size(), &count, nullptr, nullptr);
    if (rc == HX_ERR_INVALID_PARAMETER && count > tmp.size()) {
      tmp.resize(count);
      rc = hx_decode_neighbor_row(layer, blob + row_offsets[i], len, tmp.data(), tmp.size(), &count, nullptr, nullptr);
    }
    if (rc) return rc;
    nbrs.insert(nbrs.end(), tmp.begin(), tmp.begin() + count);
    offs[i + 1] = (uint32_t)nbrs.size();
  }
  return hx_index_load_graph(ix, layer, node_ids, offs.data(), nbrs.data(), n);
}

extern "C" hx_status hx_index_export_neighbor_row(hx_index* ix, uint16_t layer, uint64_t node_id, uint8_t* out, size_t cap,
                                                  size_t* out_len) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  hx_status rc = hx_finalize_graph(ix);
  if (rc) return rc;
  uint32_t slot;
  if (!hx_slot_of(ix, node_id, &slot) || !ix->d_nbr0) {
    hx_set_error("node %llu has no rows in the device mirror", (unsigned long long)node_id);
    return HX_ERR_INDEX_NOT_FOUND;
  }
  HX_CUDA(cudaSetDevice(ix->device));
  std::vector<uint32_t> row;
  if (layer == 0) {
    uint16_t deg = 0;
    HX_CUDA(cudaMemcpy(&deg, ix->d_deg0 + slot, sizeof(deg), cudaMemcpyDeviceToHost));
    row.resize(deg);
    if (deg) HX_CUDA(cudaMemcpy(row.data(), ix->d_nbr0 + (size_t)slot * ix->stride0, deg * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  } else {
    uint8_t lvl = 0;
    uint32_t off = HX_ABSENT;
    HX_CUDA(cudaMemcpy(&lvl, ix->d_level + slot, 1, cudaMemcpyDeviceToHost));
    HX_CUDA(cudaMemcpy(&off, ix->d_upper_off + slot, 4, cudaMemcpyDeviceToHost));
    if (lvl < layer || off == HX_ABSENT) {
      hx_set_error("node %llu has no row on layer %u", (unsigned long long)node_id, layer);
      return HX_ERR_INDEX_NOT_FOUND;
    }
    uint16_t deg = 0;
    const size_t r = (size_t)off + layer - 1;
    HX_CUDA(cudaMemcpy(&deg, ix->d_upper_deg + r, sizeof(deg), cudaMemcpyDeviceToHost));
    row.resize(deg);
    if (deg) HX_CUDA(cudaMemcpy(row.data(), ix->d_upper_nbr + r * ix->stride_u, deg * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  }
  std::vector<uint64_t> ids(row.size());
  for (size_t i = 0; i < row.size(); ++i) ids[i] = ix->ids_sorted[row[i]];
  return hx_encode_neighbor_row(layer, ids.data(), ids.size(), out, cap, out_len);
}

extern "C" hx_status hx_index_set_entry(hx_index* ix, uint64_t entry_point, uint16_t max_layer) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  uint32_t slot;
  if (!hx_slot_of(ix, entry_point, &slot)) {
    hx_set_error("entry point %llu has no vector row in the device mirror", (unsigned long long)entry_point);
    return HX_ERR_INVARIANT_VIOLATION;
  }
  ix->entry_id = entry_point;
  ix->entry_slot = slot;
  ix->max_layer = max_layer;
  ix->populated = true;
  return HX_OK;
}

// Turn the staged per-layer CSR rows into the fixed-stride device image.
hx_status hx_finalize_graph(hx_index* ix) {
  if (!ix->graph_dirty.load(std::memory_order_acquire)) return HX_OK;
  // Searches may race to be the first after a load: exactly one finalises, the others wait here and then see the
  // finished image (the search path never mutates index state otherwise).
  std::lock_guard<std::mutex> fin(ix->fin_mu);
  if (!ix->graph_dirty.load(std::memory_order_acquire)) return HX_OK;
  HX_CUDA(cudaSetDevice(ix->device));
  const size_t n = ix->n;
  // free previous device graph but keep staging
  std::vector<HxLayerRows> staged;
  staged.swap(ix->staged);
  const bool pop = ix->populated;
  ix->free_graph();
  ix->populated = pop;
  ix->staged.swap(staged);
  if (n == 0) {
    ix->graph_dirty.store(false, std::memory_order_release);
    return HX_OK;
  }
  uint32_t max0 = ix->lim0, maxu = ix->cfg.m;
  for (size_t l = 0; l < ix->staged.size(); ++l) {
    const HxLayerRows& L = ix->staged[l];
    for (size_t i = 0; i + 1 < L.offsets.size(); ++i) {
      const uint32_t len = L.offsets[i + 1] - L.offsets[i];
      if (l == 0) max0 = std::max(max0, len); else maxu = std::max(maxu, len);
    }
  }
  if (max0 > 4096 || maxu > 4096) {
    hx_set_error("neighbour rows longer than 4096 are not supported");
    return HX_ERR_INVALID_PARAMETER;
  }
  ix->stride0 = round_up(max0, 32);
  ix->stride_u = round_up(maxu, 16);
  std::vector<uint8_t> level(n, 0);
  std::vector<uint32_t> nbr0(n * (size_t)ix->stride0, 0);
  std::vector<uint16_t> deg0(n, 0), raw0(n, 0);
  if (!ix->staged.empty()) {
    const HxLayerRows& L = ix->staged[0];
    for (size_t i = 0; i < L.node.size(); ++i) {
      const uint32_t s = L.node[i], b = L.offsets[i], e = L.offsets[i + 1];
      memcpy(nbr0.data() + (size_t)s * ix->stride0, L.nbr.data() + b, (size_t)(e - b) * sizeof(uint32_t));
      deg0[s] = (uint16_t)(e - b);
      raw0[s] = (uint16_t)std::min<uint32_t>(L.raw_len[i], 65535);
    }
  }
  for (size_t l = 1; l < ix->staged.size(); ++l)
    for (uint32_t s : ix->staged[l].node) level[s] = std::max<uint8_t>(level[s], (uint8_t)l);
  std::vector<uint32_t> upper_off(n, HX_ABSENT);
  size_t rows = 0;
  for (size_t s = 0; s < n; ++s)
    if (level[s] > 0) {
      upper_off[s] = (uint32_t)rows;
      rows += level[s];
    }
  ix->n_upper_rows = rows;
  std::vector<uint32_t> upper_nbr(std::max<size_t>(rows, 1) * ix->stride_u, 0);
  std::vector<uint16_t> upper_deg(std::max<size_t>(rows, 1), 0);
  for (size_t l = 1; l < ix->staged.size(); ++l) {
    const HxLayerRows& L = ix->staged[l];
    for (size_t i = 0; i < L.node.size(); ++i) {
      const uint32_t s = L.node[i], b = L.offsets[i], e = L.offsets[i + 1];
      const size_t r = (size_t)upper_off[s] + (l - 1);
      memcpy(upper_nbr.data() + r * ix->stride_u, L.nbr.data() + b, (size_t)(e - b) * sizeof(uint32_t));
      upper_deg[r] = (uint16_t)(e - b);
    }
  }
  const size_t rcap = std::max(ix->cap_rows, n);   // per-row arrays follow the vector arrays' capacity (hx_mirror.inl)
  HX_CUDA(cudaMalloc((void**)&ix->d_nbr0, rcap * (size_t)ix->stride0 * sizeof(uint32_t)));
  HX_CUDA(cudaMalloc((void**)&ix->d_deg0, rcap * sizeof(uint16_t)));
  HX_CUDA(cudaMalloc((void**)&ix->d_raw0, rcap * sizeof(uint16_t)));
  HX_CUDA(cudaMalloc((void**)&ix->d_upper_off, rcap * sizeof(uint32_t)));
  HX_CUDA(cudaMalloc((void**)&ix->d_upper_nbr, upper_nbr.size() * sizeof(uint32_t)));
  HX_CUDA(cudaMalloc((void**)&ix->d_upper_deg, upper_deg.size() * sizeof(uint16_t)));
  HX_CUDA(cudaMalloc((void**)&ix->d_level, rcap));
  if (rcap > n) {
    HX_CUDA(cudaMemset(ix->d_deg0, 0, rcap * sizeof(uint16_t)));
    HX_CUDA(cudaMemset(ix->d_raw0, 0, rcap * sizeof(uint16_t)));
    HX_CUDA(cudaMemset(ix->d_upper_off, 0xFF, rcap * sizeof(uint32_t)));
    HX_CUDA(cudaMemset(ix->d_level, 0, rcap));
  }
  HX_CUDA(cudaMemcpy(ix->d_nbr0, nbr0.data(), nbr0.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  HX_CUDA(cudaMemcpy(ix->d_deg0, deg0.data(), n * sizeof(uint16_t), cudaMemcpyHostToDevice));
  HX_CUDA(cudaMemcpy(ix->d_raw0, raw0.data(), n * sizeof(uint16_t), cudaMemcpyHostToDevice));
  HX_CUDA(cudaMemcpy(ix->d_upper_off, upper_off.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice));
  HX_CUDA(cudaMemcpy(ix->d_upper_nbr, upper_nbr.data(), upper_nbr.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  HX_CUDA(cudaMemcpy(ix->d_upper_deg, upper_deg.data(), upper_deg.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
  HX_CUDA(cudaMemcpy(ix->d_level, level.data(), n, cudaMemcpyHostToDevice));
  ix->staged.clear();
  ix->graph_dirty.store(false, std::memory_order_release);
  return HX_OK;
}

extern "C" hx_status hx_index_build(hx_index* ix, const uint16_t* levels, uint64_t seed) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  HX_CUDA(cudaSetDevice(ix->device));
  return hx_build_impl(ix, levels, seed, 0);
}

extern "C" hx_status hx_index_build_ex(hx_index* ix, const uint16_t* levels, uint64_t seed, int32_t mode) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (mode != HX_BUILD_BATCHED && mode != HX_BUILD_SEQUENTIAL) {
    hx_set_error("unknown build mode %d", mode);
    return HX_ERR_INVALID_PARAMETER;
  }
  HX_CUDA(cudaSetDevice(ix->device));
  return hx_build_impl(ix, levels, seed, mode == HX_BUILD_SEQUENTIAL ? 1 : 0);
}

extern "C" hx_status hx_index_graph_info(hx_index* ix, uint64_t* n_nodes, uint64_t* entry_point, uint16_t* max_layer,
                                         uint32_t* layer0_stride, uint32_t* upper_stride) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  hx_status rc = hx_finalize_graph(ix);
  if (rc) return rc;
  if (n_nodes) *n_nodes = ix->n;
  if (entry_point) *entry_point = ix->populated ? ix->entry_id : 0;
  if (max_layer) *max_layer = (uint16_t)(ix->populated ? ix->max_layer : 0);
  if (layer0_stride) *layer0_stride = ix->stride0;
  if (upper_stride) *upper_stride = ix->stride_u;
  return HX_OK;
}

extern "C" hx_status hx_index_download_graph(hx_index* ix, uint16_t* levels, uint32_t* deg0, uint32_t* nbr0,
                                             uint64_t* n_upper_rows, uint32_t* upper_node, uint16_t* upper_layer,
                                             uint32_t* upper_deg, uint32_t* upper_nbr, size_t upper_cap) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  hx_status rc = hx_finalize_graph(ix);
  if (rc) return rc;
  HX_CUDA(cudaSetDevice(ix->device));
  const size_t n = ix->n;
  if (n_upper_rows) *n_upper_rows = ix->n_upper_rows;
  if (n == 0 || !ix->d_nbr0) return HX_OK;
  std::vector<uint8_t> level(n);
  HX_CUDA(cudaMemcpy(level.data(), ix->d_level, n, cudaMemcpyDeviceToHost));
  if (levels)
    for (size_t i = 0; i < n; ++i) levels[i] = level[i];
  if (deg0) {
    std::vector<uint16_t> d(n);
    HX_CUDA(cudaMemcpy(d.data(), ix->d_deg0, n * sizeof(uint16_t), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; ++i) deg0[i] = d[i];
  }
  if (nbr0) HX_CUDA(cudaMemcpy(nbr0, ix->d_nbr0, n * (size_t)ix->stride0 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  if (upper_node && upper_layer && upper_deg && upper_nbr) {
    if (upper_cap < ix->n_upper_rows) {
      hx_set_error("upper row capacity %zu < %zu", upper_cap, ix->n_upper_rows);
      return HX_ERR_INVALID_PARAMETER;
    }
    const size_t rows = ix->n_upper_rows;
    if (rows) {
      std::vector<uint16_t> d(rows);
      HX_CUDA(cudaMemcpy(d.data(), ix->d_upper_deg, rows * sizeof(uint16_t), cudaMemcpyDeviceToHost));
      for (size_t r = 0; r < rows; ++r) upper_deg[r] = d[r];
      HX_CUDA(cudaMemcpy(upper_nbr, ix->d_upper_nbr, rows * (size_t)ix->stride_u * sizeof(uint32_t),
                         cudaMemcpyDeviceToHost));
      size_t r = 0;
      for (size_t s = 0; s < n; ++s)
        for (uint32_t l = 1; l <= level[s]; ++l) {
          upper_node[r] = (uint32_t)s;
          upper_layer[r] = (uint16_t)l;
          ++r;
        }
    }
  }
  return HX_OK;
}

// ------------------------------------------------------------------------------------------------
// search parameter checks (SearchParams::new / with_ef, mod.rs:480-500)
// ------------------------------------------------------------------------------------------------
static inline bool params_strict(const hx_search_params* p) {   // !requires_query_simhash() (mod.rs:556-561)
  return p->simhash_mode == HX_SIMHASH_OFF && !(p->pre_sampling_ratio >= 0.0f && p->pre_sampling_ratio < 1.0f);
}

static hx_status check_params(const hx_index* ix, const hx_search_params* p, uint32_t* k, uint32_t* ef) {
  if (!p) {
    hx_set_error("null search params");
    return HX_ERR_INVALID_PARAMETER;
  }
  if (p->k == 0) {
    hx_set_error("result count must be non-zero");   // ResultCount::try_new
    return HX_ERR_INVALID_PARAMETER;
  }
  uint32_t e = p->ef == 0 ? std::max(p->k, 100u) : p->ef;
  if (e < p->k) {
    hx_set_error("search beam width must be at least %u, got %u", p->k, e);   // SearchBeamWidth::try_new
    return HX_ERR_INVALID_PARAMETER;
  }
  if (p->simhash_mode < HX_SIMHASH_OFF || p->simhash_mode > HX_SIMHASH_ALWAYS) {
    hx_set_error("unknown SimHash mode %d", p->simhash_mode);
    return HX_ERR_INVALID_PARAMETER;
  }
  if (p->pre_sampling_ratio > 1.0f || p->pre_sampling_ratio != p->pre_sampling_ratio) {
    hx_set_error("pre-SimHash sampling ratio must lie in the unit interval");   // UnitInterval::try_new
    return HX_ERR_INVALID_PARAMETER;
  }
  if (p->query_dimension != 0 && p->query_dimension != ix->cfg.dimension) {
    hx_set_error("invalid dimension: expected %u, got %u", ix->cfg.dimension, p->query_dimension);
    return HX_ERR_INVALID_DIMENSION;
  }
  if (e > 4096) {
    hx_set_error("beam width %u above the supported maximum 4096", e);
    return HX_ERR_INVALID_PARAMETER;
  }
  *k = p->k;
  *ef = e;
  return HX_OK;
}

// Upload B host queries and produce q_hdr / q_status on the device (host-side for small B, kernel otherwise).
static hx_status stage_queries(hx_index* ix, HxScratch* s, const float* queries, size_t B, uint32_t* launches,
                               bool per_query = false) {
  const uint32_t dim = ix->cfg.dimension;
  hx_status rc;
  if ((rc = s->d_queries.reserve(B * (size_t)dim))) return rc;
  if ((rc = s->d_qhdr.reserve(B))) return rc;
  if ((rc = s->d_qstatus.reserve(B))) return rc;
  HX_CUDA(cudaMemcpyAsync(s->d_queries.p, queries, B * (size_t)dim * sizeof(float), cudaMemcpyHostToDevice, s->stream));
  float limit = 0.f;
  const bool has_limit = component_limit(ix->cfg.metric, dim, &limit);
  if (B <= 8) {
    if ((rc = s->h_qhdr.reserve(B))) return rc;
    if ((rc = s->h_status.reserve(B))) return rc;
    for (size_t b = 0; b < B; ++b) {
      const uint32_t w = host_validate(queries + b * (size_t)dim, dim, ix->cfg.metric, has_limit, limit);
      if (w != HX_ST_OK && !per_query) return status_from_word(w, b, "query");
      s->h_status.p[b] = w;   // per-query mode: the kernels skip a query whose status word is set
      s->h_qhdr.p[b] = (w == HX_ST_OK && ix->cfg.metric == HX_METRIC_COSINE) ? host_cosine_norm(queries + b * (size_t)dim, dim) : 0.0f;
    }
    HX_CUDA(cudaMemcpyAsync(s->d_qhdr.p, s->h_qhdr.p, B * sizeof(float), cudaMemcpyHostToDevice, s->stream));
    HX_CUDA(cudaMemcpyAsync(s->d_qstatus.p, s->h_status.p, B * sizeof(uint32_t), cudaMemcpyHostToDevice, s->stream));
  } else {
    k_validate_and_header<<<(unsigned)((B + 7) / 8), 256, 0, s->stream>>>(s->d_queries.p, B, dim, dim, ix->cfg.metric,
                                                                         limit, has_limit ? 1 : 0, s->d_qhdr.p,
                                                                         s->d_qstatus.p);
    HX_CUDA(cudaGetLastError());
    (*launches)++;
  }
  return HX_OK;
}

static hx_status prepare_device_queries(hx_index* ix, HxScratch* s, const float* d_queries, size_t B,
                                        cudaStream_t stream, uint32_t* launches) {
  const uint32_t dim = ix->cfg.dimension;
  hx_status rc;
  if ((rc = s->d_qhdr.reserve(B))) return rc;
  if ((rc = s->d_qstatus.reserve(B))) return rc;
  float limit = 0.f;
  const bool has_limit = component_limit(ix->cfg.metric, dim, &limit);
  k_validate_and_header<<<(unsigned)((B + 7) / 8), 256, 0, stream>>>(d_queries, B, dim, dim, ix->cfg.metric, limit,
                                                                    has_limit ? 1 : 0, s->d_qhdr.p, s->d_qstatus.p);
  HX_CUDA(cudaGetLastError());
  (*launches)++;
  return HX_OK;
}

// ---- HNSW launch ---------------------------------------------------------------------------------
#define HX_TIE_POOL_N 256u     // overflow regions shared by the queries of a launch (claimed on a query's 33rd tie)
#define HX_TIE_POOL_CAP 4096u  // entries per region: a query can hold 32 + 4096 exact ties at its beam boundary
// overflow regions of the tie stack + per-query error words on one scratch set
static hx_status setup_tie_pool(HxScratch* s, HxRingArgs* rg, cudaStream_t stream) {
  hx_status rc;
  if (!s->tiepool_init) {
    if ((rc = s->d_tiepool.reserve((size_t)HX_TIE_POOL_N * HX_TIE_POOL_CAP))) return rc;
    if ((rc = s->d_tiebusy.reserve(HX_TIE_POOL_N))) return rc;
    HX_CUDA(cudaMemsetAsync(s->d_tiebusy.p, 0, HX_TIE_POOL_N * sizeof(uint32_t), stream));
    s->tiepool_init = true;
  }
  rg->tie_pool = s->d_tiepool.p;
  rg->tie_busy = s->d_tiebusy.p;
  rg->tie_pool_n = HX_TIE_POOL_N;
  rg->tie_pool_cap = HX_TIE_POOL_CAP;
  return HX_OK;
}

// ---- CTA-per-query ring build: configuration + launch (shared by hx_search's small-batch path and the query service) ----
// Shared memory per CTA: [query (QCH == 0)] | RC row slots | beam / merge stage [ef] | tie stack | RC mbarriers | frontier |
// scores | visited table.  `budget` = dynamic shared memory the CTA may take (227 KB: one CTA per SM; ~113 KB: two).
bool hx_cta_ring_config(const hx_index* ix, uint32_t ef, uint32_t want_warps, uint32_t want_rc, uint32_t want_vt_log2,
                        size_t budget, HxCtaRingCfg* c) {
  const uint32_t chunks = ix->ld / 32;
  const size_t rowbytes = (size_t)ix->ld * 4;
  c->qch = ix->cfg.metric == HX_METRIC_MANHATTAN ? 0 : chunks <= 8 ? 8 : chunks <= 24 ? 24 : chunks <= 48 ? 48 : 0;
  c->fr_cap = round_up(std::max(std::max(ix->stride0, ix->stride_u), 32u), 32);
  uint32_t lg = 12;
  while ((1u << lg) < 64u * ef && lg < 24) lg++;
  if (want_vt_log2 >= 6 && want_vt_log2 <= 24) lg = want_vt_log2;
  uint32_t vt = 1u << lg;
  const size_t fixed0 = (c->qch == 0 ? rowbytes : 0) + (size_t)ef * 8 + HX_TIE_CAP * 8 + (size_t)c->fr_cap * 8 + 256;
  const uint32_t min_rows = want_rc ? std::min(want_rc, 8u) : 8u;
  while (vt > 1024 && fixed0 + (size_t)vt * 4 + min_rows * (rowbytes + 8) > budget) vt >>= 1;
  if (fixed0 + (size_t)vt * 4 + rowbytes + 8 > budget) return false;
  uint32_t rc = (uint32_t)std::min<size_t>(32, (budget - fixed0 - (size_t)vt * 4) / (rowbytes + 8));
  if (want_rc) rc = std::min(rc, want_rc);
  c->RC = rc;
  c->vt_cap = vt;
  c->smem = fixed0 - 256 + (size_t)vt * 4 + (size_t)rc * (rowbytes + 8);
  const uint32_t max_warps = c->qch == 48 ? 8 : 12;
  c->warps = want_warps ? std::min(want_warps, max_warps) : max_warps;
  c->ef = ef;
  return true;
}

// The dynamic-shared-memory attribute is per kernel INSTANTIATION and device: `set_for` must be one array per
// instantiation (every k_hnsw_search_cta_ring<M,Q,NB> has the same function TYPE, so a static inside a function template
// keyed by that type would be shared by all of them — the macro below declares it per expansion instead).
template <typename F>
static hx_status cta_ring_prepare(F* fn, std::atomic<size_t>* set_for, int device, size_t smem) {
  const int d = device & 63;
  if (set_for[d].load(std::memory_order_relaxed) < smem) {
    HX_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    set_for[d].store(smem, std::memory_order_relaxed);
  }
  return HX_OK;
}

hx_status hx_launch_cta_ring(hx_index* ix, const HxCtaRingCfg& c, const HxHnswArgs& a, const HxRingArgs& rg, uint32_t grid,
                             cudaStream_t stream, int* ctas_per_sm) {
  const HxDev dev = ix->dev();
  hx_status rc = HX_OK;
#define HX_CTA_GO(M, Q, NBV)                                                                                          \
  do {                                                                                                                \
    static std::atomic<size_t> set_for[64];                                                                           \
    if ((rc = cta_ring_prepare(k_hnsw_search_cta_ring<M, Q, NBV>, set_for, ix->device, c.smem))) return rc;            \
    if (ctas_per_sm)                                                                                                  \
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_per_sm, k_hnsw_search_cta_ring<M, Q, NBV>, (int)c.warps * 32, \
                                                    c.smem);                                                          \
    if (grid)                                                                                                         \
      k_hnsw_search_cta_ring<M, Q, NBV><<<grid, c.warps * 32, c.smem, stream>>>(dev, a, rg, c.RC, c.vt_cap);          \
  } while (0)
#define HX_CTA_NB(M, Q)                                                                                               \
  do {                                                                                                                \
    if (c.ef <= 128) HX_CTA_GO(M, Q, 4);                                                                              \
    else HX_CTA_GO(M, Q, 0);                                                                                          \
  } while (0)
#define HX_CTA_Q(M)                                                                                                   \
  do {                                                                                                                \
    if (c.qch == 8) HX_CTA_NB(M, 8);                                                                                  \
    else if (c.qch == 24) HX_CTA_NB(M, 24);                                                                           \
    else if (c.qch == 48) HX_CTA_NB(M, 48);                                                                           \
    else HX_CTA_NB(M, 0);                                                                                             \
  } while (0)
  if (ix->cfg.metric == HX_METRIC_EUCLIDEAN) HX_CTA_Q(HXM_EUCLIDEAN);
  else if (ix->cfg.metric == HX_METRIC_COSINE) HX_CTA_Q(HXM_COSINE);
  else HX_CTA_NB(HXM_MANHATTAN, 0);   // one thread per row, sequential chain: the query stays in shared memory
#undef HX_CTA_Q
#undef HX_CTA_NB
#undef HX_CTA_GO
  if (grid) HX_CUDA(cudaGetLastError());
  return HX_OK;
}

struct HxFusedArgs {   // pipelined host-buffer search: validation inside the ring kernel, start gated on `avail`
  const uint32_t* avail = nullptr;
  float limit = 0.f;
  int has_limit = 0;
};

// true when launch_hnsw takes the warp-per-query build for this call (the host-buffer path pipelines only that one)
static bool hnsw_uses_ring(const hx_index* ix, size_t B) { return B >= (size_t)ix->sm_count; }

// Two builds of the same algorithm (bit-identical results, every metric):
//  * B <  #SMs : one CTA per query (k_hnsw_search_cta_ring: rows spread over the CTA's warps, register beam, visited set in
//                shared memory) — lowest latency per query;
//  * B >= #SMs : one WARP per query (k_hnsw_search_ring), up to 16 queries in flight per SM — highest throughput.
// Shapes the CTA build cannot hold (a row does not fit next to the visited table) take the warp build; rows that do not fit
// a warp's share either are reduced straight from global memory (R = 0).
static hx_status launch_hnsw(hx_index* ix, HxScratch* s, const float* d_queries, size_t B, uint32_t k, uint32_t ef,
                             uint64_t* d_out_ids, float* d_out_scores, uint32_t* d_out_counts, uint32_t* d_qstats,
                             cudaStream_t stream, cudaEvent_t e0, cudaEvent_t e1, bool* timed, uint32_t* launches,
                             const HxFusedArgs* fused = nullptr, bool sticky_flags = false) {
  *timed = false;
  hx_status rc = hx_finalize_graph(ix);
  if (rc) return rc;
  if ((rc = s->d_qerr.reserve(B))) return rc;
  if (ix->n == 0 || !ix->populated || !ix->d_nbr0) {   // VectorIndexState::Empty => Ok(vec![]) (search.rs:1127-1128)
    HX_CUDA(cudaMemsetAsync(s->d_qerr.p, 0, B * sizeof(uint32_t), stream));
    HX_CUDA(cudaMemsetAsync(d_out_counts, 0, B * sizeof(uint32_t), stream));
    if (d_qstats) HX_CUDA(cudaMemsetAsync(d_qstats, 0, B * 4 * sizeof(uint32_t), stream));
    return HX_OK;
  }
  const hx_tuning& t = ix->tune;
  const bool manhattan = ix->cfg.metric == HX_METRIC_MANHATTAN;
  const uint32_t fr_cap = round_up(std::max(std::max(ix->stride0, ix->stride_u), 32u), 32);
  const size_t rowbytes = (size_t)ix->ld * 4;
  const size_t ring_budget = 227 * 1024;
  const uint32_t chunks = ix->ld / 32;
  // the query lives in registers (QCH chunks of 32) when it fits; Manhattan walks it sequentially: shared memory
  const uint32_t ring_qch = manhattan ? 0u : chunks <= 8 ? 8u : chunks <= 24 ? 24u : chunks <= 48 ? 48u : 0u;
  uint32_t lg = 12;
  while ((1u << lg) < 64u * ef && lg < 24) lg++;
  const uint32_t vt_cap = 1u << knob(t.visited_log2, lg);
  HxCtaRingCfg cta_cfg{};
  bool use_cta_ring = B < (size_t)ix->sm_count &&
                      hx_cta_ring_config(ix, ef, knob(t.lat_warps, 0), knob(t.ring_rows, 0), knob(t.visited_log2, 0), ring_budget,
                                         &cta_cfg) &&
                      cta_cfg.fr_cap == fr_cap;
  uint32_t ring_R = 0, ring_wstride = 0, ring_wpc = 0;
  if (!use_cta_ring) {
    const size_t fixed0 = (ring_qch == 0 ? rowbytes : 0) + (size_t)ef * 8 + HX_TIE_CAP * 8 + (size_t)fr_cap * 12;
    uint32_t want_wpc = knob(t.ring_warps, 16);
    if (ring_qch == 48) want_wpc = std::min(want_wpc, (uint32_t)HX_RING_QCH48_THREADS / 32u);   // launch bound of that build
    const uint32_t want_R = knob(t.ring_rows, 0);
    // few queries: fewer warps per CTA so that the batch spreads over all SMs (and each warp gets a deeper ring)
    const uint32_t spread = (uint32_t)std::max<size_t>(1, (B + ix->sm_count - 1) / (size_t)ix->sm_count);
    want_wpc = std::min(want_wpc, spread);
    for (uint32_t w = want_wpc; w >= 1 && !manhattan; --w) {
      const size_t per_warp = (ring_budget / w) & ~(size_t)127;
      if (per_warp <= fixed0 + 8 + rowbytes) continue;
      uint32_t r = (uint32_t)std::min<size_t>(32, (per_warp - fixed0) / (rowbytes + 8));
      if (want_R) r = std::min(r, want_R);
      if (r >= 4 || w == 1 || (want_R && r == want_R)) { ring_wpc = w; ring_R = r; break; }
    }
    if (ring_wpc == 0) {   // no row slots: Manhattan (one lane per row, from global memory) or rows too large to stage
      const size_t need = round_up((uint32_t)std::min<size_t>(fixed0, 1u << 30), 128);
      if (need > ring_budget) {
        hx_set_error("query working set %zu bytes exceeds shared memory (dimension %u, ef %u)", fixed0, ix->cfg.dimension, ef);
        return HX_ERR_INVALID_PARAMETER;
      }
      ring_wpc = (uint32_t)std::max<size_t>(1, std::min<size_t>(want_wpc, ring_budget / need));
    }
    ring_wstride = round_up((uint32_t)(fixed0 + (size_t)ring_R * (rowbytes + 8)), 128);
  }
  const bool use_ring = !use_cta_ring;
  uint32_t grid;
  size_t smem_launch, vslots = 0;
  if (use_ring) {
    grid = (uint32_t)std::min<size_t>((B + ring_wpc - 1) / ring_wpc, (size_t)ix->sm_count);
    smem_launch = (size_t)ring_wpc * ring_wstride;
    vslots = (size_t)grid * ring_wpc;
  } else {
    grid = (uint32_t)B;   // B < #SMs
    smem_launch = cta_cfg.smem;
  }
  HxRingArgs rg{};
  {
    const uint32_t pool_n = knob(t.visited_pool, 32);
    const uint32_t pool_cap = std::max<uint32_t>(vt_cap * 16u, 65536u);
    if (vslots && (rc = s->d_vtab.reserve(vslots * vt_cap))) return rc;
    if (s->vpool_n != pool_n || s->vpool_cap != pool_cap || !s->d_vbusy.p) {
      if ((rc = s->d_vpool.reserve((size_t)std::max(pool_n, 1u) * pool_cap))) return rc;
      if ((rc = s->d_vbusy.reserve(std::max(pool_n, 1u)))) return rc;
      HX_CUDA(cudaMemsetAsync(s->d_vbusy.p, 0, std::max(pool_n, 1u) * sizeof(uint32_t), stream));
      s->vpool_n = pool_n;
      s->vpool_cap = pool_cap;
    }
    rg.vtab = s->d_vtab.p;
    rg.vt_cap = vt_cap;
    rg.pool = s->d_vpool.p;
    rg.pool_busy = s->d_vbusy.p;
    rg.pool_n = pool_n;
    rg.pool_cap = pool_cap;
    rg.l2_hint = knob(t.l2_hint, 1);
    rg.prefetch_below = knob(t.prefetch_below, ef / 2 + 1);
    if ((rc = setup_tie_pool(s, &rg, stream))) return rc;
    rg.batch_admit = knob(t.lat_admit_seq, 0) ? 0u : 1u;
    rg.l2_spec = knob(t.lat_spec, 0);   // off: the speculative row prefetch costs more than it hides (DESIGN §5)
    if (knob(t.phase_prof, 0)) {        // diagnostics: cycle sums per phase of the latency build
      if ((rc = s->d_prof.reserve(8))) return rc;
      if (!s->prof_init) { HX_CUDA(cudaMemsetAsync(s->d_prof.p, 0, 8 * sizeof(unsigned long long), stream)); s->prof_init = true; }
      rg.prof = s->d_prof.p;
    }
  }
  const bool had_err = s->d_err.p != nullptr;
  if ((rc = s->d_err.reserve(4))) return rc;   // [0] error flags, [1] query counter of the ring build, [2] queries landed
  // device-buffer calls keep the flag word sticky (ORed over launches until hx_device_flags reads and clears it)
  if (sticky_flags && had_err) HX_CUDA(cudaMemsetAsync(s->d_err.p + 1, 0, sizeof(uint32_t), stream));
  else HX_CUDA(cudaMemsetAsync(s->d_err.p, 0, 2 * sizeof(uint32_t), stream));
  rg.counter = s->d_err.p + 1;
  HxHnswArgs a{};
  a.queries = d_queries;
  a.q_hdr = s->d_qhdr.p;
  a.q_status = s->d_qstatus.p;
  a.B = (uint32_t)B;
  a.k = k;
  a.ef = ef;
  a.out_ids = d_out_ids;
  a.out_scores = d_out_scores;
  a.out_counts = d_out_counts;
  a.q_stats = d_qstats;
  a.err_flags = s->d_err.p;
  a.q_err = s->d_qerr.p;
  a.fr_cap = fr_cap;
  if (fused) {
    if (!use_ring) {
      hx_set_error("internal: fused validation needs the warp-per-query build");
      return HX_ERR_INVARIANT_VIOLATION;
    }
    a.fused_validate = 1;
    a.q_status_w = s->d_qstatus.p;
    a.q_hdr_w = s->d_qhdr.p;
    a.limit = fused->limit;
    a.has_limit = fused->has_limit;
    a.avail = fused->avail;
  }
  const HxDev dev = ix->dev();
  HX_CUDA(cudaEventRecord(e0, stream));
#define HX_LAUNCH_RING(M, Q)                                                                                       \
  do {                                                                                                             \
    HX_CUDA(cudaFuncSetAttribute(k_hnsw_search_ring<M, Q>, cudaFuncAttributeMaxDynamicSharedMemorySize,            \
                                 (int)smem_launch));                                                               \
    k_hnsw_search_ring<M, Q><<<grid, ring_wpc * 32, smem_launch, stream>>>(dev, a, rg, ring_wstride, ring_R);      \
  } while (0)
#define HX_LAUNCH_RING_Q(M)                                                                                        \
  do {                                                                                                             \
    if (ring_qch == 8) HX_LAUNCH_RING(M, 8);                                                                       \
    else if (ring_qch == 24) HX_LAUNCH_RING(M, 24);                                                                \
    else if (ring_qch == 48) HX_LAUNCH_RING(M, 48);                                                                \
    else HX_LAUNCH_RING(M, 0);                                                                                     \
  } while (0)
  if (use_cta_ring) {
    if ((rc = hx_launch_cta_ring(ix, cta_cfg, a, rg, grid, stream, nullptr))) return rc;
  } else {
    switch (ix->cfg.metric) {
      case HX_METRIC_EUCLIDEAN: HX_LAUNCH_RING_Q(HXM_EUCLIDEAN); break;
      case HX_METRIC_COSINE: HX_LAUNCH_RING_Q(HXM_COSINE); break;
      default: HX_LAUNCH_RING(HXM_MANHATTAN, 0); break;
    }
  }
#undef HX_LAUNCH_RING_Q
#undef HX_LAUNCH_RING
  HX_CUDA(cudaGetLastError());
  HX_CUDA(cudaEventRecord(e1, stream));
  *timed = true;
  (*launches)++;
  return HX_OK;
}

static hx_status check_device_flags(uint32_t flags) {
  if (flags & HXF_INVALID_SCORE) {
    hx_set_error("vector distance kernel emitted an invalid score");   // model.rs:21-28
    return HX_ERR_INVARIANT_VIOLATION;
  }
  if (flags & HXF_COPY_TIMEOUT) {
    hx_set_error("the host-to-device copy of the queries did not complete (pipelined search gave up waiting)");
    return HX_ERR_CUDA;
  }
  if (flags & HXF_VT_OVERFLOW) {
    hx_set_error("visited-set overflow: a query visited more nodes than the overflow tables hold");
    return HX_ERR_INVARIANT_VIOLATION;
  }
  if (flags & HXF_TIE_OVERFLOW) {
    hx_set_error("more than %u exact score ties at the beam boundary (tie-stack overflow regions exhausted)",
                 (unsigned)(HX_TIE_CAP + HX_TIE_POOL_CAP));
    return HX_ERR_INVARIANT_VIOLATION;
  }
  return HX_OK;
}

// ---- result download -------------------------------------------------------------------------------------------------------
// Small calls (one query per call is the reference's usage) are dominated by fixed costs: six device-to-host copies of a few
// bytes each cost more than the data.  Their results are packed into one block by a tiny kernel and cross PCIe in ONE copy.
static __global__ void k_pack_small(const uint64_t* __restrict__ ids, const float* __restrict__ scores,
                                    const uint32_t* __restrict__ counts, const uint32_t* __restrict__ status,
                                    const uint32_t* __restrict__ qerr, const uint32_t* __restrict__ err, uint32_t n_ids,
                                    uint32_t B, unsigned char* __restrict__ out) {
  uint64_t* o_ids = reinterpret_cast<uint64_t*>(out);
  float* o_sc = reinterpret_cast<float*>(o_ids + n_ids);
  uint32_t* o_cnt = reinterpret_cast<uint32_t*>(o_sc + n_ids);
  uint32_t* o_st = o_cnt + B;
  uint32_t* o_qe = o_st + B;
  for (uint32_t i = threadIdx.x; i < n_ids; i += blockDim.x) { o_ids[i] = ids[i]; o_sc[i] = scores[i]; }
  for (uint32_t i = threadIdx.x; i < B; i += blockDim.x) { o_cnt[i] = counts[i]; o_st[i] = status[i]; o_qe[i] = qerr ? qerr[i] : 0u; }
  if (threadIdx.x == 0) o_qe[B] = err ? err[0] : 0u;
}

struct HxDownload {
  bool packed = false;
  size_t n_ids = 0, B = 0;
};
// enqueue the download of ids / scores / counts / per-query status / per-query error flags / batch flags on s->stream
static hx_status enqueue_results(HxScratch* s, size_t B, uint32_t k, uint64_t* out_ids, float* out_scores,
                                 uint32_t* out_counts, uint32_t* launches, HxDownload* dl) {
  hx_status rc;
  dl->n_ids = B * (size_t)k;
  dl->B = B;
  if ((rc = s->h_status.reserve(B))) return rc;
  if ((rc = s->h_qerr.reserve(B))) return rc;
  if ((rc = s->h_err.reserve(1))) return rc;
  s->h_err.p[0] = 0;
  const bool have_qerr = s->d_qerr.p != nullptr && s->d_qerr.cap >= B;
  if (dl->n_ids <= 4096 && s->d_err.p) {
    const size_t bytes = dl->n_ids * 12 + B * 12 + 4;
    if ((rc = s->d_block.reserve(bytes))) return rc;
    if ((rc = s->h_block.reserve(bytes))) return rc;
    k_pack_small<<<1, 256, 0, s->stream>>>(s->d_out_ids.p, s->d_out_scores.p, s->d_out_counts.p, s->d_qstatus.p,
                                          have_qerr ? s->d_qerr.p : nullptr, s->d_err.p, (uint32_t)dl->n_ids, (uint32_t)B,
                                          s->d_block.p);
    HX_CUDA(cudaGetLastError());
    (*launches)++;
    HX_CUDA(cudaMemcpyAsync(s->h_block.p, s->d_block.p, bytes, cudaMemcpyDeviceToHost, s->stream));
    dl->packed = true;
    return HX_OK;
  }
  HX_CUDA(cudaMemcpyAsync(out_ids, s->d_out_ids.p, dl->n_ids * sizeof(uint64_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(out_scores, s->d_out_scores.p, dl->n_ids * sizeof(float), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(out_counts, s->d_out_counts.p, B * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(s->h_status.p, s->d_qstatus.p, B * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  if (have_qerr) HX_CUDA(cudaMemcpyAsync(s->h_qerr.p, s->d_qerr.p, B * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  else memset(s->h_qerr.p, 0, B * sizeof(uint32_t));
  if (s->d_err.p) HX_CUDA(cudaMemcpyAsync(s->h_err.p, s->d_err.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  return HX_OK;
}
// after the stream has been synchronised
static void finish_results(HxScratch* s, const HxDownload& dl, uint64_t* out_ids, float* out_scores, uint32_t* out_counts) {
  if (!dl.packed) return;
  const unsigned char* b = s->h_block.p;
  memcpy(out_ids, b, dl.n_ids * 8);
  memcpy(out_scores, b + dl.n_ids * 8, dl.n_ids * 4);
  memcpy(out_counts, b + dl.n_ids * 12, dl.B * 4);
  memcpy(s->h_status.p, b + dl.n_ids * 12 + dl.B * 4, dl.B * 4);
  memcpy(s->h_qerr.p, b + dl.n_ids * 12 + dl.B * 8, dl.B * 4);
  memcpy(s->h_err.p, b + dl.n_ids * 12 + dl.B * 12, 4);
}

// Per-query outcome of a finished batch.  The reference runs one query per call, so one query's failure must not take
// the others down: with `out_status` every query gets its own code (and the call returns HX_OK); without it the call
// fails with the first failing query's error, like B sequential reference calls stopped at the first Err.
static hx_status report_batch(HxScratch* s, size_t B, uint32_t* out_counts, hx_status* out_status) {
  hx_status first = HX_OK;
  const uint32_t batch_flags = s->h_err.p[0];
  for (size_t b = 0; b < B; ++b) {
    hx_status st = HX_OK;
    if (s->h_status.p[b] != HX_ST_OK) st = status_from_word(s->h_status.p[b], b, "query");
    else if (s->h_qerr.p[b]) st = check_device_flags(s->h_qerr.p[b]);
    if (out_status) {
      out_status[b] = st;
      if (st) out_counts[b] = 0;
    } else if (st) {
      return st;
    }
    if (st && !first) first = st;
  }
  if (!out_status && batch_flags) {   // a flag no query owns (copy time-out)
    hx_status rc = check_device_flags(batch_flags);
    if (rc) return rc;
  }
  if (out_status && batch_flags && !first) {   // batch-level failure with no owner: every query is suspect
    const hx_status rc = check_device_flags(batch_flags);
    if (rc)
      for (size_t b = 0; b < B; ++b) { out_status[b] = rc; out_counts[b] = 0; }
  }
  return HX_OK;
}

static hx_status hx_search_strict(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                  uint64_t* out_ids, float* out_scores, uint32_t* out_counts, hx_stats* stats,
                                  hx_status* out_status = nullptr);
static hx_status hx_search_policy(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                  const hx_policy_params* policy, const uint64_t* query_simhash, uint64_t* out_ids,
                                  float* out_scores, uint32_t* out_counts, hx_stats* stats, hx_policy_stats* pstats,
                                  hx_status* out_status);

extern "C" hx_status hx_search(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                               uint64_t* out_ids, float* out_scores, uint32_t* out_counts, hx_stats* stats) {
  if (p && !(p->simhash_mode == HX_SIMHASH_OFF && !(p->pre_sampling_ratio >= 0.0f && p->pre_sampling_ratio < 1.0f)))
    return hx_search_ex(ix, queries, B, p, nullptr, nullptr, out_ids, out_scores, out_counts, stats, nullptr);
  return hx_search_strict(ix, queries, B, p, out_ids, out_scores, out_counts, stats);
}

// B independent queries with a status PER QUERY (the reference runs one query per call: one invalid query, or one
// query that exhausts a device-side bound, fails alone).  Returns HX_OK whenever the batch itself could be executed.
extern "C" hx_status hx_search_batch(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                     uint64_t* out_ids, float* out_scores, uint32_t* out_counts, hx_status* out_status,
                                     hx_stats* stats) {
  if (B && !out_status) {
    hx_set_error("hx_search_batch: out_status is required");
    return HX_ERR_INVALID_PARAMETER;
  }
  if (p && !(p->simhash_mode == HX_SIMHASH_OFF && !(p->pre_sampling_ratio >= 0.0f && p->pre_sampling_ratio < 1.0f)))
    return hx_search_policy(ix, queries, B, p, nullptr, nullptr, out_ids, out_scores, out_counts, stats, nullptr, out_status);
  return hx_search_strict(ix, queries, B, p, out_ids, out_scores, out_counts, stats, out_status);
}

static hx_status hx_search_strict(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                  uint64_t* out_ids, float* out_scores, uint32_t* out_counts, hx_stats* stats,
                                  hx_status* out_status) {
  if (!ix) {
    hx_set_error("null index handle");
    return HX_ERR_INDEX_NOT_FOUND;
  }
  uint32_t k, ef;
  hx_status rc = check_params(ix, p, &k, &ef);
  if (rc) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (B == 0) return HX_OK;
  if (!queries || !out_ids || !out_scores || !out_counts) {
    hx_set_error("hx_search: null pointer");
    return HX_ERR_INVALID_PARAMETER;
  }
  HX_CUDA(cudaSetDevice(ix->device));
  if (ix->n == 0 || !ix->populated) return answer_empty_index(ix, queries, B, out_counts, out_status);
  HxScratch* s = nullptr;
  if ((rc = hx_acquire_scratch(ix, &s))) return rc;
  ScratchGuard guard{ix, s};
  uint32_t launches = 0;
  // Large batches on the ring build are pipelined: the queries cross PCIe in chunks on a second stream, each chunk followed
  // by a 4-byte copy that publishes how many queries have landed; the search kernel is already running, validates every
  // query itself (no separate k_validate_and_header launch) and only waits for the chunk a query belongs to.
  bool pipelined = B >= 1024 && hnsw_uses_ring(ix, B) && ix->n != 0 && ix->populated;
  pipelined = pipelined && knob(ix->tune.pipeline, 1) != 0;
  HxFusedArgs fz;
  if (pipelined) {
    const uint32_t dim = ix->cfg.dimension;
    if ((rc = hx_finalize_graph(ix))) return rc;
    if (!ix->d_nbr0) pipelined = false;
    if (pipelined) {
      if ((rc = s->d_queries.reserve(B * (size_t)dim))) return rc;
      if ((rc = s->d_qhdr.reserve(B))) return rc;
      if ((rc = s->d_qstatus.reserve(B))) return rc;
      if ((rc = s->d_err.reserve(4))) return rc;
      if (!s->copy_stream) {
        HX_CUDA(cudaStreamCreateWithFlags(&s->copy_stream, cudaStreamNonBlocking));
        HX_CUDA(cudaEventCreateWithFlags(&s->ev_copy, cudaEventDisableTiming));
      }
      const size_t chunks = 8;
      if ((rc = s->h_avail.reserve(chunks))) return rc;
      HX_CUDA(cudaMemsetAsync(s->d_err.p + 2, 0, sizeof(uint32_t), s->stream));
      HX_CUDA(cudaEventRecord(s->ev_copy, s->stream));
      HX_CUDA(cudaStreamWaitEvent(s->copy_stream, s->ev_copy, 0));
      for (size_t c = 0; c < chunks; ++c) {
        const size_t lo = B * c / chunks, hi = B * (c + 1) / chunks;
        if (hi == lo) continue;
        HX_CUDA(cudaMemcpyAsync(s->d_queries.p + lo * dim, queries + lo * dim, (hi - lo) * (size_t)dim * sizeof(float),
                                cudaMemcpyHostToDevice, s->copy_stream));
        s->h_avail.p[c] = (uint32_t)hi;
        HX_CUDA(cudaMemcpyAsync(s->d_err.p + 2, s->h_avail.p + c, sizeof(uint32_t), cudaMemcpyHostToDevice, s->copy_stream));
      }
      fz.avail = s->d_err.p + 2;
      fz.has_limit = component_limit(ix->cfg.metric, dim, &fz.limit) ? 1 : 0;
    }
  }
  if (!pipelined && (rc = stage_queries(ix, s, queries, B, &launches, out_status != nullptr))) return rc;
  if ((rc = s->d_out_ids.reserve(B * (size_t)k))) return rc;
  if ((rc = s->d_out_scores.reserve(B * (size_t)k))) return rc;
  if ((rc = s->d_out_counts.reserve(B))) return rc;
  const bool want_stats = p->collect_stats != 0 && stats != nullptr;
  if (want_stats && (rc = s->d_qstats.reserve(B * 4))) return rc;
  bool timed = false;
  rc = launch_hnsw(ix, s, s->d_queries.p, B, k, ef, s->d_out_ids.p, s->d_out_scores.p, s->d_out_counts.p,
                   want_stats ? s->d_qstats.p : nullptr, s->stream, s->ev0, s->ev1, &timed, &launches,
                   pipelined ? &fz : nullptr);
  if (rc) {
    if (pipelined) cudaStreamSynchronize(s->copy_stream);   // do not leave copies in flight into a released scratch set
    return rc;
  }
  HxDownload dl;
  if ((rc = enqueue_results(s, B, k, out_ids, out_scores, out_counts, &launches, &dl))) return rc;
  if (want_stats) {
    if ((rc = s->h_qstats.reserve(B * 4))) return rc;
    HX_CUDA(cudaMemcpyAsync(s->h_qstats.p, s->d_qstats.p, B * 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  }
  HX_CUDA(cudaStreamSynchronize(s->stream));
  finish_results(s, dl, out_ids, out_scores, out_counts);
  if ((rc = report_batch(s, B, out_counts, out_status))) return rc;
  float ms = 0.f;
  if (timed && cudaEventElapsedTime(&ms, s->ev0, s->ev1) == cudaSuccess) {
    ix->last_kernel_ms = ms;
    ix->last_kernel_launches = 1;
  }
  if (stats) {
    stats->kernel_launches = launches;
    if (want_stats) {
      for (size_t b = 0; b < B; ++b) {
        stats->expansion_steps += s->h_qstats.p[b * 4 + 0];
        stats->neighbors_examined += s->h_qstats.p[b * 4 + 1];
        stats->distance_computations += s->h_qstats.p[b * 4 + 2];
        stats->upper_layer_steps += s->h_qstats.p[b * 4 + 3];
        if (s->h_qstats.p[b * 4 + 2]) stats->vectors_loaded += s->h_qstats.p[b * 4 + 2] - 1;
      }
      stats->algorithmic_bytes = stats->expansion_steps * (5ull + 8ull * ix->lim0) +
                                 stats->distance_computations * (4ull + 4ull * ix->cfg.dimension);
    }
  }
  return HX_OK;
}

extern "C" hx_status hx_search_device(hx_index* ix, const float* d_queries, size_t B, const hx_search_params* p,
                                      uint64_t* d_out_ids, float* d_out_scores, uint32_t* d_out_counts,
                                      void* cuda_stream, hx_stats* stats) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  uint32_t k, ef;
  hx_status rc = check_params(ix, p, &k, &ef);
  if (rc) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (B == 0) return HX_OK;
  if (!d_queries || !d_out_ids || !d_out_scores || !d_out_counts) return HX_ERR_INVALID_PARAMETER;
  if (!params_strict(p)) {
    hx_set_error("the device-buffer entry point executes the strict-exhaustive specialisation only; use hx_search_ex");
    return HX_ERR_UNSUPPORTED;
  }
  HX_CUDA(cudaSetDevice(ix->device));
  HxScratch* s = nullptr;
  cudaStream_t stream = (cudaStream_t)cuda_stream;
  if ((rc = dev_scratch(ix, stream, &s))) return rc;
  uint32_t launches = 0;
  // the ring build validates each query itself (ValidatedMetricVector::try_new + header by the warp that owns it): no
  // separate k_validate_and_header launch in front of it
  HxFusedArgs fz;
  bool fused = false;
  if (hnsw_uses_ring(ix, B) && ix->n != 0 && ix->populated) {
    if ((rc = hx_finalize_graph(ix))) return rc;
    fused = ix->d_nbr0 != nullptr;
  }
  if (fused) {
    if ((rc = s->d_qhdr.reserve(B))) return rc;
    if ((rc = s->d_qstatus.reserve(B))) return rc;
    fz.has_limit = component_limit(ix->cfg.metric, ix->cfg.dimension, &fz.limit) ? 1 : 0;
  } else if ((rc = prepare_device_queries(ix, s, d_queries, B, stream, &launches))) {
    return rc;
  }
  const bool want_stats = p->collect_stats != 0 && stats != nullptr;
  if (want_stats && (rc = s->d_qstats.reserve(B * 4))) return rc;
  cudaEvent_t e0, e1;
  if ((rc = s->ring_next(&e0, &e1))) return rc;
  bool timed = false;
  if ((rc = launch_hnsw(ix, s, d_queries, B, k, ef, d_out_ids, d_out_scores, d_out_counts,
                        want_stats ? s->d_qstats.p : nullptr, stream, e0, e1, &timed, &launches, fused ? &fz : nullptr,
                        /*sticky_flags=*/true)))
    return rc;
  if (!timed && s->ring_pending) s->ring_pending--;
  if (want_stats) {   // stats need a sync; the throughput path leaves collect_stats = 0
    if ((rc = s->h_qstats.reserve(B * 4))) return rc;
    HX_CUDA(cudaMemcpyAsync(s->h_qstats.p, s->d_qstats.p, B * 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    HX_CUDA(cudaStreamSynchronize(stream));
    for (size_t b = 0; b < B; ++b) {
      stats->expansion_steps += s->h_qstats.p[b * 4 + 0];
      stats->neighbors_examined += s->h_qstats.p[b * 4 + 1];
      stats->distance_computations += s->h_qstats.p[b * 4 + 2];
      stats->upper_layer_steps += s->h_qstats.p[b * 4 + 3];
      if (s->h_qstats.p[b * 4 + 2]) stats->vectors_loaded += s->h_qstats.p[b * 4 + 2] - 1;
    }
    stats->algorithmic_bytes = stats->expansion_steps * (5ull + 8ull * ix->lim0) +
                               stats->distance_computations * (4ull + 4ull * ix->cfg.dimension);
  }
  if (stats) stats->kernel_launches = launches;
  return HX_OK;
}

// Error flags raised by the device-buffer calls issued on `cuda_stream` since the previous hx_device_flags on that
// stream (ORed over launches; synchronises the stream; clears the word).  *out_status = the HelixDbError the flags map to.
extern "C" hx_status hx_device_flags(hx_index* ix, void* cuda_stream, uint32_t* out_flags, hx_status* out_status) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  HX_CUDA(cudaSetDevice(ix->device));
  cudaStream_t stream = (cudaStream_t)cuda_stream;
  HxScratch* s = nullptr;
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    auto it = ix->dev_scratch.find(stream);
    if (it != ix->dev_scratch.end()) s = it->second;
  }
  uint32_t flags = 0;
  if (s && s->d_err.p) {
    HX_CUDA(cudaMemcpyAsync(&flags, s->d_err.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    HX_CUDA(cudaMemsetAsync(s->d_err.p, 0, sizeof(uint32_t), stream));
    HX_CUDA(cudaStreamSynchronize(stream));
  } else {
    HX_CUDA(cudaStreamSynchronize(stream));
  }
  if (out_flags) *out_flags = flags;
  if (out_status) *out_status = check_device_flags(flags);
  return HX_OK;
}

// ------------------------------------------------------------------------------------------------
// restricted search
// ------------------------------------------------------------------------------------------------
extern "C" int32_t hx_restricted_plan(uint64_t n_candidates, uint32_t dimension) {
  // EXACT_CARDINALITY_THRESHOLD = 256, EXACT_VECTOR_BYTES_THRESHOLD = 4 MiB (restricted.rs:40-42,433-440)
  const uint64_t bytes = n_candidates * (uint64_t)dimension * 4ull;
  return (n_candidates <= 256 && bytes <= 4ull * 1024 * 1024) ? 0 : 1;
}

static uint32_t pick_chunk(uint64_t total_cands, int sm_count) {
  // aim for ~8 waves of CTAs (4 resident per SM) so the last partial wave costs little; one CTA pass covers 32 rows
  uint64_t c = total_cands / ((uint64_t)sm_count * 4 * 8) + 1;
  c = (c + 31) / 32 * 32;
  if (c < 32) c = 32;
  if (c > 2048) c = 2048;
  return (uint32_t)c;
}

// d_cand_slots / d_cand_offsets on the device; host knows max candidate count per query and the total.
struct HxSetRefs {   // device arrays describing one device-resident candidate set per query
  const uint32_t* const* q_slots = nullptr;
  const uint64_t* q_len = nullptr;
  const uint64_t* q_keyoff = nullptr;
};

static hx_status launch_scan_select(hx_index* ix, HxScratch* s, const float* d_queries, size_t B, uint32_t k,
                                    const uint32_t* d_slots, const uint64_t* d_offsets, bool shared, uint64_t n_shared,
                                    uint64_t max_cands, uint64_t total_keys, uint64_t* d_out_ids, float* d_out_scores,
                                    uint32_t* d_out_counts, cudaStream_t stream, cudaEvent_t e0, cudaEvent_t e1,
                                    uint32_t* launches, const HxSetRefs* sets = nullptr, const float* q_hdr = nullptr,
                                    const uint32_t* q_status = nullptr) {
  hx_status rc;
  if (!q_hdr) q_hdr = s->d_qhdr.p;   // headers / status words of the B queries (default: the call's staged queries)
  if (!q_status) q_status = s->d_qstatus.p;
  if ((rc = s->d_err.reserve(1))) return rc;
  HX_CUDA(cudaMemsetAsync(s->d_err.p, 0, sizeof(uint32_t), stream));
  const HxDev dev = ix->dev();
  // k <= 32 (the reference's default k = 10): ONE launch — scores reduced to the top k by warp shuffles inside the scan
  // kernel, the last CTA of each query merges the per-CTA lists; no key array in HBM, no k_select launch
  const uint32_t chunk_pick = pick_chunk(total_keys, ix->sm_count);
  const uint32_t n_chunks = (uint32_t)((max_cands + chunk_pick - 1) / chunk_pick);
  const bool fused_off = knob(ix->tune.scan_fused, 1) == 0;
  const bool fused_topk = !fused_off && k <= HX_TOPK && ix->cfg.metric != HX_METRIC_MANHATTAN && B <= 65535 &&
                          (size_t)B * n_chunks * HX_TOPK * 8 <= (256ull << 20);
  if (fused_topk) {
    if ((rc = s->d_partial.reserve((size_t)B * n_chunks * HX_TOPK))) return rc;
    if (s->tickets_zeroed < B || !s->d_tickets.p) {
      if ((rc = s->d_tickets.reserve(B))) return rc;
      HX_CUDA(cudaMemsetAsync(s->d_tickets.p, 0, s->d_tickets.cap * sizeof(uint32_t), stream));
      s->tickets_zeroed = s->d_tickets.cap;
    }
    HxScanArgs a{};
    a.queries = d_queries;
    a.q_hdr = q_hdr;
    a.q_status = q_status;
    a.B = (uint32_t)B;
    a.cand_slots = d_slots;
    a.cand_offsets = d_offsets;
    a.shared_set = shared ? 1u : 0u;
    a.n_shared = n_shared;
    a.chunk = chunk_pick;
    a.err_flags = s->d_err.p;
    if (sets) { a.q_slots = sets->q_slots; a.q_len = sets->q_len; a.q_keyoff = sets->q_keyoff; }
    HxTopkArgs tk{};
    tk.partial = s->d_partial.p;
    tk.tickets = s->d_tickets.p;
    tk.n_chunks = n_chunks;
    tk.k = k;
    tk.out_ids = d_out_ids;
    tk.out_scores = d_out_scores;
    tk.out_counts = d_out_counts;
    dim3 grid(n_chunks, (unsigned)B);
    const uint32_t smem = ix->ld * 4u;
    HX_CUDA(cudaEventRecord(e0, stream));
    if (ix->cfg.metric == HX_METRIC_EUCLIDEAN) {
      if (smem > 48 * 1024) HX_CUDA(cudaFuncSetAttribute(k_scan_topk<HXM_EUCLIDEAN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      k_scan_topk<HXM_EUCLIDEAN><<<grid, HX_SCAN_THREADS, smem, stream>>>(dev, a, tk);
    } else {
      if (smem > 48 * 1024) HX_CUDA(cudaFuncSetAttribute(k_scan_topk<HXM_COSINE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      k_scan_topk<HXM_COSINE><<<grid, HX_SCAN_THREADS, smem, stream>>>(dev, a, tk);
    }
    HX_CUDA(cudaGetLastError());
    HX_CUDA(cudaEventRecord(e1, stream));
    (*launches)++;
    return HX_OK;
  }
  if ((rc = s->d_keys.reserve(total_keys))) return rc;
  HxScanArgs a{};
  a.queries = d_queries;
  a.q_hdr = q_hdr;
  a.q_status = q_status;
  a.B = (uint32_t)B;
  a.cand_slots = d_slots;
  a.cand_offsets = d_offsets;
  a.keys = s->d_keys.p;
  a.shared_set = shared ? 1u : 0u;
  a.n_shared = n_shared;
  a.chunk = pick_chunk(total_keys, ix->sm_count);
  a.err_flags = s->d_err.p;
  if (sets) { a.q_slots = sets->q_slots; a.q_len = sets->q_len; a.q_keyoff = sets->q_keyoff; }
  dim3 grid((unsigned)((max_cands + a.chunk - 1) / a.chunk), (unsigned)std::min<size_t>(B, 65535));
  const uint32_t smem = ix->ld * 4u;
  HX_CUDA(cudaEventRecord(e0, stream));
  switch (ix->cfg.metric) {
    case HX_METRIC_EUCLIDEAN:
      if (smem > 48 * 1024)
        HX_CUDA(cudaFuncSetAttribute(k_scan<HXM_EUCLIDEAN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      k_scan<HXM_EUCLIDEAN><<<grid, HX_SCAN_THREADS, smem, stream>>>(dev, a);
      break;
    case HX_METRIC_COSINE:
      if (smem > 48 * 1024)
        HX_CUDA(cudaFuncSetAttribute(k_scan<HXM_COSINE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      k_scan<HXM_COSINE><<<grid, HX_SCAN_THREADS, smem, stream>>>(dev, a);
      break;
    default:
      if (smem > 48 * 1024)
        HX_CUDA(cudaFuncSetAttribute(k_scan<HXM_MANHATTAN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      k_scan<HXM_MANHATTAN><<<grid, HX_SCAN_THREADS, smem, stream>>>(dev, a);
      break;
  }
  HX_CUDA(cudaGetLastError());
  HX_CUDA(cudaEventRecord(e1, stream));
  (*launches)++;
  HxSelectArgs sa{};
  sa.keys = s->d_keys.p;
  sa.cand_slots = d_slots;
  sa.cand_offsets = d_offsets;
  sa.q_status = q_status;
  sa.B = (uint32_t)B;
  sa.k = k;
  sa.shared_set = shared ? 1u : 0u;
  sa.n_shared = n_shared;
  sa.out_ids = d_out_ids;
  sa.out_scores = d_out_scores;
  sa.out_counts = d_out_counts;
  if (sets) { sa.q_slots = sets->q_slots; sa.q_len = sets->q_len; sa.q_keyoff = sets->q_keyoff; }
  k_select<<<(unsigned)std::min<size_t>(B, 65535), HX_SEL_THREADS, 0, stream>>>(dev, sa);
  HX_CUDA(cudaGetLastError());
  (*launches)++;
  return HX_OK;
}

static hx_status restricted_host(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                 const uint64_t* cand_ids, const uint64_t* cand_offsets, size_t n_shared, bool shared,
                                 uint64_t* out_ids, float* out_scores, uint32_t* out_counts, hx_stats* stats) {
  if (!ix) {
    hx_set_error("null index handle");
    return HX_ERR_INDEX_NOT_FOUND;
  }
  uint32_t k, ef;
  hx_status rc = check_params(ix, p, &k, &ef);
  if (rc) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (B == 0) return HX_OK;
  if (!queries || !out_ids || !out_scores || !out_counts) return HX_ERR_INVALID_PARAMETER;
  // candidate-set admission (restricted.rs:356-371, 200-213): |C| <= 1e6; k' = min(k,|C|) <= 800
  uint64_t total = 0, max_c = 0;
  bool any_nonempty = false;
  for (size_t b = 0; b < B; ++b) {
    const uint64_t c = shared ? n_shared : cand_offsets[b + 1] - cand_offsets[b];
    if (c > 1000000ull) {
      hx_set_error("restricted vector search accepts at most 1000000 unique candidates");
      return HX_ERR_QUERY;
    }
    if (c > 0) {
      any_nonempty = true;
      if (std::min<uint64_t>(k, c) > 800) {
        hx_set_error("restricted vector search result count must be at most 800, got %llu",
                     (unsigned long long)std::min<uint64_t>(k, c));
        return HX_ERR_QUERY;
      }
    }
    max_c = std::max(max_c, c);
    total += shared ? 0 : c;
    if (shared) break;
  }
  if (shared) total = n_shared;
  if (!any_nonempty || total == 0) {   // RestrictedVectorCandidates::Empty => Ok(vec![]) before any I/O (:539-541)
    for (size_t b = 0; b < B; ++b) out_counts[b] = 0;
    return HX_OK;
  }
  if ((shared && !cand_ids) || (!shared && (!cand_ids || !cand_offsets))) return HX_ERR_INVALID_PARAMETER;
  // RoaringTreemap iteration order: ascending and unique within a set (the (score,id) tie rule and the "no duplicate
  // results" guarantee depend on it; hx_candidates_create checks the same)
  for (size_t b = 0; b < (shared ? 1 : B); ++b) {
    const uint64_t lo = shared ? 0 : cand_offsets[b], hi = shared ? n_shared : cand_offsets[b + 1];
    for (uint64_t i = lo + 1; i < hi; ++i)
      if (cand_ids[i] <= cand_ids[i - 1]) {
        hx_set_error("candidate ids must be ascending and unique (RoaringTreemap iteration order); set %zu position %llu",
                     b, (unsigned long long)(i - lo));
        return HX_ERR_INVALID_PARAMETER;
      }
  }
  HX_CUDA(cudaSetDevice(ix->device));
  if (ix->n == 0 || !ix->populated)   // empty index => Ok(vec![]) after query validation (:563-566)
    return answer_empty_index(ix, queries, B, out_counts, nullptr);
  HxScratch* s = nullptr;
  if ((rc = hx_acquire_scratch(ix, &s))) return rc;
  ScratchGuard guard{ix, s};
  uint32_t launches = 0;
  if ((rc = stage_queries(ix, s, queries, B, &launches))) return rc;
  if ((rc = s->d_cand_ids.reserve(total))) return rc;
  if ((rc = s->d_cand_slots.reserve(total))) return rc;
  if ((rc = s->d_cand_offsets.reserve(B + 1))) return rc;
  HX_CUDA(cudaMemcpyAsync(s->d_cand_ids.p, cand_ids + (shared ? 0 : cand_offsets[0]), total * sizeof(uint64_t),
                          cudaMemcpyHostToDevice, s->stream));
  if (!shared) {
    if ((rc = s->h_cand_offsets.reserve(B + 1))) return rc;
    for (size_t b = 0; b <= B; ++b) s->h_cand_offsets.p[b] = cand_offsets[b] - cand_offsets[0];
    HX_CUDA(cudaMemcpyAsync(s->d_cand_offsets.p, s->h_cand_offsets.p, (B + 1) * sizeof(uint64_t),
                            cudaMemcpyHostToDevice, s->stream));
  }
  k_map_candidates<<<(unsigned)((total + 255) / 256), 256, 0, s->stream>>>(
      ix->d_ids, (uint32_t)ix->n, s->d_cand_ids.p, total, s->d_cand_slots.p, ix->contiguous ? 1 : 0, ix->first_id, ix->d_deleted);
  HX_CUDA(cudaGetLastError());
  launches++;
  if ((rc = s->d_out_ids.reserve(B * (size_t)k))) return rc;
  if ((rc = s->d_out_scores.reserve(B * (size_t)k))) return rc;
  if ((rc = s->d_out_counts.reserve(B))) return rc;
  const uint64_t total_keys = shared ? (uint64_t)B * n_shared : total;
  if ((rc = launch_scan_select(ix, s, s->d_queries.p, B, k, s->d_cand_slots.p, s->d_cand_offsets.p, shared, n_shared,
                               max_c, total_keys, s->d_out_ids.p, s->d_out_scores.p, s->d_out_counts.p, s->stream,
                               s->ev0, s->ev1, &launches)))
    return rc;
  if ((rc = s->h_status.reserve(B))) return rc;
  if ((rc = s->h_err.reserve(1))) return rc;
  HX_CUDA(cudaMemcpyAsync(out_ids, s->d_out_ids.p, B * (size_t)k * sizeof(uint64_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(out_scores, s->d_out_scores.p, B * (size_t)k * sizeof(float), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(out_counts, s->d_out_counts.p, B * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(s->h_status.p, s->d_qstatus.p, B * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(s->h_err.p, s->d_err.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaStreamSynchronize(s->stream));
  for (size_t b = 0; b < B; ++b)
    if (s->h_status.p[b] != HX_ST_OK) return status_from_word(s->h_status.p[b], b, "query");
  if ((rc = check_device_flags(s->h_err.p[0]))) return rc;
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, s->ev0, s->ev1) == cudaSuccess) {
    ix->last_kernel_ms = ms;
    ix->last_kernel_launches = 1;
  }
  if (stats) {
    stats->kernel_launches = launches;
    stats->distance_computations = total_keys;
    stats->vectors_loaded = total_keys;
    stats->algorithmic_bytes = total_keys * (4ull * ix->cfg.dimension + (ix->cfg.metric == HX_METRIC_COSINE ? 4 : 0));
  }
  return HX_OK;
}

extern "C" hx_status hx_search_restricted(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                          const uint64_t* cand_ids, size_t n_cand, uint64_t* out_ids,
                                          float* out_scores, uint32_t* out_counts, hx_stats* stats) {
  return restricted_host(ix, queries, B, p, cand_ids, nullptr, n_cand, true, out_ids, out_scores, out_counts, stats);
}

extern "C" hx_status hx_search_restricted_multi(hx_index* ix, const float* queries, size_t B,
                                                const hx_search_params* p, const uint64_t* cand_ids,
                                                const uint64_t* cand_offsets, uint64_t* out_ids, float* out_scores,
                                                uint32_t* out_counts, hx_stats* stats) {
  if (B && !cand_offsets) return HX_ERR_INVALID_PARAMETER;
  return restricted_host(ix, queries, B, p, cand_ids, cand_offsets, 0, false, out_ids, out_scores, out_counts, stats);
}

// ---- device-resident candidate sets ------------------------------------------------------------------------------------------
// The reference's label / equality indexes are RoaringTreemap values keyed by the snapshot (encoding/v1/indexes/label.rs:10-14);
// a prefilter that is reused across queries need not cross PCIe as 8 bytes per candidate on every call: the ids are uploaded and
// mapped to slots once (ids without a vector row dropped, restricted.rs:615-659) and queries then name the set.
struct hx_candidates {
  hx_index* ix = nullptr;
  uint32_t* d_slots = nullptr;   // ascending; HX_ABSENT for ids without a vector row (never results)
  uint64_t n = 0;
  uint64_t generation = 0;
  std::atomic<HxResident*> resident{nullptr};   // hx_candidates_make_resident: the tensor-core view, kept across calls
  std::mutex resident_mu;                       // serialises the build; the view is published complete
};

extern "C" hx_status hx_candidates_create(hx_index* ix, const uint64_t* cand_ids, size_t n, hx_candidates** out) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (!out || (n && !cand_ids)) return HX_ERR_INVALID_PARAMETER;
  *out = nullptr;
  if (n > 1000000ull) {   // RestrictedVectorCandidates::from_ids (restricted.rs:356-371)
    hx_set_error("restricted vector search accepts at most 1000000 unique candidates");
    return HX_ERR_QUERY;
  }
  for (size_t i = 1; i < n; ++i)
    if (cand_ids[i] <= cand_ids[i - 1]) {
      hx_set_error("candidate ids must be ascending and unique (RoaringTreemap iteration order)");
      return HX_ERR_INVALID_PARAMETER;
    }
  HX_CUDA(cudaSetDevice(ix->device));
  hx_candidates* c = new hx_candidates();
  c->ix = ix;
  c->n = n;
  c->generation = ix->vector_generation;
  if (n) {
    uint64_t* d_ids = nullptr;
    cudaError_t e = cudaMalloc((void**)&d_ids, n * sizeof(uint64_t));
    if (e == cudaSuccess) e = cudaMalloc((void**)&c->d_slots, n * sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMemcpy(d_ids, cand_ids, n * sizeof(uint64_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
      k_map_candidates<<<(unsigned)((n + 255) / 256), 256>>>(ix->d_ids, (uint32_t)ix->n, d_ids, n, c->d_slots,
                                                             ix->contiguous ? 1 : 0, ix->first_id, ix->d_deleted);
      e = cudaDeviceSynchronize();
    }
    if (d_ids) cudaFree(d_ids);
    if (e != cudaSuccess) {
      hx_set_error("candidate set upload failed: %s", cudaGetErrorString(e));
      if (c->d_slots) cudaFree(c->d_slots);
      delete c;
      return e == cudaErrorMemoryAllocation ? HX_ERR_OUT_OF_MEMORY : HX_ERR_CUDA;
    }
  }
  *out = c;
  return HX_OK;
}

extern "C" void hx_candidates_destroy(hx_candidates* c) {
  if (!c) return;
  if (c->d_slots || c->resident.load()) cudaSetDevice(c->ix->device);
  if (c->d_slots) cudaFree(c->d_slots);
  hx_resident_free(c->resident.load());
  delete c;
}

extern "C" uint64_t hx_candidates_len(const hx_candidates* c) { return c ? c->n : 0; }

extern "C" hx_status hx_candidates_make_resident(hx_index* ix, hx_candidates* set) {
  if (!ix || !set) {
    hx_set_error("hx_candidates_make_resident: null argument");
    return HX_ERR_INVALID_PARAMETER;
  }
  if (ix->cfg.metric == HX_METRIC_MANHATTAN) {
    hx_set_error("the L1 metric is not a contraction: a candidate set of an L1 index has no tensor-core view");
    return HX_ERR_UNSUPPORTED;
  }
  if (set->ix != ix || set->generation != ix->vector_generation) {
    hx_set_error("candidate set does not belong to this index image (vectors were reloaded or deleted?)");
    return HX_ERR_INVARIANT_VIOLATION;
  }
  std::lock_guard<std::mutex> lk(set->resident_mu);
  if (set->resident.load()) return HX_OK;
  HX_CUDA(cudaSetDevice(ix->device));
  HxResident* r = nullptr;
  hx_status rc = hx_resident_build(ix, set->d_slots, set->n, &r);
  if (rc) return rc;
  set->resident.store(r);
  return HX_OK;
}

extern "C" uint64_t hx_candidates_resident_bytes(const hx_candidates* set) {
  const HxResident* r = set ? set->resident.load() : nullptr;
  return r ? r->bytes : 0;
}

extern "C" hx_status hx_search_restricted_sets(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                               hx_candidates* const* sets, size_t n_sets, uint64_t* out_ids,
                                               float* out_scores, uint32_t* out_counts, hx_stats* stats) {
  if (!ix) {
    hx_set_error("null index handle");
    return HX_ERR_INDEX_NOT_FOUND;
  }
  uint32_t k, ef;
  hx_status rc = check_params(ix, p, &k, &ef);
  if (rc) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (B == 0) return HX_OK;
  if (!queries || !out_ids || !out_scores || !out_counts || !sets || (n_sets != 1 && n_sets != B)) {
    hx_set_error("hx_search_restricted_sets: one set for all queries or one per query");
    return HX_ERR_INVALID_PARAMETER;
  }
  uint64_t total_keys = 0, max_c = 0;
  for (size_t b = 0; b < B; ++b) {
    const hx_candidates* c = sets[n_sets == 1 ? 0 : b];
    if (!c || c->ix != ix || c->generation != ix->vector_generation) {
      hx_set_error("candidate set %zu does not belong to this index image (vectors were reloaded?)", b);
      return HX_ERR_INVARIANT_VIOLATION;
    }
    if (c->n > 0 && std::min<uint64_t>(k, c->n) > 800) {   // RestrictedResultCount (restricted.rs:200-213)
      hx_set_error("restricted vector search result count must be at most 800, got %llu",
                   (unsigned long long)std::min<uint64_t>(k, c->n));
      return HX_ERR_QUERY;
    }
    total_keys += c->n;
    max_c = std::max<uint64_t>(max_c, c->n);
  }
  if (total_keys == 0) {
    for (size_t b = 0; b < B; ++b) out_counts[b] = 0;
    return HX_OK;
  }
  HX_CUDA(cudaSetDevice(ix->device));
  if (ix->n == 0 || !ix->populated) return answer_empty_index(ix, queries, B, out_counts, nullptr);
  HxScratch* s = nullptr;
  if ((rc = hx_acquire_scratch(ix, &s))) return rc;
  ScratchGuard guard{ix, s};
  uint32_t launches = 0;
  if ((rc = stage_queries(ix, s, queries, B, &launches))) return rc;
  // per-query (pointer, length, key offset): 24 bytes per query over PCIe instead of 8 bytes per candidate
  if ((rc = s->h_cand_offsets.reserve(3 * B))) return rc;
  if ((rc = s->d_cand_offsets.reserve(3 * B))) return rc;
  uint64_t koff = 0;
  for (size_t b = 0; b < B; ++b) {
    const hx_candidates* c = sets[n_sets == 1 ? 0 : b];
    s->h_cand_offsets.p[b] = (uint64_t)(uintptr_t)c->d_slots;
    s->h_cand_offsets.p[B + b] = c->n;
    s->h_cand_offsets.p[2 * B + b] = koff;
    koff += c->n;
  }
  HX_CUDA(cudaMemcpyAsync(s->d_cand_offsets.p, s->h_cand_offsets.p, 3 * B * sizeof(uint64_t), cudaMemcpyHostToDevice,
                          s->stream));
  HxSetRefs refs;
  refs.q_slots = reinterpret_cast<const uint32_t* const*>(s->d_cand_offsets.p);
  refs.q_len = s->d_cand_offsets.p + B;
  refs.q_keyoff = s->d_cand_offsets.p + 2 * B;
  if ((rc = s->d_out_ids.reserve(B * (size_t)k))) return rc;
  if ((rc = s->d_out_scores.reserve(B * (size_t)k))) return rc;
  if ((rc = s->d_out_counts.reserve(B))) return rc;
  if ((rc = launch_scan_select(ix, s, s->d_queries.p, B, k, nullptr, nullptr, false, 0, max_c, total_keys, s->d_out_ids.p,
                               s->d_out_scores.p, s->d_out_counts.p, s->stream, s->ev0, s->ev1, &launches, &refs)))
    return rc;
  if ((rc = s->h_status.reserve(B))) return rc;
  if ((rc = s->h_err.reserve(1))) return rc;
  HX_CUDA(cudaMemcpyAsync(out_ids, s->d_out_ids.p, B * (size_t)k * sizeof(uint64_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(out_scores, s->d_out_scores.p, B * (size_t)k * sizeof(float), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(out_counts, s->d_out_counts.p, B * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(s->h_status.p, s->d_qstatus.p, B * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(s->h_err.p, s->d_err.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaStreamSynchronize(s->stream));
  for (size_t b = 0; b < B; ++b)
    if (s->h_status.p[b] != HX_ST_OK) return status_from_word(s->h_status.p[b], b, "query");
  if ((rc = check_device_flags(s->h_err.p[0]))) return rc;
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, s->ev0, s->ev1) == cudaSuccess) {
    ix->last_kernel_ms = ms;
    ix->last_kernel_launches = 1;
  }
  if (stats) {
    stats->kernel_launches = launches;
    stats->distance_computations = total_keys;
    stats->vectors_loaded = total_keys;
    stats->algorithmic_bytes = total_keys * (4ull * ix->cfg.dimension + (ix->cfg.metric == HX_METRIC_COSINE ? 4 : 0));
  }
  return HX_OK;
}

extern "C" hx_status hx_map_candidates_device(hx_index* ix, const uint64_t* d_cand_ids, uint64_t n,
                                              uint32_t* d_out_slots, uint64_t* d_out_count, void* cuda_stream) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (n == 0) return HX_OK;
  HX_CUDA(cudaSetDevice(ix->device));
  k_map_candidates<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>(
      ix->d_ids, (uint32_t)ix->n, d_cand_ids, n, d_out_slots, ix->contiguous ? 1 : 0, ix->first_id, ix->d_deleted);
  HX_CUDA(cudaGetLastError());
  (void)d_out_count;
  return HX_OK;
}

extern "C" hx_status hx_search_restricted_device(hx_index* ix, const float* d_queries, size_t B,
                                                 const hx_search_params* p, const uint32_t* d_cand_slots,
                                                 const uint64_t* d_cand_offsets, uint64_t total_cands,
                                                 uint64_t max_cands_per_query, uint64_t* d_out_ids,
                                                 float* d_out_scores, uint32_t* d_out_counts, void* cuda_stream) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  uint32_t k, ef;
  hx_status rc = check_params(ix, p, &k, &ef);
  if (rc) return rc;
  if (B == 0) return HX_OK;
  if (!d_queries || !d_out_ids || !d_out_scores || !d_out_counts) return HX_ERR_INVALID_PARAMETER;
  const bool shared = d_cand_offsets == nullptr;
  const uint64_t max_c = shared ? total_cands : (max_cands_per_query ? max_cands_per_query : total_cands);
  if (max_c > 1000000ull) {
    hx_set_error("restricted vector search accepts at most 1000000 unique candidates");
    return HX_ERR_QUERY;
  }
  if (std::min<uint64_t>(k, max_c) > 800) {
    hx_set_error("restricted vector search result count must be at most 800");
    return HX_ERR_QUERY;
  }
  HX_CUDA(cudaSetDevice(ix->device));
  cudaStream_t stream = (cudaStream_t)cuda_stream;
  if (total_cands == 0 || ix->n == 0 || !ix->populated) {
    HX_CUDA(cudaMemsetAsync(d_out_counts, 0, B * sizeof(uint32_t), stream));
    return HX_OK;
  }
  if (!d_cand_slots) return HX_ERR_INVALID_PARAMETER;
  HxScratch* s = nullptr;
  if ((rc = dev_scratch(ix, stream, &s))) return rc;
  uint32_t launches = 0;
  if ((rc = prepare_device_queries(ix, s, d_queries, B, stream, &launches))) return rc;
  const uint64_t total_keys = shared ? (uint64_t)B * total_cands : total_cands;
  cudaEvent_t e0, e1;
  if ((rc = s->ring_next(&e0, &e1))) return rc;
  return launch_scan_select(ix, s, d_queries, B, k, d_cand_slots, d_cand_offsets, shared, total_cands, max_c,
                            total_keys, d_out_ids, d_out_scores, d_out_counts, stream, e0, e1, &launches);
}

// ------------------------------------------------------------------------------------------------
// sharded merge, dense path, timing
// ------------------------------------------------------------------------------------------------
extern "C" hx_status hx_merge_topk_device(int32_t device, const uint64_t* d_all_ids, const float* d_all_scores,
                                          const uint32_t* d_all_counts, uint32_t n_shards, size_t B, uint32_t k,
                                          uint64_t* d_out_ids, float* d_out_scores, uint32_t* d_out_counts,
                                          void* cuda_stream) {
  if (n_shards == 0 || n_shards > 128 || k == 0) {
    hx_set_error("hx_merge_topk_device: n_shards must be in 1..128 and k > 0");
    return HX_ERR_INVALID_PARAMETER;
  }
  if (B == 0) return HX_OK;
  HX_CUDA(cudaSetDevice(device));
  k_merge_topk<<<(unsigned)((B + 7) / 8), 256, 0, (cudaStream_t)cuda_stream>>>(
      reinterpret_cast<const unsigned char*>(d_all_ids), reinterpret_cast<const unsigned char*>(d_all_scores),
      reinterpret_cast<const unsigned char*>(d_all_counts), B * (size_t)k * 8, B * (size_t)k * 4, B * 4, n_shards, B, k, k,
      d_out_ids, d_out_scores, d_out_counts);
  HX_CUDA(cudaGetLastError());
  return HX_OK;
}

extern "C" hx_status hx_search_dense(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                     uint64_t* out_ids, float* out_scores, uint32_t* out_counts, hx_stats* stats) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  HX_CUDA(cudaSetDevice(ix->device));
  return hx_dense_impl(ix, queries, B, p, out_ids, out_scores, out_counts, stats);
}

extern "C" hx_status hx_search_dense_exact(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                           uint64_t* out_ids, float* out_scores, uint32_t* out_counts, uint8_t* out_how,
                                           hx_stats* stats) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  HX_CUDA(cudaSetDevice(ix->device));
  return hx_dense_impl(ix, queries, B, p, out_ids, out_scores, out_counts, stats, true, out_how);
}

// rescan, step 1: flagged query j (query flagged[j] of the call) -> row j of a contiguous batch, with its header and status
// word.  One warp per flagged query.
static __global__ void k_dense_gather(const float* __restrict__ q, const float* __restrict__ hdr,
                                      const uint32_t* __restrict__ status, const uint32_t* __restrict__ flagged, size_t F,
                                      uint32_t dim, float* __restrict__ gq, float* __restrict__ ghdr,
                                      uint32_t* __restrict__ gstatus) {
  const size_t j = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31u;
  if (j >= F) return;
  const size_t b = flagged[j];
  for (uint32_t i = lane; i < dim; i += 32) gq[j * dim + i] = q[b * dim + i];
  if (lane == 0) {
    ghdr[j] = hdr[b];
    gstatus[j] = status[b];
  }
}

// rescan, step 3: the exact answer of flagged query j replaces the output row of query flagged[j]
static __global__ void k_dense_scatter(const uint64_t* __restrict__ gids, const float* __restrict__ gsc,
                                       const uint32_t* __restrict__ gcnt, const uint32_t* __restrict__ flagged, size_t F,
                                       uint32_t k, uint64_t* __restrict__ ids, float* __restrict__ sc, uint32_t* __restrict__ cnt) {
  const size_t j = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31u;
  if (j >= F) return;
  const size_t b = flagged[j];
  const uint32_t c = gcnt[j];
  for (uint32_t i = lane; i < c; i += 32) {
    ids[b * k + i] = gids[j * k + i];
    sc[b * k + i] = gsc[j * k + i];
  }
  if (lane == 0) cnt[b] = c;
}

hx_status hx_dense_rescan(hx_index* ix, HxScratch* s, const float* d_q, uint32_t k, const uint32_t* slots,
                          size_t n_view, const HxDenseCert& cert, uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt,
                          cudaStream_t stream, cudaEvent_t e0, cudaEvent_t e1, uint32_t* launches, size_t* n_flagged,
                          uint32_t* err_before) {
  hx_status rc;
  if ((rc = s->h_x.reserve(2)) || (rc = s->d_err.reserve(1))) return rc;
  HX_CUDA(cudaMemcpyAsync(s->h_x.p, cert.n_flagged, 4, cudaMemcpyDeviceToHost, stream));
  HX_CUDA(cudaMemcpyAsync(s->h_x.p + 1, s->d_err.p, 4, cudaMemcpyDeviceToHost, stream));
  HX_CUDA(cudaStreamSynchronize(stream));
  const size_t F = s->h_x.p[0];
  *n_flagged = F;
  *err_before = s->h_x.p[1];
  if (F == 0) return HX_OK;
  const uint32_t dim = ix->cfg.dimension;
  if ((rc = s->x_queries.reserve(F * (size_t)dim)) || (rc = s->x_hdr.reserve(F)) || (rc = s->x_status.reserve(F)) ||
      (rc = s->x_ids.reserve(F * (size_t)k)) || (rc = s->x_scores.reserve(F * (size_t)k)) || (rc = s->x_counts.reserve(F)))
    return rc;
  const unsigned grid = (unsigned)((F + 7) / 8);
  k_dense_gather<<<grid, 256, 0, stream>>>(d_q, s->d_qhdr.p, s->d_qstatus.p, cert.flagged, F, dim, s->x_queries.p,
                                           s->x_hdr.p, s->x_status.p);
  HX_CUDA(cudaGetLastError());
  ++*launches;
  if ((rc = launch_scan_select(ix, s, s->x_queries.p, F, k, slots, nullptr, true, n_view, n_view, (uint64_t)F * n_view,
                               s->x_ids.p, s->x_scores.p, s->x_counts.p, stream, e0, e1, launches, nullptr, s->x_hdr.p,
                               s->x_status.p)))
    return rc;
  k_dense_scatter<<<grid, 256, 0, stream>>>(s->x_ids.p, s->x_scores.p, s->x_counts.p, cert.flagged, F, k, d_out_ids, d_out_sc,
                                            d_out_cnt);
  HX_CUDA(cudaGetLastError());
  ++*launches;
  return HX_OK;
}

// The dense path over one candidate set shared by the B queries: host ids (`cand_ids`, n_cand) or a device set (`set`).
// Admission is restricted_host's, in its order, with the dense path's metric check before anything about the set.
// `exact` (hx_search_dense_restricted_exact[_set]): the certificate follows the re-rank and the queries it cannot clear are
// rescanned over the present slots; out_how (may be null) as hx_search_dense_exact's.
static hx_status dense_restricted_host(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                       const uint64_t* cand_ids, size_t n_cand, const hx_candidates* set, bool is_set,
                                       uint64_t* out_ids, float* out_scores, uint32_t* out_counts, hx_stats* stats,
                                       bool exact = false, uint8_t* out_how = nullptr) {
  if (!ix) {
    hx_set_error("null index handle");
    return HX_ERR_INDEX_NOT_FOUND;
  }
  uint32_t k, ef;
  hx_status rc = check_params(ix, p, &k, &ef);
  if (rc) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (B == 0) return HX_OK;
  if (!queries || !out_ids || !out_scores || !out_counts || (is_set ? !set : (n_cand && !cand_ids))) return HX_ERR_INVALID_PARAMETER;
  if (ix->cfg.metric == HX_METRIC_MANHATTAN) {
    hx_set_error("the L1 metric is not a contraction: use hx_search_restricted");
    return HX_ERR_UNSUPPORTED;
  }
  if (exact && out_how) memset(out_how, 2, B);
  const uint64_t n = is_set ? set->n : n_cand;
  if (n > 1000000ull) {
    hx_set_error("restricted vector search accepts at most 1000000 unique candidates");
    return HX_ERR_QUERY;
  }
  if (n == 0) {   // RestrictedVectorCandidates::Empty => Ok(vec![]) before any I/O
    for (size_t b = 0; b < B; ++b) out_counts[b] = 0;
    return HX_OK;
  }
  if (std::min<uint64_t>(k, n) > 800) {
    hx_set_error("restricted vector search result count must be at most 800, got %llu",
                 (unsigned long long)std::min<uint64_t>(k, n));
    return HX_ERR_QUERY;
  }
  if (!is_set)
    for (uint64_t i = 1; i < n; ++i)
      if (cand_ids[i] <= cand_ids[i - 1]) {
        hx_set_error("candidate ids must be ascending and unique (RoaringTreemap iteration order); position %llu",
                     (unsigned long long)i);
        return HX_ERR_INVALID_PARAMETER;
      }
  if (is_set && (set->ix != ix || set->generation != ix->vector_generation)) {
    hx_set_error("candidate set does not belong to this index image (vectors were reloaded or deleted?)");
    return HX_ERR_INVARIANT_VIOLATION;
  }
  HX_CUDA(cudaSetDevice(ix->device));
  if (ix->n == 0 || !ix->populated) return answer_empty_index(ix, queries, B, out_counts, nullptr);
  HxScratch* s = nullptr;
  if ((rc = hx_acquire_scratch(ix, &s))) return rc;
  ScratchGuard guard{ix, s};
  uint32_t launches = 0;
  if ((rc = stage_queries(ix, s, queries, B, &launches))) return rc;
  const uint32_t* slots = nullptr;
  if (is_set) {
    slots = set->d_slots;
  } else {
    if ((rc = s->d_cand_ids.reserve(n)) || (rc = s->d_cand_slots.reserve(n))) return rc;
    HX_CUDA(cudaMemcpyAsync(s->d_cand_ids.p, cand_ids, n * sizeof(uint64_t), cudaMemcpyHostToDevice, s->stream));
    k_map_candidates<<<(unsigned)((n + 255) / 256), 256, 0, s->stream>>>(
        ix->d_ids, (uint32_t)ix->n, s->d_cand_ids.p, n, s->d_cand_slots.p, ix->contiguous ? 1 : 0, ix->first_id, ix->d_deleted);
    HX_CUDA(cudaGetLastError());
    launches++;
    slots = s->d_cand_slots.p;
  }
  // a resident set (hx_candidates_make_resident) brings its present slots, tile and view word: no compaction (and no
  // read-back of its count), no gather, no view reduction
  HxResident* res = is_set ? set->resident.load() : nullptr;
  const uint32_t* d_present = nullptr;
  size_t present = 0;
  if (res) {
    if ((rc = hx_resident_current(ix, res))) return rc;
    d_present = res->slots;
    present = res->n;
  } else if ((rc = hx_dense_compact(ix, s, slots, n, s->stream, &d_present, &present, &launches))) {
    return rc;
  }
  if ((rc = s->d_out_ids.reserve(B * (size_t)k)) || (rc = s->d_out_scores.reserve(B * (size_t)k)) ||
      (rc = s->d_out_counts.reserve(B)))
    return rc;
  // below the dense path's minimum the exact scan over the same slot list: hx_search_restricted's answer and launches
  const bool dense = present >= hx_dense_min_rows(k);
  HxDenseCert cert;
  if (dense && res)
    rc = hx_dense_resident_device(ix, s, s->d_queries.p, B, k, *res, s->d_out_ids.p, s->d_out_scores.p, s->d_out_counts.p,
                                  s->stream, s->ev0, s->ev1, &launches, exact ? &cert : nullptr);
  else if (dense)
    rc = hx_dense_restricted_device(ix, s, s->d_queries.p, B, k, d_present, present, s->d_out_ids.p, s->d_out_scores.p,
                                    s->d_out_counts.p, s->stream, s->ev0, s->ev1, &launches, exact ? &cert : nullptr);
  else
    rc = launch_scan_select(ix, s, s->d_queries.p, B, k, slots, nullptr, true, n, n, (uint64_t)B * n, s->d_out_ids.p,
                            s->d_out_scores.p, s->d_out_counts.p, s->stream, s->ev0, s->ev1, &launches);
  if (rc) return rc;
  size_t flagged = 0;
  uint32_t err_before = 0;
  if (exact && dense &&
      (rc = hx_dense_rescan(ix, s, s->d_queries.p, k, d_present, present, cert, s->d_out_ids.p, s->d_out_scores.p,
                            s->d_out_counts.p, s->stream, s->ev0, s->ev1, &launches, &flagged, &err_before)))
    return rc;
  if ((rc = s->h_status.reserve(B)) || (rc = s->h_err.reserve(1))) return rc;
  if (exact && dense && out_how) HX_CUDA(cudaMemcpyAsync(out_how, cert.how, B, cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(out_ids, s->d_out_ids.p, B * (size_t)k * sizeof(uint64_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(out_scores, s->d_out_scores.p, B * (size_t)k * sizeof(float), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(out_counts, s->d_out_counts.p, B * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(s->h_status.p, s->d_qstatus.p, B * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaMemcpyAsync(s->h_err.p, s->d_err.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaStreamSynchronize(s->stream));
  s->h_err.p[0] |= err_before;
  for (size_t b = 0; b < B; ++b)
    if (s->h_status.p[b] != HX_ST_OK) return status_from_word(s->h_status.p[b], b, "query");
  if ((rc = check_device_flags(s->h_err.p[0]))) return rc;
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, s->ev0, s->ev1) == cudaSuccess) {   // k_dense_scores, or the exact scan below the minimum
    ix->last_kernel_ms = ms;
    ix->last_kernel_launches = 1;
  }
  if (stats) {
    const uint64_t dim = ix->cfg.dimension, ldb = (dim + 63) / 64 * 64;
    stats->kernel_launches = launches;
    if (dense) {
      stats->distance_computations = (uint64_t)B * present;
      // gather (f32 rows in, bf16 tile and row terms out; none for a resident set), then the tile read once by the
      // contraction
      stats->algorithmic_bytes = (res ? 0 : present * (4 * dim + 2 * ldb + 4)) + present * 2 * ldb;
      stats->reserved = (uint64_t)(2.0 * (double)B * (double)present * (double)ldb);   // flop of the contraction
      if (flagged) {   // the rescanned queries' full scans over the present rows
        stats->distance_computations += flagged * present;
        stats->vectors_loaded += flagged * present;
        stats->algorithmic_bytes += flagged * present * (4 * dim + (ix->cfg.metric == HX_METRIC_COSINE ? 4 : 0));
      }
    } else {
      stats->distance_computations = (uint64_t)B * n;
      stats->vectors_loaded = (uint64_t)B * n;
      stats->algorithmic_bytes = (uint64_t)B * n * (4 * dim + (ix->cfg.metric == HX_METRIC_COSINE ? 4 : 0));
    }
  }
  return HX_OK;
}

extern "C" hx_status hx_search_dense_restricted(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                                const uint64_t* cand_ids, size_t n_cand, uint64_t* out_ids,
                                                float* out_scores, uint32_t* out_counts, hx_stats* stats) {
  return dense_restricted_host(ix, queries, B, p, cand_ids, n_cand, nullptr, false, out_ids, out_scores, out_counts, stats);
}

extern "C" hx_status hx_search_dense_restricted_set(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                                    const hx_candidates* set, uint64_t* out_ids, float* out_scores,
                                                    uint32_t* out_counts, hx_stats* stats) {
  return dense_restricted_host(ix, queries, B, p, nullptr, 0, set, true, out_ids, out_scores, out_counts, stats);
}

extern "C" hx_status hx_search_dense_restricted_exact(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                                      const uint64_t* cand_ids, size_t n_cand, uint64_t* out_ids,
                                                      float* out_scores, uint32_t* out_counts, uint8_t* out_how,
                                                      hx_stats* stats) {
  return dense_restricted_host(ix, queries, B, p, cand_ids, n_cand, nullptr, false, out_ids, out_scores, out_counts, stats,
                               true, out_how);
}

extern "C" hx_status hx_search_dense_restricted_exact_set(hx_index* ix, const float* queries, size_t B,
                                                          const hx_search_params* p, const hx_candidates* set,
                                                          uint64_t* out_ids, float* out_scores, uint32_t* out_counts,
                                                          uint8_t* out_how, hx_stats* stats) {
  return dense_restricted_host(ix, queries, B, p, nullptr, 0, set, true, out_ids, out_scores, out_counts, stats, true,
                               out_how);
}

// hx_search_dense_restricted_set on device buffers, through a resident set: everything on the caller's stream, no
// synchronisation once the view is current.  Admission is hx_search_dense_restricted_set's, in its order, then the set
// must be resident.  d_out_how (may be null): the certificate without the rescan (0 certified, 1 not certified), or 2
// for every query when the present rows are below hx_dense_min_rows(k) and the exact scan answered.
extern "C" hx_status hx_search_dense_restricted_set_device(hx_index* ix, const float* d_queries, size_t B,
                                                           const hx_search_params* p, const hx_candidates* set,
                                                           uint64_t* d_out_ids, float* d_out_scores, uint32_t* d_out_counts,
                                                           uint8_t* d_out_how, void* cuda_stream) {
  if (!ix) {
    hx_set_error("null index handle");
    return HX_ERR_INDEX_NOT_FOUND;
  }
  uint32_t k, ef;
  hx_status rc = check_params(ix, p, &k, &ef);
  if (rc) return rc;
  if (B == 0) return HX_OK;
  if (!d_queries || !d_out_ids || !d_out_scores || !d_out_counts || !set) return HX_ERR_INVALID_PARAMETER;
  if (ix->cfg.metric == HX_METRIC_MANHATTAN) {
    hx_set_error("the L1 metric is not a contraction: use hx_search_restricted_device");
    return HX_ERR_UNSUPPORTED;
  }
  cudaStream_t stream = (cudaStream_t)cuda_stream;
  auto answer_none = [&]() -> hx_status {   // counts 0, every query "answered by the exact scan"
    HX_CUDA(cudaSetDevice(ix->device));
    HX_CUDA(cudaMemsetAsync(d_out_counts, 0, B * sizeof(uint32_t), stream));
    if (d_out_how) HX_CUDA(cudaMemsetAsync(d_out_how, 2, B, stream));
    return HX_OK;
  };
  const uint64_t n = set->n;
  if (n > 1000000ull) {
    hx_set_error("restricted vector search accepts at most 1000000 unique candidates");
    return HX_ERR_QUERY;
  }
  if (n == 0) return answer_none();
  if (std::min<uint64_t>(k, n) > 800) {
    hx_set_error("restricted vector search result count must be at most 800, got %llu",
                 (unsigned long long)std::min<uint64_t>(k, n));
    return HX_ERR_QUERY;
  }
  if (set->ix != ix || set->generation != ix->vector_generation) {
    hx_set_error("candidate set does not belong to this index image (vectors were reloaded or deleted?)");
    return HX_ERR_INVARIANT_VIOLATION;
  }
  HxResident* res = set->resident.load();
  if (!res) {
    hx_set_error("hx_search_dense_restricted_set_device needs a resident set (hx_candidates_make_resident)");
    return HX_ERR_INVALID_PARAMETER;
  }
  HX_CUDA(cudaSetDevice(ix->device));
  if (ix->n == 0 || !ix->populated || res->n == 0) return answer_none();
  if ((rc = hx_resident_current(ix, res))) return rc;
  HxScratch* s = nullptr;
  if ((rc = dev_scratch(ix, stream, &s))) return rc;
  uint32_t launches = 0;
  if ((rc = prepare_device_queries(ix, s, d_queries, B, stream, &launches))) return rc;
  cudaEvent_t e0, e1;
  if ((rc = s->ring_next(&e0, &e1))) return rc;
  if (res->n < hx_dense_min_rows(k)) {   // the exact scan over the present slots
    if (d_out_how) HX_CUDA(cudaMemsetAsync(d_out_how, 2, B, stream));
    return launch_scan_select(ix, s, d_queries, B, k, res->slots, nullptr, true, res->n, res->n, (uint64_t)B * res->n,
                              d_out_ids, d_out_scores, d_out_counts, stream, e0, e1, &launches);
  }
  HxDenseCert cert;
  if ((rc = hx_dense_resident_device(ix, s, d_queries, B, k, *res, d_out_ids, d_out_scores, d_out_counts, stream, e0, e1,
                                     &launches, d_out_how ? &cert : nullptr)))
    return rc;
  if (d_out_how) HX_CUDA(cudaMemcpyAsync(d_out_how, cert.how, B, cudaMemcpyDeviceToDevice, stream));
  return HX_OK;
}

// ------------------------------------------------------------------------------------------------
// SimHash policy mode (search.rs:595-992, policy.rs) — the production-default SearchParams
// ------------------------------------------------------------------------------------------------
extern "C" void hx_policy_params_default(hx_policy_params* p) {   // SearchParams::new (mod.rs:482-500)
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->bypass_min_frontier = 24;
  p->bypass_window_expansions = 4;
  p->bypass_min_filter_rate = 0.12f;
  p->read_budget_multiplier = 3;
  p->sampling_ratio_override = -1.0f;
  p->failure_prob_override = -1.0f;
}

extern "C" uint64_t hx_order_code_from_simhash_bits(uint64_t bits) {   // simhash.rs:44-59
  const uint16_t b0 = (uint16_t)(bits >> 48), b1 = (uint16_t)(bits >> 32), b2 = (uint16_t)(bits >> 16), b3 = (uint16_t)bits;
  uint64_t code = 0;
  for (int bit = 15; bit >= 0; --bit) {
    code = (code << 1) | ((b0 >> bit) & 1u);
    code = (code << 1) | ((b1 >> bit) & 1u);
    code = (code << 1) | ((b2 >> bit) & 1u);
    code = (code << 1) | ((b3 >> bit) & 1u);
  }
  return code;
}

extern "C" hx_status hx_index_set_simhash_config(hx_index* ix, const hx_simhash_config* cfg) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (!cfg || cfg->simhash_threshold > 64 || !(cfg->sampling_ratio >= 0.0f && cfg->sampling_ratio <= 1.0f) ||
      !(cfg->adaptive_failure_prob > 0.0f && cfg->adaptive_failure_prob < 1.0f)) {
    hx_set_error("invalid SimHash configuration");   // CollisionThreshold / UnitInterval / FailureProbability::try_new
    return HX_ERR_INVALID_VECTOR_CONFIG;
  }
  ix->simcfg = *cfg;
  return HX_OK;
}

static hx_status ensure_simhash_arrays(hx_index* ix) {
  if (ix->n == 0) {
    hx_set_error("no vectors loaded");
    return HX_ERR_INVALID_PARAMETER;
  }
  if (!ix->d_simhash) {
    const size_t rcap = std::max(ix->cap_rows, ix->n);
    HX_CUDA(cudaMalloc((void**)&ix->d_simhash, rcap * sizeof(uint64_t)));
    HX_CUDA(cudaMalloc((void**)&ix->d_has_simhash, rcap));
    HX_CUDA(cudaMemset(ix->d_simhash, 0, rcap * sizeof(uint64_t)));
    HX_CUDA(cudaMemset(ix->d_has_simhash, 0, rcap));
    ix->simhash_count = 0;
  }
  return HX_OK;
}

extern "C" hx_status hx_index_load_simhash(hx_index* ix, const uint64_t* ids, const uint64_t* bits, size_t n) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (n && (!ids || !bits)) return HX_ERR_INVALID_PARAMETER;
  HX_CUDA(cudaSetDevice(ix->device));
  hx_status rc = ensure_simhash_arrays(ix);
  if (rc) return rc;
  std::vector<uint64_t> h(ix->n);
  std::vector<uint8_t> has(ix->n);
  HX_CUDA(cudaMemcpy(h.data(), ix->d_simhash, ix->n * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  HX_CUDA(cudaMemcpy(has.data(), ix->d_has_simhash, ix->n, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < n; ++i) {
    uint32_t slot;
    if (!hx_slot_of(ix, ids[i], &slot)) {
      hx_set_error("SimHash row for node %llu which has no vector row", (unsigned long long)ids[i]);
      return HX_ERR_INVARIANT_VIOLATION;
    }
    h[slot] = bits[i];
    has[slot] = 1;
  }
  HX_CUDA(cudaMemcpy(ix->d_simhash, h.data(), ix->n * sizeof(uint64_t), cudaMemcpyHostToDevice));
  HX_CUDA(cudaMemcpy(ix->d_has_simhash, has.data(), ix->n, cudaMemcpyHostToDevice));
  size_t c = 0;
  for (uint8_t b : has) c += b;
  ix->simhash_count = c;
  return HX_OK;
}

extern "C" hx_status hx_index_set_simhash_planes(hx_index* ix, const float* planes) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (!planes) return HX_ERR_INVALID_PARAMETER;
  HX_CUDA(cudaSetDevice(ix->device));
  const uint32_t dim = ix->cfg.dimension;
  std::vector<float> t((size_t)dim * 64);
  for (uint32_t p = 0; p < 64; ++p)
    for (uint32_t i = 0; i < dim; ++i) t[(size_t)i * 64 + p] = planes[(size_t)p * dim + i];
  if (!ix->d_planes_t) HX_CUDA(cudaMalloc((void**)&ix->d_planes_t, t.size() * sizeof(float)));
  HX_CUDA(cudaMemcpy(ix->d_planes_t, t.data(), t.size() * sizeof(float), cudaMemcpyHostToDevice));
  return HX_OK;
}

// SimHasher::hash_from_slice (unaligned_vector/simhash.rs:263-290): thread (row, plane) walks the row sequentially,
// `dot += value * plane` with two roundings; bit = dot > 0.  64 threads per row, planes transposed so a warp reads
// 32 consecutive plane values per element and the row element is a broadcast.
__global__ void k_simhash_project(const float* __restrict__ rows, size_t n, uint32_t dim, uint32_t ld,
                                  const float* __restrict__ planes_t, uint64_t* __restrict__ out, uint8_t* has) {
  const size_t row = (size_t)blockIdx.x * (blockDim.x / 64) + threadIdx.x / 64;
  const uint32_t p = threadIdx.x & 63u;
  if (row >= n) return;
  const float* v = rows + row * ld;
  float dot = 0.0f;
  for (uint32_t i = 0; i < dim; ++i) dot = __fadd_rn(dot, __fmul_rn(v[i], planes_t[(size_t)i * 64 + p]));
  const uint32_t m = __ballot_sync(0xffffffffu, dot > 0.0f);
  // the two warps of a row combine through shared memory
  __shared__ uint32_t halves[8][2];
  const uint32_t r_in_blk = threadIdx.x / 64;
  if ((threadIdx.x & 31u) == 0) halves[r_in_blk][(threadIdx.x >> 5) & 1u] = m;
  __syncthreads();
  if (p == 0) {
    out[row] = ((uint64_t)halves[r_in_blk][1] << 32) | halves[r_in_blk][0];
    if (has) has[row] = 1;
  }
}

extern "C" hx_status hx_index_compute_simhash(hx_index* ix) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  HX_CUDA(cudaSetDevice(ix->device));
  if (!ix->d_planes_t) {
    hx_set_error("SimHash hyperplanes not set (hx_index_set_simhash_planes)");
    return HX_ERR_INVALID_VECTOR_CONFIG;
  }
  hx_status rc = ensure_simhash_arrays(ix);
  if (rc) return rc;
  const unsigned blocks = (unsigned)((ix->n + 7) / 8);
  k_simhash_project<<<blocks, 512>>>(ix->d_vec, ix->n, ix->cfg.dimension, ix->ld, ix->d_planes_t, ix->d_simhash, ix->d_has_simhash);
  HX_CUDA(cudaGetLastError());
  HX_CUDA(cudaDeviceSynchronize());
  ix->simhash_count = ix->n;
  return HX_OK;
}

extern "C" hx_status hx_index_download_simhash(hx_index* ix, size_t first_slot, size_t n, uint64_t* out_bits) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  if (!ix->d_simhash || first_slot + n > ix->n || !out_bits) return HX_ERR_INVALID_PARAMETER;
  HX_CUDA(cudaSetDevice(ix->device));
  HX_CUDA(cudaMemcpy(out_bits, ix->d_simhash + first_slot, n * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  return HX_OK;
}

static hx_status launch_policy(hx_index* ix, HxScratch* s, const float* d_queries, size_t B, uint32_t k, uint32_t ef,
                               const hx_search_params* p, const hx_policy_params* pol, const uint64_t* d_qsim,
                               uint64_t* d_out_ids, float* d_out_scores, uint32_t* d_out_counts, uint32_t* d_qstats,
                               cudaStream_t stream, uint32_t* launches) {
  hx_status rc = hx_finalize_graph(ix);
  if (rc) return rc;
  if (ix->n == 0 || !ix->populated || !ix->d_nbr0) {
    HX_CUDA(cudaMemsetAsync(d_out_counts, 0, B * sizeof(uint32_t), stream));
    if (d_qstats) HX_CUDA(cudaMemsetAsync(d_qstats, 0, B * 4 * sizeof(uint32_t), stream));
    return HX_OK;
  }
  const uint32_t fr_cap = round_up(std::max(ix->stride0, ix->stride_u), 32);
  const size_t rowbytes = (size_t)ix->ld * 4;
  // the query stays in shared memory: holding it in registers (QCH = 24) spills at the 128-register cap of a 512-thread CTA
  // and was slower
  const uint32_t pol_qch = 0;
  const size_t fixed0 = (pol_qch ? 0 : rowbytes) + (size_t)ef * 8 + (size_t)k * 8 + HX_TIE_CAP * 8 + (size_t)fr_cap * 13 +
                        28 * 4 + 16;
  const size_t budget = 227 * 1024;
  uint32_t wpc = 0, R = 0;
  const uint32_t spread = (uint32_t)std::max<size_t>(1, (B + ix->sm_count - 1) / (size_t)ix->sm_count);
  const hx_tuning& t = ix->tune;
  const uint32_t pol_warps = knob(t.pol_warps, 16), pol_minR = knob(t.pol_min_rows, 3);   // fewer rows per expansion survive the gate: 3 slots suffice
  // B < #SMs: one CTA per query (warp 0 runs the query, 7 more warps reduce rows with it)
  const bool pol_cta = B < (size_t)ix->sm_count && knob(t.pol_cta, 1) != 0;
  for (uint32_t w = pol_cta ? 1u : std::min(pol_warps, spread); w >= 1; --w) {
    const size_t per_warp = (budget / w) & ~(size_t)127;
    if (per_warp <= fixed0 + 8 + rowbytes) continue;
    const uint32_t r = (uint32_t)std::min<size_t>(32, (per_warp - fixed0) / (rowbytes + 8));
    if (r >= pol_minR || w == 1) { wpc = w; R = r; break; }
  }
  if (R == 0) {
    hx_set_error("query working set exceeds shared memory (dimension %u, ef %u)", ix->cfg.dimension, ef);
    return HX_ERR_INVALID_PARAMETER;
  }
  uint32_t wstride = round_up((uint32_t)(fixed0 + (size_t)R * (rowbytes + 8)), 128);
  uint32_t lg = 12;
  while ((1u << lg) < 64u * ef && lg < 24) lg++;
  uint32_t vt_cap = 1u << knob(t.visited_log2, lg);
  size_t cta_vt_bytes = 0;
  if (pol_cta) {   // the visited set sits in shared memory behind the query's region: shrink rows / table until it fits
    while (vt_cap > 1024 && (size_t)vt_cap * 4 > budget / 4) vt_cap >>= 1;
    while (R > 4 && fixed0 + (size_t)R * (rowbytes + 8) + 256 + (size_t)vt_cap * 4 > budget) R--;
    wstride = round_up((uint32_t)(fixed0 + (size_t)R * (rowbytes + 8)), 128);
    if ((size_t)wstride + (size_t)vt_cap * 4 > budget) {
      hx_set_error("query working set exceeds shared memory (dimension %u, ef %u)", ix->cfg.dimension, ef);
      return HX_ERR_INVALID_PARAMETER;
    }
    cta_vt_bytes = (size_t)vt_cap * 4;
  }
  const uint32_t grid = (uint32_t)std::min<size_t>((B + wpc - 1) / wpc, (size_t)ix->sm_count);
  const size_t vslots = (size_t)grid * wpc;
  const uint32_t pool_n = knob(t.visited_pool, 32);
  const uint32_t pool_cap = std::max<uint32_t>(vt_cap * 16u, 65536u);
  if ((rc = s->d_vtab.reserve(vslots * vt_cap))) return rc;
  if (s->vpool_n != pool_n || s->vpool_cap != pool_cap || !s->d_vbusy.p) {
    if ((rc = s->d_vpool.reserve((size_t)std::max(pool_n, 1u) * pool_cap))) return rc;
    if ((rc = s->d_vbusy.reserve(std::max(pool_n, 1u)))) return rc;
    HX_CUDA(cudaMemsetAsync(s->d_vbusy.p, 0, std::max(pool_n, 1u) * sizeof(uint32_t), stream));
    s->vpool_n = pool_n;
    s->vpool_cap = pool_cap;
  }
  if ((rc = s->d_err.reserve(2))) return rc;
  HX_CUDA(cudaMemsetAsync(s->d_err.p, 0, 2 * sizeof(uint32_t), stream));
  if ((rc = s->d_pstats.reserve(12))) return rc;
  HX_CUDA(cudaMemsetAsync(s->d_pstats.p, 0, 12 * sizeof(unsigned long long), stream));
  HxRingArgs rg{};
  rg.vtab = s->d_vtab.p;
  rg.vt_cap = vt_cap;
  rg.pool = s->d_vpool.p;
  rg.pool_busy = s->d_vbusy.p;
  rg.pool_n = pool_n;
  rg.pool_cap = pool_cap;
  rg.counter = s->d_err.p + 1;
  rg.l2_hint = 1;
  if ((rc = setup_tie_pool(s, &rg, stream))) return rc;
  if ((rc = s->d_qerr.reserve(B))) return rc;
  rg.l2_spec = knob(t.pol_early_sim, 1);   // policy kernel: fingerprints requested together with the visited probe (0: after it)
  HxHnswArgs a{};
  a.queries = d_queries;
  a.q_hdr = s->d_qhdr.p;
  a.q_status = s->d_qstatus.p;
  a.B = (uint32_t)B;
  a.k = k;
  a.ef = ef;
  a.out_ids = d_out_ids;
  a.out_scores = d_out_scores;
  a.out_counts = d_out_counts;
  a.q_stats = d_qstats;
  a.err_flags = s->d_err.p;
  a.q_err = s->d_qerr.p;
  a.fr_cap = fr_cap;
  HxPolicyArgs pa{};
  pa.cfg.mode = p->simhash_mode;
  pa.cfg.threshold = ix->simcfg.simhash_threshold;
  pa.cfg.sampling_ratio = pol->sampling_ratio_override >= 0.0f ? pol->sampling_ratio_override : ix->simcfg.sampling_ratio;
  pa.cfg.has_pre_override = p->pre_sampling_ratio >= 0.0f ? 1 : 0;
  pa.cfg.pre_override = p->pre_sampling_ratio >= 0.0f ? p->pre_sampling_ratio : 1.0f;
  pa.cfg.adaptive_enabled = ix->simcfg.adaptive_enabled ? 1 : 0;
  pa.cfg.failure_prob = pol->failure_prob_override >= 0.0f ? pol->failure_prob_override : ix->simcfg.adaptive_failure_prob;
  pa.cfg.bypass_min_frontier = pol->bypass_min_frontier;
  pa.cfg.bypass_window_expansions = pol->bypass_window_expansions;
  pa.cfg.bypass_min_filter_rate = pol->bypass_min_filter_rate;
  pa.cfg.read_budget_multiplier = pol->read_budget_multiplier;
  pa.cfg.threshold_margin = sqrtf((64.0f * logf(1.0f / pa.cfg.failure_prob)) / 2.0f);   // policy.rs:592, host libm
  pa.node_simhash = ix->d_simhash;
  pa.node_has_simhash = ix->simhash_count == ix->n ? nullptr : ix->d_has_simhash;   // all present: skip the byte load
  pa.query_simhash = d_qsim;
  pa.pstats = s->d_pstats.p;
  const HxDev dev = ix->dev();
  const size_t smem_launch = (size_t)wpc * wstride + cta_vt_bytes;
#define HX_LAUNCH_POLICY2(M, Q)                                                                                    \
  do {                                                                                                             \
    if (pol_cta) {                                                                                                 \
      HX_CUDA(cudaFuncSetAttribute(k_hnsw_search_policy<M, Q, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                                   (int)smem_launch));                                                             \
      k_hnsw_search_policy<M, Q, true><<<grid, 8 * 32, smem_launch, stream>>>(dev, a, rg, pa, wstride, R);         \
    } else {                                                                                                       \
      HX_CUDA(cudaFuncSetAttribute(k_hnsw_search_policy<M, Q, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
                                   (int)smem_launch));                                                             \
      k_hnsw_search_policy<M, Q, false><<<grid, wpc * 32, smem_launch, stream>>>(dev, a, rg, pa, wstride, R);      \
    }                                                                                                              \
  } while (0)
#define HX_LAUNCH_POLICY(M)                                                                                        \
  do {                                                                                                             \
    HX_LAUNCH_POLICY2(M, 0);                                                                                       \
  } while (0)
  switch (ix->cfg.metric) {
    case HX_METRIC_EUCLIDEAN: HX_LAUNCH_POLICY(HXM_EUCLIDEAN); break;
    case HX_METRIC_COSINE: HX_LAUNCH_POLICY(HXM_COSINE); break;
    default: HX_LAUNCH_POLICY(HXM_MANHATTAN); break;
  }
#undef HX_LAUNCH_POLICY
#undef HX_LAUNCH_POLICY2
  HX_CUDA(cudaGetLastError());
  (*launches)++;
  return HX_OK;
}

extern "C" hx_status hx_search_ex(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                  const hx_policy_params* policy, const uint64_t* query_simhash, uint64_t* out_ids,
                                  float* out_scores, uint32_t* out_counts, hx_stats* stats, hx_policy_stats* pstats) {
  return hx_search_policy(ix, queries, B, p, policy, query_simhash, out_ids, out_scores, out_counts, stats, pstats, nullptr);
}

static hx_status hx_search_policy(hx_index* ix, const float* queries, size_t B, const hx_search_params* p,
                                  const hx_policy_params* policy, const uint64_t* query_simhash, uint64_t* out_ids,
                                  float* out_scores, uint32_t* out_counts, hx_stats* stats, hx_policy_stats* pstats,
                                  hx_status* out_status) {
  if (!ix) {
    hx_set_error("null index handle");
    return HX_ERR_INDEX_NOT_FOUND;
  }
  uint32_t k, ef;
  hx_status rc = check_params(ix, p, &k, &ef);
  if (rc) return rc;
  if (pstats) memset(pstats, 0, sizeof(*pstats));
  if (params_strict(p)) {   // the exhaustive specialisation never looks at fingerprints or the policy
    hx_search_params q = *p;
    q.simhash_mode = HX_SIMHASH_OFF;
    q.pre_sampling_ratio = 1.0f;
    return hx_search_strict(ix, queries, B, &q, out_ids, out_scores, out_counts, stats, out_status);
  }
  hx_policy_params pol;
  hx_policy_params_default(&pol);
  if (policy) pol = *policy;
  if (pol.bypass_min_frontier == 0 || pol.bypass_window_expansions == 0 || pol.read_budget_multiplier == 0 ||
      !(pol.bypass_min_filter_rate >= 0.0f && pol.bypass_min_filter_rate <= 1.0f) || pol.sampling_ratio_override > 1.0f ||
      pol.failure_prob_override >= 1.0f || pol.failure_prob_override == 0.0f) {
    hx_set_error("invalid SimHash policy parameters");   // VectorParameterError (mod.rs:563-600)
    return HX_ERR_INVALID_PARAMETER;
  }
  if (stats) memset(stats, 0, sizeof(*stats));
  if (B == 0) return HX_OK;
  if (!queries || !out_ids || !out_scores || !out_counts) {
    hx_set_error("hx_search_ex: null pointer");
    return HX_ERR_INVALID_PARAMETER;
  }
  HX_CUDA(cudaSetDevice(ix->device));
  if (ix->n == 0 || !ix->populated) return answer_empty_index(ix, queries, B, out_counts, out_status);
  // filtering needs the node fingerprints (cosine only, policy.rs:67-88); sampling needs the query's for its seed
  const bool filtering = ix->cfg.metric == HX_METRIC_COSINE && p->simhash_mode != HX_SIMHASH_OFF;
  if (filtering && ix->n && !ix->d_simhash) {
    hx_set_error("SimHash rows not loaded: call hx_index_load_simhash or hx_index_compute_simhash before a filtered search");
    return HX_ERR_INVALID_VECTOR_CONFIG;
  }
  if (!query_simhash && !ix->d_planes_t) {
    hx_set_error("no query fingerprints given and no hyperplanes set (hx_index_set_simhash_planes)");
    return HX_ERR_INVALID_VECTOR_CONFIG;
  }
  HxScratch* s = nullptr;
  if ((rc = hx_acquire_scratch(ix, &s))) return rc;
  ScratchGuard guard{ix, s};
  uint32_t launches = 0;
  if ((rc = stage_queries(ix, s, queries, B, &launches, out_status != nullptr))) return rc;
  if ((rc = s->d_out_ids.reserve(B * (size_t)k))) return rc;
  if ((rc = s->d_out_scores.reserve(B * (size_t)k))) return rc;
  if ((rc = s->d_out_counts.reserve(B))) return rc;
  if ((rc = s->d_qsim.reserve(B))) return rc;
  if (query_simhash) {
    HX_CUDA(cudaMemcpyAsync(s->d_qsim.p, query_simhash, B * sizeof(uint64_t), cudaMemcpyHostToDevice, s->stream));
  } else {
    k_simhash_project<<<(unsigned)((B + 7) / 8), 512, 0, s->stream>>>(s->d_queries.p, B, ix->cfg.dimension, ix->cfg.dimension,
                                                                     ix->d_planes_t, s->d_qsim.p, nullptr);
    HX_CUDA(cudaGetLastError());
    launches++;
  }
  const bool want_stats = p->collect_stats != 0 && stats != nullptr;
  if (want_stats && (rc = s->d_qstats.reserve(B * 4))) return rc;
  HX_CUDA(cudaEventRecord(s->ev0, s->stream));
  if ((rc = launch_policy(ix, s, s->d_queries.p, B, k, ef, p, &pol, s->d_qsim.p, s->d_out_ids.p, s->d_out_scores.p,
                          s->d_out_counts.p, want_stats ? s->d_qstats.p : nullptr, s->stream, &launches)))
    return rc;
  HX_CUDA(cudaEventRecord(s->ev1, s->stream));
  HxDownload dl;
  if ((rc = enqueue_results(s, B, k, out_ids, out_scores, out_counts, &launches, &dl))) return rc;
  if (want_stats) {
    if ((rc = s->h_qstats.reserve(B * 4))) return rc;
    HX_CUDA(cudaMemcpyAsync(s->h_qstats.p, s->d_qstats.p, B * 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s->stream));
  }
  unsigned long long hps[12] = {0};
  if (pstats && s->d_pstats.p)
    HX_CUDA(cudaMemcpyAsync(hps, s->d_pstats.p, sizeof(hps), cudaMemcpyDeviceToHost, s->stream));
  HX_CUDA(cudaStreamSynchronize(s->stream));
  finish_results(s, dl, out_ids, out_scores, out_counts);
  if ((rc = report_batch(s, B, out_counts, out_status))) return rc;
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, s->ev0, s->ev1) == cudaSuccess) {
    ix->last_kernel_ms = ms;
    ix->last_kernel_launches = 1;
  }
  if (pstats) memcpy(pstats, hps, sizeof(hps));
  if (stats) {
    stats->kernel_launches = launches;
    if (want_stats) {
      for (size_t b = 0; b < B; ++b) {
        stats->expansion_steps += s->h_qstats.p[b * 4 + 0];
        stats->neighbors_examined += s->h_qstats.p[b * 4 + 1];
        stats->distance_computations += s->h_qstats.p[b * 4 + 2];
        stats->upper_layer_steps += s->h_qstats.p[b * 4 + 3];
        if (s->h_qstats.p[b * 4 + 2]) stats->vectors_loaded += s->h_qstats.p[b * 4 + 2] - 1;
      }
      stats->algorithmic_bytes = stats->expansion_steps * (5ull + 8ull * ix->lim0) +
                                 stats->distance_computations * (4ull + 4ull * ix->cfg.dimension) +
                                 (pstats ? pstats->simhash_examined * 8ull : 0ull);
    }
  }
  return HX_OK;
}

extern "C" hx_status hx_last_kernel_ms(hx_index* ix, float* ms, uint32_t* launches) {
  if (!ix) return HX_ERR_INDEX_NOT_FOUND;
  HX_CUDA(cudaSetDevice(ix->device));
  std::vector<HxScratch*> devs;
  {
    std::lock_guard<std::mutex> lk(ix->mu);
    for (auto& kv : ix->dev_scratch) devs.push_back(kv.second);
  }
  float total = 0.f;
  uint32_t cnt = 0;
  bool any = false;
  for (HxScratch* s : devs) {
    if (s->ring_pending) {
      // device-path launches since the previous call: sum their CUDA-event durations (synchronises)
      any = true;
      const size_t cap = s->ring0.size();
      size_t idx;
      if (s->ring0.size() < 512) idx = s->ring0.size() - s->ring_pending;
      else idx = (s->ring_pos + cap - s->ring_pending) % cap;
      for (size_t i = 0; i < s->ring_pending; ++i) {
        const size_t j = (idx + i) % cap;
        float t = 0.f;
        if (cudaEventSynchronize(s->ring1[j]) == cudaSuccess &&
            cudaEventElapsedTime(&t, s->ring0[j], s->ring1[j]) == cudaSuccess) {
          total += t;
          cnt++;
        } else {
          cudaGetLastError();
        }
      }
      s->ring_pending = 0;
    }
    if (s->prof_init && s->d_prof.p) {   // HX_PHASE_PROF diagnostics: print and reset the phase cycle sums
      unsigned long long h[8];
      cudaDeviceSynchronize();
      if (cudaMemcpy(h, s->d_prof.p, sizeof(h), cudaMemcpyDeviceToHost) == cudaSuccess) {
        fprintf(stderr, "HX_PHASE_PROF cycles: pop=%llu row+deg=%llu visited+issue=%llu wait+score=%llu admit=%llu  "
                        "predicted-next hits=%llu of %llu expansions\n", h[0], h[1], h[2], h[3], h[4], h[5], h[6]);
        cudaMemset(s->d_prof.p, 0, sizeof(h));
      }
    }
  }
  if (any) {
    ix->last_kernel_ms = total;
    ix->last_kernel_launches = cnt;
  }
  if (ms) *ms = ix->last_kernel_ms;
  if (launches) *launches = ix->last_kernel_launches;
  return HX_OK;
}

#include "hx_service.inl"
#include "hx_mirror.inl"
#include "hx_filtered.inl"
