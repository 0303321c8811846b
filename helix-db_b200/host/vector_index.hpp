// vector_index.hpp — C++ host-side mirror of the reference's vector-index read API over the C ABI.
//
// The reference is compiled code (Rust) whose toolchain is absent here; this header is what a C++ host links instead.
// Names, argument meaning and error behaviour follow
//   ValidatedVectorReadIndex::<D>::{search, search_restricted}   crates/db/src/search/vector/read_index.rs:81-101
//   SearchParams                                                 crates/db/src/search/vector/mod.rs:411-621
//   RestrictedVectorCandidates::from_ids                         crates/db/src/search/vector/restricted.rs:356-371
//   SearchResult                                                 crates/db/src/search/vector/result.rs:20-40
//   HelixDbError                                                 crates/db/src/error.rs:379-661
// Header-only; link with -lhelix_b200.  No CPU fallback: every call runs on the device or throws.
#pragma once
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/helix_b200.h"

namespace helix {

struct HelixDbError : std::runtime_error {
  hx_status code;
  uint32_t index;   // component index for InvalidVectorComponent / VectorComponentMagnitudeExceeded
  HelixDbError(hx_status c, const std::string& msg, uint32_t idx = 0) : std::runtime_error(variant(c) + ": " + msg), code(c), index(idx) {}
  static std::string variant(hx_status c) {
    switch (c) {
      case HX_ERR_INDEX_NOT_FOUND: return "IndexNotFound";
      case HX_ERR_INVALID_DIMENSION: return "InvalidDimension";
      case HX_ERR_INVALID_VECTOR_COMPONENT: return "InvalidVectorComponent";
      case HX_ERR_ZERO_NORM_COSINE: return "ZeroNormCosineVector";
      case HX_ERR_MAGNITUDE_EXCEEDED: return "VectorComponentMagnitudeExceeded";
      case HX_ERR_INVALID_VECTOR_CONFIG: return "InvalidVectorConfig";
      case HX_ERR_QUERY: return "Query";
      case HX_ERR_INVARIANT_VIOLATION: return "InvariantViolation";
      case HX_ERR_INVALID_PARAMETER: return "VectorParameterError";
      case HX_ERR_UNSUPPORTED: return "Unsupported";
      default: return "Device";
    }
  }
};

inline void check(hx_status rc) {
  if (rc != HX_OK) throw HelixDbError(rc, hx_last_error(), hx_last_error_index());
}

enum class SimHashMode { Off = HX_SIMHASH_OFF, Adaptive = HX_SIMHASH_ADAPTIVE, Always = HX_SIMHASH_ALWAYS };

struct SearchResult {
  uint64_t entity_id;
  float score;   // finite, >= 0 (DistanceScore)
};

// SearchParams::new(k): ef = max(k, 100), SimHashMode::Adaptive (mod.rs:482-500)
class SearchParams {
 public:
  explicit SearchParams(uint32_t k) : k_(k), ef_(std::max(k, 100u)) {
    if (k == 0) throw HelixDbError(HX_ERR_INVALID_PARAMETER, "result count must be non-zero");
    hx_policy_params_default(&policy_);
  }
  SearchParams& with_ef(uint32_t ef) {
    if (ef < k_) throw HelixDbError(HX_ERR_INVALID_PARAMETER, "search beam width must cover k");
    ef_ = ef;
    return *this;
  }
  SearchParams& with_simhash_mode(SimHashMode m) { mode_ = m; return *this; }
  SearchParams& with_pre_simhash_sampling_ratio(float r) {
    if (!(r >= 0.0f && r <= 1.0f)) throw HelixDbError(HX_ERR_INVALID_PARAMETER, "ratio must be in the unit interval");
    ratio_ = r; has_ratio_ = true; return *this;
  }
  // mod.rs:563-613
  SearchParams& with_simhash_bypass_tuning(uint32_t min_frontier, uint32_t window_expansions, float min_filter_rate,
                                           uint32_t read_budget_multiplier) {
    if (!min_frontier || !window_expansions || !read_budget_multiplier || !(min_filter_rate >= 0.0f && min_filter_rate <= 1.0f))
      throw HelixDbError(HX_ERR_INVALID_PARAMETER, "invalid SimHash bypass tuning");
    policy_.bypass_min_frontier = min_frontier; policy_.bypass_window_expansions = window_expansions;
    policy_.bypass_min_filter_rate = min_filter_rate; policy_.read_budget_multiplier = read_budget_multiplier;
    return *this;
  }
  SearchParams& with_simhash_sampling_ratio(float r) {
    if (!(r >= 0.0f && r <= 1.0f)) throw HelixDbError(HX_ERR_INVALID_PARAMETER, "ratio must be in the unit interval");
    policy_.sampling_ratio_override = r; return *this;
  }
  SearchParams& with_simhash_failure_prob(float p) {
    if (!(p > 0.0f && p < 1.0f)) throw HelixDbError(HX_ERR_INVALID_PARAMETER, "failure probability must be in (0, 1)");
    policy_.failure_prob_override = p; return *this;
  }
  const hx_policy_params& policy() const { return policy_; }
  static SearchParams strict(uint32_t k) { return SearchParams(k).with_simhash_mode(SimHashMode::Off).with_pre_simhash_sampling_ratio(1.0f); }
  uint32_t k() const { return k_; }
  uint32_t ef() const { return ef_; }
  bool requires_query_simhash() const { return mode_ != SimHashMode::Off || (has_ratio_ && ratio_ < 1.0f); }
  hx_search_params raw(uint32_t query_dimension = 0) const {
    hx_search_params p{};
    p.k = k_;
    p.ef = ef_;
    p.simhash_mode = static_cast<int32_t>(mode_);
    p.pre_sampling_ratio = has_ratio_ ? ratio_ : -1.0f;   // negative = no override (Option::None)
    p.query_dimension = query_dimension;
    return p;
  }

 private:
  uint32_t k_, ef_;
  SimHashMode mode_ = SimHashMode::Adaptive;
  float ratio_ = 1.0f;
  bool has_ratio_ = false;
  hx_policy_params policy_{};
};

// RestrictedVectorCandidates::from_ids: duplicates collapse, ascending, at most 1e6 (restricted.rs:356-371)
class RestrictedVectorCandidates {
 public:
  static RestrictedVectorCandidates from_ids(std::vector<uint64_t> ids) {
    std::sort(ids.begin(), ids.end());
    ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
    if (ids.size() > 1000000) throw HelixDbError(HX_ERR_QUERY, "restricted vector search accepts at most 1000000 unique candidates");
    RestrictedVectorCandidates c;
    c.ids_ = std::move(ids);
    return c;
  }
  bool is_empty() const { return ids_.empty(); }
  bool contains(uint64_t id) const { return std::binary_search(ids_.begin(), ids_.end(), id); }
  const std::vector<uint64_t>& ids() const { return ids_; }

 private:
  std::vector<uint64_t> ids_;
};

class VectorIndex {
 public:
  VectorIndex(hx_metric metric, uint32_t dimension, uint32_t m = 16, uint32_t m0 = 32, uint32_t ef_construction = 200, int device = 0)
      : dim_(dimension) {
    hx_index_config cfg{};
    cfg.dimension = dimension;
    cfg.metric = metric;
    cfg.m = m;
    cfg.m0 = m0;
    cfg.ef_construction = ef_construction;
    cfg.device = device;
    check(hx_index_create(&cfg, &h_));
  }
  ~VectorIndex() { hx_index_destroy(h_); }
  VectorIndex(const VectorIndex&) = delete;
  VectorIndex& operator=(const VectorIndex&) = delete;

  void load_vectors(const std::vector<uint64_t>& ids, const std::vector<float>& rows) {
    if (rows.size() != ids.size() * dim_) throw HelixDbError(HX_ERR_INVALID_DIMENSION, "rows must be ids.size() x dimension");
    check(hx_index_load_vectors(h_, ids.data(), rows.data(), ids.size()));
  }
  void load_graph(uint16_t layer, const std::vector<uint64_t>& nodes, const std::vector<uint32_t>& offsets, const std::vector<uint64_t>& nbrs) {
    check(hx_index_load_graph(h_, layer, nodes.data(), offsets.data(), nbrs.data(), nodes.size()));
  }
  void set_entry(uint64_t entry_point, uint16_t max_layer) { check(hx_index_set_entry(h_, entry_point, max_layer)); }
  void build(uint64_t seed = 0) { check(hx_index_build(h_, nullptr, seed)); }

  // SimHash state of the production-default mode: the index configuration (config/indexes.rs:398-406), the persisted
  // [0x12] fingerprints, optionally the hyperplane table (SimHasher::hyperplanes(), 64 x dimension)
  void set_simhash_config(uint32_t threshold = 43, float sampling_ratio = 0.8f, bool adaptive_enabled = true,
                          float adaptive_failure_prob = 0.1f) {
    hx_simhash_config c{threshold, sampling_ratio, adaptive_enabled ? 1u : 0u, adaptive_failure_prob};
    check(hx_index_set_simhash_config(h_, &c));
  }
  void load_simhash(const std::vector<uint64_t>& ids, const std::vector<uint64_t>& bits) {
    if (ids.size() != bits.size()) throw HelixDbError(HX_ERR_INVALID_PARAMETER, "one fingerprint per id");
    check(hx_index_load_simhash(h_, ids.data(), bits.data(), ids.size()));
  }
  void set_simhash_planes(const std::vector<float>& planes) {
    if (planes.size() != 64u * dim_) throw HelixDbError(HX_ERR_INVALID_DIMENSION, "hyperplane table must be 64 x dimension");
    check(hx_index_set_simhash_planes(h_, planes.data()));
  }
  void compute_simhash() { check(hx_index_compute_simhash(h_)); }

  // VectorIndex::search (index.rs:1578): results sorted by (score, id), at most k.  Every SearchParams is served: the
  // strict-exhaustive specialisation and the SimHash policy modes (query fingerprint given, or projected from the planes).
  std::vector<SearchResult> search(const std::vector<float>& query, const SearchParams& params,
                                   const uint64_t* query_simhash = nullptr) const {
    hx_search_params p = params.raw(static_cast<uint32_t>(query.size()));
    std::vector<uint64_t> ids(params.k());
    std::vector<float> scores(params.k());
    uint32_t count = 0;
    check(hx_search_ex(h_, query.data(), 1, &p, &params.policy(), query_simhash, ids.data(), scores.data(), &count, nullptr,
                       nullptr));
    std::vector<SearchResult> out(count);
    for (uint32_t i = 0; i < count; ++i) out[i] = SearchResult{ids[i], scores[i]};
    return out;
  }
  // VectorIndex::search_restricted (restricted.rs:466-479), exact for every |C| <= 1e6
  std::vector<SearchResult> search_restricted(const std::vector<float>& query, const SearchParams& params,
                                              const RestrictedVectorCandidates& allowed) const {
    hx_search_params p = params.raw(static_cast<uint32_t>(query.size()));
    std::vector<uint64_t> ids(params.k());
    std::vector<float> scores(params.k());
    uint32_t count = 0;
    check(hx_search_restricted(h_, query.data(), 1, &p, allowed.ids().data(), allowed.ids().size(), ids.data(), scores.data(), &count, nullptr));
    std::vector<SearchResult> out(count);
    for (uint32_t i = 0; i < count; ++i) out[i] = SearchResult{ids[i], scores[i]};
    return out;
  }
  // A device candidate set's tensor-core view, built once and kept by the set (hx_candidates_make_resident), and the
  // device memory it holds (0 while the set is not resident)
  void make_resident(hx_candidates* set) const { check(hx_candidates_make_resident(h_, set)); }
  static uint64_t resident_bytes(const hx_candidates* set) { return hx_candidates_resident_bytes(set); }
  hx_index* raw() const { return h_; }
  uint32_t dimension() const { return dim_; }

 private:
  hx_index* h_ = nullptr;
  uint32_t dim_;
};

// hx_service: the reference's calling pattern — ONE query per call from many concurrent tasks (read_index.rs:81-101) —
// served by shared launches.  search() is the blocking drop-in; submit()/poll() is the pair an async runtime maps a task to.
class SearchService {
 public:
  // borrows an index handle (the owner keeps it alive for the service's lifetime)
  SearchService(hx_index* index, uint32_t k, uint32_t ef = 0, uint32_t capacity = 0, uint32_t max_batch = 0,
                uint32_t ctas_per_sm = 0)
      : k_(k) {
    hx_service_config c{};
    c.k = k;
    c.ef = ef;
    c.capacity = capacity;
    c.max_batch = max_batch;
    c.ctas_per_sm = ctas_per_sm;
    check(hx_service_create(index, &c, &h_));
  }
  explicit SearchService(hx_service* adopt_borrowed, uint32_t k, bool) : h_(adopt_borrowed), k_(k), owned_(false) {}
  ~SearchService() { if (owned_) hx_service_destroy(h_); }
  SearchService(const SearchService&) = delete;
  SearchService& operator=(const SearchService&) = delete;

  uint64_t submit(const float* query) const {
    uint64_t t = 0;
    check(hx_service_submit(h_, query, &t));
    return t;
  }
  // false while the query is running; true once `out` holds its results (the ticket is consumed)
  bool poll(uint64_t ticket, uint64_t* ids, float* scores, uint32_t* count) const {
    int32_t done = 0;
    check(hx_service_poll(h_, ticket, &done, ids, scores, count));
    return done != 0;
  }
  void search(const float* query, uint64_t* ids, float* scores, uint32_t* count) const {
    check(hx_service_search(h_, query, ids, scores, count));
  }
  std::vector<SearchResult> search(const std::vector<float>& query) const {
    std::vector<uint64_t> ids(k_);
    std::vector<float> scores(k_);
    uint32_t count = 0;
    search(query.data(), ids.data(), scores.data(), &count);
    std::vector<SearchResult> out(count);
    for (uint32_t i = 0; i < count; ++i) out[i] = SearchResult{ids[i], scores[i]};
    return out;
  }
  uint32_t k() const { return k_; }
  hx_service* raw() const { return h_; }

 private:
  hx_service* h_ = nullptr;
  uint32_t k_;
  bool owned_ = true;
};

// hx_restricted_service_create: search_restricted with the same calling pattern (read_index.rs:92-101) — one query and
// one candidate set per call, many concurrent tasks — served by shared exact-scan launches.  Answers are bit-identical to
// VectorIndex::search_restricted.  A device set (hx_candidates*) must outlive the tickets that name it.
class RestrictedSearchService {
 public:
  // borrows an index handle (the owner keeps it alive for the service's lifetime)
  RestrictedSearchService(hx_index* index, uint32_t k, uint64_t arena_ids = 0, uint32_t capacity = 0, uint32_t max_batch = 0)
      : k_(k) {
    hx_service_config c{};
    c.k = k;
    c.capacity = capacity;
    c.max_batch = max_batch;
    check(hx_restricted_service_create(index, &c, arena_ids, &h_));
  }
  explicit RestrictedSearchService(hx_service* adopt_borrowed, uint32_t k, bool) : h_(adopt_borrowed), k_(k), owned_(false) {}
  ~RestrictedSearchService() { if (owned_) hx_service_destroy(h_); }
  RestrictedSearchService(const RestrictedSearchService&) = delete;
  RestrictedSearchService& operator=(const RestrictedSearchService&) = delete;

  uint64_t submit(const float* query, const uint64_t* cand_ids, size_t n_cand) const {
    uint64_t t = 0;
    check(hx_service_submit_restricted(h_, query, cand_ids, n_cand, &t));
    return t;
  }
  uint64_t submit(const float* query, const hx_candidates* set) const {
    uint64_t t = 0;
    check(hx_service_submit_restricted_set(h_, query, set, &t));
    return t;
  }
  // false while the query is running; true once `out` holds its results (the ticket is consumed)
  bool poll(uint64_t ticket, uint64_t* ids, float* scores, uint32_t* count) const {
    int32_t done = 0;
    check(hx_service_poll(h_, ticket, &done, ids, scores, count));
    return done != 0;
  }
  void search(const float* query, const uint64_t* cand_ids, size_t n_cand, uint64_t* ids, float* scores,
              uint32_t* count) const {
    check(hx_service_search_restricted(h_, query, cand_ids, n_cand, ids, scores, count));
  }
  std::vector<SearchResult> search(const std::vector<float>& query, const RestrictedVectorCandidates& allowed) const {
    std::vector<uint64_t> ids(k_);
    std::vector<float> scores(k_);
    uint32_t count = 0;
    search(query.data(), allowed.ids().data(), allowed.ids().size(), ids.data(), scores.data(), &count);
    std::vector<SearchResult> out(count);
    for (uint32_t i = 0; i < count; ++i) out[i] = SearchResult{ids[i], scores[i]};
    return out;
  }
  uint32_t k() const { return k_; }
  hx_service* raw() const { return h_; }

 private:
  hx_service* h_ = nullptr;
  uint32_t k_;
  bool owned_ = true;
};

}   // namespace helix
