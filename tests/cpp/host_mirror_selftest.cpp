// Self-test of the C++ host mirror (helix-db_b200/host/vector_index.hpp) LINKED against libhelix_b200.so and executed.
// Device-free checks always run; with a GPU the reference's phase-0 known-answer test (search/vector/index.rs:2318-2411:
// Cosine d=2, m=4 / m0=8 / ef_construction=16, scripted layers [0,1,2,0], strict k=4 ef=16, query (1,0) ->
// [(1,0.0),(2,0.5),(4,0.5),(3,1.0)] bit for bit) and the validation-order KAT (tests/.../vector/search.rs:160-183) run through
// helix::VectorIndex.  Exit code 0 = pass; the last line says which part ran.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>

#include "vector_index.hpp"

static int fails = 0;
#define CHECK(cond)                                                    \
  do {                                                                 \
    if (!(cond)) {                                                     \
      std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond);    \
      ++fails;                                                         \
    }                                                                  \
  } while (0)

template <class F>
static hx_status status_of(F&& f) {
  try {
    f();
  } catch (const helix::HelixDbError& e) {
    return e.code;
  }
  return HX_OK;
}

static uint32_t bits(float x) {
  uint32_t u;
  std::memcpy(&u, &x, 4);
  return u;
}

int main() {
  using namespace helix;
  // ---- device-free: SearchParams (mod.rs:411-621), candidates (restricted.rs:356-371), pure ABI entry points ----
  CHECK(status_of([] { SearchParams p(0); }) == HX_ERR_INVALID_PARAMETER);
  SearchParams p(10);
  CHECK(p.k() == 10 && p.ef() == 100 && p.requires_query_simhash());
  CHECK(status_of([&] { p.with_ef(9); }) == HX_ERR_INVALID_PARAMETER);
  CHECK(status_of([&] { p.with_simhash_bypass_tuning(0, 1, 0.5f, 1); }) == HX_ERR_INVALID_PARAMETER);
  CHECK(status_of([&] { p.with_simhash_bypass_tuning(1, 0, 0.5f, 1); }) == HX_ERR_INVALID_PARAMETER);
  CHECK(status_of([&] { p.with_simhash_bypass_tuning(1, 1, 0.5f, 0); }) == HX_ERR_INVALID_PARAMETER);
  CHECK(status_of([&] { p.with_simhash_bypass_tuning(1, 1, std::nanf(""), 1); }) == HX_ERR_INVALID_PARAMETER);
  CHECK(status_of([&] { p.with_simhash_failure_prob(1.0f); }) == HX_ERR_INVALID_PARAMETER);
  CHECK(status_of([&] { p.with_pre_simhash_sampling_ratio(1.5f); }) == HX_ERR_INVALID_PARAMETER);
  CHECK(p.policy().bypass_min_frontier == 24 && p.policy().bypass_window_expansions == 4 && p.policy().read_budget_multiplier == 3);
  SearchParams off = SearchParams(1).with_simhash_mode(SimHashMode::Off);
  CHECK(!off.requires_query_simhash());
  CHECK(SearchParams(1).with_simhash_mode(SimHashMode::Off).with_pre_simhash_sampling_ratio(0.5f).requires_query_simhash());
  CHECK(!SearchParams::strict(3).requires_query_simhash() && SearchParams::strict(3).raw().pre_sampling_ratio == 1.0f);
  CHECK(p.raw().pre_sampling_ratio < 0.0f);   // Option::None crosses the ABI as a negative
  auto c = RestrictedVectorCandidates::from_ids({7, 7, 3});
  CHECK(c.ids().size() == 2 && c.contains(3) && c.contains(7) && !c.contains(4) && !c.is_empty());
  CHECK(RestrictedVectorCandidates::from_ids({}).is_empty());
  CHECK(hx_order_code_from_simhash_bits(0) == 0 && hx_order_code_from_simhash_bits(1ull << 47) == 1ull << 62);
  CHECK(std::strstr(hx_version(), "sm_90a") != nullptr);
  CHECK(HelixDbError::variant(HX_ERR_ZERO_NORM_COSINE) == "ZeroNormCosineVector");

  // ---- the device: no CPU fallback ----
  bool have_device = true;
  try {
    VectorIndex probe(HX_METRIC_COSINE, 2, 4, 8, 16);
  } catch (const HelixDbError& e) {
    have_device = false;
    CHECK(e.code == HX_ERR_CUDA && std::strstr(e.what(), "no CPU fallback") != nullptr);
  }
  if (!have_device) {
    if (fails) std::printf("host mirror: %d FAILED\n", fails);
    else std::printf("host mirror: device-free checks passed (no GPU: no CPU fallback, as designed)\n");
    return fails ? 1 : 0;
  }
  {
    VectorIndex ix(HX_METRIC_COSINE, 2, 4, 8, 16);
    // empty index: validation errors come first, in the reference's order, then Ok([])
    VectorIndex e3(HX_METRIC_COSINE, 3);
    CHECK(status_of([&] { e3.search({1.0f, 0.0f}, SearchParams::strict(1)); }) == HX_ERR_INVALID_DIMENSION);
    CHECK(status_of([&] { e3.search({1.0f, std::numeric_limits<float>::quiet_NaN(), 0.0f}, SearchParams::strict(1)); }) ==
          HX_ERR_INVALID_VECTOR_COMPONENT);
    CHECK(status_of([&] { e3.search({0.0f, 0.0f, 0.0f}, SearchParams::strict(1)); }) == HX_ERR_ZERO_NORM_COSINE);
    CHECK(e3.search({1.0f, 0.0f, 0.0f}, SearchParams::strict(1)).empty());
    // phase 0: the graph insert_hnsw builds for scripted layers [0,1,2,0] (every pair linked on layer 0; 2-3 on layer 1)
    ix.load_vectors({1, 2, 3, 4}, {1.0f, 0.0f, 0.0f, 1.0f, -1.0f, 0.0f, 0.0f, -1.0f});
    ix.load_graph(0, {1, 2, 3, 4}, {0, 3, 6, 9, 12}, {2, 3, 4, 1, 3, 4, 1, 2, 4, 1, 2, 3});
    ix.load_graph(1, {2, 3}, {0, 1, 2}, {3, 2});
    ix.load_graph(2, {3}, {0, 0}, {});
    ix.set_entry(3, 2);
    SearchParams strict = SearchParams::strict(4);
    strict.with_ef(16);
    auto r = ix.search({1.0f, 0.0f}, strict);
    CHECK(r.size() == 4);
    if (r.size() == 4) {
      const uint64_t want_id[4] = {1, 2, 4, 3};
      const float want_sc[4] = {0.0f, 0.5f, 0.5f, 1.0f};
      for (int i = 0; i < 4; ++i) CHECK(r[i].entity_id == want_id[i] && bits(r[i].score) == bits(want_sc[i]));
    }
    // prefiltered exact scan: tie stability by id, every result inside the candidate set
    auto rr = ix.search_restricted({1.0f, 0.0f}, SearchParams::strict(3), RestrictedVectorCandidates::from_ids({4, 2, 3, 99}));
    CHECK(rr.size() == 3 && rr[0].entity_id == 2 && rr[1].entity_id == 4 && rr[2].entity_id == 3);
    CHECK(ix.search_restricted({1.0f, 0.0f}, SearchParams::strict(3), RestrictedVectorCandidates::from_ids({})).empty());
  }
  if (fails) std::printf("host mirror: %d FAILED\n", fails);
  else std::printf("host mirror: phase-0 KAT and validation order passed on the device\n");
  return fails ? 1 : 0;
}
