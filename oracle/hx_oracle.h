/*
 * hx_oracle.h — CPU restatement of HelixDB's vector-search hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  This is the parity oracle and the CPU baseline of
 * bench.py; nothing in the product path (helix-db_b200/) may include, link or
 * call it.  Every function cites the reference file:line it restates (paths are
 * relative to helix-db/crates/db/src/search/vector/).
 *
 * Pinning: checked against the reference's own known-answer tests (SURVEY §8c,
 * tests/test_oracle_kat.py).  Strict-exhaustive search and the layer-0 policy functions are
 * pinned by values the reference's tests assert.  NOT pinned (the section at the end of this
 * header says exactly what): the stream of the query session RNG (rand 0.10.2 / chacha20 0.10.1
 * are absent from the tree; restated from their published algorithm; the ChaCha12 generator and
 * PCG32 pieces are checked against those crates' published value-stability vectors) and SimHash
 * hyperplane values (never generated here: fingerprints and planes are inputs).
 */
#ifndef HX_ORACLE_H
#define HX_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { HXO_EUCLIDEAN = 0, HXO_COSINE = 1, HXO_MANHATTAN = 2 };

/* same numeric values as hx_status in include/helix_b200.h */
enum {
  HXO_OK = 0,
  HXO_ERR_INDEX_NOT_FOUND = 1,
  HXO_ERR_INVALID_DIMENSION = 2,
  HXO_ERR_INVALID_VECTOR_COMPONENT = 3,
  HXO_ERR_ZERO_NORM_COSINE = 4,
  HXO_ERR_MAGNITUDE_EXCEEDED = 5,
  HXO_ERR_INVALID_VECTOR_CONFIG = 6,
  HXO_ERR_QUERY = 7,
  HXO_ERR_INVARIANT_VIOLATION = 8,
  HXO_ERR_INVALID_PARAMETER = 9
};

/* ---- distance kernels (spaces/simple.rs, spaces/simple_avx.rs) ---- */
float hxo_euclid_scalar(const float* u, const float* v, size_t d);      /* simple.rs:204-218 */
float hxo_dot_scalar(const float* u, const float* v, size_t d);         /* simple.rs:220-234 */
float hxo_manhattan(const float* u, const float* v, size_t d);          /* simple.rs:186-202 */
float hxo_euclid_avx_fma(const float* u, const float* v, size_t d);     /* simple_avx.rs:128-180 (intrinsics) */
float hxo_dot_avx_fma(const float* u, const float* v, size_t d);        /* simple_avx.rs:184-238 (intrinsics) */
float hxo_euclid_avx_fma_portable(const float* u, const float* v, size_t d); /* same order, fmaf() only */
float hxo_dot_avx_fma_portable(const float* u, const float* v, size_t d);
float hxo_euclidean_distance(const float* u, const float* v, size_t d); /* simple.rs:120-144 dispatch: AvxFma iff d>=32 */
float hxo_dot_product(const float* u, const float* v, size_t d);        /* simple.rs:155-177 */
int   hxo_has_avx_fma(void);

/* ---- metric headers and scores (distance/{cosine,euclidean,manhattan}.rs) ---- */
double hxo_scaled_l2_norm(const float* v, size_t d);                    /* cosine.rs:12-36 */
float  hxo_cosine_norm(const float* v, size_t d);                       /* cosine.rs:120-122 */
float  hxo_header(int metric, const float* v, size_t d);                /* new_header: cosine norm, else 0.0 bias */
float  hxo_cosine_distance(const float* p, float pn, const float* q, float qn, size_t d); /* cosine.rs:96-118 */
float  hxo_distance(int metric, const float* p, float p_hdr, const float* q, float q_hdr, size_t d);
/* DistanceScore::try_new (parameters.rs:241-258): finite, >= 0, -0 -> +0. Returns 0 if valid. */
int    hxo_score_validate(float* score);

/* ---- input domain (domain.rs:15-160) ---- */
/* Returns 1 and the limit if the metric has one (Euclidean sqrt(MAX/(8d)), Manhattan MAX/(4d)); 0 for cosine. */
int hxo_component_limit(int metric, size_t d, float* limit);
/* ValidatedMetricVector::try_new order: dimension -> finiteness -> cosine zero -> magnitude. */
int hxo_validate_vector(int metric, size_t expected_d, const float* v, size_t actual_d, uint32_t* bad_index);

/* ---- layer selection (mod.rs:769-796) ---- */
uint16_t hxo_select_layer_from_uniform(float ml, float uniform);
float    hxo_default_ml_for_m(uint32_t m);                               /* mod.rs:705-709 */

/* ---- restricted planning (restricted.rs:40-56,200-213,321-342,426-453) ---- */
int  hxo_restricted_plan(uint64_t n_candidates, uint32_t dimension);     /* 0 Exact, 1 FilteredGraph */
/* RestrictedResultCount::try_new: min(k,|C|), error if > 800 or == 0 */
int  hxo_restricted_result_count(uint32_t k, uint64_t n_candidates, uint32_t* out_k);
/* NonEmptyCandidateSet::deterministic_sample_ids over a sorted id array */
size_t hxo_deterministic_sample_ids(const uint64_t* sorted_ids, size_t n, size_t limit, uint64_t* out);

/* ---- deterministic fixtures from the reference's tests ---- */
/* tests/production_support/index_lifecycle_scale.rs:410-422 (xorshift, d values in [-1,1)) */
void hxo_fixture_xorshift_vector(uint64_t entity_id, uint32_t d, float* out);
/* scale_contracts.rs:44-48 */
void hxo_fixture_circle_vector(uint64_t entity_id, uint64_t entity_count, float* out2);
/* scale_contracts.rs:50-71; returns count written (sorted, unique, self-free) */
size_t hxo_fixture_skip_neighbors(uint64_t entity_id, uint64_t entity_count, uint64_t* out, size_t cap);

/* ---- in-memory index (flat arrays: the reference's algorithm without its KV layer) ---- */
typedef struct hxo_index hxo_index;

typedef struct {
  uint64_t expansion_steps;       /* search.rs:538-541 */
  uint64_t neighbors_examined;    /* search.rs:579-581 */
  uint64_t distance_computations; /* search.rs:511-513,931-933 */
  uint64_t vectors_loaded;        /* search.rs:893-896 (rows fetched, entry excluded) */
  uint64_t upper_layer_steps;
} hxo_stats;

hxo_index* hxo_index_new(int metric, uint32_t dim, uint32_t m, uint32_t m0, uint32_t ef_construction);
void       hxo_index_free(hxo_index* idx);
size_t     hxo_index_len(const hxo_index* idx);
int        hxo_index_state(const hxo_index* idx, uint64_t* entry_point, uint16_t* max_layer); /* 1 populated */
uint32_t   hxo_index_layer0_limit(const hxo_index* idx);                  /* max(m0, 2m) mutation.rs:179-199 */

/* Raw row mirroring (fixtures that seed rows directly, like scale_contracts.rs:96-150). */
int hxo_index_put_vector(hxo_index* idx, uint64_t id, const float* v);    /* validated */
int hxo_index_put_neighbors(hxo_index* idx, uint16_t layer, uint64_t id, const uint64_t* nbrs, size_t n);
int hxo_index_set_entry(hxo_index* idx, uint64_t entry_point, uint16_t max_layer);
/* Bulk: n rows at once (ids ascending or not). */
int hxo_index_put_vectors(hxo_index* idx, const uint64_t* ids, const float* rows, size_t n);

/* insert_with_mutation_cache + insert_hnsw (mutation.rs:642-895) with the layer given by the caller. */
int hxo_index_insert(hxo_index* idx, uint64_t id, const float* v, uint16_t layer);
/* VectorIndex::delete (mutation.rs:1606-1773): removes the node from every layer, re-links every row that named it
 * (delete_from_layer :1819, relink_neighbor :1916), drops its rows / vector / fingerprint and, when it was the entry
 * point, promotes the best live entry candidate (highest layer, then smallest id).  *existed = the item was present. */
int hxo_index_delete(hxo_index* idx, uint64_t id, int* existed);
/* VectorInsertContract::Upsert (mutation.rs:653-661): delete an existing item, then insert */
int hxo_index_upsert(hxo_index* idx, uint64_t id, const float* v, uint16_t layer);

/* Row export (for mirroring into the device index). */
size_t hxo_index_node_ids(const hxo_index* idx, uint64_t* out, size_t cap);            /* ascending */
int    hxo_index_node_level(const hxo_index* idx, uint64_t id);                        /* -1 = no rows */
size_t hxo_index_get_neighbors(const hxo_index* idx, uint16_t layer, uint64_t id, uint64_t* out, size_t cap);
int    hxo_index_get_vector(const hxo_index* idx, uint64_t id, float* out);

/* search_layer_greedy (search.rs:169-224). */
int hxo_search_layer_greedy(const hxo_index* idx, const float* query, uint64_t entry, uint16_t layer,
                            uint64_t* out_node);
/* SearchSession::run, strict-exhaustive (search.rs:1101-1230 + :267-1067 STRICT_EXHAUSTIVE). */
int hxo_search(const hxo_index* idx, const float* query, uint32_t query_dim, uint32_t k, uint32_t ef,
               uint64_t* out_ids, float* out_scores, uint32_t* out_count, hxo_stats* stats);
/* restricted_exact_scan (restricted.rs:753-835) for any |C| (ids ascending unique). */
int hxo_search_restricted(const hxo_index* idx, const float* query, uint32_t query_dim, uint32_t k,
                          const uint64_t* cand_ids, size_t n_cand, uint64_t* out_ids, float* out_scores,
                          uint32_t* out_count, uint64_t* distance_computations);

/* Filter-aware (ACORN-style) restricted search, V/restricted.rs:837-1148, for generations without the SimHash routing
 * directory: seeds = deterministic sample + entry point, bridges through non-members ranked by SimHash Hamming distance.
 * Needs the node fingerprints (hxo_index_put_simhash) and the query's.  Approximate by design (the reference's recall
 * gate for this branch is 0.92); restated so that the device walk can be compared with it step for step.
 * Pinned by: the budgets' closed forms and deterministic_sample_ids literals (tests/production_support/vector/
 * restricted.rs:532-551); SimHash VALUES are inputs (unpinned, see below). */
enum { HXO_FG_NONE = 0, HXO_FG_VECTOR_BUDGET = 1, HXO_FG_BEAM_COMPLETE = 2, HXO_FG_EXHAUSTED = 3, HXO_FG_ROUTING_BUDGET = 4,
       HXO_FG_BRIDGE_BUDGET = 5 };
typedef struct {
  uint64_t vector_payload_requests, distance_computations, routing_rows, bridge_rows, bridge_frontier_pushes,
      simhash_row_requests;
  uint32_t termination, reserved;
} hxo_filtered_stats;
typedef struct { size_t ef_filtered, routing_rows, bridge_rows, vector_payloads, sampled_seeds; } hxo_filtered_budgets_t;
void hxo_filtered_budgets(uint32_t k, uint32_t ef, uint32_t beam_percent, size_t n_cand, hxo_filtered_budgets_t* out);
int hxo_search_filtered_graph_budgets(const hxo_index* idx, const float* query, uint32_t k,
                                      const hxo_filtered_budgets_t* budgets, const uint64_t* cand_ids, size_t n_cand,
                                      uint64_t query_simhash, uint64_t* out_ids, float* out_scores, uint32_t* out_count,
                                      hxo_filtered_stats* stats);
int hxo_search_filtered_graph(const hxo_index* idx, const float* query, uint32_t k, uint32_t ef, uint32_t beam_percent,
                              const uint64_t* cand_ids, size_t n_cand, uint64_t query_simhash, uint64_t* out_ids,
                              float* out_scores, uint32_t* out_count, hxo_filtered_stats* stats);


/* exact top-k over the whole index (ground truth for recall), same (score,id) rule. */
int hxo_search_exact(const hxo_index* idx, const float* query, uint32_t k, uint64_t* out_ids,
                     float* out_scores, uint32_t* out_count);

/* Threaded drivers: one query per thread at a time (the reference's one-query-per-tokio-task model).
 * Return wall seconds spent in the parallel region. */
double hxo_search_batch(const hxo_index* idx, const float* queries, size_t nq, uint32_t k, uint32_t ef,
                        int threads, uint64_t* out_ids, float* out_scores, uint32_t* out_counts,
                        hxo_stats* stats_sum);
double hxo_search_restricted_batch(const hxo_index* idx, const float* queries, size_t nq, uint32_t k,
                                   const uint64_t* cand_ids, const uint64_t* cand_offsets, int threads,
                                   uint64_t* out_ids, float* out_scores, uint32_t* out_counts);
double hxo_search_exact_batch(const hxo_index* idx, const float* queries, size_t nq, uint32_t k, int threads,
                              uint64_t* out_ids, float* out_scores, uint32_t* out_counts);

/* Bulk graph import in slot space (slot = rank of id ascending), as downloaded from the device. */
int hxo_index_import_graph(hxo_index* idx, const uint16_t* levels, const uint32_t* deg0, const uint32_t* nbr0,
                           uint32_t layer0_stride, size_t n_upper_rows, const uint32_t* upper_node,
                           const uint16_t* upper_layer, const uint32_t* upper_deg, const uint32_t* upper_nbr,
                           uint32_t upper_stride, uint64_t entry_point, uint16_t max_layer);


/* ====================================================================================================
 * Non-exhaustive layer-0 search: SimHash filtering, sampling, adaptive bypass (SimHashMode::{Adaptive,Always},
 * or Off with a pre-sampling override < 1).  Restates policy.rs:52-597, randomness.rs:96-165,
 * unaligned_vector/simhash.rs:20-55,263-290, simhash.rs:44-59 and search.rs:267-1067 with STRICT_EXHAUSTIVE=false.
 *
 * Pinning: the policy functions are pinned by the literals of the reference's own policy tests
 * (policy.rs:641-1010: thresholds, probabilities, bypass window transitions; tests/test_oracle_kat.py).
 * PARITY UNPINNED BY THE TREE: (1) the values drawn from the query session RNG — rand 0.10.2 `StdRng` = ChaCha12 seeded
 * through rand_core's `seed_from_u64` (PCG32 expansion), `random::<f32>()` = (next_u32 >> 8) * 2^-24,
 * `random_range(0..n)` = widening-multiply with one bias-correction draw — are restated from the published algorithms
 * of those crates (absent from the reference repository; no committed value pins them; the reference's own tests only compare
 * two instances of the generator).  What narrows that gap (tests/test_oracle_kat.py, vectors quoted from the published
 * crates' own value-stability tests, not from a file in the tree): the ChaCha12 stream — round count, counter / stream
 * start, word order, `from_rng` re-seeding — reproduces rand's `test_stdrng_construction` (10719222850664546238,
 * 14064965282130556830) and rand_chacha's `test_chacha_construction` (137206642, 1325750369); PCG32's LCG step and
 * XSH-RR permutation reproduce the PCG reference demo stream (0xa15c02b7, 0x7b47f409, ...).  Still resting on the
 * restatement alone: seed_from_u64's increment constant and advance-then-output order, the f32 conversion, and the
 * range reduction of `random_range`; (2) SimHash hyperplanes (StdRng(42) Gaussian draws) are never generated here: node and query
 * fingerprints are INPUTS (the reference persists them as [0x12] rows), or are projected from caller-supplied planes.
 * The RNG is consulted only for frontiers larger than max(ef/4, 8) (policy.rs:526-556), i.e. rarely at ef=100, m0=32.
 * SimHash "filter reads" follow the resident-store case (memory_store.rs:331-337: no KV read, so the read budget of
 * the adaptive bypass is never consumed), which is what a device-resident mirror is.
 * ==================================================================================================== */
enum { HXO_SIMHASH_OFF = 0, HXO_SIMHASH_ADAPTIVE = 1, HXO_SIMHASH_ALWAYS = 2 };
enum { HXO_BYPASS_READY = 0, HXO_BYPASS_BYPASSING = 1, HXO_BYPASS_COOLING = 2 };
enum { HXO_TRIGGER_NONE = 0, HXO_TRIGGER_READ_BUDGET = 1, HXO_TRIGGER_LOW_YIELD = 2, HXO_TRIGGER_BOTH = 3 };
enum { HXO_SAMPLING_EXHAUSTIVE = 0, HXO_SAMPLING_FIXED = 1, HXO_SAMPLING_ADAPTIVE = 2 };

typedef struct {              /* index config (config/indexes.rs:398-406) + SearchParams (mod.rs:411-500) */
  int32_t  mode;              /* HXO_SIMHASH_*; SearchParams::new => Adaptive                         */
  uint32_t threshold;         /* simhash_threshold, 0..64 (default 43)                                */
  float    sampling_ratio;    /* index sampling_ratio (0.8) or the per-query override                 */
  int32_t  has_pre_override;  /* pre_simhash_sampling_ratio_override.is_some()                        */
  float    pre_override;
  int32_t  adaptive_enabled;  /* index adaptive_enabled (true)                                        */
  float    failure_prob;      /* adaptive_failure_prob (0.1) or the per-query override                */
  uint32_t bypass_min_frontier;        /* 24 */
  uint32_t bypass_window_expansions;   /* 4  */
  float    bypass_min_filter_rate;     /* 0.12 */
  uint32_t read_budget_multiplier;     /* 3  */
} hxo_policy_cfg;
void hxo_policy_defaults(hxo_policy_cfg* cfg);   /* SearchParams::new + VectorIndexConfig defaults */

typedef struct {              /* SimHashContext (policy.rs:385-395) */
  int32_t  topk_ready;
  uint32_t ef, search_frontier_len, candidate_frontier_len;
  float    current, delta;
  int32_t  bypass_state;      /* HXO_BYPASS_* */
  uint32_t bypass_remaining;
  uint64_t simhash_filter_reads, window_examined, window_filtered, window_expansions;
} hxo_policy_ctx;

typedef struct {              /* SimHashDecision (policy.rs:433-448) */
  int32_t  fetch_missing, filter_cached, has_threshold;
  uint32_t threshold;
  int32_t  pre_kind;  float pre_prob;     /* SamplingDecision + probability() */
  int32_t  samp_kind; float samp_prob;
  float    base_sampling_probability;
  int32_t  bypassed, next_state;
  uint32_t next_remaining;
  int32_t  trigger;
} hxo_policy_decision;
/* Layer0Policy::from_deployed(..).with_adaptive_bypass(AdaptiveBypassPolicy::from_deployed(..)).decide(ctx) */
void  hxo_policy_decide(int metric, const hxo_policy_cfg* cfg, const hxo_policy_ctx* ctx, hxo_policy_decision* out);
/* SamplingDecision::candidate_probability (policy.rs:415-430) */
float hxo_candidate_probability(const hxo_policy_decision* d, uint32_t similarity_bits);

/* SearchSession (randomness.rs:122-165) over StdRng = ChaCha12 (see the header note: unpinned). */
typedef struct { uint64_t seed; int32_t started; uint32_t key[8]; uint64_t block; uint32_t buf[16]; uint32_t pos; } hxo_session;
void     hxo_session_seeded(hxo_session* s, uint64_t seed);
uint64_t hxo_session_seed_for(uint64_t query_simhash, uint64_t entry_point, uint64_t ef);  /* randomness.rs:109-114 */
uint32_t hxo_session_next_u32(hxo_session* s);
/* the two halves of rand_core's seed_from_u64 expansion: PCG's LCG step and its XSH-RR output permutation */
uint32_t hxo_pcg32_xsh_rr(uint64_t state);
uint64_t hxo_pcg32_step(uint64_t state, uint64_t increment);
/* the ChaCha block function itself (words 12-13 = counter, 14-15 = stream); pinned by RFC 7539 2.3.2 at 20 rounds */
void     hxo_chacha_block(const uint32_t key[8], uint64_t counter, uint64_t stream, int rounds, uint32_t out[16]);
int      hxo_session_should_sample(hxo_session* s, float ratio);           /* :141-153 */
int64_t  hxo_session_choose_index(hxo_session* s, uint64_t count);         /* :155-158; -1 = None */

/* SimHash (unaligned_vector/simhash.rs): hash_from_slice over caller-supplied planes [64][dim]; order code. */
uint64_t hxo_simhash_from_planes(const float* planes, const float* v, uint32_t dim);   /* :263-290 */
uint32_t hxo_simhash_collision_count(uint64_t a, uint64_t b);                          /* :37-40 */
uint64_t hxo_order_code_from_simhash_bits(uint64_t bits);                              /* simhash.rs:44-59 */

typedef struct {              /* the SimHash-related SearchStats counters (mod.rs:640-700) */
  uint64_t simhash_filtered, simhash_examined, simhash_missing_hash, simhash_passed_before_sampling,
      simhash_passed_after_sampling, simhash_bypass_expansions, simhash_skipped_candidates, pre_simhash_sample_kept,
      pre_simhash_sample_dropped, simhash_bypass_trigger_budget, simhash_bypass_trigger_low_yield, rng_draws;
} hxo_policy_stats;

/* Node fingerprints ([0x12] rows).  A node without one behaves as SimHashRow::Missing (not filtered, similarity 32). */
int hxo_index_put_simhash(hxo_index* idx, const uint64_t* ids, const uint64_t* bits, size_t n);
/* SearchSession::run with the given policy and query fingerprint (search.rs:1101-1230, :267-1067). */
int hxo_search_policy(const hxo_index* idx, const float* query, uint32_t query_dim, uint32_t k, uint32_t ef,
                      const hxo_policy_cfg* cfg, uint64_t query_simhash, uint64_t* out_ids, float* out_scores,
                      uint32_t* out_count, hxo_stats* stats, hxo_policy_stats* pstats);
/* threaded driver (one query per thread at a time); returns wall seconds, < 0 on error */
double hxo_search_policy_batch(const hxo_index* idx, const float* queries, const uint64_t* query_simhash, size_t nq,
                               uint32_t k, uint32_t ef, const hxo_policy_cfg* cfg, int threads, uint64_t* out_ids,
                               float* out_scores, uint32_t* out_counts);

#ifdef __cplusplus
}
#endif
#endif
