/*
 * helix_b200.h — C ABI of the CUDA (H100, sm_90a) vector-search inner loop for HelixDB.
 *
 * This is the drop-in boundary.  Every entry point is `extern "C"`, takes plain
 * pointers and sizes, returns an `hx_status` (0 = OK) and never throws or aborts.
 * The reference (HelixDB, 100 % Rust) exposes no FFI for this path; the natural
 * seam is the pair of methods every production vector query funnels through:
 *
 *   ValidatedVectorReadIndex::<D>::search             crates/db/src/search/vector/read_index.rs:81-90
 *   ValidatedVectorReadIndex::<D>::search_restricted  crates/db/src/search/vector/read_index.rs:92-101
 *     -> VectorIndex::<D>::search                     crates/db/src/search/vector/index.rs:1578-1587
 *     -> VectorIndex::<D>::search_restricted          crates/db/src/search/vector/restricted.rs:466-479
 *
 * reached from the planner operators ExecNodeAccessPlan::VectorSearch
 * (crates/planner/src/exec/access/node.rs:69-78) and ExecOp::VectorSearch
 * (crates/planner/src/exec/op/operation.rs:26-29).  INTEGRATION.md shows the
 * Rust `extern "C"` block a maintainer would add on the reference side.
 *
 * The device index is a *disposable mirror* of the reference's KV rows (like its
 * resident VectorMemoryStore, memory_store.rs:97-130): vectors, per-row headers
 * (cosine norm), the layer-0 and upper-layer neighbour rows, entry point and
 * max layer are uploaded once and searched many times.
 *
 * Threading: an `hx_index*` may be searched concurrently from several host
 * threads: each host-buffer call takes a private stream + scratch block from a
 * pool (64 per handle, then callers queue), device-buffer calls use one scratch
 * set per caller stream, and the first search after a load finalises the graph
 * image under a lock.  One-query-per-call traffic belongs on an hx_service
 * (below), which coalesces concurrent callers into shared launches.
 * load/build calls must not overlap searches on the same handle.
 */
#ifndef HELIX_B200_H
#define HELIX_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes ------------------------------------------------------- */
/* Mirrors the HelixDbError variants the reference can return on this path
 * (crates/db/src/error.rs:379,415,433,467,631-661).  Query validation happens
 * before any traversal and in this order: dimension -> finiteness -> cosine
 * zero norm -> component magnitude (domain.rs:113-154). */
typedef int32_t hx_status;
enum {
  HX_OK = 0,
  HX_ERR_INDEX_NOT_FOUND = 1,          /* HelixDbError::IndexNotFound (null / destroyed handle)        */
  HX_ERR_INVALID_DIMENSION = 2,        /* HelixDbError::InvalidDimension{expected,got}                  */
  HX_ERR_INVALID_VECTOR_COMPONENT = 3, /* HelixDbError::InvalidVectorComponent{index} (NaN / Inf)       */
  HX_ERR_ZERO_NORM_COSINE = 4,         /* HelixDbError::ZeroNormCosineVector                             */
  HX_ERR_MAGNITUDE_EXCEEDED = 5,       /* HelixDbError::VectorComponentMagnitudeExceeded{..}             */
  HX_ERR_INVALID_VECTOR_CONFIG = 6,    /* HelixDbError::InvalidVectorConfig                              */
  HX_ERR_QUERY = 7,                    /* HelixDbError::Query(String): >1e6 candidates, restricted k>800 */
  HX_ERR_INVARIANT_VIOLATION = 8,      /* HelixDbError::InvariantViolation: NaN/negative score, bad rows */
  HX_ERR_INVALID_PARAMETER = 9,        /* VectorParameterError: k == 0, ef < k, null pointer             */
  HX_ERR_CUDA = 10,                    /* a CUDA runtime call failed (see hx_last_error)                 */
  HX_ERR_OUT_OF_MEMORY = 11,
  HX_ERR_UNSUPPORTED = 12              /* a mode or size the device path does not execute                */
};

/* ---- metrics -------------------------------------------------------------- */
/* D in {Euclidean, Cosine, Manhattan} (search/dispatch.rs:127-188).
 * Scores: Euclidean = squared L2 (spaces/simple.rs:204-218),
 *         Cosine    = (1 - cos)/2 in [0,1] (distance/cosine.rs:96-118),
 *         Manhattan = L1 (spaces/simple.rs:186-202).  All f32. */
typedef enum {
  HX_METRIC_EUCLIDEAN = 0,
  HX_METRIC_COSINE = 1,
  HX_METRIC_MANHATTAN = 2
} hx_metric;

/* ---- index configuration --------------------------------------------------- */
/* Mirrors VectorIndexDefinition / VectorIndexConfig defaults
 * (crates/db/src/config/indexes.rs:374-408): m=16, m0=32, ef_construction=200. */
typedef struct {
  uint32_t dimension;       /* > 0                                                     */
  int32_t  metric;          /* hx_metric                                               */
  uint32_t m;               /* upper-layer degree limit                                */
  uint32_t m0;              /* configured layer-0 degree; effective = max(m0, 2m)      */
  uint32_t ef_construction; /* used by hx_index_build                                  */
  int32_t  device;          /* CUDA device ordinal (one process per GPU: LOCAL_RANK)   */
  uint32_t storage;         /* 0 = f32 rows (parity path), 1 = also keep a bf16 copy
                               for the tensor-core batched path (hx_search_dense)     */
  uint32_t reserved;
} hx_index_config;

/* ---- per-query parameters ---------------------------------------------------- */
/* Mirrors SearchParams (search/vector/mod.rs:411-621).  SearchParams::new(k):
 * ef = max(k, 100), SimHashMode::Adaptive.  mode HX_SIMHASH_OFF + pre_sampling_ratio 1.0 is the
 * reference's strict-exhaustive specialisation (STRICT_EXHAUSTIVE, search.rs:296-304,595-596), whose
 * results the reference pins by value.  ADAPTIVE / ALWAYS (the production default) run the
 * SimHash filtering / sampling / adaptive-bypass policy of search.rs:595-992 + policy.rs; they need the node
 * fingerprints (hx_index_load_simhash or hx_index_compute_simhash) and are checked against the CPU oracle's
 * restatement; see hx_search_ex for what the reference itself pins there. */
typedef enum { HX_SIMHASH_OFF = 0, HX_SIMHASH_ADAPTIVE = 1, HX_SIMHASH_ALWAYS = 2 } hx_simhash_mode;

typedef struct {
  uint32_t k;                  /* results per query, > 0                                */
  uint32_t ef;                 /* beam width, >= k; 0 => max(k,100)                    */
  int32_t  simhash_mode;       /* hx_simhash_mode                                       */
  float    pre_sampling_ratio; /* pre_simhash_sampling_ratio_override: a value in [0,1] = Some(v), negative = None.
                                  OFF + 1.0 (or OFF + None) is the strict-exhaustive specialisation; every other
                                  combination runs the policy kernel (hx_search_ex semantics, default policy params) */
  uint32_t collect_stats;      /* fill hx_stats (per-call sums)                         */
  uint32_t query_dimension;    /* length of each query as the caller holds it; 0 = the
                                  index dimension.  A mismatch is InvalidDimension and is
                                  reported before any other check (domain.rs:117-122)   */
} hx_search_params;

/* Counter semantics mirror SearchStats (search/vector/mod.rs:668-679):
 * expansion_steps counts every candidate pop including the one that triggers the
 * stop test (search.rs:538-551); neighbors_examined sums full row lengths before
 * the visited filter (:579-581); distance_computations includes the entry point
 * (:511-513).  Sums over the B queries of the call. */
typedef struct {
  uint64_t expansion_steps;
  uint64_t neighbors_examined;
  uint64_t distance_computations;
  uint64_t vectors_loaded;
  uint64_t upper_layer_steps;   /* greedy moves above layer 0 (not in the reference's stats) */
  uint64_t algorithmic_bytes;   /* E*(5+8*deg) + Dc*(4+4d), SURVEY §8(d)                    */
  uint64_t kernel_launches;     /* launches of OUR kernels issued by the call               */
  uint64_t reserved;
} hx_stats;

typedef struct hx_index hx_index;

/* ---- lifecycle ------------------------------------------------------------------ */
hx_status hx_index_create(const hx_index_config* cfg, hx_index** out);
void      hx_index_destroy(hx_index* idx);

/* Upload n rows.  `ids` need not be sorted; rows are re-ordered so that device slot
 * order == ascending id order (the reference canonicalises neighbour rows to
 * ascending node id, encoding/v1/values/vectors.rs:67-110, so slot order makes the
 * (score, id) tie rule a single 64-bit compare).  Every row is validated like
 * decode_item_borrowed (mod.rs:889-949): finite, magnitude bound, non-zero for
 * cosine.  Replaces any previous contents. */
hx_status hx_index_load_vectors(hx_index* idx, const uint64_t* ids, const float* rows, size_t n);

/* Generate unit-normalised synthetic vectors on the device instead (bench only; no PCIe copy),
 * ids = first_id..first_id+n-1, keyed by the global id so id-range shards reproduce the corpus.
 * kind 0      : isolated isotropic Gaussian clusters in full dimension (the SURVEY §8d recipe);
 * kind r=2..64: Gaussian mixture in an r-dimensional latent space pushed through a fixed random
 *               projection (+2 % isotropic noise): intrinsic dimension ~r, like real embeddings.
 * Queries from the same distribution: hx_generate_queries. */
hx_status hx_index_generate_vectors(hx_index* idx, uint64_t first_id, size_t n, uint64_t seed,
                                    uint32_t n_centroids, float sigma, uint32_t kind);
hx_status hx_generate_queries(hx_index* idx, uint64_t seed, uint32_t n_centroids, float sigma,
                              uint64_t first_query, size_t n_queries, float* out_host, uint32_t kind);
/* Copy rows [first_slot, first_slot+n) (slot order) back to the host (f32, n*dimension). */
hx_status hx_index_download_vectors(hx_index* idx, size_t first_slot, size_t n, float* out_rows,
                                    uint64_t* out_ids);

/* Mirror one HNSW layer.  layer 0 rows = layer-0 neighbour rows
 * `[0x12][count u32 BE][id u64 BE x <= m0]`, layers >= 1 = upper rows
 * (encoding/v1/values/vectors/neighbors.rs:57-76) — passed here decoded, CSR style:
 * node_ids[i] owns neighbors[offsets[i] .. offsets[i+1]).  Neighbour ids without a
 * vector row are kept out of the device rows but still counted in
 * neighbors_examined (the reference skips them at fetch time, search.rs:909-913). */
hx_status hx_index_load_graph(hx_index* idx, uint16_t layer, const uint64_t* node_ids,
                              const uint32_t* offsets, const uint64_t* neighbors, size_t n_nodes);
/* VectorIndexState::Populated{entry_point,max_layer} (configuration.rs). */
hx_status hx_index_set_entry(hx_index* idx, uint64_t entry_point, uint16_t max_layer);

/* ---- row-image import / export (SURVEY §8(f).2) ----------------------------------------------
 * The reference's encoded row VALUES are accepted as they are stored, so hydration needs no
 * decode step on the Rust side.
 *  vector item rows  `[header f32][f32 x dimension]`, native endian, 4+4*dimension bytes each
 *      (encode_item, search/vector/mod.rs:866-871; golden bytes magnitude_regressions.rs:333-338).
 *      Checked like decode_item_borrowed (mod.rs:889-949): exact length, finite components,
 *      magnitude bound, and the stored header must equal the recomputed one bit for bit
 *      (cosine norm / 0.0 bias) — otherwise HX_ERR_INVARIANT_VIOLATION (HeaderMismatch).
 *  neighbour rows: layer 0  = empty | `[0x12][count u32 BE][id u64 BE...]`
 *                             | `[0x13][flags][count u32 BE][simhash u64 LE if flags&1][id u64 BE...]`
 *                  (encoding/v1/values/vectors.rs:26-200),
 *                  layer>=1 = `[count u32 BE][id u64 BE...]` (values/vectors/neighbors.rs:57-110).
 *      Exact lengths are required (trailing bytes are corruption). */
hx_status hx_index_load_vector_rows(hx_index* idx, const uint64_t* ids, const uint8_t* rows, size_t n);
hx_status hx_index_load_neighbor_rows(hx_index* idx, uint16_t layer, const uint64_t* node_ids,
                                      const uint8_t* blob, const uint64_t* row_offsets /* n+1 */, size_t n);
/* Pure codecs (no device needed). decode: returns the ids (and the SimHash bits of a 0x13 row). */
hx_status hx_decode_neighbor_row(uint16_t layer, const uint8_t* row, size_t len, uint64_t* out_ids,
                                 size_t cap, size_t* out_count, uint64_t* out_simhash, int32_t* out_has_simhash);
hx_status hx_encode_neighbor_row(uint16_t layer, const uint64_t* ids, size_t n, uint8_t* out, size_t cap,
                                 size_t* out_len);
/* Encode one row of the device graph (e.g. after hx_index_build) for persistence through the
 * reference's normal mutation path. */
hx_status hx_index_export_neighbor_row(hx_index* idx, uint16_t layer, uint64_t node_id, uint8_t* out,
                                       size_t cap, size_t* out_len);

/* ---- row KEYS of the vector families the mirror consumes (encoding/v1/keys/vectors.rs:23-52) -------
 *  HX_KEY_VECTOR           `[0xF1][index_id u64 BE][0x02][order_code u64 BE][node_id u64 BE]`  (:805-892)
 *  HX_KEY_LAYER0_NEIGHBORS `[0xF0][index_id][0x16][node_id]`                                   (:673-745)
 *  HX_KEY_UPPER_NEIGHBORS  `[0xF0][index_id][0x11][layer u16 BE][node_id]`                     (:1370-1457)
 *  HX_KEY_SIMHASH          `[0xF0][index_id][0x12][node_id]`                                   (:1459-1530)
 *  HX_KEY_UPPER_VECTOR     `[0xF0][index_id][0x13][node_id]`                                   (:1532-1603)
 *  HX_KEY_METADATA         `[0x03][0x03][index_id][0x01]`                                      (:479-544)
 * Exact lengths are required, like VectorKey::parse_from_slice (:311-470); any other vector-keyspace
 * key (prefix keys, entry candidates, reverse edges, directory, txn guard) parses as HX_KEY_OTHER so a
 * hydration loop can skip it; a key outside the vector keyspaces or with a wrong length for its kind
 * is HX_ERR_INVARIANT_VIOLATION. */
typedef enum {
  HX_KEY_OTHER = 0,
  HX_KEY_VECTOR = 1,
  HX_KEY_LAYER0_NEIGHBORS = 2,
  HX_KEY_UPPER_NEIGHBORS = 3,
  HX_KEY_SIMHASH = 4,
  HX_KEY_UPPER_VECTOR = 5,
  HX_KEY_METADATA = 6
} hx_key_kind;
typedef struct {
  int32_t  kind;        /* hx_key_kind */
  uint16_t layer;       /* HX_KEY_UPPER_NEIGHBORS only */
  uint16_t reserved;
  uint64_t index_id;
  uint64_t order_code;  /* HX_KEY_VECTOR only (SimHash-interleaved locality code, simhash.rs:44-59) */
  uint64_t node_id;
} hx_vector_key;
hx_status hx_parse_vector_key(const uint8_t* key, size_t len, hx_vector_key* out);
hx_status hx_encode_vector_key(const hx_vector_key* key, uint8_t* out, size_t cap, size_t* out_len);

/* ---- incremental mirror maintenance (SURVEY §8(f).2; memory_store.rs:105-130, read_index.rs:53-65) ------------
 * A committed write reaches the mirror as ROW PATCHES — the rows the write made dirty on the Rust side
 * (VectorMemoryDirtyRows: dirty_nodes + dirty_upper_neighbors) — followed by a new version token:
 *   hx_index_upsert_vectors        vector rows: an existing id is overwritten in place, an id above the current
 *                                  maximum is appended (ids come from a monotonic allocator); an absent id INSIDE the
 *                                  mirrored range would renumber the slots -> HX_ERR_UNSUPPORTED, re-hydrate
 *   hx_index_set_levels            the HNSW level of new nodes (allocates their empty upper rows, mutation.rs:706-739)
 *   hx_index_upsert_neighbor_rows  replaces the layer's rows of the given nodes (decoded CSR as in hx_index_load_graph)
 *   hx_index_load_simhash          (above) patches fingerprints by id
 *   hx_index_delete_vectors        the node can no longer be scored or returned; its former neighbours' repaired rows
 *                                  arrive as upserts; deleting the entry point needs a following hx_index_set_entry
 *   hx_index_set_entry             (above) new entry point / max layer
 *   hx_index_load_upper_vector_rows  `[0x13]` hot-lane item rows: inserted when the node is new, otherwise required to be
 *                                  byte-identical to the canonical row (a stale hot-lane row is an InvariantViolation)
 *   hx_index_set_version           the (generation identity, visible sequence) this image now corresponds to; the Rust
 *                                  read guard compares it with the request's snapshot before dispatching a search here
 * Patch calls must not overlap searches on the same handle (the Rust side holds its write lock, as it does around the
 * resident cache's publish).  The rkyv metadata row is decoded on the Rust side: entry point and max layer cross the
 * ABI as the two scalars of hx_index_set_entry. */
hx_status hx_index_upsert_vectors(hx_index* idx, const uint64_t* ids, const float* rows, size_t n);
hx_status hx_index_set_levels(hx_index* idx, const uint64_t* ids, const uint16_t* levels, size_t n);
hx_status hx_index_upsert_neighbor_rows(hx_index* idx, uint16_t layer, const uint64_t* node_ids,
                                        const uint32_t* offsets, const uint64_t* neighbors, size_t n_nodes);
hx_status hx_index_delete_vectors(hx_index* idx, const uint64_t* ids, size_t n);
hx_status hx_index_load_upper_vector_rows(hx_index* idx, const uint64_t* ids, const uint8_t* rows, size_t n);
hx_status hx_index_set_version(hx_index* idx, uint64_t generation, uint64_t visible_seq);
hx_status hx_index_get_version(hx_index* idx, uint64_t* generation, uint64_t* visible_seq, uint64_t* patches_applied);

/* Build the HNSW graph on the device from the loaded vectors (SURVEY §8(f).1:
 * insert_hnsw / search_layer_beam / select_diverse / add_bidirectional_link,
 * mutation.rs:787-1005,1498-1591, restated as batched concurrent insertion).
 * `levels` (n entries, slot order of ascending id) may be NULL => drawn from `seed`
 * with select_layer's law floor(-ln(U)*ml), ml = 1/ln(m) (mod.rs:769-796). */
hx_status hx_index_build(hx_index* idx, const uint16_t* levels, uint64_t seed);
/* Build modes.  HX_BUILD_BATCHED (hx_index_build): rounds of concurrent insertions — fast (1M x 768 in seconds), same
 * structural invariants and recall class as the reference, but not the same graph (nodes of one round do not see each
 * other).  HX_BUILD_SEQUENTIAL: one insert_hnsw at a time, the links of each insert applied in selection order
 * (add_bidirectional_link, mutation.rs:1498-1591) — the graph is IDENTICAL to the reference's for the same insertion
 * order (ascending id) and level assignment; two launches per node, meant for parity runs and small indexes (config C1). */
enum { HX_BUILD_BATCHED = 0, HX_BUILD_SEQUENTIAL = 1 };
hx_status hx_index_build_ex(hx_index* idx, const uint16_t* levels, uint64_t seed, int32_t mode);

/* Download the graph (for the CPU oracle to traverse the identical adjacency). */
hx_status hx_index_graph_info(hx_index* idx, uint64_t* n_nodes, uint64_t* entry_point,
                              uint16_t* max_layer, uint32_t* layer0_stride, uint32_t* upper_stride);
hx_status hx_index_download_graph(hx_index* idx, uint16_t* levels /*n*/, uint32_t* deg0 /*n*/,
                                  uint32_t* nbr0 /*n*layer0_stride, slot numbers*/,
                                  uint64_t* n_upper_rows, uint32_t* upper_node /*cap*/,
                                  uint16_t* upper_layer /*cap*/, uint32_t* upper_deg /*cap*/,
                                  uint32_t* upper_nbr /*cap*upper_stride*/, size_t upper_cap);

/* ---- search (host buffers: the reference-facing call) ------------------------------ */
/* VectorIndex::search (index.rs:1578) -> SearchSession::run (search.rs:1101-1230):
 * validate query, greedy descent layers max_layer..1 (search.rs:169-224), layer-0
 * beam (search.rs:267-1067, strict-exhaustive), results sorted by (score,id),
 * truncated to k.  B independent queries, no cross-query sharing.
 * out_ids/out_scores are B*k; out_counts[b] <= k.  Empty index => counts 0, HX_OK. */
hx_status hx_search(hx_index* idx, const float* queries, size_t B, const hx_search_params* p,
                    uint64_t* out_ids, float* out_scores, uint32_t* out_counts, hx_stats* stats);

/* VectorIndex::search_restricted (restricted.rs:466-613), exact branch
 * restricted_exact_scan (restricted.rs:753-835) executed for ANY |C| <= 1e6.
 * cand_ids: ascending unique u64 (RoaringTreemap iteration order), shared by the B
 * queries.  k is clamped to |C| and must then be <= 800 (restricted.rs:200-213).
 * Empty candidate set => counts 0 before any device work (restricted.rs:539-541). */
hx_status hx_search_restricted(hx_index* idx, const float* queries, size_t B,
                               const hx_search_params* p, const uint64_t* cand_ids, size_t n_cand,
                               uint64_t* out_ids, float* out_scores, uint32_t* out_counts,
                               hx_stats* stats);
/* Same, one candidate set per query: query b owns cand_ids[cand_offsets[b]..cand_offsets[b+1]). */
hx_status hx_search_restricted_multi(hx_index* idx, const float* queries, size_t B,
                                     const hx_search_params* p, const uint64_t* cand_ids,
                                     const uint64_t* cand_offsets, uint64_t* out_ids,
                                     float* out_scores, uint32_t* out_counts, hx_stats* stats);

/* ---- filter-aware (ACORN-style) restricted search (restricted.rs:837-1148) -------------------------------------
 * The walk the reference plans for |C| > 256 (restricted.rs:426-453), for generations without the SimHash routing
 * directory: seeds = the evenly spaced sample of the candidate set + the entry point when it is a candidate; the best
 * scored candidates' layer-0 rows are routed 16 at a time; neighbours outside the candidate set become bridges ranked by
 * SimHash Hamming distance to the query and are expanded (never scored) up to 256 at a time; at most 800 candidate vectors
 * are scored.  Approximate by design (the reference gates it at recall 0.92); hx_search_restricted answers the same
 * question exactly and is the better choice until |C| x row bytes dominates (bench.py reports the cross-over).
 * Needs the node fingerprints (hx_index_load_simhash / hx_index_compute_simhash) and the queries' (given, or projected
 * from the planes).  budgets == NULL: FilteredGraphBudgets::with_beam_percent(params, k, |C|, 150).  One candidate set for
 * the B queries.  A neighbour without its SimHash row fails the call (InvariantViolation, "missing simhash"). */
typedef struct { uint32_t ef_filtered, routing_rows, bridge_rows, vector_payloads, sampled_seeds; } hx_filtered_budgets_t;
typedef struct {   /* RestrictedSearchStats counters, summed over the B queries */
  uint64_t vector_payload_requests, distance_computations, routing_rows, bridge_rows, bridge_frontier_pushes, iterations,
      kernel_launches, reserved;
} hx_filtered_stats;
void      hx_filtered_budgets(uint32_t k, uint32_t ef, uint32_t beam_percent /*0 => 150*/, uint64_t n_cand,
                              hx_filtered_budgets_t* out);
hx_status hx_search_filtered_graph(hx_index* idx, const float* queries, size_t B, const hx_search_params* p,
                                   const hx_filtered_budgets_t* budgets, const uint64_t* cand_ids, size_t n_cand,
                                   const uint64_t* query_simhash, uint64_t* out_ids, float* out_scores,
                                   uint32_t* out_counts, hx_filtered_stats* stats);

/* ---- device-resident candidate sets (prefilter reuse) ------------------------------------------------------
 * The reference's label / equality indexes are RoaringTreemap values tied to a snapshot
 * (encoding/v1/indexes/label.rs:10-14; SURVEY §8d: "allow label bitmaps to be cached device-side keyed by the same
 * snapshot sequence").  hx_candidates_create uploads one candidate set (ascending unique ids, <= 1e6,
 * restricted.rs:356-371) and maps it to device slots once; hx_search_restricted_sets then names a set per query
 * (n_sets == B) or one for all (n_sets == 1): 24 bytes per query cross PCIe instead of 8 bytes per candidate.
 * Same exact answer as hx_search_restricted.  A set is invalidated by reloading the index's vectors. */
typedef struct hx_candidates hx_candidates;
hx_status hx_candidates_create(hx_index* idx, const uint64_t* cand_ids, size_t n, hx_candidates** out);
void      hx_candidates_destroy(hx_candidates* set);
uint64_t  hx_candidates_len(const hx_candidates* set);
hx_status hx_search_restricted_sets(hx_index* idx, const float* queries, size_t B, const hx_search_params* p,
                                    hx_candidates* const* sets, size_t n_sets, uint64_t* out_ids,
                                    float* out_scores, uint32_t* out_counts, hx_stats* stats);

/* RestrictedExecutionPlan chosen by the reference for this |C| and dimension
 * (restricted.rs:40-42,426-453): 0 = Exact, 1 = FilteredGraph.  Informational: the
 * device path always answers exactly. */
int32_t hx_restricted_plan(uint64_t n_candidates, uint32_t dimension);

/* B independent queries with a status PER QUERY.  The reference runs one query per call
 * (read_index.rs:81-101), so in a batch one invalid query (or one query that exhausts a device-side
 * bound such as the tie-stack overflow regions) must fail alone: out_status[b] carries the code
 * hx_search would have returned for query b on its own, out_counts[b] = 0 for a failed query, and the
 * call returns HX_OK whenever the batch itself could be executed.  Same kernels and results as
 * hx_search (strict-exhaustive params) / hx_search_ex with default policy (any other params). */
hx_status hx_search_batch(hx_index* idx, const float* queries, size_t B, const hx_search_params* p,
                          uint64_t* out_ids, float* out_scores, uint32_t* out_counts,
                          hx_status* out_status /* B */, hx_stats* stats);

/* ---- query service: the reference's calling pattern ---------------------------------------------
 * Production traffic reaches this path as ONE query per call from many concurrent tokio tasks, no
 * intra-query parallelism (read_index.rs:81-101, called per request from
 * execution/interpreter/access/search/storage.rs:142-192).  A service coalesces those callers: a caller
 * writes its query into a slot of a pinned submission ring (lock-free ticket), a dispatcher thread turns
 * whatever is pending into ONE launch of the CTA-per-query traversal kernel (grid = pending queries, several
 * launches in flight on a stream pool, 2-3 CTAs resident per SM), the kernel writes each query's results
 * straight into host-mapped memory and then publishes a per-query done word; nobody ever calls
 * cudaStreamSynchronize.  hx_service_submit / hx_service_poll are the async pair a tokio task maps to
 * (submit, then poll from the task's waker loop or a oneshot fed by a reaper thread); hx_service_search is
 * the blocking form (futex wait, woken by the service's completer thread).  Results are bit-identical to
 * hx_search: same kernel, same admission order.  Strict-exhaustive SearchParams; k and ef are fixed per
 * service (they size the result slots).  Thread-safe; any number of services per index. */
typedef struct hx_service hx_service;
typedef struct {
  uint32_t k;               /* results per query (> 0)                                                */
  uint32_t ef;              /* beam width; 0 => max(k, 100)                                           */
  uint32_t capacity;        /* submission-ring slots = max queries in flight; 0 => 1024 (rounded up to 2^n) */
  uint32_t max_batch;       /* max queries per launch; 0 => 128                                       */
  uint32_t n_streams;       /* launches in flight; 0 => 32                                            */
  uint32_t ctas_per_sm;     /* resident CTAs (= queries) per SM the launch shape is sized for; 0 => 2 */
  uint32_t cta_warps;       /* warps per CTA of the traversal kernel; 0 => 12 / 6 / 4 for 1 / 2 / 3+ CTAs per SM */
  uint32_t rows_in_flight;  /* vector rows staged per CTA; 0 => as many as fit                        */
  uint32_t visited_log2;    /* log2 of the shared-memory visited-table size; 0 => auto               */
  uint32_t min_batch;       /* while the device is busy a launch waits (<= batch_window_us) for this many queries; 0 => 16 */
  uint32_t batch_window_us; /* 0 => 30                                                                */
  uint32_t flags;           /* HX_SERVICE_*                                                           */
} hx_service_config;
enum { HX_SERVICE_NO_COALESCING = 1,   /* launch whatever is pending at once, always                              */
       HX_SERVICE_STAGE_QUERIES = 2 }; /* copy queries to device memory first (default: the kernel reads the pinned
                                          ring directly when the dimension is a multiple of 32)                     */
typedef struct {
  uint64_t submitted, completed, launches, max_batch_seen, dispatcher_sleeps, completer_wakes;
  uint32_t cta_warps, rows_in_flight, visited_cap, smem_bytes, ctas_per_sm, reserved;
} hx_service_stats;
hx_status hx_service_create(hx_index* idx, const hx_service_config* cfg, hx_service** out);
void      hx_service_destroy(hx_service* svc);   /* waits for queries in flight */
/* Validate (dimension known from the index; finiteness -> cosine zero norm -> magnitude, domain.rs:113-154), copy the
 * query into a ring slot and return its ticket.  Blocks only while the ring is full (back-pressure). */
hx_status hx_service_submit(hx_service* svc, const float* query, uint64_t* out_ticket);
/* Non-blocking.  *out_done = 0: still running.  *out_done = 1: results copied out (out_ids/out_scores hold k entries,
 * *out_count <= k), the return value is the query's own status, the ticket is consumed. */
hx_status hx_service_poll(hx_service* svc, uint64_t ticket, int32_t* out_done, uint64_t* out_ids, float* out_scores,
                          uint32_t* out_count);
/* Blocking: returns when the ticket's results are out (futex wait; consumes the ticket). */
hx_status hx_service_wait(hx_service* svc, uint64_t ticket, uint64_t* out_ids, float* out_scores, uint32_t* out_count);
/* submit + wait: the drop-in for one ValidatedVectorReadIndex::search call. */
hx_status hx_service_search(hx_service* svc, const float* query, uint64_t* out_ids, float* out_scores,
                            uint32_t* out_count);
hx_status hx_service_get_stats(hx_service* svc, hx_service_stats* out);

/* ---- restricted query service: search_restricted with the same calling pattern ---------------------------------
 * ValidatedVectorReadIndex::search_restricted (read_index.rs:92-101) is called like search: one (query, candidate set)
 * per call from many concurrent tasks.  A restricted service coalesces those callers exactly as above, through the same
 * ring, dispatcher, completer, poll / wait and stats; each coalesced run becomes ONE exact-scan launch that writes every
 * answer into its host-mapped result slot.  Answers are bit-identical to hx_search_restricted (ids, order, score bits,
 * count).  No graph or entry point is needed.
 * Config: k in 1..800 (restricted.rs:55); capacity, max_batch (<= 128), n_streams, min_batch, batch_window_us and flags
 * as above (HX_SERVICE_STAGE_QUERIES stages candidate ids too); ef, ctas_per_sm, cta_warps, rows_in_flight and
 * visited_log2 must be 0.  arena_ids sizes the pinned arena that holds submitted candidate ids until their launch has
 * read them: 0 => 2000000, values below 1000000 are refused (every legal set fits).  A full arena is back-pressure.
 * Device memory per service, per stream (n_streams, default 32): (arena_ids / 256 + 128) * 256 B of partial lists, and for
 * k > 32 (arena_ids + 262144) * 8 B of scores — with the defaults about 65 MB, plus about 580 MB when k > 32.  Fewer
 * streams (or a smaller arena) cost proportionally less.
 * hx_service_submit on a restricted service, and the restricted submits on an HNSW service, are HX_ERR_INVALID_PARAMETER. */
hx_status hx_restricted_service_create(hx_index* idx, const hx_service_config* cfg, uint64_t arena_ids, hx_service** out);
/* Admission on the caller's thread, in restricted_host's order: |C| > 1e6 => HX_ERR_QUERY; an empty set completes the
 * ticket at once with count 0 (no query validation, no device work); ids not ascending and unique =>
 * HX_ERR_INVALID_PARAMETER; then the query is validated (dimension -> finiteness -> cosine zero norm -> magnitude).
 * The ids are copied: the caller's array may be reused when the call returns. */
hx_status hx_service_submit_restricted(hx_service* svc, const float* query, const uint64_t* cand_ids, size_t n_cand,
                                       uint64_t* out_ticket);
/* Same with a device-resident set (hx_candidates_create): no ids cross PCIe.  A set of another index or of an older
 * vector generation is HX_ERR_INVARIANT_VIOLATION.  The set is read by the device until the ticket completes: it must
 * not be destroyed before hx_service_poll / hx_service_wait has returned the ticket's results. */
hx_status hx_service_submit_restricted_set(hx_service* svc, const float* query, const hx_candidates* set,
                                           uint64_t* out_ticket);
/* submit + wait: the drop-in for one ValidatedVectorReadIndex::search_restricted call. */
hx_status hx_service_search_restricted(hx_service* svc, const float* query, const uint64_t* cand_ids, size_t n_cand,
                                       uint64_t* out_ids, float* out_scores, uint32_t* out_count);
hx_status hx_service_search_restricted_set(hx_service* svc, const float* query, const hx_candidates* set,
                                           uint64_t* out_ids, float* out_scores, uint32_t* out_count);

/* ---- search (device buffers: inputs already resident in HBM) ------------------------- */
/* Same semantics, no validation copy, no host sync: everything is enqueued on
 * `cuda_stream` (a cudaStream_t, 0 = legacy default stream).  d_queries must have been
 * validated by the caller.  Used by bench.py for `value`, and by the sharded path. */
hx_status hx_search_device(hx_index* idx, const float* d_queries, size_t B,
                           const hx_search_params* p, uint64_t* d_out_ids, float* d_out_scores,
                           uint32_t* d_out_counts, void* cuda_stream, hx_stats* stats_or_null);
/* Device-buffer calls never synchronise, so they cannot report a per-call device error: the flags raised by the
 * launches issued on `cuda_stream` since the previous hx_device_flags on that stream are ORed into one word
 * (1 invalid score, 4 tie-stack overflow, 8 visited-set overflow, 16 copy time-out).  This call synchronises the stream,
 * returns and clears the word; *out_status = the HelixDbError it maps to (HX_OK when 0).  Device-buffer calls on
 * DIFFERENT streams use separate scratch sets and may run concurrently from different threads. */
hx_status hx_device_flags(hx_index* idx, void* cuda_stream, uint32_t* out_flags, hx_status* out_status);
/* Candidates as device slot numbers (ascending), per query CSR. */
hx_status hx_search_restricted_device(hx_index* idx, const float* d_queries, size_t B,
                                      const hx_search_params* p, const uint32_t* d_cand_slots,
                                      const uint64_t* d_cand_offsets /* NULL: one set shared by all B */,
                                      uint64_t total_cands, uint64_t max_cands_per_query /* 0: unknown */,
                                      uint64_t* d_out_ids, float* d_out_scores,
                                      uint32_t* d_out_counts, void* cuda_stream);
/* Map ascending candidate ids to device slots (absent ids dropped, restricted.rs:615-659). */
hx_status hx_map_candidates_device(hx_index* idx, const uint64_t* d_cand_ids, uint64_t n,
                                   uint32_t* d_out_slots, uint64_t* d_out_count, void* cuda_stream);

/* ---- sharded path: merge of per-shard top-k (SURVEY §8e) ------------------------------ */
/* After ONE all-gather of per-shard (score,id,count) blocks over NCCL, every rank selects
 * the k smallest by (score,id) per query.  d_all_* are [n_shards][B][k] / [n_shards][B]. */
hx_status hx_merge_topk_device(int32_t device, const uint64_t* d_all_ids, const float* d_all_scores,
                               const uint32_t* d_all_counts, uint32_t n_shards, size_t B, uint32_t k,
                               uint64_t* d_out_ids, float* d_out_scores, uint32_t* d_out_counts,
                               void* cuda_stream);

/* ---- sharded search: id-range shards, one rank per device, ONE all-gather (SURVEY §8e) -----------------
 * Each rank holds an hx_index with a contiguous id range of the corpus (hx_index_generate_vectors / load_* with
 * that range's ids, its own graph from hx_index_build or hx_index_load_graph).  A group binds the ranks with one NCCL
 * communicator (NCCL is dlopen'ed on first use; a group of 1 never touches it).  A sharded search = local search on the
 * shard, whose kernels write ids | scores | counts straight into this rank's send block -> ONE ncclAllGather of
 * the blocks -> the (score, id) merge kernel on every rank.  Every rank passes the SAME queries and receives the same
 * merged answer.  `local` holds the PER-SHARD parameters: local->k results are kept per shard (>= k_out is exact;
 * smaller trades recall for traffic) and local->ef is the per-shard beam width — a shard is 1/n_shards of the corpus, so
 * the beam that gives the unsharded index its recall is over-provisioned per shard; bench.py tunes it to iso-recall.
 * Ranks may be processes (torchrun: rank 0 calls hx_shard_unique_id and ships the 128 bytes through the host's own
 * channel) or threads of one process, one per device.  Collective: every rank must make the same sequence of calls. */
typedef struct hx_shard_group hx_shard_group;
enum { HX_SHARD_HNSW = 0 /* hx_search_device on the shard */, HX_SHARD_DENSE = 1 /* tensor-core exhaustive path */ };
#define HX_SHARD_UNIQUE_ID_BYTES 128
hx_status hx_shard_unique_id(uint8_t* out, size_t cap /* >= HX_SHARD_UNIQUE_ID_BYTES */);
hx_status hx_shard_group_create(hx_index* shard, uint32_t n_shards, uint32_t rank, const uint8_t* unique_id,
                                hx_shard_group** out);
void      hx_shard_group_destroy(hx_shard_group* g);
/* device buffers, everything enqueued on cuda_stream (no host synchronisation) */
hx_status hx_search_sharded_device(hx_shard_group* g, int32_t path, const float* d_queries, size_t B,
                                   const hx_search_params* local, uint32_t k_out, uint64_t* d_out_ids,
                                   float* d_out_scores, uint32_t* d_out_counts, void* cuda_stream);
/* host buffers (blocking) */
hx_status hx_search_sharded(hx_shard_group* g, int32_t path, const float* queries, size_t B,
                            const hx_search_params* local, uint32_t k_out, uint64_t* out_ids, float* out_scores,
                            uint32_t* out_counts);
/* restricted search across shards: every rank passes the same ascending candidate list; a shard scores the slice inside
 * its id range (an empty slice = RestrictedVectorCandidates::Empty for that shard); exact for any number of shards */
hx_status hx_search_restricted_sharded(hx_shard_group* g, const float* queries, size_t B, const hx_search_params* p,
                                       const uint64_t* cand_ids, size_t n_cand, uint64_t* out_ids, float* out_scores,
                                       uint32_t* out_counts);
/* device time of the last host-buffer sharded call: local search, and all-gather + merge */
hx_status hx_shard_group_last_ms(hx_shard_group* g, float* local_ms, float* collective_ms);

/* ---- dense batched path (tensor cores; configs C4/C5) ---------------------------------- */
/* Exhaustive top-k of B queries against all rows through the bf16 copy:
 * wgmma (Hopper tensor cores) for the B x N contraction, per-tile candidate filter, fp32 re-rank of
 * survivors with the exact kernel.  Requires cfg.storage == 1. */
hx_status hx_search_dense(hx_index* idx, const float* queries, size_t B, const hx_search_params* p,
                          uint64_t* out_ids, float* out_scores, uint32_t* out_counts,
                          hx_stats* stats);
/* The same path restricted to ONE candidate set C shared by the B queries (prefiltered search as a contraction):
 * hx_search_dense's contract over the rows of C that are present and not deleted.  Every score is the exact fp32 score,
 * results are in (score, id) order with exact ties resolved by id, the count is min(k, |C ∩ live rows|), and ids without a
 * row are never returned.  Per call the present rows of C are converted from the f32 rows into a bf16 tile (the
 * whole-corpus bf16 copy is neither built nor read, so cfg.storage may be 0; the answer is the same at 0 and 1), the
 * tensor cores nominate, and the exact kernel re-ranks.  Below 8 * min(max(4k, 64), 800) present rows the call runs the
 * exact scan instead and returns hx_search_restricted's answer bit for bit.
 * Admission, in order: params (as hx_search_restricted); B == 0 => HX_OK; null pointers => HX_ERR_INVALID_PARAMETER;
 * Manhattan => HX_ERR_UNSUPPORTED; |C| > 1e6 => HX_ERR_QUERY; |C| == 0 => counts 0 (no query validation, no device work);
 * min(k, |C|) > 800 => HX_ERR_QUERY (k is clamped to |C|; out_ids / out_scores are still B*k); ids not ascending and
 * unique => HX_ERR_INVALID_PARAMETER; a set of another index or of an older vector generation => HX_ERR_INVARIANT_VIOLATION;
 * empty or unpopulated index => counts 0 after query validation; then the queries are validated (first failing query's code).
 * Device memory, held by the call's scratch set across calls: about present * (2 * ldb + 4) bytes for the tile (ldb = the
 * dimension rounded up to 64) plus at most 16 bytes per candidate id and the nominee keys; about 1.5 GB at |C| = 1e6,
 * d = 768.
 * Per-query candidate sets stay on hx_search_restricted_multi / hx_search_restricted_sets. */
hx_status hx_search_dense_restricted(hx_index* idx, const float* queries, size_t B, const hx_search_params* p,
                                     const uint64_t* cand_ids, size_t n_cand, uint64_t* out_ids, float* out_scores,
                                     uint32_t* out_counts, hx_stats* stats);
/* Same with a device-resident set (hx_candidates_create): no ids cross PCIe. */
hx_status hx_search_dense_restricted_set(hx_index* idx, const float* queries, size_t B, const hx_search_params* p,
                                         const hx_candidates* set, uint64_t* out_ids, float* out_scores,
                                         uint32_t* out_counts, hx_stats* stats);

/* Exact tensor-core search.  The answer of hx_search_restricted over every live id (resp. over C), bit for bit: ids, order,
 * score bits and count, for every legal input.  After the re-rank a certificate bounds, per query, what the tensor-core pass
 * may have dropped (bucket tails and the nominee cut, against the bf16 / fp32 error bound derived in csrc/k_dense.cu); a
 * query it cannot prove exact is rescanned by the exact scan over every row of the view.  One more stream synchronisation
 * than the entry of the same name (a 4-byte read-back of the flagged count); a rescanned query costs a full exact scan.
 * out_how (B bytes, may be NULL): 0 = the tensor-core answer was certified, 1 = the query was rescanned because the
 * certificate failed, 2 = the corpus / present set is below hx_dense_min_rows(k) = 8 * min(max(4k, 64), 800) rows and every
 * query was answered by the exact scan outright (also for an empty index or set).  Admission and errors exactly as the
 * entry of the same name without _exact.  hx_last_kernel_ms reports the rescan's scan kernel when queries were rescanned.
 * hx_stats: kernel_launches includes the certificate, compaction, gather, scan and scatter; distance_computations and
 * algorithmic_bytes add the rescanned queries' full scans. */
hx_status hx_search_dense_exact(hx_index* idx, const float* queries, size_t B, const hx_search_params* p,
                                uint64_t* out_ids, float* out_scores, uint32_t* out_counts, uint8_t* out_how,
                                hx_stats* stats);
hx_status hx_search_dense_restricted_exact(hx_index* idx, const float* queries, size_t B, const hx_search_params* p,
                                           const uint64_t* cand_ids, size_t n_cand, uint64_t* out_ids, float* out_scores,
                                           uint32_t* out_counts, uint8_t* out_how, hx_stats* stats);
hx_status hx_search_dense_restricted_exact_set(hx_index* idx, const float* queries, size_t B, const hx_search_params* p,
                                               const hx_candidates* set, uint64_t* out_ids, float* out_scores,
                                               uint32_t* out_counts, uint8_t* out_how, hx_stats* stats);

/* Resident candidate sets.  hx_search_dense_restricted_set and _exact_set otherwise rebuild the set's tensor-core view on
 * every call: compaction of the present slots (and a stream synchronisation to read their count), gather of the present
 * rows into a bf16 tile, and for the exact entry the reduction of the view word of the certificate.  The gather is the
 * largest kernel of a call.  hx_candidates_make_resident builds that view once, blocking, and the set keeps it until
 * hx_candidates_destroy.  It holds the ascending present slots, the bf16 tile in tile placement over candidate rank, the
 * row terms and the view word, built by the kernels the per-call path runs, so an answer through a resident set is the
 * answer of the same ids through a non-resident set bit for bit.
 * With the view, the two set entries run no compaction, gather or view reduction: the plain entry synchronises once per call.
 * hx_stats: kernel_launches counts the launches actually issued; algorithmic_bytes = present * 2 * ldb (the tile read once)
 * plus any rescans.
 * Device memory: n_pad * (2 * ldb + 4) + 4 * present + 4 bytes (n_pad = present rounded up to 256, ldb = the dimension
 * rounded up to 64; 0 when no id of the set is present), about 1.5 GB at present = 1e6, d = 768.  hx_candidates_resident_bytes
 * reports it (0 while the set is not resident).
 * Admission, in order: null argument => HX_ERR_INVALID_PARAMETER; Manhattan => HX_ERR_UNSUPPORTED; a set of another index or
 * of an older vector generation => HX_ERR_INVARIANT_VIOLATION; an empty set => HX_OK, 0 bytes.  A second call is a no-op.
 * Staleness: the present list cannot change while the set is valid (deletes and reloads refuse the set; upserts do not
 * remap it), but an upsert can change row values.  The first call after any row write re-gathers the tile and the view word
 * in place, on the set's own stream, once, however many callers race to it; no caller reads a half-built tile.  A
 * stream-ordered search (hx_search_dense_restricted_set_device) counts as overlapping a patch call until its stream has
 * been synchronised: patch calls must not overlap searches, and a patch must not run while such a search may still read
 * the tile.  A set maps its ids once, at hx_candidates_create: ids appended or revived by later upserts stay absent from
 * it, resident or not. */
hx_status hx_candidates_make_resident(hx_index* idx, hx_candidates* set);
uint64_t  hx_candidates_resident_bytes(const hx_candidates* set);
/* hx_search_dense_restricted_set on device buffers, through a resident set.  Everything is enqueued on `cuda_stream`
 * (per-stream scratch, as hx_search_device); no synchronisation once the view is current (the first call after a row
 * write refreshes it as above).  Admission exactly as hx_search_dense_restricted_set, in its order; then a set that is not
 * resident => HX_ERR_INVALID_PARAMETER.  d_queries follow hx_search_device's convention: the caller validates them, an
 * invalid query gets count 0.  Device errors come out through hx_device_flags.  Below hx_dense_min_rows(k) present rows
 * the exact scan over the present slots answers, on the stream.
 * d_out_how (B bytes on the device, may be NULL) runs the certificate of the exact entries without the rescan:
 *   0 = certified: the answer is hx_search_restricted's bit for bit;
 *   1 = not certified: the plain tensor-core answer is returned, not rescanned;
 *   2 = the present rows are below hx_dense_min_rows(k): exact scan.
 * The rescan needs the flagged count on the host, so a caller that needs exactness for the queries marked 1 re-issues them
 * through hx_search_restricted_device or an exact host entry. */
hx_status hx_search_dense_restricted_set_device(hx_index* idx, const float* d_queries, size_t B, const hx_search_params* p,
                                                const hx_candidates* set, uint64_t* d_out_ids, float* d_out_scores,
                                                uint32_t* d_out_counts, uint8_t* d_out_how /* may be NULL */,
                                                void* cuda_stream);

/* ---- SimHash filtering / sampling policy: the production-default search mode ------------------------------
 * SearchParams::new(k) is SimHashMode::Adaptive: layer 0 then runs Layer0Policy::decide per expansion
 * (policy.rs:119-175: adaptive collision threshold :576-597, adaptive sampling :558-574, pre-/post-sampling activation
 * :526-556, bypass windows :196-291), gates every unvisited neighbour on its 64-bit SimHash
 * (unaligned_vector/simhash.rs:37-55: collisions = 64 - popcount(a ^ b) >= threshold; cosine only, policy.rs:67-88),
 * accounts filtered nodes as virtual beam-fill slots (search.rs:742-748,940-951) and fetches vectors only for the
 * survivors.  Index-level settings mirror VectorIndexConfig (config/indexes.rs:398-406); per-query ones the rest of
 * SearchParams (mod.rs:431-454).
 *
 * Fingerprints are DATA, not recomputed secrets: the reference persists one per node ([0x12] rows, 8 bytes LE,
 * values/vectors/simhash.rs:37-41) -> hx_index_load_simhash; the query's fingerprint is computed by the caller's
 * SimHasher (hash_from_slice, unaligned_vector/simhash.rs:263-290) and passed in, or — when the caller hands over the
 * hyperplane table (SimHasher::hyperplanes(), 64 x dimension f32) — projected on the device with the same sequential
 * `dot += v*h` order.  Bernoulli draws use the reference's query-derived seed (randomness.rs:109-114) over ChaCha12
 * (rand 0.10 StdRng, restated from the published algorithm: the reference pins no stream value); they only happen for
 * frontiers larger than max(ef/4, 8).  "SimHash filter reads" follow the resident-store case (no KV reads). */
typedef struct {
  uint32_t simhash_threshold;      /* 0..64, default 43 (simhash.rs:35)            */
  float    sampling_ratio;         /* default 0.8                                   */
  uint32_t adaptive_enabled;       /* default 1                                     */
  float    adaptive_failure_prob;  /* default 0.1, in (0,1)                         */
} hx_simhash_config;
hx_status hx_index_set_simhash_config(hx_index* idx, const hx_simhash_config* cfg);
hx_status hx_index_load_simhash(hx_index* idx, const uint64_t* ids, const uint64_t* bits, size_t n);
/* planes: 64 x dimension f32, plane-major (SimHasher::hyperplanes()). */
hx_status hx_index_set_simhash_planes(hx_index* idx, const float* planes);
/* hash_from_slice of every loaded row on the device (needs the planes); replaces loaded fingerprints. */
hx_status hx_index_compute_simhash(hx_index* idx);
hx_status hx_index_download_simhash(hx_index* idx, size_t first_slot, size_t n, uint64_t* out_bits);
/* locality order code of the canonical vector key (simhash.rs:44-59); pure */
uint64_t  hx_order_code_from_simhash_bits(uint64_t bits);

typedef struct {                      /* SearchParams fields beyond hx_search_params; hx_policy_params_default() first */
  uint32_t bypass_min_frontier;       /* 24   */
  uint32_t bypass_window_expansions;  /* 4    */
  float    bypass_min_filter_rate;    /* 0.12 */
  uint32_t read_budget_multiplier;    /* 3    */
  float    sampling_ratio_override;   /* simhash_sampling_ratio_override; negative = None */
  float    failure_prob_override;     /* simhash_failure_prob_override;   negative = None */
  uint32_t reserved[2];
} hx_policy_params;
void hx_policy_params_default(hx_policy_params* p);

/* Sums over the B queries of the SimHash-related SearchStats counters (mod.rs:640-700). */
typedef struct {
  uint64_t simhash_filtered, simhash_examined, simhash_missing_hash, simhash_passed_before_sampling,
      simhash_passed_after_sampling, simhash_bypass_expansions, simhash_skipped_candidates, pre_simhash_sample_kept,
      pre_simhash_sample_dropped, simhash_bypass_trigger_budget, simhash_bypass_trigger_low_yield, rng_draws;
} hx_policy_stats;

/* hx_search with the full SearchParams surface.  policy == NULL: SearchParams::new defaults.  query_simhash == NULL:
 * projected on the device from the planes (HX_ERR_INVALID_VECTOR_CONFIG when there are none).  The strict-exhaustive
 * combination is forwarded to the exhaustive kernels (identical results to hx_search). */
hx_status hx_search_ex(hx_index* idx, const float* queries, size_t B, const hx_search_params* p,
                       const hx_policy_params* policy, const uint64_t* query_simhash, uint64_t* out_ids,
                       float* out_scores, uint32_t* out_counts, hx_stats* stats, hx_policy_stats* policy_stats);

/* ---- diagnostics --------------------------------------------------------------------------- */
const char* hx_last_error(void);          /* thread-local, valid until the next failing call     */
uint32_t    hx_last_error_index(void);    /* component index for HX_ERR_INVALID_VECTOR_COMPONENT */
const char* hx_version(void);
/* Device time (ms, CUDA events recorded on the launch stream around the dominant kernel:
 * the traversal kernel or the scan) and launch count.  After host-buffer calls: the most recent call.
 * After device-buffer calls: the SUM over every launch since the previous hx_last_kernel_ms
 * (the call synchronises on the recorded events). */
hx_status hx_last_kernel_ms(hx_index* idx, float* ms, uint32_t* launches);

/* Launch-shape knobs of the traversal kernels, for experiments and A/B tests (every default is the measured best; results
 * are bit-identical for every setting — tests/test_gpu_parity.py::test_traversal_builds_agree).  A handle takes its values
 * from the environment ONCE, in hx_index_create (the variable named next to each field); nothing on the search path reads
 * the environment.  -1 in any field = the built-in default.  hx_index_set_tuning(idx, NULL) re-reads the environment.
 * Not synchronised with searches in flight on the same handle. */
typedef struct hx_tuning {
  int32_t ring_warps;      /* HX_RING_WARPS      warp-per-query build: warps per SM, 1..16 (16)                    */
  int32_t ring_rows;       /* HX_RING_R          row slots per warp / rows in flight per CTA, 1..32 (what fits)     */
  int32_t visited_log2;    /* HX_VT_CAP_LOG2     log2 entries of a query's visited hash set, 6..24 (64 ef rounded)  */
  int32_t visited_pool;    /* HX_VT_POOL         overflow tables, 0..1024 (32)                                     */
  int32_t l2_hint;         /* HX_L2_HINT         evict-first hint on row copies (1)                                 */
  int32_t prefetch_below;  /* HX_PREFETCH_BELOW  beam position below which an admitted row is L2-prefetched (ef/2+1)*/
  int32_t lat_warps;       /* HX_LAT_WARPS       CTA-per-query build: warps per CTA, 1..12 (12; 8 above d = 1024)   */
  int32_t lat_admit_seq;   /* HX_LAT_ADMIT=seq   CTA build: sequential instead of one-pass admission (0)           */
  int32_t lat_spec;        /* HX_LAT_SPEC        CTA build: speculative L2 prefetch of the next expansion (0)       */
  int32_t phase_prof;      /* HX_PHASE_PROF      CTA build: per-phase cycle sums, printed by hx_last_kernel_ms (0)  */
  int32_t pipeline;        /* HX_PIPELINE        chunked query upload overlapped with the search (1)               */
  int32_t scan_fused;      /* HX_SCAN_FUSED      prefilter scan: in-kernel top-k for k <= 32 (1)                    */
  int32_t pol_warps;       /* HX_POL_WARPS       default-mode kernel: warps per SM, 1..16 (16)                      */
  int32_t pol_min_rows;    /* HX_POL_MINR        default-mode kernel: least row slots per warp (3)                  */
  int32_t pol_cta;         /* HX_POL_CTA         default-mode kernel: CTA-per-query build below #SMs queries (1)    */
  int32_t pol_early_sim;   /* HX_POL_EARLY_SIM   fingerprints requested together with the visited probe (1)         */
  int32_t build_max_batch; /* HX_BUILD_MAX_BATCH device build: cap on the nodes inserted per round (n/64, <= 16384) */
} hx_tuning;
hx_status hx_index_get_tuning(const hx_index* idx, hx_tuning* out);
hx_status hx_index_set_tuning(hx_index* idx, const hx_tuning* tuning);

#ifdef __cplusplus
}
#endif
#endif /* HELIX_B200_H */
