/*
 * hx_oracle.c — CPU restatement of HelixDB's vector-search hot path (see hx_oracle.h).
 *
 * TEST INFRASTRUCTURE ONLY — never linked into the product library.
 *
 * Build with -ffp-contract=off and without -ffast-math: the reference is Rust, which
 * never contracts a*b+c and never re-associates float sums; the only fused operations
 * are the explicit _mm256_fmadd_ps calls of spaces/simple_avx.rs.
 *
 * All "V/" paths are helix-db/crates/db/src/search/vector/.
 */
#define _GNU_SOURCE
#include "hx_oracle.h"

#include <float.h>
#include <immintrin.h>
#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ------------------------------------------------------------------------------------------
 * Distance kernels
 * ------------------------------------------------------------------------------------------ */

/* V/spaces/simple.rs:204-218 — `distance += (l - r) * (l - r)`, strictly sequential, no FMA. */
float hxo_euclid_scalar(const float* u, const float* v, size_t d) {
  float distance = 0.0f;
  for (size_t i = 0; i < d; ++i) {
    float diff = u[i] - v[i];
    float sq = diff * diff;
    distance = distance + sq;
  }
  return distance;
}

/* V/spaces/simple.rs:220-234 */
float hxo_dot_scalar(const float* u, const float* v, size_t d) {
  float product = 0.0f;
  for (size_t i = 0; i < d; ++i) {
    float p = u[i] * v[i];
    product = product + p;
  }
  return product;
}

/* V/spaces/simple.rs:186-202 — `distance += (l - r).abs()`, sequential; the reference has no SIMD path. */
float hxo_manhattan(const float* u, const float* v, size_t d) {
  float distance = 0.0f;
  for (size_t i = 0; i < d; ++i) {
    float diff = u[i] - v[i];
    distance = distance + fabsf(diff);
  }
  return distance;
}

int hxo_has_avx_fma(void) {
  return __builtin_cpu_supports("avx") && __builtin_cpu_supports("fma");
}

/* V/spaces/simple_avx.rs:6-12 hsum256_ps_avx */
__attribute__((target("avx,fma"))) static float hsum256(__m256 x) {
  __m128 x128 = _mm_add_ps(_mm256_extractf128_ps(x, 1), _mm256_castps256_ps128(x));
  __m128 x64 = _mm_add_ps(x128, _mm_movehl_ps(x128, x128));
  __m128 x32 = _mm_add_ss(x64, _mm_shuffle_ps(x64, x64, 0x55));
  return _mm_cvtss_f32(x32);
}

/* V/spaces/simple_avx.rs:128-180 euclid_similarity_avx_fma */
__attribute__((target("avx,fma"))) float hxo_euclid_avx_fma(const float* p1, const float* p2, size_t n) {
  size_t m = n - (n % 32);
  __m256 s1 = _mm256_setzero_ps(), s2 = _mm256_setzero_ps(), s3 = _mm256_setzero_ps(), s4 = _mm256_setzero_ps();
  size_t i = 0;
  while (i < m) {
    __m256 d1 = _mm256_sub_ps(_mm256_loadu_ps(p1), _mm256_loadu_ps(p2));
    s1 = _mm256_fmadd_ps(d1, d1, s1);
    __m256 d2 = _mm256_sub_ps(_mm256_loadu_ps(p1 + 8), _mm256_loadu_ps(p2 + 8));
    s2 = _mm256_fmadd_ps(d2, d2, s2);
    __m256 d3 = _mm256_sub_ps(_mm256_loadu_ps(p1 + 16), _mm256_loadu_ps(p2 + 16));
    s3 = _mm256_fmadd_ps(d3, d3, s3);
    __m256 d4 = _mm256_sub_ps(_mm256_loadu_ps(p1 + 24), _mm256_loadu_ps(p2 + 24));
    s4 = _mm256_fmadd_ps(d4, d4, s4);
    p1 += 32;
    p2 += 32;
    i += 32;
  }
  __m256 sum = _mm256_add_ps(_mm256_add_ps(s1, s2), _mm256_add_ps(s3, s4));
  float result = hsum256(sum);
  for (size_t t = 0; t < n - m; ++t) {
    float a = p1[t], b = p2[t];
    float d = a - b;
    float sq = d * d;
    result = result + sq;
  }
  return result;
}

/* V/spaces/simple_avx.rs:184-238 dot_similarity_avx_fma */
__attribute__((target("avx,fma"))) float hxo_dot_avx_fma(const float* p1, const float* p2, size_t n) {
  size_t m = n - (n % 32);
  __m256 s1 = _mm256_setzero_ps(), s2 = _mm256_setzero_ps(), s3 = _mm256_setzero_ps(), s4 = _mm256_setzero_ps();
  size_t i = 0;
  while (i < m) {
    s1 = _mm256_fmadd_ps(_mm256_loadu_ps(p1), _mm256_loadu_ps(p2), s1);
    s2 = _mm256_fmadd_ps(_mm256_loadu_ps(p1 + 8), _mm256_loadu_ps(p2 + 8), s2);
    s3 = _mm256_fmadd_ps(_mm256_loadu_ps(p1 + 16), _mm256_loadu_ps(p2 + 16), s3);
    s4 = _mm256_fmadd_ps(_mm256_loadu_ps(p1 + 24), _mm256_loadu_ps(p2 + 24), s4);
    p1 += 32;
    p2 += 32;
    i += 32;
  }
  __m256 sum = _mm256_add_ps(_mm256_add_ps(s1, s2), _mm256_add_ps(s3, s4));
  float result = hsum256(sum);
  for (size_t t = 0; t < n - m; ++t) {
    float p = p1[t] * p2[t];
    result = result + p;
  }
  return result;
}

/* The same accumulation order spelled with scalar fmaf(): 32 independent accumulators
 * (accumulator a, lane j  <->  element index i with i mod 32 == 8a + j), then
 * (s1+s2)+(s3+s4) per lane, then hsum256's tree, then the scalar tail.  This is the form
 * the CUDA kernels implement; it must equal the intrinsic version bit for bit. */
static float avx_order_reduce(const float acc[32]) {
  float lane[8];
  for (int j = 0; j < 8; ++j) {
    float a = acc[j] + acc[8 + j];
    float b = acc[16 + j] + acc[24 + j];
    lane[j] = a + b;
  }
  float x128[4];
  for (int j = 0; j < 4; ++j) x128[j] = lane[4 + j] + lane[j];
  float x64_0 = x128[0] + x128[2];
  float x64_1 = x128[1] + x128[3];
  return x64_0 + x64_1;
}

float hxo_euclid_avx_fma_portable(const float* u, const float* v, size_t n) {
  size_t m = n - (n % 32);
  float acc[32];
  for (int l = 0; l < 32; ++l) acc[l] = 0.0f;
  for (size_t i = 0; i < m; i += 32)
    for (int l = 0; l < 32; ++l) {
      float d = u[i + l] - v[i + l];
      acc[l] = fmaf(d, d, acc[l]);
    }
  float result = avx_order_reduce(acc);
  for (size_t i = m; i < n; ++i) {
    float d = u[i] - v[i];
    float sq = d * d;
    result = result + sq;
  }
  return result;
}

float hxo_dot_avx_fma_portable(const float* u, const float* v, size_t n) {
  size_t m = n - (n % 32);
  float acc[32];
  for (int l = 0; l < 32; ++l) acc[l] = 0.0f;
  for (size_t i = 0; i < m; i += 32)
    for (int l = 0; l < 32; ++l) acc[l] = fmaf(u[i + l], v[i + l], acc[l]);
  float result = avx_order_reduce(acc);
  for (size_t i = m; i < n; ++i) {
    float p = u[i] * v[i];
    result = result + p;
  }
  return result;
}

/* V/spaces/simple.rs:120-144: on x86_64 with avx+fma detected, AvxFma is used iff len >= 32
 * (MIN_DIM_SIZE_AVX, simple.rs:32); because float_simd() then returns AvxFma, the Sse arm never
 * matches, so every len < 32 takes the scalar loop.  The oracle always models that machine
 * (the reference's CI kernel-equivalence matrix and this container's host both have avx+fma). */
float hxo_euclidean_distance(const float* u, const float* v, size_t d) {
  if (d >= 32) return hxo_has_avx_fma() ? hxo_euclid_avx_fma(u, v, d) : hxo_euclid_avx_fma_portable(u, v, d);
  return hxo_euclid_scalar(u, v, d);
}
/* V/spaces/simple.rs:155-177 */
float hxo_dot_product(const float* u, const float* v, size_t d) {
  if (d >= 32) return hxo_has_avx_fma() ? hxo_dot_avx_fma(u, v, d) : hxo_dot_avx_fma_portable(u, v, d);
  return hxo_dot_scalar(u, v, d);
}

/* V/distance/cosine.rs:12-36 scaled_l2_norm */
double hxo_scaled_l2_norm(const float* v, size_t d) {
  double scale = 0.0, scaled_sum = 1.0;
  for (size_t i = 0; i < d; ++i) {
    double magnitude = (double)fabsf(v[i]);
    if (magnitude == 0.0) continue;
    if (scale < magnitude) {
      double ratio = scale / magnitude;
      scaled_sum = 1.0 + scaled_sum * ratio * ratio;
      scale = magnitude;
    } else {
      double ratio = magnitude / scale;
      scaled_sum += ratio * ratio;
    }
  }
  if (scale == 0.0) return 0.0;
  return scale * sqrt(scaled_sum);
}

/* V/distance/cosine.rs:120-122 norm_no_header: `scaled_l2_norm(v).min(f32::MAX as f64) as f32` */
float hxo_cosine_norm(const float* v, size_t d) {
  double n = hxo_scaled_l2_norm(v, d);
  double mx = (double)FLT_MAX;
  if (n > mx) n = mx;
  return (float)n;
}

/* new_header: Cosine -> norm (cosine.rs:89-93); Euclidean/Manhattan -> bias 0.0 (euclidean.rs:42-44) */
float hxo_header(int metric, const float* v, size_t d) {
  return metric == HXO_COSINE ? hxo_cosine_norm(v, d) : 0.0f;
}

/* V/distance/cosine.rs:39-59 stable_half_cosine */
static float stable_half_cosine(const float* p, const float* q, size_t d) {
  double pn = hxo_scaled_l2_norm(p, d), qn = hxo_scaled_l2_norm(q, d);
  if (pn == 0.0 || qn == 0.0) return NAN;
  double dot = 0.0;
  for (size_t i = 0; i < d; ++i) dot += (double)p[i] * (double)q[i];
  double c = dot / (pn * qn);
  if (c < -1.0) c = -1.0;
  if (c > 1.0) c = 1.0;
  return (float)((1.0 - c) * 0.5);
}

/* V/distance/cosine.rs:96-118 */
float hxo_cosine_distance(const float* p, float pn, const float* q, float qn, size_t d) {
  float pq = hxo_dot_product(p, q, d);
  float pnqn = pn * qn;
  if (pn > 0.0f && qn > 0.0f && pn != FLT_MAX && qn != FLT_MAX && isnormal(pnqn) && isfinite(pq)) {
    float c = pq / pnqn;
    if (c < -1.0f) c = -1.0f;
    if (c > 1.0f) c = 1.0f;
    float one_minus = 1.0f - c;
    return one_minus / 2.0f;
  }
  return stable_half_cosine(p, q, d);
}

float hxo_distance(int metric, const float* p, float p_hdr, const float* q, float q_hdr, size_t d) {
  switch (metric) {
    case HXO_EUCLIDEAN: return hxo_euclidean_distance(p, q, d);
    case HXO_COSINE: return hxo_cosine_distance(p, p_hdr, q, q_hdr, d);
    default: return hxo_manhattan(p, q, d);
  }
}

/* V/parameters.rs:241-258 + V/model.rs:21-28: NaN / Inf / negative => InvariantViolation; -0 -> +0 */
int hxo_score_validate(float* score) {
  if (!isfinite(*score)) return HXO_ERR_INVARIANT_VIOLATION;
  if (*score < 0.0f) return HXO_ERR_INVARIANT_VIOLATION;
  if (*score == 0.0f) *score = 0.0f; /* normalize_zero */
  return HXO_OK;
}

/* ------------------------------------------------------------------------------------------
 * Input domain  V/domain.rs:15-160
 * ------------------------------------------------------------------------------------------ */
int hxo_component_limit(int metric, size_t d, float* limit) {
  double factor;
  if (metric == HXO_COSINE) return 0;
  factor = metric == HXO_EUCLIDEAN ? 8.0 : 4.0;
  double divisor = (double)((uint64_t)d * (uint64_t)factor);
  double exact = metric == HXO_EUCLIDEAN ? sqrt((double)FLT_MAX / divisor) : (double)FLT_MAX / divisor;
  float rounded = (float)exact;
  if ((double)rounded > exact) {
    uint32_t bits;
    memcpy(&bits, &rounded, 4);
    bits -= 1;
    memcpy(&rounded, &bits, 4);
  }
  *limit = rounded;
  return 1;
}

int hxo_validate_vector(int metric, size_t expected_d, const float* v, size_t actual_d, uint32_t* bad_index) {
  if (bad_index) *bad_index = 0;
  if (actual_d != expected_d) return HXO_ERR_INVALID_DIMENSION;
  for (size_t i = 0; i < actual_d; ++i)
    if (!isfinite(v[i])) {
      if (bad_index) *bad_index = (uint32_t)i;
      return HXO_ERR_INVALID_VECTOR_COMPONENT;
    }
  if (metric == HXO_COSINE) {
    int all_zero = 1;
    for (size_t i = 0; i < actual_d; ++i)
      if (!(v[i] == 0.0f)) {
        all_zero = 0;
        break;
      }
    if (all_zero) return HXO_ERR_ZERO_NORM_COSINE;
  }
  float limit;
  if (hxo_component_limit(metric, expected_d, &limit)) {
    for (size_t i = 0; i < actual_d; ++i)
      if (fabsf(v[i]) > limit) {
        if (bad_index) *bad_index = (uint32_t)i;
        return HXO_ERR_MAGNITUDE_EXCEEDED;
      }
  }
  return HXO_OK;
}

/* ------------------------------------------------------------------------------------------
 * Layer selection  V/mod.rs:705-709,769-796
 * ------------------------------------------------------------------------------------------ */
float hxo_default_ml_for_m(uint32_t m) {
  float effective_m = (float)(m < 2 ? 2 : m);
  return 1.0f / logf(effective_m);
}

uint16_t hxo_select_layer_from_uniform(float ml, float uniform) {
  if (!(isfinite(ml) && ml > 0.0f)) ml = hxo_default_ml_for_m(16);
  if (isfinite(uniform)) {
    float lo = FLT_MIN, hi = 1.0f - FLT_EPSILON;
    if (uniform < lo) uniform = lo;
    if (uniform > hi) uniform = hi;
  } else {
    uniform = 0.5f;
  }
  float neg_ln = -logf(uniform);
  float sampled = floorf(neg_ln * ml);
  if (!isfinite(sampled) || sampled <= 0.0f) return 0;
  if (sampled > 63.0f) sampled = 63.0f;
  return (uint16_t)sampled;
}

/* ------------------------------------------------------------------------------------------
 * Restricted planning  V/restricted.rs
 * ------------------------------------------------------------------------------------------ */
int hxo_restricted_plan(uint64_t n_candidates, uint32_t dimension) {
  /* restricted.rs:40-42 thresholds, :426-453 plan */
  uint64_t bytes = n_candidates * (uint64_t)dimension * 4u;
  return (n_candidates <= 256 && bytes <= 4u * 1024u * 1024u) ? 0 : 1;
}

int hxo_restricted_result_count(uint32_t k, uint64_t n_candidates, uint32_t* out_k) {
  /* restricted.rs:200-213; ResultCount::try_new rejects 0 */
  uint64_t c = k < n_candidates ? k : n_candidates;
  if (c == 0) return HXO_ERR_INVALID_PARAMETER;
  if (c > 800) return HXO_ERR_QUERY;
  *out_k = (uint32_t)c;
  return HXO_OK;
}

size_t hxo_deterministic_sample_ids(const uint64_t* ids, size_t n, size_t limit, uint64_t* out) {
  /* restricted.rs:321-342 */
  size_t sample_count = limit < n ? limit : n;
  if (sample_count == n) {
    memcpy(out, ids, n * sizeof(uint64_t));
    return n;
  }
  if (sample_count == 1) {
    out[0] = ids[0];
    return 1;
  }
  uint64_t last_rank = (uint64_t)n - 1;
  for (size_t s = 0; s < sample_count; ++s) {
    unsigned __int128 r = (unsigned __int128)s * last_rank / (unsigned __int128)(sample_count - 1);
    out[s] = ids[(size_t)r];
  }
  return sample_count;
}

/* ------------------------------------------------------------------------------------------
 * Fixtures
 * ------------------------------------------------------------------------------------------ */
void hxo_fixture_xorshift_vector(uint64_t entity_id, uint32_t d, float* out) {
  uint64_t state = entity_id + 0x9e3779b97f4a7c15ULL;
  for (uint32_t i = 0; i < d; ++i) {
    state ^= state << 13;
    state ^= state >> 7;
    state ^= state << 17;
    int32_t centered = (int32_t)(uint16_t)(state & 0xffff) - 32768;
    out[i] = (float)centered / 32768.0f;
  }
}

void hxo_fixture_circle_vector(uint64_t entity_id, uint64_t entity_count, float* out2) {
  double angle = 6.283185307179586 /* std::f64::consts::TAU */ * (double)entity_id / (double)entity_count;
  out2[0] = (float)cos(angle);
  out2[1] = (float)sin(angle);
}

static int cmp_u64(const void* a, const void* b) {
  uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
  return x < y ? -1 : (x > y ? 1 : 0);
}

size_t hxo_fixture_skip_neighbors(uint64_t entity_id, uint64_t entity_count, uint64_t* out, size_t cap) {
  uint64_t tmp[160];
  size_t n = 0;
  uint64_t offset = 1;
  while (offset < entity_count) {
    uint64_t forward = (entity_id - 1 + offset) % entity_count + 1;
    uint64_t backward = (entity_id - 1 + entity_count - offset % entity_count) % entity_count + 1;
    if (forward != entity_id && n < 160) tmp[n++] = forward;
    if (backward != entity_id && n < 160) tmp[n++] = backward;
    if (offset > UINT64_MAX / 2) break;
    offset *= 2;
  }
  qsort(tmp, n, sizeof(uint64_t), cmp_u64);
  size_t w = 0;
  for (size_t i = 0; i < n; ++i)
    if (w == 0 || tmp[w - 1] != tmp[i]) tmp[w++] = tmp[i];
  if (w > cap) w = cap;
  memcpy(out, tmp, w * sizeof(uint64_t));
  return w;
}

/* ------------------------------------------------------------------------------------------
 * In-memory index
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  uint16_t nlayers; /* rows for layers 1..nlayers (some may be absent => present[l]=0) */
  uint8_t* present; /* [nlayers] */
  uint32_t* deg;    /* [nlayers] */
  uint32_t* raw;    /* [nlayers] row length including ids without vectors */
  uint32_t* nbr;    /* [nlayers * capu_alloc] */
  uint32_t cap;     /* per-row capacity */
} upper_rows;

struct hxo_index {
  int metric;
  uint32_t dim, m, m0, efc;
  uint32_t lim_upper, lim0; /* MutationDegreeLimits: upper = m, layer0 = max(m0, 2m) (mutation.rs:179-199) */
  uint32_t stride0;         /* storage stride for layer-0 rows (>= lim0 + 1, and >= any imported row) */
  size_t n, cap;
  uint64_t* ids;
  float* vecs;
  float* hdr;
  uint8_t* has_vec;
  uint8_t* has_row0;
  uint32_t* nbr0;
  uint32_t* deg0;
  upper_rows** up;
  int32_t* level; /* highest layer with a row, -1 none */
  /* id -> slot */
  uint64_t* hk;
  uint32_t* hv;
  size_t hcap, hcount;
  int populated;
  uint64_t entry_id;
  uint16_t max_layer;
  uint64_t count;
  /* node fingerprints ([0x12] SimHash rows), allocated by hxo_index_put_simhash */
  uint64_t* simhash;
  uint8_t* has_simhash;
  size_t sim_cap;
};

static uint64_t mix64(uint64_t x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33;
  return x;
}

static void hash_grow(hxo_index* ix) {
  size_t ncap = ix->hcap ? ix->hcap * 2 : 1024;
  uint64_t* nk = (uint64_t*)malloc(ncap * sizeof(uint64_t));
  uint32_t* nv = (uint32_t*)malloc(ncap * sizeof(uint32_t));
  for (size_t i = 0; i < ncap; ++i) nv[i] = UINT32_MAX;
  for (size_t i = 0; i < ix->hcap; ++i)
    if (ix->hv[i] != UINT32_MAX) {
      size_t p = mix64(ix->hk[i]) & (ncap - 1);
      while (nv[p] != UINT32_MAX) p = (p + 1) & (ncap - 1);
      nk[p] = ix->hk[i];
      nv[p] = ix->hv[i];
    }
  free(ix->hk);
  free(ix->hv);
  ix->hk = nk;
  ix->hv = nv;
  ix->hcap = ncap;
}

static uint32_t slot_of(const hxo_index* ix, uint64_t id) {
  if (!ix->hcap) return UINT32_MAX;
  size_t p = mix64(id) & (ix->hcap - 1);
  while (ix->hv[p] != UINT32_MAX) {
    if (ix->hk[p] == id) return ix->hv[p];
    p = (p + 1) & (ix->hcap - 1);
  }
  return UINT32_MAX;
}

static void reserve_nodes(hxo_index* ix, size_t want) {
  if (want <= ix->cap) return;
  size_t ncap = ix->cap ? ix->cap : 1024;
  while (ncap < want) ncap *= 2;
  ix->ids = (uint64_t*)realloc(ix->ids, ncap * sizeof(uint64_t));
  ix->vecs = (float*)realloc(ix->vecs, ncap * (size_t)ix->dim * sizeof(float));
  ix->hdr = (float*)realloc(ix->hdr, ncap * sizeof(float));
  ix->has_vec = (uint8_t*)realloc(ix->has_vec, ncap);
  ix->has_row0 = (uint8_t*)realloc(ix->has_row0, ncap);
  ix->nbr0 = (uint32_t*)realloc(ix->nbr0, ncap * (size_t)ix->stride0 * sizeof(uint32_t));
  ix->deg0 = (uint32_t*)realloc(ix->deg0, ncap * sizeof(uint32_t));
  ix->up = (upper_rows**)realloc(ix->up, ncap * sizeof(upper_rows*));
  ix->level = (int32_t*)realloc(ix->level, ncap * sizeof(int32_t));
  ix->cap = ncap;
}

static uint32_t slot_get_or_create(hxo_index* ix, uint64_t id) {
  uint32_t s = slot_of(ix, id);
  if (s != UINT32_MAX) return s;
  if ((ix->hcount + 1) * 2 > ix->hcap) hash_grow(ix);
  reserve_nodes(ix, ix->n + 1);
  s = (uint32_t)ix->n++;
  ix->ids[s] = id;
  ix->hdr[s] = 0.0f;
  ix->has_vec[s] = 0;
  ix->has_row0[s] = 0;
  ix->deg0[s] = 0;
  ix->up[s] = NULL;
  ix->level[s] = -1;
  size_t p = mix64(id) & (ix->hcap - 1);
  while (ix->hv[p] != UINT32_MAX) p = (p + 1) & (ix->hcap - 1);
  ix->hk[p] = id;
  ix->hv[p] = s;
  ix->hcount++;
  return s;
}

hxo_index* hxo_index_new(int metric, uint32_t dim, uint32_t m, uint32_t m0, uint32_t ef_construction) {
  if (dim == 0 || m == 0 || metric < 0 || metric > 2) return NULL;
  hxo_index* ix = (hxo_index*)calloc(1, sizeof(hxo_index));
  ix->metric = metric;
  ix->dim = dim;
  ix->m = m;
  ix->m0 = m0;
  ix->efc = ef_construction;
  ix->lim_upper = m;
  ix->lim0 = m0 >= 2 * m ? m0 : 2 * m;
  ix->stride0 = ix->lim0 + 1;
  return ix;
}

void hxo_index_free(hxo_index* ix) {
  if (!ix) return;
  for (size_t i = 0; i < ix->n; ++i)
    if (ix->up[i]) {
      free(ix->up[i]->present);
      free(ix->up[i]->deg);
      free(ix->up[i]->raw);
      free(ix->up[i]->nbr);
      free(ix->up[i]);
    }
  free(ix->ids);
  free(ix->vecs);
  free(ix->hdr);
  free(ix->has_vec);
  free(ix->has_row0);
  free(ix->nbr0);
  free(ix->deg0);
  free(ix->up);
  free(ix->level);
  free(ix->hk);
  free(ix->hv);
  free(ix->simhash);
  free(ix->has_simhash);
  free(ix);
}

size_t hxo_index_len(const hxo_index* ix) { return (size_t)ix->count; }
uint32_t hxo_index_layer0_limit(const hxo_index* ix) { return ix->lim0; }

int hxo_index_state(const hxo_index* ix, uint64_t* entry_point, uint16_t* max_layer) {
  if (!ix->populated) return 0;
  if (entry_point) *entry_point = ix->entry_id;
  if (max_layer) *max_layer = ix->max_layer;
  return 1;
}

static void ensure_stride0(hxo_index* ix, uint32_t need) {
  if (need <= ix->stride0) return;
  uint32_t ns = ix->stride0;
  while (ns < need) ns *= 2;
  uint32_t* nn = (uint32_t*)malloc(ix->cap * (size_t)ns * sizeof(uint32_t));
  for (size_t s = 0; s < ix->n; ++s)
    memcpy(nn + s * (size_t)ns, ix->nbr0 + s * (size_t)ix->stride0, ix->deg0[s] * sizeof(uint32_t));
  free(ix->nbr0);
  ix->nbr0 = nn;
  ix->stride0 = ns;
}

static upper_rows* upper_ensure(hxo_index* ix, uint32_t slot, uint16_t layer, uint32_t need_cap) {
  upper_rows* u = ix->up[slot];
  uint32_t cap = ix->lim_upper + 1;
  if (need_cap > cap) cap = need_cap;
  if (!u) {
    u = (upper_rows*)calloc(1, sizeof(upper_rows));
    u->cap = cap;
    ix->up[slot] = u;
  }
  if (cap > u->cap) {
    uint32_t* nn = (uint32_t*)calloc((size_t)u->nlayers * cap + 1, sizeof(uint32_t));
    for (uint16_t l = 0; l < u->nlayers; ++l)
      memcpy(nn + (size_t)l * cap, u->nbr + (size_t)l * u->cap, u->deg[l] * sizeof(uint32_t));
    free(u->nbr);
    u->nbr = nn;
    u->cap = cap;
  }
  if (layer > u->nlayers) {
    u->present = (uint8_t*)realloc(u->present, layer);
    u->deg = (uint32_t*)realloc(u->deg, layer * sizeof(uint32_t));
    u->raw = (uint32_t*)realloc(u->raw, layer * sizeof(uint32_t));
    u->nbr = (uint32_t*)realloc(u->nbr, (size_t)layer * u->cap * sizeof(uint32_t));
    for (uint16_t l = u->nlayers; l < layer; ++l) {
      u->present[l] = 0;
      u->deg[l] = 0;
      u->raw[l] = 0;
    }
    u->nlayers = layer;
  }
  return u;
}

/* neighbour-row accessors: a missing row is the deployed empty-neighbour state
 * (search.rs:152-153 `unwrap_or_default`, :201-203) */
static const uint32_t* row_get(const hxo_index* ix, uint16_t layer, uint32_t slot, uint32_t* deg) {
  if (layer == 0) {
    *deg = ix->has_row0[slot] ? ix->deg0[slot] : 0;
    return ix->nbr0 + (size_t)slot * ix->stride0;
  }
  const upper_rows* u = ix->up[slot];
  if (!u || layer > u->nlayers || !u->present[layer - 1]) {
    *deg = 0;
    return NULL;
  }
  *deg = u->deg[layer - 1];
  return u->nbr + (size_t)(layer - 1) * u->cap;
}

static int cmp_slot_by_id_ctx(const void* a, const void* b, void* ctx) {
  const hxo_index* ix = (const hxo_index*)ctx;
  uint64_t x = ix->ids[*(const uint32_t*)a], y = ix->ids[*(const uint32_t*)b];
  return x < y ? -1 : (x > y ? 1 : 0);
}

/* stage_neighbors_vec_for_mutation (mutation.rs:1291-1307): canonical ascending node-id order */
static void row_set(hxo_index* ix, uint16_t layer, uint32_t slot, const uint32_t* nbrs, uint32_t n) {
  uint32_t* dst;
  if (layer == 0) {
    ensure_stride0(ix, n);
    dst = ix->nbr0 + (size_t)slot * ix->stride0;
    ix->has_row0[slot] = 1;
    ix->deg0[slot] = n;
  } else {
    upper_rows* u = upper_ensure(ix, slot, layer, n);
    dst = u->nbr + (size_t)(layer - 1) * u->cap;
    u->present[layer - 1] = 1;
    u->deg[layer - 1] = n;
    u->raw[layer - 1] = n;
  }
  if (n) memmove(dst, nbrs, n * sizeof(uint32_t));
  qsort_r(dst, n, sizeof(uint32_t), cmp_slot_by_id_ctx, ix);
  if ((int32_t)layer > ix->level[slot]) ix->level[slot] = layer;
}

int hxo_index_put_vector(hxo_index* ix, uint64_t id, const float* v) {
  uint32_t bad;
  int rc = hxo_validate_vector(ix->metric, ix->dim, v, ix->dim, &bad);
  if (rc) return rc;
  uint32_t s = slot_get_or_create(ix, id);
  memcpy(ix->vecs + (size_t)s * ix->dim, v, ix->dim * sizeof(float));
  ix->hdr[s] = hxo_header(ix->metric, v, ix->dim);
  if (!ix->has_vec[s]) ix->count++;
  ix->has_vec[s] = 1;
  return HXO_OK;
}

int hxo_index_put_vectors(hxo_index* ix, const uint64_t* ids, const float* rows, size_t n) {
  reserve_nodes(ix, ix->n + n);
  for (size_t i = 0; i < n; ++i) {
    int rc = hxo_index_put_vector(ix, ids[i], rows + i * (size_t)ix->dim);
    if (rc) return rc;
  }
  return HXO_OK;
}

int hxo_index_put_neighbors(hxo_index* ix, uint16_t layer, uint64_t id, const uint64_t* nbrs, size_t n) {
  uint32_t s = slot_get_or_create(ix, id);
  uint32_t* tmp = (uint32_t*)malloc((n + 1) * sizeof(uint32_t));
  for (size_t i = 0; i < n; ++i) tmp[i] = slot_get_or_create(ix, nbrs[i]);
  row_set(ix, layer, s, tmp, (uint32_t)n);
  free(tmp);
  return HXO_OK;
}

int hxo_index_set_entry(hxo_index* ix, uint64_t entry_point, uint16_t max_layer) {
  ix->populated = 1;
  ix->entry_id = entry_point;
  ix->max_layer = max_layer;
  return HXO_OK;
}

size_t hxo_index_node_ids(const hxo_index* ix, uint64_t* out, size_t cap) {
  size_t w = 0;
  for (size_t s = 0; s < ix->n && w < cap; ++s)
    if (ix->has_vec[s]) out[w++] = ix->ids[s];
  qsort(out, w, sizeof(uint64_t), cmp_u64);
  return w;
}

int hxo_index_node_level(const hxo_index* ix, uint64_t id) {
  uint32_t s = slot_of(ix, id);
  return s == UINT32_MAX ? -1 : ix->level[s];
}

size_t hxo_index_get_neighbors(const hxo_index* ix, uint16_t layer, uint64_t id, uint64_t* out, size_t cap) {
  uint32_t s = slot_of(ix, id);
  if (s == UINT32_MAX) return 0;
  uint32_t deg;
  const uint32_t* r = row_get(ix, layer, s, &deg);
  size_t w = 0;
  for (uint32_t i = 0; i < deg && w < cap; ++i) out[w++] = ix->ids[r[i]];
  return w;
}

int hxo_index_get_vector(const hxo_index* ix, uint64_t id, float* out) {
  uint32_t s = slot_of(ix, id);
  if (s == UINT32_MAX || !ix->has_vec[s]) return HXO_ERR_INDEX_NOT_FOUND;
  memcpy(out, ix->vecs + (size_t)s * ix->dim, ix->dim * sizeof(float));
  return HXO_OK;
}

/* ------------------------------------------------------------------------------------------
 * Candidate ordering  V/model.rs:41-61: (score, then node_id)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  float score;
  uint32_t slot;
} cand;

static inline int cand_less(const hxo_index* ix, cand a, cand b) {
  if (a.score < b.score) return 1;
  if (a.score > b.score) return 0;
  return ix->ids[a.slot] < ix->ids[b.slot];
}

typedef struct {
  cand* a;
  size_t n, cap;
} heap;

static void heap_reserve(heap* h, size_t want) {
  if (want <= h->cap) return;
  size_t nc = h->cap ? h->cap * 2 : 256;
  while (nc < want) nc *= 2;
  h->a = (cand*)realloc(h->a, nc * sizeof(cand));
  h->cap = nc;
}
/* max==0: min-heap (BinaryHeap<Reverse<Candidate>>); max==1: max-heap (BinaryHeap<Candidate>) */
static inline int heap_before(const hxo_index* ix, int max, cand a, cand b) {
  return max ? cand_less(ix, b, a) : cand_less(ix, a, b);
}
static void heap_push(const hxo_index* ix, heap* h, int max, cand c) {
  heap_reserve(h, h->n + 1);
  size_t i = h->n++;
  while (i > 0) {
    size_t p = (i - 1) / 2;
    if (!heap_before(ix, max, c, h->a[p])) break;
    h->a[i] = h->a[p];
    i = p;
  }
  h->a[i] = c;
}
static cand heap_pop(const hxo_index* ix, heap* h, int max) {
  cand top = h->a[0];
  cand last = h->a[--h->n];
  size_t i = 0;
  for (;;) {
    size_t l = 2 * i + 1, r = l + 1;
    if (l >= h->n) break;
    size_t c = (r < h->n && heap_before(ix, max, h->a[r], h->a[l])) ? r : l;
    if (!heap_before(ix, max, h->a[c], last)) break;
    h->a[i] = h->a[c];
    i = c;
  }
  if (h->n) h->a[i] = last;
  return top;
}

static int cmp_cand_ctx(const void* a, const void* b, void* ctx) {
  const hxo_index* ix = (const hxo_index*)ctx;
  cand x = *(const cand*)a, y = *(const cand*)b;
  if (cand_less(ix, x, y)) return -1;
  if (cand_less(ix, y, x)) return 1;
  return 0;
}

/* per-thread scratch */
typedef struct {
  uint32_t* stamp;
  size_t stamp_n;
  uint32_t epoch;
  heap cands, w;
  uint32_t* frontier;
  size_t frontier_cap;
} scratch;

static void scratch_begin(scratch* sc, size_t n) {
  if (sc->stamp_n < n) {
    free(sc->stamp);
    sc->stamp = (uint32_t*)calloc(n, sizeof(uint32_t));
    sc->stamp_n = n;
    sc->epoch = 0;
  }
  if (++sc->epoch == 0) {
    memset(sc->stamp, 0, sc->stamp_n * sizeof(uint32_t));
    sc->epoch = 1;
  }
  sc->cands.n = 0;
  sc->w.n = 0;
}
static void scratch_free(scratch* sc) {
  free(sc->stamp);
  free(sc->cands.a);
  free(sc->w.a);
  free(sc->frontier);
  memset(sc, 0, sizeof(*sc));
}
static inline int visited_insert(scratch* sc, uint32_t slot) { /* HashSet::insert: 1 if newly inserted */
  if (sc->stamp[slot] == sc->epoch) return 0;
  sc->stamp[slot] = sc->epoch;
  return 1;
}
static inline int visited_contains(const scratch* sc, uint32_t slot) { return sc->stamp[slot] == sc->epoch; }

static inline float dist_q(const hxo_index* ix, const float* q, float q_hdr, uint32_t slot) {
  return hxo_distance(ix->metric, q, q_hdr, ix->vecs + (size_t)slot * ix->dim, ix->hdr[slot], ix->dim);
}

/* V/search.rs:169-224 search_layer_greedy (and its mutation twin mutation.rs:1008-1064) */
static int greedy_slot(const hxo_index* ix, scratch* sc, const float* q, float q_hdr, uint32_t entry_slot,
                       uint16_t layer, uint32_t* out_slot, hxo_stats* st) {
  scratch_begin(sc, ix->n);
  uint32_t current = entry_slot;
  if (entry_slot == UINT32_MAX || !ix->has_vec[entry_slot]) { /* missing entry item: return entry unchanged */
    *out_slot = entry_slot;
    return HXO_OK;
  }
  float current_dist = dist_q(ix, q, q_hdr, current);
  int rc = hxo_score_validate(&current_dist);
  if (rc) return rc;
  visited_insert(sc, current);
  for (;;) {
    uint32_t deg;
    const uint32_t* nbrs = row_get(ix, layer, current, &deg);
    int changed = 0;
    for (uint32_t i = 0; i < deg; ++i) {
      uint32_t nb = nbrs[i];
      if (!visited_insert(sc, nb)) continue;
      if (!ix->has_vec[nb]) continue;
      float d = dist_q(ix, q, q_hdr, nb);
      rc = hxo_score_validate(&d);
      if (rc) return rc;
      if (d < current_dist) {
        current = nb;
        current_dist = d;
        changed = 1;
      }
    }
    if (!changed) break;
    if (st) st->upper_layer_steps++;
  }
  *out_slot = current;
  return HXO_OK;
}

static __thread scratch tls_scratch;

int hxo_search_layer_greedy(const hxo_index* ix, const float* query, uint64_t entry, uint16_t layer,
                            uint64_t* out_node) {
  uint32_t es = slot_of(ix, entry);
  if (es == UINT32_MAX) { /* unknown entry is returned unchanged (tests/.../search.rs:268-274) */
    *out_node = entry;
    return HXO_OK;
  }
  float qh = hxo_header(ix->metric, query, ix->dim);
  uint32_t out;
  int rc = greedy_slot(ix, &tls_scratch, query, qh, es, layer, &out, NULL);
  if (rc) return rc;
  *out_node = ix->ids[out];
  return HXO_OK;
}

/* V/search.rs:267-1067 with STRICT_EXHAUSTIVE = true: SimHashDecision::exhaustive() (:595-596), no
 * pre-sampling, no filter, every unvisited neighbour admitted to scoring and marked visited
 * (:830-831, mark_sampled_neighbors_visited :89-97), simhash_fill_slots stays 0. */
static int layer0_strict(const hxo_index* ix, scratch* sc, const float* q, float q_hdr, uint32_t entry_slot,
                         uint32_t ef, hxo_stats* st) {
  scratch_begin(sc, ix->n);
  if (entry_slot == UINT32_MAX || !ix->has_vec[entry_slot]) return HXO_OK; /* :463-499 empty results */
  float entry_dist = dist_q(ix, q, q_hdr, entry_slot);
  if (st) st->distance_computations++;
  int rc = hxo_score_validate(&entry_dist);
  if (rc) return rc;
  cand e = {entry_dist, entry_slot};
  heap_push(ix, &sc->cands, 0, e);
  heap_push(ix, &sc->w, 1, e);
  visited_insert(sc, entry_slot);

  while (sc->cands.n) {
    if (st) st->expansion_steps++;
    cand current = heap_pop(ix, &sc->cands, 0);
    if (sc->w.n >= ef && current.score > sc->w.a[0].score) break; /* :549 */

    uint32_t deg;
    const uint32_t* nbrs = row_get(ix, 0, current.slot, &deg);
    if (st) st->neighbors_examined += deg;
    if (sc->frontier_cap < deg) {
      sc->frontier = (uint32_t*)realloc(sc->frontier, (deg + 64) * sizeof(uint32_t));
      sc->frontier_cap = deg + 64;
    }
    uint32_t nf = 0;
    for (uint32_t i = 0; i < deg; ++i)
      if (!visited_contains(sc, nbrs[i])) sc->frontier[nf++] = nbrs[i]; /* :583-589 */
    if (!nf) continue;
    for (uint32_t i = 0; i < nf; ++i) visited_insert(sc, sc->frontier[i]); /* :830-831 */
    for (uint32_t i = 0; i < nf; ++i) {                                     /* :909-953, neighbour-id order */
      uint32_t nb = sc->frontier[i];
      if (!ix->has_vec[nb]) continue; /* :910-912 */
      if (st) st->vectors_loaded++;
      float d = dist_q(ix, q, q_hdr, nb);
      if (st) st->distance_computations++;
      rc = hxo_score_validate(&d);
      if (rc) return rc;
      if (d < sc->w.a[0].score || sc->w.n < ef) { /* :935 */
        cand c = {d, nb};
        heap_push(ix, &sc->cands, 0, c);
        heap_push(ix, &sc->w, 1, c);
        while (sc->w.n > ef) heap_pop(ix, &sc->w, 1); /* :947-952 */
      }
    }
  }
  return HXO_OK;
}

static int search_impl(const hxo_index* ix, scratch* sc, const float* query, uint32_t query_dim, uint32_t k,
                       uint32_t ef, uint64_t* out_ids, float* out_scores, uint32_t* out_count, hxo_stats* st) {
  *out_count = 0;
  if (k == 0) return HXO_ERR_INVALID_PARAMETER;      /* ResultCount::try_new */
  if (ef == 0) ef = k > 100 ? k : 100;               /* SearchParams::new mod.rs:482-487 */
  if (ef < k) return HXO_ERR_INVALID_PARAMETER;      /* SearchBeamWidth::try_new */
  uint32_t bad;
  int rc = hxo_validate_vector(ix->metric, ix->dim, query, query_dim, &bad); /* search.rs:1120-1125 */
  if (rc) return rc;
  if (!ix->populated) return HXO_OK;                 /* search.rs:1127-1128 */
  float qh = hxo_header(ix->metric, query, ix->dim); /* search.rs:1135-1138 */
  uint32_t entry = slot_of(ix, ix->entry_id);
  for (int layer = ix->max_layer; layer >= 1; --layer) { /* search.rs:1150-1156 */
    if (entry == UINT32_MAX) break;
    rc = greedy_slot(ix, sc, query, qh, entry, (uint16_t)layer, &entry, st);
    if (rc) return rc;
  }
  rc = layer0_strict(ix, sc, query, qh, entry, ef, st);
  if (rc) return rc;
  /* search.rs:994-1004 sort by (score,id); :1229 take(k) */
  qsort_r(sc->w.a, sc->w.n, sizeof(cand), cmp_cand_ctx, (void*)ix);
  uint32_t n = sc->w.n < k ? (uint32_t)sc->w.n : k;
  for (uint32_t i = 0; i < n; ++i) {
    out_ids[i] = ix->ids[sc->w.a[i].slot];
    out_scores[i] = sc->w.a[i].score;
  }
  *out_count = n;
  return HXO_OK;
}

int hxo_search(const hxo_index* ix, const float* query, uint32_t query_dim, uint32_t k, uint32_t ef,
               uint64_t* out_ids, float* out_scores, uint32_t* out_count, hxo_stats* stats) {
  if (stats) memset(stats, 0, sizeof(*stats));
  return search_impl(ix, &tls_scratch, query, query_dim, k, ef, out_ids, out_scores, out_count, stats);
}

/* V/restricted.rs:753-835 restricted_exact_scan (+ :661-704 restricted_score_keys): iterate the bitmap
 * ascending, skip ids without a vector row (:615-659 — an id present in the graph but lacking its
 * SimHash row is an error there; the flat image has no SimHash rows), keep the k smallest by
 * (score,id) in a max-heap, sort. */
static int restricted_impl(const hxo_index* ix, scratch* sc, const float* query, uint32_t query_dim, uint32_t k,
                           const uint64_t* cand_ids, size_t n_cand, uint64_t* out_ids, float* out_scores,
                           uint32_t* out_count, uint64_t* ndist) {
  *out_count = 0;
  if (ndist) *ndist = 0;
  if (n_cand == 0) return HXO_OK; /* RestrictedVectorCandidates::Empty, restricted.rs:539-541 */
  if (n_cand > 1000000) return HXO_ERR_QUERY; /* restricted.rs:40,356-371 */
  uint32_t kk;
  int rc = hxo_restricted_result_count(k, n_cand, &kk);
  if (rc) return rc;
  uint32_t bad;
  rc = hxo_validate_vector(ix->metric, ix->dim, query, query_dim, &bad);
  if (rc) return rc;
  if (!ix->populated) return HXO_OK; /* restricted.rs:563-566 */
  float qh = hxo_header(ix->metric, query, ix->dim);
  sc->w.n = 0;
  for (size_t i = 0; i < n_cand; ++i) {
    uint32_t s = slot_of(ix, cand_ids[i]);
    if (s == UINT32_MAX || !ix->has_vec[s]) continue;
    float d = dist_q(ix, query, qh, s);
    if (ndist) (*ndist)++;
    rc = hxo_score_validate(&d);
    if (rc) return rc;
    cand c = {d, s};
    heap_push(ix, &sc->w, 1, c);
    if (sc->w.n > kk) heap_pop(ix, &sc->w, 1);
  }
  qsort_r(sc->w.a, sc->w.n, sizeof(cand), cmp_cand_ctx, (void*)ix);
  for (size_t i = 0; i < sc->w.n; ++i) {
    out_ids[i] = ix->ids[sc->w.a[i].slot];
    out_scores[i] = sc->w.a[i].score;
  }
  *out_count = (uint32_t)sc->w.n;
  return HXO_OK;
}

int hxo_search_restricted(const hxo_index* ix, const float* query, uint32_t query_dim, uint32_t k,
                          const uint64_t* cand_ids, size_t n_cand, uint64_t* out_ids, float* out_scores,
                          uint32_t* out_count, uint64_t* distance_computations) {
  return restricted_impl(ix, &tls_scratch, query, query_dim, k, cand_ids, n_cand, out_ids, out_scores,
                         out_count, distance_computations);
}

static int exact_impl(const hxo_index* ix, scratch* sc, const float* query, uint32_t k, uint64_t* out_ids,
                      float* out_scores, uint32_t* out_count) {
  *out_count = 0;
  if (k == 0) return HXO_ERR_INVALID_PARAMETER;
  float qh = hxo_header(ix->metric, query, ix->dim);
  sc->w.n = 0;
  for (size_t s = 0; s < ix->n; ++s) {
    if (!ix->has_vec[s]) continue;
    float d = dist_q(ix, query, qh, (uint32_t)s);
    int rc = hxo_score_validate(&d);
    if (rc) return rc;
    if (sc->w.n == k && !(d < sc->w.a[0].score || (d == sc->w.a[0].score && ix->ids[s] < ix->ids[sc->w.a[0].slot])))
      continue;
    cand c = {d, (uint32_t)s};
    heap_push(ix, &sc->w, 1, c);
    if (sc->w.n > k) heap_pop(ix, &sc->w, 1);
  }
  qsort_r(sc->w.a, sc->w.n, sizeof(cand), cmp_cand_ctx, (void*)ix);
  for (size_t i = 0; i < sc->w.n; ++i) {
    out_ids[i] = ix->ids[sc->w.a[i].slot];
    out_scores[i] = sc->w.a[i].score;
  }
  *out_count = (uint32_t)sc->w.n;
  return HXO_OK;
}

int hxo_search_exact(const hxo_index* ix, const float* query, uint32_t k, uint64_t* out_ids, float* out_scores,
                     uint32_t* out_count) {
  return exact_impl(ix, &tls_scratch, query, k, out_ids, out_scores, out_count);
}

/* ------------------------------------------------------------------------------------------
 * Filter-aware (ACORN-style) restricted search  V/restricted.rs:837-1148
 *   budgets :220-260, deterministic seeds :321-342, candidate keys :615-659, scoring :661-704,
 *   bridges :706-751.  Restated for generations WITHOUT the SimHash routing directory
 *   (simhash_directory_enabled() == false => no directory seeds, :866-925 skipped): seeds are the
 *   evenly spaced sample of the candidate set plus the entry point when it is a candidate.
 * Every heap / set is the reference's (BinaryHeap<Reverse<Candidate>>, BinaryHeap<Candidate>,
 * BinaryHeap<Reverse<(u32, NodeId)>>, HashSet<NodeId>); only their iteration-independent behaviour is used.
 * The scoring order inside one batch (physical key order) only permutes heap pushes and cannot change a result.
 * ------------------------------------------------------------------------------------------ */
typedef struct { uint64_t* k; size_t cap, n; } idset;   /* open addressing, key + 1 stored (0 = empty) */
static void idset_init(idset* s, size_t cap) {
  size_t c = 64;
  while (c < cap * 2) c <<= 1;
  s->k = (uint64_t*)calloc(c, sizeof(uint64_t));
  s->cap = c;
  s->n = 0;
}
static void idset_grow(idset* s);
static int idset_insert(idset* s, uint64_t id) { /* 1 if newly inserted */
  if ((s->n + 1) * 2 > s->cap) idset_grow(s);
  size_t h = (size_t)((id * 0x9E3779B97F4A7C15ULL) >> 17) & (s->cap - 1);
  for (;;) {
    if (s->k[h] == 0) { s->k[h] = id + 1; s->n++; return 1; }
    if (s->k[h] == id + 1) return 0;
    h = (h + 1) & (s->cap - 1);
  }
}
static int idset_contains(const idset* s, uint64_t id) {
  size_t h = (size_t)((id * 0x9E3779B97F4A7C15ULL) >> 17) & (s->cap - 1);
  for (;;) {
    if (s->k[h] == 0) return 0;
    if (s->k[h] == id + 1) return 1;
    h = (h + 1) & (s->cap - 1);
  }
}
static void idset_grow(idset* s) {
  idset o = *s;
  s->cap = o.cap * 2;
  s->k = (uint64_t*)calloc(s->cap, sizeof(uint64_t));
  s->n = 0;
  for (size_t i = 0; i < o.cap; ++i)
    if (o.k[i]) idset_insert(s, o.k[i] - 1);
  free(o.k);
}

typedef struct { uint32_t ham; uint64_t id; } bridge_key;
typedef struct { bridge_key* a; size_t n, cap; } bridge_heap;   /* min-heap on (hamming, id) */
static int bridge_less(bridge_key x, bridge_key y) { return x.ham < y.ham || (x.ham == y.ham && x.id < y.id); }
static void bridge_push(bridge_heap* h, bridge_key c) {
  if (h->n == h->cap) { h->cap = h->cap ? h->cap * 2 : 256; h->a = (bridge_key*)realloc(h->a, h->cap * sizeof(bridge_key)); }
  size_t i = h->n++;
  while (i > 0) {
    size_t p = (i - 1) / 2;
    if (!bridge_less(c, h->a[p])) break;
    h->a[i] = h->a[p];
    i = p;
  }
  h->a[i] = c;
}
static bridge_key bridge_pop(bridge_heap* h) {
  bridge_key top = h->a[0], last = h->a[--h->n];
  size_t i = 0;
  for (;;) {
    size_t l = 2 * i + 1, r = l + 1;
    if (l >= h->n) break;
    size_t c = (r < h->n && bridge_less(h->a[r], h->a[l])) ? r : l;
    if (!bridge_less(h->a[c], last)) break;
    h->a[i] = h->a[c];
    i = c;
  }
  if (h->n) h->a[i] = last;
  return top;
}

static int allowed_contains(const uint64_t* c, size_t n, uint64_t id) {
  size_t lo = 0, hi = n;
  while (lo < hi) {
    size_t mid = lo + (hi - lo) / 2;
    if (c[mid] < id) lo = mid + 1; else hi = mid;
  }
  return lo < n && c[lo] == id;
}

typedef struct {
  const hxo_index* ix;
  const float* q;
  float qh;
  heap frontier, top;   /* min-heap / max-heap of cand (oracle slots) */
  idset scored;
  size_t beam_width;
  hxo_filtered_stats* st;
} fg_score;

/* restricted_candidate_keys (:615-659) + restricted_score_keys (:661-704) for `ids` (already de-duplicated by the caller) */
static int fg_score_ids(fg_score* f, const uint64_t* ids, size_t n) {
  size_t nkeys = 0;
  uint32_t* slots = (uint32_t*)malloc((n + 1) * sizeof(uint32_t));
  for (size_t i = 0; i < n; ++i) {
    const uint32_t s = slot_of(f->ix, ids[i]);
    f->st->simhash_row_requests++;
    if (s == UINT32_MAX || !f->ix->has_vec[s]) continue;                      /* absent candidate: skipped */
    if (!f->ix->simhash || !f->ix->has_simhash[s]) { free(slots); return HXO_ERR_INVARIANT_VIOLATION; }   /* missing_simhash_error */
    if (idset_contains(&f->scored, ids[i])) continue;                         /* keyed.retain(!scored) */
    slots[nkeys++] = s;
  }
  if (nkeys) {
    f->st->vector_payload_requests += nkeys;
    for (size_t i = 0; i < nkeys; ++i) {
      float d = dist_q(f->ix, f->q, f->qh, slots[i]);
      int rc = hxo_score_validate(&d);
      if (rc) { free(slots); return rc; }
      f->st->distance_computations++;
      cand c = {d, slots[i]};
      idset_insert(&f->scored, f->ix->ids[slots[i]]);
      heap_push(f->ix, &f->frontier, 0, c);
      heap_push(f->ix, &f->top, 1, c);
      if (f->top.n > f->beam_width) heap_pop(f->ix, &f->top, 1);
    }
  }
  free(slots);
  return HXO_OK;
}

/* restricted_enqueue_bridges (:706-751) */
static int fg_enqueue_bridges(const hxo_index* ix, uint64_t qsim, const uint64_t* ids, size_t n, idset* queued,
                              bridge_heap* bh, hxo_filtered_stats* st) {
  for (size_t i = 0; i < n; ++i) {
    if (!idset_insert(queued, ids[i])) continue;
    const uint32_t s = slot_of(ix, ids[i]);
    st->simhash_row_requests++;
    if (s == UINT32_MAX || !ix->simhash || !ix->has_simhash[s]) return HXO_ERR_INVARIANT_VIOLATION;   /* mandatory companion */
    bridge_key b = {(uint32_t)__builtin_popcountll(ix->simhash[s] ^ qsim), ids[i]};
    bridge_push(bh, b);
    st->bridge_frontier_pushes++;
  }
  return HXO_OK;
}

/* FilteredGraphBudgets::with_beam_percent (:232-260) */
void hxo_filtered_budgets(uint32_t k_req, uint32_t ef, uint32_t beam_percent, size_t n_cand, hxo_filtered_budgets_t* b) {
  const size_t k = k_req < n_cand ? k_req : n_cand;
  if (beam_percent == 0) beam_percent = 150;                          /* FILTERED_BEAM_PERCENT */
  if (ef == 0) ef = k_req > 100 ? k_req : 100;
  size_t ef_filtered = (size_t)ef * beam_percent / 100;
  if (ef_filtered < k * 4) ef_filtered = k * 4;
  if (ef_filtered > n_cand) ef_filtered = n_cand;
  b->ef_filtered = ef_filtered;
  b->routing_rows = ef_filtered * 16;
  b->bridge_rows = ef_filtered * 8;
  b->vector_payloads = n_cand < 800 ? n_cand : 800;
  b->sampled_seeds = n_cand < 64 ? n_cand : 64;
}

int hxo_search_filtered_graph(const hxo_index* ix, const float* query, uint32_t k_req, uint32_t ef, uint32_t beam_percent,
                              const uint64_t* cand_ids, size_t n_cand, uint64_t query_simhash, uint64_t* out_ids,
                              float* out_scores, uint32_t* out_count, hxo_filtered_stats* stats) {
  hxo_filtered_budgets_t b;
  hxo_filtered_budgets(k_req, ef, beam_percent, n_cand, &b);
  return hxo_search_filtered_graph_budgets(ix, query, k_req, &b, cand_ids, n_cand, query_simhash, out_ids, out_scores,
                                           out_count, stats);
}

int hxo_search_filtered_graph_budgets(const hxo_index* ix, const float* query, uint32_t k_req,
                                      const hxo_filtered_budgets_t* budgets, const uint64_t* cand_ids, size_t n_cand,
                                      uint64_t query_simhash, uint64_t* out_ids, float* out_scores, uint32_t* out_count,
                                      hxo_filtered_stats* stats) {
  hxo_filtered_stats local;
  if (!stats) stats = &local;
  memset(stats, 0, sizeof(*stats));
  *out_count = 0;
  if (k_req == 0 || n_cand == 0) return n_cand == 0 ? HXO_OK : HXO_ERR_INVALID_PARAMETER;
  if (n_cand > 1000000) return HXO_ERR_QUERY;
  const size_t k = k_req < n_cand ? k_req : n_cand;                   /* RestrictedResultCount (:200-213) */
  if (k > 800) return HXO_ERR_QUERY;
  if (!ix->populated) return HXO_OK;
  const size_t ef_filtered = budgets->ef_filtered, routing_rows = budgets->routing_rows, bridge_rows = budgets->bridge_rows;
  const size_t vector_payloads = budgets->vector_payloads, sampled_seeds = budgets->sampled_seeds;
  const uint64_t entry = ix->entry_id;
  const int entry_allowed = allowed_contains(cand_ids, n_cand, entry);

  fg_score f;
  memset(&f, 0, sizeof(f));
  f.ix = ix;
  f.q = query;
  f.qh = hxo_header(ix->metric, query, ix->dim);
  f.beam_width = ef_filtered;
  f.st = stats;
  idset_init(&f.scored, 1024);
  idset attempted, expanded, queued, eligible_seen;
  idset_init(&attempted, 1024);
  idset_init(&expanded, 1024);
  idset_init(&queued, 1024);
  idset_init(&eligible_seen, 256);
  bridge_heap bh = {0, 0, 0};
  uint64_t* buf = (uint64_t*)malloc((sampled_seeds + 2) * sizeof(uint64_t));
  uint64_t* routing = (uint64_t*)malloc(17 * sizeof(uint64_t));
  uint64_t* bridges = (uint64_t*)malloc(257 * sizeof(uint64_t));
  size_t elig_cap = 1024, rej_cap = 1024, n_elig = 0, n_rej = 0;
  uint64_t* eligible = (uint64_t*)malloc(elig_cap * sizeof(uint64_t));
  uint64_t* rejected = (uint64_t*)malloc(rej_cap * sizeof(uint64_t));
  int rc = HXO_OK;

  /* seeds: the evenly spaced sample, then the entry point when it is a candidate; truncated to the payload budget */
  size_t n_init = hxo_deterministic_sample_ids(cand_ids, n_cand, sampled_seeds, buf);
  for (size_t i = 0; i < n_init; ++i) idset_insert(&attempted, buf[i]);
  {   /* restricted_candidate_keys: an id without a vector row has no key (:629-640) */
    size_t w = 0;
    for (size_t i = 0; i < n_init; ++i) {
      const uint32_t s = slot_of(ix, buf[i]);
      if (s == UINT32_MAX || !ix->has_vec[s]) { stats->simhash_row_requests++; continue; }
      buf[w++] = buf[i];
    }
    n_init = w;
  }
  if (entry_allowed && idset_insert(&attempted, entry)) buf[n_init++] = entry;   /* :948-960 */
  if (n_init > vector_payloads) n_init = vector_payloads;                        /* initial_keys.truncate (:961) */
  rc = fg_score_ids(&f, buf, n_init);
  if (!rc && !entry_allowed) rc = fg_enqueue_bridges(ix, query_simhash, &entry, 1, &queued, &bh, stats);

#define FG_CLASSIFY(node_slot)                                                                          \
  do {                                                                                                  \
    if (ix->has_row0[node_slot]) {                                                                      \
      const uint32_t* row = ix->nbr0 + (size_t)(node_slot) * ix->stride0;                               \
      for (uint32_t j = 0; j < ix->deg0[node_slot]; ++j) {                                              \
        const uint64_t nid = ix->ids[row[j]];                                                           \
        if (allowed_contains(cand_ids, n_cand, nid)) {                                                  \
          if (!idset_contains(&attempted, nid) && idset_insert(&eligible_seen, nid)) {                  \
            if (n_elig == elig_cap) { elig_cap *= 2; eligible = (uint64_t*)realloc(eligible, elig_cap * sizeof(uint64_t)); } \
            eligible[n_elig++] = nid;                                                                   \
          }                                                                                             \
        } else {                                                                                        \
          if (n_rej == rej_cap) { rej_cap *= 2; rejected = (uint64_t*)realloc(rejected, rej_cap * sizeof(uint64_t)); } \
          rejected[n_rej++] = nid;                                                                      \
        }                                                                                               \
      }                                                                                                 \
    }                                                                                                   \
  } while (0)

  while (!rc) {
    if (stats->vector_payload_requests >= vector_payloads) { stats->termination = HXO_FG_VECTOR_BUDGET; break; }
    if (bh.n == 0 && f.top.n >= ef_filtered && f.frontier.n && f.top.n &&
        cand_less(ix, f.top.a[0], f.frontier.a[0])) {               /* next > worst */
      stats->termination = HXO_FG_BEAM_COMPLETE;
      break;
    }
    size_t n_routing = 0;
    while (n_routing < 16 && f.frontier.n) {
      cand c = heap_pop(ix, &f.frontier, 0);
      if (idset_insert(&expanded, ix->ids[c.slot])) routing[n_routing++] = ix->ids[c.slot];
    }
    if (n_routing == 0 && bh.n == 0) { stats->termination = HXO_FG_EXHAUSTED; break; }
    size_t routing_remaining = routing_rows > stats->routing_rows ? routing_rows - stats->routing_rows : 0;
    if (routing_remaining == 0) { stats->termination = HXO_FG_ROUTING_BUDGET; break; }
    if (n_routing > routing_remaining) n_routing = routing_remaining;
    n_elig = 0;
    n_rej = 0;
    memset(eligible_seen.k, 0, eligible_seen.cap * sizeof(uint64_t));
    eligible_seen.n = 0;
    if (n_routing) {
      stats->routing_rows += n_routing;
      routing_remaining -= n_routing;
      for (size_t i = 0; i < n_routing; ++i) {
        const uint32_t s = slot_of(ix, routing[i]);
        if (s != UINT32_MAX) FG_CLASSIFY(s);
      }
    }
    rc = fg_enqueue_bridges(ix, query_simhash, rejected, n_rej, &queued, &bh, stats);
    if (rc) break;
    n_rej = 0;
    const size_t bridge_remaining = bridge_rows > stats->bridge_rows ? bridge_rows - stats->bridge_rows : 0;
    size_t bl = bridge_remaining < routing_remaining ? bridge_remaining : routing_remaining;
    if (bl > 256) bl = 256;
    if (bl > bh.n) bl = bh.n;
    if (bl) {
      for (size_t i = 0; i < bl; ++i) bridges[i] = bridge_pop(&bh).id;
      stats->routing_rows += bl;
      stats->bridge_rows += bl;
      for (size_t i = 0; i < bl; ++i) {
        const uint32_t s = slot_of(ix, bridges[i]);
        if (s != UINT32_MAX) FG_CLASSIFY(s);
      }
      rc = fg_enqueue_bridges(ix, query_simhash, rejected, n_rej, &queued, &bh, stats);
      if (rc) break;
    } else if (n_routing == 0 && bh.n) {
      stats->termination = HXO_FG_BRIDGE_BUDGET;
      break;
    }
    const size_t vector_remaining = vector_payloads > stats->vector_payload_requests
                                        ? vector_payloads - stats->vector_payload_requests : 0;
    if (vector_remaining == 0) { stats->termination = HXO_FG_VECTOR_BUDGET; break; }
    size_t take = vector_remaining < ef_filtered ? vector_remaining : ef_filtered;
    if (n_elig > take) n_elig = take;
    if (n_elig == 0) continue;
    for (size_t i = 0; i < n_elig; ++i) idset_insert(&attempted, eligible[i]);
    rc = fg_score_ids(&f, eligible, n_elig);
  }
#undef FG_CLASSIFY
  if (!rc) {
    qsort_r(f.top.a, f.top.n, sizeof(cand), cmp_cand_ctx, (void*)ix);
    const size_t n = f.top.n < k ? f.top.n : k;
    for (size_t i = 0; i < n; ++i) {
      out_ids[i] = ix->ids[f.top.a[i].slot];
      out_scores[i] = f.top.a[i].score;
    }
    *out_count = (uint32_t)n;
  }
  free(f.frontier.a); free(f.top.a); free(f.scored.k); free(attempted.k); free(expanded.k); free(queued.k);
  free(eligible_seen.k); free(bh.a); free(buf); free(routing); free(bridges); free(eligible); free(rejected);
  return rc;
}

/* ------------------------------------------------------------------------------------------
 * Build: V/mutation.rs:642-1005,1498-1591 + V/mod.rs:809-856
 * ------------------------------------------------------------------------------------------ */

/* search_layer_beam (mutation.rs:904-1005): visited on discovery; admit `w.len() < ef || d < w.max`;
 * result sorted ascending by (score,id). Output in sc->w.a[0..sc->w.n). */
static int beam_for_insert(const hxo_index* ix, scratch* sc, const float* q, float q_hdr, uint32_t entry_slot,
                           uint16_t layer, uint32_t ef) {
  scratch_begin(sc, ix->n);
  if (entry_slot == UINT32_MAX || !ix->has_vec[entry_slot]) return HXO_OK;
  float ed = dist_q(ix, q, q_hdr, entry_slot);
  int rc = hxo_score_validate(&ed);
  if (rc) return rc;
  cand e = {ed, entry_slot};
  heap_push(ix, &sc->cands, 0, e);
  heap_push(ix, &sc->w, 1, e);
  visited_insert(sc, entry_slot);
  while (sc->cands.n) {
    cand current = heap_pop(ix, &sc->cands, 0);
    if (sc->w.n >= ef && current.score > sc->w.a[0].score) break;
    uint32_t deg;
    const uint32_t* nbrs = row_get(ix, layer, current.slot, &deg);
    if (sc->frontier_cap < deg) {
      sc->frontier = (uint32_t*)realloc(sc->frontier, (deg + 64) * sizeof(uint32_t));
      sc->frontier_cap = deg + 64;
    }
    uint32_t nf = 0;
    for (uint32_t i = 0; i < deg; ++i)
      if (visited_insert(sc, nbrs[i])) sc->frontier[nf++] = nbrs[i];
    for (uint32_t i = 0; i < nf; ++i) {
      uint32_t nb = sc->frontier[i];
      if (!ix->has_vec[nb]) continue;
      float d = dist_q(ix, q, q_hdr, nb);
      rc = hxo_score_validate(&d);
      if (rc) return rc;
      if (sc->w.n < ef || d < sc->w.a[0].score) {
        cand c = {d, nb};
        heap_push(ix, &sc->cands, 0, c);
        heap_push(ix, &sc->w, 1, c);
        if (sc->w.n > ef) heap_pop(ix, &sc->w, 1);
      }
    }
  }
  qsort_r(sc->w.a, sc->w.n, sizeof(cand), cmp_cand_ctx, (void*)ix);
  return HXO_OK;
}

/* select_diverse (mod.rs:809-856).  `resolvable[i]` = get_item(candidates[i]) is Some.
 * Returns number selected into out (selection order). */
static int select_diverse(const hxo_index* ix, const cand* candidates, size_t nc, const uint8_t* resolvable,
                          uint32_t m, uint32_t* out, uint32_t* out_n) {
  uint32_t ns = 0;
  uint8_t* taken = (uint8_t*)calloc(nc + 1, 1);
  for (size_t i = 0; i < nc && ns < m; ++i) {
    if (!resolvable[i]) continue;
    uint32_t c = candidates[i].slot;
    int diverse = 1;
    for (uint32_t s = 0; s < ns; ++s) {
      float pd = hxo_distance(ix->metric, ix->vecs + (size_t)c * ix->dim, ix->hdr[c],
                              ix->vecs + (size_t)out[s] * ix->dim, ix->hdr[out[s]], ix->dim);
      int rc = hxo_score_validate(&pd);
      if (rc) {
        free(taken);
        return rc;
      }
      if (pd < candidates[i].score) {
        diverse = 0;
        break;
      }
    }
    if (diverse) {
      out[ns++] = c;
      taken[i] = 1;
    }
  }
  if (ns < m) { /* backfill with closest remaining resolvable */
    for (size_t i = 0; i < nc && ns < m; ++i) {
      if (!resolvable[i] || taken[i]) continue;
      /* selected_ids.insert(c.node_id): candidates are unique per list */
      out[ns++] = candidates[i].slot;
      taken[i] = 1;
    }
  }
  free(taken);
  *out_n = ns;
  return HXO_OK;
}

static int row_contains(const uint32_t* r, uint32_t n, uint32_t x) {
  for (uint32_t i = 0; i < n; ++i)
    if (r[i] == x) return 1;
  return 0;
}

/* remove_edge_from_neighbor (mutation.rs:1890-1908) */
static void remove_edge(hxo_index* ix, uint16_t layer, uint32_t neighbor, uint32_t node_to_remove) {
  uint32_t deg;
  const uint32_t* r = row_get(ix, layer, neighbor, &deg);
  if (!row_contains(r, deg, node_to_remove)) return;
  uint32_t* tmp = (uint32_t*)malloc((deg + 1) * sizeof(uint32_t));
  uint32_t w = 0;
  for (uint32_t i = 0; i < deg; ++i)
    if (r[i] != node_to_remove) tmp[w++] = r[i];
  row_set(ix, layer, neighbor, tmp, w);
  free(tmp);
}

/* add_bidirectional_link (mutation.rs:1498-1591) */
static int add_bidirectional_link(hxo_index* ix, uint16_t layer, uint32_t from, uint32_t to, uint32_t max_nbrs) {
  uint32_t deg;
  const uint32_t* r = row_get(ix, layer, to, &deg);
  uint32_t n = deg;
  uint32_t* to_nbrs = (uint32_t*)malloc((deg + 2) * sizeof(uint32_t));
  memcpy(to_nbrs, r, deg * sizeof(uint32_t));
  if (!row_contains(to_nbrs, n, from)) to_nbrs[n++] = from;
  uint32_t ncand = n;
  uint32_t* candidate_nbrs = (uint32_t*)malloc((ncand + 1) * sizeof(uint32_t));
  memcpy(candidate_nbrs, to_nbrs, ncand * sizeof(uint32_t));
  int rc = HXO_OK;
  if (n > max_nbrs) {
    if (ix->has_vec[to]) {
      cand* distances = (cand*)malloc(n * sizeof(cand));
      uint8_t* resolvable = (uint8_t*)malloc(n);
      uint32_t nd = 0;
      const float* tv = ix->vecs + (size_t)to * ix->dim;
      for (uint32_t i = 0; i < n; ++i) {
        uint32_t nb = to_nbrs[i];
        if (!ix->has_vec[nb]) continue;
        float d = hxo_distance(ix->metric, tv, ix->hdr[to], ix->vecs + (size_t)nb * ix->dim, ix->hdr[nb], ix->dim);
        rc = hxo_score_validate(&d);
        if (rc) break;
        distances[nd].score = d;
        distances[nd].slot = nb;
        resolvable[nd] = 1;
        nd++;
      }
      if (!rc) {
        qsort_r(distances, nd, sizeof(cand), cmp_cand_ctx, ix);
        uint32_t ns;
        rc = select_diverse(ix, distances, nd, resolvable, max_nbrs, to_nbrs, &ns);
        n = ns;
      }
      free(distances);
      free(resolvable);
    } else {
      n = max_nbrs; /* truncate */
    }
  }
  if (!rc) {
    row_set(ix, layer, to, to_nbrs, n);
    uint32_t rdeg;
    const uint32_t* retained = row_get(ix, layer, to, &rdeg);
    /* copy retained since remove_edge may realloc rows */
    uint32_t* ret = (uint32_t*)malloc((rdeg + 1) * sizeof(uint32_t));
    memcpy(ret, retained, rdeg * sizeof(uint32_t));
    for (uint32_t i = 0; i < ncand; ++i)
      if (!row_contains(ret, rdeg, candidate_nbrs[i])) remove_edge(ix, layer, candidate_nbrs[i], to);
    free(ret);
  }
  free(to_nbrs);
  free(candidate_nbrs);
  return rc;
}

/* insert_with_mutation_cache (mutation.rs:642-780) + insert_hnsw (:787-895) */
int hxo_index_insert(hxo_index* ix, uint64_t id, const float* v, uint16_t node_layer) {
  if (slot_of(ix, id) != UINT32_MAX && ix->has_vec[slot_of(ix, id)]) return HXO_ERR_INVALID_PARAMETER; /* fresh build only */
  int rc = hxo_index_put_vector(ix, id, v);
  if (rc) return rc;
  uint32_t node = slot_of(ix, id);
  scratch* sc = &tls_scratch;
  const float* q = ix->vecs + (size_t)node * ix->dim;
  float qh = ix->hdr[node];

  if (!ix->populated) { /* mutation.rs:706-739 */
    ix->populated = 1;
    ix->entry_id = id;
    ix->max_layer = node_layer;
    for (uint16_t l = 0; l <= node_layer; ++l) row_set(ix, l, node, NULL, 0);
    return HXO_OK;
  }
  uint16_t old_max = ix->max_layer;
  uint32_t cur = slot_of(ix, ix->entry_id);
  if (node_layer < old_max) {
    for (int layer = old_max; layer >= (int)node_layer + 1; --layer) {
      rc = greedy_slot(ix, sc, q, qh, cur, (uint16_t)layer, &cur, NULL);
      if (rc) return rc;
    }
  }
  uint16_t top = old_max < node_layer ? old_max : node_layer;
  for (int layer = top; layer >= 0; --layer) {
    uint32_t ef = layer == 0 ? (ix->efc > ix->lim0 ? ix->efc : ix->lim0)
                             : (ix->efc > 2 * ix->lim_upper ? ix->efc : 2 * ix->lim_upper);
    rc = beam_for_insert(ix, sc, q, qh, cur, (uint16_t)layer, ef);
    if (rc) return rc;
    size_t nc = sc->w.n;
    cand* candidates = (cand*)malloc((nc + 1) * sizeof(cand));
    memcpy(candidates, sc->w.a, nc * sizeof(cand));
    uint32_t max_nbrs = layer == 0 ? ix->lim0 : ix->lim_upper;
    /* select_neighbors_heuristic (mutation.rs:1072-1098): items only for the first 2*max candidates */
    uint8_t* resolvable = (uint8_t*)calloc(nc + 1, 1);
    for (size_t i = 0; i < nc && i < (size_t)max_nbrs * 2; ++i) resolvable[i] = ix->has_vec[candidates[i].slot];
    uint32_t* nbrs = (uint32_t*)malloc((max_nbrs + 1) * sizeof(uint32_t));
    uint32_t nn;
    rc = select_diverse(ix, candidates, nc, resolvable, max_nbrs, nbrs, &nn);
    if (!rc) {
      row_set(ix, (uint16_t)layer, node, nbrs, nn); /* stage_new_neighbors_for_mutation */
      for (uint32_t i = 0; i < nn && !rc; ++i) rc = add_bidirectional_link(ix, (uint16_t)layer, node, nbrs[i], max_nbrs);
      if (nc) cur = candidates[0].slot; /* mutation.rs:876-878 */
    }
    free(candidates);
    free(resolvable);
    free(nbrs);
    if (rc) return rc;
  }
  if (node_layer > old_max) {
    for (uint16_t l = old_max + 1; l <= node_layer; ++l) row_set(ix, l, node, NULL, 0);
    ix->entry_id = id; /* mutation.rs:769-772 */
    ix->max_layer = node_layer;
  }
  return HXO_OK;
}

/* ------------------------------------------------------------------------------------------
 * Delete: stage_delete_with_metadata (mutation.rs:1658-1773), delete_from_layer (:1819-1888),
 * remove_edge_from_neighbor (:1890-1908), relink_neighbor (:1916-2050), find_best_entry_candidate (:340-394).
 * The reference finds the rows that name the node through its reverse-locator rows (one prefix scan); this in-memory
 * restatement recomputes that set by scanning the rows.  Items resolve at every layer through the canonical row
 * (index.rs:1544-1557 falls back to get_item), i.e. has_vec.  Entry candidates are every live node keyed
 * (u16::MAX - layer, node id): the scan yields the highest layer first, ascending id within it.
 * ------------------------------------------------------------------------------------------ */
static uint32_t* row_copy(const hxo_index* ix, uint16_t layer, uint32_t slot, uint32_t extra, uint32_t* n) {
  uint32_t deg;
  const uint32_t* r = row_get(ix, layer, slot, &deg);
  uint32_t* out = (uint32_t*)malloc(((size_t)deg + extra + 1) * sizeof(uint32_t));
  if (deg) memcpy(out, r, deg * sizeof(uint32_t));
  *n = deg;
  return out;
}

/* distances from `owner` to every member of `members` that has an item, sorted by (score, id) */
static int ranked_from(const hxo_index* ix, uint32_t owner, const uint32_t* members, uint32_t n, uint32_t skip, cand** out,
                       uint32_t* out_n) {
  cand* d = (cand*)malloc(((size_t)n + 1) * sizeof(cand));
  uint32_t nd = 0;
  const float* ov = ix->vecs + (size_t)owner * ix->dim;
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t c = members[i];
    if (c == skip || !ix->has_vec[c]) continue;
    float sc = hxo_distance(ix->metric, ov, ix->hdr[owner], ix->vecs + (size_t)c * ix->dim, ix->hdr[c], ix->dim);
    const int rc = hxo_score_validate(&sc); /* Candidate::try_new */
    if (rc) {
      free(d);
      return rc;
    }
    d[nd].score = sc;
    d[nd].slot = c;
    nd++;
  }
  qsort_r(d, nd, sizeof(cand), cmp_cand_ctx, (void*)ix);
  *out = d;
  *out_n = nd;
  return HXO_OK;
}

static int prune_to_limit(const hxo_index* ix, uint32_t owner, uint32_t* members, uint32_t* n, uint32_t max_nbrs) {
  cand* d;
  uint32_t nd;
  int rc = ranked_from(ix, owner, members, *n, UINT32_MAX, &d, &nd);
  if (rc) return rc;
  uint8_t* resolvable = (uint8_t*)malloc((size_t)nd + 1);
  memset(resolvable, 1, (size_t)nd + 1);
  rc = select_diverse(ix, d, nd, resolvable, max_nbrs, members, n);
  free(resolvable);
  free(d);
  return rc;
}

static int relink_neighbor(hxo_index* ix, uint16_t layer, uint32_t nb, const uint32_t* cands, uint32_t ncands,
                           uint32_t max_nbrs) {
  if (!ix->has_vec[nb]) return HXO_OK; /* :1925-1930 */
  uint32_t n_old, n_cur;
  uint32_t* old = row_copy(ix, layer, nb, 0, &n_old);
  uint32_t* cur = row_copy(ix, layer, nb, max_nbrs + 1, &n_cur);
  cand* ranked;
  uint32_t nr;
  int rc = ranked_from(ix, nb, cands, ncands, nb, &ranked, &nr); /* :1935-1953: HashSet order is erased by the sort */
  if (!rc) {
    for (uint32_t i = 0; i < nr && i < max_nbrs; ++i) /* :1954-1958 */
      if (!row_contains(cur, n_cur, ranked[i].slot)) cur[n_cur++] = ranked[i].slot;
    free(ranked);
    if (n_cur > max_nbrs) rc = prune_to_limit(ix, nb, cur, &n_cur, max_nbrs); /* :1960-1983 */
  }
  if (!rc) {
    row_set(ix, layer, nb, cur, n_cur); /* :1985-1993 (row_set sorts its own copy; `cur` keeps the selection order) */
    for (uint32_t i = 0; i < n_cur && !rc; ++i) { /* :1994-2047: every NEW connection gets its reciprocal edge */
      const uint32_t nn = cur[i];
      if (row_contains(old, n_old, nn)) continue;
      uint32_t n_rev;
      uint32_t* rev = row_copy(ix, layer, nn, 1, &n_rev);
      if (!row_contains(rev, n_rev, nb)) {
        rev[n_rev++] = nb;
        if (n_rev > max_nbrs && ix->has_vec[nn]) rc = prune_to_limit(ix, nn, rev, &n_rev, max_nbrs);
        /* no item for the reverse owner: the over-long row is staged as it is (:2006-2017) */
        if (!rc) row_set(ix, layer, nn, rev, n_rev);
      }
      free(rev);
    }
  }
  free(old);
  free(cur);
  return rc;
}

static int delete_from_layer(hxo_index* ix, uint16_t layer, uint32_t node, uint32_t max_nbrs, const uint32_t* extra,
                             uint32_t n_extra) {
  uint32_t n_out;
  uint32_t* outgoing = row_copy(ix, layer, node, 0, &n_out);
  /* affected = (outgoing \ {node}) U (extra \ {node}), ascending id (BTreeSet) */
  uint32_t* affected = (uint32_t*)malloc(((size_t)n_out + n_extra + 1) * sizeof(uint32_t));
  uint8_t* mandatory = (uint8_t*)calloc((size_t)n_out + n_extra + 1, 1);
  uint32_t na = 0;
  for (uint32_t i = 0; i < n_out; ++i)
    if (outgoing[i] != node && !row_contains(affected, na, outgoing[i])) affected[na++] = outgoing[i];
  const uint32_t n_mand = na;
  for (uint32_t i = 0; i < n_extra; ++i)
    if (extra[i] != node && !row_contains(affected, na, extra[i])) affected[na++] = extra[i];
  int rc = HXO_OK;
  if (na) {
    /* sort by id, carrying the "came from the outgoing row" flag */
    uint32_t* order = (uint32_t*)malloc((size_t)na * sizeof(uint32_t));
    memcpy(order, affected, (size_t)na * sizeof(uint32_t));
    qsort_r(order, na, sizeof(uint32_t), cmp_slot_by_id_ctx, ix);
    for (uint32_t i = 0; i < na; ++i) mandatory[i] = row_contains(affected, n_mand, order[i]) ? 1 : 0;
    uint32_t* relink = (uint32_t*)malloc((size_t)na * sizeof(uint32_t));
    uint32_t nrl = 0;
    for (uint32_t i = 0; i < na; ++i) { /* :1848-1856 */
      uint32_t deg;
      const uint32_t* r = row_get(ix, layer, order[i], &deg);
      const int had_edge = row_contains(r, deg, node);
      if (had_edge) remove_edge(ix, layer, order[i], node);
      if (mandatory[i] || had_edge) relink[nrl++] = order[i]; /* ascending id: `order` is */
    }
    if (nrl) {
      /* candidates (:1861-1876): the relink sources and their remaining neighbours, minus the node */
      size_t cap = nrl;
      for (uint32_t i = 0; i < nrl; ++i) {
        uint32_t deg;
        row_get(ix, layer, relink[i], &deg);
        cap += deg;
      }
      uint32_t* cands = (uint32_t*)malloc((cap + 1) * sizeof(uint32_t));
      uint32_t nc = 0;
      for (uint32_t i = 0; i < nrl; ++i)
        if (relink[i] != node && !row_contains(cands, nc, relink[i])) cands[nc++] = relink[i];
      for (uint32_t i = 0; i < nrl; ++i) {
        uint32_t deg;
        const uint32_t* r = row_get(ix, layer, relink[i], &deg);
        for (uint32_t j = 0; j < deg; ++j)
          if (r[j] != node && r[j] != relink[i] && !row_contains(cands, nc, r[j])) cands[nc++] = r[j];
      }
      for (uint32_t i = 0; i < nrl && !rc; ++i) rc = relink_neighbor(ix, layer, relink[i], cands, nc, max_nbrs);
      free(cands);
    }
    free(relink);
    free(order);
  }
  free(mandatory);
  free(affected);
  free(outgoing);
  return rc;
}

int hxo_index_delete(hxo_index* ix, uint64_t id, int* existed) {
  if (existed) *existed = 0;
  const uint32_t node = slot_of(ix, id);
  if (node == UINT32_MAX) return HXO_OK; /* nothing names an id this index never saw */
  const int item_existed = ix->has_vec[node] ? 1 : 0;
  const int node_max_layer = ix->level[node] > 0 ? ix->level[node] : 0; /* get_node_max_layer_cached :1788-1811 */
  int top = node_max_layer;
  if ((int)ix->max_layer > top) top = ix->max_layer;
  for (size_t s = 0; s < ix->n; ++s)
    if (ix->level[s] > top) top = ix->level[s];
  int rc = HXO_OK;
  uint32_t* src = (uint32_t*)malloc((ix->n + 1) * sizeof(uint32_t));
  for (int layer = top; layer >= 0 && !rc; --layer) { /* layers_to_process, highest first (:1681-1702) */
    uint32_t ns = 0;
    for (size_t s = 0; s < ix->n; ++s) { /* the reverse locators of (layer, node) */
      if ((uint32_t)s == node) continue;
      uint32_t deg;
      const uint32_t* r = row_get(ix, (uint16_t)layer, (uint32_t)s, &deg);
      if (deg && row_contains(r, deg, node)) src[ns++] = (uint32_t)s;
    }
    if (layer > node_max_layer && ns == 0) continue;
    rc = delete_from_layer(ix, (uint16_t)layer, node, layer == 0 ? ix->lim0 : ix->lim_upper, src, ns);
  }
  free(src);
  if (rc) return rc;
  /* the node's own rows, vector and fingerprint (:1711-1737) */
  if (item_existed) {
    ix->has_vec[node] = 0;
    ix->count--;
  }
  ix->has_row0[node] = 0;
  ix->deg0[node] = 0;
  if (ix->up[node]) memset(ix->up[node]->present, 0, ix->up[node]->nlayers);
  ix->level[node] = -1;
  if (ix->has_simhash && node < ix->sim_cap) ix->has_simhash[node] = 0;
  if (ix->populated && ix->entry_id == id) { /* :1751-1763 */
    int best_level = -1;
    uint64_t best_id = 0;
    for (size_t s = 0; s < ix->n; ++s) {
      if (!ix->has_vec[s] || ix->level[s] < 0) continue;
      if (ix->level[s] > best_level || (ix->level[s] == best_level && ix->ids[s] < best_id)) {
        best_level = ix->level[s];
        best_id = ix->ids[s];
      }
    }
    if (best_level < 0) {
      ix->populated = 0; /* entry_point = None, max_layer = 0 */
      ix->entry_id = 0;
      ix->max_layer = 0;
    } else {
      ix->entry_id = best_id;
      ix->max_layer = (uint16_t)best_level;
    }
  }
  if (existed) *existed = item_existed;
  return HXO_OK;
}

/* VectorInsertContract::Upsert (mutation.rs:653-661): an existing item is deleted through the full delete path first,
 * then the vector is inserted like a fresh one (new layer draw, new links). */
int hxo_index_upsert(hxo_index* ix, uint64_t id, const float* v, uint16_t node_layer) {
  const uint32_t s = slot_of(ix, id);
  if (s != UINT32_MAX && ix->has_vec[s]) {
    uint32_t bad;
    int rc = hxo_validate_vector(ix->metric, ix->dim, v, ix->dim, &bad); /* validation precedes every write */
    if (rc) return rc;
    rc = hxo_index_delete(ix, id, NULL);
    if (rc) return rc;
  }
  return hxo_index_insert(ix, id, v, node_layer);
}

/* ------------------------------------------------------------------------------------------
 * Bulk graph import (slot space = rank of ascending id), as downloaded from the device
 * ------------------------------------------------------------------------------------------ */
int hxo_index_import_graph(hxo_index* ix, const uint16_t* levels, const uint32_t* deg0, const uint32_t* nbr0,
                           uint32_t layer0_stride, size_t n_upper_rows, const uint32_t* upper_node,
                           const uint16_t* upper_layer, const uint32_t* upper_deg, const uint32_t* upper_nbr,
                           uint32_t upper_stride, uint64_t entry_point, uint16_t max_layer) {
  /* rank -> oracle slot */
  size_t n = 0;
  uint64_t* sorted = (uint64_t*)malloc(ix->n * sizeof(uint64_t) + 8);
  n = hxo_index_node_ids(ix, sorted, ix->n);
  uint32_t* rank2slot = (uint32_t*)malloc((n + 1) * sizeof(uint32_t));
  for (size_t r = 0; r < n; ++r) rank2slot[r] = slot_of(ix, sorted[r]);
  free(sorted);
  uint32_t* tmp = (uint32_t*)malloc(((size_t)layer0_stride + upper_stride + 2) * sizeof(uint32_t));
  for (size_t r = 0; r < n; ++r) {
    uint32_t d = deg0[r];
    for (uint32_t j = 0; j < d; ++j) tmp[j] = rank2slot[nbr0[r * (size_t)layer0_stride + j]];
    row_set(ix, 0, rank2slot[r], tmp, d);
    (void)levels;
  }
  for (size_t u = 0; u < n_upper_rows; ++u) {
    uint32_t d = upper_deg[u];
    for (uint32_t j = 0; j < d; ++j) tmp[j] = rank2slot[upper_nbr[u * (size_t)upper_stride + j]];
    row_set(ix, upper_layer[u], rank2slot[upper_node[u]], tmp, d);
  }
  free(tmp);
  free(rank2slot);
  return hxo_index_set_entry(ix, entry_point, max_layer);
}

/* ==========================================================================================
 * Non-exhaustive layer 0: policy, session RNG, SimHash (see hx_oracle.h for what is pinned)
 * ========================================================================================== */
void hxo_policy_defaults(hxo_policy_cfg* c) { /* SearchParams::new mod.rs:482-500; config/indexes.rs:398-406 */
  memset(c, 0, sizeof(*c));
  c->mode = HXO_SIMHASH_ADAPTIVE;
  c->threshold = 43;
  c->sampling_ratio = 0.8f;
  c->has_pre_override = 0;
  c->pre_override = 1.0f;
  c->adaptive_enabled = 1;
  c->failure_prob = 0.1f;
  c->bypass_min_frontier = 24;
  c->bypass_window_expansions = 4;
  c->bypass_min_filter_rate = 0.12f;
  c->read_budget_multiplier = 3;
}

static inline float clampf(float x, float lo, float hi) { /* f32::clamp */
  if (x < lo) return lo;
  if (x > hi) return hi;
  return x;
}
static inline float maxf_(float a, float b) { return a > b ? a : b; } /* f32::max for non-NaN operands */
static inline float minf_(float a, float b) { return a < b ? a : b; }
static inline uint32_t max_u32(uint32_t a, uint32_t b) { return a > b ? a : b; }

/* policy.rs:558-574 */
static float adaptive_sampling_ratio(float base, const hxo_policy_ctx* c) {
  if (base >= 1.0f) return base;
  if (c->search_frontier_len < max_u32(c->ef / 3, 8)) return 1.0f;
  const float current = c->current, delta = c->delta;
  if (delta <= 1e-6f) return base;
  const float relative_quality = clampf(1.0f - clampf(current / delta, 0.0f, 1.0f), 0.0f, 1.0f);
  return minf_(clampf(base + (1.0f - base) * relative_quality, base, 1.0f), maxf_(0.90f, base));
}
/* policy.rs:576-597 */
static uint32_t adaptive_threshold(const hxo_policy_ctx* c, uint32_t configured, float failure) {
  uint32_t value;
  if (configured == 0) {
    value = 0;
  } else if (!c->topk_ready) {
    value = 1;
  } else {
    const float normalized = clampf(c->delta, 0.0f, 1.0f);
    const float cosine_similarity = clampf(1.0f - 2.0f * normalized, -1.0f, 1.0f);
    const float collision = 1.0f - acosf(cosine_similarity) / 3.14159274101257324f; /* std::f32::consts::PI */
    const float bits = 64.0f;
    const float margin = sqrtf((bits * logf(1.0f / failure)) / 2.0f);
    const float t = clampf(floorf(bits * collision - margin), 1.0f, bits);
    value = (uint32_t)t;
    if (value > configured) value = configured;
  }
  return value;
}
/* policy.rs:526-537 */
static void activate_sampling(int kind, float prob, uint32_t frontier_len, uint32_t ef, int* out_kind, float* out_prob) {
  if (prob <= 0.0f || prob >= 1.0f || frontier_len > max_u32(ef / 4, 8)) {
    *out_kind = kind;
    *out_prob = prob;
  } else {
    *out_kind = HXO_SAMPLING_EXHAUSTIVE;
    *out_prob = 1.0f;
  }
}
/* policy.rs:539-556 */
static void pre_sampling_decision(float base_ratio, uint32_t frontier_len, uint32_t ef, int* out_kind, float* out_prob) {
  if (base_ratio >= 1.0f || frontier_len <= max_u32(ef / 4, 8)) {
    *out_kind = HXO_SAMPLING_EXHAUSTIVE;
    *out_prob = 1.0f;
    return;
  }
  float ratio = clampf(base_ratio * 0.65f, 0.25f, 0.9f);
  const uint64_t twice = (uint64_t)ef * 2u;
  if (base_ratio <= 0.0f) {
    ratio = 0.0f;
  } else if ((uint64_t)frontier_len > (twice > 32 ? twice : 32)) {
    ratio = maxf_(ratio * 0.8f, 0.20f);
  }
  *out_kind = HXO_SAMPLING_FIXED;
  *out_prob = ratio;
}

void hxo_policy_decide(int metric, const hxo_policy_cfg* cfg, const hxo_policy_ctx* ctx, hxo_policy_decision* d) {
  memset(d, 0, sizeof(*d));
  /* --- AdaptiveBypassPolicy::from_deployed + decide (policy.rs:196-291) */
  int bypassed = 0, next_state = HXO_BYPASS_READY, trigger = HXO_TRIGGER_NONE;
  uint32_t next_remaining = 0;
  if (cfg->mode == HXO_SIMHASH_ADAPTIVE) {
    const uint32_t window = cfg->bypass_window_expansions;
    uint64_t rb = (uint64_t)ctx->ef * cfg->read_budget_multiplier; /* saturating_mul on usize: no overflow here */
    if (rb < cfg->bypass_min_frontier) rb = cfg->bypass_min_frontier;
    int decided = 0;
    if (ctx->bypass_state == HXO_BYPASS_BYPASSING) {
      bypassed = 1;
      if (ctx->bypass_remaining - 1 > 0) {
        next_state = HXO_BYPASS_BYPASSING;
        next_remaining = ctx->bypass_remaining - 1;
      } else {
        next_state = HXO_BYPASS_COOLING;
        next_remaining = window;
      }
      decided = 1;
    } else if (ctx->bypass_state == HXO_BYPASS_COOLING && ctx->bypass_remaining > 1) {
      next_state = HXO_BYPASS_COOLING;
      next_remaining = ctx->bypass_remaining - 1;
      decided = 1;
    }
    if (!decided) {
      const int budget_exhausted = ctx->simhash_filter_reads >= rb;
      const float filter_rate =
          ctx->window_examined == 0 ? 1.0f : (float)ctx->window_filtered / (float)ctx->window_examined;
      const int low_yield = ctx->window_expansions >= window && filter_rate < cfg->bypass_min_filter_rate;
      const int trg = (budget_exhausted ? 1 : 0) | (low_yield ? 2 : 0);
      if (ctx->candidate_frontier_len < cfg->bypass_min_frontier || trg == HXO_TRIGGER_NONE) {
        /* inactive(): not bypassed, Ready, None */
      } else {
        bypassed = 1;
        trigger = trg;
        if (window - 1 > 0) {
          next_state = HXO_BYPASS_BYPASSING;
          next_remaining = window - 1;
        } else {
          next_state = HXO_BYPASS_COOLING;
          next_remaining = window;
        }
      }
    }
  }
  /* --- Layer0Policy::from_deployed (policy.rs:58-107) */
  enum { F_DISABLED, F_FIXED, F_ADAPTIVE } filtering = F_DISABLED;
  if (cfg->mode != HXO_SIMHASH_OFF && metric == HXO_COSINE) {
    if (cfg->mode == HXO_SIMHASH_ALWAYS) filtering = F_FIXED;
    else filtering = cfg->adaptive_enabled ? F_ADAPTIVE : F_FIXED;
  }
  int base_kind;
  float base_prob;
  if (cfg->mode == HXO_SIMHASH_OFF) {
    base_kind = HXO_SAMPLING_EXHAUSTIVE;
    base_prob = 1.0f;
  } else if (cfg->mode == HXO_SIMHASH_ADAPTIVE && cfg->adaptive_enabled) {
    base_kind = HXO_SAMPLING_ADAPTIVE;
    base_prob = adaptive_sampling_ratio(cfg->sampling_ratio, ctx);
  } else {
    base_kind = HXO_SAMPLING_FIXED;
    base_prob = cfg->sampling_ratio;
  }
  /* --- decide (policy.rs:119-175) */
  activate_sampling(base_kind, base_prob, ctx->candidate_frontier_len, ctx->ef, &d->samp_kind, &d->samp_prob);
  d->base_sampling_probability = base_prob;
  pre_sampling_decision(cfg->has_pre_override ? cfg->pre_override : base_prob, ctx->candidate_frontier_len, ctx->ef,
                        &d->pre_kind, &d->pre_prob);
  d->next_state = next_state;
  d->next_remaining = next_remaining;
  d->trigger = trigger;
  if (bypassed) {
    d->bypassed = 1;
    return;
  }
  if (filtering == F_DISABLED) return;
  d->fetch_missing = 1;
  d->filter_cached = 1;
  d->has_threshold = 1;
  d->threshold = filtering == F_FIXED ? cfg->threshold : adaptive_threshold(ctx, cfg->threshold, cfg->failure_prob);
}

float hxo_candidate_probability(const hxo_policy_decision* d, uint32_t similarity_bits) { /* policy.rs:415-430 */
  const float base = d->samp_kind == HXO_SAMPLING_EXHAUSTIVE ? 1.0f : d->samp_prob;
  if (d->samp_kind != HXO_SAMPLING_ADAPTIVE) return base;
  if (base <= 0.0f || base >= 1.0f) return base;
  const float similarity_ratio = (float)(similarity_bits < 64 ? similarity_bits : 64) / 64.0f;
  const float threshold_ratio = d->has_threshold ? (float)d->threshold / 64.0f : 0.0f;
  return clampf(base + (1.0f - base) * maxf_(similarity_ratio - threshold_ratio, 0.0f), base, 1.0f);
}

/* ---- session RNG: rand 0.10 StdRng = ChaCha12; seed_from_u64 = PCG32 expansion (rand_core) -------- */
static inline uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
static inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
#define HXO_QR(a, b, c, d) \
  a += b; d ^= a; d = rotl32(d, 16); c += d; b ^= c; b = rotl32(b, 12); \
  a += b; d ^= a; d = rotl32(d, 8);  c += d; b ^= c; b = rotl32(b, 7);
void hxo_chacha_block(const uint32_t key[8], uint64_t counter, uint64_t stream, int rounds, uint32_t out[16]) {
  uint32_t in[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key[0], key[1], key[2], key[3],
                     key[4],      key[5],      key[6],      key[7],      (uint32_t)counter, (uint32_t)(counter >> 32),
                     (uint32_t)stream, (uint32_t)(stream >> 32)};
  uint32_t x[16];
  memcpy(x, in, sizeof(x));
  for (int i = 0; i < rounds / 2; ++i) {
    HXO_QR(x[0], x[4], x[8], x[12]) HXO_QR(x[1], x[5], x[9], x[13]) HXO_QR(x[2], x[6], x[10], x[14]) HXO_QR(x[3], x[7], x[11], x[15])
    HXO_QR(x[0], x[5], x[10], x[15]) HXO_QR(x[1], x[6], x[11], x[12]) HXO_QR(x[2], x[7], x[8], x[13]) HXO_QR(x[3], x[4], x[9], x[14])
  }
  for (int i = 0; i < 16; ++i) out[i] = x[i] + in[i];
}
void hxo_session_seeded(hxo_session* s, uint64_t seed) { /* randomness.rs:122-132: the RNG is built lazily */
  memset(s, 0, sizeof(*s));
  s->seed = seed;
}
uint64_t hxo_session_seed_for(uint64_t query_simhash, uint64_t entry_point, uint64_t ef) { /* randomness.rs:109-114 */
  return query_simhash ^ rotl64(entry_point, 17) ^ rotl64(ef, 7);
}
/* PCG32's output permutation XSH-RR (xorshift high bits, random rotate) of a 64-bit LCG state; the LCG multiplier is PCG's
 * 6364136223846793005.  Pinned by the PCG reference implementation's demo stream (tests/test_oracle_kat.py). */
uint32_t hxo_pcg32_xsh_rr(uint64_t state) {
  const uint32_t xorshifted = (uint32_t)(((state >> 18) ^ state) >> 27);
  const uint32_t rot = (uint32_t)(state >> 59);
  return (xorshifted >> rot) | (xorshifted << ((32 - rot) & 31)); /* rotate_right */
}
uint64_t hxo_pcg32_step(uint64_t state, uint64_t increment) { return state * 6364136223846793005ull + increment; }
static void session_start(hxo_session* s) { /* SeedableRng::seed_from_u64: PCG32 fills the 32-byte key */
  uint64_t state = s->seed;
  for (int i = 0; i < 8; ++i) {
    state = hxo_pcg32_step(state, 11634580027462260723ull); /* advance FIRST (away from a low-weight seed), then output */
    s->key[i] = hxo_pcg32_xsh_rr(state);                    /* little-endian words of the 32-byte seed */
  }
  s->block = 0;
  s->pos = 16;
  s->started = 1;
}
uint32_t hxo_session_next_u32(hxo_session* s) {
  if (!s->started) session_start(s);
  if (s->pos >= 16) {
    hxo_chacha_block(s->key, s->block++, 0, 12, s->buf); /* ChaCha12, 64-bit block counter, stream 0 */
    s->pos = 0;
  }
  return s->buf[s->pos++];
}
int hxo_session_should_sample(hxo_session* s, float ratio) { /* randomness.rs:141-153 */
  if (ratio >= 1.0f) return 1;
  if (ratio <= 0.0f) return 0;
  const float u = (float)(hxo_session_next_u32(s) >> 8) * (1.0f / 16777216.0f); /* StandardUniform for f32 */
  return u < ratio;
}
int64_t hxo_session_choose_index(hxo_session* s, uint64_t count) { /* randomness.rs:155-158 */
  if (count == 0) return -1;
  if (count > 0xffffffffull) { /* UniformUsize falls to u64 sampling above u32::MAX: not reachable (row lengths) */
    return -1;
  }
  const uint32_t range = (uint32_t)count;
  const uint64_t m = (uint64_t)hxo_session_next_u32(s) * range;
  uint32_t result = (uint32_t)(m >> 32);
  const uint32_t lo_order = (uint32_t)m;
  if (lo_order > (uint32_t)(0u - range)) {
    const uint32_t new_hi = (uint32_t)(((uint64_t)hxo_session_next_u32(s) * range) >> 32);
    if ((uint64_t)lo_order + new_hi > 0xffffffffull) result += 1;
  }
  return (int64_t)result;
}

/* ---- SimHash ------------------------------------------------------------------------------------------ */
uint64_t hxo_simhash_from_planes(const float* planes, const float* v, uint32_t dim) { /* unaligned_vector/simhash.rs:263-290 */
  uint64_t bits = 0;
  for (uint32_t p = 0; p < 64; ++p) {
    float dot = 0.0f;
    const float* h = planes + (size_t)p * dim;
    for (uint32_t i = 0; i < dim; ++i) dot += v[i] * h[i]; /* two roundings (-ffp-contract=off) */
    if (dot > 0.0f) bits |= 1ull << p;
  }
  return bits;
}
uint32_t hxo_simhash_collision_count(uint64_t a, uint64_t b) { return 64u - (uint32_t)__builtin_popcountll(a ^ b); }
uint64_t hxo_order_code_from_simhash_bits(uint64_t bits) { /* simhash.rs:44-59 */
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

int hxo_index_put_simhash(hxo_index* ix, const uint64_t* ids, const uint64_t* bits, size_t n) {
  if (ix->sim_cap < ix->cap) {
    ix->simhash = (uint64_t*)realloc(ix->simhash, ix->cap * sizeof(uint64_t));
    ix->has_simhash = (uint8_t*)realloc(ix->has_simhash, ix->cap);
    memset(ix->has_simhash + ix->sim_cap, 0, ix->cap - ix->sim_cap);
    ix->sim_cap = ix->cap;
  }
  for (size_t i = 0; i < n; ++i) {
    const uint32_t s = slot_of(ix, ids[i]);
    if (s == UINT32_MAX) return HXO_ERR_INVARIANT_VIOLATION;
    ix->simhash[s] = bits[i];
    ix->has_simhash[s] = 1;
  }
  return HXO_OK;
}

/* V/search.rs:267-1067 with STRICT_EXHAUSTIVE = false */
typedef struct { uint32_t slot; uint32_t sim; } sampled_nb;
static int layer0_policy(const hxo_index* ix, scratch* sc, const float* q, float q_hdr, uint32_t entry_slot, uint64_t entry_id,
                         uint32_t k, uint32_t ef, const hxo_policy_cfg* cfg, uint64_t qsim, hxo_stats* st,
                         hxo_policy_stats* ps) {
  scratch_begin(sc, ix->n);
  if (entry_slot == UINT32_MAX || !ix->has_vec[entry_slot]) return HXO_OK;
  hxo_session session;
  hxo_session_seeded(&session, hxo_session_seed_for(qsim, entry_id, ef)); /* search.rs:343-348 */
  heap topk = {0};
  const uint32_t topk_target = k > 1 ? k : 1;
  uint64_t window_examined = 0, window_filtered = 0, window_expansions = 0;
  int bypass_state = HXO_BYPASS_READY;
  uint32_t bypass_remaining = 0;
  const uint64_t simhash_filter_reads = 0; /* resident store: memory_store.rs:331-337 */
  size_t fill = 0;                         /* simhash_fill_slots */
  int rc = HXO_OK;
  sampled_nb *sampled = NULL, *deferred = NULL;
  uint32_t* simfront = NULL;
  size_t cap = 0;

  float entry_dist = dist_q(ix, q, q_hdr, entry_slot);
  if (st) st->distance_computations++;
  rc = hxo_score_validate(&entry_dist);
  if (rc) return rc;
  cand e = {entry_dist, entry_slot};
  heap_push(ix, &sc->cands, 0, e);
  heap_push(ix, &sc->w, 1, e);
  heap_push(ix, &topk, 1, e);
  visited_insert(sc, entry_slot);

  while (sc->cands.n) {
    if (st) st->expansion_steps++;
    cand current = heap_pop(ix, &sc->cands, 0);
    if (sc->w.n + fill >= ef && current.score > sc->w.a[0].score) break; /* :544-551 */
    uint32_t deg;
    const uint32_t* nbrs = row_get(ix, 0, current.slot, &deg);
    if (st) st->neighbors_examined += deg;
    if (cap < deg + 1) {
      cap = deg + 64;
      sc->frontier = (uint32_t*)realloc(sc->frontier, cap * sizeof(uint32_t));
      sc->frontier_cap = cap;
      simfront = (uint32_t*)realloc(simfront, cap * sizeof(uint32_t));
      sampled = (sampled_nb*)realloc(sampled, cap * sizeof(sampled_nb));
      deferred = (sampled_nb*)realloc(deferred, cap * sizeof(sampled_nb));
    }
    uint32_t nf = 0;
    for (uint32_t i = 0; i < deg; ++i)
      if (!visited_contains(sc, nbrs[i])) sc->frontier[nf++] = nbrs[i]; /* :583-589 */
    if (!nf) continue;

    /* :603-637 decision */
    hxo_policy_ctx ctx;
    memset(&ctx, 0, sizeof(ctx));
    ctx.topk_ready = topk.n >= topk_target;
    ctx.ef = ef;
    ctx.search_frontier_len = (uint32_t)sc->w.n;
    ctx.candidate_frontier_len = nf;
    ctx.current = current.score;
    ctx.delta = topk.n ? topk.a[0].score : current.score;
    ctx.bypass_state = bypass_state;
    ctx.bypass_remaining = bypass_remaining;
    ctx.simhash_filter_reads = simhash_filter_reads;
    ctx.window_examined = window_examined;
    ctx.window_filtered = window_filtered;
    ctx.window_expansions = window_expansions;
    hxo_policy_decision dec;
    hxo_policy_decide(ix->metric, cfg, &ctx, &dec);
    bypass_state = dec.next_state;
    bypass_remaining = dec.next_remaining;
    if (ps) {
      if (dec.trigger & HXO_TRIGGER_READ_BUDGET) ps->simhash_bypass_trigger_budget++;
      if (dec.trigger & HXO_TRIGGER_LOW_YIELD) ps->simhash_bypass_trigger_low_yield++;
    }
    const float active_sampling_ratio = dec.samp_kind == HXO_SAMPLING_EXHAUSTIVE ? 1.0f : dec.samp_prob;
    const uint32_t active_threshold = dec.has_threshold ? dec.threshold : 0;

    /* :651-678 stage-0 pre-sampling */
    uint32_t nsf = 0;
    const int pre_enabled = dec.pre_kind != HXO_SAMPLING_EXHAUSTIVE;
    if (pre_enabled) {
      for (uint32_t i = 0; i < nf; ++i) {
        if (hxo_session_should_sample(&session, dec.pre_prob)) simfront[nsf++] = sc->frontier[i];
        else if (ps) ps->pre_simhash_sample_dropped++;
      }
      if (nsf == 0) {
        const int64_t idx = hxo_session_choose_index(&session, nf);
        if (idx < 0) continue;
        simfront[nsf++] = sc->frontier[idx];
      }
      if (ps) ps->pre_simhash_sample_kept += nsf;
    } else {
      memcpy(simfront, sc->frontier, nf * sizeof(uint32_t));
      nsf = nf;
    }
    if (ps && dec.bypassed) { /* :681-685 */
      ps->simhash_bypass_expansions++;
      ps->simhash_skipped_candidates += nsf;
    }

    /* :709-786 threshold gate + sampling */
    uint32_t ns = 0, nd = 0;
    const int should_sample = !pre_enabled && dec.samp_kind != HXO_SAMPLING_EXHAUSTIVE && active_sampling_ratio > 0.0f;
    uint64_t examined_round = 0, filtered_round = 0;
    for (uint32_t i = 0; i < nsf; ++i) {
      const uint32_t nb = simfront[i];
      const int has_hash = dec.filter_cached && ix->has_simhash && ix->has_simhash[nb];
      if (has_hash) {
        examined_round++;
        if (ps) ps->simhash_examined++;
        if (hxo_simhash_collision_count(ix->simhash[nb], qsim) < active_threshold) { /* !passes_threshold */
          if (ps) ps->simhash_filtered++;
          filtered_round++;
          if (visited_insert(sc, nb) && sc->w.n + fill < ef) fill++; /* :742-748 */
          continue;
        }
      } else if (ps && dec.fetch_missing) {
        ps->simhash_missing_hash++;
      }
      if (ps) ps->simhash_passed_before_sampling++;
      const uint32_t similarity_bits = has_hash ? hxo_simhash_collision_count(ix->simhash[nb], qsim) : 32u; /* 64 - hamming */
      if (should_sample) {
        const float p = hxo_candidate_probability(&dec, similarity_bits);
        if (hxo_session_should_sample(&session, p)) sampled[ns++] = (sampled_nb){nb, similarity_bits};
        else deferred[nd++] = (sampled_nb){nb, similarity_bits};
      } else if (active_sampling_ratio <= 0.0f) {
        deferred[nd++] = (sampled_nb){nb, similarity_bits};
      } else {
        sampled[ns++] = (sampled_nb){nb, similarity_bits};
      }
    }
    if (dec.filter_cached && examined_round > 0) { /* :788-800 */
      window_examined += examined_round;
      window_filtered += filtered_round;
      window_expansions += 1;
      if (window_expansions > cfg->bypass_window_expansions) {
        window_examined /= 2;
        window_filtered /= 2;
        window_expansions = cfg->bypass_window_expansions / 2;
      }
    }
    if (active_sampling_ratio > 0.0f && ns == 0 && nd > 0) { /* :802-823 */
      uint32_t best = 0;
      for (uint32_t i = 0; i < nd; ++i)
        if (deferred[i].sim > best) best = deferred[i].sim;
      uint32_t nbest = 0;
      for (uint32_t i = 0; i < nd; ++i)
        if (deferred[i].sim == best) nbest++;
      const int64_t idx = hxo_session_choose_index(&session, nbest);
      if (idx < 0) continue;
      uint32_t seen = 0;
      for (uint32_t i = 0; i < nd; ++i)
        if (deferred[i].sim == best && seen++ == (uint32_t)idx) { /* swap_remove(idx) returns element idx */
          sampled[ns++] = deferred[i];
          break;
        }
    }
    if (ps) ps->simhash_passed_after_sampling += ns;

    /* :830-953 mark visited, score, admit */
    for (uint32_t i = 0; i < ns; ++i) {
      const uint32_t nb = sampled[i].slot;
      if (!visited_insert(sc, nb)) continue; /* mark_sampled_neighbors_visited */
      if (!ix->has_vec[nb]) continue;
      if (st) st->vectors_loaded++;
      float d = dist_q(ix, q, q_hdr, nb);
      if (st) st->distance_computations++;
      rc = hxo_score_validate(&d);
      if (rc) goto done;
      if (d < sc->w.a[0].score || sc->w.n + fill < ef) { /* :927-928 */
        cand c = {d, nb};
        heap_push(ix, &sc->cands, 0, c);
        heap_push(ix, &sc->w, 1, c);
        heap_push(ix, &topk, 1, c);
        if (topk.n > topk_target) heap_pop(ix, &topk, 1);
        while (sc->w.n + fill > ef) { /* :940-951 */
          if (fill > 0) fill--;
          else if (sc->w.n > ef) heap_pop(ix, &sc->w, 1);
          else break;
        }
      }
    }
  }
done:
  if (ps) ps->rng_draws = session.started ? session.block * 16 - (16 - session.pos) : 0;
  free(topk.a);
  free(sampled);
  free(deferred);
  free(simfront);
  return rc;
}

int hxo_search_policy(const hxo_index* ix, const float* query, uint32_t query_dim, uint32_t k, uint32_t ef,
                      const hxo_policy_cfg* cfg, uint64_t qsim, uint64_t* out_ids, float* out_scores, uint32_t* out_count,
                      hxo_stats* st, hxo_policy_stats* ps) {
  scratch* sc = &tls_scratch;
  if (st) memset(st, 0, sizeof(*st));
  if (ps) memset(ps, 0, sizeof(*ps));
  *out_count = 0;
  if (k == 0) return HXO_ERR_INVALID_PARAMETER;
  if (ef == 0) ef = k > 100 ? k : 100;
  if (ef < k) return HXO_ERR_INVALID_PARAMETER;
  uint32_t bad;
  int rc = hxo_validate_vector(ix->metric, ix->dim, query, query_dim, &bad);
  if (rc) return rc;
  if (!ix->populated) return HXO_OK;
  const float qh = hxo_header(ix->metric, query, ix->dim);
  uint32_t entry = slot_of(ix, ix->entry_id);
  for (int layer = ix->max_layer; layer >= 1; --layer) {
    if (entry == UINT32_MAX) break;
    rc = greedy_slot(ix, sc, query, qh, entry, (uint16_t)layer, &entry, st);
    if (rc) return rc;
  }
  /* requires_query_simhash() false (Off, no pre-sampling override < 1) is the strict-exhaustive specialisation */
  const int strict = cfg->mode == HXO_SIMHASH_OFF && !(cfg->has_pre_override && cfg->pre_override < 1.0f);
  if (strict) rc = layer0_strict(ix, sc, query, qh, entry, ef, st);
  else rc = layer0_policy(ix, sc, query, qh, entry, entry == UINT32_MAX ? 0 : ix->ids[entry], k, ef, cfg, qsim, st, ps);
  if (rc) return rc;
  qsort_r(sc->w.a, sc->w.n, sizeof(cand), cmp_cand_ctx, (void*)ix);
  const uint32_t n = sc->w.n < k ? (uint32_t)sc->w.n : k;
  for (uint32_t i = 0; i < n; ++i) {
    out_ids[i] = ix->ids[sc->w.a[i].slot];
    out_scores[i] = sc->w.a[i].score;
  }
  *out_count = n;
  return HXO_OK;
}

/* ------------------------------------------------------------------------------------------
 * Threaded drivers (one query per thread at a time; no intra-query parallelism, like the reference)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  const hxo_index* ix;
  const float* queries;
  size_t nq;
  uint32_t k, ef;
  const uint64_t* cand_ids;
  const uint64_t* cand_offsets;
  uint64_t* out_ids;
  float* out_scores;
  uint32_t* out_counts;
  hxo_stats* stats_sum;
  int mode; /* 0 hnsw, 1 restricted, 2 exact */
  size_t next;
  pthread_mutex_t mu;
  int rc;
} batch_job;

static void* batch_worker(void* arg) {
  batch_job* job = (batch_job*)arg;
  scratch sc;
  memset(&sc, 0, sizeof(sc));
  hxo_stats local;
  memset(&local, 0, sizeof(local));
  for (;;) {
    size_t i = __atomic_fetch_add(&job->next, 1, __ATOMIC_RELAXED);
    if (i >= job->nq) break;
    const float* q = job->queries + i * (size_t)job->ix->dim;
    uint64_t* oi = job->out_ids + i * (size_t)job->k;
    float* os = job->out_scores + i * (size_t)job->k;
    int rc;
    if (job->mode == 0) {
      rc = search_impl(job->ix, &sc, q, job->ix->dim, job->k, job->ef, oi, os, &job->out_counts[i], &local);
    } else if (job->mode == 1) {
      size_t b = job->cand_offsets[i], e = job->cand_offsets[i + 1];
      rc = restricted_impl(job->ix, &sc, q, job->ix->dim, job->k, job->cand_ids + b, e - b, oi, os,
                           &job->out_counts[i], NULL);
    } else {
      rc = exact_impl(job->ix, &sc, q, job->k, oi, os, &job->out_counts[i]);
    }
    if (rc) job->rc = rc;
  }
  if (job->stats_sum) {
    pthread_mutex_lock(&job->mu);
    job->stats_sum->expansion_steps += local.expansion_steps;
    job->stats_sum->neighbors_examined += local.neighbors_examined;
    job->stats_sum->distance_computations += local.distance_computations;
    job->stats_sum->vectors_loaded += local.vectors_loaded;
    job->stats_sum->upper_layer_steps += local.upper_layer_steps;
    pthread_mutex_unlock(&job->mu);
  }
  scratch_free(&sc);
  return NULL;
}

static double run_batch(batch_job* job, int threads) {
  if (threads < 1) threads = 1;
  if (threads > 256) threads = 256;
  pthread_mutex_init(&job->mu, NULL);
  job->next = 0;
  job->rc = 0;
  struct timespec t0, t1;
  clock_gettime(CLOCK_MONOTONIC, &t0);
  pthread_t th[256];
  for (int t = 0; t < threads; ++t) pthread_create(&th[t], NULL, batch_worker, job);
  for (int t = 0; t < threads; ++t) pthread_join(th[t], NULL);
  clock_gettime(CLOCK_MONOTONIC, &t1);
  pthread_mutex_destroy(&job->mu);
  double s = (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
  return job->rc ? -1.0 : s;
}

double hxo_search_batch(const hxo_index* ix, const float* queries, size_t nq, uint32_t k, uint32_t ef, int threads,
                        uint64_t* out_ids, float* out_scores, uint32_t* out_counts, hxo_stats* stats_sum) {
  batch_job job;
  memset(&job, 0, sizeof(job));
  if (stats_sum) memset(stats_sum, 0, sizeof(*stats_sum));
  job.ix = ix;
  job.queries = queries;
  job.nq = nq;
  job.k = k;
  job.ef = ef;
  job.out_ids = out_ids;
  job.out_scores = out_scores;
  job.out_counts = out_counts;
  job.stats_sum = stats_sum;
  job.mode = 0;
  return run_batch(&job, threads);
}

double hxo_search_restricted_batch(const hxo_index* ix, const float* queries, size_t nq, uint32_t k,
                                   const uint64_t* cand_ids, const uint64_t* cand_offsets, int threads,
                                   uint64_t* out_ids, float* out_scores, uint32_t* out_counts) {
  batch_job job;
  memset(&job, 0, sizeof(job));
  job.ix = ix;
  job.queries = queries;
  job.nq = nq;
  job.k = k;
  job.cand_ids = cand_ids;
  job.cand_offsets = cand_offsets;
  job.out_ids = out_ids;
  job.out_scores = out_scores;
  job.out_counts = out_counts;
  job.mode = 1;
  return run_batch(&job, threads);
}

double hxo_search_exact_batch(const hxo_index* ix, const float* queries, size_t nq, uint32_t k, int threads,
                              uint64_t* out_ids, float* out_scores, uint32_t* out_counts) {
  batch_job job;
  memset(&job, 0, sizeof(job));
  job.ix = ix;
  job.queries = queries;
  job.nq = nq;
  job.k = k;
  job.out_ids = out_ids;
  job.out_scores = out_scores;
  job.out_counts = out_counts;
  job.mode = 2;
  return run_batch(&job, threads);
}

/* Threaded driver for the non-exhaustive mode (one query per thread at a time, like hxo_search_batch). */
typedef struct {
  const hxo_index* ix;
  const float* queries;
  const uint64_t* qsim;
  size_t nq;
  uint32_t k, ef;
  const hxo_policy_cfg* cfg;
  uint64_t* out_ids;
  float* out_scores;
  uint32_t* out_counts;
  size_t next;
  pthread_mutex_t mu;
  int rc;
} policy_job;

static void* policy_worker(void* arg) {
  policy_job* j = (policy_job*)arg;
  for (;;) {
    pthread_mutex_lock(&j->mu);
    const size_t q = j->next++;
    pthread_mutex_unlock(&j->mu);
    if (q >= j->nq) break;
    uint32_t cnt = 0;
    const int rc = hxo_search_policy(j->ix, j->queries + q * j->ix->dim, j->ix->dim, j->k, j->ef, j->cfg, j->qsim[q],
                                     j->out_ids + q * j->k, j->out_scores + q * j->k, &cnt, NULL, NULL);
    j->out_counts[q] = cnt;
    if (rc) j->rc = rc;
  }
  scratch_free(&tls_scratch);
  return NULL;
}

double hxo_search_policy_batch(const hxo_index* ix, const float* queries, const uint64_t* qsim, size_t nq, uint32_t k,
                               uint32_t ef, const hxo_policy_cfg* cfg, int threads, uint64_t* out_ids, float* out_scores,
                               uint32_t* out_counts) {
  policy_job j;
  memset(&j, 0, sizeof(j));
  j.ix = ix; j.queries = queries; j.qsim = qsim; j.nq = nq; j.k = k; j.ef = ef; j.cfg = cfg;
  j.out_ids = out_ids; j.out_scores = out_scores; j.out_counts = out_counts;
  pthread_mutex_init(&j.mu, NULL);
  if (threads < 1) threads = 1;
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * (size_t)threads);
  struct timespec t0, t1;
  clock_gettime(CLOCK_MONOTONIC, &t0);
  for (int i = 0; i < threads; ++i) pthread_create(&th[i], NULL, policy_worker, &j);
  for (int i = 0; i < threads; ++i) pthread_join(th[i], NULL);
  clock_gettime(CLOCK_MONOTONIC, &t1);
  free(th);
  pthread_mutex_destroy(&j.mu);
  if (j.rc) return -1.0;
  return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
