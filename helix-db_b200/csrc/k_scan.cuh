// k_scan.cuh — prefiltered brute-force scan + top-k selection.
//
// Restates VectorIndex::restricted_exact_scan (search/vector/restricted.rs:753-835) with
// restricted_score_keys (:661-704): every present candidate is scored with D::distance and the k
// smallest by (score, id) are returned sorted.  The reference takes this branch only for |C| <= 256
// (restricted.rs:40-42,426-453) and otherwise walks the graph approximately; on the device the exact
// scan is HBM-bound and cheap, so it answers every |C| <= 1e6 exactly (SURVEY §8 a11/a12).
//
// k_scan: grid (candidate chunks, queries).  One octet per candidate row (bit-exact octet kernel, rows
// read with coalesced 128-bit loads, each row exactly once per query); emits one 64-bit key
// score_bits<<32 | rank per candidate (rank = position in the ascending candidate list, so key order is
// the reference's (score,id) order).  Algorithmic bytes per candidate: 4*dim (+4 header for cosine).
// k_select: one CTA per query keeps the k smallest keys (threshold filter + bitonic merge in smem).
#pragma once
#include "hx_common.cuh"

#define HX_SCAN_THREADS 256
#define HX_SEL_THREADS 512
#define HX_SEL_HALF 1024            // max k' (restricted k <= 800, restricted.rs:55)

struct HxScanArgs {
  const float* queries;          // [B][dim]
  const float* q_hdr;            // [B]
  const uint32_t* q_status;      // [B]
  uint32_t B;
  const uint32_t* cand_slots;    // candidate slots (HX_ABSENT = id without a vector row: skipped)
  const uint64_t* cand_offsets;  // [B+1] (ignored when shared_set)
  uint64_t* keys;                // one key per (query, candidate)
  uint32_t shared_set;           // all queries scan cand_slots[0 .. n_shared)
  uint64_t n_shared;
  uint32_t chunk;                // candidates per CTA (multiple of 32)
  uint32_t* err_flags;
  // device-resident candidate sets (hx_candidates): per query a pointer, a length and the position of its keys
  const uint32_t* const* q_slots;  // [B] or nullptr
  const uint64_t* q_len;           // [B]
  const uint64_t* q_keyoff;        // [B]
};

template <int METRIC>
static __global__ void __launch_bounds__(HX_SCAN_THREADS) k_scan(HxDev ix, HxScanArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  float* sq = reinterpret_cast<float*>(smem);
  const uint32_t tid = threadIdx.x, t = tid & 7u, oct = tid >> 3;
  for (uint32_t q = blockIdx.y; q < a.B; q += gridDim.y) {
    const uint64_t base = a.q_slots ? 0ull : (a.shared_set ? 0ull : a.cand_offsets[q]);
    const uint64_t n = a.q_slots ? a.q_len[q] : (a.shared_set ? a.n_shared : (a.cand_offsets[q + 1] - base));
    const uint64_t start = (uint64_t)blockIdx.x * a.chunk;
    if (start >= n || a.q_status[q] != 0u) continue;   // uniform per CTA
    const uint64_t end = (start + a.chunk < n) ? start + a.chunk : n;
    const float q_hdr = a.q_hdr[q];
    for (uint32_t i = tid; i < ix.ld; i += HX_SCAN_THREADS)
      sq[i] = i < ix.dim ? a.queries[(size_t)q * ix.dim + i] : 0.0f;
    __syncthreads();
    uint64_t* keys_out = a.keys + (a.q_slots ? a.q_keyoff[q] : (a.shared_set ? (uint64_t)q * a.n_shared : base));
    const uint32_t* slots = a.q_slots ? a.q_slots[q] : a.cand_slots + base;
    if (METRIC == HXM_MANHATTAN) {
      for (uint64_t r = start + tid; r < end; r += HX_SCAN_THREADS) {
        const uint32_t slot = slots[r];
        uint64_t key = HX_KEY_MAX;
        if (slot != HX_ABSENT) {
          float s = hx_manhattan_seq(ix.vec + (size_t)slot * ix.ld, sq, ix.dim);
          if (!hx_score_ok(s)) atomicOr(a.err_flags, HXF_INVALID_SCORE);
          key = hx_make_key(s, (uint32_t)r);
        }
        keys_out[r] = key;
      }
    } else {
      for (uint64_t r = start + oct; r < end; r += HX_SCAN_THREADS / 8) {
        const uint32_t slot = slots[r];
        uint64_t key = HX_KEY_MAX;
        if (slot != HX_ABSENT) {
          float s = hx_octet_score<METRIC>(ix, sq, q_hdr, slot, t);
          if (t == 0) {
            if (!hx_score_ok(s)) atomicOr(a.err_flags, HXF_INVALID_SCORE);
            key = hx_make_key(s, (uint32_t)r);
          }
        }
        if (t == 0) keys_out[r] = key;
      }
    }
    __syncthreads();
  }
}

// ---- fused scan + top-k (k <= 32): ONE launch, no key array ---------------------------------------------------------------
// north_star: "warp-shuffle top-k reduction".  Same grid and the same bit-exact octet scoring as k_scan, but a candidate's
// key never goes to HBM: every warp keeps its HX_TOPK smallest keys sorted across its lanes (lane i = i-th smallest; an
// insertion is one ballot for the rank and one shuffle-up for the shift), the 8 warps of the CTA merge through shared
// memory, the CTA writes its HX_TOPK keys to a small partial array, and the LAST CTA of a query (atomic ticket) merges the
// partials and writes ids / scores / count.  The ticket counter resets itself, so nothing is zeroed per launch.
#define HX_TOPK 32

struct HxTopkArgs {
  uint64_t* partial;        // [B][n_chunks][HX_TOPK]
  uint32_t* tickets;        // [B] zero before the first launch; self-resetting
  uint32_t n_chunks;        // gridDim.x
  uint32_t k;               // requested k (<= HX_TOPK); clamped to |C_q| per query (restricted.rs:200-213)
  uint64_t* out_ids;        // [B][k]
  float* out_scores;
  uint32_t* out_counts;
};

// insert `key` into the warp's sorted list (lane i holds the i-th smallest, HX_KEY_MAX = empty); warp-uniform call
__device__ __forceinline__ void hx_topk_insert(uint64_t& mine, uint64_t key, uint32_t lane) {
  const unsigned FULL = 0xffffffffu;
  const uint32_t pos = __popc(__ballot_sync(FULL, mine < key));   // keys are distinct (rank in the low word)
  if (pos >= HX_TOPK) return;
  const uint64_t up = __shfl_up_sync(FULL, mine, 1);
  if (lane > pos) mine = up;
  else if (lane == pos) mine = key;
}

// top-32 of the union of two ascending 32-lists (lane i holds the i-th smallest of each): min(A[i], B[31-i]) is a
// bitonic sequence made of exactly the 32 smallest keys; five compare-exchange stages sort it.  ~12 shuffles instead of
// up to 32 insertions.
__device__ __forceinline__ uint64_t hx_topk_merge32(uint64_t mine, uint64_t other, uint32_t lane) {
  const unsigned FULL = 0xffffffffu;
  const uint64_t rev = __shfl_sync(FULL, other, 31u - lane);
  uint64_t v = mine < rev ? mine : rev;
#pragma unroll
  for (uint32_t s = 16; s > 0; s >>= 1) {
    const uint64_t p = __shfl_xor_sync(FULL, v, s);
    const bool lower = (lane & s) == 0u;
    v = (lower == (v < p)) ? v : p;   // lower half keeps the min, upper half the max
  }
  return v;
}

template <int METRIC>
static __global__ void __launch_bounds__(HX_SCAN_THREADS, 4) k_scan_topk(HxDev ix, HxScanArgs a, HxTopkArgs tk) {
  extern __shared__ __align__(128) unsigned char smem[];
  float* sq = reinterpret_cast<float*>(smem);
  __shared__ uint64_t s_lists[HX_SCAN_THREADS / 32][HX_TOPK];
  __shared__ uint32_t s_last;
  const uint32_t tid = threadIdx.x, t = tid & 7u, oct = tid >> 3, lane = tid & 31u, warp = tid >> 5;
  const unsigned FULL = 0xffffffffu;
  for (uint32_t q = blockIdx.y; q < a.B; q += gridDim.y) {
    const uint64_t base = a.q_slots ? 0ull : (a.shared_set ? 0ull : a.cand_offsets[q]);
    const uint64_t n = a.q_slots ? a.q_len[q] : (a.shared_set ? a.n_shared : (a.cand_offsets[q + 1] - base));
    const uint64_t start = (uint64_t)blockIdx.x * a.chunk;
    const bool live = a.q_status[q] == 0u && start < n;            // uniform per CTA
    uint64_t mine = HX_KEY_MAX;
    if (live) {
      const uint64_t end = (start + a.chunk < n) ? start + a.chunk : n;
      const float q_hdr = a.q_hdr[q];
      for (uint32_t i = tid; i < ix.ld; i += HX_SCAN_THREADS)
        sq[i] = i < ix.dim ? a.queries[(size_t)q * ix.dim + i] : 0.0f;
      __syncthreads();
      const uint32_t* slots = a.q_slots ? a.q_slots[q] : a.cand_slots + base;
      // every warp walks the chunk in steps of 32 rows (4 octets per warp: rows r, r+1, r+2, r+3 of its step)
      for (uint64_t r0 = start; r0 < end; r0 += HX_SCAN_THREADS / 8) {
        const uint64_t r = r0 + oct;
        uint64_t key = HX_KEY_MAX;
        if (r < end) {
          const uint32_t slot = slots[r];
          if (slot != HX_ABSENT) {
            float s;
            if (METRIC == HXM_MANHATTAN) s = hx_manhattan_seq(ix.vec + (size_t)slot * ix.ld, sq, ix.dim);
            else s = hx_octet_score<METRIC>(ix, sq, q_hdr, slot, t);
            if (!hx_score_ok(s)) atomicOr(a.err_flags, HXF_INVALID_SCORE);
            key = hx_make_key(s, (uint32_t)r);
          }
        }
        // the warp's four candidates of this step, tested against its current k-th before any insertion work
        const uint64_t kth = __shfl_sync(FULL, mine, HX_TOPK - 1);
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const uint64_t c = __shfl_sync(FULL, key, o * 8);
          if (c < kth) hx_topk_insert(mine, c, lane);   // warp-uniform branch (c and kth are broadcasts)
        }
      }
      s_lists[warp][lane] = mine;
    }
    __syncthreads();
    if (live && warp == 0) {   // merge the 8 warp lists (warp 0's own list is already in `mine`)
#pragma unroll
      for (uint32_t w = 1; w < HX_SCAN_THREADS / 32; ++w) mine = hx_topk_merge32(mine, s_lists[w][lane], lane);
    }
    if (warp == 0) {
      // every CTA of the grid row reports (an empty list when it had nothing to scan) so that the ticket count is exact
      tk.partial[((size_t)q * tk.n_chunks + blockIdx.x) * HX_TOPK + lane] = live ? mine : HX_KEY_MAX;
      __threadfence();
      __syncwarp();
      if (lane == 0) {
        const uint32_t tkt = atomicAdd(tk.tickets + q, 1u);
        s_last = (tkt == tk.n_chunks - 1u) ? 1u : 0u;
      }
    }
    __syncthreads();
    if (s_last) {   // the last CTA of this query merges the partial lists: warp w takes chunks w, w+8, ...
      __threadfence();
      uint64_t best = HX_KEY_MAX;
      const uint64_t* P = tk.partial + (size_t)q * tk.n_chunks * HX_TOPK;
      for (uint32_t c = warp; c < tk.n_chunks; c += HX_SCAN_THREADS / 32)
        best = hx_topk_merge32(best, __ldcg(P + (size_t)c * HX_TOPK + lane), lane);
      s_lists[warp][lane] = best;
      __syncthreads();
      if (warp == 0) {
#pragma unroll
        for (uint32_t w = 1; w < HX_SCAN_THREADS / 32; ++w) best = hx_topk_merge32(best, s_lists[w][lane], lane);
        const uint32_t kk = (uint64_t)tk.k < n ? tk.k : (uint32_t)n;   // k' = min(k, |C|)
        const bool have = lane < kk && best != HX_KEY_MAX && a.q_status[q] == 0u;
        if (have) {
          const uint32_t rank = (uint32_t)(best & 0xffffffffu);
          const uint32_t* slots = a.q_slots ? a.q_slots[q] : a.cand_slots + base;
          tk.out_ids[(size_t)q * tk.k + lane] = ix.ids[slots[rank]];
          tk.out_scores[(size_t)q * tk.k + lane] = hx_key_score(best);
        }
        const uint32_t cnt = __popc(__ballot_sync(FULL, have));
        if (lane == 0) {
          tk.out_counts[q] = cnt;
          tk.tickets[q] = 0u;   // ready for the next launch
        }
      }
    }
    __syncthreads();
  }
}

// ---- top-k selection -----------------------------------------------------------------------------------
struct HxSelectArgs {
  const uint64_t* keys;
  const uint32_t* cand_slots;
  const uint64_t* cand_offsets;
  const uint32_t* q_status;
  uint32_t B, k;                 // k as requested; clamped to |C_q| per query (restricted.rs:200-213)
  uint32_t shared_set;           // 0: per-query CSR sets, 1: one shared set, 2: keys carry global slots (no indirection)
  uint64_t n_shared;
  uint64_t* out_ids;             // [B][k] (mode 2: the slot itself)
  float* out_scores;
  uint32_t* out_counts;
  const uint32_t* const* q_slots;  // device-resident candidate sets (see HxScanArgs)
  const uint64_t* q_len;
  const uint64_t* q_keyoff;
};

// bitonic sort of 2*HX_SEL_HALF keys in shared memory, ascending, by a block of THREADS threads
template <uint32_t THREADS>
__device__ __forceinline__ void hx_bitonic_sort_2048(uint64_t* s, uint32_t tid) {
  const uint32_t N = 2 * HX_SEL_HALF;
  for (uint32_t size = 2; size <= N; size <<= 1) {
    for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (uint32_t p = tid; p < N / 2; p += THREADS) {
        const uint32_t i = 2 * p - (p & (stride - 1));   // index of the lower element of the pair
        const uint32_t j = i + stride;
        const bool up = ((i & size) == 0);
        const uint64_t x = s[i], y = s[j];
        if ((x > y) == up) { s[i] = y; s[j] = x; }
      }
    }
  }
  __syncthreads();
}

// The kk (<= HX_SEL_HALF) smallest of keys[0, n) into buf[0, kk), ascending; buf[kk..] holds larger keys or HX_KEY_MAX.
// Threshold filter + bitonic merge in shared memory, run by the whole block (block-uniform call; buf = 2*HX_SEL_HALF
// keys).  The keys are read from L2 (__ldcg): the service kernel selects over keys other CTAs of the same launch wrote.
template <uint32_t THREADS>
__device__ __forceinline__ void hx_select_keys(const uint64_t* keys, uint64_t n, uint32_t kk, uint64_t* buf, uint32_t* s_cnt,
                                               uint64_t* s_thr, uint32_t tid) {
  for (uint32_t i = tid; i < 2 * HX_SEL_HALF; i += THREADS) buf[i] = HX_KEY_MAX;
  if (tid == 0) { *s_cnt = 0; *s_thr = HX_KEY_MAX; }
  __syncthreads();
  for (uint64_t b0 = 0; b0 < n; b0 += THREADS) {
    const uint64_t r = b0 + tid;
    if (r < n) {
      const uint64_t key = __ldcg(keys + r);
      if (key < *s_thr) {
        const uint32_t p = atomicAdd(s_cnt, 1u);
        buf[HX_SEL_HALF + p] = key;            // p < HX_SEL_HALF guaranteed by the flush rule below
      }
    }
    __syncthreads();
    const uint32_t filled = *s_cnt;   // snapshot between two barriers: no thread can bump s_cnt before all have read it
    __syncthreads();
    if (filled + THREADS > HX_SEL_HALF) {   // next step could overflow: merge now (block-uniform)
      hx_bitonic_sort_2048<THREADS>(buf, tid);
      for (uint32_t i = tid; i < HX_SEL_HALF; i += THREADS) buf[HX_SEL_HALF + i] = HX_KEY_MAX;
      if (tid == 0) { *s_cnt = 0; *s_thr = buf[kk - 1]; }   // HX_KEY_MAX until kk keys are known
      __syncthreads();
    }
  }
  hx_bitonic_sort_2048<THREADS>(buf, tid);
}

static __global__ void __launch_bounds__(HX_SEL_THREADS) k_select(HxDev ix, HxSelectArgs a) {
  __shared__ uint64_t buf[2 * HX_SEL_HALF];   // [0,1024): best so far (sorted), [1024,2048): incoming survivors
  __shared__ uint32_t s_cnt;
  __shared__ uint64_t s_thr;
  const uint32_t tid = threadIdx.x;
  for (uint32_t q = blockIdx.x; q < a.B; q += gridDim.x) {
    const uint64_t base = a.q_slots ? 0ull : (a.shared_set ? 0ull : a.cand_offsets[q]);
    const uint64_t n = a.q_slots ? a.q_len[q] : (a.shared_set ? a.n_shared : (a.cand_offsets[q + 1] - base));
    if (a.q_status[q] != 0u || n == 0) {
      if (tid == 0) a.out_counts[q] = 0;
      continue;
    }
    const uint64_t* keys = a.keys + (a.q_slots ? a.q_keyoff[q] : (a.shared_set ? (uint64_t)q * a.n_shared : base));
    const uint32_t kk = (uint64_t)a.k < n ? a.k : (uint32_t)n;   // k' = min(k, |C|)
    hx_select_keys<HX_SEL_THREADS>(keys, n, kk, buf, &s_cnt, &s_thr, tid);
    // count valid (absent candidates carry HX_KEY_MAX and are never results)
    const uint32_t* slots = a.q_slots ? a.q_slots[q] : a.cand_slots + base;
    uint32_t cnt = 0;
    for (uint32_t i = tid; i < kk; i += HX_SEL_THREADS) {
      const uint64_t key = buf[i];
      if (key != HX_KEY_MAX) {
        const uint32_t rank = (uint32_t)(key & 0xffffffffu);
        a.out_ids[(size_t)q * a.k + i] = a.shared_set == 2 ? (uint64_t)rank : ix.ids[slots[rank]];
        a.out_scores[(size_t)q * a.k + i] = hx_key_score(key);
        cnt++;
      }
    }
    // block reduce of cnt
    __shared__ uint32_t s_total;
    if (tid == 0) s_total = 0;
    __syncthreads();
    if (cnt) atomicAdd(&s_total, cnt);
    __syncthreads();
    if (tid == 0) a.out_counts[q] = s_total;
    __syncthreads();
  }
}

// ---- candidate id -> slot mapping (restricted.rs:615-659: ids without a vector row are skipped) ----------
__device__ __forceinline__ uint32_t hx_candidate_slot(const uint64_t* __restrict__ ids_sorted, uint32_t n, uint64_t id,
                                                      int contiguous, uint64_t first_id, const uint8_t* __restrict__ deleted) {
  uint32_t slot = HX_ABSENT;
  if (contiguous) {
    if (id >= first_id && id - first_id < (uint64_t)n) slot = (uint32_t)(id - first_id);
  } else {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
      const uint32_t mid = lo + ((hi - lo) >> 1);
      if (ids_sorted[mid] < id) lo = mid + 1; else hi = mid;
    }
    if (lo < n && ids_sorted[lo] == id) slot = lo;
  }
  if (deleted && slot != HX_ABSENT && deleted[slot]) slot = HX_ABSENT;   // hx_index_delete_vectors: the row is gone
  return slot;
}

static __global__ void k_map_candidates(const uint64_t* __restrict__ ids_sorted, uint32_t n, const uint64_t* __restrict__ cand,
                                 uint64_t n_cand, uint32_t* __restrict__ out_slots, int contiguous, uint64_t first_id,
                                 const uint8_t* __restrict__ deleted) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_cand) return;
  out_slots[i] = hx_candidate_slot(ids_sorted, n, cand[i], contiguous, first_id, deleted);
}

// ---- restricted query service: one launch per coalesced batch of one-query callers (hx_service_submit_restricted) ---------
// The grid is the batch's flattened work list: query q owns units [unit0[q], unit0[q+1]), one CTA per `chunk` candidates
// (chunk >= 256, so the reference's exact-plan shape |C| <= 256 is one CTA: no ticket, no partial list).  A CTA stages the
// query and its chunk's candidate slots in shared memory (list submissions: ids read from the pinned arena and mapped
// with hx_candidate_slot; device sets: slots as stored), scores every present row with the bit-exact octet kernel (one
// thread per row for Manhattan) and keys it score_bits<<32 | rank, exactly as k_scan does.
//   k <= 32: warp lists (hx_topk_insert / hx_topk_merge32) as in k_scan_topk; a query of several units merges the
//            per-CTA lists in its last CTA (self-resetting ticket).
//   k >  32: keys go to scratch; the query's last CTA selects with hx_select_keys (k_select's logic).
// The CTA that finishes a query writes ids / scores / count into the host-mapped result slot, __threadfence_system, then
// the slot's done word 0x80000000 | flags (the hx_query_done protocol).
#define HX_RSVC_MAX_BATCH 128       // queries per launch: the descriptor travels as the kernel parameter
#define HX_RSVC_CHUNK_MIN 256
#define HX_RSVC_CHUNK_MAX 2048

struct HxRsvcQuery {
  const void* cand;     // list: ascending uint64 ids; device set: uint32 slots (HX_ABSENT = no vector row)
  uint32_t n;           // |C| (> 0)
  uint32_t is_set;
};

struct HxRsvcArgs {
  const float* queries;          // [B][dim]  (the pinned ring itself or its device copy)
  const float* q_hdr;            // [B]
  const uint8_t* deleted;
  int contiguous;
  uint64_t first_id;
  uint32_t B, k, chunk;
  uint64_t* partial;             // [units][HX_TOPK]    (k <= 32)
  uint64_t* keys;                // [units * chunk]     (k > 32): query q's keys start at unit0[q] * chunk
  uint32_t* tickets;             // [B] zero; self-resetting
  uint32_t* qflags;              // [B] zero; self-resetting
  uint64_t* out_ids;             // [B][k]  host-mapped result slots
  float* out_scores;             // [B][k]
  uint32_t* out_counts;          // [B]
  uint32_t* done;                // [B]
  uint32_t unit0[HX_RSVC_MAX_BATCH + 1];
  HxRsvcQuery q[HX_RSVC_MAX_BATCH];
};

template <int METRIC, bool BIGK>
static __global__ void __launch_bounds__(HX_SCAN_THREADS, 4) k_scan_service(HxDev ix, const __grid_constant__ HxRsvcArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  float* sq = reinterpret_cast<float*>(smem);
  __shared__ uint32_t s_slots[HX_RSVC_CHUNK_MAX];
  __shared__ uint64_t s_lists[HX_SCAN_THREADS / 32][HX_TOPK];
  __shared__ uint64_t s_buf[BIGK ? 2 * HX_SEL_HALF : 1];
  __shared__ uint64_t s_thr;
  __shared__ uint32_t s_cnt, s_last, s_flags;
  const uint32_t tid = threadIdx.x, t = tid & 7u, oct = tid >> 3, lane = tid & 31u, warp = tid >> 5;
  const unsigned FULL = 0xffffffffu;
  const uint32_t unit = blockIdx.x;
  // the owning query: the last q with unit0[q] <= unit (a query without units shares unit0 with its successor)
  uint32_t q = 0, hi = a.B;
  while (hi - q > 1) {
    const uint32_t mid = (q + hi) >> 1;
    if (a.unit0[mid] <= unit) q = mid; else hi = mid;
  }
  const HxRsvcQuery Q = a.q[q];
  const uint32_t n = Q.n, first = a.unit0[q], nunits = a.unit0[q + 1] - first;
  const uint32_t start = (unit - first) * a.chunk, end = min(start + a.chunk, n);
  for (uint32_t i = tid; i < ix.ld; i += HX_SCAN_THREADS) sq[i] = i < ix.dim ? a.queries[(size_t)q * ix.dim + i] : 0.0f;
  for (uint32_t r = start + tid; r < end; r += HX_SCAN_THREADS)
    s_slots[r - start] = Q.is_set ? static_cast<const uint32_t*>(Q.cand)[r]
                                  : hx_candidate_slot(ix.ids, ix.n, static_cast<const uint64_t*>(Q.cand)[r], a.contiguous,
                                                      a.first_id, a.deleted);
  if (tid == 0) s_flags = 0u;
  const float q_hdr = a.q_hdr[q];
  __syncthreads();
  // scan: octets own rows (4 per warp per step), Manhattan one row per thread (32 per warp per step)
  const uint32_t step = METRIC == HXM_MANHATTAN ? HX_SCAN_THREADS : HX_SCAN_THREADS / 8;
  uint64_t mine = HX_KEY_MAX;
  uint32_t flags = 0u;
  for (uint32_t r0 = start; r0 < end; r0 += step) {
    const uint32_t r = r0 + (METRIC == HXM_MANHATTAN ? tid : oct);
    uint64_t key = HX_KEY_MAX;
    if (r < end) {
      const uint32_t slot = s_slots[r - start];
      if (slot != HX_ABSENT) {
        float s;
        if (METRIC == HXM_MANHATTAN) s = hx_manhattan_seq(ix.vec + (size_t)slot * ix.ld, sq, ix.dim);
        else s = hx_octet_score<METRIC>(ix, sq, q_hdr, slot, t);
        if (!hx_score_ok(s)) flags |= HXF_INVALID_SCORE;
        key = hx_make_key(s, r);
      }
    }
    if (BIGK) {
      if (r < end && (METRIC == HXM_MANHATTAN || t == 0)) a.keys[(size_t)first * a.chunk + r] = key;
    } else {
      uint64_t kth = __shfl_sync(FULL, mine, HX_TOPK - 1);
      constexpr int PER_WARP = METRIC == HXM_MANHATTAN ? 32 : 4;
#pragma unroll 4
      for (int o = 0; o < PER_WARP; ++o) {
        const uint64_t c = __shfl_sync(FULL, key, METRIC == HXM_MANHATTAN ? o : o * 8);
        if (c < kth) {   // warp-uniform branch (c and kth are broadcasts)
          hx_topk_insert(mine, c, lane);
          kth = __shfl_sync(FULL, mine, HX_TOPK - 1);
        }
      }
    }
  }
  if (flags) atomicOr(&s_flags, flags);
  if (!BIGK) s_lists[warp][lane] = mine;
  __syncthreads();
  if (!BIGK && warp == 0) {
#pragma unroll
    for (uint32_t w = 1; w < HX_SCAN_THREADS / 32; ++w) mine = hx_topk_merge32(mine, s_lists[w][lane], lane);
  }
  uint32_t qf = s_flags;
  if (nunits > 1) {   // publish this CTA's part; the last CTA of the query finishes it
    if (!BIGK && warp == 0) a.partial[(size_t)unit * HX_TOPK + lane] = mine;
    if (tid == 0 && qf) atomicOr(a.qflags + q, qf);
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(a.tickets + q, 1u) == nunits - 1u ? 1u : 0u;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    qf = __ldcg(a.qflags + q);
    if (!BIGK) {   // warp w merges units w, w + 8, ... of the query
      uint64_t best = HX_KEY_MAX;
      for (uint32_t u = first + warp; u < first + nunits; u += HX_SCAN_THREADS / 32)
        best = hx_topk_merge32(best, __ldcg(a.partial + (size_t)u * HX_TOPK + lane), lane);
      s_lists[warp][lane] = best;
      __syncthreads();
      if (warp == 0) {
        mine = best;
#pragma unroll
        for (uint32_t w = 1; w < HX_SCAN_THREADS / 32; ++w) mine = hx_topk_merge32(mine, s_lists[w][lane], lane);
      }
    }
    __syncthreads();
    if (tid == 0) { a.tickets[q] = 0u; a.qflags[q] = 0u; }   // ready for the next launch on this scratch
  }
  const uint32_t kk = a.k < n ? a.k : n;   // k' = min(k, |C|)
  uint32_t cnt = 0;
  auto result_id = [&](uint32_t rank) -> uint64_t {
    return Q.is_set ? ix.ids[static_cast<const uint32_t*>(Q.cand)[rank]] : static_cast<const uint64_t*>(Q.cand)[rank];
  };
  if (!BIGK) {
    if (warp != 0) return;
    const bool have = lane < kk && mine != HX_KEY_MAX;
    if (have) {
      a.out_ids[(size_t)q * a.k + lane] = result_id((uint32_t)(mine & 0xffffffffu));
      a.out_scores[(size_t)q * a.k + lane] = hx_key_score(mine);
    }
    cnt = __popc(__ballot_sync(FULL, have));
    __threadfence_system();   // results before the done word
    __syncwarp();
    if (lane == 0) {
      a.out_counts[q] = cnt;
      __threadfence_system();
      *((volatile uint32_t*)a.done + q) = 0x80000000u | qf;
    }
    return;
  }
  hx_select_keys<HX_SCAN_THREADS>(a.keys + (size_t)first * a.chunk, n, kk, s_buf, &s_cnt, &s_thr, tid);
  for (uint32_t i = tid; i < kk; i += HX_SCAN_THREADS) {
    const uint64_t key = s_buf[i];
    if (key != HX_KEY_MAX) {
      a.out_ids[(size_t)q * a.k + i] = result_id((uint32_t)(key & 0xffffffffu));
      a.out_scores[(size_t)q * a.k + i] = hx_key_score(key);
      cnt++;
    }
  }
  if (tid == 0) s_cnt = 0u;
  __syncthreads();
  if (cnt) atomicAdd(&s_cnt, cnt);
  __threadfence_system();
  __syncthreads();
  if (tid == 0) {
    a.out_counts[q] = s_cnt;
    __threadfence_system();
    *((volatile uint32_t*)a.done + q) = 0x80000000u | qf;
  }
}
