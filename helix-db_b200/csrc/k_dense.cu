// k_dense.cu — tensor-core batched distance path (configs C4/C5): exhaustive top-k of B queries against every row.
//
// The only place on this hot path where the work is a dense contraction: S[b][i] = <q_b, x_i> for B = 1024..4096
// queries against the whole shard is a (B x d) x (d x N) GEMM with arithmetic intensity ~B flop/byte, far beyond the
// HBM ridge.  It runs on the Hopper tensor cores (sm_90a):
//   * operands in bf16 (a bf16 copy of the corpus is kept when hx_index_config.storage == 1), fp32 accumulation in the
//     registers of the issuing warpgroup;
//   * one persistent CTA per SM.  A producer warp streams (128 queries | 128 corpus rows) x 64-element k-blocks with TMA
//     (128-byte swizzle) into a 4-stage shared-memory ring whose slots are handed over by mbarriers (full: bytes landed,
//     empty: the MMAs that read the slot have completed).  Two consumer warpgroups each issue wgmma.m64n128k16 for 64 of
//     the 128 queries with both operands read straight from shared memory, keeping one wgmma group in flight while the
//     next slot is waited for;
//   * fused epilogue: the accumulators of each 128 x 128 half tile are written to shared memory (row stride 129 floats, so
//     the column-order reads below are free of bank conflicts); each of the 256 consumer threads — one query row x one
//     64-column quarter — turns them into the metric's score order with the stored row norms and keeps the HXD_T best rows
//     per (query, run of tiles, column quarter) by register insertion, emitting score_bits<<32|row keys — the B x N
//     score matrix is never written.  Per half tile the epilogue is 64 columns per thread against the 4 x ldb/64 wgmma
//     steps of the contraction, so it runs between the MMAs of consecutive half tiles instead of beside them.
// The approximate (bf16) keys only NOMINATE candidates: k_select keeps the k' best keys per query and the exact fp32
// scan kernel (bit-exact reference arithmetic) re-ranks them, so returned scores are exact and ordering follows the
// reference's (score, id) rule; recall vs the exhaustive exact scan is measured, not assumed.
//
// Reference behaviour this stands in for: the same answer VectorIndex::search_restricted gives with every id as a
// candidate (restricted_exact_scan, search/vector/restricted.rs:753-835), i.e. exact brute-force top-k.
#include <cuda.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "hx_index.hpp"
#include "k_scan.cuh"
#include "k_util.cuh"

#define HXD_BM 128          // queries per CTA tile: two consumer warpgroups x 64 (wgmma M)
#define HXD_BN 256          // corpus rows per placement tile (the unit of the row interleave and of the column quarters)
#define HXD_BH 128          // corpus rows per MMA tile (wgmma N): a placement tile is contracted in two halves
#define HXD_BK 64           // bf16 elements per k-block = 128 bytes = one swizzle atom
#define HXD_STAGES 4
#define HXD_PARTS 4         // 64-column quarters of a placement tile: one bucket of the fused top-T per (query, run, quarter)
#ifndef HXD_T
#define HXD_T 8             // best rows kept per (query, run of n-tiles, column quarter): 32 per (query, run)
#endif
// Row placement inside a 256-row corpus tile.  A bucket of the fused top-T is (query, run of tiles, 64-COLUMN quarter) and keeps
// HXD_T rows.  With rows placed in id order a quarter is 64 CONSECUTIVE ids, so a query whose true neighbours are consecutive
// ids (near-duplicate rows inserted back to back: chunks of one document) could have more than HXD_T of them in one bucket and
// lose the rest.  HXD_INTERLEAVE = 1 stores row j of a tile at position (j % 4) * 64 + j / 4: consecutive ids land in different
// quarters (a run of 32 consecutive ids puts at most 8 into any bucket), at no cost to the kernel (same loads, same MMAs; only
// the slot a column stands for changes).  tests/test_gpu_zz_reference_contracts.py::test_dense_path_keeps_id_clustered_neighbours
// is the fixture on which id order loses neighbours.  Default on.
#ifndef HXD_INTERLEAVE
#define HXD_INTERLEAVE 1
#endif
// position of tile row j / tile row held at position c (inverse of each other)
__host__ __device__ __forceinline__ uint32_t hxd_pos_of_row(uint32_t j) {
#if HXD_INTERLEAVE
  return (j & 3u) * (HXD_BN / HXD_PARTS) + (j >> 2);
#else
  return j;
#endif
}
__host__ __device__ __forceinline__ uint32_t hxd_row_at_pos(uint32_t c) {
#if HXD_INTERLEAVE
  return (c & (HXD_BN / HXD_PARTS - 1u)) * HXD_PARTS + c / (HXD_BN / HXD_PARTS);
#else
  return c;
#endif
}
#define HXD_CONSUMERS 256   // warps 0-7: two consumer warpgroups (MMA + epilogue); warp 8: TMA producer
#define HXD_THREADS (HXD_CONSUMERS + 32)
#define HXD_A_BYTES (HXD_BM * HXD_BK * 2)
#define HXD_B_BYTES (HXD_BH * HXD_BK * 2)
#define HXD_STAGE_BYTES (HXD_A_BYTES + HXD_B_BYTES)
#define HXD_ACC_LD (HXD_BH + 1)   // floats per row of the accumulator tile in shared memory

// ---- PTX wrappers ------------------------------------------------------------------------------------------------------
// tile -> shared memory; the bytes are counted on `bar`
__device__ __forceinline__ void hxd_tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          hx_smem_u32(smem_dst)),
      "l"(map), "r"(hx_smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void hxd_prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void hxd_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void hxd_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void hxd_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// ties the accumulator registers to the surrounding asm so that no read of them moves across a wgmma wait
__device__ __forceinline__ void hxd_fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, bf16 operands from shared memory (both K-major), fp32 accumulate in registers.
// Thread layout of D (warp w of the warpgroup, lane l): d[4j + 2h + e] = D[16w + l/4 + 8h][8j + 2(l%4) + e].
__device__ __forceinline__ void hxd_wgmma(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// K-major operand tile stored by TMA with the 128-byte swizzle: rows of 128 bytes, 8-row groups 1024 bytes apart.
// wgmma matrix descriptor: start>>4 [0,14) | LBO>>4 [16,30) = 1 (unused for swizzled K-major) | SBO>>4 [32,46) = 64 |
// base offset [49,52) = 0 (tiles are 1024-byte aligned) | layout [62,64) = 1 (SWIZZLE_128B).
__device__ __forceinline__ uint64_t hxd_make_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3fffu);
  d |= (uint64_t)1u << 16;
  d |= (uint64_t)64u << 32;
  d |= (uint64_t)1u << 62;
  return d;
}

struct HxDenseArgs {
  uint32_t n_rows;            // rows of the bf16 copy = live corpus rows (unpadded)
  uint32_t n_queries;         // B (unpadded)
  uint32_t k_blocks;          // ldb / 64
  uint32_t m_tiles, n_tiles;  // 128-query tiles, 256-row corpus tiles
  uint32_t n_split;           // work unit u: query tile u % m_tiles, n-tiles [r*n_tiles/n_split, (r+1)*n_tiles/n_split), r = u / m_tiles
  const float* row_aux;       // cosine: 1/|x_i|   ; euclidean: |x_i|^2            (from the bf16-rounded rows)
  const float* q_aux;         // cosine: 1/|q_b|   ; euclidean: |q_b|^2
  uint64_t* keys;             // [B][n_split][HXD_PARTS][HXD_T]
  int32_t metric;
};

// insert (t, slot) into a descending best-T list (ties keep the earlier column)
__device__ __forceinline__ void hxd_insert(float (&bt)[HXD_T], uint32_t (&bs)[HXD_T], float t, uint32_t slot) {
  bt[HXD_T - 1] = t;
  bs[HXD_T - 1] = slot;
#pragma unroll
  for (int j = HXD_T - 1; j > 0; --j)
    if (bt[j] > bt[j - 1]) {
      const float tf = bt[j]; bt[j] = bt[j - 1]; bt[j - 1] = tf;
      const uint32_t tsl = bs[j]; bs[j] = bs[j - 1]; bs[j - 1] = tsl;
    }
}

__global__ void __launch_bounds__(HXD_THREADS, 1)
k_dense_scores(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_x, HxDenseArgs a) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  // HXD_STAGES x (A 16 KB | B 16 KB); the 128-byte swizzle needs 1024-byte aligned tiles: align inside the window
  unsigned char* smem = smem_raw + ((1024u - (hx_smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* tiles = smem;
  float* accs = reinterpret_cast<float*>(smem + HXD_STAGES * HXD_STAGE_BYTES);   // [HXD_BM][HXD_ACC_LD] accumulators of a half tile
  float* ax = accs + HXD_BM * HXD_ACC_LD;                                         // [HXD_BH] row terms of that half tile
  uint64_t* full = reinterpret_cast<uint64_t*>(ax + HXD_BH);                      // [HXD_STAGES] slot filled (TMA bytes landed)
  uint64_t* empty = full + HXD_STAGES;                                            // [HXD_STAGES] slot read by every consumer warp

  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  if (threadIdx.x == 0) {
    hxd_prefetch_tmap(&map_q);
    hxd_prefetch_tmap(&map_x);
    for (int s = 0; s < HXD_STAGES; ++s) {
      hx_mbar_init(full + s, 1);                       // the producer's arrive.expect_tx
      hx_mbar_init(empty + s, HXD_CONSUMERS / 32);     // one arrive per consumer warp
    }
    hx_fence_mbar_init();
  }
  __syncthreads();
  const uint32_t total_units = a.m_tiles * a.n_split;

  if (warp == HXD_CONSUMERS / 32) {
    // ===== TMA producer (one lane) =====
    if (lane == 0) {
      uint32_t stage = 0, ph = 0;
      for (uint32_t u = blockIdx.x; u < total_units; u += gridDim.x) {
        // units with the same n-range and different query tiles run on neighbouring CTAs in step: the corpus tile is
        // read from HBM once and served to the others by L2
        const uint32_t mt = u % a.m_tiles, r = u / a.m_tiles;
        const uint32_t nt0 = (uint32_t)((uint64_t)r * a.n_tiles / a.n_split), nt1 = (uint32_t)((uint64_t)(r + 1) * a.n_tiles / a.n_split);
        for (uint32_t nt = nt0; nt < nt1; ++nt)
          for (uint32_t h = 0; h < HXD_BN / HXD_BH; ++h)
            for (uint32_t kb = 0; kb < a.k_blocks; ++kb) {
              hx_mbar_wait(empty + stage, ph ^ 1u);
              unsigned char* sa = tiles + (size_t)stage * HXD_STAGE_BYTES;
              hx_mbar_expect_tx(full + stage, HXD_STAGE_BYTES);
              hxd_tma_load_2d(sa, &map_q, full + stage, (int)(kb * HXD_BK), (int)(mt * HXD_BM));
              hxd_tma_load_2d(sa + HXD_A_BYTES, &map_x, full + stage, (int)(kb * HXD_BK), (int)(nt * HXD_BN + h * HXD_BH));
              if (++stage == HXD_STAGES) { stage = 0; ph ^= 1u; }
            }
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg issues the MMAs of queries 64*wg .. 64*wg+63; all 256 threads run the epilogue =====
  const uint32_t wg = warp >> 2;
  const uint32_t erow = threadIdx.x & (HXD_BM - 1u);   // epilogue: query row of the tile ...
  const uint32_t eq = threadIdx.x / HXD_BM;            // ... and 64-column quarter within the half tile
  uint32_t stage = 0, ph = 0;
  for (uint32_t u = blockIdx.x; u < total_units; u += gridDim.x) {
    const uint32_t mt = u % a.m_tiles, r = u / a.m_tiles;
    const uint32_t nt0 = (uint32_t)((uint64_t)r * a.n_tiles / a.n_split), nt1 = (uint32_t)((uint64_t)(r + 1) * a.n_tiles / a.n_split);
    const uint32_t qrow = mt * HXD_BM + erow;
    const float qa = qrow < a.n_queries ? a.q_aux[qrow] : 0.f;
    // running best-T (largest t) of this query over the run, for quarter eq (first half) and quarter 2 + eq (second half);
    // t = s*ax (cosine) or 2s - ax (euclidean)
    float bt0[HXD_T], bt1[HXD_T];
    uint32_t bs0[HXD_T], bs1[HXD_T];
#pragma unroll
    for (int i = 0; i < HXD_T; ++i) {
      bt0[i] = bt1[i] = -__int_as_float(0x7f800000);
      bs0[i] = bs1[i] = HX_ABSENT;
    }
    for (uint32_t nt = nt0; nt < nt1; ++nt) {
      const uint32_t n0 = nt * HXD_BN;
      for (uint32_t h = 0; h < HXD_BN / HXD_BH; ++h) {
        float d[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] = 0.f;
        uint32_t prev = 0;
        for (uint32_t kb = 0; kb < a.k_blocks; ++kb) {
          hx_mbar_wait(full + stage, ph);
          const uint32_t sa = hx_smem_u32(tiles + (size_t)stage * HXD_STAGE_BYTES);
          const uint64_t adesc = hxd_make_desc(sa + wg * (HXD_A_BYTES / 2)), bdesc = hxd_make_desc(sa + HXD_A_BYTES);
          hxd_wgmma_fence();
#pragma unroll
          for (uint32_t k = 0; k < HXD_BK / 16; ++k)   // 16 bf16 = 32 bytes along K inside the swizzle atom: start address += 2
            hxd_wgmma(d, adesc + 2ull * k, bdesc + 2ull * k, (kb | k) ? 1u : 0u);
          hxd_wgmma_commit();
          hxd_wgmma_wait<1>();                       // the group of k-block kb-1 has completed: its slot is free
          if (kb > 0 && lane == 0) hx_mbar_arrive(empty + prev);
          prev = stage;
          if (++stage == HXD_STAGES) { stage = 0; ph ^= 1u; }
        }
        hxd_wgmma_wait<0>();
        hxd_fence_acc(d);
        if (lane == 0) hx_mbar_arrive(empty + prev);
        {   // accumulators -> shared memory (layout of hxd_wgmma), row terms of the half tile
          float* p0 = accs + (64u * wg + 16u * (warp & 3u) + (lane >> 2)) * HXD_ACC_LD + 2u * (lane & 3u);
          float* p1 = p0 + 8 * HXD_ACC_LD;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            p0[8 * j] = d[4 * j]; p0[8 * j + 1] = d[4 * j + 1];
            p1[8 * j] = d[4 * j + 2]; p1[8 * j + 1] = d[4 * j + 3];
          }
          const uint32_t c = threadIdx.x;
          if (c < HXD_BH) {
            const uint32_t pos = h * HXD_BH + c;
            const bool live = n0 + hxd_row_at_pos(pos) < a.n_rows;   // row_aux is indexed by POSITION, the bound is on the row there
            float v = live ? a.row_aux[n0 + pos] : 0.f;
            if (!live) v = a.metric == HXM_COSINE ? -__int_as_float(0x7f800000) : __int_as_float(0x7f800000);
            ax[c] = v;                                  // padded rows: t = NaN / -inf never beats the threshold
          }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        {
          const uint32_t part = h * (HXD_BH / 64) + eq;   // column quarter of the placement tile
          const float* rowp = accs + erow * HXD_ACC_LD + eq * 64u;
          const float* axp = ax + eq * 64u;
          // one instance of the insertion network per bucket: the loop is kept rolled (instruction cache)
          auto scan = [&](float (&bt)[HXD_T], uint32_t (&bs)[HXD_T]) {
#pragma unroll 4
            for (uint32_t c = 0; c < 64; ++c) {
              const float s = rowp[c], x = axp[c];
              const float t = a.metric == HXM_COSINE ? s * x : fmaf(2.0f, s, -x);
              if (t > bt[HXD_T - 1]) hxd_insert(bt, bs, t, n0 + hxd_row_at_pos(part * 64u + c));
            }
          };
          if (h == 0) scan(bt0, bs0);
          else scan(bt1, bs1);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");   // the accumulator tile is free for the next half
      }
    }
    if (qrow < a.n_queries) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const uint32_t part = hh * (HXD_BH / 64) + eq;
        uint64_t* out = a.keys + (((size_t)qrow * a.n_split + r) * HXD_PARTS + part) * HXD_T;
#pragma unroll
        for (int i = 0; i < HXD_T; ++i) {
          const float t = hh ? bt1[i] : bt0[i];
          const uint32_t s = hh ? bs1[i] : bs0[i];
          uint64_t key = HX_KEY_MAX;
          if (s != HX_ABSENT) {
            float sc = a.metric == HXM_COSINE ? 0.5f - 0.5f * t * qa : qa - t;   // (1-cos)/2 ; |q|^2 + |x|^2 - 2<q,x>
            sc = fmaxf(sc, 0.0f);
            key = hx_make_key(sc, s);
          }
          out[i] = key;
        }
      }
    }
  }
}

// f32 rows -> bf16 rows (round to nearest even) with zero padding to ldb, plus the per-row aux term computed from the
// ROUNDED values (so that approximate scores are self-consistent)
// `tiled`: the corpus copy — row w goes to its tile position (hxd_pos_of_row); queries keep their order
// `src_rows`: row w of the copy is source row src_rows[w] (the live slots: deleted rows are left out); nullptr = row w
// Cosine is scale-free, and cosine vectors have no component limit: before rounding, each row / query is multiplied by the
// power of two that brings its largest |component| into [1, 2) (exact).  Without it a norm of ~1e19 or more makes the fp32
// sum of squares inf, one of ~1e-29 or less makes it 0 (the row term 0: every approximate score 0.5), and FLT_MAX rounds to
// a bf16 inf.  Euclidean rows keep their scale: the score is not scale-free, and every legal row fits (component limit).
__global__ void k_to_bf16(const float* __restrict__ src, size_t rows, uint32_t dim, size_t ld_src, __nv_bfloat16* __restrict__ dst,
                          uint32_t ldb, float* __restrict__ aux, int metric, int tiled, const uint32_t* __restrict__ src_rows) {
  const size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31u;
  if (w >= rows) return;
  const size_t pos = tiled ? (w / HXD_BN) * HXD_BN + hxd_pos_of_row((uint32_t)(w % HXD_BN)) : w;
  const float* s = src + (src_rows ? (size_t)src_rows[w] : w) * ld_src;
  __nv_bfloat16* d = dst + pos * (size_t)ldb;
  int shift = 0;
  if (metric == HXM_COSINE) {
    float mx = 0.f;
    for (uint32_t j = lane; j < dim; j += 32) mx = fmaxf(mx, fabsf(s[j]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 16)); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 8));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 4));  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    if (mx > 0.f) {
      int e;
      frexpf(mx, &e);   // mx = m * 2^e, m in [0.5, 1): mx * 2^(1-e) is in [1, 2)
      shift = 1 - e;
    }
  }
  float ss = 0.f;
  for (uint32_t j = lane; j < ldb; j += 32) {
    const float x = j < dim ? ldexpf(s[j], shift) : 0.f;
    const __nv_bfloat16 b = __float2bfloat16_rn(x);
    d[j] = b;
    const float xb = __bfloat162float(b);
    ss += xb * xb;
  }
  ss += __shfl_xor_sync(0xffffffffu, ss, 16); ss += __shfl_xor_sync(0xffffffffu, ss, 8);
  ss += __shfl_xor_sync(0xffffffffu, ss, 4);  ss += __shfl_xor_sync(0xffffffffu, ss, 2);
  ss += __shfl_xor_sync(0xffffffffu, ss, 1);
  if (lane == 0) aux[pos] = metric == HXM_COSINE ? (ss > 0.f ? rsqrtf(ss) : 0.f) : ss;
}

// The k' nominees of a query (rows of the bf16 copy in the low word, in approximate-score order; HX_ABSENT = unfilled) ->
// its candidate slot list for the exact re-rank, ASCENDING.  k_scan keys a candidate by its position in this list, so
// ascending slots make exact ties resolve by id — the reference's (score, id) rule — in order and in which tied rows
// make the cut, instead of by their bf16 scores.  One CTA per query sorts `width` (a power of two >= k') entries.
#define HXD_SORT_THREADS 256
#define HXD_SORT_MAX 1024
__global__ void __launch_bounds__(HXD_SORT_THREADS) k_nominee_slots(const uint64_t* __restrict__ sel, size_t B, uint32_t kprime,
                                                                   uint32_t width, const uint32_t* __restrict__ live_slots,
                                                                   uint32_t* __restrict__ out) {
  __shared__ uint32_t s[HXD_SORT_MAX];
  for (size_t q = blockIdx.x; q < B; q += gridDim.x) {
    for (uint32_t i = threadIdx.x; i < width; i += HXD_SORT_THREADS) {
      uint32_t v = HX_ABSENT;
      if (i < kprime) {
        const uint32_t w = (uint32_t)sel[q * kprime + i];
        if (w != HX_ABSENT) v = live_slots[w];
      }
      s[i] = v;
    }
    for (uint32_t size = 2; size <= width; size <<= 1)
      for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
        __syncthreads();
        for (uint32_t p = threadIdx.x; p < width / 2; p += HXD_SORT_THREADS) {
          const uint32_t i = 2 * p - (p & (stride - 1)), j = i + stride;
          const bool up = (i & size) == 0;
          const uint32_t x = s[i], y = s[j];
          if ((x > y) == up) { s[i] = y; s[j] = x; }
        }
      }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < kprime; i += HXD_SORT_THREADS) out[q * kprime + i] = s[i];
    __syncthreads();
  }
}

// ---- order-preserving compaction of a candidate slot list (hx_search_dense_restricted) ----------------------------------------
// Drops the HX_ABSENT entries (ids without a row, deleted rows) of an ascending slot list and keeps the rest in order, so
// that the gathered tile holds present rows only: an absent row left in the tile would take a column and bucket space and
// could leave the count short of min(k, present).  Two launches: per-tile counts, then each tile sums the counts before it
// and scatters.  Tile = HXD_CPT_ROWS rows of 256 slots; row r of a tile is slots [256 r, 256 r + 256), one per thread, so
// the loads are coalesced and a present slot's rank is (rank of its warp within the row, ballot prefix within the warp).
#define HXD_CPT_THREADS 256
#define HXD_CPT_ROWS 16
#define HXD_CPT_TILE (HXD_CPT_THREADS * HXD_CPT_ROWS)

__global__ void __launch_bounds__(HXD_CPT_THREADS) k_compact_count(const uint32_t* __restrict__ slots, size_t n,
                                                                  uint32_t* __restrict__ tile_counts) {
  __shared__ uint32_t ws[HXD_CPT_THREADS / 32];
  const size_t t0 = (size_t)blockIdx.x * HXD_CPT_TILE;
  uint32_t c = 0;
#pragma unroll
  for (int r = 0; r < HXD_CPT_ROWS; ++r) {
    const size_t i = t0 + (size_t)r * HXD_CPT_THREADS + threadIdx.x;
    c += i < n && slots[i] != HX_ABSENT;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31u) == 0) ws[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t s = 0;
    for (int w = 0; w < HXD_CPT_THREADS / 32; ++w) s += ws[w];
    tile_counts[blockIdx.x] = s;
  }
}

__global__ void __launch_bounds__(HXD_CPT_THREADS) k_compact_scatter(const uint32_t* __restrict__ slots, size_t n,
                                                                    const uint32_t* __restrict__ tile_counts,
                                                                    uint32_t* __restrict__ out, uint32_t* __restrict__ out_count) {
  __shared__ uint32_t ws[HXD_CPT_THREADS / 32];
  __shared__ uint32_t off[HXD_CPT_ROWS * (HXD_CPT_THREADS / 32)];   // output offsets of the (row, warp) groups, in that order
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const size_t t0 = (size_t)blockIdx.x * HXD_CPT_TILE;
  // present slots of the tiles before this one
  uint32_t base = 0;
  for (uint32_t t = threadIdx.x; t < blockIdx.x; t += HXD_CPT_THREADS) base += tile_counts[t];
  base = __reduce_add_sync(0xffffffffu, base);
  if (lane == 0) ws[warp] = base;
  uint32_t v[HXD_CPT_ROWS], mask[HXD_CPT_ROWS];
#pragma unroll
  for (int r = 0; r < HXD_CPT_ROWS; ++r) {
    const size_t i = t0 + (size_t)r * HXD_CPT_THREADS + threadIdx.x;
    v[r] = i < n ? slots[i] : HX_ABSENT;
    mask[r] = __ballot_sync(0xffffffffu, v[r] != HX_ABSENT);
    if (lane == 0) off[r * (HXD_CPT_THREADS / 32) + warp] = __popc(mask[r]);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t s = 0;
    for (int w = 0; w < HXD_CPT_THREADS / 32; ++w) s += ws[w];
    for (int j = 0; j < HXD_CPT_ROWS * (HXD_CPT_THREADS / 32); ++j) {
      const uint32_t c = off[j];
      off[j] = s;
      s += c;
    }
    if (blockIdx.x == gridDim.x - 1) *out_count = s;
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < HXD_CPT_ROWS; ++r)
    if (v[r] != HX_ABSENT) out[off[r * (HXD_CPT_THREADS / 32) + warp] + __popc(mask[r] & ((1u << lane) - 1u))] = v[r];
}

// ---- the certificate of the exact entries (hx_search_dense_exact, hx_search_dense_restricted_exact[_set]) ------------------
// After the re-rank, query q's answer is exact unless a row the pass dropped belongs in it.  A dropped row r has approximate
// score ŝ_r (a key of k_dense_scores) >= L_q, the smaller of
//   * the tail (key HXD_T - 1) of every FULL bucket (tail != HX_KEY_MAX): a bucket keeps the HXD_T largest t and sc is
//     monotone (non-increasing) in t, fmaxf clamp included, so every row it dropped has ŝ >= its tail;
//   * the k'-th nominee's approximate score, when the first k_select kept k' keys (otherwise it dropped none).
// With S_k the k-th exact score of the answer (the reference's fp32 bits), the query is certified iff
//   floor(L_q) > S_k,   floor(L) = a lower bound on the reference's fp32 score of ANY row of the view with ŝ >= L,
// i.e. L_q > S_k + E_q with E_q = L_q - floor(L_q).  floor is non-decreasing in L, so bounding at ŝ = L_q covers every
// dropped row: each has exact score > S_k, so it is neither better than the k-th row nor tied with it.
//
// The bound (hxd_exact_floor; tests/test_dense_exact_reference.py restates it and checks it against the oracle).  Notation:
// u = 2^-24 (fp32), u_b = 2^-8 (bf16: 8 significant bits), γ(n) = n u / (1 - n u), ldb = dim rounded up to 64.  q^, x^ are
// the bf16 operands; Q = |q^|, X = |x^|.  Three error sources:
//  (a) the pass's own fp32 arithmetic.  Tensor-core accumulation is not IEEE-specified; it is bounded as if every one of
//      the ldb additions truncated (2^-23) and flushed anything below 2^-126 (inputs included):
//        |s - <q^,x^>| <= c_acc Σ|q^_i x^_i| + 2 (ldb + 16) 2^-126 + 2^-126 Σ(|q^_i| + |x^_i|),  c_acc = (ldb + 16) 2^-22.
//      The row / query terms are fp32 sums of exact bf16 squares, depth ldb/32 + 5: |qa - Q^2| <= γ_sq Q^2 + ldb 2^-150.
//      Euclidean, sc = qa - fma(2, s, -ax) (two roundings, |operands| <= M = (Q + X)^2):
//        |sc - |q^ - x^|^2| <= (γ_sq + c_acc + 3u) M + 2 ldb 2^-150 + 2 a_acc + 2^-150.
//      Cosine, sc = 0.5 - 0.5 (s ax) qa with ax, qa = rsqrtf (2 ulp = 4u) of the sums; after k_to_bf16's power-of-two step
//      every nonzero operand has its largest component in [1, 2), so Q, X >= 1 and every absolute term is relative:
//        |sc - (1 - cos^)/2| <= 0.5 (c_acc + 1.01 Ψ) + 1.6u + 2^-100,  Ψ = 1.01 (2 ψ + u),  ψ = 1.01 (γ_sq + ldb 2^-150 + 4u).
//      sc >= that error below the true value is all that is used: the clamp only raises ŝ, and the true value is >= 0.
//  (b) bf16 rounding, in the distance domain, where it is a contraction.  |x^_i - x_i| <= u_b |x_i| + 2^-134 (bf16
//      subnormal spacing 2^-133), so |x^ - x| <= u_b |x| + a, a = sqrt(ldb) 2^-134, and |x| <= (X + a) / (1 - u_b).
//      Euclidean: D = |q - x| >= |q^ - x^| - |q^ - q| - |x^ - x| >= sqrt(ŝ - err) - β,
//        β = u_b (Q + R + 2a) / (1 - u_b) + 2a,  R = an upper bound on X over the view (max of the row terms).
//      Cosine: the score is |e_q - e_x|^2 / 4 over unit vectors e.  Scaling by 2^j changes no direction; rounding a vector
//      w with |w^ - w| <= η |w| (η = u_b + sqrt(ldb) 2^-133, ldexpf's own rounding included) turns its direction by an
//      angle whose chord is <= η' = 1.01 η / (1 - η).  So sqrt(score) >= sqrt(ŝ - err) - η'.  No norms enter.
//  (c) the reference's fp32 score of the dropped row, since S_k is the reference's bits.  Euclidean: every term (q_i - x_i)^2
//      is positive and sees at most 2 dim + 10 roundings (subtraction, fma chain, tree, scalar tail) plus at most that many
//      underflows of 2^-150: s_ref >= (1 - γ(2 dim + 10)) D^2 - (2 dim + 10) 2^-150.  Cosine: the fast path runs only when
//      |q||x| is a normal float, so the dot's underflow is another γ of |q||x|; with the norms' and the division's roundings
//      |cos_ref - cos| <= 2 γ(2 dim + 10) + 6u, and 1 - cos plus the halving add 2u: |s_ref - s| <= 1.01 (γ + 3u) + 2u.  The
//      f64 fallback is far more accurate than this.
// Everything is evaluated in double with a relative margin of 2^-30 on the comparison.  A query is flagged — never
// certified on an unproven bound — when its status word is not OK, its count is not k, S_k, L_q or the bound is not a
// finite number (a NaN bound compares false), or (cosine) the query's or a row's fp32 norm is below FLT_MIN, where the
// reference's own rounding of the norm is not relative (see k_dense_view_bound).
#define HXD_U (1.0 / 16777216.0)
__host__ __device__ inline double hxd_gamma(double n) { return n * HXD_U / (1.0 - n * HXD_U); }

// lower bound on the reference's fp32 score of any row of the view whose approximate score is >= L (see above).
// q_aux: the pass's query term (euclidean |q^|^2); r2: the largest row term of the view (euclidean |x^|^2)
__host__ __device__ inline double hxd_exact_floor(int metric, uint32_t dim, uint32_t ldb, double L, double q_aux, double r2) {
  const double u = HXD_U, ub = 1.0 / 256.0, sub = 0x1p-150, tiny = 0x1p-126, sd = sqrt((double)ldb);
  const double c_acc = (ldb + 16.0) * 4.0 * u, g_sq = hxd_gamma(ldb / 32 + 5.0), n_ref = 2.0 * dim + 10.0;
  if (metric == HXM_COSINE) {
    const double psi = 1.01 * (g_sq + ldb * sub + 4.0 * u), Psi = 1.01 * (2.0 * psi + u);
    const double err = 0.5 * (c_acc + 1.01 * Psi) + 1.6 * u + 0x1p-100;
    const double eta = ub + sd * 0x1p-133, eta1 = 1.01 * eta / (1.0 - eta);
    const double h = fmax(sqrt(fmax(L - err, 0.0)) - eta1, 0.0);   // <= half the chord between the true unit vectors
    return h * h - (1.01 * (hxd_gamma(n_ref) + 3.0 * u) + 2.0 * u);
  }
  const double Q = sqrt((q_aux + ldb * sub) / (1.0 - g_sq)), X = sqrt((r2 + ldb * sub) / (1.0 - g_sq));
  const double M = (Q + X) * (Q + X);
  const double a_acc = 2.0 * (ldb + 16.0) * tiny + tiny * sd * (Q + X);
  const double err = (g_sq + c_acc + 3.0 * u) * M + 2.0 * ldb * sub + 2.0 * a_acc + sub;
  const double a = sd * 0x1p-134, beta = ub * (Q + X + 2.0 * a) / (1.0 - ub) + 2.0 * a;
  const double D = fmax(sqrt(fmax(L - err, 0.0)) - beta, 0.0);   // <= |q - x|
  return (1.0 - hxd_gamma(n_ref)) * D * D - n_ref * sub;
}

// What the bound needs from the whole view, one word; *out must be 0 before the launch.
//   euclidean: the largest row term |x^|^2 over the positions that hold a row, as float bits (non-negative floats order
//              like their bits): R^2;
//   cosine:    1 when a row's exact header (its fp32 norm) is below FLT_MIN.  The reference's fast path divides by that
//              norm, whose fp32 rounding is then not relative (a row of +-2^-149 has a norm 15% off), so part (c) of the
//              bound does not hold for that row and no query of the call can be certified.
__global__ void k_dense_view_bound(const float* __restrict__ aux, const float* __restrict__ hdr,
                                   const uint32_t* __restrict__ slots, size_t n, int metric, uint32_t* __restrict__ out) {
  const size_t n_pad = (n + HXD_BN - 1) / HXD_BN * HXD_BN;
  uint32_t m = 0;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < n_pad; p += (size_t)gridDim.x * blockDim.x) {
    if (metric == HXM_COSINE) {
      if (p < n && !(hdr[slots[p]] >= FLT_MIN)) m = 1u;
    } else if (p / HXD_BN * HXD_BN + hxd_row_at_pos((uint32_t)(p % HXD_BN)) < n) {
      m = max(m, __float_as_uint(aux[p]));
    }
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31u) == 0 && m) atomicMax(out, m);
}

struct HxCertArgs {
  const uint64_t* keys;        // HxDensePassOut
  uint32_t n_split, kprime;
  const float* sel_sc;
  const uint32_t* sel_cnt;
  const float* q_aux;
  const float* out_sc;         // [B][k] the re-ranked answer
  const uint32_t* out_cnt;
  const uint32_t* q_status;
  const float* q_hdr;          // [B] exact query headers (cosine: fp32 norm)
  const uint32_t* view_word;   // k_dense_view_bound's word
  uint32_t B, k, dim, ldb;
  int32_t metric;
  uint32_t* flag;              // [B] q when the query must be rescanned, HX_ABSENT when certified (k_compact_* input)
  uint8_t* how;                // [B] 0 certified, 1 rescanned
};

// one warp per query: the warp takes the minimum over its n_split * HXD_PARTS bucket tails, lane 0 decides
__global__ void __launch_bounds__(256) k_dense_certify(HxCertArgs a) {
  const size_t q = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31u;
  if (q >= a.B) return;
  const uint32_t nb = a.n_split * HXD_PARTS;
  const uint64_t* kq = a.keys + q * nb * HXD_T;
  uint32_t lb = 0x7f800000u;   // +inf: no full bucket
  for (uint32_t i = lane; i < nb; i += 32) {
    const uint64_t tail = kq[(size_t)i * HXD_T + HXD_T - 1];
    if (tail != HX_KEY_MAX) lb = min(lb, (uint32_t)(tail >> 32));
  }
  lb = __reduce_min_sync(0xffffffffu, lb);
  if (lane != 0) return;
  float L = __uint_as_float(lb);
  if (a.sel_cnt[q] == a.kprime) L = fminf(L, a.sel_sc[q * a.kprime + a.kprime - 1]);
  bool ok = a.q_status[q] == 0u && a.out_cnt[q] == a.k;
  const float sk = ok ? a.out_sc[q * a.k + a.k - 1] : 0.f;
  ok = ok && isfinite(L) && isfinite(sk);
  // cosine: the reference's norms of the query and of every row must be normal floats (k_dense_view_bound)
  if (a.metric == HXM_COSINE) ok = ok && *a.view_word == 0u && a.q_hdr[q] >= FLT_MIN;
  if (ok) {
    const double r2 = a.metric == HXM_COSINE ? 0.0 : (double)__uint_as_float(*a.view_word);
    const double lo = hxd_exact_floor(a.metric, a.dim, a.ldb, (double)L, (double)a.q_aux[q], r2);
    ok = lo * (1.0 - 0x1p-30) > (double)sk;   // false for a NaN bound
  }
  a.flag[q] = ok ? HX_ABSENT : (uint32_t)q;
  a.how[q] = ok ? 0 : 1;
}

// ---- host ------------------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static hx_status make_map(CUtensorMap* map, void* base, uint64_t rows, uint32_t ldb, uint32_t box_rows) {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) {
      hx_set_error("cuTensorMapEncodeTiled is not available from the driver");
      return HX_ERR_CUDA;
    }
    fn = (PFN_encodeTiled)p;
  }
  const cuuint64_t dims[2] = {ldb, rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ldb * 2};
  const cuuint32_t box[2] = {HXD_BK, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    hx_set_error("cuTensorMapEncodeTiled failed (%d)", (int)r);
    return HX_ERR_CUDA;
  }
  return HX_OK;
}

// Lazily build the dense path's view of the corpus (dropped by every mirror write, hx_mirror.inl: invalidate_bf16): the
// ascending live slots and, when `need_bf16`, the bf16 copy of the live rows compacted in slot order (deleted rows take
// no tile column and no bucket space).  The work is enqueued on the calling stream and the pointers are published under
// ix->dense_mu only after that stream has completed it, so a caller on any other stream never reads a half-built copy,
// and concurrent first callers build it once.
static hx_status ensure_dense_state(hx_index* ix, uint32_t ldb, bool need_bf16, cudaStream_t stream) {
  std::lock_guard<std::mutex> lk(ix->dense_mu);
  if (!ix->d_live_slots) {
    std::vector<uint32_t> live;
    live.reserve(ix->n - std::min(ix->n, ix->n_deleted));
    for (size_t s = 0; s < ix->n; ++s)
      if (ix->host_deleted.empty() || !ix->host_deleted[s]) live.push_back((uint32_t)s);
    uint32_t* d = nullptr;
    HX_CUDA(cudaMalloc((void**)&d, std::max<size_t>(live.size(), 1) * sizeof(uint32_t)));
    cudaError_t e = cudaMemcpyAsync(d, live.data(), live.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) {
      cudaFree(d);
      hx_set_error("dense path live-row table: %s", cudaGetErrorString(e));
      return HX_ERR_CUDA;
    }
    ix->d_live_slots = d;
    ix->n_live = live.size();
  }
  if (!need_bf16 || ix->d_vec_bf16) return HX_OK;
  const size_t n = ix->n_live, n_pad = (n + HXD_BN - 1) / HXD_BN * HXD_BN;
  void* vb = nullptr;
  float* aux = nullptr;
  cudaError_t e = cudaMalloc(&vb, n_pad * (size_t)ldb * 2);
  if (e == cudaSuccess) e = cudaMalloc((void**)&aux, n_pad * sizeof(float));
  if (e == cudaSuccess) e = cudaMemsetAsync(vb, 0, n_pad * (size_t)ldb * 2, stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(aux, 0, n_pad * sizeof(float), stream);
  if (e == cudaSuccess) {
    k_to_bf16<<<(unsigned)((n + 7) / 8), 256, 0, stream>>>(ix->d_vec, n, ix->cfg.dimension, ix->ld, (__nv_bfloat16*)vb, ldb, aux,
                                                          ix->cfg.metric, 1, ix->d_live_slots);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  if (e != cudaSuccess) {
    if (vb) cudaFree(vb);
    if (aux) cudaFree(aux);
    hx_set_error("dense path bf16 copy: %s", cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? HX_ERR_OUT_OF_MEMORY : HX_ERR_CUDA;
  }
  ix->d_vec_bf16 = vb;
  ix->d_sqnorm = aux;
  return HX_OK;
}

// iota of the nominee CSR offsets (b * k')
static __global__ void k_dense_offsets(uint64_t* __restrict__ offs, size_t B, uint32_t kprime) {
  const size_t b = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b <= B) offs[b] = b * (uint64_t)kprime;
}

static hx_status dense_check(hx_index* ix, const hx_search_params* p) {
  if (!p || p->k == 0) {
    hx_set_error("result count must be non-zero");
    return HX_ERR_INVALID_PARAMETER;
  }
  if (p->k > 800) {
    hx_set_error("dense search result count must be at most 800");
    return HX_ERR_QUERY;
  }
  if (ix->cfg.storage != 1) {
    hx_set_error("hx_search_dense needs hx_index_config.storage == 1 (bf16 copy of the corpus)");
    return HX_ERR_INVALID_PARAMETER;
  }
  if (ix->cfg.metric == HX_METRIC_MANHATTAN) {
    hx_set_error("the L1 metric is not a contraction: use hx_search_restricted");
    return HX_ERR_UNSUPPORTED;
  }
  if (p->query_dimension != 0 && p->query_dimension != ix->cfg.dimension) {
    hx_set_error("invalid dimension: expected %u, got %u", ix->cfg.dimension, p->query_dimension);
    return HX_ERR_INVALID_DIMENSION;
  }
  return HX_OK;
}

// validation + exact headers (same order of checks as every other entry point)
static void dense_validate(hx_index* ix, const float* d_q, size_t B, float* d_qhdr, uint32_t* d_status, cudaStream_t stream) {
  const uint32_t dim = ix->cfg.dimension;
  float limit = 0.f;
  bool has_limit = false;
  if (ix->cfg.metric == HX_METRIC_EUCLIDEAN) {
    const double exact = std::sqrt((double)FLT_MAX / ((double)dim * 8.0));
    limit = (float)exact;
    if ((double)limit > exact) limit = std::nextafter(limit, 0.0f);
    has_limit = true;
  }
  k_validate_and_header<<<(unsigned)((B + 7) / 8), 256, 0, stream>>>(d_q, B, dim, dim, ix->cfg.metric, limit, has_limit ? 1 : 0,
                                                                    d_qhdr, d_status);
}

// Small corpora (see hx_dense_device): every query scans every live row with the exact kernel, keyed by position in the
// ascending live-slot table, and keeps the k smallest (score, id) — the answer of restricted_exact_scan over all ids.
static hx_status dense_exact_scan(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, const hx_search_params* p,
                                  uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt, cudaStream_t stream,
                                  cudaEvent_t e0, cudaEvent_t e1, uint32_t* launches_out) {
  const size_t n = ix->n_live;
  if (n == 0) {
    HX_CUDA(cudaMemsetAsync(d_out_cnt, 0, B * sizeof(uint32_t), stream));
    if (launches_out) *launches_out = 0;
    return HX_OK;
  }
  hx_status rc;
  DevBuf<uint8_t>& kb = scr->misc[15];   // not one of the tensor-core pass's buffers: its cached tensor maps stay valid
  if ((rc = kb.reserve(B * n * 8)) || (rc = scr->d_qhdr.reserve(B)) || (rc = scr->d_qstatus.reserve(B)) ||
      (rc = scr->d_err.reserve(4)))
    return rc;
  uint64_t* d_keys = reinterpret_cast<uint64_t*>(kb.p);
  HX_CUDA(cudaMemsetAsync(scr->d_err.p, 0, 4, stream));
  dense_validate(ix, d_q, B, scr->d_qhdr.p, scr->d_qstatus.p, stream);
  HxDev dev = ix->dev();
  HxScanArgs sa{};
  sa.queries = d_q;
  sa.q_hdr = scr->d_qhdr.p;
  sa.q_status = scr->d_qstatus.p;
  sa.B = (uint32_t)B;
  sa.cand_slots = ix->d_live_slots;
  sa.keys = d_keys;
  sa.shared_set = 1;
  sa.n_shared = n;
  sa.chunk = 1024;
  sa.err_flags = scr->d_err.p;
  dim3 g((unsigned)((n + sa.chunk - 1) / sa.chunk), (unsigned)std::min<size_t>(B, 65535));
  const uint32_t sm = ix->ld * 4u;
  if (e0) HX_CUDA(cudaEventRecord(e0, stream));
  if (ix->cfg.metric == HX_METRIC_COSINE) k_scan<HXM_COSINE><<<g, HX_SCAN_THREADS, sm, stream>>>(dev, sa);
  else k_scan<HXM_EUCLIDEAN><<<g, HX_SCAN_THREADS, sm, stream>>>(dev, sa);
  if (e1) HX_CUDA(cudaEventRecord(e1, stream));
  HxSelectArgs s2{};
  s2.keys = d_keys;
  s2.cand_slots = ix->d_live_slots;
  s2.q_status = scr->d_qstatus.p;
  s2.B = (uint32_t)B;
  s2.k = p->k;
  s2.shared_set = 1;
  s2.n_shared = n;
  s2.out_ids = d_out_ids;
  s2.out_scores = d_out_sc;
  s2.out_counts = d_out_cnt;
  k_select<<<(unsigned)std::min<size_t>(B, 65535), HX_SEL_THREADS, 0, stream>>>(dev, s2);
  HX_CUDA(cudaGetLastError());
  if (launches_out) *launches_out = 3;
  return HX_OK;
}

// Small corpora get the exact scan.  The tensor-core pass hands each query at most HXD_PARTS * HXD_T = 32 nominees per run
// of tiles, and a run is at least one 256-row tile, so a corpus of few tiles cannot fill k' = min(max(4k, 64), 800, rows)
// nominees, and its count could fall short of min(k, rows).  From 8 * min(max(4k, 64), 800) rows on, every run but the
// last holds a full tile (32 nominees), which covers k' (n_split below is at least k'/4 runs or every tile).  Below that
// the exact scan costs at most 6400 rows per query.
size_t hx_dense_min_rows(uint32_t k) { return 8 * (size_t)std::min<uint32_t>(std::max<uint32_t>(4 * k, 64), 800); }

// The corpus a tensor-core pass runs over: `n` bf16 rows in tile placement (k_to_bf16 with tiled = 1), their row terms
// (indexed by position), and the ascending slot table that maps row w of the view to its corpus slot.
struct HxDenseView {
  const void* rows;
  const float* aux;
  const uint32_t* slots;
  size_t n;
};

// What a tensor-core pass leaves behind that bounds what it may have dropped (read by the certificate, k_dense_certify)
struct HxDensePassOut {
  const uint64_t* keys;      // [B][n_split][HXD_PARTS][HXD_T] bucket lists of k_dense_scores
  uint32_t n_split;
  const float* sel_sc;       // [B][kprime] approximate scores of the nominees, ascending
  const uint32_t* sel_cnt;   // [B] nominees per query
  uint32_t kprime;
  const float* q_aux;        // [B] query terms of the pass (euclidean: |q^|^2)
};

// Tensor-core nomination over the view, then the exact re-rank with the reference arithmetic.  Needs
// n >= hx_dense_min_rows(k) and k <= 800, and the queries' exact headers and status words in scr->d_qhdr / d_qstatus.
// Everything is enqueued on `stream`; nothing synchronises with the host (buffers, the query tensor map and the nominee
// offsets are cached in the scratch set across calls; the corpus map is keyed on the view's (base, rows)).
// `pass_out` (may be null) receives the pass's internal buffers; they stay valid until the scratch set's next dense pass.
static hx_status dense_pass(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, uint32_t k, const HxDenseView& v,
                            uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt, cudaStream_t stream, cudaEvent_t e0,
                            cudaEvent_t e1, uint32_t* launches_out, HxDensePassOut* pass_out = nullptr) {
  hx_status rc;
  const uint32_t dim = ix->cfg.dimension;
  const uint32_t ldb = (dim + HXD_BK - 1) / HXD_BK * HXD_BK;
  const size_t n = v.n;
  const uint32_t kcap = std::min<uint32_t>(std::max<uint32_t>(4 * k, 64), 800);
  const uint32_t m_tiles = (uint32_t)((B + HXD_BM - 1) / HXD_BM), n_tiles = (uint32_t)((n + HXD_BN - 1) / HXD_BN);
  const size_t B_pad = (size_t)m_tiles * HXD_BM, n_pad = (size_t)n_tiles * HXD_BN;
  const size_t n_ctas = (size_t)std::max(1, ix->sm_count);   // one persistent CTA per SM
  const uint32_t kprime = (uint32_t)std::min<size_t>(kcap, n);
  // runs per query tile: enough units to fill the CTAs, and enough that one run's best-T comfortably covers its share
  // of the k' nominees even when the true neighbours cluster in id space (8x head-room)
  uint32_t n_split = (uint32_t)std::max<size_t>(1, std::min<size_t>(n_tiles,
      std::max<size_t>(std::max<size_t>(4, n_ctas / m_tiles), (8 * (size_t)kprime + HXD_PARTS * HXD_T - 1) / (HXD_PARTS * HXD_T))));
  // the grid is one persistent CTA per SM: make the number of work units a multiple of it so that the last wave is full
  // (1024 queries = 8 query tiles: 32 runs = 256 units = 1.94 waves of 132 CTAs; 33 runs = 264 units = exactly 2 waves)
  if ((size_t)m_tiles * n_split > n_ctas)
    for (uint32_t cand = n_split; cand <= std::min<uint32_t>(n_tiles, 2 * n_split); ++cand)
      if (((size_t)m_tiles * cand) % n_ctas == 0) { n_split = cand; break; }
  const size_t nkeys = B * (size_t)n_split * HXD_PARTS * HXD_T;
  int mi = 0;
  bool grew = false;
  auto take = [&](size_t bytes, void** out) -> hx_status {
    const unsigned char* before = scr->misc[mi].p;
    hx_status r = scr->misc[mi].reserve(bytes + 256);
    if (scr->misc[mi].p != before) grew = true;
    *out = scr->misc[mi].p;
    ++mi;
    return r;
  };
  float *d_qaux, *d_sel_sc;
  __nv_bfloat16* d_qb;
  uint64_t *d_keys, *d_sel_ids, *d_keys2, *d_coffs;
  uint32_t *d_sel_cnt, *d_cslots;
  if ((rc = take(B_pad * (size_t)ldb * 2, (void**)&d_qb)) || (rc = take(B_pad * 4, (void**)&d_qaux)) ||
      (rc = take(nkeys * 8, (void**)&d_keys)) || (rc = take(B * (size_t)kprime * 8, (void**)&d_sel_ids)) ||
      (rc = take(B * (size_t)kprime * 4, (void**)&d_sel_sc)) || (rc = take(B * 4, (void**)&d_sel_cnt)) ||
      (rc = take(B * (size_t)kprime * 4, (void**)&d_cslots)) || (rc = take((B + 1) * 8, (void**)&d_coffs)) ||
      (rc = take(B * (size_t)kprime * 8, (void**)&d_keys2)))
    return rc;
  if ((rc = scr->d_qhdr.reserve(B)) || (rc = scr->d_qstatus.reserve(B)) || (rc = scr->d_err.reserve(4))) return rc;
  float* d_qhdr = scr->d_qhdr.p;
  uint32_t* d_status = scr->d_qstatus.p;
  uint32_t* d_err = scr->d_err.p;
  HxDenseCache& dc = scr->dense;
  const bool shape_changed = grew || dc.B != B || dc.kprime != kprime || dc.ldb != ldb;
  HX_CUDA(cudaMemsetAsync(d_err, 0, 4, stream));
  HX_CUDA(cudaMemsetAsync(d_sel_ids, 0xFF, B * (size_t)kprime * 8, stream));   // unfilled nominee slots read as HX_ABSENT
  if (shape_changed) {   // pad rows / pad columns of the bf16 query tile and the nominee offsets: once per shape
    HX_CUDA(cudaMemsetAsync(d_qb, 0, B_pad * (size_t)ldb * 2, stream));
    HX_CUDA(cudaMemsetAsync(d_qaux, 0, B_pad * 4, stream));
    k_dense_offsets<<<(unsigned)((B + 256) / 256), 256, 0, stream>>>(d_coffs, B, kprime);
    if ((rc = make_map(reinterpret_cast<CUtensorMap*>(dc.map_q), d_qb, B_pad, ldb, HXD_BM))) return rc;
    dc.B = B;
    dc.kprime = kprime;
    dc.ldb = ldb;
  }
  if (dc.map_x_base != v.rows || dc.map_x_rows != n_pad) {
    if ((rc = make_map(reinterpret_cast<CUtensorMap*>(dc.map_x), const_cast<void*>(v.rows), n_pad, ldb, HXD_BH))) return rc;   // one MMA tile = half a placement tile
    dc.map_x_base = v.rows;
    dc.map_x_rows = n_pad;
  }
  uint32_t launches = 0;
  k_to_bf16<<<(unsigned)((B + 7) / 8), 256, 0, stream>>>(d_q, B, dim, dim, d_qb, ldb, d_qaux, ix->cfg.metric, 0, nullptr);
  launches += 1;
  HX_CUDA(cudaGetLastError());
  // ---- tensor-core pass ----
  HxDenseArgs a{};
  a.n_rows = (uint32_t)n;
  a.n_queries = (uint32_t)B;
  a.k_blocks = ldb / HXD_BK;
  a.m_tiles = m_tiles;
  a.n_tiles = n_tiles;
  a.n_split = n_split;
  a.row_aux = v.aux;
  a.q_aux = d_qaux;
  a.keys = d_keys;
  a.metric = ix->cfg.metric;
  const size_t smem = (size_t)HXD_STAGES * HXD_STAGE_BYTES + (size_t)HXD_BM * HXD_ACC_LD * 4 + HXD_BH * 4 + 2 * HXD_STAGES * 8 + 1024;
  static std::atomic<int> attr_set[64];
  if (!attr_set[ix->device & 63].load()) {
    HX_CUDA(cudaFuncSetAttribute(k_dense_scores, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set[ix->device & 63].store(1);
  }
  const uint32_t grid = (uint32_t)std::min<size_t>((size_t)m_tiles * n_split, n_ctas);
  if (e0) HX_CUDA(cudaEventRecord(e0, stream));
  k_dense_scores<<<grid, HXD_THREADS, smem, stream>>>(*reinterpret_cast<CUtensorMap*>(dc.map_q),
                                                      *reinterpret_cast<CUtensorMap*>(dc.map_x), a);
  if (e1) HX_CUDA(cudaEventRecord(e1, stream));
  launches++;
  HX_CUDA(cudaGetLastError());
  // ---- k' nominees per query by approximate key, then the exact re-rank with the reference arithmetic ----
  HxDev dev = ix->dev();
  HxSelectArgs s1{};
  s1.keys = d_keys;
  s1.q_status = d_status;
  s1.B = (uint32_t)B;
  s1.k = kprime;
  s1.shared_set = 2;   // keys carry rows of the bf16 copy in their low word (no candidate indirection)
  s1.n_shared = (uint64_t)n_split * HXD_PARTS * HXD_T;
  s1.out_ids = d_sel_ids;
  s1.out_scores = d_sel_sc;
  s1.out_counts = d_sel_cnt;
  k_select<<<(unsigned)std::min<size_t>(B, 65535), HX_SEL_THREADS, 0, stream>>>(dev, s1);
  uint32_t width = 32;
  while (width < kprime) width <<= 1;
  k_nominee_slots<<<(unsigned)std::min<size_t>(B, 65535), HXD_SORT_THREADS, 0, stream>>>(d_sel_ids, B, kprime, width,
                                                                                       v.slots, d_cslots);
  launches += 2;
  HxScanArgs sa{};
  sa.queries = d_q;
  sa.q_hdr = d_qhdr;
  sa.q_status = d_status;
  sa.B = (uint32_t)B;
  sa.cand_slots = d_cslots;
  sa.cand_offsets = d_coffs;
  sa.keys = d_keys2;
  sa.shared_set = 0;
  sa.n_shared = 0;
  sa.chunk = 32 * ((kprime + 31) / 32);
  sa.err_flags = d_err;
  {
    dim3 g(1, (unsigned)std::min<size_t>(B, 65535));
    const uint32_t sm = ix->ld * 4u;
    if (ix->cfg.metric == HX_METRIC_COSINE) k_scan<HXM_COSINE><<<g, HX_SCAN_THREADS, sm, stream>>>(dev, sa);
    else k_scan<HXM_EUCLIDEAN><<<g, HX_SCAN_THREADS, sm, stream>>>(dev, sa);
  }
  HxSelectArgs s2{};
  s2.keys = d_keys2;
  s2.cand_slots = d_cslots;
  s2.cand_offsets = d_coffs;
  s2.q_status = d_status;
  s2.B = (uint32_t)B;
  s2.k = k;
  s2.shared_set = 0;
  s2.n_shared = 0;
  s2.out_ids = d_out_ids;
  s2.out_scores = d_out_sc;
  s2.out_counts = d_out_cnt;
  k_select<<<(unsigned)std::min<size_t>(B, 65535), HX_SEL_THREADS, 0, stream>>>(dev, s2);
  launches += 2;
  HX_CUDA(cudaGetLastError());
  if (launches_out) *launches_out = launches;
  if (pass_out) *pass_out = HxDensePassOut{d_keys, n_split, d_sel_sc, d_sel_cnt, kprime, d_qaux};
  return HX_OK;
}

// k_dense_view_bound over view `v` into *word (zeroed first), enqueued on `stream`
static hx_status dense_view_word(hx_index* ix, const HxDenseView& v, uint32_t* word, cudaStream_t stream) {
  HX_CUDA(cudaMemsetAsync(word, 0, 4, stream));
  const size_t n_pad = (v.n + HXD_BN - 1) / HXD_BN * HXD_BN;
  const unsigned grid = (unsigned)std::min<size_t>((n_pad + 255) / 256, 4 * (size_t)std::max(1, ix->sm_count));
  k_dense_view_bound<<<grid, 256, 0, stream>>>(v.aux, ix->d_hdr, v.slots, v.n, ix->cfg.metric, word);
  HX_CUDA(cudaGetLastError());
  return HX_OK;
}

// The certificate after a pass over view `v` (see k_dense_certify), then the order-preserving compaction of the flagged
// query indices.  Enqueued on `stream`, no synchronisation.  Buffers: the scratch set's x_flag / x_how, none of the pass's.
// `resident_word`: the view's word as a resident view holds it (null: reduced here, one more launch).
static hx_status dense_certify(hx_index* ix, HxScratch* scr, size_t B, uint32_t k, const HxDenseView& v,
                               const HxDensePassOut& po, const float* d_out_sc, const uint32_t* d_out_cnt, HxDenseCert* cert,
                               cudaStream_t stream, uint32_t* launches, const uint32_t* resident_word = nullptr) {
  hx_status rc;
  const size_t tiles = (B + HXD_CPT_TILE - 1) / HXD_CPT_TILE;
  if ((rc = scr->x_flag.reserve(2 * B + tiles + 2)) || (rc = scr->x_how.reserve(B))) return rc;
  uint32_t* flag = scr->x_flag.p;          // [B] per query
  uint32_t* flagged = flag + B;            // [B] compacted
  uint32_t* counts = flagged + B;          // [tiles] + the total
  const uint32_t* view_word = resident_word;
  if (!view_word) {
    uint32_t* w = counts + tiles + 1;
    if ((rc = dense_view_word(ix, v, w, stream))) return rc;
    view_word = w;
    ++*launches;
  }
  HxCertArgs a{};
  a.keys = po.keys;
  a.n_split = po.n_split;
  a.kprime = po.kprime;
  a.sel_sc = po.sel_sc;
  a.sel_cnt = po.sel_cnt;
  a.q_aux = po.q_aux;
  a.out_sc = d_out_sc;
  a.out_cnt = d_out_cnt;
  a.q_status = scr->d_qstatus.p;
  a.q_hdr = scr->d_qhdr.p;
  a.view_word = view_word;
  a.B = (uint32_t)B;
  a.k = k;
  a.dim = ix->cfg.dimension;
  a.ldb = (ix->cfg.dimension + HXD_BK - 1) / HXD_BK * HXD_BK;
  a.metric = ix->cfg.metric;
  a.flag = flag;
  a.how = scr->x_how.p;
  k_dense_certify<<<(unsigned)((B + 7) / 8), 256, 0, stream>>>(a);
  k_compact_count<<<(unsigned)tiles, HXD_CPT_THREADS, 0, stream>>>(flag, B, counts);
  k_compact_scatter<<<(unsigned)tiles, HXD_CPT_THREADS, 0, stream>>>(flag, B, counts, flagged, counts + tiles);
  HX_CUDA(cudaGetLastError());
  *launches += 3;
  cert->small = false;
  cert->flagged = flagged;
  cert->n_flagged = counts + tiles;
  cert->how = scr->x_how.p;
  return HX_OK;
}

// hx_search_dense over every live row.  Everything below is enqueued on `stream`; nothing synchronises with the host once
// the dense state exists.  d_queries: B x dim f32 on the device.  Per-query validation status is left in s->d_qstatus
// (a query that fails validation yields count 0); error flags accumulate in s->d_err[0].
hx_status hx_dense_device(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, const hx_search_params* p,
                          uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt, cudaStream_t stream,
                          cudaEvent_t e0, cudaEvent_t e1, uint32_t* launches_out, HxDenseCert* cert) {
  hx_status rc = dense_check(ix, p);
  if (rc) return rc;
  if (B == 0) return HX_OK;
  if (ix->n == 0 || !ix->populated) {
    HX_CUDA(cudaMemsetAsync(d_out_cnt, 0, B * sizeof(uint32_t), stream));
    return HX_OK;
  }
  const uint32_t ldb = (ix->cfg.dimension + HXD_BK - 1) / HXD_BK * HXD_BK;
  if ((rc = ensure_dense_state(ix, ldb, false, stream))) return rc;
  const size_t n = ix->n_live;   // rows of the bf16 copy: the live rows, compacted
  if (n < hx_dense_min_rows(p->k)) {
    if (cert) cert->small = true;
    return dense_exact_scan(ix, scr, d_q, B, p, d_out_ids, d_out_sc, d_out_cnt, stream, e0, e1, launches_out);
  }
  if ((rc = ensure_dense_state(ix, ldb, true, stream))) return rc;
  if ((rc = scr->d_qhdr.reserve(B)) || (rc = scr->d_qstatus.reserve(B))) return rc;
  dense_validate(ix, d_q, B, scr->d_qhdr.p, scr->d_qstatus.p, stream);
  const HxDenseView v{ix->d_vec_bf16, ix->d_sqnorm, ix->d_live_slots, n};
  HxDensePassOut po{};
  rc = dense_pass(ix, scr, d_q, B, p->k, v, d_out_ids, d_out_sc, d_out_cnt, stream, e0, e1, launches_out, cert ? &po : nullptr);
  if (!rc && launches_out) *launches_out += 1;
  if (!rc && cert) {
    uint32_t l = 0;
    rc = dense_certify(ix, scr, B, p->k, v, po, d_out_sc, d_out_cnt, cert, stream, &l);
    if (launches_out) *launches_out += l;
  }
  return rc;
}

// hx_search_dense_restricted, step 1: the present entries of the ascending candidate slot list `d_slots` (n entries,
// HX_ABSENT for ids without a row and for deleted rows), compacted in order into scratch.  Synchronises the stream to read
// the count back (4 bytes).
hx_status hx_dense_compact(hx_index* ix, HxScratch* scr, const uint32_t* d_slots, size_t n, cudaStream_t stream,
                           const uint32_t** d_present, size_t* n_present, uint32_t* launches) {
  hx_status rc;
  const size_t tiles = (n + HXD_CPT_TILE - 1) / HXD_CPT_TILE;
  if ((rc = scr->misc[11].reserve(n * 4)) || (rc = scr->misc[12].reserve((tiles + 1) * 4)) || (rc = scr->h_err.reserve(1)))
    return rc;
  uint32_t* out = reinterpret_cast<uint32_t*>(scr->misc[11].p);
  uint32_t* counts = reinterpret_cast<uint32_t*>(scr->misc[12].p);   // [tiles] per-tile counts, then the total
  k_compact_count<<<(unsigned)tiles, HXD_CPT_THREADS, 0, stream>>>(d_slots, n, counts);
  k_compact_scatter<<<(unsigned)tiles, HXD_CPT_THREADS, 0, stream>>>(d_slots, n, counts, out, counts + tiles);
  HX_CUDA(cudaGetLastError());
  *launches += 2;
  HX_CUDA(cudaMemcpyAsync(scr->h_err.p, counts + tiles, 4, cudaMemcpyDeviceToHost, stream));
  HX_CUDA(cudaStreamSynchronize(stream));
  *d_present = out;
  *n_present = scr->h_err.p[0];
  return HX_OK;
}

// The tensor-core pass over a candidate view, then (cert != null) the certificate; `view_word` as dense_certify's
// resident_word.  Adds the launches it issues to *launches.
static hx_status dense_view_search(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, uint32_t k, const HxDenseView& v,
                                   const uint32_t* view_word, uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt,
                                   cudaStream_t stream, cudaEvent_t e0, cudaEvent_t e1, uint32_t* launches,
                                   HxDenseCert* cert) {
  hx_status rc;
  uint32_t pass_launches = 0;
  HxDensePassOut po{};
  if ((rc = dense_pass(ix, scr, d_q, B, k, v, d_out_ids, d_out_sc, d_out_cnt, stream, e0, e1, &pass_launches,
                       cert ? &po : nullptr)))
    return rc;
  *launches += pass_launches;
  if (cert) return dense_certify(ix, scr, B, k, v, po, d_out_sc, d_out_cnt, cert, stream, launches, view_word);
  return HX_OK;
}

// hx_search_dense_restricted, step 2 (n_present >= hx_dense_min_rows(k)): the present rows, converted from the f32 rows into
// a bf16 tile of this scratch set's own (k_to_bf16: tile placement over candidate RANK, cosine power-of-two scaling, row
// terms), then the tensor-core pass over that tile with the compacted slots as its slot table.  The whole-corpus bf16 copy
// is neither built nor read.  The queries' headers and status words must be in scr->d_qhdr / d_qstatus.
hx_status hx_dense_restricted_device(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, uint32_t k,
                                     const uint32_t* d_present, size_t n_present, uint64_t* d_out_ids, float* d_out_sc,
                                     uint32_t* d_out_cnt, cudaStream_t stream, cudaEvent_t e0, cudaEvent_t e1,
                                     uint32_t* launches, HxDenseCert* cert) {
  hx_status rc;
  const uint32_t ldb = (ix->cfg.dimension + HXD_BK - 1) / HXD_BK * HXD_BK;
  const size_t n_pad = (n_present + HXD_BN - 1) / HXD_BN * HXD_BN;
  if ((rc = scr->misc[9].reserve(n_pad * (size_t)ldb * 2)) || (rc = scr->misc[10].reserve(n_pad * 4))) return rc;
  void* tile = scr->misc[9].p;
  float* aux = reinterpret_cast<float*>(scr->misc[10].p);
  // the positions of the last placement tile that no candidate fills read as zero rows
  HX_CUDA(cudaMemsetAsync(static_cast<unsigned char*>(tile) + (n_pad - HXD_BN) * (size_t)ldb * 2, 0, (size_t)HXD_BN * ldb * 2,
                          stream));
  k_to_bf16<<<(unsigned)((n_present + 7) / 8), 256, 0, stream>>>(ix->d_vec, n_present, ix->cfg.dimension, ix->ld,
                                                                 (__nv_bfloat16*)tile, ldb, aux, ix->cfg.metric, 1, d_present);
  HX_CUDA(cudaGetLastError());
  *launches += 1;
  return dense_view_search(ix, scr, d_q, B, k, HxDenseView{tile, aux, d_present, n_present}, nullptr, d_out_ids, d_out_sc,
                           d_out_cnt, stream, e0, e1, launches, cert);
}

// ---- resident candidate views (hx_candidates_make_resident) -------------------------------------------------------------------
// The tile, its row terms and the view word of a resident view, from the current f32 rows of its present slots: the same
// kernels, on the same rows, as hx_dense_restricted_device and dense_certify run per call, so a search through the view
// returns the non-resident set's answer bit for bit.  Enqueued on r->stream, then ONE synchronisation.
static hx_status resident_fill(hx_index* ix, HxResident* r) {
  const uint32_t ldb = (ix->cfg.dimension + HXD_BK - 1) / HXD_BK * HXD_BK;
  k_to_bf16<<<(unsigned)((r->n + 7) / 8), 256, 0, r->stream>>>(ix->d_vec, r->n, ix->cfg.dimension, ix->ld,
                                                                (__nv_bfloat16*)r->rows, ldb, r->aux, ix->cfg.metric, 1,
                                                                r->slots);
  HX_CUDA(cudaGetLastError());
  hx_status rc = dense_view_word(ix, HxDenseView{r->rows, r->aux, r->slots, r->n}, r->word, r->stream);
  if (rc) return rc;
  HX_CUDA(cudaStreamSynchronize(r->stream));
  return HX_OK;
}

void hx_resident_free(HxResident* r) {
  if (!r) return;
  if (r->stream) cudaStreamDestroy(r->stream);
  if (r->slots) cudaFree(r->slots);
  if (r->rows) cudaFree(r->rows);
  if (r->aux) cudaFree(r->aux);
  delete r;
}

hx_status hx_resident_build(hx_index* ix, const uint32_t* d_slots, size_t n_slots, HxResident** out) {
  HxResident* r = new HxResident();
  struct Free { HxResident*& r; ~Free() { hx_resident_free(r); } } fr{r};   // unless published below
  const uint64_t epoch = ix->content_epoch.load(std::memory_order_acquire);
  HX_CUDA(cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking));
  if (n_slots) {
    HxScratch* s = nullptr;
    hx_status rc = hx_acquire_scratch(ix, &s);
    if (rc) return rc;
    struct Rel { hx_index* ix; HxScratch* s; ~Rel() { hx_release_scratch(ix, s); } } rel{ix, s};
    const uint32_t* d_present = nullptr;
    uint32_t launches = 0;
    if ((rc = hx_dense_compact(ix, s, d_slots, n_slots, r->stream, &d_present, &r->n, &launches))) return rc;
    if (r->n) {
      const uint32_t ldb = (ix->cfg.dimension + HXD_BK - 1) / HXD_BK * HXD_BK;
      const size_t n_pad = (r->n + HXD_BN - 1) / HXD_BN * HXD_BN;
      HX_CUDA(cudaMalloc((void**)&r->slots, r->n * 4));
      HX_CUDA(cudaMalloc(&r->rows, n_pad * (size_t)ldb * 2));
      HX_CUDA(cudaMalloc((void**)&r->aux, (n_pad + 1) * 4));
      r->word = reinterpret_cast<uint32_t*>(r->aux + n_pad);
      r->bytes = n_pad * (uint64_t)(2 * ldb + 4) + 4 * (uint64_t)r->n + 4;
      HX_CUDA(cudaMemcpyAsync(r->slots, d_present, r->n * 4, cudaMemcpyDeviceToDevice, r->stream));
      // the positions of the last placement tile that no candidate fills read as zero rows, for good: refreshes rewrite
      // the present positions only
      HX_CUDA(cudaMemsetAsync(r->rows, 0, n_pad * (size_t)ldb * 2, r->stream));
      HX_CUDA(cudaMemsetAsync(r->aux, 0, n_pad * 4, r->stream));
      if ((rc = resident_fill(ix, r))) return rc;
    }
  }
  r->epoch.store(epoch, std::memory_order_release);
  *out = r;
  r = nullptr;
  return HX_OK;
}

// The pattern of ensure_dense_state: a caller that finds the view stale takes the view's mutex, re-checks, re-gathers on the
// view's own stream, synchronises once and only then publishes the epoch; concurrent first callers wait on the mutex and
// find it current, so the tile is rebuilt once and never read half built.  In place: a stream-ordered search that still
// reads the tile counts as overlapping the row write that made it stale (patch calls must not overlap searches).
hx_status hx_resident_current(hx_index* ix, HxResident* r) {
  const uint64_t want = ix->content_epoch.load(std::memory_order_acquire);
  if (r->n == 0 || r->epoch.load(std::memory_order_acquire) == want) return HX_OK;
  std::lock_guard<std::mutex> lk(r->mu);
  if (r->epoch.load(std::memory_order_acquire) == want) return HX_OK;
  hx_status rc = resident_fill(ix, r);
  if (rc) return rc;
  r->epoch.store(want, std::memory_order_release);
  return HX_OK;
}

hx_status hx_dense_resident_device(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, uint32_t k, const HxResident& r,
                                   uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt, cudaStream_t stream,
                                   cudaEvent_t e0, cudaEvent_t e1, uint32_t* launches, HxDenseCert* cert) {
  return dense_view_search(ix, scr, d_q, B, k, HxDenseView{r.rows, r.aux, r.slots, r.n}, r.word, d_out_ids, d_out_sc,
                           d_out_cnt, stream, e0, e1, launches, cert);
}

// Host-buffer entry point: a private stream + scratch set per call, the queries cross PCIe with one async copy, results
// and per-query status come back with four, ONE stream synchronisation.  `exact` (hx_search_dense_exact): the certificate
// follows the re-rank and the queries it cannot clear are rescanned (hx_dense_rescan: one more synchronisation, for the
// flagged count); out_how (may be null) receives 0 / 1 per query, or 2 for every query when the exact scan answered all.
hx_status hx_dense_impl(hx_index* ix, const float* queries, size_t B, const hx_search_params* p, uint64_t* out_ids,
                        float* out_scores, uint32_t* out_counts, hx_stats* stats, bool exact, uint8_t* out_how) {
  hx_status rc = dense_check(ix, p);
  if (rc) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (B == 0) return HX_OK;
  if (!queries || !out_ids || !out_scores || !out_counts) return HX_ERR_INVALID_PARAMETER;
  if (exact && out_how) memset(out_how, 2, B);
  if (ix->n == 0 || !ix->populated) {
    for (size_t b = 0; b < B; ++b) out_counts[b] = 0;
    return HX_OK;
  }
  const uint32_t dim = ix->cfg.dimension, k = p->k;
  HxScratch* scr = nullptr;
  if ((rc = hx_acquire_scratch(ix, &scr))) return rc;
  struct Rel { hx_index* ix; HxScratch* s; ~Rel() { hx_release_scratch(ix, s); } } rel{ix, scr};
  if ((rc = scr->d_queries.reserve(B * (size_t)dim)) || (rc = scr->d_out_ids.reserve(B * (size_t)k)) ||
      (rc = scr->d_out_scores.reserve(B * (size_t)k)) || (rc = scr->d_out_counts.reserve(B)) ||
      (rc = scr->h_status.reserve(B)) || (rc = scr->h_err.reserve(1)))
    return rc;
  cudaStream_t st = scr->stream;
  HX_CUDA(cudaMemcpyAsync(scr->d_queries.p, queries, B * (size_t)dim * 4, cudaMemcpyHostToDevice, st));
  uint32_t launches = 0;
  HxDenseCert cert;
  if ((rc = hx_dense_device(ix, scr, scr->d_queries.p, B, p, scr->d_out_ids.p, scr->d_out_scores.p, scr->d_out_counts.p, st,
                            scr->ev0, scr->ev1, &launches, exact ? &cert : nullptr)))
    return rc;
  size_t flagged = 0;
  uint32_t err_before = 0;
  if (exact && !cert.small &&
      (rc = hx_dense_rescan(ix, scr, scr->d_queries.p, k, ix->d_live_slots, ix->n_live, cert, scr->d_out_ids.p,
                            scr->d_out_scores.p, scr->d_out_counts.p, st, scr->ev0, scr->ev1, &launches, &flagged,
                            &err_before)))
    return rc;
  HX_CUDA(cudaMemcpyAsync(out_ids, scr->d_out_ids.p, B * (size_t)k * 8, cudaMemcpyDeviceToHost, st));
  HX_CUDA(cudaMemcpyAsync(out_scores, scr->d_out_scores.p, B * (size_t)k * 4, cudaMemcpyDeviceToHost, st));
  HX_CUDA(cudaMemcpyAsync(out_counts, scr->d_out_counts.p, B * 4, cudaMemcpyDeviceToHost, st));
  HX_CUDA(cudaMemcpyAsync(scr->h_status.p, scr->d_qstatus.p, B * 4, cudaMemcpyDeviceToHost, st));
  HX_CUDA(cudaMemcpyAsync(scr->h_err.p, scr->d_err.p, 4, cudaMemcpyDeviceToHost, st));
  if (exact && !cert.small && out_how) HX_CUDA(cudaMemcpyAsync(out_how, cert.how, B, cudaMemcpyDeviceToHost, st));
  HX_CUDA(cudaStreamSynchronize(st));
  scr->h_err.p[0] |= err_before;
  for (size_t b = 0; b < B; ++b)
    if (scr->h_status.p[b] != HX_ST_OK) {
      const uint32_t w = scr->h_status.p[b], code = w >> 24;
      hx_set_error_index(w & 0xffffffu);
      hx_set_error("query %zu failed validation (code %u)", b, code);
      return code == HX_ST_COMPONENT ? HX_ERR_INVALID_VECTOR_COMPONENT
                                     : (code == HX_ST_ZERO_NORM ? HX_ERR_ZERO_NORM_COSINE : HX_ERR_MAGNITUDE_EXCEEDED);
    }
  if (scr->h_err.p[0] & HXF_INVALID_SCORE) {
    hx_set_error("vector distance kernel emitted an invalid score");
    return HX_ERR_INVARIANT_VIOLATION;
  }
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, scr->ev0, scr->ev1) == cudaSuccess) {
    ix->last_kernel_ms = ms;
    ix->last_kernel_launches = 1;
  }
  if (stats) {
    const uint32_t ldb = (dim + HXD_BK - 1) / HXD_BK * HXD_BK;
    stats->kernel_launches = launches;
    stats->distance_computations = (uint64_t)B * ix->n;
    stats->algorithmic_bytes = (uint64_t)ix->n * ldb * 2;   // corpus streamed once; the bound is the tensor pipe: 2*B*N*d flop
    stats->reserved = (uint64_t)(2.0 * (double)B * (double)ix->n * (double)ldb);   // flop of the contraction
    if (flagged) {   // the rescanned queries' full scans
      stats->distance_computations += flagged * ix->n_live;
      stats->algorithmic_bytes += flagged * ix->n_live * (4ull * dim + (ix->cfg.metric == HX_METRIC_COSINE ? 4 : 0));
    }
  }
  return HX_OK;
}
