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
//     per (query, run of tiles, column quarter) by register insertion, emitting score_bits<<32|slot keys — the B x N
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
  uint32_t n_rows;            // corpus rows (unpadded)
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
__global__ void k_to_bf16(const float* __restrict__ src, size_t rows, uint32_t dim, size_t ld_src, __nv_bfloat16* __restrict__ dst,
                          uint32_t ldb, float* __restrict__ aux, int metric, int tiled) {
  const size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31u;
  if (w >= rows) return;
  const size_t pos = tiled ? (w / HXD_BN) * HXD_BN + hxd_pos_of_row((uint32_t)(w % HXD_BN)) : w;
  const float* s = src + w * ld_src;
  __nv_bfloat16* d = dst + pos * (size_t)ldb;
  float ss = 0.f;
  for (uint32_t j = lane; j < ldb; j += 32) {
    const float x = j < dim ? s[j] : 0.f;
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

// keys[q][j] hold GLOBAL slots in their low word; turn the selected ones into a per-query candidate slot list
__global__ void k_keys_to_slots(const uint64_t* __restrict__ sel_ids_as_slots, size_t total, uint32_t* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) out[i] = (uint32_t)sel_ids_as_slots[i];
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

// lazily build the bf16 copy of the corpus
static hx_status ensure_bf16(hx_index* ix, uint32_t ldb) {
  if (ix->d_vec_bf16) return HX_OK;
  const size_t n_pad = (ix->n + HXD_BN - 1) / HXD_BN * HXD_BN;
  HX_CUDA(cudaMalloc(&ix->d_vec_bf16, n_pad * (size_t)ldb * 2));
  HX_CUDA(cudaMemset(ix->d_vec_bf16, 0, n_pad * (size_t)ldb * 2));
  HX_CUDA(cudaMalloc((void**)&ix->d_sqnorm, n_pad * sizeof(float)));
  HX_CUDA(cudaMemset(ix->d_sqnorm, 0, n_pad * sizeof(float)));
  k_to_bf16<<<(unsigned)((ix->n + 7) / 8), 256>>>(ix->d_vec, ix->n, ix->cfg.dimension, ix->ld, (__nv_bfloat16*)ix->d_vec_bf16, ldb,
                                                  ix->d_sqnorm, ix->cfg.metric, 1);
  HX_CUDA(cudaGetLastError());
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

// Everything below is enqueued on `stream`; nothing synchronises with the host (buffers, tensor maps and the nominee
// offsets are cached in the scratch set across calls).  d_queries: B x dim f32 on the device.  Per-query validation status
// is left in s->d_qstatus (a query that fails validation yields count 0); error flags accumulate in s->d_err[0].
hx_status hx_dense_device(hx_index* ix, HxScratch* scr, const float* d_q, size_t B, const hx_search_params* p,
                          uint64_t* d_out_ids, float* d_out_sc, uint32_t* d_out_cnt, cudaStream_t stream,
                          cudaEvent_t e0, cudaEvent_t e1, uint32_t* launches_out) {
  hx_status rc = dense_check(ix, p);
  if (rc) return rc;
  if (B == 0) return HX_OK;
  if (ix->n == 0 || !ix->populated) {
    HX_CUDA(cudaMemsetAsync(d_out_cnt, 0, B * sizeof(uint32_t), stream));
    return HX_OK;
  }
  const uint32_t dim = ix->cfg.dimension, k = p->k;
  const uint32_t ldb = (dim + HXD_BK - 1) / HXD_BK * HXD_BK;
  if ((rc = ensure_bf16(ix, ldb))) return rc;
  const size_t n = ix->n;
  const uint32_t m_tiles = (uint32_t)((B + HXD_BM - 1) / HXD_BM), n_tiles = (uint32_t)((n + HXD_BN - 1) / HXD_BN);
  const size_t B_pad = (size_t)m_tiles * HXD_BM, n_pad = (size_t)n_tiles * HXD_BN;
  const size_t n_ctas = (size_t)std::max(1, ix->sm_count);   // one persistent CTA per SM
  const uint32_t kprime = (uint32_t)std::min<size_t>(std::max<uint32_t>(4 * k, 64), std::min<size_t>(800, n));
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
  if (dc.map_x_base != ix->d_vec_bf16 || dc.map_x_rows != n_pad) {
    if ((rc = make_map(reinterpret_cast<CUtensorMap*>(dc.map_x), ix->d_vec_bf16, n_pad, ldb, HXD_BH))) return rc;   // one MMA tile = half a placement tile
    dc.map_x_base = ix->d_vec_bf16;
    dc.map_x_rows = n_pad;
  }
  uint32_t launches = 0;
  // validation + exact headers (same order of checks as every other entry point)
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
  k_to_bf16<<<(unsigned)((B + 7) / 8), 256, 0, stream>>>(d_q, B, dim, dim, d_qb, ldb, d_qaux, ix->cfg.metric, 0);
  launches += 2;
  HX_CUDA(cudaGetLastError());
  // ---- tensor-core pass ----
  HxDenseArgs a{};
  a.n_rows = (uint32_t)n;
  a.n_queries = (uint32_t)B;
  a.k_blocks = ldb / HXD_BK;
  a.m_tiles = m_tiles;
  a.n_tiles = n_tiles;
  a.n_split = n_split;
  a.row_aux = ix->d_sqnorm;
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
  s1.shared_set = 2;   // keys carry global slots in their low word (no candidate indirection)
  s1.n_shared = (uint64_t)n_split * HXD_PARTS * HXD_T;
  s1.out_ids = d_sel_ids;
  s1.out_scores = d_sel_sc;
  s1.out_counts = d_sel_cnt;
  k_select<<<(unsigned)std::min<size_t>(B, 65535), HX_SEL_THREADS, 0, stream>>>(dev, s1);
  k_keys_to_slots<<<(unsigned)((B * (size_t)kprime + 255) / 256), 256, 0, stream>>>(d_sel_ids, B * (size_t)kprime, d_cslots);
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
  return HX_OK;
}

// Host-buffer entry point: a private stream + scratch set per call, the queries cross PCIe with one async copy, results
// and per-query status come back with four, ONE stream synchronisation.
hx_status hx_dense_impl(hx_index* ix, const float* queries, size_t B, const hx_search_params* p, uint64_t* out_ids,
                        float* out_scores, uint32_t* out_counts, hx_stats* stats) {
  hx_status rc = dense_check(ix, p);
  if (rc) return rc;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (B == 0) return HX_OK;
  if (!queries || !out_ids || !out_scores || !out_counts) return HX_ERR_INVALID_PARAMETER;
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
  if ((rc = hx_dense_device(ix, scr, scr->d_queries.p, B, p, scr->d_out_ids.p, scr->d_out_scores.p, scr->d_out_counts.p, st,
                            scr->ev0, scr->ev1, &launches)))
    return rc;
  HX_CUDA(cudaMemcpyAsync(out_ids, scr->d_out_ids.p, B * (size_t)k * 8, cudaMemcpyDeviceToHost, st));
  HX_CUDA(cudaMemcpyAsync(out_scores, scr->d_out_scores.p, B * (size_t)k * 4, cudaMemcpyDeviceToHost, st));
  HX_CUDA(cudaMemcpyAsync(out_counts, scr->d_out_counts.p, B * 4, cudaMemcpyDeviceToHost, st));
  HX_CUDA(cudaMemcpyAsync(scr->h_status.p, scr->d_qstatus.p, B * 4, cudaMemcpyDeviceToHost, st));
  HX_CUDA(cudaMemcpyAsync(scr->h_err.p, scr->d_err.p, 4, cudaMemcpyDeviceToHost, st));
  HX_CUDA(cudaStreamSynchronize(st));
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
  }
  return HX_OK;
}
