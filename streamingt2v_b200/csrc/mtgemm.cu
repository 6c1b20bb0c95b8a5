// Multi-tap tensor-core GEMM for sm_90a.
// TMA (rank-5 activation view) -> smem stage ring (128B swizzle) -> wgmma (fp32 accumulators in registers)
// -> fused epilogue from registers.  See include/b200svd.h for the contract.
//
// Replaces, underneath StreamingWrapper.forward (reference code/models/diffusion/wrappers.py:23-78):
//   nn.Linear            code/models/svd/sgm/modules/attention.py:94-120,262-351, video_attention.py:23-168
//   Conv2d 3x3 (s1, s2)  code/models/svd/sgm/modules/diffusionmodules/openaimodel.py:107-207,257-305
//   Conv3d (3,1,1)       code/models/diffusion/video_model.py:46-59 (ResBlock dims=3)
//   + their elementwise neighbours (bias, emb add openaimodel.py:346-352, GEGLU attention.py:94-101,
//     residual / AlphaBlender diffusionmodules/util.py:358-370).
//
// Persistent CTAs (one per SM) walk the output tiles with a grid stride (N tile fastest).  Three warpgroups:
//   warpgroup 0     TMA producer for A/B (one thread; the stage ring runs ahead across tiles, so the next tile's
//                   operands stream in while the consumers run the epilogue of the current one)
//   warpgroups 1-2  consumers: each owns 64 rows of the 128-row tile, issues m64nBNk16 wgmma on the shared B stage
//                   and applies the epilogue straight from its accumulator registers.
// A convolution tap is a shifted box of the same activation view, so taps and K blocks form one reduction loop.
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/b200svd.h"
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace b200 {

struct GemmDev {
  int32_t tap_off[B200SVD_MAX_TAPS][5];
  uint32_t taps, kblocks;
  uint32_t n;  // GEMM N (weight rows)
  uint32_t n_tiles;
  uint32_t total_tiles;
  uint32_t m_ext[3];
  uint32_t m_lb[3];  // log2 of box
  uint32_t m_tiles[3];
  uint32_t m_adim[3];
  int64_t out_rs[3];
  void* out;
  int64_t ldo;
  int32_t out_fp32;
  const float* bias;
  const float* fvec;
  int64_t ldf;
  uint32_t rows_per_frame;
  int32_t act;
  float s_acc;
  const __nv_bfloat16* res1;
  int64_t ld1;
  float s1;
  const __nv_bfloat16* res2;
  int64_t ld2;
  float s2;
  float* gn_part;  // GroupNorm partial sums of the output, see b200svd.h
  int32_t* gn_slot_sample;
  int64_t gn_ld;
  uint32_t gn_rows;
};

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int NUM_THREADS = 3 * 128;        // producer warpgroup + two consumer warpgroups
constexpr int SMEM_LIMIT = 232448;          // 227 KB of dynamic shared memory per block

template <int BN>
struct TileCfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int GN_BYTES = 4 * BN * 8;  // per 32-row quadrant: (sum, sum of squares) per column
  static constexpr int FIXED_BYTES = GN_BYTES + 256;
  static constexpr int STAGES_FIT = (SMEM_LIMIT - FIXED_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 6 ? 6 : STAGES_FIT;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + FIXED_BYTES;
  // accumulator registers per consumer thread: BN / 2; the 256-wide tile needs the producer's registers
  static constexpr int CONSUMER_REGS = BN > 128 ? 232 : 160;
  static constexpr int PRODUCER_REGS = 40;
  static_assert(STAGES >= 3, "pipeline depth");
  static_assert(SMEM_BYTES <= SMEM_LIMIT, "shared memory budget");
  static_assert(STAGE_BYTES % 1024 == 0, "stage alignment");
  static_assert(2 * (STAGES + 0) * 8 <= 256 - 8, "barrier area");
};

// `tile` enumerates (N tile fastest, then M tile).  An M tile decodes to the box origin of each of the three output
// row dimensions.
__device__ __forceinline__ void decode_tile(const GemmDev& p, uint32_t tile, uint32_t& n_tile, uint32_t& mb1,
                                            uint32_t& mb2, uint32_t& mb3) {
  n_tile = tile % p.n_tiles;
  uint32_t mt = tile / p.n_tiles;
  const uint32_t t1 = mt % p.m_tiles[0];
  mt /= p.m_tiles[0];
  const uint32_t t2 = mt % p.m_tiles[1];
  const uint32_t t3 = mt / p.m_tiles[1];
  mb1 = t1 << p.m_lb[0];
  mb2 = t2 << p.m_lb[1];
  mb3 = t3 << p.m_lb[2];
}

__device__ __forceinline__ float ldg_bf16(const __nv_bfloat16* p) { return __bfloat162float(p[0]); }

// Two adjacent bf16 elements at index i (and i + 1 if `both`): one 32-bit load when aligned.
__device__ __forceinline__ void load_bf16_pair(const __nv_bfloat16* base, int64_t i, bool both, float& a, float& b) {
  if (both && (i & 1) == 0) {
    const uint32_t w = __ldg(reinterpret_cast<const unsigned int*>(base + i));
    a = bf16_lo(w);
    b = bf16_hi(w);
  } else {
    a = ldg_bf16(base + i);
    b = both ? ldg_bf16(base + i + 1) : 0.f;
  }
}

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
mtgemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmDev p) {
  using Cfg = TileCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int R = BN / 2;  // accumulator registers per thread (m64nBN: 64 x BN over 128 threads)
  extern __shared__ __align__(1024) uint8_t smem[];  // SWIZZLE_128B operands need 1024-byte alignment
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  float* gn_x = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);  // [4 quadrants][BN][2]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES + Cfg::GN_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const uint32_t iters_per_tile = p.taps * p.kblocks;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::PRODUCER_REGS));
    if (threadIdx.x == 0) {
      // ===================== TMA producer (A, B) =====================
      uint32_t it = 0;
      for (uint32_t tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        uint32_t n_tile, mb1, mb2, mb3;
        decode_tile(p, tile, n_tile, mb1, mb2, mb3);
        int base[5] = {0, 0, 0, 0, 0};
        base[p.m_adim[0]] += (int)mb1;
        base[p.m_adim[1]] += (int)mb2;
        base[p.m_adim[2]] += (int)mb3;
        const int n0 = (int)(n_tile * BN);
        for (uint32_t tap = 0; tap < p.taps; ++tap) {
          const int c0 = p.tap_off[tap][0];
          const int c1 = base[1] + p.tap_off[tap][1];
          const int c2 = base[2] + p.tap_off[tap][2];
          const int c3 = base[3] + p.tap_off[tap][3];
          const int c4 = base[4] + p.tap_off[tap][4];
          for (uint32_t kb = 0; kb < p.kblocks; ++kb, ++it) {
            const uint32_t s = it % STAGES;
            const uint32_t ph = (it / STAGES) & 1;
            mbar_wait_parked(&empty_bar[s], ph ^ 1);
            uint8_t* sa = smem + s * Cfg::STAGE_BYTES;
            mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
            tma_load_5d(sa, &tmA, &full_bar[s], c0 + (int)(kb * BK), c1, c2, c3, c4);
            tma_load_3d(sa + A_STAGE_BYTES, &tmB, &full_bar[s], (int)(kb * BK), n0, (int)tap);
          }
        }
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::CONSUMER_REGS));

  // ===================== consumer warpgroups =====================
  const int cw = wg - 1;   // rows [64 cw, 64 cw + 64) of the tile
  const int wl = warp & 3;  // warp of the warpgroup: rows 16 wl .. 16 wl + 15 of those 64
  const int rq = lane >> 2, cq = lane & 3;
  const bool geglu = (p.act == B200SVD_ACT_GEGLU);
  const uint32_t n_out = geglu ? p.n / 2 : p.n;
  const uint32_t tile_out_w = geglu ? (uint32_t)BN / 2 : (uint32_t)BN;
  const uint32_t lb1 = p.m_lb[0], lb2 = p.m_lb[1];
  const int quad = 2 * cw + (wl >> 1);  // 32-row quadrant of the tile
  const bool gn = p.gn_part != nullptr;
  const bool gn_sender = (wl & 1) != 0;
  const int gn_bar = 1 + quad;
  float* gxq = gn_x + quad * BN * 2;
  uint32_t it = 0;
  float acc[R];

  for (uint32_t tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
#pragma unroll
    for (int i = 0; i < R; ++i) acc[i] = 0.f;
    for (uint32_t i = 0; i < iters_per_tile; ++i, ++it) {
      const uint32_t s = it % STAGES;
      mbar_wait(&full_bar[s], (it / STAGES) & 1);
      const uint32_t sa = smem_u32(smem + s * Cfg::STAGE_BYTES);
      const uint64_t adesc = smem_desc_k_sw128(sa + cw * (A_STAGE_BYTES / 2));
      const uint64_t bdesc = smem_desc_k_sw128(sa + A_STAGE_BYTES);
      wgmma_fence_regs(acc);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk)  // +16 elements along K = +32 B inside the swizzle atom
        Wgmma<BN>::ss(acc, adesc + (uint64_t)(kk * 2), bdesc + (uint64_t)(kk * 2), 1u);
      wgmma_commit();
      wgmma_fence_regs(acc);
      // the MMAs of the previous stage have completed: hand it back to the producer
      wgmma_wait<1>();
      if (i > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);

    // ----- epilogue: thread holds rows r0 and r0 + 8, columns 8 j + 2 cq + {0, 1} (acc[4 j + 2 h + e]) -----
    uint32_t n_tile, mb1, mb2, mb3;
    decode_tile(p, tile, n_tile, mb1, mb2, mb3);
    const uint32_t n0 = n_tile * BN;
    const uint32_t otile0 = n_tile * tile_out_w;
    bool valid[2];
    int64_t row[2];
    const float* fv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t r = (uint32_t)(64 * cw + 16 * wl + rq + 8 * h);
      const uint32_t m1 = mb1 + (r & ((1u << lb1) - 1));
      const uint32_t m2 = mb2 + ((r >> lb1) & ((1u << lb2) - 1));
      const uint32_t m3 = mb3 + (r >> (lb1 + lb2));
      valid[h] = (m1 < p.m_ext[0]) && (m2 < p.m_ext[1]) && (m3 < p.m_ext[2]);
      row[h] = (int64_t)m1 * p.out_rs[0] + (int64_t)m2 * p.out_rs[1] + (int64_t)m3 * p.out_rs[2];
      fv[h] = (p.fvec != nullptr && valid[h]) ? p.fvec + (int64_t)((uint32_t)row[h] / p.rows_per_frame) * p.ldf
                                              : nullptr;
    }
    constexpr int NJ = BN / 8;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      if (geglu && j >= NJ / 2) break;  // gate columns are consumed with their value columns
      const uint32_t tcol = 8 * j + 2 * cq;  // column in the tile (value column for GEGLU)
      const uint32_t ocol = otile0 + tcol;
      const bool in0 = ocol < n_out, in1 = ocol + 1 < n_out;
      float gs0 = 0.f, gs1 = 0.f, gq0 = 0.f, gq1 = 0.f;  // GroupNorm partials of the two columns
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (!valid[h] || !in0) continue;
        if (p.bias != nullptr) {
          v0 += __ldg(p.bias + n0 + tcol);
          if (in1) v1 += __ldg(p.bias + n0 + tcol + 1);
        }
        if (fv[h] != nullptr) {
          v0 += __ldg(fv[h] + ocol);
          if (in1) v1 += __ldg(fv[h] + ocol + 1);
        }
        if (p.act == B200SVD_ACT_SILU) {
          v0 = silu_fast(v0);
          v1 = silu_fast(v1);
        } else if (p.act == B200SVD_ACT_GELU) {
          v0 = gelu_fast(v0);
          v1 = gelu_fast(v1);
        } else if (geglu) {
          float g0 = acc[4 * (j + NJ / 2) + 2 * h], g1 = acc[4 * (j + NJ / 2) + 2 * h + 1];
          if (p.bias != nullptr) {
            g0 += __ldg(p.bias + n0 + BN / 2 + tcol);
            if (in1) g1 += __ldg(p.bias + n0 + BN / 2 + tcol + 1);
          }
          v0 *= gelu_fast(g0);
          v1 *= gelu_fast(g1);
        }
        v0 *= p.s_acc;
        v1 *= p.s_acc;
        if (p.res1 != nullptr) {
          float a, b;
          load_bf16_pair(p.res1, row[h] * p.ld1 + ocol, in1, a, b);
          v0 += p.s1 * a;
          v1 += p.s1 * b;
        }
        if (p.res2 != nullptr) {
          float a, b;
          load_bf16_pair(p.res2, row[h] * p.ld2 + ocol, in1, a, b);
          v0 += p.s2 * a;
          v1 += p.s2 * b;
        }
        if (p.out_fp32) {
          float* op = reinterpret_cast<float*>(p.out) + row[h] * p.ldo + ocol;
          if (in1 && ((row[h] * p.ldo + ocol) & 1) == 0) {
            *reinterpret_cast<float2*>(op) = make_float2(v0, v1);
          } else {
            op[0] = v0;
            if (in1) op[1] = v1;
          }
        } else {
          __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(p.out) + row[h] * p.ldo + ocol;
          const uint32_t w = pack_bf16x2(v0, v1);
          if (in1) {
            *reinterpret_cast<uint32_t*>(op) = w;  // ldo % 8 == 0 and an even column: 4-byte aligned
          } else {
            op[0] = __float2bfloat16(v0);
          }
          // statistics of the bf16-ROUNDED values, the ones the consumer reads
          const float r0 = bf16_lo(w), r1 = in1 ? bf16_hi(w) : 0.f;
          gs0 += r0;
          gs1 += r1;
          gq0 += r0 * r0;
          gq1 += r1 * r1;
        }
      }
      if (gn) {
        // column sums over the warp's 16 rows (lanes of equal cq), then over the quadrant's two warps via smem
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          gs0 += __shfl_xor_sync(0xffffffffu, gs0, o);
          gs1 += __shfl_xor_sync(0xffffffffu, gs1, o);
          gq0 += __shfl_xor_sync(0xffffffffu, gq0, o);
          gq1 += __shfl_xor_sync(0xffffffffu, gq1, o);
        }
        if (gn_sender && rq == 0)
          *reinterpret_cast<float4*>(gxq + 2 * tcol) = make_float4(gs0, gq0, gs1, gq1);
        if (!gn_sender) {
          acc[4 * j] = gs0;  // the accumulators of this column block are consumed: park the partials there
          acc[4 * j + 1] = gq0;
          acc[4 * j + 2] = gs1;
          acc[4 * j + 3] = gq1;
        }
      }
    }
    if (gn) {
      named_bar_sync(gn_bar, 64);  // the partner warp's partials are in shared memory
      if (!gn_sender) {
        const uint32_t slot = (tile / p.n_tiles) * 4u + (uint32_t)quad;
        if (rq == 0) {
          float2* dst = reinterpret_cast<float2*>(p.gn_part) + (int64_t)slot * p.gn_ld;
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            const uint32_t tcol = 8 * j + 2 * cq;
            const uint32_t ocol = otile0 + tcol;
            if (ocol < n_out) {
              const float4 o = *reinterpret_cast<const float4*>(gxq + 2 * tcol);
              dst[ocol] = make_float2(acc[4 * j] + o.x, acc[4 * j + 1] + o.y);
              if (ocol + 1 < n_out) dst[ocol + 1] = make_float2(acc[4 * j + 2] + o.z, acc[4 * j + 3] + o.w);
            }
          }
        }
        // lane 0 holds the first row of the quadrant: if it is out of range, so is every row of the quadrant
        if (lane == 0 && n_tile == 0) p.gn_slot_sample[slot] = valid[0] ? (int32_t)((uint32_t)row[0] / p.gn_rows) : -1;
      }
      named_bar_sync(gn_bar, 64);  // read before the next tile overwrites
    }
  }
}

static int ilog2_exact(uint32_t v) {
  if (v == 0 || (v & (v - 1)) != 0) return -1;
  int l = 0;
  while ((1u << l) < v) ++l;
  return l;
}

template <int BN>
static int launch(const b200svd_gemm_params* p, const CUtensorMap& tmA, const GemmDev& d, cudaStream_t st) {
  using Cfg = TileCfg<BN>;
  // weights [taps][n][k] -> TMA dims (k, n, taps)
  CUtensorMap tmB;
  uint64_t bd[3] = {p->k, p->n, p->taps};
  uint64_t bs[2] = {(uint64_t)p->k * 2, (uint64_t)p->k * 2 * p->n};
  uint32_t bb[3] = {64, (uint32_t)BN, 1};
  if (encode_tmap_bf16(&tmB, p->w_ptr, 3, bd, bs, bb)) return 1;
  GemmDev dd = d;
  dd.n_tiles = (p->n + BN - 1) / BN;
  const int slot = dev_slot();
  static bool attr_set[B200_MAX_DEVICES] = {};
  if (!attr_set[slot]) {
    cudaError_t e = cudaFuncSetAttribute(mtgemm_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(mtgemm)");
    attr_set[slot] = true;
  }
  const uint64_t m_tiles = (uint64_t)dd.m_tiles[0] * dd.m_tiles[1] * dd.m_tiles[2];
  const uint64_t total = (uint64_t)dd.n_tiles * m_tiles;
  if (total == 0 || total > 0x7FFFFFFFull) {
    set_error("mtgemm: bad tile count %llu", (unsigned long long)total);
    return 1;
  }
  dd.total_tiles = (uint32_t)total;
  const uint32_t grid = (uint32_t)(total < (uint64_t)sm_count() ? total : (uint64_t)sm_count());
  mtgemm_kernel<BN><<<grid, NUM_THREADS, Cfg::SMEM_BYTES, st>>>(tmA, tmB, dd);
  B200_CHECK_LAUNCH("mtgemm launch");
  return 0;
}

// Kept for the C ABI: CTA-pair (cta_group::2) tiles do not exist on sm_90, every launch uses single-CTA tiles.
static int g_pair_mode = 2;

}  // namespace b200

extern "C" int b200svd_gemm_pair_mode(int mode) {
  const int prev = b200::g_pair_mode;
  if (mode >= 0 && mode <= 3) b200::g_pair_mode = mode;
  return prev;
}

extern "C" int b200svd_gemm(const b200svd_gemm_params* p, void* stream) {
  using namespace b200;
  if (p == nullptr) {
    set_error("b200svd_gemm: null params");
    return 1;
  }
  if (p->taps == 0 || p->taps > B200SVD_MAX_TAPS) {
    set_error("b200svd_gemm: taps=%u out of range", p->taps);
    return 1;
  }
  if (p->a_box[0] != 64 || (uint64_t)p->a_box[1] * p->a_box[2] * p->a_box[3] * p->a_box[4] != 128) {
    set_error("b200svd_gemm: A box must be 64 x (product 128), got [%u,%u,%u,%u,%u]", p->a_box[0], p->a_box[1],
              p->a_box[2], p->a_box[3], p->a_box[4]);
    return 1;
  }
  if (p->k % 8 != 0) {
    set_error("b200svd_gemm: K=%u must be a multiple of 8 (16-byte TMA rows)", p->k);
    return 1;
  }
  GemmDev d;
  memset(&d, 0, sizeof(d));
  for (uint32_t t = 0; t < p->taps; ++t)
    for (int i = 0; i < 5; ++i) d.tap_off[t][i] = p->tap_off[t][i];
  d.taps = p->taps;
  d.kblocks = (p->k + 63) / 64;
  d.n = p->n;
  uint32_t prod = 1;
  for (int i = 0; i < 3; ++i) {
    int lb = ilog2_exact(p->m_box[i]);
    if (lb < 0) {
      set_error("b200svd_gemm: m_box[%d]=%u is not a power of two", i, p->m_box[i]);
      return 1;
    }
    if (p->m_adim[i] < 1 || p->m_adim[i] > 4) {
      set_error("b200svd_gemm: m_adim[%d]=%u must be in 1..4", i, p->m_adim[i]);
      return 1;
    }
    if (p->a_box[p->m_adim[i]] != p->m_box[i]) {
      set_error("b200svd_gemm: a_box[%u]=%u != m_box[%d]=%u", p->m_adim[i], p->a_box[p->m_adim[i]], i, p->m_box[i]);
      return 1;
    }
    if (i > 0 && p->m_adim[i] <= p->m_adim[i - 1]) {
      set_error("b200svd_gemm: m_adim must be increasing");
      return 1;
    }
    prod *= p->m_box[i];
    d.m_ext[i] = p->m_ext[i];
    d.m_lb[i] = (uint32_t)lb;
    d.m_tiles[i] = (p->m_ext[i] + p->m_box[i] - 1) / p->m_box[i];
    d.m_adim[i] = p->m_adim[i];
    d.out_rs[i] = p->out_rs[i];
  }
  if (prod != 128) {
    set_error("b200svd_gemm: m_box product %u != 128", prod);
    return 1;
  }
  d.out = p->out;
  d.ldo = p->ldo;
  d.out_fp32 = p->out_fp32;
  d.bias = p->bias;
  d.fvec = p->fvec;
  d.ldf = p->ldf;
  d.rows_per_frame = p->rows_per_frame ? p->rows_per_frame : 1;
  d.act = p->act;
  d.s_acc = p->s_acc;
  d.res1 = reinterpret_cast<const __nv_bfloat16*>(p->res1);
  d.ld1 = p->ld1;
  d.s1 = p->s1;
  d.res2 = reinterpret_cast<const __nv_bfloat16*>(p->res2);
  d.ld2 = p->ld2;
  d.s2 = p->s2;
  d.gn_part = p->gn_part;
  d.gn_slot_sample = p->gn_slot_sample;
  d.gn_ld = p->gn_ld;
  d.gn_rows = p->gn_rows ? p->gn_rows : 1;

  int bn = p->bn;
  if (p->act == B200SVD_ACT_GEGLU) {
    if (bn == 0) bn = 256;
    if (bn != 256 || (p->n % 256) != 0) {
      set_error("b200svd_gemm: GEGLU needs n (%u) divisible by 256 and the 256-wide tile (weights interleaved per tile)",
                p->n);
      return 1;
    }
  }
  const uint64_t m_tiles_all = (uint64_t)d.m_tiles[0] * d.m_tiles[1] * d.m_tiles[2];
  if (bn == 0) {
    if (p->n <= 32) bn = 32;
    else if (p->n <= 64) bn = 64;
    else if (p->n <= 128) bn = 128;
    else if (p->n == 160 || p->n == 320) bn = 160;  // no ragged N tile
    // a single M tile: the 128-wide tile spreads such a (weight-streaming) GEMM over more SMs
    else bn = m_tiles_all < 2 ? 128 : 256;
  }
  // wgmma takes N <= 256: a 320-wide tile is computed as two 160-wide tiles
  if (bn == 320) bn = 160;
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  // The epilogue stores column pairs as one word (bf16x2 or float2) and loads residual pairs as one 32-bit word
  // whenever the element offset from the base is even, so every base must be aligned to that word.
  const bool res_ok = (p->res1 == nullptr || (p->ld1 % 8 == 0 && al16(p->res1))) &&
                      (p->res2 == nullptr || (p->ld2 % 8 == 0 && al16(p->res2)));
  const bool bf16_ok = p->ldo % 8 == 0 && al16(p->out);
  if (!res_ok || (!p->out_fp32 && !bf16_ok)) {
    set_error("b200svd_gemm: bf16 outputs/residuals need 16-byte aligned bases and leading dims that are multiples of 8");
    return 1;
  }
  if (p->out_fp32 && (reinterpret_cast<uintptr_t>(p->out) & 7) != 0) {
    set_error("b200svd_gemm: an fp32 output needs an 8-byte aligned base");
    return 1;
  }
  const uint32_t n_out = p->act == B200SVD_ACT_GEGLU ? p->n / 2 : p->n;
  if (p->gn_part != nullptr &&
      (p->act != B200SVD_ACT_NONE || p->out_fp32 || (n_out % 16) != 0 || bn < 128 || p->gn_slot_sample == nullptr ||
       p->gn_ld < (int64_t)p->n || (p->gn_ld % 2) != 0 || (reinterpret_cast<uintptr_t>(p->gn_part) & 7) != 0)) {
    set_error("b200svd_gemm: gn_part needs the activation-free bf16 epilogue (n %% 16 == 0, n > 64), gn_slot_sample and "
              "an 8-byte aligned partial buffer with gn_ld >= n");
    return 1;
  }

  CUtensorMap tmA;
  if (encode_tmap_bf16(&tmA, p->a_ptr, 5, p->a_dims, p->a_strides, p->a_box)) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (bn) {
    case 32: return launch<32>(p, tmA, d, st);
    case 64: return launch<64>(p, tmA, d, st);
    case 128: return launch<128>(p, tmA, d, st);
    case 160: return launch<160>(p, tmA, d, st);
    case 256: return launch<256>(p, tmA, d, st);
    default: set_error("b200svd_gemm: unsupported N tile %d", bn); return 1;
  }
}
