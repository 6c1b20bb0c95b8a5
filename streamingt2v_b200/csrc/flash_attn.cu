// FlashAttention forward for sm_90a, head dim 64: wgmma for S = Q K^T and O += P V with the accumulators in
// registers, TMA-fed Q/K/V tiles read straight from the fused QKV projection output [(n s), 3C] (no head split /
// transpose in HBM).
//
// Replaces the spatial self-attention core of BasicTransformerBlock.attn1
// (reference code/models/svd/sgm/modules/attention.py:320-351 SDPA / :427-446 xformers), batch = frames,
// heads = C/64, sequence = H*W.
//
// CTA = one 128-row query tile of one (frame, head), three warpgroups:
//   warpgroup 0      TMA producer (Q once; K/V ring of FA_KV_STAGES 128-key blocks)
//   warpgroups 1, 2  64 query rows each.  Per key block:
//     S[64x128] = Q K_j^T            4 x wgmma m64n128k16, both operands from shared memory
//     online softmax in registers    row max over the quad of threads sharing a row, P = exp2(S*c - m), O and l
//                                    rescaled when the running max rises
//     O[64x64] += P V_j              8 x wgmma m64n64k16, A = P (bf16) from registers, B = V MN-major from smem
#include <cuda.h>
#include <cuda_bf16.h>
#include <math.h>

#include "../../include/b200svd.h"
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace b200 {

constexpr int FA_BQ = 128;
constexpr int FA_BK = 128;
constexpr int FA_D = 64;
constexpr int FA_KV_STAGES = 4;
constexpr int FA_Q_BYTES = FA_BQ * FA_D * 2;        // 16 KB
constexpr int FA_KV_TILE_BYTES = FA_BK * FA_D * 2;  // 16 KB each for K and V
constexpr int FA_SMEM_BYTES = FA_Q_BYTES + FA_KV_STAGES * 2 * FA_KV_TILE_BYTES + 256;
constexpr int FA_THREADS = 3 * 128;

struct FaParams {
  __nv_bfloat16* out;
  int64_t ldo;
  int S, heads, C;
  float scale_log2;
};

__global__ void __launch_bounds__(FA_THREADS, 1)
flash_attn_kernel(const __grid_constant__ CUtensorMap tmQKV, const FaParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];  // SWIZZLE_128B tiles need 1024-byte alignment
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + FA_Q_BYTES;  // stage s: K at sKV + s*32K, V at +16K
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + FA_KV_STAGES * 2 * FA_KV_TILE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                 // [FA_KV_STAGES]
  uint64_t* kv_empty = kv_full + FA_KV_STAGES;  // [FA_KV_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int head = blockIdx.y, n = blockIdx.z;
  const int q0 = blockIdx.x * FA_BQ;
  const int nkb = (p.S + FA_BK - 1) / FA_BK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmQKV);
    mbar_init(q_full, 1);
    for (int s = 0; s < FA_KV_STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      // ===================== TMA producer =====================
      mbar_expect_tx(q_full, FA_Q_BYTES);
      tma_load_3d(sQ, &tmQKV, q_full, head * FA_D, q0, n);
      for (int j = 0; j < nkb; ++j) {
        const int s = j % FA_KV_STAGES;
        mbar_wait_parked(&kv_empty[s], ((j / FA_KV_STAGES) & 1) ^ 1);
        uint8_t* sk = sKV + s * 2 * FA_KV_TILE_BYTES;
        mbar_expect_tx(&kv_full[s], 2 * FA_KV_TILE_BYTES);
        tma_load_3d(sk, &tmQKV, &kv_full[s], p.C + head * FA_D, j * FA_BK, n);
        tma_load_3d(sk + FA_KV_TILE_BYTES, &tmQKV, &kv_full[s], 2 * p.C + head * FA_D, j * FA_BK, n);
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");

  // ===================== consumer warpgroups: rows 64 cw + 16 wl + rq (+ 8) of the tile =====================
  const int cw = wg - 1, wl = warp & 3;
  const int rq = lane >> 2, cq = lane & 3;
  const float c = p.scale_log2;
  const uint64_t qdesc = smem_desc_k_sw128(smem_u32(sQ + cw * (FA_Q_BYTES / 2)));
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};  // running max, already scaled by c (log2 units)
  float l_run[2] = {0.f, 0.f};              // this thread's part of the row sum
  mbar_wait(q_full, 0);

  for (int j = 0; j < nkb; ++j) {
    const int st = j % FA_KV_STAGES;
    mbar_wait(&kv_full[st], (j / FA_KV_STAGES) & 1);
    const uint32_t sk = smem_u32(sKV + st * 2 * FA_KV_TILE_BYTES);
    float sacc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) sacc[i] = 0.f;
    wgmma_fence_regs(sacc);
    wgmma_fence();
    const uint64_t kdesc = smem_desc_k_sw128(sk);
#pragma unroll
    for (int kk = 0; kk < FA_D / 16; ++kk) Wgmma<128>::ss(sacc, qdesc + (uint64_t)(kk * 2), kdesc + (uint64_t)(kk * 2), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sacc);

    const int kbase = j * FA_BK;
    if (kbase + FA_BK > p.S) {  // ragged last block: keys past the sequence do not exist
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (kbase + 8 * jj + 2 * cq + e >= p.S) {
            sacc[4 * jj + e] = -INFINITY;
            sacc[4 * jj + 2 + e] = -INFINITY;
          }
    }
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(sacc[4 * jj + 2 * h], sacc[4 * jj + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx * c);
      alpha[h] = ex2_approx(m_run[h] - m_new);  // 0 on the first block (m_run = -inf)
      m_run[h] = m_new;
      float l = 0.f;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float pr = ex2_approx(fmaf(sacc[4 * jj + 2 * h + e], c, -m_new));
          sacc[4 * jj + 2 * h + e] = pr;
          l += pr;
        }
      }
      l_run[h] = l_run[h] * alpha[h] + l;
    }
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      o[4 * jj] *= alpha[0];
      o[4 * jj + 1] *= alpha[0];
      o[4 * jj + 2] *= alpha[1];
      o[4 * jj + 3] *= alpha[1];
    }
    // P as the A operand of m64k16: the accumulator layout of two 8-column blocks is the A fragment layout
    uint32_t pa[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      pa[kk][0] = pack_bf16x2(sacc[8 * kk + 0], sacc[8 * kk + 1]);
      pa[kk][1] = pack_bf16x2(sacc[8 * kk + 2], sacc[8 * kk + 3]);
      pa[kk][2] = pack_bf16x2(sacc[8 * kk + 4], sacc[8 * kk + 5]);
      pa[kk][3] = pack_bf16x2(sacc[8 * kk + 6], sacc[8 * kk + 7]);
    }
    const uint64_t vdesc = smem_desc_mn_sw128(sk + FA_KV_TILE_BYTES);
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)  // 16 keys = 16 rows of V = 2048 B (+128 in the address field)
      Wgmma<64>::rs_tb(o, pa[kk], vdesc + (uint64_t)(kk * 128), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[st]);
  }

  // epilogue: O / l -> bf16
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const int qrow = q0 + 64 * cw + 16 * wl + rq + 8 * h;
    if (qrow < p.S) {
      __nv_bfloat16* dst = p.out + ((int64_t)n * p.S + qrow) * p.ldo + head * FA_D + 2 * cq;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    }
  }
}

// Kept for the C ABI: the sm_90 kernel has a single softmax organisation; the value is recorded and reported only.
static int g_fa_variant = 4;

}  // namespace b200

extern "C" int b200svd_flash_attn_variant(int v) {
  const int prev = b200::g_fa_variant;
  if (v >= 3 && v <= 5) b200::g_fa_variant = v;
  return prev;
}

// qkv: [(n s), ldqkv] bf16 with columns [q | k | v], each C = heads*64 wide; out: [(n s), ldo] bf16 (C columns).
extern "C" int b200svd_flash_attn(const void* qkv, int64_t ldqkv, void* out, int64_t ldo, int n, int s, int heads,
                                  float scale, void* stream) {
  using namespace b200;
  if (ldqkv % 8 || ldo % 8) {
    set_error("flash_attn: leading dims must be multiples of 8");
    return 1;
  }
  if ((reinterpret_cast<uintptr_t>(out) & 15) != 0) {  // the epilogue stores 4-byte words from a 16-byte base
    set_error("flash_attn: out must be 16-byte aligned");
    return 1;
  }
  const int C = heads * FA_D;
  CUtensorMap tm;
  uint64_t dims[3] = {(uint64_t)3 * C, (uint64_t)s, (uint64_t)n};
  uint64_t strides[2] = {(uint64_t)ldqkv * 2, (uint64_t)ldqkv * 2 * (uint64_t)s};
  uint32_t box[3] = {64, 128, 1};
  if (encode_tmap_bf16(&tm, qkv, 3, dims, strides, box)) return 1;
  static bool attr_set[B200_MAX_DEVICES] = {};
  const int slot = dev_slot();
  if (!attr_set[slot]) {
    cudaError_t e = cudaFuncSetAttribute(flash_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FA_SMEM_BYTES);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(flash_attn)");
    attr_set[slot] = true;
  }
  FaParams p;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;
  p.S = s;
  p.heads = heads;
  p.C = C;
  p.scale_log2 = scale * 1.4426950408889634f;
  dim3 grid((s + FA_BQ - 1) / FA_BQ, heads, n);
  flash_attn_kernel<<<grid, FA_THREADS, FA_SMEM_BYTES, reinterpret_cast<cudaStream_t>(stream)>>>(tm, p);
  B200_CHECK_LAUNCH("flash_attn");
  return 0;
}
