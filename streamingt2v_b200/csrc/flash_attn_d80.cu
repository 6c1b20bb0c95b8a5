// FlashAttention forward for sm_90a, head dim 80: the self-attention of the OpenCLIP ViT-H/14 image tower
// (open_clip transformer.py ResidualAttentionBlock -> nn.MultiheadAttention, width 1280, 16 heads; called per chunk by
// the SVD conditioner, reference code/models/svd/sgm/modules/encoders/modules.py:697-729).  Same contract and pipeline
// as the head-dim-64 kernel (flash_attn.cu): wgmma for S = Q K^T and O += P V with the accumulators in registers,
// TMA-fed Q/K/V tiles read straight from the fused in_proj output [(n s), ldqkv] (no head split / transpose in HBM).
//
// A 160-byte head row does not fit one 128-byte swizzle atom, so every 128-row Q/K/V tile is loaded as two TMA boxes:
//   columns  0..63   SWIZZLE_128B box (128 B rows)   -> 4 k16 steps of Q K^T, the n64 half of P V
//   columns 64..79   SWIZZLE_32B  box ( 32 B rows)   -> the 5th k16 step of Q K^T, the n16 half of P V
//
// CTA = one 128-row query tile of one (image, head), three warpgroups:
//   warpgroup 0      TMA producer (Q once; K/V ring of F8_KV_STAGES 128-key blocks)
//   warpgroups 1, 2  64 query rows each.  Per key block:
//     S[64x128] = Q K_j^T            5 x wgmma m64n128k16, both operands from shared memory
//     online softmax in registers    as flash_attn.cu; keys past the sequence (ragged last block) are -inf
//     O[64x80] += P V_j              8 x (wgmma m64n64k16 + m64n16k16), A = P (bf16) from registers, B = V MN-major
#include <cuda.h>
#include <cuda_bf16.h>
#include <math.h>

#include "../../include/b200svd.h"
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace b200 {

constexpr int F8_BQ = 128;
constexpr int F8_BK = 128;
constexpr int F8_D = 80;
constexpr int F8_KV_STAGES = 4;
constexpr int F8_WIDE_BYTES = 128 * 64 * 2;                  // 16 KB: columns 0..63 of a 128-row tile (SW128)
constexpr int F8_NARROW_BYTES = 128 * 16 * 2;                // 4 KB: columns 64..79 (SW32)
constexpr int F8_TILE_BYTES = F8_WIDE_BYTES + F8_NARROW_BYTES;  // 20 KB per Q, K or V tile
constexpr int F8_SMEM_BYTES = F8_TILE_BYTES + F8_KV_STAGES * 2 * F8_TILE_BYTES + 256;
constexpr int F8_THREADS = 3 * 128;

struct Fa80Params {
  __nv_bfloat16* out;
  int64_t ldo;
  int S, C;
  float scale_log2;
};

__global__ void __launch_bounds__(F8_THREADS, 1)
flash_attn_d80_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmN,
                      const Fa80Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];  // SWIZZLE_128B tiles need 1024-byte alignment
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sQ = smem;                 // [wide 16 KB | narrow 4 KB]
  uint8_t* sKV = sQ + F8_TILE_BYTES;  // stage s: K tile at sKV + s*40K, V tile at +20K
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + F8_KV_STAGES * 2 * F8_TILE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                 // [F8_KV_STAGES]
  uint64_t* kv_empty = kv_full + F8_KV_STAGES;  // [F8_KV_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int head = blockIdx.y, n = blockIdx.z;
  const int q0 = blockIdx.x * F8_BQ;
  const int nkb = (p.S + F8_BK - 1) / F8_BK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmW);
    prefetch_tmap(&tmN);
    mbar_init(q_full, 1);
    for (int s = 0; s < F8_KV_STAGES; ++s) {
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
      const int cq = head * F8_D;
      mbar_expect_tx(q_full, F8_TILE_BYTES);
      tma_load_3d(sQ, &tmW, q_full, cq, q0, n);
      tma_load_3d(sQ + F8_WIDE_BYTES, &tmN, q_full, cq + 64, q0, n);
      for (int j = 0; j < nkb; ++j) {
        const int s = j % F8_KV_STAGES;
        mbar_wait_parked(&kv_empty[s], ((j / F8_KV_STAGES) & 1) ^ 1);
        uint8_t* sk = sKV + s * 2 * F8_TILE_BYTES;
        uint8_t* sv = sk + F8_TILE_BYTES;
        mbar_expect_tx(&kv_full[s], 2 * F8_TILE_BYTES);
        tma_load_3d(sk, &tmW, &kv_full[s], p.C + cq, j * F8_BK, n);
        tma_load_3d(sk + F8_WIDE_BYTES, &tmN, &kv_full[s], p.C + cq + 64, j * F8_BK, n);
        tma_load_3d(sv, &tmW, &kv_full[s], 2 * p.C + cq, j * F8_BK, n);
        tma_load_3d(sv + F8_WIDE_BYTES, &tmN, &kv_full[s], 2 * p.C + cq + 64, j * F8_BK, n);
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");

  // ===================== consumer warpgroups: rows 64 cw + 16 wl + rq (+ 8) of the tile =====================
  const int cw = wg - 1, wl = warp & 3;
  const int rq = lane >> 2, cq = lane & 3;
  const float c = p.scale_log2;
  const uint64_t qdesc_w = smem_desc_k_sw128(smem_u32(sQ + cw * (F8_WIDE_BYTES / 2)));
  const uint64_t qdesc_n = smem_desc_k_sw32(smem_u32(sQ + F8_WIDE_BYTES + cw * (F8_NARROW_BYTES / 2)));
  float o[32];  // output columns 0..63
  float o16[8];  // output columns 64..79
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) o16[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};  // running max, already scaled by c (log2 units)
  float l_run[2] = {0.f, 0.f};              // this thread's part of the row sum
  mbar_wait(q_full, 0);

  for (int j = 0; j < nkb; ++j) {
    const int st = j % F8_KV_STAGES;
    mbar_wait(&kv_full[st], (j / F8_KV_STAGES) & 1);
    const uint32_t sk = smem_u32(sKV + st * 2 * F8_TILE_BYTES);
    const uint32_t sv = sk + F8_TILE_BYTES;
    float sacc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) sacc[i] = 0.f;
    wgmma_fence_regs(sacc);
    wgmma_fence();
    const uint64_t kdesc_w = smem_desc_k_sw128(sk);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      Wgmma<128>::ss(sacc, qdesc_w + (uint64_t)(kk * 2), kdesc_w + (uint64_t)(kk * 2), 1u);
    Wgmma<128>::ss(sacc, qdesc_n, smem_desc_k_sw32(sk + F8_WIDE_BYTES), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sacc);

    const int kbase = j * F8_BK;
    if (kbase + F8_BK > p.S) {  // ragged last block: keys past the sequence do not exist
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
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      o16[4 * jj] *= alpha[0];
      o16[4 * jj + 1] *= alpha[0];
      o16[4 * jj + 2] *= alpha[1];
      o16[4 * jj + 3] *= alpha[1];
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
    const uint64_t vdesc_w = smem_desc_mn_sw128(sv);
    const uint64_t vdesc_n = smem_desc_mn_sw32(sv + F8_WIDE_BYTES);
    wgmma_fence_regs(o);
    wgmma_fence_regs(o16);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      // 16 keys = 16 rows of V: 2048 B of the wide box (+128 in the address field), 512 B of the narrow one (+32)
      Wgmma<64>::rs_tb(o, pa[kk], vdesc_w + (uint64_t)(kk * 128), 1u);
      Wgmma<16>::rs_tb(o16, pa[kk], vdesc_n + (uint64_t)(kk * 32), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    wgmma_fence_regs(o16);
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
      __nv_bfloat16* dst = p.out + ((int64_t)n * p.S + qrow) * p.ldo + head * F8_D + 2 * cq;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
#pragma unroll
      for (int jj = 0; jj < 2; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 64 + 8 * jj) =
            pack_bf16x2(o16[4 * jj + 2 * h] * inv, o16[4 * jj + 2 * h + 1] * inv);
    }
  }
}

}  // namespace b200

// qkv: [(n s), ldqkv] bf16 with columns [q | k | v], each C = heads*80 wide; out: [(n s), ldo] bf16 (C columns).
extern "C" int b200svd_flash_attn_d80(const void* qkv, int64_t ldqkv, void* out, int64_t ldo, int n, int s, int heads,
                                      float scale, void* stream) {
  using namespace b200;
  if (n <= 0 || s <= 0 || heads <= 0 || n > 65535 || heads > 65535) {
    set_error("flash_attn_d80: need n, s, heads >= 1 (n, heads <= 65535), got n=%d s=%d heads=%d", n, s, heads);
    return 1;
  }
  if (ldqkv % 8 || ldo % 8) {
    set_error("flash_attn_d80: leading dims must be multiples of 8");
    return 1;
  }
  const int C = heads * F8_D;
  if (ldqkv < 3 * (int64_t)C || ldo < (int64_t)C) {
    set_error("flash_attn_d80: ldqkv (%lld) must be >= 3*heads*80 and ldo (%lld) >= heads*80 (%d)", (long long)ldqkv,
              (long long)ldo, C);
    return 1;
  }
  if ((reinterpret_cast<uintptr_t>(qkv) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 15) != 0) {
    set_error("flash_attn_d80: qkv and out must be 16-byte aligned");
    return 1;
  }
  CUtensorMap tmW, tmN;
  uint64_t dims[3] = {(uint64_t)3 * C, (uint64_t)s, (uint64_t)n};
  uint64_t strides[2] = {(uint64_t)ldqkv * 2, (uint64_t)ldqkv * 2 * (uint64_t)s};
  uint32_t box_w[3] = {64, 128, 1};
  uint32_t box_n[3] = {16, 128, 1};
  if (encode_tmap_bf16(&tmW, qkv, 3, dims, strides, box_w)) return 1;
  if (encode_tmap_bf16_sw32(&tmN, qkv, 3, dims, strides, box_n)) return 1;
  static bool attr_set[B200_MAX_DEVICES] = {};
  const int slot = dev_slot();
  if (!attr_set[slot]) {
    cudaError_t e =
        cudaFuncSetAttribute(flash_attn_d80_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, F8_SMEM_BYTES);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(flash_attn_d80)");
    attr_set[slot] = true;
  }
  Fa80Params p;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;
  p.S = s;
  p.C = C;
  p.scale_log2 = scale * 1.4426950408889634f;
  dim3 grid((s + F8_BQ - 1) / F8_BQ, heads, n);
  flash_attn_d80_kernel<<<grid, F8_THREADS, F8_SMEM_BYTES, reinterpret_cast<cudaStream_t>(stream)>>>(tmW, tmN, p);
  B200_CHECK_LAUNCH("flash_attn_d80");
  return 0;
}
