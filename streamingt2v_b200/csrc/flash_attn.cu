// FlashAttention forward for sm_90a, head dim D = 64 or 80: wgmma for S = Q K^T and O += P V with the accumulators in
// registers, TMA-fed Q/K/V tiles read straight from the fused QKV projection output [(n s), ldqkv] (no head split /
// transpose in HBM).
//
// D = 64 replaces the spatial self-attention core of BasicTransformerBlock.attn1
// (reference code/models/svd/sgm/modules/attention.py:320-351 SDPA / :427-446 xformers), batch = frames,
// heads = C/64, sequence = H*W.
// D = 80 is the self-attention of the OpenCLIP ViT-H/14 image tower (open_clip transformer.py ResidualAttentionBlock ->
// nn.MultiheadAttention, width 1280, 16 heads; called per chunk by the SVD conditioner, reference
// code/models/svd/sgm/modules/encoders/modules.py:697-729), batch = images, sequence = 257 tokens.
//
// A head row wider than the 128-byte swizzle atom is split: every 128-row Q/K/V tile is loaded as
//   columns  0..63   SWIZZLE_128B box (128 B rows)   -> 4 k16 steps of Q K^T, the n64 part of P V
//   columns 64..D-1  SWIZZLE_32B  box ( 32 B rows)   -> the 5th k16 step of Q K^T, the n16 part of P V (D = 80 only)
//
// CTA = one 128-row query tile of one (frame, head), three warpgroups:
//   warpgroup 0      TMA producer (Q once; K/V ring of FA_KV_STAGES 128-key blocks)
//   warpgroups 1, 2  64 query rows each.  Per key block:
//     S[64x128] = Q K_j^T            D/16 x wgmma m64n128k16, both operands from shared memory
//     online softmax in registers    row max over the quad of threads sharing a row, P = exp2(S*c - m), O and l
//                                    rescaled when the running max rises; keys past the sequence are -inf
//     O[64xD] += P V_j               8 x wgmma m64n64k16 (+ m64n16k16 for the tail), A = P (bf16) from registers,
//                                    B = V MN-major from smem
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
constexpr int FA_KV_STAGES = 4;
constexpr int FA_THREADS = 3 * 128;
constexpr int FA_WIDE_BYTES = 128 * 64 * 2;  // 16 KB: columns 0..63 of a 128-row tile (SW128)

// One 128-row Q, K or V tile is [wide 16 KB | tail 128 x (D - 64) columns (SW32)].
constexpr int fa_tile_bytes(int D) { return 128 * D * 2; }
constexpr int fa_smem_bytes(int D) { return fa_tile_bytes(D) + FA_KV_STAGES * 2 * fa_tile_bytes(D) + 256; }

struct FaParams {
  __nv_bfloat16* out;
  int64_t ldo;
  int S, C;
  float scale_log2;
};

// The kernel body for head dim D; tmT maps the tail columns (SWIZZLE_32B box) and is not read when D = 64.  The maps
// are the kernels' __grid_constant__ parameters: TMA needs their parameter-space addresses.
template <int D>
__device__ __forceinline__ void flash_attn_body(const CUtensorMap& tmW, const CUtensorMap& tmT, const FaParams& p) {
  // The tail is one 16-column SWIZZLE_32B box: one k16 step of Q K^T and one m64n16 wgmma of P V.
  static_assert(D == 64 || D == 80, "head dim 64, or 64 + one 16-column tail");
  constexpr int TAIL = D - 64;
  constexpr int TAIL_BYTES = 128 * TAIL * 2;
  constexpr int TILE_BYTES = fa_tile_bytes(D);

  extern __shared__ __align__(1024) uint8_t smem[];  // SWIZZLE_128B tiles need 1024-byte alignment
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + TILE_BYTES;  // stage s: K tile at sKV + s*2*TILE_BYTES, V tile at +TILE_BYTES
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + FA_KV_STAGES * 2 * TILE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                 // [FA_KV_STAGES]
  uint64_t* kv_empty = kv_full + FA_KV_STAGES;  // [FA_KV_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int head = blockIdx.y, n = blockIdx.z;
  const int q0 = blockIdx.x * FA_BQ;
  const int nkb = (p.S + FA_BK - 1) / FA_BK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmW);
    if constexpr (TAIL > 0) prefetch_tmap(&tmT);
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
      const int col = head * D;
      mbar_expect_tx(q_full, TILE_BYTES);
      tma_load_3d(sQ, &tmW, q_full, col, q0, n);
      if constexpr (TAIL > 0) tma_load_3d(sQ + FA_WIDE_BYTES, &tmT, q_full, col + 64, q0, n);
      for (int j = 0; j < nkb; ++j) {
        const int s = j % FA_KV_STAGES;
        mbar_wait_parked(&kv_empty[s], ((j / FA_KV_STAGES) & 1) ^ 1);
        uint8_t* sk = sKV + s * 2 * TILE_BYTES;
        uint8_t* sv = sk + TILE_BYTES;
        mbar_expect_tx(&kv_full[s], 2 * TILE_BYTES);
        tma_load_3d(sk, &tmW, &kv_full[s], p.C + col, j * FA_BK, n);
        if constexpr (TAIL > 0) tma_load_3d(sk + FA_WIDE_BYTES, &tmT, &kv_full[s], p.C + col + 64, j * FA_BK, n);
        tma_load_3d(sv, &tmW, &kv_full[s], 2 * p.C + col, j * FA_BK, n);
        if constexpr (TAIL > 0) tma_load_3d(sv + FA_WIDE_BYTES, &tmT, &kv_full[s], 2 * p.C + col + 64, j * FA_BK, n);
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");

  // ===================== consumer warpgroups: rows 64 cw + 16 wl + rq (+ 8) of the tile =====================
  const int cw = wg - 1, wl = warp & 3;
  const int rq = lane >> 2, cq = lane & 3;
  const float c = p.scale_log2;
  const uint64_t qdesc = smem_desc_k_sw128(smem_u32(sQ + cw * (FA_WIDE_BYTES / 2)));
  const uint64_t qdesc_t = smem_desc_k_sw32(smem_u32(sQ + FA_WIDE_BYTES + cw * (TAIL_BYTES / 2)));
  float o[32];                         // output columns 0..63
  float ot[TAIL > 0 ? TAIL / 2 : 1];   // output columns 64..D-1
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
#pragma unroll
  for (int i = 0; i < TAIL / 2; ++i) ot[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};  // running max, already scaled by c (log2 units)
  float l_run[2] = {0.f, 0.f};              // this thread's part of the row sum
  mbar_wait(q_full, 0);

  for (int j = 0; j < nkb; ++j) {
    const int st = j % FA_KV_STAGES;
    mbar_wait(&kv_full[st], (j / FA_KV_STAGES) & 1);
    const uint32_t sk = smem_u32(sKV + st * 2 * TILE_BYTES);
    const uint32_t sv = sk + TILE_BYTES;
    float sacc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) sacc[i] = 0.f;
    wgmma_fence_regs(sacc);
    wgmma_fence();
    const uint64_t kdesc = smem_desc_k_sw128(sk);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) Wgmma<128>::ss(sacc, qdesc + (uint64_t)(kk * 2), kdesc + (uint64_t)(kk * 2), 1u);
    if constexpr (TAIL > 0) Wgmma<128>::ss(sacc, qdesc_t, smem_desc_k_sw32(sk + FA_WIDE_BYTES), 1u);
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
#pragma unroll
    for (int jj = 0; jj < TAIL / 8; ++jj) {
      ot[4 * jj] *= alpha[0];
      ot[4 * jj + 1] *= alpha[0];
      ot[4 * jj + 2] *= alpha[1];
      ot[4 * jj + 3] *= alpha[1];
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
    const uint64_t vdesc = smem_desc_mn_sw128(sv);
    const uint64_t vdesc_t = smem_desc_mn_sw32(sv + FA_WIDE_BYTES);
    wgmma_fence_regs(o);
    if constexpr (TAIL > 0) wgmma_fence_regs(ot);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      // 16 keys = 16 rows of V: 2048 B of the wide box (+128 in the address field), 512 B of the tail box (+32)
      Wgmma<64>::rs_tb(o, pa[kk], vdesc + (uint64_t)(kk * 128), 1u);
      if constexpr (TAIL > 0) Wgmma<TAIL>::rs_tb(ot, pa[kk], vdesc_t + (uint64_t)(kk * 32), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if constexpr (TAIL > 0) wgmma_fence_regs(ot);
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
      __nv_bfloat16* dst = p.out + ((int64_t)n * p.S + qrow) * p.ldo + head * D + 2 * cq;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
#pragma unroll
      for (int jj = 0; jj < TAIL / 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 64 + 8 * jj) =
            pack_bf16x2(ot[4 * jj + 2 * h] * inv, ot[4 * jj + 2 * h + 1] * inv);
    }
  }
}

// One named entry point per head dim, so that SASS listings and profiler traces tell the two apart.
__global__ void __launch_bounds__(FA_THREADS, 1)
flash_attn_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmT, const FaParams p) {
  flash_attn_body<64>(tmW, tmT, p);
}

__global__ void __launch_bounds__(FA_THREADS, 1)
flash_attn_d80_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmT,
                      const FaParams p) {
  flash_attn_body<80>(tmW, tmT, p);
}

// qkv: [(n s), ldqkv] bf16 with columns [q | k | v], each C = heads*D wide; out: [(n s), ldo] bf16 (C columns).
// Every argument is checked before any tensor-map encode or launch.
template <int D>
static int flash_attn_launch(const char* name, const void* qkv, int64_t ldqkv, void* out, int64_t ldo, int n, int s,
                             int heads, float scale, void* stream) {
  if (n <= 0 || s <= 0 || heads <= 0 || n > 65535 || heads > 65535) {  // grid.y, grid.z
    set_error("%s: need n, s, heads >= 1 (n, heads <= 65535), got n=%d s=%d heads=%d", name, n, s, heads);
    return 1;
  }
  if (ldqkv % 8 || ldo % 8) {
    set_error("%s: leading dims must be multiples of 8", name);
    return 1;
  }
  const int C = heads * D;
  if (ldqkv < 3 * (int64_t)C || ldo < (int64_t)C) {
    set_error("%s: ldqkv (%lld) must be >= 3*heads*%d and ldo (%lld) >= heads*%d (%d)", name, (long long)ldqkv, D,
              (long long)ldo, D, C);
    return 1;
  }
  // TMA reads qkv in 16-byte units; the epilogue stores 4-byte words from a 16-byte base
  if ((reinterpret_cast<uintptr_t>(qkv) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 15) != 0) {
    set_error("%s: qkv and out must be 16-byte aligned", name);
    return 1;
  }
  CUtensorMap tmW, tmT = {};
  uint64_t dims[3] = {(uint64_t)3 * C, (uint64_t)s, (uint64_t)n};
  uint64_t strides[2] = {(uint64_t)ldqkv * 2, (uint64_t)ldqkv * 2 * (uint64_t)s};
  uint32_t box_w[3] = {64, 128, 1};
  if (encode_tmap_bf16(&tmW, qkv, 3, dims, strides, box_w)) return 1;
  if constexpr (D > 64) {
    uint32_t box_t[3] = {D - 64, 128, 1};
    if (encode_tmap_bf16_sw32(&tmT, qkv, 3, dims, strides, box_t)) return 1;
  }
  auto* kernel = D == 64 ? flash_attn_kernel : flash_attn_d80_kernel;
  static bool attr_set[B200_MAX_DEVICES] = {};
  const int slot = dev_slot();
  if (!attr_set[slot]) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, fa_smem_bytes(D));
    if (e != cudaSuccess) return cuda_fail(e, name);
    attr_set[slot] = true;
  }
  FaParams p;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;
  p.S = s;
  p.C = C;
  p.scale_log2 = scale * 1.4426950408889634f;
  dim3 grid((s + FA_BQ - 1) / FA_BQ, heads, n);
  kernel<<<grid, FA_THREADS, fa_smem_bytes(D), reinterpret_cast<cudaStream_t>(stream)>>>(tmW, tmT, p);
  B200_CHECK_LAUNCH(name);
  return 0;
}

// Kept for the C ABI: the sm_90 kernel has a single softmax organisation; the value is recorded and reported only.
static int g_fa_variant = 4;

}  // namespace b200

extern "C" int b200svd_flash_attn_variant(int v) {
  const int prev = b200::g_fa_variant;
  if (v >= 3 && v <= 5) b200::g_fa_variant = v;
  return prev;
}

extern "C" int b200svd_flash_attn(const void* qkv, int64_t ldqkv, void* out, int64_t ldo, int n, int s, int heads,
                                  float scale, void* stream) {
  return b200::flash_attn_launch<64>("flash_attn", qkv, ldqkv, out, ldo, n, s, heads, scale, stream);
}

extern "C" int b200svd_flash_attn_d80(const void* qkv, int64_t ldqkv, void* out, int64_t ldo, int n, int s, int heads,
                                      float scale, void* stream) {
  return b200::flash_attn_launch<80>("flash_attn_d80", qkv, ldqkv, out, ldo, n, s, heads, scale, stream);
}
