// Per-pixel attention over frames on the tensor cores (head dim 64): temporal self-attention (Lq = Lk = T) and
// CAM cross-frame attention (Lq = T, Lk = number of control frames), K/V per pixel.
//
// Replaces VideoTransformerBlock.attn1 (reference code/models/svd/sgm/modules/video_attention.py:145-148, after the
// "(b t) s c -> (b s) t c" transpose of :131) and the CAM CrossAttention core (code/models/cam/conditioning.py:65-68).
//
// One CTA = 4 pixels x 1 head, two warpgroups of two pixels each.  The 2 x 32 (frames padded to 32) query rows of a
// warpgroup form one 64-row wgmma tile, the same pixels' 2 x 32 key rows one 64-key block; S = Q K^T is computed for
// the whole block by wgmma and only the block diagonal (same pixel) is kept.  The frame-strided rows of a pixel are
// gathered by TMA (box = 64 channels x 1 pixel x 32 frames; frames beyond L are zero-filled), so the reference's
// transpose never exists in HBM.  Softmax and P stay in registers; P is the register A operand of O = P V.
#include <cuda.h>
#include <cuda_bf16.h>
#include <math.h>

#include "../../include/b200svd.h"
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace b200 {

constexpr int PA_TILE_BYTES = 128 * 64 * 2;  // 16 KB: Q, K, V tiles of 4 pixels
constexpr int PA_SMEM_BYTES = 3 * PA_TILE_BYTES + 128;
constexpr int PA_THREADS = 2 * 128;

struct PaParams {
  __nv_bfloat16* out;
  int64_t ldo;
  int S, Lq, Lk;
  float scale_log2;
};

__global__ void __launch_bounds__(PA_THREADS)
pixel_attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                  const __grid_constant__ CUtensorMap tmV, const PaParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + PA_TILE_BYTES;
  uint8_t* sV = sK + PA_TILE_BYTES;
  uint64_t* ld_full = reinterpret_cast<uint64_t*>(sV + PA_TILE_BYTES);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pix0 = blockIdx.x * 4, head = blockIdx.y, b = blockIdx.z;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmK);
    prefetch_tmap(&tmV);
    mbar_init(ld_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // TMA: 4 pixels x {Q, K, V}; each box = 64 channels x 1 pixel x 32 frames -> 4 KB, rows ordered (pixel, frame)
    mbar_expect_tx(ld_full, 3 * PA_TILE_BYTES);
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      tma_load_4d(sQ + px * 4096, &tmQ, ld_full, head * 64, pix0 + px, 0, b);
      tma_load_4d(sK + px * 4096, &tmK, ld_full, head * 64, pix0 + px, 0, b);
      tma_load_4d(sV + px * 4096, &tmV, ld_full, head * 64, pix0 + px, 0, b);
    }
  }
  // warpgroup cw: pixels 2 cw, 2 cw + 1 of the CTA; warp wl: 16 query rows of pixel wl / 2
  const int cw = warp >> 2, wl = warp & 3;
  const int rq = lane >> 2, cq = lane & 3;
  const int wpix = wl >> 1;  // pixel of this warp's rows inside the warpgroup
  mbar_wait(ld_full, 0);

  float sacc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) sacc[i] = 0.f;
  const uint64_t qdesc = smem_desc_k_sw128(smem_u32(sQ + cw * 8192));
  const uint64_t kdesc = smem_desc_k_sw128(smem_u32(sK + cw * 8192));
  wgmma_fence_regs(sacc);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) Wgmma<64>::ss(sacc, qdesc + (uint64_t)(kk * 2), kdesc + (uint64_t)(kk * 2), 1u);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(sacc);

  // keep the block diagonal: key column 8 jj + 2 cq + e belongs to pixel jj / 4, frame (8 jj + 2 cq + e) % 32
  uint32_t pa[4][4];
  float inv[2];
  {
    float pr[32];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if ((jj >> 2) == wpix && ((8 * jj + 2 * cq + e) & 31) < p.Lk) mx = fmaxf(mx, sacc[4 * jj + 2 * h + e]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mb = mx * p.scale_log2;
      float l = 0.f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const bool keep = (jj >> 2) == wpix && ((8 * jj + 2 * cq + e) & 31) < p.Lk;
          const float v = keep ? ex2_approx(fmaf(sacc[4 * jj + 2 * h + e], p.scale_log2, -mb)) : 0.f;
          pr[4 * jj + 2 * h + e] = v;
          l += v;
        }
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      inv[h] = 1.0f / l;
    }
    // normalised probabilities as the A operand of m64k16 (accumulator layout of two 8-column blocks)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      pa[kk][0] = pack_bf16x2(pr[8 * kk + 0] * inv[0], pr[8 * kk + 1] * inv[0]);
      pa[kk][1] = pack_bf16x2(pr[8 * kk + 2] * inv[1], pr[8 * kk + 3] * inv[1]);
      pa[kk][2] = pack_bf16x2(pr[8 * kk + 4] * inv[0], pr[8 * kk + 5] * inv[0]);
      pa[kk][3] = pack_bf16x2(pr[8 * kk + 6] * inv[1], pr[8 * kk + 7] * inv[1]);
    }
  }
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  const uint64_t vdesc = smem_desc_mn_sw128(smem_u32(sV + cw * 8192));
  wgmma_fence_regs(o);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) Wgmma<64>::rs_tb(o, pa[kk], vdesc + (uint64_t)(kk * 128), 1u);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(o);

  const int pix = pix0 + 2 * cw + wpix;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int frame = (16 * wl + rq + 8 * h) & 31;
    if (frame < p.Lq && pix < p.S) {
      __nv_bfloat16* dst = p.out + (((int64_t)b * p.Lq + frame) * p.S + pix) * p.ldo + head * 64 + 2 * cq;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h], o[4 * jj + 2 * h + 1]);
    }
  }
}

// rows (b, l, s) of a [(b l s), ld] matrix with `cols` usable columns -> TMA view (cols, S, L, B), box (64, 1, 32, 1)
static int encode_pixel_view(CUtensorMap* tm, const void* base, int64_t ld, int cols, int b, int s, int l) {
  uint64_t dims[4] = {(uint64_t)cols, (uint64_t)s, (uint64_t)l, (uint64_t)b};
  uint64_t str[3] = {(uint64_t)ld * 2, (uint64_t)ld * 2 * (uint64_t)s, (uint64_t)ld * 2 * (uint64_t)s * (uint64_t)l};
  uint32_t box[4] = {64, 1, 32, 1};
  return encode_tmap_bf16(tm, base, 4, dims, str, box);
}

}  // namespace b200

// q/out rows (b, i < lq, s); k/v rows (b, j < lk, s); head dim 64; lq, lk <= 32.
extern "C" int b200svd_pixel_attn(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                  void* o, int64_t ldo, int b, int s, int heads, int lq, int lk, float scale,
                                  void* stream) {
  using namespace b200;
  if (lq < 1 || lq > 32 || lk < 1 || lk > 32) {
    set_error("pixel_attn: Lq=%d / Lk=%d must be in 1..32", lq, lk);
    return 1;
  }
  if (ldq % 8 || ldk % 8 || ldv % 8 || ldo % 8) {
    set_error("pixel_attn: leading dims must be multiples of 8");
    return 1;
  }
  for (const void* t : {q, k, v, static_cast<const void*>(o)}) {
    if ((reinterpret_cast<uintptr_t>(t) & 15) != 0) {
      set_error("pixel_attn: q/k/v/o must be 16-byte aligned");
      return 1;
    }
  }
  const int C = heads * 64;
  CUtensorMap tmQ, tmK, tmV;
  if (encode_pixel_view(&tmQ, q, ldq, C, b, s, lq)) return 1;
  if (encode_pixel_view(&tmK, k, ldk, C, b, s, lk)) return 1;
  if (encode_pixel_view(&tmV, v, ldv, C, b, s, lk)) return 1;
  static bool attr_set[B200_MAX_DEVICES] = {};
  const int slot = dev_slot();
  if (!attr_set[slot]) {
    cudaError_t e = cudaFuncSetAttribute(pixel_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PA_SMEM_BYTES);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(pixel_attn)");
    attr_set[slot] = true;
  }
  PaParams p;
  p.out = reinterpret_cast<__nv_bfloat16*>(o);
  p.ldo = ldo;
  p.S = s;
  p.Lq = lq;
  p.Lk = lk;
  p.scale_log2 = scale * 1.4426950408889634f;
  dim3 grid((s + 3) / 4, heads, b);
  pixel_attn_kernel<<<grid, PA_THREADS, PA_SMEM_BYTES, reinterpret_cast<cudaStream_t>(stream)>>>(tmQ, tmK, tmV, p);
  B200_CHECK_LAUNCH("pixel_attn");
  return 0;
}
