// Small-sequence attention (head dim 64): one warp per (batch b, pixel s, head h) problem; every lane owns one
// query row, keys/values of the problem are staged in shared memory and broadcast.  The "(b t) s c -> (b s) t c"
// transposes of the reference never touch HBM: rows are addressed with their native frame stride.
//
// Replaces:
//   temporal self-attention   VideoTransformerBlock attn1 (reference code/models/svd/sgm/modules/video_attention.py:145-148)
//                             Lq = Lk = T (25), K/V per pixel
//   CAM cross-frame attention CrossAttention.forward (code/models/cam/conditioning.py:65-68), Lq = T, Lk = 7, K/V per pixel
//   temporal cross-attention  VideoTransformerBlock attn2 with APM tokens (video_attention.py:150-154), Lk = 17, K/V per batch
// Row addressing (elements): q/out row of (b, i, s) = ((b*Lq + i)*S + s); k/v row of (b, j, s) = ((b*Lk + j)*Skv + s*kv_pp)
// with Skv = S, kv_pp = 1 (per-pixel K/V) or Skv = 1, kv_pp = 0 (K/V shared by all pixels of a batch).
#include <cuda_bf16.h>
#include <math.h>

#include "../../include/b200svd.h"
#include "common.h"
#include "ptx.cuh"

namespace b200 {

constexpr int SA_MAXL = 32;
constexpr int SA_WARPS = 4;

struct SmallAttnParams {
  const __nv_bfloat16* q;
  const __nv_bfloat16* k;
  const __nv_bfloat16* v;
  __nv_bfloat16* o;
  int64_t ldq, ldk, ldv, ldo;
  int B, S, H, Lq, Lk;
  int Skv, kv_pp;
  float scale_log2;  // softmax scale * log2(e)
  int64_t total;     // B*S*H problems
};

__global__ void __launch_bounds__(SA_WARPS * 32) small_attn_kernel(const SmallAttnParams p) {
  __shared__ __align__(16) __nv_bfloat16 ks[SA_WARPS][SA_MAXL][64];
  __shared__ __align__(16) __nv_bfloat16 vs[SA_WARPS][SA_MAXL][64];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t prob = (int64_t)blockIdx.x * SA_WARPS + warp;
  if (prob >= p.total) return;
  // problem order: head fastest, then pixel, then batch -> neighbouring warps read neighbouring 128-byte segments
  const int h = (int)(prob % p.H);
  const int64_t bs = prob / p.H;
  const int s = (int)(bs % p.S);
  const int b = (int)(bs / p.S);

  // stage K, V (Lk rows x 128 B) with cp.async so that the Q loads below overlap them:
  // lane -> (row = lane/8 + 4*it, 16-byte chunk = lane%8)
  {
    const int chunk = lane & 7;
    for (int j = lane >> 3; j < p.Lk; j += 4) {
      const int64_t row = ((int64_t)b * p.Lk + j) * p.Skv + (int64_t)s * p.kv_pp;
      const void* gk = reinterpret_cast<const uint4*>(p.k + row * p.ldk + h * 64) + chunk;
      const void* gv = reinterpret_cast<const uint4*>(p.v + row * p.ldv + h * 64) + chunk;
      const uint32_t sk = smem_u32(reinterpret_cast<uint4*>(&ks[warp][j][0]) + chunk);
      const uint32_t sv = smem_u32(reinterpret_cast<uint4*>(&vs[warp][j][0]) + chunk);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sk), "l"(gk) : "memory");
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sv), "l"(gv) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  const int qi = lane < p.Lq ? lane : p.Lq - 1;  // idle lanes shadow the last query (no divergence on the loads)
  const int64_t qrow = ((int64_t)b * p.Lq + qi) * p.S + s;
  uint32_t qp[32];
  {
    const uint4* qsrc = reinterpret_cast<const uint4*>(p.q + qrow * p.ldq + h * 64);
    uint4 u[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) u[c] = __ldg(qsrc + c);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      qp[4 * c] = u[c].x;
      qp[4 * c + 1] = u[c].y;
      qp[4 * c + 2] = u[c].z;
      qp[4 * c + 3] = u[c].w;
    }
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncwarp();
  if (lane >= p.Lq) return;

  float sc[SA_MAXL];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < SA_MAXL; ++j) {
    if (j < p.Lk) {
      float acc = 0.f;
      const uint4* kr = reinterpret_cast<const uint4*>(&ks[warp][j][0]);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint4 u = kr[c];
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          acc = fmaf(bf16_lo(qp[4 * c + e]), bf16_lo(w[e]), acc);
          acc = fmaf(bf16_hi(qp[4 * c + e]), bf16_hi(w[e]), acc);
        }
      }
      sc[j] = acc * p.scale_log2;
      mx = fmaxf(mx, sc[j]);
    } else {
      sc[j] = -INFINITY;
    }
  }
  float den = 0.f;
#pragma unroll
  for (int j = 0; j < SA_MAXL; ++j) {
    const float e = (j < p.Lk) ? exp2f(sc[j] - mx) : 0.f;
    sc[j] = e;
    den += e;
  }
  const float inv = 1.0f / den;
  float o[64];
#pragma unroll
  for (int d = 0; d < 64; ++d) o[d] = 0.f;
#pragma unroll
  for (int j = 0; j < SA_MAXL; ++j) {
    if (j < p.Lk) {
      const float pj = sc[j] * inv;
      const uint4* vr = reinterpret_cast<const uint4*>(&vs[warp][j][0]);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint4 u = vr[c];
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          o[8 * c + 2 * e] = fmaf(pj, bf16_lo(w[e]), o[8 * c + 2 * e]);
          o[8 * c + 2 * e + 1] = fmaf(pj, bf16_hi(w[e]), o[8 * c + 2 * e + 1]);
        }
      }
    }
  }
  uint4* dst = reinterpret_cast<uint4*>(p.o + qrow * p.ldo + h * 64);
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    dst[c] = make_uint4(pack_bf16x2(o[8 * c], o[8 * c + 1]), pack_bf16x2(o[8 * c + 2], o[8 * c + 3]),
                        pack_bf16x2(o[8 * c + 4], o[8 * c + 5]), pack_bf16x2(o[8 * c + 6], o[8 * c + 7]));
  }
}

}  // namespace b200

extern "C" int b200svd_small_attn(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                  void* o, int64_t ldo, int b, int s, int heads, int lq, int lk, int kv_per_pixel,
                                  float scale, void* stream) {
  using namespace b200;
  if (lq < 1 || lq > SA_MAXL || lk < 1 || lk > SA_MAXL) {
    set_error("small_attn: Lq=%d / Lk=%d must be in 1..%d", lq, lk, SA_MAXL);
    return 1;
  }
  if (ldq % 8 || ldk % 8 || ldv % 8 || ldo % 8) {
    set_error("small_attn: leading dims must be multiples of 8");
    return 1;
  }
  for (const void* t : {q, k, v, static_cast<const void*>(o)}) {  // 16-byte cp.async and uint4 loads / stores
    if ((reinterpret_cast<uintptr_t>(t) & 15) != 0) {
      set_error("small_attn: q/k/v/o must be 16-byte aligned");
      return 1;
    }
  }
  SmallAttnParams p;
  p.q = reinterpret_cast<const __nv_bfloat16*>(q);
  p.k = reinterpret_cast<const __nv_bfloat16*>(k);
  p.v = reinterpret_cast<const __nv_bfloat16*>(v);
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.ldq = ldq;
  p.ldk = ldk;
  p.ldv = ldv;
  p.ldo = ldo;
  p.B = b;
  p.S = s;
  p.H = heads;
  p.Lq = lq;
  p.Lk = lk;
  p.Skv = kv_per_pixel ? s : 1;
  p.kv_pp = kv_per_pixel ? 1 : 0;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.total = (int64_t)b * s * heads;
  const int64_t blocks = (p.total + SA_WARPS - 1) / SA_WARPS;
  if (blocks <= 0 || blocks > 0x7FFFFFFF) {
    set_error("small_attn: bad problem count");
    return 1;
  }
  small_attn_kernel<<<(unsigned)blocks, SA_WARPS * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  B200_CHECK_LAUNCH("small_attn");
  return 0;
}
