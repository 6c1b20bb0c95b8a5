// EMA-VFI frame interpolation (the reference's interpolate stage, i2v_enhance/thirdparty/VFI): the kernels of the
// network that are not GEMMs or LayerNorms.  Everything here is bandwidth- or latency-bound CUDA-core code.
//
//   window_attn   InterFrameAttention on 7x7 windows (feature_extractor.py:146-172) with the window partition, the
//                 centre padding, the shift roll and the frame pairing of MotionFormerBlock.forward (:213-277) done
//                 by addressing.  One block per (window, head, image).  Per block QK^T and P.V are 49x49x32 and the
//                 motion term 49x49x8: 0.35 MFLOP against 7.5 KB of bf16 operands, so fp32 CUDA cores with the
//                 operands in shared memory; at 720x1280 the whole pair's attention is ~21 GFLOP.
//   warp          warplayer.warp: grid_sample(bilinear, border, align_corners=True) at linspace grid + flow.
//   resize        F.interpolate(bilinear, align_corners=False) by 1/4, 1/2, 2, 4, times a power-of-two multiplier,
//                 optionally added to the output (flow / mask accumulation of MultiScaleFlow.forward).
//   dwconv_gelu   DWConv + GELU of the Mlp (feature_extractor.py:101-108, 500-511).
//   head_gather   Head input: cat([t mf[:B], (1-t) mf[B:], af[:B], af[B:]]) then PixelShuffle(2) twice.
//   merge         sigmoid mask blend + refinement residual + clamp (flow_estimation.py:133-140), the fast-TTA
//                 average (Trainer.py:95-99) and vfi_process's uint8 truncation and BGR->RGB flip.
//   pair_input / frames_to_bgr   the network's input batch and vfi_process's uint8 -> /255 BGR conversion.
//
// Arithmetic follows PyTorch's CUDA kernels (the reference runs the network on the GPU): linspace's two-sided
// formula, division by a host scalar as a multiply by its float reciprocal, grid_sample's unnormalise and
// corner weights, upsample_bilinear2d's source index and lambdas.
#include <cuda_bf16.h>
#include <math.h>

#include "../../include/b200svd.h"
#include "common.h"

namespace b200 {

static constexpr int VW = 7;         // window side
static constexpr int VN = VW * VW;   // tokens per window
static constexpr int VHD = 32;       // head dim
static constexpr int VMD = 8;        // motion dim per head
static constexpr int VFI_THREADS = 256;

static inline unsigned vfi_blocks(int64_t total) { return (unsigned)((total + VFI_THREADS - 1) / VFI_THREADS); }

struct VfiWinGeom {
  int h, w;      // token grid
  int hp, wp;    // padded to multiples of 7
  int pt, pl;    // top / left padding (pad // 2)
  int shift;     // 0 or 3
  int nwx;       // windows per row
};

__device__ __forceinline__ int vfi_region3(int v, int a, int b) { return v < a ? 0 : (v < b ? 1 : 2); }

// Token of window position `pos`: its index in the (unpadded) image or -1 for padding, and its mask label.  Two
// positions get the additive -100 iff their labels differ: the shift-mask label on the rolled grid
// (MotionFormerBlock.forward :226-243) and the padding label on the unrolled grid (pad_if_needed :32-56), which the
// reference also applies unrolled in the shifted blocks (:245-247).
__device__ __forceinline__ void vfi_win_token(const VfiWinGeom& g, int win, int pos, int& src, int& label) {
  const int Y = (win / g.nwx) * VW + pos / VW, X = (win % g.nwx) * VW + pos % VW;
  int sl = 0;
  int ys = Y, xs = X;
  if (g.shift) {
    sl = vfi_region3(Y, g.hp - VW, g.hp - g.shift) * 3 + vfi_region3(X, g.wp - VW, g.wp - g.shift);
    ys = (Y + g.shift) % g.hp;  // torch.roll by -shift
    xs = (X + g.shift) % g.wp;
  }
  const bool padded = g.hp != g.h || g.wp != g.w;
  const int pl = padded ? vfi_region3(Y, g.pt, g.pt + g.h) * 3 + vfi_region3(X, g.pl, g.pl + g.w) : 0;
  label = sl * 9 + pl;
  const int y = ys - g.pt, x = xs - g.pl;
  src = (y >= 0 && y < g.h && x >= 0 && x < g.w) ? y * g.w + x : -1;
}

__device__ __forceinline__ void vfi_load8(const __nv_bfloat16* p, float* d) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(h[i]);
    d[2 * i] = f.x;
    d[2 * i + 1] = f.y;
  }
}

// qkv rows: image b token p at row b*hw + p, row 2*pairs*hw = the padding token (q/k/v of LayerNorm(0) = beta);
// columns [q | k | v], each heads*32.  ce rows: token p (the grid is the same in every image), row hw = padding.
// Image b attends to image (b + pairs) mod 2*pairs (x_reverse, :264).
__global__ void __launch_bounds__(128) vfi_window_attn_kernel(const __nv_bfloat16* __restrict__ qkv, int64_t ldq,
                                                          const __nv_bfloat16* __restrict__ ce, int64_t ldc,
                                                          __nv_bfloat16* __restrict__ out, int64_t ldo,
                                                          __nv_bfloat16* __restrict__ mot, int64_t ldm, int heads,
                                                          int pairs, VfiWinGeom g, float scale) {
  __shared__ float sq[VN][VHD + 1], sk[VN][VHD + 1], sv[VN][VHD + 1], sc[VN][VMD + 1], sp[VN][VN + 1];
  __shared__ int ssrc[VN], slab[VN];
  const int win = blockIdx.x, head = blockIdx.y, img = blockIdx.z;
  const int kimg = (img + pairs) % (2 * pairs);
  const int64_t hw = (int64_t)g.h * g.w;
  const int64_t pad_row = 2 * pairs * hw;
  const int C = heads * VHD;
  const int tid = threadIdx.x;
  if (tid < VN) vfi_win_token(g, win, tid, ssrc[tid], slab[tid]);
  __syncthreads();
  for (int i = tid; i < VN * 13; i += blockDim.x) {
    const int pos = i / 13, part = i % 13;  // 4 vectors each of q, k, v, 1 of the motion embedding
    const int s = ssrc[pos];
    float d[8];
    if (part < 12) {
      const int t = part / 4, v = part % 4;
      const int64_t row = s < 0 ? pad_row : (int64_t)(t == 0 ? img : kimg) * hw + s;
      vfi_load8(qkv + row * ldq + t * C + head * VHD + v * 8, d);
      float(*dst)[VHD + 1] = t == 0 ? sq : (t == 1 ? sk : sv);
#pragma unroll
      for (int e = 0; e < 8; ++e) dst[pos][v * 8 + e] = d[e];
    } else {
      vfi_load8(ce + (s < 0 ? hw : (int64_t)s) * ldc + head * VMD, d);
#pragma unroll
      for (int e = 0; e < 8; ++e) sc[pos][e] = d[e];
    }
  }
  __syncthreads();
  for (int i = tid; i < VN * VN; i += blockDim.x) {
    const int r = i / VN, c = i % VN;
    float acc = 0.f;
#pragma unroll
    for (int d = 0; d < VHD; ++d) acc = fmaf(sq[r][d], sk[c][d], acc);
    acc = acc * scale;
    if (slab[r] != slab[c]) acc = acc + -100.f;
    sp[r][c] = acc;
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  for (int r = warp; r < VN; r += blockDim.x / 32) {
    const float a = sp[r][lane];
    const float b = lane + 32 < VN ? sp[r][lane + 32] : -INFINITY;
    float m = fmaxf(a, b);
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const float ea = expf(a - m), eb = lane + 32 < VN ? expf(b - m) : 0.f;
    float s = ea + eb;
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    sp[r][lane] = ea / s;
    if (lane + 32 < VN) sp[r][lane + 32] = eb / s;
  }
  __syncthreads();
  for (int i = tid; i < VN * VHD; i += blockDim.x) {
    const int r = i / VHD, d = i % VHD;
    const int s = ssrc[r];
    if (s < 0) continue;  // padding rows are cut off again (depad_if_needed)
    float acc = 0.f;
    for (int c = 0; c < VN; ++c) acc = fmaf(sp[r][c], sv[c][d], acc);
    out[((int64_t)img * hw + s) * ldo + head * VHD + d] = __float2bfloat16(acc);
  }
  for (int i = tid; i < VN * VMD; i += blockDim.x) {
    const int r = i / VMD, e = i % VMD;
    const int s = ssrc[r];
    if (s < 0) continue;
    float acc = 0.f;
    for (int c = 0; c < VN; ++c) acc = fmaf(sp[r][c], sc[c][e], acc);
    mot[((int64_t)img * hw + s) * ldm + head * VMD + e] = __float2bfloat16(acc - sc[r][e]);
  }
}

// torch.linspace(-1, 1, n)[i] (float): the step from the end points, the first half counted from the start, the
// second from the end
__device__ __forceinline__ float vfi_linspace_pm1(int i, int n) {
  const float step = 2.f / (float)(n - 1);
  return i < n / 2 ? fmaf(step, (float)i, -1.f) : fmaf(-step, (float)(n - 1 - i), 1.f);
}

template <typename T>
__device__ __forceinline__ float vfi_ldf(const T* p) {
  if constexpr (sizeof(T) == 2) return __bfloat162float(*p);
  else return __ldg(p);
}
template <typename T>
__device__ __forceinline__ void vfi_stf(T* p, float v) {
  if constexpr (sizeof(T) == 2) *p = __float2bfloat16(v);
  else *p = v;
}

struct VfiStr4 {
  int64_t n, c, y, x;  // element strides
};

// One thread per output pixel, all channels.  grid = linspace + flow / ((size - 1) / 2) (warplayer.py:11-21),
// unnormalised with align_corners=True, clamped to the border, then the four corner weights in grid_sample's order.
template <typename TI, typename TO>
__global__ void vfi_warp_kernel(const TI* __restrict__ in, VfiStr4 is, const float* __restrict__ flow, VfiStr4 fs,
                            TO* __restrict__ out, VfiStr4 os, int n, int c, int h, int w) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * h * w) return;
  const int x = (int)(i % w), y = (int)((i / w) % h), b = (int)(i / ((int64_t)w * h));
  const float* f = flow + b * fs.n + y * fs.y + x * fs.x;
  const float inv_x = 1.f / (float)((w - 1.0) / 2.0), inv_y = 1.f / (float)((h - 1.0) / 2.0);
  const float gx = vfi_linspace_pm1(x, w) + __ldg(f) * inv_x;
  const float gy = vfi_linspace_pm1(y, h) + __ldg(f + fs.c) * inv_y;
  float ix = ((gx + 1.f) / 2) * (float)(w - 1);
  float iy = ((gy + 1.f) / 2) * (float)(h - 1);
  ix = fminf((float)(w - 1), fmaxf(ix, 0.f));
  iy = fminf((float)(h - 1), fmaxf(iy, 0.f));
  const int x0 = (int)floorf(ix), y0 = (int)floorf(iy);
  const int x1 = x0 + 1, y1 = y0 + 1;
  const float wnw = ((float)x1 - ix) * ((float)y1 - iy);
  const float wne = (ix - (float)x0) * ((float)y1 - iy);
  const float wsw = ((float)x1 - ix) * (iy - (float)y0);
  const float wse = (ix - (float)x0) * (iy - (float)y0);
  const bool bx1 = x1 < w, by1 = y1 < h;
  const TI* src = in + b * is.n;
  TO* dst = out + b * os.n + y * os.y + x * os.x;
  for (int ch = 0; ch < c; ++ch) {
    const TI* s = src + ch * is.c;
    float v = 0.f;
    v = fmaf(vfi_ldf(s + y0 * is.y + x0 * is.x), wnw, v);
    if (bx1) v = fmaf(vfi_ldf(s + y0 * is.y + x1 * is.x), wne, v);
    if (by1) v = fmaf(vfi_ldf(s + y1 * is.y + x0 * is.x), wsw, v);
    if (bx1 && by1) v = fmaf(vfi_ldf(s + y1 * is.y + x1 * is.x), wse, v);
    vfi_stf(dst + ch * os.c, v);
  }
}

// upsample_bilinear2d (align_corners=False) with the scale factor given: source index max((d + 0.5) / f - 0.5, 0)
template <typename TO>
__global__ void vfi_resize_kernel(const float* __restrict__ in, VfiStr4 is, TO* __restrict__ out, VfiStr4 os, int n, int c,
                              int hi, int wi, int ho, int wo, float rscale, float mul, int accumulate) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * c * ho * wo) return;
  const int x = (int)(i % wo);
  int64_t r = i / wo;
  const int y = (int)(r % ho);
  r /= ho;
  const int ch = (int)(r % c), b = (int)(r / c);
  const float hr = fmaxf(rscale * ((float)y + 0.5f) - 0.5f, 0.f);
  const float wr = fmaxf(rscale * ((float)x + 0.5f) - 0.5f, 0.f);
  const int h1 = (int)hr, w1 = (int)wr;
  const int h1p = h1 < hi - 1 ? 1 : 0, w1p = w1 < wi - 1 ? 1 : 0;
  const float h1l = hr - (float)h1, h0l = 1.f - h1l;
  const float w1l = wr - (float)w1, w0l = 1.f - w1l;
  const float* s = in + b * is.n + ch * is.c;
  const float a00 = __ldg(s + h1 * is.y + w1 * is.x), a01 = __ldg(s + h1 * is.y + (w1 + w1p) * is.x);
  const float a10 = __ldg(s + (h1 + h1p) * is.y + w1 * is.x), a11 = __ldg(s + (h1 + h1p) * is.y + (w1 + w1p) * is.x);
  const float v = h0l * (w0l * a00 + w1l * a01) + h1l * (w0l * a10 + w1l * a11);
  TO* d = out + b * os.n + ch * os.c + y * os.y + x * os.x;
  float res = v * mul;
  if (accumulate) res = vfi_ldf(d) + res;
  vfi_stf(d, res);
}

// depthwise 3x3 (zero pad 1) + bias, then exact GELU; one thread per pixel and 8 channels
__global__ void vfi_dwconv_gelu_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int n, int h,
                                   int w, int c, const float* __restrict__ wt, const float* __restrict__ bias) {
  const int cv = c / 8;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * h * w * cv) return;
  const int c0 = (int)(i % cv) * 8;
  const int64_t p = i / cv;
  const int px = (int)(p % w), py = (int)((p / w) % h);
  const int64_t img = p / ((int64_t)w * h);
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
  for (int kh = 0; kh < 3; ++kh) {
    const int yy = py + kh - 1;
    if (yy < 0 || yy >= h) continue;
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      const int xx = px + kw - 1;
      if (xx < 0 || xx >= w) continue;
      float v[8];
      vfi_load8(x + ((img * h + yy) * w + xx) * c + c0, v);
      const float* wk = wt + (kh * 3 + kw) * c + c0;
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = fmaf(v[e], __ldg(wk + e), acc[e]);
    }
  }
  uint4 o;
  __nv_bfloat162* oh = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float a = acc[2 * e] + __ldg(bias + c0 + 2 * e), b = acc[2 * e + 1] + __ldg(bias + c0 + 2 * e + 1);
    a = 0.5f * a * (1.f + erff(a * 0.70710678118654752f));
    b = 0.5f * b * (1.f + erff(b * 0.70710678118654752f));
    oh[e] = __floats2bfloat162_rn(a, b);
  }
  *reinterpret_cast<uint4*>(y + p * c + c0) = o;
}

// out[b][4i + 2a + a'][4j + 2b + b'][ch] = src channel s = 16 ch + 8 a' + 4 b' + 2 a + b of the concat
// [0.5 mf[b] | 0.5 mf[b + pairs] | af[b] | af[b + pairs]] at (i, j), each block c channels (timestep 0.5)
__global__ void vfi_head_gather_kernel(const __nv_bfloat16* __restrict__ mf, int64_t ldm,
                                   const __nv_bfloat16* __restrict__ af, int64_t lda, int pairs, int h, int w, int c,
                                   __nv_bfloat16* __restrict__ out, int64_t ldo) {
  const int co = c / 4;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)pairs * 16 * h * w * co) return;
  const int ch = (int)(i % co);
  int64_t r = i / co;
  const int X = (int)(r % (4 * w));
  r /= 4 * w;
  const int Y = (int)(r % (4 * h));
  const int b = (int)(r / (4 * h));
  const int s = 16 * ch + 8 * (Y & 1) + 4 * (X & 1) + 2 * ((Y >> 1) & 1) + ((X >> 1) & 1);
  const int blk = s / c, sc = s % c;
  const int64_t pix = (int64_t)(Y >> 2) * w + (X >> 2);
  const int img = (blk & 1) ? b + pairs : b;
  const int64_t row = (int64_t)img * h * w + pix;
  float v;
  if (blk < 2) v = 0.5f * __bfloat162float(mf[row * ldm + sc]);
  else v = __bfloat162float(af[row * lda + sc]);
  out[((int64_t)b * 16 * h * w + (int64_t)Y * 4 * w + X) * ldo + ch] = __float2bfloat16(v);
}

__device__ __forceinline__ float vfi_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// pred_b = clamp(w0 m + w1 (1 - m) + (2 sigmoid(u) - 1), 0, 1), m = sigmoid(mask), for the pair (b = 0) and its
// flipped copy (b = 1, read at the mirrored pixel); out = (pred_0 + pred_1) / 2.  Each step one fp32 operation, as the
// reference's separate elementwise kernels round.
__global__ void vfi_merge_kernel(const float* __restrict__ w0, const float* __restrict__ w1, const float* __restrict__ fm,
                             const float* __restrict__ u, int64_t ldu, int h, int w, float* __restrict__ pred,
                             uint8_t* __restrict__ frame) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t hw = (int64_t)h * w;
  if (i >= hw) return;
  const int x = (int)(i % w), y = (int)(i / w);
  float avg[3];
  float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const int64_t p = b == 0 ? i : (int64_t)(h - 1 - y) * w + (w - 1 - x);
    const float m = vfi_sigmoid(__ldg(fm + (b * 5 + 4) * hw + p));
    const float om = __fsub_rn(1.f, m);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float merged = __fadd_rn(__fmul_rn(__ldg(w0 + (b * 3 + c) * hw + p), m),
                                     __fmul_rn(__ldg(w1 + (b * 3 + c) * hw + p), om));
      const float res = __fsub_rn(__fmul_rn(vfi_sigmoid(__ldg(u + (b * hw + p) * ldu + c)), 2.f), 1.f);
      const float pv = fminf(fmaxf(__fadd_rn(merged, res), 0.f), 1.f);
      acc[c] = b == 0 ? pv : __fadd_rn(acc[c], pv);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) avg[c] = acc[c] / 2.f;
  if (pred != nullptr) {
#pragma unroll
    for (int c = 0; c < 3; ++c) pred[c * hw + i] = avg[c];
  }
  if (frame != nullptr) {
#pragma unroll
    for (int c = 0; c < 3; ++c) frame[i * 3 + (2 - c)] = (uint8_t)(int)__fmul_rn(avg[c], 255.f);  // truncates
  }
}

// imgs [4][3][h][w] = [img0, flip(img0), img1, flip(img1)] (flip = both spatial axes), x8 [4][h][w][8] bf16 with
// channels 3..7 zero: the first conv's A operand
__global__ void vfi_pair_input_kernel(const float* __restrict__ img0, const float* __restrict__ img1, int h, int w,
                                  float* __restrict__ imgs, __nv_bfloat16* __restrict__ x8) {
  const int64_t hw = (int64_t)h * w;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 4 * hw) return;
  const int n = (int)(i / hw);
  const int64_t p = i % hw;
  const int64_t q = (n & 1) ? hw - 1 - p : p;
  const float* src = n < 2 ? img0 : img1;
  uint4 o = make_uint4(0, 0, 0, 0);
  __nv_bfloat16* oh = reinterpret_cast<__nv_bfloat16*>(&o);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = __ldg(src + c * hw + q);
    imgs[(n * 3 + c) * hw + p] = v;
    oh[c] = __float2bfloat16(v);
  }
  reinterpret_cast<uint4*>(x8)[i] = o;
}

// uint8 RGB [n][h][w][3] -> fp32 BGR [n][3][h][w], value (float)(u / 255.0) as numpy's float64 division then the
// float32 cast
__global__ void vfi_frames_to_bgr_kernel(const uint8_t* __restrict__ fr, int64_t total_px, int64_t hw,
                                     float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total_px) return;
  const int64_t f = i / hw, p = i % hw;
#pragma unroll
  for (int c = 0; c < 3; ++c) out[(f * 3 + c) * hw + p] = (float)((double)fr[i * 3 + (2 - c)] / 255.0);
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200svd_vfi_window_attn(const void* qkv, int64_t ldq, const void* cor_embed, int64_t ldc, void* out, int64_t ldo,
                            void* motion, int64_t ldm, int pairs, int h, int w, int heads, int shift, float scale,
                            void* stream) {
  if (pairs < 0 || h < 0 || w < 0 || heads < 0 || heads > 65535 || pairs > 32767 || (shift != 0 && shift != 3)) {
    set_error("b200svd_vfi_window_attn: pairs=%d h=%d w=%d heads=%d shift=%d out of range (heads <= 65535, "
              "2*pairs <= 65535, shift 0 or 3)", pairs, h, w, heads, shift);
    return 1;
  }
  if ((int64_t)pairs * h * w * heads == 0) return 0;
  if (!aligned(qkv, 16) || !aligned(cor_embed, 16) || ldq % 8 || ldc % 8 || ldq < 3 * heads * VHD ||
      ldc < heads * VMD || ldo < heads * VHD || ldm < heads * VMD) {
    set_error("b200svd_vfi_window_attn: qkv / cor_embed need 16-byte aligned bases and leading dims that are multiples "
              "of 8, and every leading dim must hold its heads");
    return 1;
  }
  VfiWinGeom g;
  g.h = h;
  g.w = w;
  g.hp = (h + VW - 1) / VW * VW;
  g.wp = (w + VW - 1) / VW * VW;
  g.pt = (g.hp - h) / 2;
  g.pl = (g.wp - w) / 2;
  g.shift = shift;
  g.nwx = g.wp / VW;
  const dim3 grid((unsigned)((g.hp / VW) * g.nwx), (unsigned)heads, (unsigned)(2 * pairs));
  vfi_window_attn_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)qkv, ldq, (const __nv_bfloat16*)cor_embed, ldc, (__nv_bfloat16*)out, ldo,
      (__nv_bfloat16*)motion, ldm, heads, pairs, g, scale);
  B200_CHECK_LAUNCH("b200svd_vfi_window_attn");
  return 0;
}

int b200svd_vfi_warp(const void* in, int in_bf16, int64_t isn, int64_t isc, int64_t isy, int64_t isx,
                     const float* flow, int64_t fsn, int64_t fsc, int64_t fsy, int64_t fsx, void* out, int out_bf16,
                     int64_t osn, int64_t osc, int64_t osy, int64_t osx, int n, int c, int h, int w, void* stream) {
  if (in_bf16 != out_bf16) {
    set_error("b200svd_vfi_warp: in and out must both be fp32 or both bf16 (in_bf16=%d out_bf16=%d)", in_bf16,
              out_bf16);
    return 1;
  }
  if (n < 0 || c < 0 || h < 0 || w < 0) {
    set_error("b200svd_vfi_warp: n=%d c=%d h=%d w=%d out of range", n, c, h, w);
    return 1;
  }
  const int64_t total = (int64_t)n * h * w;
  if (total == 0 || c == 0) return 0;
  if (h < 2 || w < 2) {  // the grid's (size - 1) / 2 normalisation
    set_error("b200svd_vfi_warp: h=%d w=%d, both must be >= 2", h, w);
    return 1;
  }
  const VfiStr4 is{isn, isc, isy, isx}, fs{fsn, fsc, fsy, fsx}, os{osn, osc, osy, osx};
  cudaStream_t st = (cudaStream_t)stream;
  if (in_bf16)
    vfi_warp_kernel<<<vfi_blocks(total), VFI_THREADS, 0, st>>>((const __nv_bfloat16*)in, is, flow, fs,
                                                           (__nv_bfloat16*)out, os, n, c, h, w);
  else
    vfi_warp_kernel<<<vfi_blocks(total), VFI_THREADS, 0, st>>>((const float*)in, is, flow, fs, (float*)out, os, n, c, h,
                                                           w);
  B200_CHECK_LAUNCH("b200svd_vfi_warp");
  return 0;
}

int b200svd_vfi_resize(const float* in, int64_t isn, int64_t isc, int64_t isy, int64_t isx, void* out, int out_bf16,
                       int64_t osn, int64_t osc, int64_t osy, int64_t osx, int n, int c, int h, int w, int factor_log2,
                       float mul, int accumulate, void* stream) {
  if (factor_log2 < -2 || factor_log2 > 2 || factor_log2 == 0 || n < 0 || c < 0 || h < 0 || w < 0 ||
      (out_bf16 && accumulate)) {
    set_error("b200svd_vfi_resize: factor 2^%d (must be 1/4, 1/2, 2 or 4), n=%d c=%d h=%d w=%d, accumulate=%d "
              "(fp32 outputs only)", factor_log2, n, c, h, w, accumulate);
    return 1;
  }
  int ho, wo;
  float rscale;
  if (factor_log2 > 0) {
    ho = h << factor_log2;
    wo = w << factor_log2;
    rscale = 1.f / (float)(1 << factor_log2);
  } else {
    ho = h >> -factor_log2;  // floor(h * factor), as F.interpolate sizes its output
    wo = w >> -factor_log2;
    rscale = (float)(1 << -factor_log2);
  }
  const int64_t total = (int64_t)n * c * ho * wo;
  if (total == 0) return 0;
  const VfiStr4 is{isn, isc, isy, isx}, os{osn, osc, osy, osx};
  if (out_bf16)
    vfi_resize_kernel<<<vfi_blocks(total), VFI_THREADS, 0, (cudaStream_t)stream>>>(in, is, (__nv_bfloat16*)out, os, n, c, h,
                                                                               w, ho, wo, rscale, mul, 0);
  else
    vfi_resize_kernel<<<vfi_blocks(total), VFI_THREADS, 0, (cudaStream_t)stream>>>(in, is, (float*)out, os, n, c, h, w, ho,
                                                                               wo, rscale, mul, accumulate);
  B200_CHECK_LAUNCH("b200svd_vfi_resize");
  return 0;
}

int b200svd_vfi_dwconv_gelu(const void* x, void* y, int n, int h, int w, int c, const float* wt, const float* bias,
                            void* stream) {
  if (n < 0 || h < 0 || w < 0 || c < 0 || c % 8 || !aligned(x, 16) || !aligned(y, 16)) {
    set_error("b200svd_vfi_dwconv_gelu: c=%d must be a multiple of 8 and x, y 16-byte aligned", c);
    return 1;
  }
  const int64_t total = (int64_t)n * h * w * (c / 8);
  if (total == 0) return 0;
  vfi_dwconv_gelu_kernel<<<vfi_blocks(total), VFI_THREADS, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x, (__nv_bfloat16*)y, n, h, w, c, wt, bias);
  B200_CHECK_LAUNCH("b200svd_vfi_dwconv_gelu");
  return 0;
}

int b200svd_vfi_head_gather(const void* mf, int64_t ldm, const void* af, int64_t lda, int pairs, int h, int w, int c,
                            void* out, int64_t ldo, void* stream) {
  if (pairs < 0 || h < 0 || w < 0 || c < 0 || c % 4 || ldm < c || lda < c || ldo < c / 4) {
    set_error("b200svd_vfi_head_gather: c=%d must be a multiple of 4 and fit the leading dims", c);
    return 1;
  }
  const int64_t total = (int64_t)pairs * 16 * h * w * (c / 4);
  if (total == 0) return 0;
  vfi_head_gather_kernel<<<vfi_blocks(total), VFI_THREADS, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)mf, ldm, (const __nv_bfloat16*)af, lda, pairs, h, w, c, (__nv_bfloat16*)out, ldo);
  B200_CHECK_LAUNCH("b200svd_vfi_head_gather");
  return 0;
}

int b200svd_vfi_merge(const float* warped0, const float* warped1, const float* fm, const float* res, int64_t ldr,
                      int h, int w, float* pred, void* frame, void* stream) {
  if (h < 0 || w < 0 || ldr < 3) {
    set_error("b200svd_vfi_merge: h=%d w=%d ldr=%lld out of range", h, w, (long long)ldr);
    return 1;
  }
  const int64_t total = (int64_t)h * w;
  if (total == 0) return 0;
  vfi_merge_kernel<<<vfi_blocks(total), VFI_THREADS, 0, (cudaStream_t)stream>>>(warped0, warped1, fm, res, ldr, h, w, pred,
                                                                            (uint8_t*)frame);
  B200_CHECK_LAUNCH("b200svd_vfi_merge");
  return 0;
}

int b200svd_vfi_pair_input(const float* img0, const float* img1, int h, int w, float* imgs, void* x8, void* stream) {
  if (h < 0 || w < 0 || !aligned(x8, 16)) {
    set_error("b200svd_vfi_pair_input: h=%d w=%d, x8 must be 16-byte aligned", h, w);
    return 1;
  }
  const int64_t total = 4 * (int64_t)h * w;
  if (total == 0) return 0;
  vfi_pair_input_kernel<<<vfi_blocks(total), VFI_THREADS, 0, (cudaStream_t)stream>>>(img0, img1, h, w, imgs,
                                                                                 (__nv_bfloat16*)x8);
  B200_CHECK_LAUNCH("b200svd_vfi_pair_input");
  return 0;
}

int b200svd_vfi_frames_to_bgr(const void* frames, int64_t n, int h, int w, float* out, void* stream) {
  if (n < 0 || h < 0 || w < 0) {
    set_error("b200svd_vfi_frames_to_bgr: n=%lld h=%d w=%d out of range", (long long)n, h, w);
    return 1;
  }
  const int64_t hw = (int64_t)h * w, total = n * hw;
  if (total == 0) return 0;
  vfi_frames_to_bgr_kernel<<<vfi_blocks(total), VFI_THREADS, 0, (cudaStream_t)stream>>>((const uint8_t*)frames, total, hw,
                                                                                    out);
  B200_CHECK_LAUNCH("b200svd_vfi_frames_to_bgr");
  return 0;
}

}  // extern "C"
