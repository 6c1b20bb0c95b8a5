// CLIP image preprocessing of the SVD conditioner, fused with the patch gather of the ViT-H/14 patch embedding.
//
// Replaces FrozenOpenCLIPImageEmbedder.preprocess (reference code/models/svd/sgm/modules/encoders/modules.py:624-636):
//   kornia.geometry.resize(x, (224, 224), interpolation="bicubic", align_corners=True, antialias=True)
//     = separable Gaussian blur (reflect borders; taps computed on the host from kornia 0.7.2's formulas) when
//       downscaling, then F.interpolate(bicubic, align_corners=True) (A = -0.75, clamped neighbour indices)
//   (x + 1) / 2, then kornia.enhance.normalize with the CLIP mean / std
// and the im2col of open_clip's `conv1` (14 x 14, stride 14, no bias): the output is the A operand of the patch GEMM,
// bf16 rows [(n 256), ldp], row = image * 256 + patch_y * 16 + patch_x, column = (kh * 14 + kw) * 3 + channel,
// columns 588..ldp-1 zero.  One thread per output element; the blur is evaluated only at the 4 x 4 source pixels the
// bicubic taps of that element read, so no intermediate image is written.  fp32 arithmetic throughout.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200svd.h"
#include "common.h"

namespace b200 {

constexpr int CP_OUT = 224;
constexpr int CP_PATCH = 14;
constexpr int CP_GRID = CP_OUT / CP_PATCH;  // 16 patches per side
constexpr int CP_K = CP_PATCH * CP_PATCH * 3;  // 588
constexpr int CP_MAX_TAPS = 63;

struct ClipPrepParams {
  const float* x;
  __nv_bfloat16* out;
  int64_t ldp;
  int n, H, W;
  int ky, kx;
  float gy[CP_MAX_TAPS];
  float gx[CP_MAX_TAPS];
};

__device__ __forceinline__ int reflect_idx(int i, int n) {  // torch F.pad(mode="reflect"), pad < n
  i = i < 0 ? -i : i;
  return i >= n ? 2 * (n - 1) - i : i;
}

// torch's upsample_bicubic2d weight of tap a (0..3, source index floor(s) - 1 + a) at fraction t (A = -0.75):
// taps 0 and 3 at distance 1 + t and 2 - t, taps 1 and 2 at distance t and 1 - t
__device__ __forceinline__ float cubic_weight(int a, float t) {
  const float A = -0.75f;
  const float d = a == 0 ? t + 1.0f : a == 1 ? t : a == 2 ? 1.0f - t : 2.0f - t;
  return (a == 0 || a == 3) ? ((A * d - 5.0f * A) * d + 8.0f * A) * d - 4.0f * A
                            : ((A + 2.0f) * d - (A + 3.0f)) * d * d + 1.0f;
}

__global__ void clip_preprocess_kernel(const __grid_constant__ ClipPrepParams p) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = (int64_t)p.n * CP_GRID * CP_GRID * p.ldp;
  if (i >= total) return;
  const int col = (int)(i % p.ldp);
  const int64_t row = i / p.ldp;
  if (col >= CP_K) {
    p.out[i] = __float2bfloat16(0.0f);
    return;
  }
  const int img = (int)(row / (CP_GRID * CP_GRID));
  const int patch = (int)(row % (CP_GRID * CP_GRID));
  const int ch = col % 3, kk = col / 3;
  const int oy = (patch / CP_GRID) * CP_PATCH + kk / CP_PATCH;
  const int ox = (patch % CP_GRID) * CP_PATCH + kk % CP_PATCH;
  const int H = p.H, W = p.W;
  // align_corners source coordinate, in fp32 as torch computes it
  const float sy = ((float)(H - 1) / (float)(CP_OUT - 1)) * (float)oy;
  const float sx = ((float)(W - 1) / (float)(CP_OUT - 1)) * (float)ox;
  const int iy = (int)floorf(sy), ix = (int)floorf(sx);
  const float ty = sy - (float)iy, tx = sx - (float)ix;
  const float* src = p.x + ((int64_t)img * 3 + ch) * H * W;
  const int hy = p.ky / 2, hx = p.kx / 2;
  float acc = 0.0f;
  for (int a = 0; a < 4; ++a) {
    const int r = min(max(iy - 1 + a, 0), H - 1);
    float rowv = 0.0f;
    for (int b = 0; b < 4; ++b) {
      const int q = min(max(ix - 1 + b, 0), W - 1);
      // blurred source pixel (r, q): sum_u gy[u] sum_v gx[v] x[reflect(r + u - hy), reflect(q + v - hx)]
      float blur = 0.0f;
      for (int u = 0; u < p.ky; ++u) {
        const float* srow = src + (int64_t)reflect_idx(r + u - hy, H) * W;
        float hs = 0.0f;
        for (int v = 0; v < p.kx; ++v) hs = fmaf(p.gx[v], __ldg(srow + reflect_idx(q + v - hx, W)), hs);
        blur = fmaf(p.gy[u], hs, blur);
      }
      rowv = fmaf(cubic_weight(b, tx), blur, rowv);
    }
    acc = fmaf(cubic_weight(a, ty), rowv, acc);
  }
  const float mean = ch == 0 ? 0.48145466f : ch == 1 ? 0.4578275f : 0.40821073f;
  const float stdv = ch == 0 ? 0.26862954f : ch == 1 ? 0.26130258f : 0.27577711f;
  p.out[i] = __float2bfloat16(((acc + 1.0f) / 2.0f - mean) / stdv);
}

}  // namespace b200

extern "C" int b200svd_clip_preprocess(const float* x, int n, int h, int w, void* out, int64_t ldp,
                                       const float* taps_y, int ky, const float* taps_x, int kx, void* stream) {
  using namespace b200;
  if (n <= 0 || h <= 0 || w <= 0) {
    set_error("clip_preprocess: need n, h, w >= 1, got n=%d h=%d w=%d", n, h, w);
    return 1;
  }
  if (ldp % 8 != 0 || ldp < ((CP_K + 7) / 8) * 8) {
    set_error("clip_preprocess: ldp (%lld) must be a multiple of 8 and >= 592", (long long)ldp);
    return 1;
  }
  if ((reinterpret_cast<uintptr_t>(x) & 3) != 0 || (reinterpret_cast<uintptr_t>(out) & 15) != 0) {
    set_error("clip_preprocess: x must be 4-byte aligned and out 16-byte aligned");
    return 1;
  }
  if (ky < 1 || kx < 1 || ky > CP_MAX_TAPS || kx > CP_MAX_TAPS || ky % 2 == 0 || kx % 2 == 0 || !taps_y || !taps_x) {
    set_error("clip_preprocess: blur taps must be odd counts in 1..%d (got %d, %d)", CP_MAX_TAPS, ky, kx);
    return 1;
  }
  if (ky / 2 >= h || kx / 2 >= w) {
    set_error("clip_preprocess: reflect padding (%d, %d) must be smaller than the image (%d x %d)", ky / 2, kx / 2, h, w);
    return 1;
  }
  ClipPrepParams p;
  p.x = x;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ldp = ldp;
  p.n = n;
  p.H = h;
  p.W = w;
  p.ky = ky;
  p.kx = kx;
  for (int i = 0; i < CP_MAX_TAPS; ++i) {
    p.gy[i] = i < ky ? taps_y[i] : 0.0f;
    p.gx[i] = i < kx ? taps_x[i] : 0.0f;
  }
  const int64_t total = (int64_t)n * CP_GRID * CP_GRID * ldp;
  clip_preprocess_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  B200_CHECK_LAUNCH("clip_preprocess");
  return 0;
}
