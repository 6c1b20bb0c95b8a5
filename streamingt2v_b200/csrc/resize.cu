// PIL's BICUBIC resize of uint8 RGB frames, bit for bit: `Image.resize((W, H))` as the reference's enhance stage
// calls it on the first stage's 1024x576 frames (code/inference_i2v.py:197-199) and on the request image
// (IImage.resize, :194-195).
//
// Pillow's 8-bit path (libImaging/Resample.c) is separable: a horizontal pass into a uint8 image, then a vertical
// pass, each skipped when its axis keeps its size.  Output index xx of a pass reads n consecutive source samples from
// xmin with integer coefficients k (weights scaled by 2^22 and rounded away from zero), all computed on the host
// (ops.bicubic_taps), and writes clip((2^21 + sum k * p) >> 22, 0, 255) in int32.  One thread per output pixel, three
// channels each; the horizontal pass writes [n, h_in, w_out, 3] into the caller's workspace.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200svd.h"
#include "common.h"

namespace b200 {

constexpr int RS_PRECISION = 22;  // Pillow's PRECISION_BITS for 8-bit images (32 - 8 - 2)

__device__ __forceinline__ uint8_t rs_clip8(int32_t acc) {
  return (uint8_t)min(max(acc >> RS_PRECISION, 0), 255);
}

// One pass along an axis.  Output pixel (o, i, c) of [outer, n_out, inner] pixels reads source pixels
// (o, xmin + j, c), j < n, of [outer, n_in, inner]: the horizontal pass has inner = 1, the vertical inner = width.
__global__ void resize_pass_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int64_t outer,
                                   int n_in, int n_out, int64_t inner, const int2* __restrict__ bounds,
                                   const int32_t* __restrict__ taps, int k) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= outer * n_out * inner) return;
  const int64_t c = p % inner;
  const int64_t oi = p / inner;
  const int i = (int)(oi % n_out);
  const int64_t o = oi / n_out;
  const int2 b = __ldg(bounds + i);  // (xmin, n)
  const int32_t* kk = taps + (int64_t)i * k;
  const uint8_t* src = in + ((o * n_in + b.x) * inner + c) * 3;
  const int64_t step = inner * 3;
  int32_t a0 = 1 << (RS_PRECISION - 1), a1 = a0, a2 = a0;
  for (int j = 0; j < b.y; ++j) {
    const int32_t w = __ldg(kk + j);
    a0 += (int32_t)__ldg(src) * w;
    a1 += (int32_t)__ldg(src + 1) * w;
    a2 += (int32_t)__ldg(src + 2) * w;
    src += step;
  }
  uint8_t* dst = out + p * 3;
  dst[0] = rs_clip8(a0);
  dst[1] = rs_clip8(a1);
  dst[2] = rs_clip8(a2);
}

int resize_pass(const uint8_t* in, uint8_t* out, int64_t outer, int n_in, int n_out, int64_t inner,
                const int32_t* bounds, const int32_t* taps, int k, cudaStream_t stream) {
  const int64_t total = outer * n_out * inner;
  resize_pass_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(
      in, out, outer, n_in, n_out, inner, reinterpret_cast<const int2*>(bounds), taps, k);
  B200_CHECK_LAUNCH("resize_bicubic_u8");
  return 0;
}

}  // namespace b200

extern "C" int b200svd_resize_bicubic_u8(const void* x, int64_t n, int h_in, int w_in, void* out, int h_out,
                                         int w_out, const int32_t* bounds_x, const int32_t* taps_x, int kx,
                                         const int32_t* bounds_y, const int32_t* taps_y, int ky, void* workspace,
                                         void* stream) {
  using namespace b200;
  if (n < 0 || h_in < 1 || w_in < 1 || h_out < 1 || w_out < 1) {
    set_error("resize_bicubic_u8: need n >= 0 and sizes >= 1, got n=%lld %dx%d -> %dx%d", (long long)n, w_in, h_in,
              w_out, h_out);
    return 1;
  }
  if (n == 0) return 0;
  const bool horizontal = w_out != w_in, vertical = h_out != h_in;
  if ((horizontal && (!bounds_x || !taps_x || kx < 1)) || (vertical && (!bounds_y || !taps_y || ky < 1))) {
    set_error("resize_bicubic_u8: a pass that changes its axis needs its bounds, taps and a tap count >= 1");
    return 1;
  }
  if ((horizontal && !aligned(bounds_x, 8)) || (vertical && !aligned(bounds_y, 8))) {
    set_error("resize_bicubic_u8: bounds arrays must be 8-byte aligned");
    return 1;
  }
  if (horizontal && vertical && !workspace) {
    set_error("resize_bicubic_u8: resizing both axes needs a workspace of n * h_in * w_out * 3 bytes");
    return 1;
  }
  auto s = reinterpret_cast<cudaStream_t>(stream);
  auto src = reinterpret_cast<const uint8_t*>(x);
  auto dst = reinterpret_cast<uint8_t*>(out);
  if (!horizontal && !vertical) {
    const cudaError_t e = cudaMemcpyAsync(dst, src, (size_t)n * h_in * w_in * 3, cudaMemcpyDeviceToDevice, s);
    return e == cudaSuccess ? 0 : cuda_fail(e, "resize_bicubic_u8: copy");
  }
  if (horizontal) {
    uint8_t* hout = vertical ? reinterpret_cast<uint8_t*>(workspace) : dst;
    if (resize_pass(src, hout, n * h_in, w_in, w_out, 1, bounds_x, taps_x, kx, s)) return 1;
    src = hout;
  }
  if (vertical) return resize_pass(src, dst, n, h_in, h_out, w_out, bounds_y, taps_y, ky, s);
  return 0;
}
