// Layout / glue kernels (HBM-bound, vectorised): NCHW fp32 <-> channel-last bf16 at the module seam, nearest 2x
// upsample, sinusoidal timestep embedding, embedding finalisation, APM context mix.
//
// Replaces the reference's torch.cat / rearrange / F.interpolate / timestep_embedding glue:
//   wrappers.py:33 (cat latents + concat cond), openaimodel.py:107-157 (Upsample nearest),
//   diffusionmodules/util.py:207-231 (timestep_embedding), video_model.py:561-567 (emb = time_embed + label_emb),
//   attention.py:612-620 (APM context mix).
#include <cuda_bf16.h>
#include <math.h>

#include "../../include/b200svd.h"
#include "common.h"
#include "ptx.cuh"

namespace b200 {

// src: [N][Csrc][H][W] fp32 (frame stride given, lets the caller slice frames) -> dst[(n*HW + p)*ldd + c_off + c] bf16
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, int64_t src_frame_stride, int Csrc, int64_t HW,
                                    __nv_bfloat16* __restrict__ dst, int64_t ldd, int c_off, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int64_t p = i % HW;
  const int64_t n = i / HW;
  const float* s = src + n * src_frame_stride + p;
  __nv_bfloat16* d = dst + i * ldd + c_off;
  for (int c = 0; c < Csrc; ++c) d[c] = __float2bfloat16(__ldg(s + (int64_t)c * HW));
}

// src: [rows][lds] (fp32 or bf16 rows, first C columns) -> dst [N][C][HW] fp32
template <typename T>
__global__ void nhwc_to_nchw_kernel(const T* __restrict__ src, int64_t lds, int C, int64_t HW, float* __restrict__ dst,
                                    int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // over N*C*HW, p fastest (coalesced writes)
  if (i >= total) return;
  const int64_t p = i % HW;
  const int64_t c = (i / HW) % C;
  const int64_t n = i / (HW * C);
  dst[i] = (float)src[(n * HW + p) * lds + c];
}

// nearest-neighbour 2x upsample, channel-last: x [N][H][W][C] -> y [N][2H][2W][C]; one thread per output 16 B vector
__global__ void upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int H, int W, int vecs,
                                  int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int v = (int)(i % vecs);
  int64_t r = i / vecs;
  const int ox = (int)(r % (2 * W));
  r /= (2 * W);
  const int oy = (int)(r % (2 * H));
  const int64_t n = r / (2 * H);
  y[i] = __ldg(x + ((n * H + (oy >> 1)) * W + (ox >> 1)) * vecs + v);
}

// out[n][0:half] = cos(t*f), out[n][half:] = sin(t*f), f_i = exp(-ln(max_period) * i / half); bf16
__global__ void timestep_embed_kernel(const float* __restrict__ t, int n, int dim, float max_period,
                                      __nv_bfloat16* __restrict__ out, int64_t ldo) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = dim / 2;
  if (i >= n * half) return;
  const int r = i / half, c = i % half;
  const float f = expf(-logf(max_period) * (float)c / (float)half);
  const float a = t[r] * f;
  out[(int64_t)r * ldo + c] = __float2bfloat16(cosf(a));
  out[(int64_t)r * ldo + half + c] = __float2bfloat16(sinf(a));
}

// out = bf16( silu(a + b) )  (b may be null)
__global__ void add_silu_kernel(const float* __restrict__ a, const float* __restrict__ b, __nv_bfloat16* __restrict__ out,
                                int64_t total, int apply_silu) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  float v = a[i] + (b ? b[i] : 0.f);
  if (apply_silu) v = silu_f(v);
  out[i] = __float2bfloat16(v);
}

// strided bf16 row copy: dst[r*ldd + c] = src[r*lds + c], cols multiple of 8
__global__ void copy2d_kernel(const __nv_bfloat16* __restrict__ src, int64_t lds, __nv_bfloat16* __restrict__ dst,
                              int64_t ldd, int vecs, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int v = (int)(i % vecs);
  const int64_t r = i / vecs;
  *reinterpret_cast<uint4*>(dst + r * ldd + v * 8) = __ldg(reinterpret_cast<const uint4*>(src + r * lds + v * 8));
}

// dst[r*ldd + c] += src[(r % src_rows)*lds + c]   (ControlNet Merger "addition", controlnet.py:23-48)
__global__ void add_rows_kernel(__nv_bfloat16* __restrict__ dst, int64_t ldd, const __nv_bfloat16* __restrict__ src,
                                int64_t lds, int64_t src_rows, int vecs, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int v = (int)(i % vecs);
  const int64_t r = i / vecs;
  uint4* dp = reinterpret_cast<uint4*>(dst + r * ldd + v * 8);
  const uint4 a = *dp;
  const uint4 b = __ldg(reinterpret_cast<const uint4*>(src + (r % src_rows) * lds + v * 8));
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j)
    o[j] = pack_bf16x2(bf16_lo(aw[j]) + bf16_lo(bw[j]), bf16_hi(aw[j]) + bf16_hi(bw[j]));
  *dp = make_uint4(o[0], o[1], o[2], o[3]);
}

// APM: ctx [N][L][D] fp32 -> out [N][D] bf16 = ctx[:,0] + LN_D(conv1d_{L->1,k=3,pad=1 over D}(ctx)) * silu(alpha)
// one block per n; D <= 4096.
__global__ void apm_mix_kernel(const float* __restrict__ ctx, int L, int D, const float* __restrict__ w /*[L][3]*/,
                               const float* __restrict__ wb /*[1]*/, const float* __restrict__ ln_g,
                               const float* __restrict__ ln_b, const float* __restrict__ alpha,
                               __nv_bfloat16* __restrict__ out) {
  extern __shared__ float mix[];  // [D]
  __shared__ float red[64];
  const int n = blockIdx.x;
  const float* c = ctx + (int64_t)n * L * D;
  float lsum = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = wb[0];
    for (int l = 0; l < L; ++l) {
      const float* row = c + (int64_t)l * D;
      const float xm = d > 0 ? row[d - 1] : 0.f, x0 = row[d], xp = d + 1 < D ? row[d + 1] : 0.f;
      acc += w[l * 3] * xm + w[l * 3 + 1] * x0 + w[l * 3 + 2] * xp;
    }
    mix[d] = acc;
    lsum += acc;
  }
  // block reduce (sum)
  for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lsum;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
  const float mean = tot / (float)D;
  __syncthreads();
  float lsq = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const float t = mix[d] - mean;
    lsq += t * t;
  }
  for (int o = 16; o > 0; o >>= 1) lsq += __shfl_xor_sync(0xffffffffu, lsq, o);
  if ((threadIdx.x & 31) == 0) red[32 + (threadIdx.x >> 5)] = lsq;
  __syncthreads();
  float tq = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tq += red[32 + i];
  const float rstd = rsqrtf(tq / (float)D + 1e-5f);
  const float sa = silu_f(alpha[0]);
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const float m = (mix[d] - mean) * rstd * ln_g[d] + ln_b[d];
    out[(int64_t)n * D + d] = __float2bfloat16(c[d] + m * sa);
  }
}

static inline unsigned blocks_for(int64_t total, int threads) { return (unsigned)((total + threads - 1) / threads); }


// Sampler arithmetic around the denoiser seam (fp32, elementwise).
// prepare: xin2 = cat([x, x]) * c_in            (guiders.py:97 doubled batch, denoiser.py:36 input scaling)
__global__ void sampler_prepare_kernel(const float* __restrict__ x, float* __restrict__ xin2, int64_t n, float c_in) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = __ldg(x + i) * c_in;
  xin2[i] = v;
  xin2[n + i] = v;
}
// step: denoised = c_skip*x + c_out*(net_u + s_t*(net_c - net_u))   (denoiser.py:33-39 + guiders.py:78-86; both
//       halves of the doubled batch carry the same x); d = (x - denoised)/sigma; x_next = x + (sigma_next - sigma)*d
//       (sampling.py:100-103, 213-215).  Evaluated in the reference's operation order so that fp32 rounding matches.
__global__ void sampler_step_kernel(const float* __restrict__ net, const float* __restrict__ x,
                                    float* __restrict__ x_next, int64_t n, int64_t chw, int num_frames,
                                    const float* __restrict__ scale, float c_skip, float c_out, float sigma,
                                    float next_sigma) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float xv = __ldg(x + i);
  const float s = __ldg(scale + (int)((i / chw) % num_frames));
  const float du = __ldg(net + i) * c_out + xv * c_skip;
  const float dc = __ldg(net + n + i) * c_out + xv * c_skip;
  const float den = du + s * (dc - du);
  const float d = (xv - den) / sigma;
  x_next[i] = xv + (next_sigma - sigma) * d;
}

}  // namespace b200

extern "C" {

int b200svd_nchw_to_nhwc(const float* src, int64_t src_frame_stride, int n, int c_src, int64_t hw, void* dst,
                         int64_t ldd, int c_off, void* stream) {
  using namespace b200;
  if (n <= 0 || hw <= 0) return 0;
  const int64_t total = (int64_t)n * hw;
  nchw_to_nhwc_kernel<<<blocks_for(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src, src_frame_stride, c_src, hw, reinterpret_cast<__nv_bfloat16*>(dst), ldd, c_off, total);
  B200_CHECK_LAUNCH("nchw_to_nhwc");
  return 0;
}

int b200svd_nhwc_to_nchw(const void* src, int src_is_fp32, int64_t lds, int n, int c, int64_t hw, float* dst,
                         void* stream) {
  using namespace b200;
  if (n <= 0 || c <= 0 || hw <= 0) return 0;
  const int64_t total = (int64_t)n * c * hw;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (src_is_fp32)
    nhwc_to_nchw_kernel<float><<<blocks_for(total, 256), 256, 0, st>>>(reinterpret_cast<const float*>(src), lds, c, hw,
                                                                       dst, total);
  else
    nhwc_to_nchw_kernel<__nv_bfloat16><<<blocks_for(total, 256), 256, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(src), lds, c, hw, dst, total);
  B200_CHECK_LAUNCH("nhwc_to_nchw");
  return 0;
}

int b200svd_upsample2x(const void* x, void* y, int n, int h, int w, int c, void* stream) {
  using namespace b200;
  if (c % 8) {
    set_error("upsample2x: channels must be a multiple of 8");
    return 1;
  }
  if (n <= 0 || h <= 0 || w <= 0 || c <= 0) return 0;
  if (!aligned(x, 16) || !aligned(y, 16)) {  // one 16-byte vector per thread
    set_error("upsample2x: x and y must be 16-byte aligned");
    return 1;
  }
  const int vecs = c / 8;
  const int64_t total = (int64_t)n * 2 * h * 2 * w * vecs;
  upsample2x_kernel<<<blocks_for(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(y), h, w, vecs, total);
  B200_CHECK_LAUNCH("upsample2x");
  return 0;
}

int b200svd_timestep_embed(const float* t, int n, int dim, float max_period, void* out, int64_t ldo, void* stream) {
  using namespace b200;
  if (dim % 2) {
    set_error("timestep_embed: odd dim unsupported");
    return 1;
  }
  if (n <= 0 || dim <= 0) return 0;
  const int total = n * (dim / 2);
  timestep_embed_kernel<<<blocks_for(total, 128), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      t, n, dim, max_period, reinterpret_cast<__nv_bfloat16*>(out), ldo);
  B200_CHECK_LAUNCH("timestep_embed");
  return 0;
}

int b200svd_add_silu(const float* a, const float* b, void* out, int64_t total, int apply_silu, void* stream) {
  using namespace b200;
  if (total <= 0) return 0;
  add_silu_kernel<<<blocks_for(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      a, b, reinterpret_cast<__nv_bfloat16*>(out), total, apply_silu);
  B200_CHECK_LAUNCH("add_silu");
  return 0;
}

int b200svd_copy2d(const void* src, int64_t lds, void* dst, int64_t ldd, int64_t rows, int cols, void* stream) {
  using namespace b200;
  if (cols % 8 || lds % 8 || ldd % 8) {
    set_error("copy2d: cols and leading dims must be multiples of 8");
    return 1;
  }
  if (rows <= 0 || cols <= 0) return 0;
  if (!aligned(src, 16) || !aligned(dst, 16)) {  // 16-byte vectors
    set_error("copy2d: src and dst must be 16-byte aligned");
    return 1;
  }
  const int vecs = cols / 8;
  const int64_t total = rows * vecs;
  copy2d_kernel<<<blocks_for(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(src), lds, reinterpret_cast<__nv_bfloat16*>(dst), ldd, vecs, total);
  B200_CHECK_LAUNCH("copy2d");
  return 0;
}

int b200svd_add_rows(void* dst, int64_t ldd, const void* src, int64_t lds, int64_t rows, int64_t src_rows, int cols,
                     void* stream) {
  using namespace b200;
  if (cols % 8 || lds % 8 || ldd % 8) {
    set_error("add_rows: cols and leading dims must be multiples of 8");
    return 1;
  }
  if (src_rows < 1) {  // dst row r adds src row r % src_rows
    set_error("add_rows: src_rows must be >= 1 (got %lld)", (long long)src_rows);
    return 1;
  }
  if (rows <= 0 || cols <= 0) return 0;
  if (!aligned(dst, 16) || !aligned(src, 16)) {  // 16-byte vectors
    set_error("add_rows: dst and src must be 16-byte aligned");
    return 1;
  }
  const int vecs = cols / 8;
  const int64_t total = rows * vecs;
  add_rows_kernel<<<blocks_for(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<__nv_bfloat16*>(dst), ldd, reinterpret_cast<const __nv_bfloat16*>(src), lds, src_rows, vecs,
      total);
  B200_CHECK_LAUNCH("add_rows");
  return 0;
}

int b200svd_apm_mix(const float* ctx, int n, int l, int d, const float* w, const float* wb, const float* ln_g,
                    const float* ln_b, const float* alpha, void* out, void* stream) {
  using namespace b200;
  if (d > 8192) {
    set_error("apm_mix: D too large");
    return 1;
  }
  if (n <= 0 || d <= 0) return 0;
  apm_mix_kernel<<<n, 256, d * sizeof(float), reinterpret_cast<cudaStream_t>(stream)>>>(
      ctx, l, d, w, wb, ln_g, ln_b, alpha, reinterpret_cast<__nv_bfloat16*>(out));
  B200_CHECK_LAUNCH("apm_mix");
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------------
// Single-head attention helpers for the VAE decoder's AttnBlock (reference diffusionmodules/model.py:180-195):
// row softmax of fp32 scores -> bf16 probabilities, and a bf16 matrix transpose (V^T as the K-major GEMM operand).
// ------------------------------------------------------------------------------------------------------------------
namespace b200 {

// one block per row; in: fp32 [rows][lds] (already scaled), out: bf16 [rows][ldo]; cols % 4 == 0
__global__ void softmax_rows_kernel(const float* __restrict__ in, int64_t lds, __nv_bfloat16* __restrict__ out,
                                    int64_t ldo, int cols) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const float4* src = reinterpret_cast<const float4*>(in + row * lds);
  const int nv = cols >> 2;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const float4 v = __ldg(src + i);
    mx = fmaxf(mx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const float4 v = __ldg(src + i);
    sum += __expf(v.x - mx) + __expf(v.y - mx) + __expf(v.z - mx) + __expf(v.w - mx);
  }
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
  const float inv = 1.0f / tot;
  uint2* dst = reinterpret_cast<uint2*>(out + row * ldo);
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const float4 v = __ldg(src + i);
    dst[i] = make_uint2(pack_bf16x2(__expf(v.x - mx) * inv, __expf(v.y - mx) * inv),
                        pack_bf16x2(__expf(v.z - mx) * inv, __expf(v.w - mx) * inv));
  }
}

// out[c][r] = in[r][c]; 32 x 32 tiles through shared memory
__global__ void transpose_kernel(const __nv_bfloat16* __restrict__ in, int64_t ldi, __nv_bfloat16* __restrict__ out,
                                 int64_t ldo, int rows, int cols) {
  __shared__ __nv_bfloat16 tile[32][34];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    if (r < rows && c < cols) tile[i][threadIdx.x] = in[(int64_t)r * ldi + c];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < rows && c < cols) out[(int64_t)c * ldo + r] = tile[threadIdx.x][i];
  }
}

// One DDIM step (eta = 0) of one randomized-blending chunk with the classifier-free-guidance combine, written straight
// into the blended latent (reference code/i2v_enhance/pipeline_i2vgen_xl.py:868-903; scheduler arithmetic restated
// from diffusers==0.30.2 DDIMScheduler.step).  Layout [C][frames][hw] fp32 (batch 1).  noise: [2 or 1][C][cs][hw].
__global__ void ddim_blend_step_kernel(const float* __restrict__ noise, const float* __restrict__ lat,
                                       float* __restrict__ out, int64_t n, int cs, int64_t hw, int lat_frames,
                                       int lat_start, int out_frames, int out_start, int offset, int cfg,
                                       float guidance, float sa, float sb, float sap, float dir, int v_pred) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t px = i % hw;
  const int f = (int)((i / hw) % cs);
  const int64_t c = i / (hw * cs);
  if (f < offset) return;
  float e = noise[i];
  if (cfg) e = e + guidance * (noise[n + i] - e);                       // uncond + g (text - uncond)
  const float x = lat[(c * lat_frames + lat_start + f) * hw + px];
  float x0, eps;
  if (v_pred) {
    x0 = sa * x - sb * e;
    eps = sa * e + sb * x;
  } else {
    x0 = (x - sb * e) / sa;
    eps = e;
  }
  out[(c * out_frames + out_start + f) * hw + px] = sap * x0 + dir * eps;
}

// Frames for the media container: float NCHW in [vmin, vmax] -> uint8 NHWC, exactly the arithmetic of the reference's
// torch2np (code/lib/farancia/libimage/iimage.py:21-39): 255 * (clip(x) - vmin) / (vmax - vmin), truncated to uint8.
__global__ void frames_to_uint8_kernel(const float* __restrict__ x, uint8_t* __restrict__ out, int64_t n, int c,
                                       int64_t hw, float vmin, float vmax) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // over (frame, pixel)
  if (i >= n * hw) return;
  const int64_t f = i / hw, px = i % hw;
  for (int ch = 0; ch < c; ++ch) {
    float v = x[(f * c + ch) * hw + px];
    v = fminf(fmaxf(v, vmin), vmax);
    v = 255.0f * (v - vmin) / (vmax - vmin);   // same operation order as the reference expression (IEEE division)
    out[i * c + ch] = (uint8_t)v;               // float -> uint8 truncates toward zero, like torch's .to(torch.uint8)
  }
}

// The uint8 image round trip of the first chunk, in place of diffusers' postprocess_video(output_type="pil") followed by
// torchvision's ToTensor() and `* 2.0 - 1` (streaming_svd.py:390-393).  Each step is one fp32 operation rounded to
// nearest, in the reference's order; the explicit _rn intrinsics keep nvcc from contracting them into FMAs.
// 255 is not a power of two, so neither `* 255` nor `/ 255` is exact and the order matters.
__global__ void frames_quantize_kernel(const float* x, float* out, int64_t n) {  // out may alias x
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = __fadd_rn(__fdiv_rn(x[i], 2.0f), 0.5f);   // x / 2 + 0.5
  v = fminf(fmaxf(v, 0.0f), 1.0f);                    // .clamp(0, 1)
  v = rintf(__fmul_rn(v, 255.0f));                    // (v * 255).round(): numpy rounds half to even, as rintf does
  v = __fdiv_rn(v, 255.0f);                           // ToTensor: uint8 -> float / 255
  out[i] = __fsub_rn(__fmul_rn(v, 2.0f), 1.0f);       // * 2.0 - 1
}

}  // namespace b200

extern "C" {

int b200svd_frames_to_uint8(const float* x, void* out, int64_t n, int c, int64_t hw, float vmin, float vmax,
                            void* stream) {
  using namespace b200;
  if (!(vmax > vmin) || c < 1 || c > 4) {
    set_error("frames_to_uint8: need vmax > vmin and 1..4 channels");
    return 1;
  }
  const int64_t tot = n * hw;
  if (tot <= 0) return 0;
  frames_to_uint8_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, reinterpret_cast<uint8_t*>(out), n, c, hw, vmin, vmax);
  B200_CHECK_LAUNCH("frames_to_uint8");
  return 0;
}

int b200svd_frames_quantize(const float* x, float* out, int64_t n, void* stream) {
  using namespace b200;
  if (n < 0) {
    set_error("frames_quantize: negative element count");
    return 1;
  }
  if (n == 0) return 0;
  frames_quantize_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, out, n);
  B200_CHECK_LAUNCH("frames_quantize");
  return 0;
}

int b200svd_ddim_blend_step(const float* noise, const float* lat, float* out, int channels, int cs, int64_t hw,
                            int lat_frames, int lat_start, int out_frames, int out_start, int offset, int cfg,
                            float guidance, float alpha_t, float alpha_prev, int v_pred, void* stream) {
  using namespace b200;
  if (cs < 1 || offset < 0 || offset > cs || lat_start < 0 || lat_start + cs > lat_frames || out_start < 0 ||
      out_start + cs > out_frames) {
    set_error("ddim_blend_step: bad frame window (cs %d offset %d lat %d+%d/%d out %d+%d/%d)", cs, offset, lat_start, cs,
              lat_frames, out_start, cs, out_frames);
    return 1;
  }
  if (!(alpha_t > 0.f) || alpha_t > 1.f || alpha_prev < 0.f || alpha_prev > 1.f) {
    set_error("ddim_blend_step: alphas_cumprod out of range");
    return 1;
  }
  const int64_t n = (int64_t)channels * cs * hw;
  if (n <= 0) return 0;
  ddim_blend_step_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      noise, lat, out, n, cs, hw, lat_frames, lat_start, out_frames, out_start, offset, cfg, guidance, sqrtf(alpha_t),
      sqrtf(1.f - alpha_t), sqrtf(alpha_prev), sqrtf(1.f - alpha_prev), v_pred);
  B200_CHECK_LAUNCH("ddim_blend_step");
  return 0;
}

int b200svd_softmax_rows(const float* in, int64_t lds, void* out, int64_t ldo, int64_t rows, int cols, void* stream) {
  using namespace b200;
  if (cols % 4 || lds % 4 || ldo % 4) {
    set_error("softmax_rows: cols and leading dims must be multiples of 4");
    return 1;
  }
  if (rows <= 0 || cols <= 0) return 0;
  if (!aligned(in, 16) || !aligned(out, 8)) {  // float4 loads, 4 x bf16 (8-byte) stores
    set_error("softmax_rows: in must be 16-byte and out 8-byte aligned");
    return 1;
  }
  softmax_rows_kernel<<<(unsigned)rows, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      in, lds, reinterpret_cast<__nv_bfloat16*>(out), ldo, cols);
  B200_CHECK_LAUNCH("softmax_rows");
  return 0;
}

int b200svd_transpose(const void* in, int64_t ldi, void* out, int64_t ldo, int rows, int cols, void* stream) {
  using namespace b200;
  if (rows <= 0 || cols <= 0) return 0;
  dim3 grid((cols + 31) / 32, (rows + 31) / 32), block(32, 8);
  transpose_kernel<<<grid, block, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(in), ldi, reinterpret_cast<__nv_bfloat16*>(out), ldo, rows, cols);
  B200_CHECK_LAUNCH("transpose");
  return 0;
}

int b200svd_sampler_prepare(const float* x, float* xin2, int64_t rows, int64_t chw, float c_in, void* stream) {
  using namespace b200;
  const int64_t n = rows * chw;
  if (n <= 0) return 0;
  sampler_prepare_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, xin2, n,
                                                                                                         c_in);
  B200_CHECK_LAUNCH("sampler_prepare");
  return 0;
}

int b200svd_sampler_step(const float* net, const float* x, float* x_next, int64_t rows, int64_t chw, int num_frames,
                         const float* scale, float c_skip, float c_out, float sigma, float next_sigma, void* stream) {
  using namespace b200;
  if (num_frames < 1 || rows % num_frames != 0) {
    set_error("sampler_step: rows (%lld) must be a multiple of num_frames (%d)", (long long)rows, num_frames);
    return 1;
  }
  if (!(sigma > 0.f)) {
    set_error("sampler_step: sigma must be positive");
    return 1;
  }
  const int64_t n = rows * chw;
  if (n <= 0) return 0;
  sampler_step_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      net, x, x_next, n, chw, num_frames, scale, c_skip, c_out, sigma, next_sigma);
  B200_CHECK_LAUNCH("sampler_step");
  return 0;
}

}  // extern "C"
