// GroupNorm (32 groups, channel-last) and LayerNorm kernels — HBM-bound, 16-byte vectorised, fp32 statistics.
//
// Replaces: GroupNorm32 (reference code/models/svd/sgm/modules/diffusionmodules/util.py:274-276, eps 1e-5),
// Normalize (attention.py:132-135, eps 1e-6), the CAM joint (C/32,F,H,W) GroupNorm (code/models/cam/conditioning.py:57-59),
// nn.LayerNorm (attention.py:528-530, video_attention.py:59,87,101-102; controlnet.py:113-118).
#include <cuda_bf16.h>
#include <limits.h>

#include "../../include/b200svd.h"
#include "common.h"
#include "ptx.cuh"

namespace b200 {

// ------------------------------------------------------------------------------------------------------------
// GroupNorm statistics -> sums [N][32][2] (double: sum, sum of squares), deterministic (fixed summation order, no
// floating-point atomics): every block folds its per-channel fp32 sums into 32 group partials in double and writes
// them to partial[n][chunk][32][2]; the LAST block of sample n (atomic ticket) adds the chunk partials of the sample
// in chunk order.  grid = (chunks, N).
// ------------------------------------------------------------------------------------------------------------

// sm [rstep][2][C]: per-channel sums (sum, then sum of squares) of the block; threads 0-63 each add one group's
// channels, each channel's rstep copies in order in fp32, then the channels in order in double.
__device__ __forceinline__ void gn_fold_groups(const float* sm, int C, int rstep, double* __restrict__ partial, int n) {
  if (threadIdx.x < 64) {
    const int g = threadIdx.x & 31, which = threadIdx.x >> 5;  // which: 0 = sum, 1 = sum of squares
    const int cpg = C >> 5;
    double a = 0.0;
    for (int j = 0; j < cpg; ++j) {
      float c = 0.f;
      for (int r = 0; r < rstep; ++r) c += sm[(size_t)r * 2 * C + which * C + g * cpg + j];
      a += (double)c;
    }
    partial[(((int64_t)n * gridDim.x + blockIdx.x) * 32 + g) * 2 + which] = a;
  }
}

// True, in every thread, in the block that finishes sample n last; that block resets the sample's ticket counter
// for the next launch.
__device__ __forceinline__ bool gn_last_block(int* __restrict__ counters, int n) {
  __shared__ int is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int ticket = atomicAdd(&counters[n], 1);
    is_last = (ticket == (int)gridDim.x - 1);
    if (is_last) counters[n] = 0;
  }
  __syncthreads();
  if (is_last) __threadfence();
  return is_last;
}

// The last block's reduction of sample n's chunk partials into sums[n], spread over the whole block: thread t owns
// pair t % 64 and the chunks congruent to t / 64 modulo parts = blockDim / 64 (>= 2); the parts are then added in
// order.  W independent accumulators, folded pairwise, keep W loads in flight per thread (the chain of dependent
// double adds over up to ~1000 chunk partials, one L2 round trip each, used to dominate the launch for few, large
// samples); the summation order stays fixed.  dsm: parts * 64 doubles.
template <int W>
__device__ __forceinline__ void gn_reduce_chunks(const double* __restrict__ partial, int n, double* dsm,
                                                 double* __restrict__ sums) {
  const int chunks = gridDim.x, parts = blockDim.x / 64;
  const int pr = threadIdx.x % 64, part = threadIdx.x / 64;
  if (part < parts) {
    const double* src = partial + (int64_t)n * chunks * 64 + (pr & 31) * 2 + (pr >> 5);
    double a[W];
#pragma unroll
    for (int i = 0; i < W; ++i) a[i] = 0.0;
    int c = part;
    for (; c + (W - 1) * parts < chunks; c += W * parts) {
#pragma unroll
      for (int i = 0; i < W; ++i) a[i] += src[(int64_t)(c + i * parts) * 64];
    }
    for (; c < chunks; c += parts) a[0] += src[(int64_t)c * 64];
#pragma unroll
    for (int w = W / 2; w > 0; w >>= 1)
#pragma unroll
      for (int i = 0; i < w; ++i) a[i] += a[i + w];
    dsm[part * 64 + pr] = a[0];
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    double a = 0.0;
    for (int q = 0; q < parts; ++q) a += dsm[q * 64 + threadIdx.x];
    sums[((int64_t)n * 32 + (threadIdx.x & 31)) * 2 + (threadIdx.x >> 5)] = a;
  }
}

// Calls f(p, u) for the rows p, p + rstep, ... below p1, u the 16 bytes at row p of xb; 4 loads in flight per thread.
template <class F>
__device__ __forceinline__ void gn_for_rows(const __nv_bfloat16* xb, int64_t ldx, int p, int p1, int rstep, F&& f) {
  constexpr int U = 4;
  for (; p + (U - 1) * rstep < p1; p += U * rstep) {
    uint4 u[U];
#pragma unroll
    for (int i = 0; i < U; ++i) u[i] = __ldg(reinterpret_cast<const uint4*>(xb + (int64_t)(p + i * rstep) * ldx));
#pragma unroll
    for (int i = 0; i < U; ++i) f(p + i * rstep, u[i]);
  }
  for (; p < p1; p += rstep) f(p, __ldg(reinterpret_cast<const uint4*>(xb + (int64_t)p * ldx)));
}

// x [N][P][C] bf16 (row stride ldx).  block = (C/8) * rows_per_iter threads; each thread owns one 8-channel vector
// column: thread partials -> smem [rstep][2][C] -> gn_fold_groups.
__global__ void gn_stats_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, int P, int C, int rows_per_chunk,
                                double* __restrict__ sums, double* __restrict__ partial, int* __restrict__ counters) {
  extern __shared__ float sm[];  // [rstep][2][C]; the last block reuses it for blockDim / 64 * 64 doubles
  const int vecs = C >> 3;
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * rows_per_chunk;
  const int p1 = min(P, p0 + rows_per_chunk);
  const int v = threadIdx.x % vecs;
  const int r0 = threadIdx.x / vecs;
  const int rstep = blockDim.x / vecs;
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  gn_for_rows(x + ((int64_t)n * P) * ldx + v * 8, ldx, p0 + r0, p1, rstep, [&](int, const uint4& u) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = bf16_lo(w[j]), b = bf16_hi(w[j]);
      s[2 * j] += a;
      q[2 * j] += a * a;
      s[2 * j + 1] += b;
      q[2 * j + 1] += b * b;
    }
  });
  float* mine = sm + (size_t)r0 * 2 * C;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    mine[v * 8 + j] = s[j];
    mine[C + v * 8 + j] = q[j];
  }
  __syncthreads();
  gn_fold_groups(sm, C, rstep, partial, n);
  if (gn_last_block(counters, n)) gn_reduce_chunks<16>(partial, n, reinterpret_cast<double*>(sm), sums);
}

// From the per-quadrant partials written by the GEMM epilogue (mtgemm.cu, gn_part): part [n_slots][ld][2] fp32 (sum,
// sum of squares per channel over the <= 32 rows of a slot), slot_sample [n_slots].  A block takes 64 slots and adds
// those of ITS sample in slot order.
constexpr int GNP_SLOTS = 64;
constexpr int GNP_THREADS = 256;
__global__ void __launch_bounds__(GNP_THREADS)
gn_stats_partials_kernel(const float2* __restrict__ part, const int* __restrict__ slot_sample, int64_t n_slots,
                         int64_t ld, int C, double* __restrict__ sums, double* __restrict__ partial,
                         int* __restrict__ counters) {
  extern __shared__ float sm[];  // [2][C]; the last block reuses it for 4 * 64 doubles (C >= 256: checked on host)
  __shared__ int hit[GNP_SLOTS];
  const int n = blockIdx.y;
  const int64_t s0 = (int64_t)blockIdx.x * GNP_SLOTS;
  if (threadIdx.x < GNP_SLOTS) {
    const int64_t sl = s0 + threadIdx.x;
    hit[threadIdx.x] = (sl < n_slots && slot_sample[sl] == n) ? 1 : 0;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += GNP_THREADS) {
    float a = 0.f, b = 0.f;
    for (int i = 0; i < GNP_SLOTS; ++i) {
      if (hit[i]) {
        const float2 v = __ldg(part + (s0 + i) * ld + c);
        a += v.x;
        b += v.y;
      }
    }
    sm[c] = a;
    sm[C + c] = b;
  }
  __syncthreads();
  gn_fold_groups(sm, C, 1, partial, n);
  if (gn_last_block(counters, n)) gn_reduce_chunks<8>(partial, n, reinterpret_cast<double*>(sm), sums);
}

// y = [silu]((x - mean) * rstd * gamma + beta), bf16 out (row stride ldy).
__global__ void gn_apply_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, __nv_bfloat16* __restrict__ y,
                                int64_t ldy, int P, int C, int rows_per_chunk, const double* __restrict__ sums,
                                const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                int apply_silu) {
  const int vecs = C >> 3;
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * rows_per_chunk;
  const int p1 = min(P, p0 + rows_per_chunk);
  const int v = threadIdx.x % vecs;
  const int r0 = threadIdx.x / vecs;
  const int rstep = blockDim.x / vecs;
  const int cpg = C >> 5;
  const double cnt = (double)P * (double)cpg;
  float sc[8], sh[8];
  int gprev = -1;
  float mean_f = 0.f, rstd = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = v * 8 + j;
    const int g = c / cpg;
    if (g != gprev) {  // the double-precision statistics are evaluated once per distinct group (<= 2 for C >= 256)
      const double su = sums[((int64_t)n * 32 + g) * 2], sq = sums[((int64_t)n * 32 + g) * 2 + 1];
      const double mean = su / cnt;
      double var = sq / cnt - mean * mean;
      if (var < 0.0) var = 0.0;
      rstd = rsqrtf((float)var + eps);
      mean_f = (float)mean;
      gprev = g;
    }
    const float ga = __ldg(gamma + c), be = __ldg(beta + c);
    sc[j] = rstd * ga;
    sh[j] = be - mean_f * rstd * ga;
  }
  __nv_bfloat16* yb = y + ((int64_t)n * P) * ldy + v * 8;
  gn_for_rows(x + ((int64_t)n * P) * ldx + v * 8, ldx, p0 + r0, p1, rstep, [&](int p, const uint4& u) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float a = bf16_lo(w[j]) * sc[2 * j] + sh[2 * j];
      float b = bf16_hi(w[j]) * sc[2 * j + 1] + sh[2 * j + 1];
      if (apply_silu) {
        a = silu_fast(a);
        b = silu_fast(b);
      }
      o[j] = pack_bf16x2(a, b);
    }
    *reinterpret_cast<uint4*>(yb + (int64_t)p * ldy) = make_uint4(o[0], o[1], o[2], o[3]);
  });
}

// ------------------------------------------------------------------------------------------------------------
// LayerNorm over the channel dim, fp32 two-pass statistics:  y = [silu](((x [+ fvec[row/rpf]]) - mean) * rstd * gamma
// + beta).  With xsum, also writes xsum = bf16(x + fvec), which the caller uses as the residual stream, and normalises
// that rounded sum.  LPR lanes own one row (32 / LPR rows per warp), lane li its 16-byte vectors li + i * LPR for
// i < V; vectors past C/8 are skipped.  VEC: gamma, beta and fvec are 16-byte aligned and load as float4 pairs, else
// one float at a time.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void load8(const float* __restrict__ p, float (&o)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w;
  o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}

template <int LPR, int V, bool VEC>
__global__ void __launch_bounds__(256) layernorm_kernel(
    const __nv_bfloat16* __restrict__ x, int64_t ldx, __nv_bfloat16* __restrict__ y, int64_t ldy, int64_t rows, int C,
    const float* __restrict__ gamma, const float* __restrict__ beta, float eps, const float* __restrict__ fvec,
    int64_t ldf, int rows_per_frame, __nv_bfloat16* __restrict__ xsum, int64_t ldxs, int apply_silu) {
  const int lane = threadIdx.x & 31, li = lane % LPR;
  const int64_t row = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * (32 / LPR) + lane / LPR;
  if (LPR == 32 && row >= rows) return;
  // a row past the end (LPR < 32) stores nothing, but reads the last row so that its lanes still take part in their
  // warp's shuffles
  const bool active = row < rows;
  const int64_t rr = active ? row : rows - 1;
  // V = 5 runs only at C = 40 LPR: every vector is owned, and the constant lets the compiler drop the checks
  const int vecs = V == 5 ? 5 * LPR : C >> 3;
  auto own = [&](int i) { return li + i * LPR < vecs; };
  const __nv_bfloat16* xr = x + rr * ldx;
  const float* fr = fvec ? fvec + (rr / rows_per_frame) * ldf : nullptr;
  uint4 u[V];  // every load issued before the first use
#pragma unroll
  for (int i = 0; i < V; ++i)
    if (own(i)) u[i] = __ldg(reinterpret_cast<const uint4*>(xr + (li + i * LPR) * 8));
  float val[V][8];
#pragma unroll
  for (int i = 0; i < V; ++i) {
    if (!own(i)) continue;
    const int c0 = (li + i * LPR) * 8;
    const uint32_t w[4] = {u[i].x, u[i].y, u[i].z, u[i].w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      val[i][2 * j] = bf16_lo(w[j]);
      val[i][2 * j + 1] = bf16_hi(w[j]);
    }
    if (fr) {
      float f[8];
      if constexpr (VEC) load8(fr + c0, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) val[i][j] += VEC ? f[j] : __ldg(fr + c0 + j);
    }
  }
  if (fr && xsum) {
    // every per-frame load is issued before the first store
#pragma unroll
    for (int i = 0; i < V; ++i) {
      if (!active || !own(i)) continue;
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] = pack_bf16x2(val[i][2 * j], val[i][2 * j + 1]);
      *reinterpret_cast<uint4*>(xsum + row * ldxs + (li + i * LPR) * 8) = make_uint4(o[0], o[1], o[2], o[3]);
      // the residual stream is the bf16-rounded sum; normalise exactly what the consumer will see
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        val[i][2 * j] = bf16_lo(o[j]);
        val[i][2 * j + 1] = bf16_hi(o[j]);
      }
    }
  }
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i)
    if (own(i))
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += val[i][j];
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i)
    if (own(i))
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = val[i][j] - mean;
        sq += d * d;
      }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / (float)C + eps);
  __nv_bfloat16* yr = y + row * ldy;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    if (!active || !own(i)) continue;
    const int c0 = (li + i * LPR) * 8;
    float g[8], b[8], o8[8];
    if constexpr (VEC) {
      load8(gamma + c0, g);
      load8(beta + c0, b);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float t = (val[i][j] - mean) * rstd * (VEC ? g[j] : __ldg(gamma + c0 + j)) + (VEC ? b[j] : __ldg(beta + c0 + j));
      if (apply_silu) t = silu_fast(t);
      o8[j] = t;
    }
    *reinterpret_cast<uint4*>(yr + c0) = make_uint4(pack_bf16x2(o8[0], o8[1]), pack_bf16x2(o8[2], o8[3]),
                                                    pack_bf16x2(o8[4], o8[5]), pack_bf16x2(o8[6], o8[7]));
  }
}

static int gn_geometry(int C, int64_t n, int P, int* threads, int* rows_per_chunk, int* chunks) {
  if (C % 8 != 0 || C % 32 != 0) return 1;
  const int vecs = C / 8;
  if (vecs > 1024) return 1;
  int rpi = 256 / vecs;
  if (rpi < 1) rpi = 1;
  *threads = vecs * rpi;
  // Enough CTAs to cover the GPU several times over (these kernels are latency-bound otherwise): aim for
  // >= 8 CTAs per SM, but never less than one 4-deep unrolled batch of rows per thread, never more than 256 rows.
  const int min_rpc = rpi * 4;
  const int64_t target_ctas = (int64_t)sm_count() * 8;
  int64_t rpc = ((int64_t)P * n + target_ctas - 1) / target_ctas;
  rpc = ((rpc + min_rpc - 1) / min_rpc) * min_rpc;
  if (rpc < min_rpc) rpc = min_rpc;
  int64_t cap = 256;
  while ((int64_t)P / cap > 2048 && cap < 4096) cap *= 2;  // bound the number of chunk partials per sample
  if (rpc > cap) rpc = cap / min_rpc * min_rpc > 0 ? cap / min_rpc * min_rpc : min_rpc;
  if (rpc > P) rpc = P;
  *rows_per_chunk = (int)rpc;
  *chunks = (int)((P + rpc - 1) / rpc);
  return 0;
}

// Shapes every GroupNorm entry point accepts: 32 <= c <= 8192 in whole groups of channels (gn_geometry), p within the
// kernels' int row index, n within gridDim.y.  n = 0 or p = 0 is valid and launches nothing.
static int gn_check_shape(const char* who, int64_t n, int64_t p, int c) {
  if (c < 32 || c > 8192 || c % 32 != 0) {
    set_error("%s: unsupported channel count %d (need a multiple of 32, 32 <= c <= 8192)", who, c);
    return 1;
  }
  if (n < 0 || n > 65535 || p < 0 || p > INT_MAX) {
    set_error("%s: need 0 <= n <= 65535 and 0 <= p <= %d (n %lld, p %lld)", who, INT_MAX, (long long)n, (long long)p);
    return 1;
  }
  return 0;
}

// Lets kernel K take smem bytes of dynamic shared memory: past the default 48 KB the limit is raised, per device, to
// the largest size asked for so far.
template <auto K>
static int allow_dynamic_smem(size_t smem, const char* what) {
  static size_t smem_set_dev[B200_MAX_DEVICES] = {};
  size_t& smem_set = smem_set_dev[dev_slot()];
  if (smem > 48 * 1024 && smem > smem_set) {
    cudaError_t e = cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_fail(e, what);
    smem_set = smem;
  }
  return 0;
}

using LayerNormKernel = decltype(&layernorm_kernel<32, 1, false>);

}  // namespace b200

extern "C" {

// sums: n*32*2 doubles (out).  scratch: at least b200svd_gn_scratch_doubles(n, p, c) doubles.  counters: n int32,
// zero-initialised once by the caller (the kernel leaves them zero).
int64_t b200svd_gn_scratch_doubles(int64_t n, int64_t p, int c) {
  using namespace b200;
  if (gn_check_shape("gn_scratch_doubles", n, p, c)) return -1;
  if (n == 0 || p == 0) return 0;
  int threads, rpc, chunks;
  if (gn_geometry(c, n, (int)p, &threads, &rpc, &chunks)) return -1;
  return n * (int64_t)chunks * 64;
}

int b200svd_gn_stats_partials(const float* gn_part, const int32_t* gn_slot_sample, int64_t n_slots, int64_t gn_ld,
                              int c, int64_t n, void* sums, void* scratch, void* counters, void* stream) {
  using namespace b200;
  if (c % 32 != 0 || c < 256 || c > 8192 || gn_ld < c || n_slots < 1 || n < 1 || n > 65535) {
    set_error("gn_stats_partials: need 256 <= c <= 8192, c %% 32 == 0, gn_ld >= c, n_slots >= 1, 1 <= n <= 65535 "
              "(c %d, ld %lld, slots %lld, n %lld)", c, (long long)gn_ld, (long long)n_slots, (long long)n);
    return 1;
  }
  const int64_t chunks = (n_slots + GNP_SLOTS - 1) / GNP_SLOTS;
  dim3 grid((unsigned)chunks, (unsigned)n);
  const size_t smem = (size_t)2 * c * sizeof(float);
  if (allow_dynamic_smem<gn_stats_partials_kernel>(smem, "cudaFuncSetAttribute(gn_stats_partials)")) return 1;
  gn_stats_partials_kernel<<<grid, GNP_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float2*>(gn_part), gn_slot_sample, n_slots, gn_ld, c, reinterpret_cast<double*>(sums),
      reinterpret_cast<double*>(scratch), reinterpret_cast<int*>(counters));
  B200_CHECK_LAUNCH("gn_stats_partials");
  return 0;
}

int b200svd_gn_stats(const void* x, int64_t ldx, int64_t n, int64_t p, int c, void* sums, void* scratch,
                     void* counters, void* stream) {
  using namespace b200;
  if (gn_check_shape("gn_stats", n, p, c)) return 1;
  if (ldx % 8 != 0) {
    set_error("gn_stats: ldx must be a multiple of 8");
    return 1;
  }
  if (n == 0 || p == 0) return 0;
  if (!aligned(x, 16)) {  // 16-byte (8-channel) loads
    set_error("gn_stats: x must be 16-byte aligned");
    return 1;
  }
  int threads, rpc, chunks;
  if (gn_geometry(c, n, (int)p, &threads, &rpc, &chunks)) {
    set_error("gn_stats: unsupported channel count %d", c);
    return 1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  dim3 grid(chunks, (unsigned)n);
  const int rstep = threads / (c / 8);
  const size_t smem = (size_t)rstep * 2 * c * sizeof(float);
  if (allow_dynamic_smem<gn_stats_kernel>(smem, "gn_stats smem attribute")) return 1;
  gn_stats_kernel<<<grid, threads, smem, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), ldx, (int)p, c, rpc,
                                             reinterpret_cast<double*>(sums), reinterpret_cast<double*>(scratch),
                                             reinterpret_cast<int*>(counters));
  B200_CHECK_LAUNCH("gn_stats");
  return 0;
}

int b200svd_gn_apply(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t n, int64_t p, int c, const void* sums,
                     const float* gamma, const float* beta, float eps, int apply_silu, void* stream) {
  using namespace b200;
  if (gn_check_shape("gn_apply", n, p, c)) return 1;
  if (ldx % 8 != 0 || ldy % 8 != 0) {
    set_error("gn_apply: leading dims must be multiples of 8");
    return 1;
  }
  if (n == 0 || p == 0) return 0;
  if (!aligned(x, 16) || !aligned(y, 16)) {  // 16-byte (8-channel) loads and stores
    set_error("gn_apply: x and y must be 16-byte aligned");
    return 1;
  }
  int threads, rpc, chunks;
  if (gn_geometry(c, n, (int)p, &threads, &rpc, &chunks)) {
    set_error("gn_apply: unsupported channel count %d", c);
    return 1;
  }
  // one thread per 8-channel column: past c = 2048 a block has c / 8 threads, and the kernel's register use caps the
  // block below 1024 threads (at 66 registers, 896: c <= 7168)
  static int max_threads_dev[B200_MAX_DEVICES] = {};
  int& max_threads = max_threads_dev[dev_slot()];
  if (max_threads == 0) {
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, gn_apply_kernel);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncGetAttributes(gn_apply)");
    max_threads = fa.maxThreadsPerBlock;
  }
  if (threads > max_threads) {
    set_error("gn_apply: c = %d needs %d threads per block, the kernel launches at most %d (c <= %d)", c, threads,
              max_threads, max_threads / 4 * 32);
    return 1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  dim3 grid(chunks, (unsigned)n);
  gn_apply_kernel<<<grid, threads, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), ldx,
                                            reinterpret_cast<__nv_bfloat16*>(y), ldy, (int)p, c, rpc,
                                            reinterpret_cast<const double*>(sums), gamma, beta, eps, apply_silu);
  B200_CHECK_LAUNCH("gn_apply");
  return 0;
}

int b200svd_layernorm(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int c, const float* gamma,
                      const float* beta, float eps, const float* fvec, int64_t ldf, int rows_per_frame, void* xsum,
                      int64_t ldxs, int apply_silu, void* stream) {
  using namespace b200;
  if (c < 0 || c % 8 != 0 || c > 8 * 32 * 8) {
    set_error("layernorm: unsupported width %d (multiple of 8, <= 2048)", c);
    return 1;
  }
  if (ldx % 8 != 0 || ldy % 8 != 0 || (xsum && ldxs % 8 != 0)) {
    set_error("layernorm: leading dims must be multiples of 8");
    return 1;
  }
  if (xsum && !fvec) {  // the kernels write xsum = bf16(x + fvec) only while adding fvec
    set_error("layernorm: xsum needs fvec (xsum = bf16(x + fvec)); pass both or neither");
    return 1;
  }
  if (rows <= 0 || c == 0) return 0;
  // x, y and xsum move in 16-byte vectors; gamma / beta / fvec fall back to the scalar kernel below when misaligned
  if (!aligned(x, 16) || !aligned(y, 16) || !aligned(xsum, 16)) {
    set_error("layernorm: x, y and xsum must be 16-byte aligned");
    return 1;
  }
  if (rows_per_frame <= 0) rows_per_frame = 1;
  const int vecs = c / 8;
  const bool f_ok = (fvec == nullptr) || (ldf % 4 == 0 && (reinterpret_cast<uintptr_t>(fvec) & 15) == 0);
  const bool gb_ok = ((reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) & 15) == 0;
  // layernorm_kernel<lanes per row, vectors per lane, float4 parameter loads>
  LayerNormKernel kernel;
  int lpr;
  const char* name;
  if ((c == 320 || c == 640 || c == 1280) && f_ok && gb_ok) {  // C = 40 * LPR: 5 vectors per lane, no idle lanes
    lpr = c / 40;
    kernel = lpr == 8 ? layernorm_kernel<8, 5, true> : lpr == 16 ? layernorm_kernel<16, 5, true>
                                                                 : layernorm_kernel<32, 5, true>;
    name = "layernorm5";
  } else if (vecs <= 32 && fvec == nullptr && xsum == nullptr && gb_ok) {
    // narrow rows (C <= 256: the ControlNet condition-embedding norms): a warp issues full-width loads for several rows
    lpr = vecs <= 4 ? 4 : vecs <= 8 ? 8 : vecs <= 16 ? 16 : 32;
    kernel = lpr == 4    ? layernorm_kernel<4, 1, true>
             : lpr == 8  ? layernorm_kernel<8, 1, true>
             : lpr == 16 ? layernorm_kernel<16, 1, true>
                         : layernorm_kernel<32, 1, true>;
    name = "layernorm_narrow";
  } else {
    lpr = 32;
    kernel = vecs <= 32    ? layernorm_kernel<32, 1, false>
             : vecs <= 64  ? layernorm_kernel<32, 2, false>
             : vecs <= 128 ? layernorm_kernel<32, 4, false>
                           : layernorm_kernel<32, 8, false>;
    name = "layernorm";
  }
  const int wpb = 8;
  const int64_t rows_per_block = (int64_t)wpb * (32 / lpr);
  const unsigned grid = (unsigned)((rows + rows_per_block - 1) / rows_per_block);
  kernel<<<grid, wpb * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, reinterpret_cast<__nv_bfloat16*>(y), ldy, rows, c, gamma, beta,
      eps, fvec, ldf, rows_per_frame, reinterpret_cast<__nv_bfloat16*>(xsum), ldxs, apply_silu);
  B200_CHECK_LAUNCH(name);
  return 0;
}

}  // extern "C"
