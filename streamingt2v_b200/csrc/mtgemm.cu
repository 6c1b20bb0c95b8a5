// Multi-tap tensor-core GEMM for sm_90a.
// TMA (rank-5 activation view) -> smem stage ring (128B swizzle) -> wgmma (fp32 accumulators in registers)
// -> fused epilogue (bf16 outputs staged through shared memory and written by TMA stores).
// See include/b200svd.h for the contract.
//
// Replaces, underneath StreamingWrapper.forward (reference code/models/diffusion/wrappers.py:23-78):
//   nn.Linear            code/models/svd/sgm/modules/attention.py:94-120,262-351, video_attention.py:23-168
//   Conv2d 3x3 (s1, s2)  code/models/svd/sgm/modules/diffusionmodules/openaimodel.py:107-207,257-305
//   Conv3d (3,1,1)       code/models/diffusion/video_model.py:46-59 (ResBlock dims=3)
//   + their elementwise neighbours (bias, emb add openaimodel.py:346-352, GEGLU attention.py:94-101,
//     residual / AlphaBlender diffusionmodules/util.py:358-370).
//
// Persistent CTAs (one per SM) walk the output tiles with a grid stride (N tile fastest).  Three warpgroups:
//   warpgroup 0     TMA producers: thread 0 loads A/B (the stage ring runs ahead across tiles, so the next tile's
//                   operands stream in while the consumers run the epilogue of the current one); thread 32 loads the
//                   residuals of bf16 outputs into their own ring
//   warpgroups 1-2  consumers: each owns 64 rows of the 128-row tile, issues m64nBNk16 wgmma on the shared B stage
//                   and applies the epilogue to its accumulator registers.  bf16 outputs are written 32 columns at a
//                   time through a shared-memory staging buffer and a TMA store; fp32 outputs are stored directly.
// A convolution tap is a shifted box of the same activation view, so taps and K blocks form one reduction loop.
//
// Two schedules share the producers and the epilogue arithmetic.  "Cooperative" (mtgemm_kernel) is the one above.
// "Alternating" (mtgemm_alt_kernel) gives whole 128 x BN tiles to the consumer warpgroups in turn (warpgroup w takes
// the CTA's tiles w, w + 2, ...), so the epilogue of one tile runs under the MMAs of the next; it is chosen for bf16
// launches of many short-K tiles, where the epilogue is a large share of a tile (b200svd_gemm_schedule).
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/b200svd.h"
#include "common.h"
#include "mtgemm_ring.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace b200 {

struct GemmDev {
  int32_t tap_off[B200SVD_MAX_TAPS][5];
  uint32_t taps, kblocks;
  uint32_t n;  // GEMM N (weight rows)
  uint32_t n_tiles;
  uint32_t total_tiles;
  uint32_t m_ext[3];
  uint32_t m_lb[3];  // log2 of box
  uint32_t m_tiles[3];
  uint32_t m_adim[3];
  int64_t out_rs[3];
  void* out;
  int64_t ldo;
  int32_t out_fp32;
  const float* bias;
  const float* fvec;
  int64_t ldf;
  uint32_t rows_per_frame;
  int32_t act;
  float s_acc;
  const __nv_bfloat16* res1;
  int64_t ld1;
  float s1;
  const __nv_bfloat16* res2;
  int64_t ld2;
  float s2;
  float* gn_part;  // GroupNorm partial sums of the output, see b200svd.h
  int32_t* gn_slot_sample;
  int64_t gn_ld;
  uint32_t gn_rows;
  int32_t staged;      // bf16 output through shared memory and TMA stores (else straight from registers)
  int32_t epi_kind;    // B200SVD_EPI_*: the compile-time epilogue body of a staged launch, 0 = the generic one
  uint32_t stages;     // depth of the A/B stage ring
  uint32_t res_slots;  // depth of the residual ring (bf16 outputs with residuals, else 0)
  uint32_t wg_off[3];  // row-box origin of the second consumer warpgroup's 64 rows (bf16 output stores)
  const float* slope;  // PReLU slope per GEMM column (act = B200SVD_ACT_PRELU)
#ifdef MTGEMM_PHASE_CLOCKS
  long long* phase_buf;  // [CTA][role][PC_N] clock sums, see PhaseClock
#endif
};

// Where a thread's clocks go.  Only the measuring build (-DMTGEMM_PHASE_CLOCKS, scripts/bench_gemm_shapes.py) reads
// the clock: mark(i) adds the time since the previous mark to counter i.  In the product build every call is empty.
enum {
  PC_RING_WAIT = 0,   // producer: waiting for a free stage; consumer: waiting for a full one
  PC_MMA = 1,         // consumer: first wgmma of a stage to the wait that retires it
  PC_RES_WAIT = 2,    // epilogue: waiting for a residual slot
  PC_STORE_WAIT = 3,  // epilogue: until the previous TMA store has read its staging buffer, plus the named barrier
  PC_EPI = 4,         // epilogue: everything else
  PC_OTHER = 5,       // issue work of the producer, stepping over the other warpgroup's tiles
  PC_TOTAL = 7,       // lifetime of the thread
  PC_N = 8
};
#ifdef MTGEMM_PHASE_CLOCKS
struct PhaseClock {
  long long t0, last, acc[PC_N];
  __device__ __forceinline__ PhaseClock() {
    t0 = last = clock64();
#pragma unroll
    for (int i = 0; i < PC_N; ++i) acc[i] = 0;
  }
  __device__ __forceinline__ void mark(int i) {
    const long long n = clock64();
    acc[i] += n - last;
    last = n;
  }
  // role: 0 = A/B producer, 1 and 2 = leader of the consumer warpgroups
  __device__ __forceinline__ void write(long long* buf, int role) {
    if (buf == nullptr) return;
    acc[PC_TOTAL] = clock64() - t0;
#pragma unroll
    for (int i = 0; i < PC_N; ++i) buf[((size_t)blockIdx.x * 3 + role) * PC_N + i] += acc[i];
  }
};
#define PC_BUF(p) ((p).phase_buf)
#else
struct PhaseClock {
  __device__ __forceinline__ void mark(int) {}
  __device__ __forceinline__ void write(long long*, int) {}
};
#define PC_BUF(p) nullptr
#endif

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int NUM_THREADS = 3 * 128;        // producer warpgroup + two consumer warpgroups
constexpr int SMEM_LIMIT = 232448;          // 227 KB of dynamic shared memory per block
constexpr int MAX_STAGES = 6;
constexpr int MIN_STAGES = 3;
// bf16 epilogue: the tile is processed in 32-column sub-tiles (64-byte rows, SWIZZLE_64B)
constexpr int SUB_W = 32;
constexpr int STG_SLOT_BYTES = 64 * SUB_W * 2;    // one warpgroup's 64 rows of one sub-tile: 4 KB
constexpr int STG_SLOTS = 2;                      // staging buffers per consumer warpgroup
constexpr int STG_BYTES = 2 * STG_SLOTS * STG_SLOT_BYTES;
constexpr int RES_SLOT_BYTES = BM * SUB_W * 2;    // one residual sub-tile, both warpgroups: 8 KB
constexpr int MAX_RES_SLOTS = 16;
constexpr int GN_BYTES = 2 * 2 * 2 * SUB_W * 8;  // [warpgroup][buffer][quadrant][column][sum, sum of squares]
constexpr int BAR_BYTES = 512;
constexpr int FIXED_BYTES = STG_BYTES + GN_BYTES + BAR_BYTES;
static_assert(2 * (MAX_STAGES + MAX_RES_SLOTS) * 8 + 16 <= BAR_BYTES, "barrier area and the tile counters");

// Shared memory (offsets in bytes, every region 1024-byte aligned):
//   [0, stages * STAGE_BYTES)   A/B stage ring
//   res_slots * RES_SLOT_BYTES  residual ring (bf16 outputs with residuals)
//   STG_BYTES                   output staging, per consumer warpgroup
//   GN_BYTES                    GroupNorm partials of the partner warp
//   BAR_BYTES                   mbarriers
// The stage count and the residual ring are chosen per launch (launch<BN>): a launch with residuals trades A/B
// stages (not below MIN_STAGES) for a residual ring that holds a whole tile's residuals where it fits.
template <int BN>
struct TileCfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int FIXED = FIXED_BYTES;
  static constexpr int STAGES_FIT = (SMEM_LIMIT - FIXED_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > MAX_STAGES ? MAX_STAGES : STAGES_FIT;
  static constexpr int SUBTILES = BN / SUB_W;
  // accumulator registers per consumer thread: BN / 2; the 256-wide tile needs the producer's registers
  static constexpr int CONSUMER_REGS = BN > 128 ? 232 : 160;
  static constexpr int PRODUCER_REGS = 40;
  static constexpr int RES_SLOTS_AT_MIN = (SMEM_LIMIT - FIXED_BYTES - MIN_STAGES * STAGE_BYTES) / RES_SLOT_BYTES;
  static int res_slots_fit(int stages) { return (SMEM_LIMIT - FIXED_BYTES - stages * STAGE_BYTES) / RES_SLOT_BYTES; }
  static_assert(STAGES >= 4, "pipeline depth without residuals");
  static_assert(RES_SLOTS_AT_MIN >= 2, "two residuals need two ring slots");
  static_assert(STAGES * STAGE_BYTES + FIXED_BYTES <= SMEM_LIMIT, "shared memory budget");
  static_assert(STAGE_BYTES % 1024 == 0, "stage alignment");
  static_assert(BN % SUB_W == 0, "sub-tiles");
};

// Alternating schedule: a consumer warpgroup holds the whole 128 x BN accumulator (BN registers per thread, so
// BN <= 128) and stages 128-row sub-tiles (8 KB, two buffers per warpgroup); no GroupNorm partials.
constexpr int ALT_STG_SLOT_BYTES = BM * SUB_W * 2;
constexpr int ALT_STG_BYTES = 2 * STG_SLOTS * ALT_STG_SLOT_BYTES;
template <int BN>
struct AltCfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int FIXED = ALT_STG_BYTES + BAR_BYTES;
  static constexpr int STAGES_FIT = (SMEM_LIMIT - FIXED) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > MAX_STAGES ? MAX_STAGES : STAGES_FIT;
  static constexpr int SUBTILES = BN / SUB_W;
  static constexpr int CONSUMER_REGS = 232;
  static constexpr int PRODUCER_REGS = 40;
  static constexpr int RES_SLOTS_AT_MIN = (SMEM_LIMIT - FIXED - MIN_STAGES * STAGE_BYTES) / RES_SLOT_BYTES;
  static int res_slots_fit(int stages) { return (SMEM_LIMIT - FIXED - stages * STAGE_BYTES) / RES_SLOT_BYTES; }
  static_assert(BN <= 128, "128 x BN accumulator in one warpgroup's registers");
  static_assert(2 * 128 * CONSUMER_REGS + 128 * PRODUCER_REGS <= 65536, "register file");
  static_assert(STAGES >= 4, "pipeline depth without residuals");
  static_assert(RES_SLOTS_AT_MIN >= 2, "two residuals need two ring slots");
  static_assert(STAGES * STAGE_BYTES + FIXED <= SMEM_LIMIT, "shared memory budget");
  static_assert(STAGE_BYTES % 1024 == 0, "stage alignment");
  static_assert(BN % SUB_W == 0, "sub-tiles");
};

// `tile` enumerates (N tile fastest, then M tile).  An M tile decodes to the box origin of each of the three output
// row dimensions.
__device__ __forceinline__ void decode_tile(const GemmDev& p, uint32_t tile, uint32_t& n_tile, uint32_t& mb1,
                                            uint32_t& mb2, uint32_t& mb3) {
  n_tile = tile % p.n_tiles;
  uint32_t mt = tile / p.n_tiles;
  const uint32_t t1 = mt % p.m_tiles[0];
  mt /= p.m_tiles[0];
  const uint32_t t2 = mt % p.m_tiles[1];
  const uint32_t t3 = mt / p.m_tiles[1];
  mb1 = t1 << p.m_lb[0];
  mb2 = t2 << p.m_lb[1];
  mb3 = t3 << p.m_lb[2];
}

__device__ __forceinline__ float ldg_bf16(const __nv_bfloat16* p) { return __bfloat162float(p[0]); }

// Two adjacent bf16 elements at index i (and i + 1 if `both`): one 32-bit load when aligned.
__device__ __forceinline__ void load_bf16_pair(const __nv_bfloat16* base, int64_t i, bool both, float& a, float& b) {
  if (both && (i & 1) == 0) {
    const uint32_t w = __ldg(reinterpret_cast<const unsigned int*>(base + i));
    a = bf16_lo(w);
    b = bf16_hi(w);
  } else {
    a = ldg_bf16(base + i);
    b = both ? ldg_bf16(base + i + 1) : 0.f;
  }
}

// The epilogue arithmetic after bias and per-frame vector, shared by the fp32 and the bf16 output paths so that both
// round the same fp32 value: activation (GEGLU: value * GELU(gate + gate bias), the gate bias already added; PReLU: g is
// the column's slope), scale.
// Multiplies and fused multiply-adds are written out so that the compiler cannot contract them differently.  An
// activation known at compile time folds the tests away.
__device__ __forceinline__ float epi_act(int act, float s_acc, float v, float g) {
  if (act == B200SVD_ACT_SILU) {
    v = silu_fast(v);
  } else if (act == B200SVD_ACT_GELU) {
    v = gelu_fast(v);
  } else if (act == B200SVD_ACT_GEGLU) {
    v = __fmul_rn(v, gelu_fast(g));
  } else if (act == B200SVD_ACT_PRELU) {
    v = v > 0.f ? v : __fmul_rn(g, v);
  }
  return __fmul_rn(v, s_acc);
}

// byte offset of (row, 4-byte column pair `cp` of 16-byte chunk `ch`) in a 64-byte-row SWIZZLE_64B sub-tile buffer
__device__ __forceinline__ uint32_t sw64_off(uint32_t row, uint32_t ch, uint32_t cp) {
  return row * 64u + ((ch ^ ((row >> 1) & 3u)) << 4) + cp * 4u;
}

// ---- epilogue kinds of the staged bf16 output ----
// Testing activation, bias, per-frame vector and residuals per element, and the global loads sitting between those
// tests, is what a consumer warp would spend its epilogue on.  The combinations the network launches
// (b200svd_gemm_epilogue_kind) are compiled as branch-free bodies instead, one switch per tile picking the body;
// EpiGeneric reads the same flags from the launch parameters and keeps every other combination.  All of them run one
// body (epi_stage_half), whose accessors are constants for a compiled kind, so per element the arithmetic is the same
// operation for operation and the output is bitwise the same.
template <int ACT_, bool BIAS_, bool FVEC_, int NRES_>
struct Epi {
  static constexpr bool GENERIC = false;
  __device__ static int act(const GemmDev&) { return ACT_; }
  __device__ static bool geglu(const GemmDev&) { return ACT_ == B200SVD_ACT_GEGLU; }
  __device__ static bool bias(const GemmDev&) { return BIAS_; }
  __device__ static bool fvec(const GemmDev&) { return FVEC_; }
  __device__ static bool res1(const GemmDev&) { return NRES_ >= 1; }
  __device__ static bool res2(const GemmDev&) { return NRES_ >= 2; }
};
struct EpiGeneric {
  static constexpr bool GENERIC = true;
  __device__ static int act(const GemmDev& p) { return p.act; }
  __device__ static bool geglu(const GemmDev& p) { return p.act == B200SVD_ACT_GEGLU; }
  __device__ static bool bias(const GemmDev& p) { return p.bias != nullptr; }
  __device__ static bool fvec(const GemmDev& p) { return p.fvec != nullptr; }
  __device__ static bool res1(const GemmDev& p) { return p.res1 != nullptr; }
  __device__ static bool res2(const GemmDev& p) { return p.res2 != nullptr; }
};
// X(kind id, activation, bias, per-frame vector, residuals): what the two kernels instantiate
#define MTGEMM_EPI_KINDS(X)                                    \
  X(B200SVD_EPI_PLAIN, B200SVD_ACT_NONE, false, false, 0)      \
  X(B200SVD_EPI_BIAS, B200SVD_ACT_NONE, true, false, 0)        \
  X(B200SVD_EPI_BIAS_RES1, B200SVD_ACT_NONE, true, false, 1)   \
  X(B200SVD_EPI_BIAS_RES1_FVEC, B200SVD_ACT_NONE, true, true, 1) \
  X(B200SVD_EPI_BIAS_FVEC, B200SVD_ACT_NONE, true, true, 0)    \
  X(B200SVD_EPI_BIAS_GEGLU, B200SVD_ACT_GEGLU, true, false, 0) \
  X(B200SVD_EPI_BIAS_RES2, B200SVD_ACT_NONE, true, false, 2)   \
  X(B200SVD_EPI_BIAS_SILU, B200SVD_ACT_SILU, true, false, 0)   \
  X(B200SVD_EPI_BIAS_GELU, B200SVD_ACT_GELU, true, false, 0)

// What a consumer thread knows about its tile
struct EpiTile {
  uint32_t n0, otile0, n_out;  // first GEMM column, first output column, output width
  uint32_t mb1, mb2, mb3;      // row box origin
  uint32_t mt;                 // M tile (the tile's GroupNorm partial-sum rows are 4 mt .. 4 mt + 3)
};

// Where row r (0-127) of the tile goes: whether it lies inside the output, its output row, and its per-frame vector
// row (p.fvec itself for a row outside the output: any readable row will do, such a row is never stored).
struct OutRow {
  bool valid;
  int64_t row;
  const float* fv;
};
__device__ __forceinline__ OutRow out_row(const GemmDev& p, const EpiTile& t, uint32_t r) {
  const uint32_t lb1 = p.m_lb[0], lb2 = p.m_lb[1];
  const uint32_t m1 = t.mb1 + (r & ((1u << lb1) - 1));
  const uint32_t m2 = t.mb2 + ((r >> lb1) & ((1u << lb2) - 1));
  const uint32_t m3 = t.mb3 + (r >> (lb1 + lb2));
  OutRow o;
  o.valid = (m1 < p.m_ext[0]) && (m2 < p.m_ext[1]) && (m3 < p.m_ext[2]);
  o.row = (int64_t)m1 * p.out_rs[0] + (int64_t)m2 * p.out_rs[1] + (int64_t)m3 * p.out_rs[2];
  o.fv = p.fvec != nullptr && o.valid ? p.fvec + (int64_t)((uint32_t)o.row / p.rows_per_frame) * p.ldf : p.fvec;
  return o;
}

// Bias and GEGLU gate bias of the thread's 8 columns of sub-tile c, loaded in one batch ahead of the residual waits
// and the arithmetic.  Columns past the output width read nothing.
template <int BN, class E>
__device__ __forceinline__ void epi_load_bias(const GemmDev& p, const EpiTile& t, int c, uint32_t cq, float (&bv)[4][2],
                                              float (&gbv)[4][2]) {
  if (E::bias(p)) {
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const uint32_t tcol = (uint32_t)(8 * (4 * c + jj)) + 2 * cq;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        bv[jj][e] = t.otile0 + tcol + e < t.n_out ? __ldg(p.bias + t.n0 + tcol + e) : 0.f;
        if (E::geglu(p)) gbv[jj][e] = __ldg(p.bias + t.n0 + BN / 2 + tcol + e);  // n is a multiple of BN
      }
    }
  }
}

// One 64-row half of sub-tile c: the thread's rows rbase and rbase + 8 (of the 64), 8 columns each, from the m64nBN
// accumulator fragment `acc` to the staging buffer `stg`; r1s / r2s are the residual sub-tiles of the same 64 rows.
// rows[h] is where row h goes; the half's 16 per-frame values are loaded in one batch ahead of the arithmetic.
// Order per element: bias, per-frame, gate bias, activation, s_acc, res1, res2, round.  An absent term is skipped,
// not added as zero (-0 + 0 is +0).
template <int BN, class E>
__device__ __forceinline__ void epi_stage_half(const GemmDev& p, const EpiTile& t, const float* acc, int c,
                                               uint32_t rbase, uint32_t cq, uint8_t* stg, const uint8_t* r1s,
                                               const uint8_t* r2s, const float (&bv)[4][2], const float (&gbv)[4][2],
                                               const OutRow (&rows)[2]) {
  constexpr int NJ = BN / 8;
  float fvv[2][4][2];
  if (E::fvec(p)) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const uint32_t ocol = t.otile0 + (uint32_t)(8 * (4 * c + jj)) + 2 * cq;
#pragma unroll
        for (int e = 0; e < 2; ++e) fvv[h][jj][e] = ocol + e < t.n_out ? __ldg(rows[h].fv + ocol + e) : 0.f;
      }
  }
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = 4 * c + jj;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t off = sw64_off(rbase + 8u * h, (uint32_t)jj, cq);
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      float g0 = 0.f, g1 = 0.f;
      if (E::bias(p)) {
        v0 += bv[jj][0];
        v1 += bv[jj][1];
      }
      if (E::fvec(p)) {
        v0 += fvv[h][jj][0];
        v1 += fvv[h][jj][1];
      }
      // GEGLU launches only the 128- and 256-wide tiles, and only value columns (j < NJ / 2) reach here: the gate
      // index stays inside the accumulator fragment at compile time.
      if constexpr (BN == 128 || BN == 256) {
        if (E::geglu(p) && j < NJ / 2) {
          g0 = acc[4 * (j + NJ / 2) + 2 * h];
          g1 = acc[4 * (j + NJ / 2) + 2 * h + 1];
          if (E::bias(p)) {
            g0 += gbv[jj][0];
            g1 += gbv[jj][1];
          }
        }
      }
      v0 = epi_act(E::act(p), p.s_acc, v0, g0);
      v1 = epi_act(E::act(p), p.s_acc, v1, g1);
      if (E::res1(p)) {
        const uint32_t w = *reinterpret_cast<const uint32_t*>(r1s + off);
        v0 = __fmaf_rn(p.s1, bf16_lo(w), v0);
        v1 = __fmaf_rn(p.s1, bf16_hi(w), v1);
      }
      if (E::res2(p)) {
        const uint32_t w = *reinterpret_cast<const uint32_t*>(r2s + off);
        v0 = __fmaf_rn(p.s2, bf16_lo(w), v0);
        v1 = __fmaf_rn(p.s2, bf16_hi(w), v1);
      }
      *reinterpret_cast<uint32_t*>(stg + off) = pack_bf16x2(v0, v1);
    }
  }
}

// GroupNorm partials of sub-tile c (cooperative generic launches with gn_part), summed from the bf16 words this
// thread has just staged (the values the GroupNorm reads; the same thread wrote them, so no barrier is needed): column
// sums over the warp's 16 rows (lanes of equal cq), then over the quadrant's two warps.  The odd warp of the quadrant
// hands its sums to the even one through gxb; the even one parks its own in the accumulators of the sub-tile, which
// are consumed, until gn_write_partials.
template <int BN>
__device__ __forceinline__ void gn_sum_partials(const EpiTile& t, float* acc, int c, uint32_t rbase, uint32_t cq,
                                                const uint8_t* stg, const OutRow (&rows)[2], float* gxb, bool sender,
                                                bool first_row) {
  // every staged word is read back first, outside the tests, so that the reads overlap the shuffles
  uint32_t sw[4][2];
#pragma unroll
  for (int jj = 0; jj < 4; ++jj)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      sw[jj][h] = *reinterpret_cast<const uint32_t*>(stg + sw64_off(rbase + 8u * h, (uint32_t)jj, cq));
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = 4 * c + jj;
    const uint32_t ocol = t.otile0 + (uint32_t)(8 * j) + 2 * cq;
    const bool in0 = ocol < t.n_out, in1 = ocol + 1 < t.n_out;
    float gs0 = 0.f, gs1 = 0.f, gq0 = 0.f, gq1 = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (rows[h].valid && in0) {
        const uint32_t w = sw[jj][h];
        const float r0 = bf16_lo(w), r1 = in1 ? bf16_hi(w) : 0.f;
        gs0 += r0;
        gs1 += r1;
        gq0 = __fmaf_rn(r0, r0, gq0);
        gq1 = __fmaf_rn(r1, r1, gq1);
      }
    }
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      gs0 += __shfl_xor_sync(0xffffffffu, gs0, o);
      gs1 += __shfl_xor_sync(0xffffffffu, gs1, o);
      gq0 += __shfl_xor_sync(0xffffffffu, gq0, o);
      gq1 += __shfl_xor_sync(0xffffffffu, gq1, o);
    }
    if (sender && first_row) *reinterpret_cast<float4*>(gxb + 2 * (8 * jj + 2 * cq)) = make_float4(gs0, gq0, gs1, gq1);
    if (!sender) {
      acc[4 * j] = gs0;
      acc[4 * j + 1] = gq0;
      acc[4 * j + 2] = gs1;
      acc[4 * j + 3] = gq1;
    }
  }
}

// After the named barrier: the even warp of the quadrant adds the partner's sums from gxb to its own and writes the
// quadrant's partials of sub-tile c to partial-sum row `slot`.
__device__ __forceinline__ void gn_write_partials(const GemmDev& p, const EpiTile& t, const float* acc, int c,
                                                  uint32_t cq, const float* gxb, uint32_t slot) {
  float2* dst = reinterpret_cast<float2*>(p.gn_part) + (int64_t)slot * p.gn_ld;
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = 4 * c + jj;
    const uint32_t ocol = t.otile0 + (uint32_t)(8 * j) + 2 * cq;
    if (ocol < t.n_out) {
      const float4 o = *reinterpret_cast<const float4*>(gxb + 2 * (8 * jj + 2 * cq));
      dst[ocol] = make_float2(acc[4 * j] + o.x, acc[4 * j + 1] + o.y);
      if (ocol + 1 < t.n_out) dst[ocol + 1] = make_float2(acc[4 * j + 2] + o.z, acc[4 * j + 3] + o.w);
    }
  }
}

// TMA producer of the A/B stage ring (one thread): the CTA's tiles in order, taps and K blocks of each.  Both
// schedules run it unchanged; the ring is what orders the consumers.
template <int BN>
__device__ __forceinline__ void produce_ab(const GemmDev& p, const CUtensorMap* tmA, const CUtensorMap* tmB,
                                           uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar) {
  constexpr int STAGE_BYTES = A_STAGE_BYTES + BN * BK * 2;
  PhaseClock pc;
  uint32_t st = 0, ph = 0;
  for (uint32_t tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    uint32_t n_tile, mb1, mb2, mb3;
    decode_tile(p, tile, n_tile, mb1, mb2, mb3);
    int base[5] = {0, 0, 0, 0, 0};
    base[p.m_adim[0]] += (int)mb1;
    base[p.m_adim[1]] += (int)mb2;
    base[p.m_adim[2]] += (int)mb3;
    const int n0 = (int)(n_tile * BN);
    for (uint32_t tap = 0; tap < p.taps; ++tap) {
      const int c0 = p.tap_off[tap][0];
      const int c1 = base[1] + p.tap_off[tap][1];
      const int c2 = base[2] + p.tap_off[tap][2];
      const int c3 = base[3] + p.tap_off[tap][3];
      const int c4 = base[4] + p.tap_off[tap][4];
#pragma unroll 1
      for (uint32_t kb = 0; kb < p.kblocks; ++kb) {
        pc.mark(PC_OTHER);
        mbar_wait_parked(&empty_bar[st], ph ^ 1);
        pc.mark(PC_RING_WAIT);
        uint8_t* sa = smem + st * STAGE_BYTES;
        mbar_expect_tx(&full_bar[st], STAGE_BYTES);
        tma_load_5d(sa, tmA, &full_bar[st], c0 + (int)(kb * BK), c1, c2, c3, c4);
        tma_load_3d(sa + A_STAGE_BYTES, tmB, &full_bar[st], (int)(kb * BK), n0, (int)tap);
        if (++st == p.stages) {
          st = 0;
          ph ^= 1;
        }
      }
    }
  }
  pc.write(PC_BUF(p), 0);
}

// TMA producer of the residual ring (one thread; bf16 outputs): sub-tile by sub-tile, res1 then res2, 128 rows x 32
// columns a slot.  It runs ahead of the consumers by the depth of the ring, so a tile's residuals stream in during
// its MMAs.
__device__ __forceinline__ void produce_residuals(const GemmDev& p, const CUtensorMap* tmR1, const CUtensorMap* tmR2,
                                                  uint8_t* res_smem, uint64_t* res_full, uint64_t* res_empty,
                                                  uint32_t tile_out_w, uint32_t n_out) {
  if (p.res1 != nullptr) prefetch_tmap(tmR1);
  if (p.res2 != nullptr) prefetch_tmap(tmR2);
  uint32_t slot = 0, ph = 0;
  for (uint32_t tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    uint32_t n_tile, mb1, mb2, mb3;
    decode_tile(p, tile, n_tile, mb1, mb2, mb3);
    const uint32_t otile0 = n_tile * tile_out_w;
    for (uint32_t c = 0; c < tile_out_w / SUB_W && otile0 + c * SUB_W < n_out; ++c) {
      for (int r = 0; r < 2; ++r) {
        if ((r == 0 ? p.res1 : p.res2) == nullptr) continue;
        mbar_wait_parked(&res_empty[slot], ph ^ 1);
        mbar_expect_tx(&res_full[slot], RES_SLOT_BYTES);
        tma_load_4d(res_smem + slot * RES_SLOT_BYTES, r == 0 ? tmR1 : tmR2, &res_full[slot],
                    (int)(otile0 + c * SUB_W), (int)mb1, (int)mb2, (int)mb3);
        if (++slot == p.res_slots) {
          slot = 0;
          ph ^= 1;
        }
      }
    }
  }
}

// The staged bf16 epilogue of one tile for epilogue kind E on either schedule.  A consumer warpgroup holds HALVES
// 64-row halves of the tile: 1 on the cooperative schedule (its own 64 rows, 4 KB staging slots, its rows of each
// residual slot at cw * STG_SLOT_BYTES, stores at the box origin moved by wg_off), 2 on the alternating one (the whole
// tile, 8 KB slots, stores at the tile's box).  Sub-tile by sub-tile: bias loads, the residual waits in the order the
// residual producer loads them, the arithmetic into one of the warpgroup's two staging slots, and one TMA store once
// the store issued a sub-tile ago has read the other slot.  gn_x is the GroupNorm exchange area (cooperative only).
template <int BN, class E, int HALVES>
__device__ __forceinline__ void epilogue_staged(const GemmDev& p, const CUtensorMap* tmO, const EpiTile& t,
                                                float* const (&acc)[HALVES], const OutRow (&rows)[HALVES][2],
                                                uint8_t* stg_smem, const uint8_t* res_smem, uint64_t* res_full,
                                                uint64_t* res_empty, RingPos& rr, uint32_t& stg_it, uint32_t cw,
                                                uint32_t rbase, uint32_t cq, bool leader, float* gn_x, PhaseClock& pc) {
  constexpr uint32_t SLOT_BYTES = HALVES * STG_SLOT_BYTES;
  const uint8_t* res_rows = res_smem + (HALVES == 1 ? cw * STG_SLOT_BYTES : 0u);
  const uint32_t wl = rbase >> 4, rq = rbase & 7u;  // warp of the warpgroup, row of the lane in its 8-row group
#pragma unroll
  for (int c = 0; c < BN / SUB_W; ++c) {
    if (E::geglu(p) && c >= BN / SUB_W / 2) break;  // gate columns are consumed with their value columns
    if (t.otile0 + (uint32_t)(c * SUB_W) >= t.n_out) break;
    uint8_t* stg = stg_smem + (cw * STG_SLOTS + (stg_it & 1)) * SLOT_BYTES;
    float bv[4][2], gbv[4][2];
    epi_load_bias<BN, E>(p, t, c, cq, bv, gbv);
    const uint8_t* r1s = res_rows;
    const uint8_t* r2s = res_rows;
    uint32_t r1slot = 0, r2slot = 0;
    pc.mark(PC_EPI);
    if (E::res1(p)) {
      r1slot = rr.idx;
      mbar_wait(&res_full[rr.idx], rr.phase);
      r1s = res_rows + rr.idx * RES_SLOT_BYTES;
      ring_step(rr, p.res_slots);
    }
    if (E::res2(p)) {
      r2slot = rr.idx;
      mbar_wait(&res_full[rr.idx], rr.phase);
      r2s = res_rows + rr.idx * RES_SLOT_BYTES;
      ring_step(rr, p.res_slots);
    }
    pc.mark(PC_RES_WAIT);
#pragma unroll
    for (int hh = 0; hh < HALVES; ++hh)
      epi_stage_half<BN, E>(p, t, acc[hh], c, rbase, cq, stg + hh * STG_SLOT_BYTES, r1s + hh * STG_SLOT_BYTES,
                            r2s + hh * STG_SLOT_BYTES, bv, gbv, rows[hh]);
    float* gxb = nullptr;
    if constexpr (HALVES == 1 && E::GENERIC) {
      gxb = gn_x + ((cw * 2 + (stg_it & 1)) * 2 + (wl >> 1)) * (SUB_W * 2);
      if (p.gn_part != nullptr) gn_sum_partials<BN>(t, acc[0], c, rbase, cq, stg, rows[0], gxb, wl & 1, rq == 0);
    }
    fence_proxy_async_smem();  // the staged values are read by the TMA store (async proxy)
    pc.mark(PC_EPI);
    // the store issued one sub-tile ago has read the other staging buffer: it may be refilled next sub-tile
    if (leader) tma_store_wait_read0();
    named_bar_sync(5 + (int)cw, 128);
    pc.mark(PC_STORE_WAIT);
    if (leader) {
      if (E::res1(p)) mbar_arrive(&res_empty[r1slot]);
      if (E::res2(p)) mbar_arrive(&res_empty[r2slot]);
      // cooperative: the warpgroup's 64 rows, the tile's row box halved in its outermost non-unit dimension
      const bool second = HALVES == 1 && cw != 0;
      tma_store_4d(tmO, stg, (int)(t.otile0 + c * SUB_W), (int)(t.mb1 + (second ? p.wg_off[0] : 0u)),
                   (int)(t.mb2 + (second ? p.wg_off[1] : 0u)), (int)(t.mb3 + (second ? p.wg_off[2] : 0u)));
      tma_store_commit();
    }
    if constexpr (HALVES == 1 && E::GENERIC) {
      if (p.gn_part != nullptr && (wl & 1) == 0 && rq == 0)
        gn_write_partials(p, t, acc[0], c, cq, gxb, t.mt * 4u + 2 * cw + (wl >> 1));
    }
    ++stg_it;
  }
}

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
mtgemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
              const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmR1,
              const __grid_constant__ CUtensorMap tmR2, const GemmDev p) {
  using Cfg = TileCfg<BN>;
  constexpr int R = BN / 2;  // accumulator registers per thread (m64nBN: 64 x BN over 128 threads)
  extern __shared__ __align__(1024) uint8_t smem[];  // SWIZZLE_128B operands need 1024-byte alignment
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  const uint32_t stages = p.stages, rslots = p.res_slots;
  uint8_t* res_smem = smem + stages * Cfg::STAGE_BYTES;
  uint8_t* stg_smem = res_smem + rslots * RES_SLOT_BYTES;
  float* gn_x = reinterpret_cast<float*>(stg_smem + STG_BYTES);  // [warpgroup][buffer][quadrant][32 columns][2]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg_smem + STG_BYTES + GN_BYTES);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  uint64_t* res_full = empty_bar + MAX_STAGES;
  uint64_t* res_empty = res_full + MAX_RES_SLOTS;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const uint32_t iters_per_tile = p.taps * p.kblocks;
  const bool geglu = (p.act == B200SVD_ACT_GEGLU);
  const uint32_t n_out = geglu ? p.n / 2 : p.n;
  const uint32_t tile_out_w = geglu ? (uint32_t)BN / 2 : (uint32_t)BN;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if (p.staged) prefetch_tmap(&tmO);
    for (uint32_t s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per consumer warpgroup
    }
    for (uint32_t s = 0; s < rslots; ++s) {
      mbar_init(&res_full[s], 1);
      mbar_init(&res_empty[s], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::PRODUCER_REGS));
    if (threadIdx.x == 0) {
      produce_ab<BN>(p, &tmA, &tmB, smem, full_bar, empty_bar);
    } else if (threadIdx.x == 32 && rslots != 0) {
      produce_residuals(p, &tmR1, &tmR2, res_smem, res_full, res_empty, tile_out_w, n_out);
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::CONSUMER_REGS));

  // ===================== consumer warpgroups =====================
  const int cw = wg - 1;   // rows [64 cw, 64 cw + 64) of the tile
  const int wl = warp & 3;  // warp of the warpgroup: rows 16 wl .. 16 wl + 15 of those 64
  const int rq = lane >> 2, cq = lane & 3;
  const bool leader = (threadIdx.x & 127) == 0;
  const uint32_t rbase = (uint32_t)(16 * wl + rq);
  RingPos ab = {0, 0};   // A/B ring position
  RingPos rr = {0, 0};   // residual ring position
  uint32_t stg_it = 0;   // sub-tiles staged by this warpgroup so far
  float acc[R];
  PhaseClock pc;

  for (uint32_t tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    pc.mark(PC_EPI);
#pragma unroll
    for (int i = 0; i < R; ++i) acc[i] = 0.f;
    uint32_t prev = 0;
    for (uint32_t i = 0; i < iters_per_tile; ++i) {
      mbar_wait(&full_bar[ab.idx], ab.phase);
      pc.mark(PC_RING_WAIT);
      const uint32_t sa = smem_u32(smem + ab.idx * Cfg::STAGE_BYTES);
      const uint64_t adesc = smem_desc_k_sw128(sa + cw * (A_STAGE_BYTES / 2));
      const uint64_t bdesc = smem_desc_k_sw128(sa + A_STAGE_BYTES);
      wgmma_fence_regs(acc);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk)  // +16 elements along K = +32 B inside the swizzle atom
        Wgmma<BN>::ss(acc, adesc + (uint64_t)(kk * 2), bdesc + (uint64_t)(kk * 2), 1u);
      wgmma_commit();
      wgmma_fence_regs(acc);
      // the MMAs of the previous stage have completed: hand it back to the producer
      wgmma_wait<1>();
      pc.mark(PC_MMA);
      if (i > 0 && leader) mbar_arrive(&empty_bar[prev]);
      prev = ab.idx;
      ring_step(ab, stages);
    }
    wgmma_wait<0>();
    pc.mark(PC_MMA);
    wgmma_fence_regs(acc);
    if (leader) mbar_arrive(&empty_bar[prev]);

    // ----- epilogue: thread holds rows r0 and r0 + 8, columns 8 j + 2 cq + {0, 1} (acc[4 j + 2 h + e]) -----
    uint32_t n_tile, mb1, mb2, mb3;
    decode_tile(p, tile, n_tile, mb1, mb2, mb3);
    const EpiTile et = {n_tile * BN, n_tile * tile_out_w, n_out, mb1, mb2, mb3, tile / p.n_tiles};
    const OutRow rows[1][2] = {{out_row(p, et, 64 * cw + rbase), out_row(p, et, 64 * cw + rbase + 8)}};
    if (p.staged) {
      // ----- bf16 output: 32-column sub-tiles staged in shared memory (SWIZZLE_64B, conflict-free fragment
      // writes), written by one TMA store per warpgroup and sub-tile; residuals come from the TMA-fed ring.  The
      // epilogue kind is launch-uniform: one switch per tile -----
      float* const accs[1] = {acc};
      switch (p.epi_kind) {
        case B200SVD_EPI_GENERIC:
          epilogue_staged<BN, EpiGeneric, 1>(p, &tmO, et, accs, rows, stg_smem, res_smem, res_full, res_empty, rr,
                                             stg_it, cw, rbase, cq, leader, gn_x, pc);
          break;
#define MTGEMM_CASE(ID, ACT, BIAS, FVEC, NRES)                                                                    \
  case ID:                                                                                                        \
    if constexpr (ACT != B200SVD_ACT_GEGLU || BN == 128 || BN == 256)                                             \
      epilogue_staged<BN, Epi<ACT, BIAS, FVEC, NRES>, 1>(p, &tmO, et, accs, rows, stg_smem, res_smem, res_full,   \
                                                         res_empty, rr, stg_it, cw, rbase, cq, leader, gn_x, pc); \
    break;
        MTGEMM_EPI_KINDS(MTGEMM_CASE)
#undef MTGEMM_CASE
      }
      if (p.gn_part != nullptr && (wl & 1) == 0 && lane == 0 && n_tile == 0) {
        // lane 0 holds the first row of the quadrant: if it is out of range, so is every row of the quadrant
        const uint32_t slot = et.mt * 4u + (uint32_t)(2 * cw + (wl >> 1));
        p.gn_slot_sample[slot] = rows[0][0].valid ? (int32_t)((uint32_t)rows[0][0].row / p.gn_rows) : -1;
      }
      continue;
    }
    // ----- fp32 output (pitches a tensor map cannot describe), or a bf16 output whose width is not a whole number
    // of 16-byte chunks (a TMA store writes whole chunks): straight from the accumulator registers -----
    constexpr int NJ = BN / 8;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      if (geglu && j >= NJ / 2) break;  // gate columns are consumed with their value columns
      const uint32_t tcol = 8 * j + 2 * cq;  // column in the tile (value column for GEGLU)
      const uint32_t ocol = et.otile0 + tcol;
      const bool in0 = ocol < n_out, in1 = ocol + 1 < n_out;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (!rows[0][h].valid || !in0) continue;
        const int64_t row = rows[0][h].row;
        if (p.bias != nullptr) {
          v0 += __ldg(p.bias + et.n0 + tcol);
          if (in1) v1 += __ldg(p.bias + et.n0 + tcol + 1);
        }
        if (p.fvec != nullptr) {
          v0 += __ldg(rows[0][h].fv + ocol);
          if (in1) v1 += __ldg(rows[0][h].fv + ocol + 1);
        }
        float g0 = 0.f, g1 = 0.f;
        if (geglu) {
          g0 = acc[4 * (j + NJ / 2) + 2 * h];
          g1 = acc[4 * (j + NJ / 2) + 2 * h + 1];
          if (p.bias != nullptr) {
            g0 += __ldg(p.bias + et.n0 + BN / 2 + tcol);
            if (in1) g1 += __ldg(p.bias + et.n0 + BN / 2 + tcol + 1);
          }
        } else if (p.act == B200SVD_ACT_PRELU) {
          g0 = __ldg(p.slope + et.n0 + tcol);
          if (in1) g1 = __ldg(p.slope + et.n0 + tcol + 1);
        }
        v0 = epi_act(p.act, p.s_acc, v0, g0);
        v1 = epi_act(p.act, p.s_acc, v1, g1);
        if (p.res1 != nullptr) {
          float a, b;
          load_bf16_pair(p.res1, row * p.ld1 + ocol, in1, a, b);
          v0 = __fmaf_rn(p.s1, a, v0);
          v1 = __fmaf_rn(p.s1, b, v1);
        }
        if (p.res2 != nullptr) {
          float a, b;
          load_bf16_pair(p.res2, row * p.ld2 + ocol, in1, a, b);
          v0 = __fmaf_rn(p.s2, a, v0);
          v1 = __fmaf_rn(p.s2, b, v1);
        }
        if (p.out_fp32) {
          float* op = reinterpret_cast<float*>(p.out) + row * p.ldo + ocol;
          if (in1 && ((row * p.ldo + ocol) & 1) == 0) {
            *reinterpret_cast<float2*>(op) = make_float2(v0, v1);
          } else {
            op[0] = v0;
            if (in1) op[1] = v1;
          }
        } else {
          __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(p.out) + row * p.ldo + ocol;
          if (in1) {
            *reinterpret_cast<uint32_t*>(op) = pack_bf16x2(v0, v1);  // ldo % 8 == 0 and an even column: 4-byte aligned
          } else {
            op[0] = __float2bfloat16(v0);
          }
        }
      }
    }
  }
  pc.mark(PC_EPI);
  if (leader) pc.write(PC_BUF(p), 1 + cw);
  if (p.staged && leader) tma_store_wait_all();  // shared memory must outlive the last stores' reads
}

// The alternating schedule.  Producers, tile order and ring contents are those of mtgemm_kernel; what changes is who
// consumes a tile.  Warpgroup w computes the CTA's tiles w, w + 2, ... whole (two m64nBNk16 per k16 step, rows 0-63
// and 64-127 of the A stage against the same B descriptor) and is the only one to release their stages and residual
// slots, so every "empty" barrier counts one arrival.  It steps over the other warpgroup's tiles by ring arithmetic
// alone (mtgemm_ring.h).  Because the ring is filled in tile order, a warpgroup's next tile becomes full as the other
// one nears the end of its MMAs: one warpgroup's epilogue runs under the other's MMAs.
// An mbarrier wait sees one bit of phase, so a wait for fill j of a buffer also passes while fill j - 1 of that buffer
// has not landed (the barrier is two phases behind: the same parity).  A warpgroup that only did arithmetic over the
// other's tile could be that far ahead.  Two monotonic tile counters per warpgroup in shared memory rule it out: a
// warpgroup starts the MMAs (the residual waits) of its tile t only when the other one has passed every stage wait
// (residual wait) of tile t - 1, so every earlier fill of every buffer has landed.  The tensor cores are shared, so
// waiting for the other warpgroup's MMAs costs nothing that was not already spent.
// Per output element the k order, the wgmma k16 steps and the epilogue arithmetic are those of
// mtgemm_kernel, so the results are bitwise the same.  bf16 staged outputs only, no GroupNorm partials.
template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
mtgemm_alt_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmR1,
                  const __grid_constant__ CUtensorMap tmR2, const GemmDev p) {
  using Cfg = AltCfg<BN>;
  constexpr int R = BN / 2;  // accumulator registers per thread and 64-row half
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  const uint32_t stages = p.stages, rslots = p.res_slots;
  uint8_t* res_smem = smem + stages * Cfg::STAGE_BYTES;
  uint8_t* stg_smem = res_smem + rslots * RES_SLOT_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg_smem + ALT_STG_BYTES);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  uint64_t* res_full = empty_bar + MAX_STAGES;
  uint64_t* res_empty = res_full + MAX_RES_SLOTS;
  // tiles of the CTA's sequence whose stage waits / residual waits warpgroup w has passed: [w], [2 + w]
  uint32_t* tiles_done = reinterpret_cast<uint32_t*>(res_empty + MAX_RES_SLOTS);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const uint32_t iters_per_tile = p.taps * p.kblocks;
  const bool geglu = (p.act == B200SVD_ACT_GEGLU);
  const uint32_t n_out = geglu ? p.n / 2 : p.n;
  const uint32_t tile_out_w = geglu ? (uint32_t)BN / 2 : (uint32_t)BN;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    prefetch_tmap(&tmO);
    for (int i = 0; i < 4; ++i) tiles_done[i] = 0;
    for (uint32_t s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);  // released by the warpgroup that owns the tile
    }
    for (uint32_t s = 0; s < rslots; ++s) {
      mbar_init(&res_full[s], 1);
      mbar_init(&res_empty[s], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::PRODUCER_REGS));
    if (threadIdx.x == 0) {
      produce_ab<BN>(p, &tmA, &tmB, smem, full_bar, empty_bar);
    } else if (threadIdx.x == 32 && rslots != 0) {
      produce_residuals(p, &tmR1, &tmR2, res_smem, res_full, res_empty, tile_out_w, n_out);
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::CONSUMER_REGS));

  // ===================== consumer warpgroups =====================
  const uint32_t cw = (uint32_t)(wg - 1);
  const int wl = warp & 3;  // warp of the warpgroup: rows 16 wl .. 16 wl + 15 of both 64-row halves
  const int rq = lane >> 2, cq = lane & 3;
  const bool leader = (threadIdx.x & 127) == 0;
  const uint32_t rbase = (uint32_t)(16 * wl + rq);
  const uint32_t nres = (p.res1 != nullptr ? 1u : 0u) + (p.res2 != nullptr ? 1u : 0u);
  RingPos ab = {0, 0};   // A/B ring position
  RingPos rr = {0, 0};   // residual ring position
  uint32_t stg_it = 0;   // sub-tiles staged by this warpgroup so far
  float acc0[R], acc1[R];  // rows 0-63 and 64-127 of the tile
  PhaseClock pc;

  uint32_t t = 0;  // index of the tile in this CTA's sequence
  for (uint32_t tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++t) {
    pc.mark(PC_EPI);
    if (alt_owner(t) != cw) {
      // The other warpgroup's tile: step over its stages and residual slots.  If none of this warpgroup's follows,
      // it is done.
      if (tile + gridDim.x >= p.total_tiles) break;
      ring_advance(ab, iters_per_tile, stages);
      if (rslots != 0) ring_advance(rr, tile_res_slots(tile % p.n_tiles, tile_out_w, n_out, SUB_W, nres), rslots);
      continue;
    }
    while (ld_acquire_shared(&tiles_done[1 - cw]) < t) {  // the other warpgroup has seen tile t - 1's stages land
    }
    pc.mark(PC_OTHER);
#pragma unroll
    for (int i = 0; i < R; ++i) acc0[i] = acc1[i] = 0.f;
    uint32_t prev = 0;
    for (uint32_t i = 0; i < iters_per_tile; ++i) {
      mbar_wait(&full_bar[ab.idx], ab.phase);
      pc.mark(PC_RING_WAIT);
      // the tile's last stage has landed: the other warpgroup may queue its MMAs behind these
      if (leader && i + 1 == iters_per_tile) st_release_shared(&tiles_done[cw], t + 1);
      const uint32_t sa = smem_u32(smem + ab.idx * Cfg::STAGE_BYTES);
      const uint64_t adesc0 = smem_desc_k_sw128(sa);
      const uint64_t adesc1 = smem_desc_k_sw128(sa + A_STAGE_BYTES / 2);
      const uint64_t bdesc = smem_desc_k_sw128(sa + A_STAGE_BYTES);
      wgmma_fence_regs(acc0);
      wgmma_fence_regs(acc1);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk) {  // +16 elements along K = +32 B inside the swizzle atom
        Wgmma<BN>::ss(acc0, adesc0 + (uint64_t)(kk * 2), bdesc + (uint64_t)(kk * 2), 1u);
        Wgmma<BN>::ss(acc1, adesc1 + (uint64_t)(kk * 2), bdesc + (uint64_t)(kk * 2), 1u);
      }
      wgmma_commit();
      wgmma_fence_regs(acc0);
      wgmma_fence_regs(acc1);
      // the MMAs of the previous stage have completed: hand it back to the producer
      wgmma_wait<1>();
      pc.mark(PC_MMA);
      if (i > 0 && leader) mbar_arrive(&empty_bar[prev]);
      prev = ab.idx;
      ring_step(ab, stages);
    }
    wgmma_wait<0>();
    pc.mark(PC_MMA);
    wgmma_fence_regs(acc0);
    wgmma_fence_regs(acc1);
    if (leader) mbar_arrive(&empty_bar[prev]);

    // ----- epilogue: thread holds rows 64 hh + 16 wl + rq + 8 h, columns 8 j + 2 cq + {0, 1} (accHH[4 j + 2 h + e])
    uint32_t n_tile, mb1, mb2, mb3;
    decode_tile(p, tile, n_tile, mb1, mb2, mb3);
    const EpiTile et = {n_tile * BN, n_tile * tile_out_w, n_out, mb1, mb2, mb3, tile / p.n_tiles};
    const OutRow rows[2][2] = {{out_row(p, et, rbase), out_row(p, et, rbase + 8)},
                               {out_row(p, et, 64 + rbase), out_row(p, et, 64 + rbase + 8)}};
    if (rslots != 0) {
      pc.mark(PC_EPI);
      while (ld_acquire_shared(&tiles_done[2 + 1 - cw]) < t) {  // ... and tile t - 1's residual slots
      }
      pc.mark(PC_RES_WAIT);
    }
    // the epilogue kind is launch-uniform: one switch per tile
    float* const accs[2] = {acc0, acc1};
    switch (p.epi_kind) {
      case B200SVD_EPI_GENERIC:
        epilogue_staged<BN, EpiGeneric, 2>(p, &tmO, et, accs, rows, stg_smem, res_smem, res_full, res_empty, rr,
                                           stg_it, cw, rbase, cq, leader, nullptr, pc);
        break;
#define MTGEMM_CASE(ID, ACT, BIAS, FVEC, NRES)                                                                    \
  case ID:                                                                                                        \
    if constexpr (ACT != B200SVD_ACT_GEGLU || BN == 128)                                                          \
      epilogue_staged<BN, Epi<ACT, BIAS, FVEC, NRES>, 2>(p, &tmO, et, accs, rows, stg_smem, res_smem, res_full,   \
                                                         res_empty, rr, stg_it, cw, rbase, cq, leader, nullptr,   \
                                                         pc);                                                     \
    break;
      MTGEMM_EPI_KINDS(MTGEMM_CASE)
#undef MTGEMM_CASE
    }
    if (leader && rslots != 0) st_release_shared(&tiles_done[2 + cw], t + 1);
  }
  pc.mark(PC_EPI);
  if (leader) pc.write(PC_BUF(p), 1 + (int)cw);
  if (leader) tma_store_wait_all();  // shared memory must outlive the last stores' reads
}

static int ilog2_exact(uint32_t v) {
  if (v == 0 || (v & (v - 1)) != 0) return -1;
  int l = 0;
  while ((1u << l) < v) ++l;
  return l;
}

// Tensor maps of the bf16 epilogue: the output, res1 and res2 as (n_out, m1, m2, m3) views with row strides
// out_rs[i] * leading dimension, and a 32-column box (SWIZZLE_64B).  Hardware clipping handles ragged M in each of
// the three row dimensions, the N edge and column slices of wider buffers.
struct EpiMaps {
  CUtensorMap out, res1, res2;
};

#ifdef MTGEMM_PHASE_CLOCKS
static long long* g_phase_buf = nullptr;
#endif

template <int BN, bool ALT>
struct SchedCfg {
  using type = TileCfg<BN>;
  static constexpr auto kernel = mtgemm_kernel<BN>;
};
template <int BN>
struct SchedCfg<BN, true> {
  using type = AltCfg<BN>;
  static constexpr auto kernel = mtgemm_alt_kernel<BN>;
};

template <int BN, bool ALT = false>
static int launch(const b200svd_gemm_params* p, const CUtensorMap& tmA, const EpiMaps& em, const GemmDev& d,
                  cudaStream_t st) {
  using Cfg = typename SchedCfg<BN, ALT>::type;
  constexpr auto kernel = SchedCfg<BN, ALT>::kernel;
  // weights [taps][n][k] -> TMA dims (k, n, taps)
  CUtensorMap tmB;
  uint64_t bd[3] = {p->k, p->n, p->taps};
  uint64_t bs[2] = {(uint64_t)p->k * 2, (uint64_t)p->k * 2 * p->n};
  uint32_t bb[3] = {64, (uint32_t)BN, 1};
  if (encode_tmap_bf16(&tmB, p->w_ptr, 3, bd, bs, bb)) return 1;
  GemmDev dd = d;
#ifdef MTGEMM_PHASE_CLOCKS
  dd.phase_buf = g_phase_buf;
#endif
  dd.n_tiles = (p->n + BN - 1) / BN;
  // Ring depths.  Without residuals every byte past the fixed areas goes to A/B stages.  With residuals (bf16
  // output) stages are given up, down to MIN_STAGES, until the residual ring holds a whole tile's residual sub-tiles.
  int stages = Cfg::STAGES, res_slots = 0;
  const int nres = d.staged ? (p->res1 != nullptr) + (p->res2 != nullptr) : 0;
  if (nres > 0) {
    const int tile_out_w = p->act == B200SVD_ACT_GEGLU ? BN / 2 : BN;
    int want = nres * (tile_out_w / SUB_W);
    if (want > MAX_RES_SLOTS) want = MAX_RES_SLOTS;
    while (stages > MIN_STAGES && Cfg::res_slots_fit(stages) < want) --stages;
    res_slots = Cfg::res_slots_fit(stages);
    if (res_slots > want) res_slots = want;
  }
  dd.stages = (uint32_t)stages;
  dd.res_slots = (uint32_t)res_slots;
  const int smem_bytes = stages * Cfg::STAGE_BYTES + res_slots * RES_SLOT_BYTES + Cfg::FIXED;
  const int slot = dev_slot();
  static bool attr_set[B200_MAX_DEVICES] = {};
  if (!attr_set[slot]) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(mtgemm)");
    attr_set[slot] = true;
  }
  const uint64_t m_tiles = (uint64_t)dd.m_tiles[0] * dd.m_tiles[1] * dd.m_tiles[2];
  const uint64_t total = (uint64_t)dd.n_tiles * m_tiles;
  if (total == 0 || total > 0x7FFFFFFFull) {
    set_error("mtgemm: bad tile count %llu", (unsigned long long)total);
    return 1;
  }
  dd.total_tiles = (uint32_t)total;
  const uint32_t grid = (uint32_t)(total < (uint64_t)sm_count() ? total : (uint64_t)sm_count());
  kernel<<<grid, NUM_THREADS, smem_bytes, st>>>(tmA, tmB, em.out, em.res1, em.res2, dd);
  B200_CHECK_LAUNCH("mtgemm launch");
  return 0;
}

// Kept for the C ABI: CTA-pair (cta_group::2) tiles do not exist on sm_90, every launch uses single-CTA tiles.
static int g_pair_mode = 2;

// Schedule choice, see b200svd_gemm_schedule in b200svd.h.  The alternating schedule pays for hiding the epilogue
// with narrower tiles (about a third more bytes from L2 into shared memory per MMA at 128 against 256 columns), so
// the rule keeps it to tiles whose MMAs are short enough for the epilogue to matter: taps x kblocks x 2 x BN tensor
// core clocks per tile.
static int g_schedule = 2;
constexpr uint64_t ALT_MAX_TILE_MMA_CLOCKS = 20000;

// N tile of the alternating schedule for a launch whose cooperative tile is `bn`, 0 if it has none.  A GEGLU launch
// cannot change its tile: the weights are interleaved per tile.  The 160-wide tile (N = 160, 320) has none: it
// measured slower alternating than cooperative (M 460800, K 1280, N 320 with a residual: 3.2 ms against 1.4 ms on an
// H100 at 700 W), and its 160 accumulator registers per thread leave the batched epilogue loads no room.
static int alt_tile(int bn, bool geglu) {
  if (bn == 256 && !geglu) return 128;
  return bn <= 128 ? bn : 0;
}

// Epilogue body choice, see b200svd_gemm_epilogue in b200svd.h.
static int g_epilogue = 1;

// The compile-time epilogue kind of a launch (MTGEMM_EPI_KINDS), B200SVD_EPI_GENERIC if it has none: outputs that are
// not staged bf16, GroupNorm partials, and every combination the list does not name.
static int epilogue_kind(const b200svd_gemm_params* p) {
  const uint32_t n_out = p->act == B200SVD_ACT_GEGLU ? p->n / 2 : p->n;
  if (p->out_fp32 || n_out % 8 != 0 || p->gn_part != nullptr) return B200SVD_EPI_GENERIC;
  const bool bias = p->bias != nullptr, fvec = p->fvec != nullptr;
  const int nres = p->res1 == nullptr ? (p->res2 == nullptr ? 0 : -1) : (p->res2 == nullptr ? 1 : 2);
  if (!bias) return p->act == B200SVD_ACT_NONE && !fvec && nres == 0 ? B200SVD_EPI_PLAIN : B200SVD_EPI_GENERIC;
  switch (p->act) {
    case B200SVD_ACT_NONE:
      if (nres == 0) return fvec ? B200SVD_EPI_BIAS_FVEC : B200SVD_EPI_BIAS;
      if (nres == 1) return fvec ? B200SVD_EPI_BIAS_RES1_FVEC : B200SVD_EPI_BIAS_RES1;
      return nres == 2 && !fvec ? B200SVD_EPI_BIAS_RES2 : B200SVD_EPI_GENERIC;
    case B200SVD_ACT_SILU: return !fvec && nres == 0 ? B200SVD_EPI_BIAS_SILU : B200SVD_EPI_GENERIC;
    case B200SVD_ACT_GELU: return !fvec && nres == 0 ? B200SVD_EPI_BIAS_GELU : B200SVD_EPI_GENERIC;
    case B200SVD_ACT_GEGLU: return !fvec && nres == 0 ? B200SVD_EPI_BIAS_GEGLU : B200SVD_EPI_GENERIC;
    default: return B200SVD_EPI_GENERIC;
  }
}

}  // namespace b200

extern "C" int b200svd_gemm_epilogue(int mode) {
  const int prev = b200::g_epilogue;
  if (mode == 0 || mode == 1) b200::g_epilogue = mode;
  return prev;
}

extern "C" int b200svd_gemm_epilogue_kind(const b200svd_gemm_params* p) {
  if (p == nullptr || b200::g_epilogue == 0) return B200SVD_EPI_GENERIC;
  return b200::epilogue_kind(p);
}

extern "C" int b200svd_gemm_schedule(int mode) {
  const int prev = b200::g_schedule;
  if (mode >= 0 && mode <= 2) b200::g_schedule = mode;
  return prev;
}

#ifdef MTGEMM_PHASE_CLOCKS
// Measuring build only: device buffer of [CTA][3 roles][8] int64 clock sums that every following launch adds to.
extern "C" int b200svd_gemm_phase_buffer(void* buf) {
  b200::g_phase_buf = reinterpret_cast<long long*>(buf);
  return 0;
}
#endif

extern "C" int b200svd_gemm_pair_mode(int mode) {
  const int prev = b200::g_pair_mode;
  if (mode >= 0 && mode <= 3) b200::g_pair_mode = mode;
  return prev;
}

extern "C" int b200svd_gemm(const b200svd_gemm_params* p, void* stream) {
  using namespace b200;
  if (p == nullptr) {
    set_error("b200svd_gemm: null params");
    return 1;
  }
  if (p->taps == 0 || p->taps > B200SVD_MAX_TAPS) {
    set_error("b200svd_gemm: taps=%u out of range", p->taps);
    return 1;
  }
  if (p->a_box[0] != 64 || (uint64_t)p->a_box[1] * p->a_box[2] * p->a_box[3] * p->a_box[4] != 128) {
    set_error("b200svd_gemm: A box must be 64 x (product 128), got [%u,%u,%u,%u,%u]", p->a_box[0], p->a_box[1],
              p->a_box[2], p->a_box[3], p->a_box[4]);
    return 1;
  }
  if (p->k % 8 != 0) {
    set_error("b200svd_gemm: K=%u must be a multiple of 8 (16-byte TMA rows)", p->k);
    return 1;
  }
  GemmDev d;
  memset(&d, 0, sizeof(d));
  for (uint32_t t = 0; t < p->taps; ++t)
    for (int i = 0; i < 5; ++i) d.tap_off[t][i] = p->tap_off[t][i];
  d.taps = p->taps;
  d.kblocks = (p->k + 63) / 64;
  d.n = p->n;
  uint32_t prod = 1;
  for (int i = 0; i < 3; ++i) {
    int lb = ilog2_exact(p->m_box[i]);
    if (lb < 0) {
      set_error("b200svd_gemm: m_box[%d]=%u is not a power of two", i, p->m_box[i]);
      return 1;
    }
    if (p->m_adim[i] < 1 || p->m_adim[i] > 4) {
      set_error("b200svd_gemm: m_adim[%d]=%u must be in 1..4", i, p->m_adim[i]);
      return 1;
    }
    if (p->a_box[p->m_adim[i]] != p->m_box[i]) {
      set_error("b200svd_gemm: a_box[%u]=%u != m_box[%d]=%u", p->m_adim[i], p->a_box[p->m_adim[i]], i, p->m_box[i]);
      return 1;
    }
    if (i > 0 && p->m_adim[i] <= p->m_adim[i - 1]) {
      set_error("b200svd_gemm: m_adim must be increasing");
      return 1;
    }
    prod *= p->m_box[i];
    d.m_ext[i] = p->m_ext[i];
    d.m_lb[i] = (uint32_t)lb;
    d.m_tiles[i] = (p->m_ext[i] + p->m_box[i] - 1) / p->m_box[i];
    d.m_adim[i] = p->m_adim[i];
    d.out_rs[i] = p->out_rs[i];
  }
  if (prod != 128) {
    set_error("b200svd_gemm: m_box product %u != 128", prod);
    return 1;
  }
  d.out = p->out;
  d.ldo = p->ldo;
  d.out_fp32 = p->out_fp32;
  d.bias = p->bias;
  d.fvec = p->fvec;
  d.ldf = p->ldf;
  d.rows_per_frame = p->rows_per_frame ? p->rows_per_frame : 1;
  d.act = p->act;
  d.s_acc = p->s_acc;
  d.res1 = reinterpret_cast<const __nv_bfloat16*>(p->res1);
  d.ld1 = p->ld1;
  d.s1 = p->s1;
  d.res2 = reinterpret_cast<const __nv_bfloat16*>(p->res2);
  d.ld2 = p->ld2;
  d.s2 = p->s2;
  d.gn_part = p->gn_part;
  d.gn_slot_sample = p->gn_slot_sample;
  d.gn_ld = p->gn_ld;
  d.gn_rows = p->gn_rows ? p->gn_rows : 1;
  if (p->act < B200SVD_ACT_NONE || p->act > B200SVD_ACT_PRELU || (p->act == B200SVD_ACT_PRELU && p->slope == nullptr)) {
    set_error("b200svd_gemm: act=%d is not a B200SVD_ACT_* value, or PReLU without slopes", (int)p->act);
    return 1;
  }
  d.slope = p->slope;

  int bn = p->bn;
  if (p->act == B200SVD_ACT_GEGLU) {
    if (bn == 0) bn = 256;
    if ((bn != 256 && bn != 128) || (p->n % (uint32_t)bn) != 0) {
      set_error("b200svd_gemm: GEGLU needs the 128- or 256-wide tile its weights were interleaved for and n (%u) "
                "divisible by it, got bn=%d", p->n, bn);
      return 1;
    }
  }
  const uint64_t m_tiles_all = (uint64_t)d.m_tiles[0] * d.m_tiles[1] * d.m_tiles[2];
  if (bn == 0) {
    if (p->n <= 32) bn = 32;
    else if (p->n <= 64) bn = 64;
    else if (p->n <= 128) bn = 128;
    else if (p->n == 160 || p->n == 320) bn = 160;  // no ragged N tile
    // a single M tile: the 128-wide tile spreads such a (weight-streaming) GEMM over more SMs
    else bn = m_tiles_all < 2 ? 128 : 256;
  }
  // wgmma takes N <= 256: a 320-wide tile is computed as two 160-wide tiles
  if (bn == 320) bn = 160;
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  // The epilogue stores column pairs as one word (bf16x2 or float2) and loads residual pairs as one 32-bit word
  // whenever the element offset from the base is even, so every base must be aligned to that word.
  const bool res_ok = (p->res1 == nullptr || (p->ld1 % 8 == 0 && al16(p->res1))) &&
                      (p->res2 == nullptr || (p->ld2 % 8 == 0 && al16(p->res2)));
  const bool bf16_ok = p->ldo % 8 == 0 && al16(p->out);
  if (!res_ok || (!p->out_fp32 && !bf16_ok)) {
    set_error("b200svd_gemm: bf16 outputs/residuals need 16-byte aligned bases and leading dims that are multiples of 8");
    return 1;
  }
  if (p->out_fp32 && (reinterpret_cast<uintptr_t>(p->out) & 7) != 0) {
    set_error("b200svd_gemm: an fp32 output needs an 8-byte aligned base");
    return 1;
  }
  const uint32_t n_out = p->act == B200SVD_ACT_GEGLU ? p->n / 2 : p->n;
  if (p->gn_part != nullptr &&
      (p->act != B200SVD_ACT_NONE || p->out_fp32 || (n_out % 16) != 0 || bn < 128 || p->gn_slot_sample == nullptr ||
       p->gn_ld < (int64_t)p->n || (p->gn_ld % 2) != 0 || (reinterpret_cast<uintptr_t>(p->gn_part) & 7) != 0)) {
    set_error("b200svd_gemm: gn_part needs the activation-free bf16 epilogue (n %% 16 == 0, n > 64), gn_slot_sample and "
              "an 8-byte aligned partial buffer with gn_ld >= n");
    return 1;
  }

  // bf16 outputs are staged in shared memory and written by TMA stores, their residuals read by TMA loads.  A TMA
  // store writes whole 16-byte chunks of a row, so this needs an output width that is a multiple of 8.
  EpiMaps em;
  memset(&em, 0, sizeof(em));
  // PReLU stores from registers: its per-column slopes in the staged body would cost the cooperative 128-wide kernel
  // registers it does not have (ptxas spills), and no other launch uses them.
  d.staged = !p->out_fp32 && n_out % 8 == 0 && p->act != B200SVD_ACT_PRELU;
  d.epi_kind = g_epilogue != 0 ? epilogue_kind(p) : B200SVD_EPI_GENERIC;
  int alt_bn = 0;
  if (d.staged && p->gn_part == nullptr && g_schedule != 0) {
    alt_bn = alt_tile(bn, p->act == B200SVD_ACT_GEGLU);
    if (alt_bn != 0 && g_schedule == 2) {
      const uint64_t tiles = m_tiles_all * ((p->n + alt_bn - 1) / alt_bn);
      const uint64_t mma_clocks = (uint64_t)d.taps * d.kblocks * 2 * alt_bn;
      if (tiles < 2 * (uint64_t)sm_count() || mma_clocks >= ALT_MAX_TILE_MMA_CLOCKS) alt_bn = 0;
    }
  }
  if (d.staged) {
    for (int i = 0; i < 3; ++i) {
      if (p->out_rs[i] <= 0) {
        set_error("b200svd_gemm: a bf16 output needs positive row strides, got out_rs[%d]=%lld", i,
                  (long long)p->out_rs[i]);
        return 1;
      }
    }
    const uint64_t od[4] = {n_out, p->m_ext[0], p->m_ext[1], p->m_ext[2]};
    auto row_strides = [&](int64_t ld, uint64_t* s) {
      for (int i = 0; i < 3; ++i) s[i] = (uint64_t)p->out_rs[i] * (uint64_t)ld * 2;
    };
    // each consumer warpgroup stores its 64 rows: the row box halved in its outermost non-unit dimension
    uint32_t ob[4] = {(uint32_t)SUB_W, p->m_box[0], p->m_box[1], p->m_box[2]};
    const int hd = p->m_box[2] > 1 ? 2 : (p->m_box[1] > 1 ? 1 : 0);
    if (alt_bn == 0) {  // the alternating schedule stores the whole row box
      ob[1 + hd] /= 2;
      d.wg_off[hd] = ob[1 + hd];
    }
    uint64_t os[3];
    row_strides(p->ldo, os);
    if (encode_tmap_bf16_sw64(&em.out, p->out, 4, od, os, ob)) return 1;
    const uint32_t rb[4] = {(uint32_t)SUB_W, p->m_box[0], p->m_box[1], p->m_box[2]};
    if (p->res1 != nullptr) {
      row_strides(p->ld1, os);
      if (encode_tmap_bf16_sw64(&em.res1, p->res1, 4, od, os, rb)) return 1;
    }
    if (p->res2 != nullptr) {
      row_strides(p->ld2, os);
      if (encode_tmap_bf16_sw64(&em.res2, p->res2, 4, od, os, rb)) return 1;
    }
  }

  CUtensorMap tmA;
  if (encode_tmap_bf16(&tmA, p->a_ptr, 5, p->a_dims, p->a_strides, p->a_box)) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (alt_bn) {
    case 0: break;
    case 32: return launch<32, true>(p, tmA, em, d, st);
    case 64: return launch<64, true>(p, tmA, em, d, st);
    case 128: return launch<128, true>(p, tmA, em, d, st);
  }
  switch (bn) {
    case 32: return launch<32>(p, tmA, em, d, st);
    case 64: return launch<64>(p, tmA, em, d, st);
    case 128: return launch<128>(p, tmA, em, d, st);
    case 160: return launch<160>(p, tmA, em, d, st);
    case 256: return launch<256>(p, tmA, em, d, st);
    default: set_error("b200svd_gemm: unsupported N tile %d", bn); return 1;
  }
}
