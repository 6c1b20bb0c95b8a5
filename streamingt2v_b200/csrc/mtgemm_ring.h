// Ring arithmetic of the wgmma GEMM's alternating schedule (mtgemm.cu), shared with the host-side protocol
// simulation (tests/test_gemm_schedule.py), so both run the same code.
//
// A ring is `depth` buffers, each guarded by a "full" and an "empty" mbarrier.  A position is the buffer index and
// the parity of the number of times the ring has wrapped: the parity a wait on that buffer's barrier takes.  The
// producer fills the ring in tile order; in the alternating schedule consumer warpgroup w owns the CTA's tiles
// w, w + 2, ... and steps over the other warpgroup's tiles without consuming them.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define MTGEMM_RING_FN __host__ __device__ __forceinline__
#else
#define MTGEMM_RING_FN inline
#endif

namespace b200 {

struct RingPos {
  uint32_t idx, phase;
};

MTGEMM_RING_FN void ring_step(RingPos& r, uint32_t depth) {
  if (++r.idx == depth) {
    r.idx = 0;
    r.phase ^= 1u;
  }
}

MTGEMM_RING_FN void ring_advance(RingPos& r, uint32_t n, uint32_t depth) {
  const uint32_t t = r.idx + n;
  r.phase ^= (t / depth) & 1u;
  r.idx = t % depth;
}

// Which consumer warpgroup (0 or 1) owns the CTA's t-th tile.
MTGEMM_RING_FN uint32_t alt_owner(uint32_t t) { return t & 1u; }

// Residual-ring slots of one tile: the residual producer's loop bound.  `tile_out_w` output columns per tile in
// sub-tiles of `sub_w` columns, clipped at the output width `n_out`, one slot per sub-tile and residual.
MTGEMM_RING_FN uint32_t tile_res_slots(uint32_t n_tile, uint32_t tile_out_w, uint32_t n_out, uint32_t sub_w,
                                       uint32_t nres) {
  const uint32_t o0 = n_tile * tile_out_w;
  if (o0 >= n_out) return 0;
  uint32_t c = (n_out - o0 + sub_w - 1) / sub_w;
  if (c > tile_out_w / sub_w) c = tile_out_w / sub_w;
  return c * nres;
}

}  // namespace b200
