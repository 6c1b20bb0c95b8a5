// Host-side helpers shared by the .cu translation units of libb200svd.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

namespace b200 {

void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);  // records the error, returns non-zero

// cuTensorMapEncodeTiled resolved through cudaGetDriverEntryPoint (no link-time libcuda dependency).
// bf16 elements, 128-byte swizzle, zero fill out of bounds.
int encode_tmap_bf16(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                     const uint32_t* box);
// same, no swizzle (dense smem box)
int encode_tmap_bf16_noswz(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims,
                           const uint64_t* strides_bytes, const uint32_t* box);
// same, 64-byte swizzle (inner box extent 32 bf16)
int encode_tmap_bf16_sw64(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box);
// same, 32-byte swizzle (inner box extent 16 bf16)
int encode_tmap_bf16_sw32(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box);

int sm_count();

// true if p is a multiple of `bytes` (a power of two): the base a kernel's 8- or 16-byte vector accesses need
inline bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// Launch-attribute caches (cudaFuncSetAttribute results, occupancy queries) are kept PER DEVICE: function attributes
// belong to a device's context, and one process may drive several GPUs (the reference does not, but the caches must not
// silently assume it).  Index of the calling thread's current device, folded into [0, B200_MAX_DEVICES).
constexpr int B200_MAX_DEVICES = 16;
inline int dev_slot() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev & (B200_MAX_DEVICES - 1);
}

#define B200_CHECK_LAUNCH(name)                               \
  do {                                                        \
    cudaError_t e__ = cudaGetLastError();                     \
    if (e__ != cudaSuccess) return b200::cuda_fail(e__, name); \
  } while (0)

}  // namespace b200
