// Library-level plumbing: error string, device check, TMA descriptor encoding.
#include "common.h"

#include <string.h>

#include "../../include/b200svd.h"

namespace b200 {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
  return 1;
}

typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_tiled_fn g_encode = nullptr;

static int resolve_encode() {
  if (g_encode) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess) return cuda_fail(e, "cudaGetDriverEntryPoint(cuTensorMapEncodeTiled)");
  if (qres != cudaDriverEntryPointSuccess || fn == nullptr) {
    set_error("cuTensorMapEncodeTiled not available from the driver (query result %d)", (int)qres);
    return 1;
  }
  g_encode = reinterpret_cast<encode_tiled_fn>(fn);
  return 0;
}

static int encode_impl(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims,
                       const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz) {
  if (resolve_encode()) return 1;
  cuuint64_t gdims[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  if ((reinterpret_cast<uintptr_t>(gptr) & 15) != 0) {
    set_error("TMA: global address %p is not 16-byte aligned", gptr);
    return 1;
  }
  for (int i = 0; i + 1 < rank; ++i) {
    if (gstr[i] % 16 != 0) {
      set_error("TMA: stride[%d]=%llu bytes is not a multiple of 16", i + 1, (unsigned long long)gstr[i]);
      return 1;
    }
  }
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(gptr), gdims, gstr,
                        bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error(
        "cuTensorMapEncodeTiled failed (CUresult %d) rank=%d dims=[%llu,%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u,%u] "
        "stride1=%llu",
        (int)r, rank, (unsigned long long)gdims[0], (unsigned long long)(rank > 1 ? gdims[1] : 0),
        (unsigned long long)(rank > 2 ? gdims[2] : 0), (unsigned long long)(rank > 3 ? gdims[3] : 0),
        (unsigned long long)(rank > 4 ? gdims[4] : 0), bx[0], rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0,
        rank > 3 ? bx[3] : 0, rank > 4 ? bx[4] : 0, (unsigned long long)(rank > 1 ? gstr[0] : 0));
    return 1;
  }
  return 0;
}

int encode_tmap_bf16(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                     const uint32_t* box) {
  return encode_impl(out, gptr, rank, dims, strides_bytes, box, CU_TENSOR_MAP_SWIZZLE_128B);
}
int encode_tmap_bf16_noswz(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims,
                           const uint64_t* strides_bytes, const uint32_t* box) {
  return encode_impl(out, gptr, rank, dims, strides_bytes, box, CU_TENSOR_MAP_SWIZZLE_NONE);
}

int encode_tmap_bf16_sw64(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box) {
  return encode_impl(out, gptr, rank, dims, strides_bytes, box, CU_TENSOR_MAP_SWIZZLE_64B);
}

int encode_tmap_bf16_sw32(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box) {
  return encode_impl(out, gptr, rank, dims, strides_bytes, box, CU_TENSOR_MAP_SWIZZLE_32B);
}

int sm_count() {
  static int n[B200_MAX_DEVICES] = {};
  const int slot = dev_slot();
  if (n[slot] == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n[slot], cudaDevAttrMultiProcessorCount, dev);
    if (n[slot] <= 0) n[slot] = 132;
  }
  return n[slot];
}

}  // namespace b200

extern "C" {

const char* b200svd_last_error(void) { return b200::g_err; }

int b200svd_version(void) { return 100; }

int b200svd_init(int device) {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess) return b200::cuda_fail(e, "cudaGetDeviceCount");
  if (device < 0 || device >= count) {
    b200::set_error("device %d out of range (%d devices)", device, count);
    return 1;
  }
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) return b200::cuda_fail(e, "cudaGetDeviceProperties");
  if (prop.major != 9 || prop.minor != 0) {
    b200::set_error("b200svd requires an sm_90 GPU (Hopper H100); device %d is sm_%d%d — no fallback path",
                    device, prop.major, prop.minor);
    return 1;
  }
  // no cudaSetDevice here: the caller (PyTorch) owns the current device; launches go to the caller's stream
  return b200::resolve_encode();
}

}  // extern "C"
