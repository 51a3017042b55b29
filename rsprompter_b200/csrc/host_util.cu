#include "host_util.h"

#include <stdarg.h>

#include <mutex>

namespace rsp {

static thread_local char g_last_error[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

const char* last_error() { return g_last_error; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(out, base, rank, dims, strides_bytes, box, 0);
}

int make_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
              const uint32_t* box, int is_f32) {
  return make_tmap_swizzled(out, base, rank, dims, strides_bytes, box, is_f32, 128);
}

int make_tmap_swizzled(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                       const uint64_t* strides_bytes, const uint32_t* box, int is_f32, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return RSP_ERR_CUDA;
  }
  RSP_CHECK_ARG(rank >= 2 && rank <= 5, "tensor map rank %d", rank);
  RSP_CHECK_ARG((reinterpret_cast<uintptr_t>(base) & 15) == 0, "tensor map base not 16B aligned");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    RSP_CHECK_ARG(box[i] >= 1 && box[i] <= 256, "tensor map box[%d]=%u", i, box[i]);
  }
  for (int i = 0; i < rank - 1; ++i) {
    gstr[i] = strides_bytes[i];
    RSP_CHECK_ARG((strides_bytes[i] & 15) == 0, "tensor map stride[%d]=%llu not 16B multiple", i,
                  (unsigned long long)strides_bytes[i]);
  }
  RSP_CHECK_ARG(swizzle_bytes == 32 || swizzle_bytes == 64 || swizzle_bytes == 128, "swizzle %d", swizzle_bytes);
  RSP_CHECK_ARG(box[0] * (is_f32 ? 4 : 2) <= static_cast<uint32_t>(swizzle_bytes),
                "swizzle-%dB inner box must be <= %d bytes", swizzle_bytes, swizzle_bytes);
  const CUtensorMapSwizzle sw = swizzle_bytes == 128  ? CU_TENSOR_MAP_SWIZZLE_128B
                                : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                      : CU_TENSOR_MAP_SWIZZLE_32B;
  CUresult r = fn(out, is_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base),
                  gdim, gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed: CUresult %d (rank %d dims %llu,%llu box %u,%u)",
                   (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0],
                   box[1]);
    return RSP_ERR_CUDA;
  }
  return RSP_OK;
}

int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev < 0 ? 0 : (dev >= kMaxDevices ? kMaxDevices - 1 : dev);
}

int num_sms() {
  static int n[kMaxDevices] = {};
  const int dev = current_device();
  if (n[dev] == 0) {
    cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
    if (n[dev] <= 0) n[dev] = 132;
  }
  return n[dev];
}

}  // namespace rsp
