// Host-side helpers: error plumbing for the C ABI and TMA tensor-map construction.
// cuTensorMapEncodeTiled is fetched through cudaGetDriverEntryPoint so the library has no
// link-time dependency on libcuda (it must load on a box without a GPU for the symbol test).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace rsp {

enum Status : int {
  RSP_OK = 0,
  RSP_ERR_INVALID = 1,   // bad argument (shape / alignment / null pointer)
  RSP_ERR_CUDA = 2,      // CUDA runtime or driver error
  RSP_ERR_UNSUPPORTED = 3
};

void set_last_error(const char* fmt, ...);

#define RSP_CHECK_ARG(cond, ...)            \
  do {                                      \
    if (!(cond)) {                          \
      ::rsp::set_last_error(__VA_ARGS__);   \
      return ::rsp::RSP_ERR_INVALID;        \
    }                                       \
  } while (0)

#define RSP_CHECK_CUDA(expr)                                                              \
  do {                                                                                    \
    cudaError_t e_ = (expr);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      ::rsp::set_last_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr,                  \
                            cudaGetErrorString(e_));                                      \
      return ::rsp::RSP_ERR_CUDA;                                                         \
    }                                                                                     \
  } while (0)

#define RSP_CHECK_LAUNCH() RSP_CHECK_CUDA(cudaGetLastError())

#define RSP_TRY(expr)            \
  do {                           \
    int s_ = (expr);             \
    if (s_ != 0) return s_;      \
  } while (0)

// bf16 tensor map with 128-byte swizzle.  dims/strides innermost first; strides in bytes
// for dims 1..rank-1 (dim 0 is contiguous).  Out-of-bounds box elements read as zero.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box);
// same for bf16 (is_f32 = 0) or fp32 elements; also used for TMA stores (out-of-range box parts are clipped)
int make_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
              const uint32_t* box, int is_f32);
// same with a 32-, 64- or 128-byte swizzle (the inner box must fit in one swizzle span)
int make_tmap_swizzled(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                       const uint64_t* strides_bytes, const uint32_t* box, int is_f32, int swizzle_bytes);

inline int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                             uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols) {
  uint64_t dims[2] = {cols, rows};
  uint64_t strides[1] = {row_stride_bytes};
  uint32_t box[2] = {box_cols, box_rows};
  return make_tmap_bf16(out, base, 2, dims, strides, box);
}

int num_sms();   // of the current device

constexpr int kMaxDevices = 64;
int current_device();   // cudaGetDevice, clamped to [0, kMaxDevices)

}  // namespace rsp
