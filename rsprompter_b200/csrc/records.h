#pragma once
#include "host_util.h"

namespace rsp {

int pack_mask_bits(const unsigned char* masks, unsigned char* bits, long long rows, int W, cudaStream_t stream);
int unpack_mask_bits(const unsigned char* bits, unsigned char* masks, long long rows, int W, cudaStream_t stream);
int preprocess_u8(const unsigned char* img, int h, int w, long long stride_c, long long stride_y, long long stride_x,
                  float* out, int H, int W, const float* mean3, const float* std3, int swap_rb, float pad_value,
                  cudaStream_t stream);
int resize_pad_u8(const long long* desc, const long long* desc_host, int B, float* out, int Hp, int Wp,
                  const float* mean3, const float* std3, int swap_rb, const float* pad3, cudaStream_t stream);
int resize_aa_pad_u8_ws_bytes(const long long* desc_host, int B, long long* bytes);
int resize_aa_pad_u8(const long long* desc, const long long* desc_host, const int* tab, const int* tab_host,
                     long long n_tab, int B, unsigned char* ws, long long ws_bytes, float* out, int Hp, int Wp,
                     const float* mean3, const float* std3, int swap_rb, const float* pad3, cudaStream_t stream);
int patchify16_u8(const unsigned char* img, int hwc, void* out, int B, int H, int W, const float* mean3,
                  const float* std3, int swap_rb, cudaStream_t stream);

}  // namespace rsp
