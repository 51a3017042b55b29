#pragma once
#include "host_util.h"

namespace rsp {

// COCO compressed RLE of binary masks (pycocotools maskApi.c rleEncode + rleToString).  desc / desc_host:
// int64 [n, 3] = (byte offset of mask i from src, H, W), on the device and its host copy (checked before launch).
// packed = 0: uint8 [H, W] masks, any nonzero byte is set; packed = 1: [H, ceil(W/8)] bytes, pixel x = bit x % 8.
int mask_rle_lengths(const unsigned char* src, int packed, const long long* desc, const long long* desc_host, int n,
                     long long* offsets, cudaStream_t stream);
int mask_rle_write(const unsigned char* src, int packed, const long long* desc, int n, const long long* offsets,
                   char* pool, int* lengths, cudaStream_t stream);

}  // namespace rsp
