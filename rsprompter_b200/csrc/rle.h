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
// The same encoding of canvases that hold one mask each: desc / desc_host int64 [n, 9] = (byte offset of the source
// mask from src, source row bytes, source rows, visible h, w, canvas H, W, origin y0, x0); the canvas is H x W zeros
// with canvas[y0 + y, x0 + x] = mask[y, x] for y < h, x < w.  Work is proportional to h x w, not to H x W.
int mask_rle_placed_lengths(const unsigned char* src, int packed, const long long* desc, const long long* desc_host,
                            int n, long long* offsets, cudaStream_t stream);
int mask_rle_placed_write(const unsigned char* src, int packed, const long long* desc, int n, const long long* offsets,
                          char* pool, int* lengths, cudaStream_t stream);
int mask_rle_union_lengths(const unsigned char* src, int packed, const long long* desc, const long long* desc_host,
                           int n, const long long* parts, const long long* parts_host, int num_parts, long long* offsets,
                           cudaStream_t stream);
int mask_rle_union_write(const unsigned char* src, int packed, const long long* desc, int n, const long long* parts,
                         const long long* offsets, char* pool, int* lengths, cudaStream_t stream);

}  // namespace rsp
