#pragma once
#include "host_util.h"

namespace rsp {

constexpr int kChainApproxNone = 1;     // cv2.CHAIN_APPROX_NONE
constexpr int kChainApproxSimple = 2;   // cv2.CHAIN_APPROX_SIMPLE

// cv2.findContours(canvas, RETR_CCOMP, approx) of canvases that are each the OR of K >= 1 placed bit-packed parts.
// desc / desc_host int64 [n, 4] = (canvas H, W, first part, K), parts / parts_host int64 [num_parts, 7] = (byte
// offset from src, row bytes, rows, visible h, w, canvas y0, x0), as mask_rle_union_* takes them.  The workspace
// (mask_contours_ws_bytes) holds the union of each canvas's parts' bounding rectangle plus a one-pixel border and its
// labels; mask_contours_write reads what mask_contours_lengths left there.
int mask_contours_ws_bytes(const long long* desc_host, int n, const long long* parts_host, int num_parts,
                           long long* bytes);
int mask_contours_lengths(const unsigned char* src, const long long* desc, const long long* desc_host, int n,
                          const long long* parts, const long long* parts_host, int num_parts, int approx, void* ws,
                          long long ws_bytes, long long* contour_offsets, long long* point_offsets,
                          cudaStream_t stream);
int mask_contours_write(const long long* desc_host, int n, const long long* parts_host, int num_parts, int approx,
                        const void* ws, long long ws_bytes, const long long* contour_offsets,
                        const long long* canvas_points, long long num_contours, int* points, long long* point_offsets,
                        int* parents, cudaStream_t stream);

}  // namespace rsp
