#pragma once
#include "host_util.h"

namespace rsp {

int rpn_decode(const float* head_out, int ld, const long long* topk_idx, int K, int B, int H, int W,
               int A, int stride, const float* base_anchors, const float* stds4, float img_h, float img_w,
               const float* img_shapes, float min_size, int out_off, int out_ld, float* boxes, float* scores,
               cudaStream_t stream);   // img_shapes: device fp32 [B, 2] (h, w) per image, or null = (img_h, img_w)
int bbox_cls_decode(const float* cls, int ld_cls, const float* reg, int ld_reg, const float* rois,
                    const unsigned char* roi_valid, int n, int C, const float* stds4, float img_h, float img_w,
                    const float* img_shapes, float score_thr, float* scores, float* boxes, long long* labels,
                    cudaStream_t stream);
int nms_batched(const float* boxes, const long long* ids, const int* nvalid, int B, int n, float thr,
                unsigned long long* mask_ws, float* max_coord_ws, unsigned char* keep, int max_keep,
                cudaStream_t stream);   // max_keep > 0: flags past the first max_keep kept candidates may be 0
int nmm_batched(const float* boxes, const long long* labels, const int* nvalid, int B, int n, float thr, int metric,
                unsigned long long* mask_ws, unsigned char* keep, int* owner, cudaStream_t stream);
int compact_keep(const unsigned char* keep, const float* boxes, const float* scores, const long long* labels,
                 int B, int n, int K, float* out_boxes, float* out_scores, long long* out_labels,
                 int* out_index, int* counts, cudaStream_t stream);
size_t soft_nms_workspace_bytes(int B, int n, int G);
int soft_nms_batched(const float* boxes, const float* scores, const long long* ids, const int* nvalid, int B, int n,
                     int G, float iou_thr, float sigma, float min_score, int method, int split_thr, int K, void* ws,
                     size_t ws_bytes, float* out_boxes, float* out_scores, long long* out_labels, int* out_index,
                     int* counts, cudaStream_t stream);
int roi_align_nhwc(const void* const* feats, const float* const* pes, const int* Hs, const int* Ws,
                   const float* scales, int num_levels, const float* rois, int n, int C, int P,
                   float finest_scale, void* out, cudaStream_t stream);
int mask_paste(const float* maps, unsigned char* out, int n, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w,
               int H, int W, int Hr, int Wr, int packed, float thr, int mode, cudaStream_t stream);   // Hb = 0: one resize
int mask_paste_boxes(const float* probs, const float* boxes, unsigned char* out, int n, int hm, int wm, int H, int W,
                     float thr, int packed, cudaStream_t stream);
int sam_mask_stats(const float* maps, int n, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w, int H, int W,
                   float thr, float thr_hi, float thr_lo, const float* iou, float pred_iou_thresh,
                   float stability_thresh, int crop_x0, int crop_y0, int crop_x1, int crop_y1, int scene_h,
                   int scene_w, int* part_ws, int* counts, int* boxes, float* stability, unsigned char* keep,
                   cudaStream_t stream);   // scene_h = 0: no crop-edge rule
int sigmoid_f32(const float* in, float* out, long long n, cudaStream_t stream);
int pool2_nhwc(const void* in, void* out, int B, int H, int W, int C, int mode, cudaStream_t stream);
int zero_border_nhwc(void* x, int N, int H, int W, int C, cudaStream_t stream);
int sin_fold(const float* in, float* out, long long n_out, cudaStream_t stream);

}  // namespace rsp
