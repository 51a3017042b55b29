#pragma once
#include "host_util.h"

namespace rsp {

int groupnorm_nhwc(const void* x, float* stats_ws, const float* gamma, const float* beta, const void* up, void* out,
                   int B, int H, int W, int C, int G, float eps, int relu, cudaStream_t stream);
int ms_deform_attn_sample(const void* value, const float* ow, int ld_ow, const int* hs, const int* ws, int L, int P,
                          int B, int NQ, void* out, int channels, cudaStream_t stream);   // channels = 8 heads x {16, 32}
int mha_small(const void* Q, int ldq, const void* K, int ldk, const void* V, int ldv, const unsigned long long* mask,
              int B, int nq, int nk, void* out, int head_dim, cudaStream_t stream);        // 8 heads x head_dim {16, 32}
int attn_mask_bits(const float* logits, int ld, int rows, int nk, unsigned long long* out, cudaStream_t stream);
int resize_bilinear_nhwc(const void* x, int B, int H, int W, int C, int h, int w, void* out, cudaStream_t stream);
int mask_embed_src(const float* mpp, const float* const* wts, const float* emb, const float* pos, int N, int n_per_img,
                   int hm, int wm, int h, int w, float eps, void* src, void* src_pe, cudaStream_t stream);
int sam_mask_embed(const float* masks, const float* const* wts, int B, int hm, int wm, int h, int w, float eps,
                   float* dense, cudaStream_t stream);
int query_postprocess(const float* logits, const int* sel, const float* cls_scores, int n_inst, int hm, int wm, int Hb,
                      int Wb, int crop_h, int crop_w, int H, int W, int Hr, int Wr, int packed, unsigned char* masks,
                      float* part_ws, float* scores, float* boxes, cudaStream_t stream);   // Hb = 0: one resize
int panoptic_postprocess(const float* logits, const uint8_t* keep, const float* scores, const int* labels, int n_img,
                         int nq, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w, int H, int W, int num_things,
                         int num_classes, const double* iou_thr, int filter_low_score, uint16_t* idx_ws,
                         uint32_t* bits_ws, int* areas, int* seg, int* pan, cudaStream_t stream);   // Hb = 0: one resize

}  // namespace rsp
