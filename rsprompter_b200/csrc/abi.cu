// extern "C" surface of librsp_b200.so (declared in include/rsp_b200.h).
#include "../../include/rsp_b200.h"

#include "attention.h"
#include "gemm.h"
#include "rowops.h"

namespace rsp { const char* last_error(); }
using namespace rsp;

static inline cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }

extern "C" {

int rsp_abi_version(void) { return RSP_ABI_VERSION; }
const char* rsp_last_error(void) { return rsp::last_error(); }

static GemmArgs make_gemm_args(const void* A, int lda, const void* W, int ldw, void* out, int ldo,
                               int M, int N, int K, const float* bias, const void* residual, int ldr,
                               int res_fp32, int res_mod, const int32_t* row_map, int act,
                               int out_fp32) {
  GemmArgs a;
  a.A = A; a.lda = lda; a.W = W; a.ldw = ldw; a.out = out; a.ldo = ldo;
  a.M = M; a.N = N; a.K = K; a.bias = bias; a.residual = residual; a.ldr = ldr;
  a.res_fp32 = res_fp32; a.res_mod = res_mod; a.row_map = row_map; a.act = act;
  a.out_fp32 = out_fp32;
  return a;
}

int rsp_gemm_bf16(const void* A, int lda, const void* W, int ldw, void* out, int ldo, int M, int N,
                  int K, const float* bias, const void* residual, int ldr, int res_fp32, int res_mod,
                  const int32_t* row_map, int act, int out_fp32, int epi_mode, const float* ln_gamma,
                  const float* ln_beta, float ln_eps, const int32_t* res_block_map, int res_block_rows,
                  const float* hyper, float* mask_out, int grid_h, int grid_w, void* stream) {
  GemmArgs a = make_gemm_args(A, lda, W, ldw, out, ldo, M, N, K, bias, residual, ldr, res_fp32,
                              res_mod, row_map, act, out_fp32);
  a.epi_mode = epi_mode; a.ln_gamma = ln_gamma; a.ln_beta = ln_beta; a.ln_eps = ln_eps;
  a.res_block_map = res_block_map; a.res_block_rows = res_block_rows;
  a.hyper = hyper; a.mask_out = mask_out; a.grid_h = grid_h; a.grid_w = grid_w;
  return gemm_bf16(a, S(stream));
}

int rsp_gemm_bf16_grouped(const void* A, int lda, const void* W, int ldw, void* out, int ldo, int M, int N, int K,
                          int m_group_rows, int w_group_rows, const int32_t* row_map, int out_fp32, void* stream) {
  GemmArgs a = make_gemm_args(A, lda, W, ldw, out, ldo, M, N, K, nullptr, nullptr, 0, 1, 0, row_map, 0, out_fp32);
  a.m_group_rows = m_group_rows; a.w_group_rows = w_group_rows;
  return gemm_bf16(a, S(stream));
}

int rsp_conv3x3_nhwc_bf16(const void* x, int B, int H, int W, int C, const void* Wt, int ldw, void* out, int ldo,
                          int N, const float* bias, const void* residual, int ldr, int res_fp32, int act,
                          int out_fp32, void* stream) {
  GemmArgs a = make_gemm_args(x, C, Wt, ldw, out, ldo, B * H * W, N, 9 * C, bias, residual, ldr, res_fp32, 0,
                              nullptr, act, out_fp32);
  a.conv_b = B; a.conv_h = H; a.conv_w = W; a.conv_c = C;
  return conv3x3_bf16(a, S(stream));
}

int rsp_conv3x3_geometry_ok(int B, int H, int W, int C) { return conv3x3_geometry_ok(B, H, W, C) ? 1 : 0; }

int rsp_gemm_bf16_simt(const void* A, int lda, const void* W, int ldw, void* out, int ldo, int M,
                       int N, int K, const float* bias, const void* residual, int ldr, int res_fp32,
                       int res_mod, const int32_t* row_map, int act, int out_fp32, void* stream) {
  return gemm_bf16_simt(make_gemm_args(A, lda, W, ldw, out, ldo, M, N, K, bias, residual, ldr,
                                       res_fp32, res_mod, row_map, act, out_fp32), S(stream));
}

static AttentionArgs make_att_args(const void* qkv, const void* rel_h, const void* rel_w, void* out,
                                   int n_seq, int T, int Sg, int H, int hd, const int32_t* out_row_map = nullptr) {
  AttentionArgs a;
  a.qkv = qkv; a.rel_h = rel_h; a.rel_w = rel_w; a.out = out;
  a.n_seq = n_seq; a.T = T; a.S = Sg; a.H = H; a.hd = hd; a.out_row_map = out_row_map;
  return a;
}

int rsp_vit_attention(const void* qkv, const void* rel_h, const void* rel_w, void* out, int n_seq, int T, int Sg,
                      int H, int hd, const int32_t* out_row_map, void* stream) {
  return vit_attention(make_att_args(qkv, rel_h, rel_w, out, n_seq, T, Sg, H, hd, out_row_map), S(stream));
}

int rsp_vit_attention_simt(const void* qkv, const void* rel_h, const void* rel_w, void* out,
                           int n_seq, int T, int Sg, int H, int hd, void* stream) {
  return vit_attention_simt(make_att_args(qkv, rel_h, rel_w, out, n_seq, T, Sg, H, hd), S(stream));
}

int rsp_attn_softmax_bias(const float* scores, int lds, const float* tab, int ldt, int NT, void* P, int ldp, int n_rows,
                          int T, int Sg, float scale, void* stream) {
  return attn_softmax_bias(scores, lds, tab, ldt, NT, P, ldp, n_rows, T, Sg, scale, S(stream));
}

int rsp_transpose_cols(const void* in, int ld, int col0, int C, int n_seq, int T, void* out, void* stream) {
  return transpose_cols(in, ld, col0, C, n_seq, T, out, S(stream));
}

int rsp_split_heads(const void* in, int ld, int col0, int H, int hd, int n_seq, int T, void* out, void* stream) {
  return split_heads(in, ld, col0, H, hd, n_seq, T, out, S(stream));
}

int rsp_layernorm(const void* in, int in_fp32, int ld_in, void* out, int out_fp32, int ld_out,
                  const float* gamma, const float* beta, const int32_t* src_map, int rows_out, int C,
                  float eps, int act, void* copy_out, int ld_copy, void* stream) {
  LayerNormArgs a;
  a.copy_out = copy_out; a.ld_copy = ld_copy;
  a.in = in; a.in_fp32 = in_fp32; a.ld_in = ld_in; a.out = out; a.out_fp32 = out_fp32;
  a.ld_out = ld_out; a.gamma = gamma; a.beta = beta; a.src_map = src_map; a.rows_out = rows_out;
  a.C = C; a.eps = eps; a.act = act;
  return layernorm_rows(a, S(stream));
}

int rsp_layernorm_add(const void* x, const void* res, int res_fp32, const int32_t* res_block_map,
                      int res_block_rows, const float* gamma, const float* beta, void* out, const float* pos,
                      int pos_mod, void* out_pe, long long rows, int C, float eps, void* stream) {
  return layernorm_add(x, res, res_fp32, res_block_map, res_block_rows, gamma, beta, out, pos, pos_mod, out_pe, rows,
                       C, eps, S(stream));
}

int rsp_patchify16(const float* img, void* out, int B, int H, int W, void* stream) {
  return patchify16(img, out, B, H, W, S(stream));
}

int rsp_im2col_nhwc(const void* in, void* out, int B, int H, int W, int C, int KH, int KW,
                    int stride, int pad, void* stream) {
  return im2col_nhwc(in, out, B, H, W, C, KH, KW, stride, pad, S(stream));
}

int rsp_nhwc_to_nchw(const void* in, int in_fp32, float* out, int B, int HW, int C, void* stream) {
  return nhwc_to_nchw(in, in_fp32, out, B, HW, C, S(stream));
}

int rsp_cast_f32_bf16(const float* in, void* out, long long n, void* stream) {
  return cast_f32_bf16(in, out, n, S(stream));
}

int rsp_add_table_bf16(const void* x, const float* table, void* out, long long n, long long period, void* stream) {
  return add_table_bf16(x, table, out, n, period, S(stream));
}

}  // extern "C"

#include "decoder.h"

extern "C" {

int rsp_gemm_upscale_masks(const void* A, int lda, const void* W, int ldw, int M, int K, const float* bias,
                           const float* hyper, int n_out, float* mask_out, int grid_h, int grid_w, void* stream) {
  GemmArgs a = make_gemm_args(A, lda, W, ldw, nullptr, 0, M, 128, K, bias, nullptr, 0, 1, 0, nullptr, 0, 0);
  a.epi_mode = 3; a.hyper = hyper; a.mask_out = mask_out; a.grid_h = grid_h; a.grid_w = grid_w;
  return gemm_upscale_masks(a, n_out, S(stream));
}

int rsp_add_cast_bf16(const float* a, const float* b, void* out, long long n, long long b_mod,
                      void* stream) {
  return add_cast_bf16(a, b, out, n, b_mod, S(stream));
}

int rsp_token_self_attention(const void* q, const void* k, const void* v, void* out, int N, int T,
                             int heads, int c, void* stream) {
  return token_self_attention(q, k, v, out, N, T, heads, c, S(stream));
}

int rsp_t2i_attention(const void* q, const void* K, const void* V, int ldkv, const int32_t* kv_block, void* out,
                      int N, int Tq, int HW, void* stream) {
  return t2i_attention(q, K, V, ldkv, kv_block, out, N, Tq, HW, S(stream));
}

int rsp_i2t_attention(const void* Q, const int32_t* q_block, const void* ktok, const void* vtok,
                      void* out, int N, int Tq, int HW, void* stream) {
  return i2t_attention(Q, q_block, ktok, vtok, out, N, Tq, HW, S(stream));
}

int rsp_t2i_fused(const void* keys, int ldk, const void* kvw, const float* kvb, const void* pe_kv, const void* q,
                  void* out, int N, int Tq, int HW, void* stream) {
  return t2i_fused(keys, ldk, kvw, kvb, pe_kv, q, out, N, Tq, HW, S(stream));
}

int rsp_i2t_fused(const void* keys, int ldk, const void* wq, const float* qb, const void* pe_q, const void* ktok,
                  const void* vtok, const void* wo, const float* ob, const float* ln_g, const float* ln_b, float eps,
                  void* out, int N, int Tq, int HW, void* stream) {
  return i2t_fused(keys, ldk, wq, qb, pe_q, ktok, vtok, wo, ob, ln_g, ln_b, eps, out, N, Tq, HW, S(stream));
}

}  // extern "C"

#include "detect.h"

extern "C" {

int rsp_rpn_decode(const float* head_out, int ld, const int64_t* topk_idx, int K, int B, int H, int W, int A, int stride,
                   const float* base_anchors, const float* stds4, float img_h, float img_w, const float* img_shapes,
                   float min_size, int out_off, int out_ld, float* boxes, float* scores, void* stream) {
  return rpn_decode(head_out, ld, reinterpret_cast<const long long*>(topk_idx), K, B, H, W, A, stride,
                    base_anchors, stds4, img_h, img_w, img_shapes, min_size, out_off, out_ld, boxes, scores, S(stream));
}

int rsp_bbox_cls_decode(const float* cls, int ld_cls, const float* reg, int ld_reg, const float* rois,
                        const uint8_t* roi_valid, int n, int C, const float* stds4, float img_h, float img_w,
                        const float* img_shapes, float score_thr, float* scores, float* boxes, int64_t* labels,
                        void* stream) {
  return bbox_cls_decode(cls, ld_cls, reg, ld_reg, rois, roi_valid, n, C, stds4, img_h, img_w, img_shapes, score_thr,
                         scores, boxes, reinterpret_cast<long long*>(labels), S(stream));
}

int rsp_nms_batched(const float* boxes, const int64_t* ids, const int32_t* nvalid, int B, int n, float thr,
                    void* mask_ws, float* max_coord_ws, uint8_t* keep, int max_keep, void* stream) {
  return nms_batched(boxes, reinterpret_cast<const long long*>(ids), nvalid, B, n, thr,
                     static_cast<unsigned long long*>(mask_ws), max_coord_ws, keep, max_keep, S(stream));
}

int rsp_nmm_batched(const float* boxes, const int64_t* labels, const int32_t* nvalid, int B, int n, float thr,
                    int metric, void* mask_ws, uint8_t* keep, int32_t* owner, void* stream) {
  return nmm_batched(boxes, reinterpret_cast<const long long*>(labels), nvalid, B, n, thr, metric,
                     static_cast<unsigned long long*>(mask_ws), keep, owner, S(stream));
}

int rsp_compact_keep(const uint8_t* keep, const float* boxes, const float* scores, const int64_t* labels,
                     int B, int n, int K, float* out_boxes, float* out_scores, int64_t* out_labels,
                     int32_t* out_index, int32_t* counts, void* stream) {
  return compact_keep(keep, boxes, scores, reinterpret_cast<const long long*>(labels), B, n, K, out_boxes,
                      out_scores, reinterpret_cast<long long*>(out_labels), out_index, counts, S(stream));
}

int rsp_soft_nms_workspace_bytes(int B, int n, int G, size_t* bytes) {
  RSP_CHECK_ARG(bytes && B > 0 && n > 0 && G >= 1, "soft_nms_workspace_bytes: bad args");
  *bytes = soft_nms_workspace_bytes(B, n, G);
  return RSP_OK;
}

int rsp_soft_nms_batched(const float* boxes, const float* scores, const int64_t* ids, const int32_t* nvalid, int B,
                         int n, int G, float iou_thr, float sigma, float min_score, int method, int split_thr, int K,
                         void* ws, size_t ws_bytes, float* out_boxes, float* out_scores, int64_t* out_labels,
                         int32_t* out_index, int32_t* counts, void* stream) {
  return soft_nms_batched(boxes, scores, reinterpret_cast<const long long*>(ids), nvalid, B, n, G, iou_thr, sigma,
                          min_score, method, split_thr, K, ws, ws_bytes, out_boxes, out_scores,
                          reinterpret_cast<long long*>(out_labels), out_index, counts, S(stream));
}

int rsp_roi_align_nhwc(const void* const* feats, const float* const* pes, const int32_t* Hs,
                       const int32_t* Ws, const float* scales, int num_levels, const float* rois, int n,
                       int C, int P, float finest_scale, void* out, void* stream) {
  return roi_align_nhwc(feats, pes, Hs, Ws, scales, num_levels, rois, n, C, P, finest_scale, out, S(stream));
}

int rsp_mask_paste(const float* maps, uint8_t* out, int n, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w,
                   int H, int W, int Hr, int Wr, int packed, float thr, int mode, void* stream) {
  return mask_paste(maps, out, n, hm, wm, Hb, Wb, crop_h, crop_w, H, W, Hr, Wr, packed, thr, mode, S(stream));
}

int rsp_sigmoid_f32(const float* in, float* out, long long n, void* stream) {
  return sigmoid_f32(in, out, n, S(stream));
}

int rsp_pool2_nhwc(const void* in, void* out, int B, int H, int W, int C, int mode, void* stream) {
  return pool2_nhwc(in, out, B, H, W, C, mode, S(stream));
}

int rsp_zero_border_nhwc(void* x, int N, int H, int W, int C, void* stream) {
  return zero_border_nhwc(x, N, H, W, C, S(stream));
}

int rsp_sin_fold(const float* in, float* out, long long n_out, void* stream) {
  return sin_fold(in, out, n_out, S(stream));
}

}  // extern "C"

#include "query.h"

extern "C" {

int rsp_groupnorm_nhwc(const void* x, float* stats_ws, const float* gamma, const float* beta, const void* up,
                       void* out, int B, int H, int W, int C, int G, float eps, int relu, void* stream) {
  return groupnorm_nhwc(x, stats_ws, gamma, beta, up, out, B, H, W, C, G, eps, relu, S(stream));
}

int rsp_ms_deform_attn_sample(const void* value, const float* ow, int ld_ow, const int32_t* hs, const int32_t* ws,
                              int L, int P, int B, int NQ, void* out, int channels, void* stream) {
  return ms_deform_attn_sample(value, ow, ld_ow, hs, ws, L, P, B, NQ, out, channels, S(stream));
}

int rsp_mha_small(const void* Q, int ldq, const void* K, int ldk, const void* V, int ldv, const uint64_t* mask_bits,
                  int B, int nq, int nk, void* out, int head_dim, void* stream) {
  return mha_small(Q, ldq, K, ldk, V, ldv, reinterpret_cast<const unsigned long long*>(mask_bits), B, nq, nk, out,
                   head_dim, S(stream));
}

int rsp_attn_mask_bits(const float* logits, int ld, int rows, int nk, uint64_t* mask_bits, void* stream) {
  return attn_mask_bits(logits, ld, rows, nk, reinterpret_cast<unsigned long long*>(mask_bits), S(stream));
}

int rsp_resize_bilinear_nhwc(const void* x, int B, int H, int W, int C, int h, int w, void* out, void* stream) {
  return resize_bilinear_nhwc(x, B, H, W, C, h, w, out, S(stream));
}

int rsp_mask_embed_src(const float* mpp, const float* const* wts, const float* emb, const float* pos, int N,
                       int n_per_img, int hm, int wm, int h, int w, float eps, void* src, void* src_pe, void* stream) {
  return mask_embed_src(mpp, wts, emb, pos, N, n_per_img, hm, wm, h, w, eps, src, src_pe, S(stream));
}

int rsp_sam_mask_embed(const float* masks, const float* const* wts, int B, int hm, int wm, int h, int w, float eps,
                       float* dense, void* stream) {
  return sam_mask_embed(masks, wts, B, hm, wm, h, w, eps, dense, S(stream));
}

int rsp_query_postprocess(const float* logits, const int32_t* sel, const float* cls_scores, int n_inst, int hm, int wm,
                          int Hb, int Wb, int crop_h, int crop_w, int H, int W, int Hr, int Wr, int packed,
                          uint8_t* masks, float* part_ws, float* scores, float* boxes, void* stream) {
  return query_postprocess(logits, sel, cls_scores, n_inst, hm, wm, Hb, Wb, crop_h, crop_w, H, W, Hr, Wr, packed, masks,
                           part_ws, scores, boxes, S(stream));
}

int rsp_mask_paste_boxes(const float* probs, const float* boxes, uint8_t* out, int n, int hm, int wm, int H, int W,
                         float thr, int packed, void* stream) {
  return mask_paste_boxes(probs, boxes, out, n, hm, wm, H, W, thr, packed, S(stream));
}

int rsp_panoptic_postprocess(const float* logits, const uint8_t* keep, const float* scores, const int32_t* labels,
                             int n_img, int nq, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w, int H, int W,
                             int num_things, int num_classes, const double* iou_thr, int filter_low_score,
                             uint16_t* idx_ws, uint32_t* bits_ws, int32_t* areas, int32_t* seg, int32_t* pan,
                             void* stream) {
  return panoptic_postprocess(logits, keep, scores, labels, n_img, nq, hm, wm, Hb, Wb, crop_h, crop_w, H, W, num_things,
                              num_classes, iou_thr, filter_low_score, idx_ws, bits_ws, areas, seg, pan, S(stream));
}

int rsp_sam_mask_stats(const float* maps, int n, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w, int H, int W,
                       float thr, float thr_hi, float thr_lo, const float* iou, float pred_iou_thresh,
                       float stability_score_thresh, int crop_x0, int crop_y0, int crop_x1, int crop_y1, int scene_h,
                       int scene_w, int32_t* part_ws, int32_t* counts, int32_t* boxes, float* stability, uint8_t* keep,
                       void* stream) {
  return sam_mask_stats(maps, n, hm, wm, Hb, Wb, crop_h, crop_w, H, W, thr, thr_hi, thr_lo, iou, pred_iou_thresh,
                        stability_score_thresh, crop_x0, crop_y0, crop_x1, crop_y1, scene_h, scene_w, part_ws, counts,
                        boxes, stability, keep, S(stream));
}

}  // extern "C"

#include "records.h"

extern "C" {

int rsp_pack_mask_bits(const uint8_t* masks, uint8_t* bits, long long rows, int W, void* stream) {
  return pack_mask_bits(masks, bits, rows, W, S(stream));
}

int rsp_unpack_mask_bits(const uint8_t* bits, uint8_t* masks, long long rows, int W, void* stream) {
  return unpack_mask_bits(bits, masks, rows, W, S(stream));
}

int rsp_preprocess_u8(const uint8_t* img, int h, int w, long long stride_c, long long stride_y, long long stride_x,
                      float* out, int H, int W, const float* mean3, const float* std3, int swap_rb, float pad_value,
                      void* stream) {
  return preprocess_u8(img, h, w, stride_c, stride_y, stride_x, out, H, W, mean3, std3, swap_rb, pad_value, S(stream));
}

int rsp_resize_pad_u8(const int64_t* desc, const int64_t* desc_host, int B, float* out, int Hp, int Wp,
                      const float* mean3, const float* std3, int swap_rb, const float* pad3, void* stream) {
  return resize_pad_u8(reinterpret_cast<const long long*>(desc), reinterpret_cast<const long long*>(desc_host), B, out,
                       Hp, Wp, mean3, std3, swap_rb, pad3, S(stream));
}

int rsp_resize_aa_pad_u8_ws_bytes(const int64_t* desc_host, int B, long long* bytes) {
  return resize_aa_pad_u8_ws_bytes(reinterpret_cast<const long long*>(desc_host), B, bytes);
}

int rsp_resize_aa_pad_u8(const int64_t* desc, const int64_t* desc_host, const int32_t* tab, const int32_t* tab_host,
                         long long n_tab, int B, uint8_t* ws, long long ws_bytes, float* out, int Hp, int Wp,
                         const float* mean3, const float* std3, int swap_rb, const float* pad3, void* stream) {
  return resize_aa_pad_u8(reinterpret_cast<const long long*>(desc), reinterpret_cast<const long long*>(desc_host), tab,
                          tab_host, n_tab, B, ws, ws_bytes, out, Hp, Wp, mean3, std3, swap_rb, pad3, S(stream));
}

int rsp_patchify16_u8(const uint8_t* img, int hwc, void* out, int B, int H, int W, const float* mean3, const float* std3,
                      int swap_rb, void* stream) {
  return patchify16_u8(img, hwc, out, B, H, W, mean3, std3, swap_rb, S(stream));
}

}  // extern "C"

#include "rle.h"

extern "C" {

int rsp_mask_rle_lengths(const uint8_t* src, int packed, const int64_t* desc, const int64_t* desc_host, int n,
                         int64_t* offsets, void* stream) {
  return mask_rle_lengths(src, packed, reinterpret_cast<const long long*>(desc),
                          reinterpret_cast<const long long*>(desc_host), n, reinterpret_cast<long long*>(offsets),
                          S(stream));
}

int rsp_mask_rle_write(const uint8_t* src, int packed, const int64_t* desc, int n, const int64_t* offsets, char* pool,
                       int32_t* lengths, void* stream) {
  return mask_rle_write(src, packed, reinterpret_cast<const long long*>(desc), n,
                        reinterpret_cast<const long long*>(offsets), pool, lengths, S(stream));
}

int rsp_mask_rle_placed_lengths(const uint8_t* src, int packed, const int64_t* desc, const int64_t* desc_host, int n,
                                int64_t* offsets, void* stream) {
  return mask_rle_placed_lengths(src, packed, reinterpret_cast<const long long*>(desc),
                                 reinterpret_cast<const long long*>(desc_host), n, reinterpret_cast<long long*>(offsets),
                                 S(stream));
}

int rsp_mask_rle_placed_write(const uint8_t* src, int packed, const int64_t* desc, int n, const int64_t* offsets,
                              char* pool, int32_t* lengths, void* stream) {
  return mask_rle_placed_write(src, packed, reinterpret_cast<const long long*>(desc), n,
                               reinterpret_cast<const long long*>(offsets), pool, lengths, S(stream));
}

int rsp_mask_rle_union_lengths(const uint8_t* src, int packed, const int64_t* desc, const int64_t* desc_host, int n,
                               const int64_t* parts, const int64_t* parts_host, int num_parts, int64_t* offsets,
                               void* stream) {
  return mask_rle_union_lengths(src, packed, reinterpret_cast<const long long*>(desc),
                                reinterpret_cast<const long long*>(desc_host), n,
                                reinterpret_cast<const long long*>(parts),
                                reinterpret_cast<const long long*>(parts_host), num_parts,
                                reinterpret_cast<long long*>(offsets), S(stream));
}

int rsp_mask_rle_union_write(const uint8_t* src, int packed, const int64_t* desc, int n, const int64_t* parts,
                             const int64_t* offsets, char* pool, int32_t* lengths, void* stream) {
  return mask_rle_union_write(src, packed, reinterpret_cast<const long long*>(desc), n,
                              reinterpret_cast<const long long*>(parts), reinterpret_cast<const long long*>(offsets),
                              pool, lengths, S(stream));
}

}  // extern "C"

#include "contours.h"

extern "C" {

int rsp_mask_contours_ws_bytes(const int64_t* desc_host, int n, const int64_t* parts_host, int num_parts,
                               long long* bytes) {
  return mask_contours_ws_bytes(reinterpret_cast<const long long*>(desc_host), n,
                                reinterpret_cast<const long long*>(parts_host), num_parts, bytes);
}

int rsp_mask_contours_lengths(const uint8_t* src, const int64_t* desc, const int64_t* desc_host, int n,
                              const int64_t* parts, const int64_t* parts_host, int num_parts, int approx, void* ws,
                              long long ws_bytes, int64_t* contour_offsets, int64_t* point_offsets, void* stream) {
  return mask_contours_lengths(src, reinterpret_cast<const long long*>(desc),
                               reinterpret_cast<const long long*>(desc_host), n,
                               reinterpret_cast<const long long*>(parts),
                               reinterpret_cast<const long long*>(parts_host), num_parts, approx, ws, ws_bytes,
                               reinterpret_cast<long long*>(contour_offsets), reinterpret_cast<long long*>(point_offsets),
                               S(stream));
}

int rsp_mask_contours_write(const int64_t* desc_host, int n, const int64_t* parts_host, int num_parts, int approx,
                            const void* ws, long long ws_bytes, const int64_t* contour_offsets,
                            const int64_t* canvas_points, long long num_contours, int32_t* points,
                            int64_t* point_offsets, int32_t* parents, void* stream) {
  return mask_contours_write(reinterpret_cast<const long long*>(desc_host), n,
                             reinterpret_cast<const long long*>(parts_host), num_parts, approx, ws, ws_bytes,
                             reinterpret_cast<const long long*>(contour_offsets),
                             reinterpret_cast<const long long*>(canvas_points), num_contours, points,
                             reinterpret_cast<long long*>(point_offsets), parents, S(stream));
}

}  // extern "C"

#include "regions.h"

extern "C" {

int rsp_mask_small_regions_bits(const uint8_t* in, uint8_t* out, int n, int H, int W, int ld, long long min_area,
                                int mode, void* ws, uint8_t* changed, int32_t* boxes, void* stream) {
  return mask_small_regions_bits(in, out, n, H, W, ld, min_area, mode, ws, changed, boxes, S(stream));
}

}  // extern "C"
