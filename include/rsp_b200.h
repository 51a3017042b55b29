/* rsp_b200.h -- C ABI of librsp_b200.so: the H100 (sm_90a) kernels behind the RSPrompter
 * inference hot path (SAM ViT encoder -> prompt-generator heads -> SAM mask decoder).
 *
 * The reference (KyanChen/RSPrompter) has no native code and no FFI: every operation below
 * replaces a PyTorch / cuDNN / cuBLAS / mmcv.ops call made from Python.  Each entry point
 * cites the reference call site it stands in for (paths relative to the reference tree;
 * "HF:" = transformers/models/sam/modeling_sam.py, the un-vendored dependency that holds
 * the encoder / decoder arithmetic, "VS:" = mmpretrain/models/backbones/vit_sam.py,
 * "M:" = mmdet/rsprompter/models.py).
 *
 * Conventions
 *   - plain C: pointers, ints, floats.  No torch types, no C++ exceptions cross the boundary.
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch allocates); the
 *     library allocates nothing and keeps no reference after the call returns.
 *   - `stream` is a cudaStream_t passed as void*; launches are asynchronous, no hidden syncs.
 *   - return value: 0 = ok, 1 = invalid argument, 2 = CUDA error, 3 = unsupported shape;
 *     rsp_last_error() returns a thread-local message for the last non-zero return.
 *   - bf16 = __nv_bfloat16 storage; matrices are row-major with an explicit leading
 *     dimension counted in elements.
 *   - an optional input is a NULL pointer or a zero size; options never get sibling entry points.
 */
#ifndef RSP_B200_H_
#define RSP_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RSP_ABI_VERSION 3

int rsp_abi_version(void);
const char* rsp_last_error(void);

/* Dense contraction with fused epilogue (wgmma + TMA):
 *   out[row_map[m], n] = act(sum_k A[m,k] * W[n,k] + bias[n]) + residual[row_map[m] % res_mod, n]
 * A bf16 [M,K]; W bf16 [N,K] (nn.Linear layout); out bf16 (out_fp32=0) or fp32.
 * act: 0 none, 1 GELU(erf), 2 ReLU.  row_map NULL = identity, -1 entries drop the row
 * (window_unpartition + crop, HF:925-952 / VS:47-75).  residual NULL or fp32/bf16 [*, ldr]
 * (res_fp32 selects), may alias out.  res_mod > 0 broadcasts the residual over the batch
 * (absolute position embedding, HF:1065-1066 / VS:576-588).
 * Replaces: nn.Linear in SamVisionAttention.qkv/.proj (HF:717-718), SamMLPBlock (HF:132-143),
 * mmcv FFN (VS:282-288), patch-embed / 1x1 / im2col'ed 3x3 convs (HF:116,975-992; M:1009-1057,
 * 1296-1363; mmdet rpn_head.py:93-97), bbox-head FCs, and the SamAttention projections of the
 * mask decoder (HF:231-270).
 * The fused epilogues of the SAM mask decoder (HF:461-543):
 *   epi_mode 0  standard (as above)
 *   epi_mode 1  out = LayerNorm_N(acc + bias + residual) * ln_gamma + ln_beta, N % 32 == 0, N <= 256:
 *               layer_norm1-4 / layer_norm_final_attn fused into the preceding out_proj / lin2
 *               (HF:316-347, 398-404)
 *   epi_mode 2  columns = (tap, 64 ch): out = GELU(LN_64(acc + bias)): upscale_conv1 as a GEMM over the
 *               2x2 taps + upscale_layer_norm + GELU (HF:519-520); output rows are then (pixel, tap)
 *   epi_mode 3  rows = (prompt, y, x, tap1), columns = (tap2, 32 ch): mask_out[prompt, 4y+.., 4x+..] =
 *               sum_c GELU(acc + bias)[tap2, c] * hyper[prompt, c]: upscale_conv2 + GELU + the
 *               hypernetwork product (HF:521-531); `out` is unused
 * ln_gamma / ln_beta / ln_eps serve epi_mode 1 and 2, hyper / mask_out / grid_h / grid_w epi_mode 3.
 * res_block_map (int32 [M / res_block_rows], NULL = none) redirects the residual of row r to row
 * map[r / res_block_rows] * res_block_rows + r % res_block_rows: prompts of one image share its
 * embedding without the repeat_interleave copies of M:367-368 / M:1682-1683.
 * epi_mode 0 with a NULL res_block_map is the plain GEMM above.
 * Alignment (a call that breaks it returns RSP_ERR_INVALID, nothing launched):
 *   epi_mode 1  out, residual, bias, ln_gamma, ln_beta 16-byte aligned; ldo, ldr % 8 == 0
 *   epi_mode 2  N % 128 == 0, out 8-byte aligned, ldo % 4 == 0; bias, ln_gamma, ln_beta 16-byte aligned
 *   epi_mode 3  hyper and bias 16-byte aligned, mask_out 8-byte aligned */
int rsp_gemm_bf16(const void* A, int lda, const void* W, int ldw, void* out, int ldo, int M, int N,
                  int K, const float* bias, const void* residual, int ldr, int res_fp32, int res_mod,
                  const int32_t* row_map, int act, int out_fp32, int epi_mode, const float* ln_gamma,
                  const float* ln_beta, float ln_eps, const int32_t* res_block_map, int res_block_rows,
                  const float* hyper, float* mask_out, int grid_h, int grid_w, void* stream);

/* 3x3 / stride 1 / pad 1 convolution on a bf16 NHWC map as an implicit GEMM (replaces F.conv2d of the FPN / RPN /
 * pixel-decoder ConvModules, e.g. M:1205-1216, dense_heads/rpn_head.py:60-75): x [B,H,W,C], Wt bf16 [N, 9*C] with
 * K ordered (ky, kx, c), out [B*H*W, ldo] bf16 or fp32 = act(conv + bias) + residual.  No im2col matrix is built:
 * each tap's A tile is one 4-D TMA box whose halo is zero-filled.  Needs C % 64 == 0 and a pixel grid whose
 * 128-pixel tiles are boxes (rsp_conv3x3_geometry_ok); otherwise RSP_ERR_INVALID. */
int rsp_conv3x3_nhwc_bf16(const void* x, int B, int H, int W, int C, const void* Wt, int ldw, void* out, int ldo,
                          int N, const float* bias, const void* residual, int ldr, int res_fp32, int act,
                          int out_fp32, void* stream);
int rsp_conv3x3_geometry_ok(int B, int H, int W, int C);

/* rsp_gemm_bf16's standard epilogue (epi_mode 0, no res_block_map) on CUDA cores (one thread per output, GELU with
 * erff): the independent check of the tensor-core kernel in tests. */
int rsp_gemm_bf16_simt(const void* A, int lda, const void* W, int ldw, void* out, int ldo, int M,
                       int N, int K, const float* bias, const void* residual, int ldr, int res_fp32,
                       int res_mod, const int32_t* row_map, int act, int out_fp32, void* stream);

/* ViT-SAM attention core: out = softmax(hd^-0.5 * q k^T + rel_h + rel_w) v per (sequence, head).
 * qkv bf16 [n_seq*T, 3*H*hd] (columns [q|k|v], heads contiguous inside each); rel_h / rel_w
 * bf16 [2S-1, hd]; out bf16 [n_seq*T, H*hd].  T = S*S; S = 14 (windows) or 32 / 64 (global) on the
 * tensor cores, other S on rsp_vit_attention_simt; hd = 64 or 80.  The T x T bias of get_decomposed_rel_pos is
 * never materialised.  The tensor-core kernel multiplies P by V in fp16 (V converted from bf16): the output is
 * finite and within the float64 bound of oracle/encoder_attention.py for |v| <= 65280 (the largest bf16 that is a
 * finite fp16; larger |v| become inf), and each |v| below 2^-14 (fp16 subnormal) carries an absolute error of up
 * to 2^-25.
 * out_row_map NULL: output rows in order.  Otherwise window_unpartition + crop (HF:925-952) is fused into the store:
 * output row r of the (window-ordered) sequences goes to row out_row_map[r] of `out` (int32 [n_seq*T], -1 = padding
 * token, dropped), so the projection that follows is a plain GEMM over the B*g*g token rows.
 * Replaces: SamVisionAttention.forward after the qkv Linear and before proj (HF:803-831,
 * HF:729-801) / Attention.forward + add_decomposed_rel_pos (VS:202-221, VS:117-157).
 * rsp_vit_attention_simt: the same on CUDA cores, without out_row_map (rows in order). */
int rsp_vit_attention(const void* qkv, const void* rel_h, const void* rel_w, void* out, int n_seq,
                      int T, int S, int H, int hd, const int32_t* out_row_map, void* stream);

int rsp_vit_attention_simt(const void* qkv, const void* rel_h, const void* rel_w, void* out,
                           int n_seq, int T, int S, int H, int hd, void* stream);

/* LayerNorm over the last dim of [rows, C] (+ optional GELU), fp32 statistics.
 * src_map (int32 [rows_out], NULL = identity): out row i is LN(in[src_map[i]]), or zeros when
 * src_map[i] < 0 -- window_partition's zero padding after LN1 (HF:959-962, HF:900-922).
 * copy_out (bf16 [rows_in, ld_copy] or NULL, fp32 input only): every source row read is also written back as bf16 -
 * the hidden states RSFeatureAggregator consumes (M:1046-1050) leave the encoder without a separate cast pass.
 * Replaces nn.LayerNorm (HF:894-896), SamLayerNorm channels_first (HF:147-170), mmpretrain
 * LayerNorm2d (norm.py:64-89) and LN2d (M:33-50) on channels-last data.
 * C % 4 == 0, C <= 1280, ld_in and ld_out multiples of 4; in and out 16-byte aligned when fp32, 8-byte when bf16;
 * gamma and beta 16-byte aligned; copy_out 8-byte aligned.  Anything else returns RSP_ERR_INVALID. */
int rsp_layernorm(const void* in, int in_fp32, int ld_in, void* out, int out_fp32, int ld_out,
                  const float* gamma, const float* beta, const int32_t* src_map, int rows_out, int C,
                  float eps, int act, void* copy_out, int ld_copy, void* stream);

/* out = LayerNorm(x + residual) over bf16 rows of C <= 256 channels (fp32 statistics): x bf16 [rows, C];
 * residual fp32 or bf16 [*, C], optionally block-mapped as in rsp_gemm_bf16.  The
 * keys = layer_norm4(keys + attn_out) step of SamTwoWayAttentionBlock (HF:345-347).  If out_pe is not
 * NULL it also receives bf16(out + pos[row % pos_mod]) (pos fp32 [pos_mod, C]): "key = keys +
 * key_point_embedding" (HF:326,339), the operand of the following k / q projections. */
int rsp_layernorm_add(const void* x, const void* res, int res_fp32, const int32_t* res_block_map,
                      int res_block_rows, const float* gamma, const float* beta, void* out, const float* pos,
                      int pos_mod, void* out_pe, long long rows, int C, float eps, void* stream);

/* fp32 NCHW image [B,3,H,W] -> bf16 [B*(H/16)*(W/16), 768] patch rows, k = c*256 + ky*16 + kx,
 * so that patch embedding (HF:116,128; mmcv PatchEmbed VS:455) is one rsp_gemm_bf16.
 * B, H, W > 0, H and W multiples of 16, img and out 16-byte aligned; else RSP_ERR_INVALID. */
int rsp_patchify16(const float* img, void* out, int B, int H, int W, void* stream);

/* bf16 NHWC [B,H,W,C] -> [B*Ho*Wo, KH*KW*C] rows, k = (ky*KW + kx)*C + c, zero padding;
 * Ho = (H + 2 pad - KH) / stride + 1, Wo likewise.  B, H, W > 0, C a positive multiple of 8, KH, KW, stride >= 1,
 * pad >= 0, KH <= H + 2 pad and KW <= W + 2 pad (Ho, Wo >= 1), in and out 16-byte aligned; else RSP_ERR_INVALID. */
int rsp_im2col_nhwc(const void* in, void* out, int B, int H, int W, int C, int KH, int KW,
                    int stride, int pad, void* stream);

/* [B, HW, C] (bf16 or fp32) -> fp32 [B, C, HW]: hands NCHW tensors back at module boundaries. */
int rsp_nhwc_to_nchw(const void* in, int in_fp32, float* out, int B, int HW, int C, void* stream);

/* epi_mode 3 for n_out (1..3) hypernetwork vectors per prompt in one GEMM: A bf16 [M, K] up1 rows (prompt, y, x,
 * tap1), W bf16 [128, K], hyper fp32 [prompts, n_out, 32] -> mask_out fp32 [prompts, n_out, 4*grid_h, 4*grid_w].
 * The multimask_output upscale of SamMaskDecoder (HF:521-531, mask_slice 1:): each accumulator tile of
 * upscale_conv2 feeds all n_out products, so the up1 rows are read once.  Output o has the bytes of
 * rsp_gemm_bf16(epi_mode 3) with hyper[:, o].  hyper, bias 16-byte and mask_out 8-byte aligned. */
int rsp_gemm_upscale_masks(const void* A, int lda, const void* W, int ldw, int M, int K, const float* bias,
                           const float* hyper, int n_out, float* mask_out, int grid_h, int grid_w, void* stream);

/* out = bf16(a + b[i % b_mod]) over n fp32 elements (b NULL = plain cast; n, b_mod % 4 == 0):
 * "queries + query_point_embedding" before a projection (HF:318,325,338). */
int rsp_add_cast_bf16(const float* a, const float* b, void* out, long long n, long long b_mod,
                      void* stream);

/* SamAttention core (HF:253-267) for the three shapes the two-way transformer uses; q/k/v are the
 * already-projected bf16 matrices, softmax in fp32, scale = c^-0.5.
 *   token self-attention: q,k,v [N, T, heads*c], T <= 16, c = 32 (or 16)
 *   t2i: q [N, Tq, 128] (8 heads x 16) attends to K,V rows kv_block[n]*HW .. +HW (NULL: n); K / V are 128-column
 *        slices with row stride ldkv (both halves of one fused k|v projection, or two [*,128] matrices)
 *   i2t: Q [*, 128] rows q_block[n]*HW .. +HW attend to ktok,vtok [N, Tq, 128]; out [N*HW, 128] */
int rsp_token_self_attention(const void* q, const void* k, const void* v, void* out, int N, int T,
                             int heads, int c, void* stream);
int rsp_t2i_attention(const void* q, const void* K, const void* V, int ldkv, const int32_t* kv_block, void* out,
                      int N, int Tq, int HW, void* stream);
int rsp_i2t_attention(const void* Q, const int32_t* q_block, const void* ktok, const void* vtok,
                      void* out, int N, int Tq, int HW, void* stream);

/* t2i with the k | v projection of per-prompt image tokens fused in: out = t2i(q, K, V) with
 * [K | V] = bf16((keys Wkv^T + kvb) + pe_kv[row % HW]), keys bf16 [N*HW, 256] (row stride ldk), Wkv bf16 [256, 256]
 * (k_proj rows, then v_proj rows), kvb fp32 [256], pe_kv bf16 [HW, 256], q / out bf16 [N, Tq, 128].  K and V never
 * reach global memory; the bytes equal rsp_gemm_bf16 (residual = pe_kv, res_mod = HW) followed by rsp_t2i_attention. */
int rsp_t2i_fused(const void* keys, int ldk, const void* kvw, const float* kvb, const void* pe_kv, const void* q,
                  void* out, int N, int Tq, int HW, void* stream);

/* The image -> token step of a two-way layer for per-prompt keys, fused:
 *   out = LN((i2t(Q, ktok, vtok) Wo^T + ob) + keys),  Q = bf16((keys Wq^T + qb) + pe_q[row % HW])
 * keys bf16 [N*HW, 256] (row stride ldk; also the residual), Wq bf16 [128, 256], qb fp32 [128], pe_q bf16 [HW, 128],
 * ktok / vtok bf16 [N, Tq, 128], Wo bf16 [256, 128], ob / ln_g / ln_b fp32 [256], out bf16 [N*HW, 256]; HW % 64 == 0.
 * Q and the attention output never reach global memory; the bytes equal rsp_gemm_bf16 (Qimg) ->
 * rsp_i2t_attention -> rsp_gemm_bf16 (epi_mode 1, residual = keys). */
int rsp_i2t_fused(const void* keys, int ldk, const void* wq, const float* qb, const void* pe_q, const void* ktok,
                  const void* vtok, const void* wo, const float* ob, const float* ln_g, const float* ln_b, float eps,
                  void* out, int N, int Tq, int HW, void* stream);

/* ---- detection side of the anchor variant: batched over B images with fixed-size padded
 * candidate lists (score -1 = filtered / padding), so RPN -> RoI head -> mask head runs without
 * host synchronisation.  All arithmetic that decides indices is fp32 without FMA contraction. ---- */

/* RPN: for the K top anchors of one level (topk_idx int64 [B, K] into the (h, w, anchor) order of
 * rpn_head.py:188-190) emit sigmoid scores and decoded, clipped boxes into boxes[B, out_ld, 4] /
 * scores[B, out_ld] at column out_off.  head_out fp32 [B*H*W, ld]: columns [0,A) objectness logits,
 * [A, 5A) deltas.  Anchors are generated analytically (AnchorGenerator, anchor_generator.py:161-301,
 * base_anchors fp32 [A, 4]); boxes failing min_bbox_size get score -1 (rpn_head.py:267-271).
 * stds4: HOST array of the coder's 4 target_stds (bbox_coder.stds; means must be 0).  Boxes are clipped to
 * (img_h, img_w) when img_shapes is NULL, otherwise every image to its own img_meta['img_shape']
 * (rpn_head.py:208-215): img_shapes = DEVICE fp32 [B, 2] (h, w) per image - batches whose images were padded to a
 * common shape by DetDataPreprocessor; img_h / img_w are then unused.
 * Replaces RPNHead._predict_by_feat_single's per-level body + DeltaXYWHBBoxCoder.decode
 * (rpn_head.py:188-226; delta_xywh_bbox_coder.py:325-359). */
int rsp_rpn_decode(const float* head_out, int ld, const int64_t* topk_idx, int K, int B, int H, int W,
                   int A, int stride, const float* base_anchors, const float* stds4, float img_h, float img_w,
                   const float* img_shapes, float min_size, int out_off, int out_ld, float* boxes, float* scores,
                   void* stream);

/* RoI bbox head post-processing before NMS: softmax over C+1 logits, per-class delta2bbox with the
 * coder's target_stds (stds4: HOST array of 4 floats), score_thr filter; rois fp32 [n, 5], roi_valid uint8 [n] or NULL.  Outputs
 * scores [n*C] (-1 = filtered), boxes [n*C, 4], labels int64 [n*C].  Boxes are clipped to (img_h, img_w) when
 * img_shapes is NULL, otherwise to the per-image img_shape (bbox_head.py:545-548): img_shapes DEVICE fp32 [B, 2],
 * indexed by rois[:, 0]; img_h / img_w are then unused.
 * Replaces BBoxHead._predict_by_feat_single up to multiclass_nms (bbox_head.py:520-555,
 * bbox_nms.py:45-75). */
int rsp_bbox_cls_decode(const float* cls, int ld_cls, const float* reg, int ld_reg, const float* rois,
                        const uint8_t* roi_valid, int n, int C, const float* stds4, float img_h, float img_w,
                        const float* img_shapes, float score_thr, float* scores, float* boxes, int64_t* labels,
                        void* stream);

/* mmcv.ops.batched_nms semantics on score-sorted candidates: boxes fp32 [B, n, 4], ids int64 [B, n]
 * (level or class; boxes are offset by id * (max_coord + 1) exactly as mmcv does), nvalid int32 [B]
 * = length of the valid sorted prefix; keep uint8 [B, n].  Suppression when IoU > thr.
 * Workspaces: mask_ws uint64 [B, n, ceil(n/64)], max_coord_ws fp32 [B].  max_keep 0 scans every candidate; max_keep > 0
 * is for callers that only read the first max_keep kept candidates (batched_nms(...)[:max_per_img],
 * rpn_head.py:285-291, bbox_nms.py:95-103): the greedy scan stops once max_keep candidates are kept, later keep flags
 * are 0.
 * Replaces mmcv.ops.batched_nms / nms (rpn_head.py:285, bbox_nms.py:95). */
int rsp_nms_batched(const float* boxes, const int64_t* ids, const int32_t* nvalid, int B, int n, float thr,
                    void* mask_ws, float* max_coord_ws, uint8_t* keep, int max_keep, void* stream);

/* Greedy non-maximum merging (sahi's GREEDYNMM postprocess; no reference counterpart: the reference's large-image
 * merge is mmcv batched_nms).  Score-sorted candidates as rsp_nms_batched takes them: boxes fp32 [B, n, 4], labels
 * int64 [B, n], nvalid int32 [B].  Candidates i < j match when their labels are equal and the metric of their boxes as
 * given (no label offset) is >= thr: metric 0 IoU = inter / ((area_i + area_j) - inter), metric 1 IoS = inter /
 * min(area_i, area_j), area = (x2 - x1) * (y2 - y1), inter = max(0, min(x2) - max(x1)) * max(0, min(y2) - max(y1)),
 * fp32 without contraction; a NaN (0 / 0) does not match.  Greedy in order: a candidate no keeper absorbed is kept
 * (keep uint8 [B, n], as rsp_nms_batched with this match) and absorbs every later unabsorbed candidate it matches;
 * owner int32 [B, n] = the index of the keeper that absorbed candidate i, -1 for keepers and invalid slots.
 * Workspace: mask_ws uint64 [B, n, ceil(n/64)]; at most 393 216 candidates per image. */
int rsp_nmm_batched(const float* boxes, const int64_t* labels, const int32_t* nvalid, int B, int n, float thr,
                    int metric, void* mask_ws, uint8_t* keep, int32_t* owner, void* stream);

/* First K kept candidates per image, in order, zero padded; counts int32 [B].  labels / out_labels /
 * out_index may be NULL.  Replaces results[keep][:max_per_img] (rpn_head.py:289, bbox_nms.py:97-99). */
int rsp_compact_keep(const uint8_t* keep, const float* boxes, const float* scores, const int64_t* labels,
                     int B, int n, int K, float* out_boxes, float* out_scores, int64_t* out_labels,
                     int32_t* out_index, int32_t* counts, void* stream);

/* mmcv.ops.batched_nms with nms_cfg type='soft_nms' (mmcv.ops.soft_nms, softnms_cpu in mmcv/ops/csrc/pytorch/cpu/nms.cpp;
 * rpn_head.py:285-291, bbox_nms.py:95-103, mmdet/utils/large_image.py:76-104).  Candidates in the caller's input order
 * (that order breaks ties): boxes fp32 [B, n, 4], scores fp32 [B, n], ids int64 [B, n] in [0, G), nvalid int32 [B] =
 * length of the valid prefix.  Boxes are offset by id * (max_coord + 1) as mmcv does; below split_thr valid candidates
 * one soft-NMS runs (output in selection order), otherwise one per id, merged by decayed score (ties: lower id, then
 * selection order; mmcv's sort leaves them unordered).  method 0 naive, 1 linear, 2 gaussian; offset 0.  Arithmetic is
 * fp32 without contraction in softnms_cpu's order; gaussian's exp runs in double on the fp32 argument, rounded once.
 * Outputs as rsp_compact_keep: the first K selections, boxes un-offset, scores decayed, zero padded, index -1 past
 * counts; out_labels / out_index may be NULL.  The loop stops after K selections per problem, so K = max_per_img
 * costs K steps.  ws: *bytes from rsp_soft_nms_workspace_bytes(B, n, G, bytes) of device memory, O(B * n + B * G).
 * 1 <= G <= 1024. */
int rsp_soft_nms_workspace_bytes(int B, int n, int G, size_t* bytes);
int rsp_soft_nms_batched(const float* boxes, const float* scores, const int64_t* ids, const int32_t* nvalid, int B,
                         int n, int G, float iou_thr, float sigma, float min_score, int method, int split_thr, int K,
                         void* ws, size_t ws_bytes, float* out_boxes, float* out_scores, int64_t* out_labels,
                         int32_t* out_index, int32_t* counts, void* stream);

/* SingleRoIExtractor + mmcv RoIAlign(output_size=P, sampling_ratio=0, aligned=True, avg)
 * (single_level_roi_extractor.py:55-119, base_roi_extractor.py:58-67) on up to 4 channels-last bf16
 * levels: feats[l] [B, Hs[l], Ws[l], C]; rois fp32 [n, 5] = (batch, x1, y1, x2, y2); level =
 * clamp(floor(log2(sqrt(area) / finest_scale + 1e-6))).  pes (NULL or per-level fp32 [H, W, C]) is the
 * batch-independent extra positional encoding of M:1566-1574, sampled and added on the fly.
 * out bf16 [n, P*P*C] in (ph, pw, c) order.  feats / pes / Hs / Ws / scales are HOST arrays. */
int rsp_roi_align_nhwc(const void* const* feats, const float* const* pes, const int32_t* Hs,
                       const int32_t* Ws, const float* scales, int num_levels, const float* rois, int n,
                       int C, int P, float finest_scale, void* out, void* stream);

/* Mask post-processing: maps fp32 [n, hm, wm] -> thresholded masks, bilinear with align_corners=False.
 * mode 0: bilinear(sigmoid(x)) >= thr (M:1758-1780); mode 1: bilinear(x) > thr (M:652-656 +
 * maskformer_fusion_head.py:169); mode 2: as mode 0 on input that rsp_sigmoid_f32 has already activated (one exp
 * per low-resolution pixel instead of four per output pixel).
 * Hb == 0: one resize (hm, wm) -> (H, W); Wb, crop_h, crop_w are unused.  Otherwise the mask resize of
 * RSPrompterAnchorMaskHead._predict_by_feat_single for resized / padded images (M:1763-1777), modes 1 and 2 only:
 * bilinear to (Hb, Wb) = batch_input_shape -> crop [:crop_h, :crop_w] (the resized, unpadded image) -> bilinear to
 * (H, W) = ori_shape -> threshold.  The intermediate map is never formed.
 * packed = 0: out uint8 [n, H, W], (Hr, Wr) = (H, W).  packed = 1: out holds the masks bit-packed into record slots
 * of Hr x Wr (H <= Hr, W <= Wr, Wr % 16 == 0, out 2-byte aligned): uint8 [n, Hr, Wr/8], pixel x = bit x % 8 of byte
 * x / 8, the (H, W) mask at the slot's top-left, every other pixel 0.  With (Hr, Wr) = (H, W) the bits are
 * rsp_pack_mask_bits of the byte output exactly (predict_records of resized images).
 * One resize writes bytes for W % 16 == 0; it writes bits on the x4 path only (anchor variant, M:1758-1780 when
 * ori_shape == batch shape): (H, W) = (4*hm, 4*wm) = (Hr, Wr), wm % 4 == 0, maps 16-byte aligned, mode 1 or 2.
 * Any other combination returns RSP_ERR_INVALID, nothing launched. */
int rsp_mask_paste(const float* maps, uint8_t* out, int n, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w,
                   int H, int W, int Hr, int Wr, int packed, float thr, int mode, void* stream);

/* out = 1 / (1 + exp(-in)) over n fp32 values (n % 4 == 0): mask_preds.sigmoid() (M:1758). */
int rsp_sigmoid_f32(const float* in, float* out, long long n, void* stream);

/* bf16 NHWC pooling: mode 0 = MaxPool2d(2, 2) (M:1307), mode 1 = max_pool2d(k=1, stride=2) (M:1362). */
int rsp_pool2_nhwc(const void* in, void* out, int B, int H, int W, int C, int mode, void* stream);

/* Zero the 1-pixel border of bf16 NHWC maps [N, H, W, C] in place (C % 8 == 0).  FCNMaskHead's 3x3 convolutions
 * (fcn_mask_head.py:84-98) run on 14x14 RoI maps embedded in 16x16 canvases so that the implicit-GEMM convolution
 * (rsp_conv3x3_nhwc) applies; the border is the convolutions' zero padding and is restored after every layer. */
int rsp_zero_border_nhwc(void* x, int N, int H, int W, int C, void* stream);

/* out[i] = sin(in[2i]) + in[2i+1]: the sin/identity fold of the point embeddings (M:348, M:1672). */
int rsp_sin_fold(const float* in, float* out, long long n_out, void* stream);

/* ---- RSPrompter-query head (M:274-715) ---- */

/* GroupNorm(G) over channels-last bf16 [B,H,W,C] (C/G = 4).  stats_ws: 16-byte aligned fp32 workspace of
 * B*G*2 * (1 + ceil(H*W/256)) floats: (mean, rstd) [B,G,2] followed by the per-256-pixel-block (sum, sumsq) partials,
 * which are folded in fp64 without atomics (bit-reproducible, no E[x^2]-mean^2 cancellation in fp32); optional `up` bf16 [B,H/2,W/2,C] is bilinearly x2-upsampled (align_corners=False) and added after the
 * affine, optional ReLU last: the ConvModule(norm=GN) tails and the FPN top-down add of MSDeformAttnPixelDecoder
 * (msdeformattn_pixel_decoder.py:94-109, 230-240). */
int rsp_groupnorm_nhwc(const void* x, float* stats_ws, const float* gamma, const float* beta, const void* up,
                       void* out, int B, int H, int W, int C, int G, float eps, int relu, void* stream);

/* mmcv MultiScaleDeformableAttention core (deformable_detr_layers.py:237-249): value bf16 [B,NQ,128] (8 heads x 16,
 * already value_proj'ed), ow fp32 [B*NQ, ld_ow] = [sampling_offsets (8*L*P*2) | attention logits (8*L*P)] from one
 * GEMM, levels hs/ws (HOST int arrays, low -> high resolution, sum h*w = NQ).  Softmax over L*P, reference point =
 * the query's own cell centre, bilinear zero-padded sampling as grid_sample(align_corners=False).  out bf16.
 * channels = 8 heads x 16 (128) or 8 heads x 32 (256: the stock Mask2FormerHead's pixel decoder,
 * configs/rsprompter/_base_/samseg-mask2former.py:104-112); value and out are [B, NQ, channels]. */
int rsp_ms_deform_attn_sample(const void* value, const float* ow, int ld_ow, const int32_t* hs, const int32_t* ws,
                              int L, int P, int B, int NQ, void* out, int channels, void* stream);

/* nn.MultiheadAttention core, 8 heads x head_dim (mma.sync flash form): Q bf16 [B,nq,ldq], K / V bf16 [B,nk,ld*],
 * mask_bits uint64 [B*nq, ceil(nk/64)] (bit k%64 of word k/64 set = key k masked, shared by the heads) or NULL;
 * out bf16 [B,nq,8*head_dim].  head_dim 16 (128 channels): masked cross-attention / self-attention of
 * Mask2FormerTransformerDecoderLayer (mask2former_layers.py:113-135); head_dim 32 (256 channels): the stock
 * Mask2FormerTransformerDecoder of samseg-mask2former.py:120-140, where 1/sqrt(32) multiplies the fp32 scores. */
int rsp_mha_small(const void* Q, int ldq, const void* K, int ldk, const void* V, int ldv, const uint64_t* mask_bits,
                  int B, int nq, int nk, void* out, int head_dim, void* stream);

/* attn_mask = sigmoid(x) < 0.5 (= x < 0) per row of level-sized mask logits fp32 [rows, ld >= nk]; a row whose keys
 * are all masked is cleared (M:386-392, M:439-442).  The logits are mask_embed x (bilinearly resized
 * mask_feature)^T: F.interpolate is linear, so resizing the features once replaces resizing every query's map. */
int rsp_attn_mask_bits(const float* logits, int ld, int rows, int nk, uint64_t* mask_bits, void* stream);

/* F.interpolate(x, (h, w), mode='bilinear', align_corners=False) on bf16 NHWC maps (C % 8 == 0). */
int rsp_resize_bilinear_nhwc(const void* x, int B, int H, int W, int C, int h, int w, void* out, void* stream);

/* SamMaskEmbedding (HF:569-593) on mask_pred_plus + image embedding + key PE: for prompt n (image n / n_per_img)
 * src = emb[img] + mask_embed(mpp[n]) bf16 [N*h*w, 256], the mask decoder's source tensor (M:359-368, HF:499), and
 * optionally (src_pe != NULL) src + pos.  wts = HOST array of 10 device pointers (conv1 w,b, ln1 g,b, conv2 w,b,
 * ln2 g,b, conv3 w,b).  emb fp32 [imgs*h*w, 256], pos fp32 [h*w, 256], mpp fp32 [N, 4h, 4w]. */
int rsp_mask_embed_src(const float* mpp, const float* const* wts, const float* emb, const float* pos, int N,
                       int n_per_img, int hm, int wm, int h, int w, float eps, void* src, void* src_pe, void* stream);

/* SamMaskEmbedding.forward (HF:583-593) alone: masks fp32 [B, 4h, 4w] (a low-res mask prompt) -> dense fp32
 * [B*h*w, 256] channels-last rows, the dense_embeddings of SamPromptEncoder.forward with input_masks (HF:691-692).
 * wts as in rsp_mask_embed_src; dense 8-byte aligned. */
int rsp_sam_mask_embed(const float* masks, const float* const* wts, int B, int hm, int wm, int h, int w, float eps,
                       float* dense, void* stream);

/* Instance post-processing of the query variant (M:652-656; maskformer_fusion_head.py:149-182; mask/utils.py:56-77):
 * for instance i (map sel[i] of logits fp32 [*, hm, wm]): bilinear to H x W, mask = > 0, score = cls_scores[i] *
 * mean sigmoid over the positive pixels, tight box.  part_ws fp32 [n_inst, ceil(Hr/16), 6].
 * Hb == 0: one resize (hm, wm) -> (H, W); Wb, crop_h, crop_w are unused.  Otherwise resized / padded images
 * (M:652-656 + 679-691): logits -> (Hb, Wb) -> crop [:crop_h, :crop_w] -> (H, W), then mask, score and box as above.
 * packed = 0: masks uint8 [n_inst, H, W], (Hr, Wr) = (H, W).  packed = 1: the masks bit-packed into record slots
 * uint8 [n_inst, Hr, Wr/8] as rsp_mask_paste writes them; scores and boxes are bit-identical to the byte layout's.
 * One resize writes bytes for W % 4 == 0; it writes bits on the x4 path only ((H, W) = (4*hm, 4*wm) = (Hr, Wr): the
 * mask decoder always emits image/4 logits; wm % 4 == 0, logits 16-byte aligned).  Two resizes write bits for
 * Wr <= 16384.  Any other combination returns RSP_ERR_INVALID, nothing launched. */
int rsp_query_postprocess(const float* logits, const int32_t* sel, const float* cls_scores, int n_inst, int hm, int wm,
                          int Hb, int Wb, int crop_h, int crop_w, int H, int W, int Hr, int Wr, int packed,
                          uint8_t* masks, float* part_ws, float* scores, float* boxes, void* stream);

/* ---- global attention on grids the flash kernel does not specialise (S = 48 / 80: 768^2 / 1280^2 inputs, VS:570-602):
 * three passes per image, all heads batched (rows stacked [H*T]), the two contractions on the wgmma GEMM:
 *   Qh, Kh = rsp_split_heads(qkv)  (bf16 [H*T, hd] each),  Vt = rsp_transpose_cols(qkv)  (bf16 [H*hd, T])
 *   scores = rsp_gemm_bf16_grouped(Qh, Kh)            fp32 [H*T, T]    (group h: Q_h K_h^T)
 *   tab    = rsp_gemm_bf16(Qh, [Rh; Rw])              fp32 [H*T, 2*NT] (NT >= 2S-1 zero-padded table rows)
 *   P      = rsp_attn_softmax_bias(scores, tab)       bf16 [H*T, T]
 *            softmax_k(scale * scores[q, k] + tab[q, qh-kh+S-1] + tab[q, NT + qw-kw+S-1])
 *   out    = rsp_gemm_bf16_grouped(P, Vt, row_map)    bf16 [T, H*hd]   (row_map scatters (h, t) to token t, head h)
 * Replaces HF:803-831 + HF:760-801 / VS:202-221 + VS:117-157 for those grids. ---- */
int rsp_attn_softmax_bias(const float* scores, int lds, const float* tab, int ldt, int NT, void* P, int ldp, int n_rows,
                          int T, int S, float scale, void* stream);

/* bf16 [n_seq*T, ld] columns [col0, col0+C) -> bf16 [n_seq, C, T] (per-head V as the K-contiguous operand of P V). */
int rsp_transpose_cols(const void* in, int ld, int col0, int C, int n_seq, int T, void* out, void* stream);

/* bf16 [n_seq*T, ld] columns [col0 + h*hd, +hd) -> bf16 [n_seq, H, T, hd] (hd % 8 == 0): contiguous per-head operands. */
int rsp_split_heads(const void* in, int ld, int col0, int H, int hd, int n_seq, int T, void* out, void* stream);

/* rsp_gemm_bf16 with one weight matrix per row group: rows [g*m_group_rows, +m_group_rows) of A (m_group_rows % 128
 * == 0, M % m_group_rows == 0) are multiplied with W rows [g*w_group_rows, +N):
 *   out[row_map[m], n] = sum_k A[m, k] * W[(m / m_group_rows) * w_group_rows + n, k]
 * (batched Q K^T / P V; also the per-image  mask_embed x mask_feature  products of the query head, M:352). */
int rsp_gemm_bf16_grouped(const void* A, int lda, const void* W, int ldw, void* out, int ldo, int M, int N, int K,
                          int m_group_rows, int w_group_rows, const int32_t* row_map, int out_fp32, void* stream);

/* ---- result record payload (SURVEY 8(e)/(f1)): masks leave the device bit-packed.  Bit layout everywhere: a mask
 * row of W pixels is ceil(W/8) bytes, pixel x = bit (x % 8) of byte x / 8 (numpy.packbits(bitorder='little')).  This
 * is the device-side stand-in for encode_mask_results + collect_results (coco_metric.py:346-400, :365). ---- */

/* Panoptic post-processing of the query variants: MaskFormerFusionHead.panoptic_postprocess
 * (mmdet/models/seg_heads/panoptic_fusion_heads/maskformer_fusion_head.py:41-106) after the resize of
 * RSMaskFormerFusionHead.predict (M:663-715; M:652-656 up-sampling), for n_img images of nq queries each, with no host
 * read.  Per image i, over the queries q with keep[i*nq+q] (softmax max score > object_mask_thr, label != num_classes,
 * computed by the caller), in ascending q:
 *   sig = 1 / (1 + expf(-v)) of the resized logit v, prob = scores[i*nq+q] * sig; per pixel the argmax of prob (the
 *   lowest q on ties); mask_area = #(argmax == q), original_area = #(sig >= 0.5); q is skipped unless both are > 0 and
 *   (double) mask_area / original_area >= *iou_thr; a stuff label (>= num_things) writes the label, a thing writes
 *   label + 1000 * instance_id (instance_id from 1, advancing on written things); with filter_low_score only pixels
 *   with sig >= 0.5 of their argmax query are written.  Every other pixel is num_classes.
 * logits fp32 [n_img*nq, hm, wm]; keep uint8 / scores fp32 / labels int32 [n_img*nq]; iou_thr: a HOST pointer to one
 * double (Python's float).  Workspaces: idx_ws uint16 [n_img, H*W], bits_ws uint32 [n_img, ceil(H*W/32)].  Outputs:
 * areas int32 [2, n_img*nq] (mask_area, then original_area; 0 for queries not kept), seg int32 [n_img*nq] (the segment
 * id of q, -1 when skipped or not kept), pan int32 [n_img, H, W].  nq < 65535, num_classes < 1000.
 * Hb == 0: one bilinear resize (hm, wm) -> (H, W) (the batch shape); Wb, crop_h, crop_w are unused.  Otherwise the
 * two resizes of a resized / padded image (M:652-656 + 679-691): logits -> (Hb, Wb) -> crop [:crop_h, :crop_w] ->
 * (H, W) (ori_shape with rescale, the crop itself without). */
int rsp_panoptic_postprocess(const float* logits, const uint8_t* keep, const float* scores, const int32_t* labels,
                             int n_img, int nq, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w, int H, int W,
                             int num_things, int num_classes, const double* iou_thr, int filter_low_score,
                             uint16_t* idx_ws, uint32_t* bits_ws, int32_t* areas, int32_t* seg, int32_t* pan,
                             void* stream);

/* SAM automatic mask generation, per candidate mask, without the original-size fp32 mask ever existing.  Replaces, for
 * one crop layer, HF SamImageProcessor.post_process_masks(binarize=False) (image_processing_sam.py:423-425) followed by
 * filter_masks (:350-363): iou_scores > pred_iou_thresh, _compute_stability_score (:449-457), masks > mask_threshold and
 * _batched_mask_to_box (:460-506).  maps fp32 [n, hm, wm] low-res logits, geometry as rsp_mask_paste's two resizes
 * (bilinear to (Hb, Wb), crop, bilinear to (H, W); Hb > 0); every pixel is that kernel's sample, so the > thr
 * decisions are its bits exactly.  Outputs per mask: counts int32 [n, 3] = pixels > thr_hi, > thr_lo, > thr
 * (thr_hi / thr_lo = mask_threshold +/- stability_score_offset, rounded to fp32 as torch compares with a python
 * scalar); boxes int32 [n, 4] inclusive pixel xyxy of > thr, [0, 0, 0, 0] when empty; stability fp32 [n] =
 * fp32(count_hi) / fp32(count_lo) (NaN for 0 / 0).
 * With iou fp32 [n] non-null, keep uint8 [n] = (pred_iou_thresh <= 0 or iou > pred_iou_thresh) and
 * (stability_score_thresh <= 0 or stability > stability_score_thresh).  part_ws int32 [n, ceil(H / 16), 7].
 * scene_h == 0: no crop-edge rule; crop_x0 .. scene_w are unused.  Otherwise the masks are those of one crop of a
 * larger scene, with HF filter_masks' crop-edge rule in the keep flag (image_processing_sam.py
 * _is_box_near_crop_edge(box, crop_box, [0, 0, scene_w, scene_h], atol=20)): the H x W masks are the crop box
 * (crop_x0, crop_y0, crop_x1, crop_y1) of a scene_h x scene_w scene, and a mask is also dropped when a side of its box
 * (its empty-mask [0, 0, 0, 0] included), shifted by (crop_x0, crop_y0) and rounded to fp32, lies within 20 of the
 * crop box's side and not within 20 of the scene's.  Applied in the same launch as the other tests; iou is required.
 * Integer reductions only: two calls give identical outputs.  n > 0, H * W < 2^31, n * ceil(H / 16) < 2^31. */
int rsp_sam_mask_stats(const float* maps, int n, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w, int H, int W,
                       float thr, float thr_hi, float thr_lo, const float* iou, float pred_iou_thresh,
                       float stability_score_thresh, int crop_x0, int crop_y0, int crop_x1, int crop_y1, int scene_h,
                       int scene_w, int32_t* part_ws, int32_t* counts, int32_t* boxes, float* stability,
                       uint8_t* keep, void* stream);

/* SAM automatic mask generation's small-region removal (min_mask_region_area) on bit-packed masks.  Replaces, per
 * kept mask, segment_anything/utils/amg.py remove_small_regions(mask, area_thresh, mode) as
 * SamAutomaticMaskGenerator.postprocess_small_regions calls it (cv2.connectedComponentsWithStats(., 8) + np.isin), and
 * batched_mask_to_box of its result.  in / out uint8 [n, H, ld] bit rows (pixel x = bit x % 8 of byte x / 8, ld even,
 * 8 * ld >= W, ld <= 4 * ceil(W / 32); rsp_mask_paste's packed ld = ceil(W / 16) * 2); bits at x >= W are
 * ignored on input and written as 0; out must not overlap in.  The working mask is ~mask (mode 0, holes) or mask
 * (mode 1, islands); its 8-connected components of area < min_area are "small":
 *   holes    out = mask | (every small component)
 *   islands  out = the components of area >= min_area; when there are none, only the largest (ties: the component
 *            whose first 2 x 2 pixel block (y / 2, x / 2) comes first in raster order, cv2's label order)
 *   changed  uint8 [n] = some component is small (even when out equals the mask, as in SAM)
 *   boxes    int32 [n, 4] inclusive pixel xyxy of out, [0, 0, 0, 0] when empty.
 * ws: n * (32 + 4 * ceil(H / 2) * ceil(W / 2)) bytes, 8-byte aligned.  Atomics touch intermediate labels only: two
 * calls give identical outputs.  n > 0, H * W < 2^31. */
int rsp_mask_small_regions_bits(const uint8_t* in, uint8_t* out, int n, int H, int W, int ld, long long min_area,
                                int mode, void* ws, uint8_t* changed, int32_t* boxes, void* stream);

/* FCNMaskHead mask paste (SAMSegMaskRCNN; fcn_mask_head.py:_do_paste_mask + threshold :388-392): activated RoI masks
 * probs fp32 [n, hm, wm] are sampled with F.grid_sample(bilinear, align_corners=False, zero padding) semantics at the
 * image pixel centres mapped into boxes fp32 [n, 4] (x1, y1, x2, y2) -> out uint8 [n, H, W] = (value >= thr); packed != 0 (W % 16 == 0): the
 * result-record layout uint8 [n, H, W/8], pixel x = bit x % 8 of byte x / 8. */
int rsp_mask_paste_boxes(const float* probs, const float* boxes, uint8_t* out, int n, int hm, int wm, int H, int W,
                         float thr, int packed, void* stream);

/* Generic pack / unpack between uint8 {0,1} masks [rows, W] and the payload [rows, ceil(W/8)] (masks produced in
 * the byte layout; unpack is for consumers that want torch.bool masks back). */
int rsp_pack_mask_bits(const uint8_t* masks, uint8_t* bits, long long rows, int W, void* stream);
int rsp_unpack_mask_bits(const uint8_t* bits, uint8_t* masks, long long rows, int W, void* stream);

/* ---- COCO RLE of predicted masks on the device (SURVEY 8(f) rank 1, the RLE half).  Replaces the host encode of every
 * predicted mask in CocoMetric.process: encode_mask_results(pred['masks'].detach().cpu().numpy())
 * (coco_metric.py:365) -> pycocotools mask_util.encode per mask on a Fortran-order copy (mmdet/structures/mask/
 * utils.py:37-53).  The output is pycocotools' compressed string (maskApi.c rleEncode + rleToString) byte for byte.
 * Masks: desc int64 [n, 3] = (byte offset of mask i from src, H, W) in DEVICE memory and desc_host, the same values in
 * host memory; every mask must have 1 .. 2^31 - 1 pixels (else RSP_ERR_INVALID, nothing launched).  packed = 0:
 * uint8 [H, W] row-major, any nonzero byte is set (torch.bool masks); packed = 1: [H, ceil(W/8)] bytes, pixel x = bit
 * x % 8 of byte x / 8 (the result-record payload).  One call covers masks of different sizes.  Two passes size the
 * output exactly:
 *   rsp_mask_rle_lengths  offsets int64 [n + 1]: offsets[i] = first char of mask i, offsets[n] = total chars
 *   rsp_mask_rle_write    chars of mask i into pool[offsets[i], offsets[i + 1]) (pool: offsets[n] bytes) and
 *                         lengths int32 [n] (-1: longer than INT32_MAX chars); src, packed, desc and offsets as
 *                         given to / produced by rsp_mask_rle_lengths.  No write leaves a mask's range.
 * No atomics: two calls give identical bytes. */
int rsp_mask_rle_lengths(const uint8_t* src, int packed, const int64_t* desc, const int64_t* desc_host, int n,
                         int64_t* offsets, void* stream);
int rsp_mask_rle_write(const uint8_t* src, int packed, const int64_t* desc, int n, const int64_t* offsets, char* pool,
                       int32_t* lengths, void* stream);
/* ... of masks placed in larger canvases (a tile's mask in scene coordinates, sahi shift_masks followed by the encode:
 * mmdet/utils/large_image.py:27-73).  desc int64 [n, 9] = (byte offset of the source mask from src, source row bytes,
 * source rows, visible h, w, canvas H, W, origin y0, x0): the string of the H x W canvas that is zero except
 * canvas[y0 + y, x0 + x] = mask[y, x] for y < h, x < w, without that canvas ever existing (the work is proportional to
 * h x w).  RSP_ERR_INVALID, nothing launched, unless 1 <= H*W <= 2^31 - 1, 0 <= y0 < H, 0 <= x0 < W, 1 <= h <= H - y0,
 * 1 <= w <= W - x0, h <= source rows and w <= source row bytes (x 8 when packed).  Pool, offsets and lengths as above. */
int rsp_mask_rle_placed_lengths(const uint8_t* src, int packed, const int64_t* desc, const int64_t* desc_host, int n,
                                int64_t* offsets, void* stream);
int rsp_mask_rle_placed_write(const uint8_t* src, int packed, const int64_t* desc, int n, const int64_t* offsets,
                              char* pool, int32_t* lengths, void* stream);
/* ... of canvases that are each the OR of K >= 1 placed parts (the union mask of a group of tiles' masks that greedy
 * non-maximum merging joined: sahi's GREEDYNMM postprocess ORs the members' shifted masks; no reference counterpart).
 * desc int64 [n, 4] = (canvas H, W, first part, K), parts int64 [num_parts, 7] = (byte offset of the source mask from
 * src, source row bytes, source rows, visible h, w, origin y0, x0), each in DEVICE and HOST memory (the write pass
 * takes the device copies only).  Canvas i is zero except where one of its parts, placed as in
 * rsp_mask_rle_placed_*, is set; neither the canvas nor the OR is formed (the work is proportional to the parts'
 * bounding rectangle times K).  With K = 1 the string is rsp_mask_rle_placed_*'s.  RSP_ERR_INVALID, nothing launched,
 * unless every canvas has 1 .. 2^31 - 1 pixels and parts within [0, num_parts), and every part passes the placed
 * checks.  Pool, offsets and lengths as above. */
int rsp_mask_rle_union_lengths(const uint8_t* src, int packed, const int64_t* desc, const int64_t* desc_host, int n,
                               const int64_t* parts, const int64_t* parts_host, int num_parts, int64_t* offsets,
                               void* stream);
int rsp_mask_rle_union_write(const uint8_t* src, int packed, const int64_t* desc, int n, const int64_t* parts,
                             const int64_t* offsets, char* pool, int32_t* lengths, void* stream);

/* ---- Mask borders as polygons: cv2.findContours(mask, RETR_CCOMP, approx) of every canvas, the call
 * mmdet.structures.mask.bitmap_to_polygon makes per mask on the host (mmdet/structures/mask/structures.py:1166-1194:
 * outs = cv2.findContours(bitmap.astype(np.uint8), cv2.RETR_CCOMP, cv2.CHAIN_APPROX_NONE)), which DetLocalVisualizer
 * calls on every drawn mask.  approx = 1 (cv2.CHAIN_APPROX_NONE) or 2 (cv2.CHAIN_APPROX_SIMPLE).  Canvases are
 * addressed as in rsp_mask_rle_union_* with bit-packed parts (pixel x = bit x % 8 of byte x / 8): desc int64 [n, 4] =
 * (canvas H, W, first part, K), parts int64 [num_parts, 7] = (byte offset from src, row bytes, rows, visible h, w,
 * origin y0, x0), in DEVICE memory and desc_host / parts_host, the same values in host memory.  One part covers a
 * record slot or a tile mask placed in a scene; K > 1 the OR of greedy_nmm's members.  The union is formed only in
 * the workspace, over the rectangle bounding the parts plus a one-pixel zero border; points are canvas coordinates.
 * RSP_ERR_INVALID, nothing launched, on rsp_mask_rle_union_lengths's descriptor checks (with their messages), on a
 * bounding rectangle of more than 2^31 - 1 pixels with its border, or on a workspace smaller than
 * rsp_mask_contours_ws_bytes's (17 bytes per rectangle pixel, plus 40 per canvas).
 *   rsp_mask_contours_lengths  contour_offsets int64 [n + 1]: first contour of canvas i, [n] = all contours;
 *                              point_offsets int64 [n + 1]: first point of canvas i, [n] = all points (negative if a
 *                              canvas has 2^31 points or more)
 *   rsp_mask_contours_write    with the descriptors, approx and workspace the lengths call was given (it reads what
 *                              that call left there) and its two arrays (canvas_points = its point_offsets):
 *                              points int32 [all points, 2] of (x, y); point_offsets int64 [num_contours + 1], the
 *                              first point of every contour; parents int32 [num_contours], the index of a hole's outer
 *                              border within its canvas's list, -1 for an outer border.
 * Per canvas, the contours come in cv2's order with cv2's start points; cv2's hierarchy follows from the parents.
 * Atomics touch intermediate labels only: two calls give identical bytes. */
int rsp_mask_contours_ws_bytes(const int64_t* desc_host, int n, const int64_t* parts_host, int num_parts,
                               long long* bytes);
int rsp_mask_contours_lengths(const uint8_t* src, const int64_t* desc, const int64_t* desc_host, int n,
                              const int64_t* parts, const int64_t* parts_host, int num_parts, int approx, void* ws,
                              long long ws_bytes, int64_t* contour_offsets, int64_t* point_offsets, void* stream);
int rsp_mask_contours_write(const int64_t* desc_host, int n, const int64_t* parts_host, int num_parts, int approx,
                            const void* ws, long long ws_bytes, const int64_t* contour_offsets,
                            const int64_t* canvas_points, long long num_contours, int32_t* points,
                            int64_t* point_offsets, int32_t* parents, void* stream);

/* ---- DetDataPreprocessor on the device (SURVEY 8(f2); data_preprocessor.py:110-148, ImgDataPreprocessor.forward,
 * BatchFixedSizePad :300).  mean3 / std3: HOST arrays of 3 floats in OUTPUT channel order. ---- */

/* One image: uint8 pixels addressed by byte strides (stride_c, stride_y, stride_x): CHW planes as PackDetInputs emits
 * them = (h*w, w, 1), decoded HWC = (1, 3w, 3) -> fp32 planes out[3, H, W]: channel c = input channel
 * (swap_rb ? 2 - c : c), (x - mean[c]) / std[c] with true fp32 division, pixels outside (h, w) = pad_value. */
int rsp_preprocess_u8(const uint8_t* img, int h, int w, long long stride_c, long long stride_y, long long stride_x,
                      float* out, int H, int W, const float* mean3, const float* std3, int swap_rb, float pad_value,
                      void* stream);

/* The test pipeline's keep-ratio Resize + Pad + DetDataPreprocessor for a batch of images of different sizes, one
 * launch.  Replaces, per image, mmcv Resize(keep_ratio=True) -> imrescale -> cv2.resize(float32, INTER_LINEAR)
 * (mmcv/image/geometric.py rescale_size / imresize; cv2 imgproc/src/resize.cpp resizeGeneric, HResizeLinear,
 * VResizeLinear), mmcv Pad(size, pad_val) (mmcv/transforms/processing.py Pad.transform) and data_preprocessor.py:110-148
 * (the configs' test_pipeline, configs/rsprompter/_base_/rsprompter_anchor.py, rsprompter_query.py,
 * samseg-maskrcnn.py, samseg-mask2former.py).  desc / desc_host int64 [B, 8], the same values in DEVICE and HOST
 * memory, per image: (source address, byte strides c, y, x, h, w, new_h, new_w); sources are uint8 CHW planes or HWC
 * views read in place, new_h <= Hp, new_w <= Wp.  out fp32 [B, 3, Hp, Wp]: channel c from input channel
 * (swap_rb ? 2 - c : c), bilinear with cv2's coefficients (computed in double, rounded to float; borders clamped;
 * horizontal pass first), then (x - mean[c]) / std[c] with true fp32 division; outside (new_h, new_w) the raw pad3
 * (HOST, 3 floats in INPUT channel order) normalised the same way.  new == source size reproduces
 * rsp_preprocess_u8 bit for bit. */
int rsp_resize_pad_u8(const int64_t* desc, const int64_t* desc_host, int B, float* out, int Hp, int Wp,
                      const float* mean3, const float* std3, int swap_rb, const float* pad3, void* stream);

/* SamImageProcessor's resize for a batch of images of different sizes, one call (two launches): the keep-ratio
 * resize of transformers 5.5's TorchvisionBackend, tvF.resize(uint8, BILINEAR, antialias=True)
 * (image_processing_backends.py:251), whose filter support widens with the downscale, where rsp_resize_pad_u8 is cv2
 * INTER_LINEAR (2 x 2 taps at any scale, which aliases at 4-20x).  Grey levels byte-identical to torchvision's CPU
 * uint8 path: per axis whose size changes, a triangle filter of support max(in / out, 1) with weights computed in
 * double and fixed to int(w * 2^prec + 0.5), each output clamp((2^(prec-1) + sum(p * w)) >> prec, 0, 255); horizontal
 * pass first, to uint8, then vertical.  The host builds the weight tables (rsprompter_b200._lib.resize_aa_table); an
 * axis whose size does not change gets the identity table (one tap, weight 2^prec), which is exact.
 * desc / desc_host int64 [B, 16], DEVICE and HOST copies: rsp_resize_pad_u8's 8 fields, then (workspace byte offset,
 * x table offset, x row length, x prec, y table offset, y row length, y prec, 0); workspace offsets are the prefix
 * sums of 3 * h * new_w in image order.  tab / tab_host int32 [n_tab], DEVICE and HOST copies: per axis, one row per
 * output index of (first tap, tap count, weights), every tap inside the source axis.  ws: DEVICE uint8 of at least
 * *bytes of rsp_resize_aa_pad_u8_ws_bytes(desc_host, B, bytes) = sum of 3 * h * new_w, the horizontal pass of each image
 * (61 MB for a 20 000^2 scene to 1024).  out, normalisation, channel order and pad exactly as rsp_resize_pad_u8,
 * applied to the resized uint8 pixel. */
int rsp_resize_aa_pad_u8_ws_bytes(const int64_t* desc_host, int B, long long* bytes);
int rsp_resize_aa_pad_u8(const int64_t* desc, const int64_t* desc_host, const int32_t* tab, const int32_t* tab_host,
                         long long n_tab, int B, uint8_t* ws, long long ws_bytes, float* out, int Hp, int Wp,
                         const float* mean3, const float* std3, int swap_rb, const float* pad3, void* stream);

/* The same arithmetic fused into the patch-embed operand loader: uint8 batch [B, 3, H, W] (hwc = 0) or [B, H, W, 3]
 * (hwc = 1), contiguous, 16-byte aligned, H, W % 16 == 0 -> bf16 patch rows [B*(H/16)*(W/16), 768] in (c, ky, kx)
 * order = rsp_patchify16(rsp_preprocess_u8(img)) bit for bit; the fp32 image never exists. */
int rsp_patchify16_u8(const uint8_t* img, int hwc, void* out, int B, int H, int W, const float* mean3, const float* std3,
                      int swap_rb, void* stream);

/* fp32 -> bf16, round to nearest even (n % 4 == 0, in 16-byte and out 8-byte aligned): feeds fp32 hidden states to
 * the bf16 tensor-core GEMMs. */
int rsp_cast_f32_bf16(const float* in, void* out, long long n, void* stream);

/* out = bf16(x + table[i % period]) on bf16 x: the RoI head's extra positional encoding added to one pyramid level
 * (x = [xi + pe_i ...], M:1566-1574), table fp32 [H*W*C], n and period multiples of 8, x, table and out 16-byte
 * aligned. */
int rsp_add_table_bf16(const void* x, const float* table, void* out, long long n, long long period, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RSP_B200_H_ */
