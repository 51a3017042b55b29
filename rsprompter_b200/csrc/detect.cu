// Detection-side kernels of the RSPrompter-anchor path: all batched over images with fixed-size
// padded candidate lists, so the whole RPN -> RoI -> mask pipeline runs without host syncs.
//
//   rpn_decode        top-k anchor indices -> sigmoid scores + delta2bbox boxes (rpn_head.py:188-226,
//                     anchor_generator.py:161-301, delta_xywh_bbox_coder.py:325-359)
//   bbox_cls_decode   softmax class scores + per-class delta2bbox (bbox_head.py:520-545)
//   nms_batched       mmcv.ops.batched_nms semantics: boxes offset by id * (max + 1), greedy NMS,
//                     suppress when IoU > thr (bbox_nms.py:95, rpn_head.py:285)
//   nmm_batched       greedy non-maximum merging (sahi GREEDYNMM, no reference counterpart): the NMS bitmask of
//                     an IoU or IoS >= thr match within a label, and the greedy scan also records which keeper
//                     absorbed each candidate
//   compact_keep      first K kept candidates per image -> dense [B, K] outputs + counts
//   roi_align_nhwc    mmcv RoIAlign(aligned=True, sampling_ratio=0, avg) over 4 FPN levels with the
//                     level mapping of SingleRoIExtractor (single_level_roi_extractor.py:55-119); the
//                     extra sine PE of M:1566-1574 is sampled from a per-level table and added
//                     (RoIAlign is linear, so x + PE never has to be materialised)
//   mask_paste        sigmoid + bilinear x4 + threshold (M:1758-1780) / bilinear + (> 0) (M:652-656)
//   pool2_nhwc        MaxPool2d(2,2) and max_pool2d(k=1, s=2) on channels-last maps (M:1307,1362)
//   sin_fold          x[..., ::2].sin() + x[..., 1::2]  (M:348, M:1672)
#include "detect.h"
#include "sm90.cuh"
#include "upsample4.cuh"

#include <climits>

namespace rsp {

// exact-rounding helpers: no FMA contraction, so IoU / box arithmetic matches the fp32 reference
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }

struct Stds4 { float v[4]; };   // DeltaXYWHBBoxCoder target_stds (host array -> kernel parameter)

__device__ __forceinline__ void delta2bbox_one(const float r[4], const float d[4], const float stds[4],
                                               float max_h, float max_w, float out[4]) {
  const float max_ratio = 4.135166556742356f;  // |log(16/1000)|
  const float dx = fmul(d[0], stds[0]), dy = fmul(d[1], stds[1]);
  float dw = fmul(d[2], stds[2]), dh = fmul(d[3], stds[3]);
  const float px = fmul(fadd(r[0], r[2]), 0.5f), py = fmul(fadd(r[1], r[3]), 0.5f);
  const float pw = fsub(r[2], r[0]), ph = fsub(r[3], r[1]);
  dw = fminf(fmaxf(dw, -max_ratio), max_ratio);
  dh = fminf(fmaxf(dh, -max_ratio), max_ratio);
  const float gx = fadd(px, fmul(pw, dx)), gy = fadd(py, fmul(ph, dy));
  const float gw = fmul(pw, expf(dw)), gh = fmul(ph, expf(dh));
  out[0] = fminf(fmaxf(fsub(gx, fmul(gw, 0.5f)), 0.f), max_w);
  out[1] = fminf(fmaxf(fsub(gy, fmul(gh, 0.5f)), 0.f), max_h);
  out[2] = fminf(fmaxf(fadd(gx, fmul(gw, 0.5f)), 0.f), max_w);
  out[3] = fminf(fmaxf(fadd(gy, fmul(gh, 0.5f)), 0.f), max_h);
}

// ---------------------------------------------------------------------------------------
// head_out: fp32 [B*H*W, ld] rows = pixels, columns [0, A) cls logits, [A, 5A) box deltas (a*4 + k)
__global__ void rpn_decode_kernel(const float* __restrict__ head_out, int ld,
                                  const long long* __restrict__ topk_idx, int K, int B, int H, int W,
                                  int A, int stride, const float* __restrict__ base_anchors, Stds4 sd,
                                  float img_h, float img_w, const float* __restrict__ img_shapes, float min_size,
                                  int out_off, int out_ld, float* __restrict__ boxes, float* __restrict__ scores) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * K) return;
  const int b = i / K, k = i - b * K;
  if (img_shapes) { img_h = img_shapes[2 * b]; img_w = img_shapes[2 * b + 1]; }   // per-image img_meta['img_shape']
  const long long idx = topk_idx[i];
  const int a = static_cast<int>(idx % A);
  const long long pix = idx / A;
  const int x = static_cast<int>(pix % W), y = static_cast<int>(pix / W);
  const float* row = head_out + (static_cast<size_t>(b) * H * W + pix) * ld;
  const float logit = row[a];
  const float d[4] = {row[A + a * 4], row[A + a * 4 + 1], row[A + a * 4 + 2], row[A + a * 4 + 3]};
  const float sx = static_cast<float>(x * stride), sy = static_cast<float>(y * stride);
  const float r[4] = {base_anchors[a * 4] + sx, base_anchors[a * 4 + 1] + sy,
                      base_anchors[a * 4 + 2] + sx, base_anchors[a * 4 + 3] + sy};
  const float stds[4] = {sd.v[0], sd.v[1], sd.v[2], sd.v[3]};
  float o[4];
  delta2bbox_one(r, d, stds, img_h, img_w, o);
  float s = 1.0f / (1.0f + expf(-logit));
  if (!(fsub(o[2], o[0]) > min_size && fsub(o[3], o[1]) > min_size)) s = -1.0f;  // filtered (rpn_head.py:267-271)
  const size_t oi = static_cast<size_t>(b) * out_ld + out_off + k;
  boxes[oi * 4] = o[0]; boxes[oi * 4 + 1] = o[1]; boxes[oi * 4 + 2] = o[2]; boxes[oi * 4 + 3] = o[3];
  scores[oi] = s;
}

int rpn_decode(const float* head_out, int ld, const long long* topk_idx, int K, int B, int H, int W,
               int A, int stride, const float* base_anchors, const float* stds4, float img_h, float img_w,
               const float* img_shapes, float min_size, int out_off, int out_ld, float* boxes, float* scores,
               cudaStream_t stream) {
  RSP_CHECK_ARG(head_out && topk_idx && base_anchors && stds4 && boxes && scores && B > 0 && K > 0,
                "rpn_decode: bad args");
  const int n = B * K;
  Stds4 sd{{stds4[0], stds4[1], stds4[2], stds4[3]}};
  rpn_decode_kernel<<<(n + 127) / 128, 128, 0, stream>>>(head_out, ld, topk_idx, K, B, H, W, A, stride,
                                                         base_anchors, sd, img_h, img_w, img_shapes, min_size,
                                                         out_off, out_ld, boxes, scores);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// cls fp32 [n, C+1], reg fp32 [n, 4C], rois fp32 [n, 5]; out scores [n*C] (-1 when <= thr or the
// roi is padding), boxes [n*C, 4], labels int64 [n*C]
__global__ void bbox_cls_decode_kernel(const float* __restrict__ cls, int ld_cls,
                                       const float* __restrict__ reg, int ld_reg,
                                       const float* __restrict__ rois, const unsigned char* __restrict__ roi_valid,
                                       int n, int C, Stds4 sd, float img_h, float img_w,
                                       const float* __restrict__ img_shapes, float score_thr,
                                       float* __restrict__ scores, float* __restrict__ boxes,
                                       long long* __restrict__ labels) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * C) return;
  const int r = i / C, c = i - r * C;
  const float* cr = cls + static_cast<size_t>(r) * ld_cls;
  float mx = cr[0];
  for (int j = 1; j <= C; ++j) mx = fmaxf(mx, cr[j]);
  float sum = 0.f;
  for (int j = 0; j <= C; ++j) sum += expf(cr[j] - mx);
  float s = expf(cr[c] - mx) / sum;
  const float* rr = rois + static_cast<size_t>(r) * 5;
  const float roi[4] = {rr[1], rr[2], rr[3], rr[4]};
  if (img_shapes) {   // per-image img_meta['img_shape'] (bbox_head.py:545-548); the RoI carries its image index
    const int b = static_cast<int>(rr[0]);
    img_h = img_shapes[2 * b]; img_w = img_shapes[2 * b + 1];
  }
  const float* dp = reg + static_cast<size_t>(r) * ld_reg + c * 4;
  const float d[4] = {dp[0], dp[1], dp[2], dp[3]};
  const float stds[4] = {sd.v[0], sd.v[1], sd.v[2], sd.v[3]};
  float o[4];
  delta2bbox_one(roi, d, stds, img_h, img_w, o);
  if (!(s > score_thr) || (roi_valid && !roi_valid[r])) s = -1.0f;
  scores[i] = s;
  boxes[static_cast<size_t>(i) * 4] = o[0]; boxes[static_cast<size_t>(i) * 4 + 1] = o[1];
  boxes[static_cast<size_t>(i) * 4 + 2] = o[2]; boxes[static_cast<size_t>(i) * 4 + 3] = o[3];
  labels[i] = c;
}

int bbox_cls_decode(const float* cls, int ld_cls, const float* reg, int ld_reg, const float* rois,
                    const unsigned char* roi_valid, int n, int C, const float* stds4, float img_h, float img_w,
                    const float* img_shapes, float score_thr, float* scores, float* boxes, long long* labels,
                    cudaStream_t stream) {
  RSP_CHECK_ARG(cls && reg && rois && stds4 && scores && boxes && labels && n > 0 && C > 0, "bbox_cls_decode: bad args");
  const int t = n * C;
  Stds4 sd{{stds4[0], stds4[1], stds4[2], stds4[3]}};
  bbox_cls_decode_kernel<<<(t + 127) / 128, 128, 0, stream>>>(cls, ld_cls, reg, ld_reg, rois, roi_valid, n, C, sd,
                                                              img_h, img_w, img_shapes, score_thr, scores, boxes,
                                                              labels);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// NMS over per-image candidate lists sorted by descending score.  boxes fp32 [B, n, 4]; ids
// int64 [B, n] (level / class); nvalid int32 [B] (sorted prefix with score >= 0).  The offset
// trick of mmcv.batched_nms is reproduced literally: box + id * (max_coord + 1), max over the
// valid boxes of the image.
__device__ __forceinline__ bool iou_gt(const float a[4], const float b[4], float thr) {
  const float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
  const float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
  const float w = fmaxf(fsub(right, left), 0.f), h = fmaxf(fsub(bottom, top), 0.f);
  const float inter = fmul(w, h);
  const float sa = fmul(fsub(a[2], a[0]), fsub(a[3], a[1]));
  const float sb = fmul(fsub(b[2], b[0]), fsub(b[3], b[1]));
  return inter / fsub(fadd(sa, sb), inter) > thr;
}

__global__ void nms_max_coord_kernel(const float* __restrict__ boxes, const int* __restrict__ nvalid,
                                     int n, float* __restrict__ max_coord) {
  __shared__ float red[256];
  const int b = blockIdx.x;
  const int nv = nvalid[b];
  float m = -INFINITY;
  for (int i = threadIdx.x; i < nv * 4; i += blockDim.x) m = fmaxf(m, boxes[static_cast<size_t>(b) * n * 4 + i]);
  red[threadIdx.x] = m;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) max_coord[b] = red[0];
}

__global__ void nms_mask_kernel(const float* __restrict__ boxes, const long long* __restrict__ ids,
                                const int* __restrict__ nvalid, const float* __restrict__ max_coord,
                                int n, float thr, unsigned long long* __restrict__ mask) {
  const int b = blockIdx.z;
  const int nv = nvalid[b];
  const int row0 = blockIdx.y * 64, col0 = blockIdx.x * 64;
  if (row0 >= nv || col0 >= nv || blockIdx.x < blockIdx.y) return;
  const float off1 = fadd(max_coord[b], 1.0f);
  __shared__ float cb[64][4];
  const int cn = min(64, nv - col0);
  if (threadIdx.x < cn) {
    const size_t j = static_cast<size_t>(b) * n + col0 + threadIdx.x;
    const float off = fmul(static_cast<float>(ids[j]), off1);
#pragma unroll
    for (int k = 0; k < 4; ++k) cb[threadIdx.x][k] = fadd(boxes[j * 4 + k], off);
  }
  __syncthreads();
  const int i = row0 + threadIdx.x;
  if (i >= nv) return;
  const size_t gi = static_cast<size_t>(b) * n + i;
  const float off = fmul(static_cast<float>(ids[gi]), off1);
  float a[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) a[k] = fadd(boxes[gi * 4 + k], off);
  unsigned long long bits = 0;
  const int start = (row0 == col0) ? threadIdx.x + 1 : 0;
  for (int j = start; j < cn; ++j)
    if (iou_gt(a, cb[j], thr)) bits |= 1ull << j;
  const int words = (n + 63) / 64;
  mask[(static_cast<size_t>(b) * n + i) * words + blockIdx.x] = bits;
}

// Greedy non-maximum merging's match bitmask, in nms_mask_kernel's layout: bit j of row i (j > i) is set when
// candidates i and j have the same label and IoU (kMetric 0) or IoS (kMetric 1) >= thr, on the boxes as given (no
// label offset, which would change the fp32 rounding).  area = (x2 - x1) * (y2 - y1), inter = max(0, min(x2) -
// max(x1)) * max(0, min(y2) - max(y1)), iou = inter / ((area_i + area_j) - inter), ios = inter / min(area_i, area_j),
// each step rounded once; a NaN (0 / 0) does not match.
template <int kMetric>
__device__ __forceinline__ bool match_ge(const float a[4], const float b[4], float thr) {
  const float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
  const float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
  const float w = fmaxf(fsub(right, left), 0.f), h = fmaxf(fsub(bottom, top), 0.f);
  const float inter = fmul(w, h);
  const float sa = fmul(fsub(a[2], a[0]), fsub(a[3], a[1]));
  const float sb = fmul(fsub(b[2], b[0]), fsub(b[3], b[1]));
  const float v = kMetric == 0 ? __fdiv_rn(inter, fsub(fadd(sa, sb), inter)) : __fdiv_rn(inter, fminf(sa, sb));
  return v >= thr;
}

template <int kMetric>
__global__ void nmm_mask_kernel(const float* __restrict__ boxes, const long long* __restrict__ labels,
                                const int* __restrict__ nvalid, int n, float thr, unsigned long long* __restrict__ mask) {
  const int b = blockIdx.z;
  const int nv = nvalid[b];
  const int row0 = blockIdx.y * 64, col0 = blockIdx.x * 64;
  if (row0 >= nv || col0 >= nv || blockIdx.x < blockIdx.y) return;
  __shared__ float cb[64][4];
  __shared__ long long cl[64];
  const int cn = min(64, nv - col0);
  if (threadIdx.x < cn) {
    const size_t j = static_cast<size_t>(b) * n + col0 + threadIdx.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) cb[threadIdx.x][k] = boxes[j * 4 + k];
    cl[threadIdx.x] = labels[j];
  }
  __syncthreads();
  const int i = row0 + threadIdx.x;
  if (i >= nv) return;
  const size_t gi = static_cast<size_t>(b) * n + i;
  float a[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) a[k] = boxes[gi * 4 + k];
  const long long la = labels[gi];
  unsigned long long bits = 0;
  const int start = (row0 == col0) ? threadIdx.x + 1 : 0;
  for (int j = start; j < cn; ++j)
    if (cl[j] == la && match_ge<kMetric>(a, cb[j], thr)) bits |= 1ull << j;
  const int words = (n + 63) / 64;
  mask[(static_cast<size_t>(b) * n + i) * words + blockIdx.x] = bits;
}

// one CTA (4 warps) per image: greedy scan in score order, 64 candidates at a time.  Warp 0 resolves a
// block serially in registers (the 64 diagonal mask words are held two per lane and broadcast by
// shuffle); then all 128 threads OR the kept rows' remaining words into the suppression bitmap,
// eight independent loads in flight per thread (the mask is L2-resident).
// kOwner (greedy merging): owner[i] = the kept row that suppressed candidate i, -1 for kept and invalid ones.  A bit
// belongs to the first kept row, in order, whose word sets it: in the diagonal block the bits dw & ~cur of a kept
// row, off the diagonal the bits a kept row's word adds to the ones of earlier kept rows (they are ORed in ascending
// row order, and remv already holds those of earlier blocks).
template <bool kOwner>
__global__ void __launch_bounds__(128)
nms_scan_kernel(const unsigned long long* __restrict__ mask, const int* __restrict__ nvalid, int n, int max_keep,
                unsigned char* __restrict__ keep, int* __restrict__ owner) {
  extern __shared__ unsigned long long remv[];
  __shared__ unsigned long long kept_s;
  const int b = blockIdx.x;
  const int nv = nvalid[b];
  const int words = (n + 63) / 64;
  const int nvw = (nv + 63) / 64;
  const int tid = threadIdx.x, lane = tid & 31;
  for (int w = tid; w < words; w += blockDim.x) remv[w] = 0ull;
  if (kOwner)
    for (int i = tid; i < n; i += blockDim.x) owner[static_cast<size_t>(b) * n + i] = -1;
  __syncthreads();
  const unsigned long long* mbase = mask + static_cast<size_t>(b) * n * words;
  int kept_total = 0;     // the caller reads only the first max_keep kept candidates (compact_keep): stop once they exist
  for (int blk = 0; blk < words; ++blk) {
    const int i0 = blk * 64;
    if (blk < nvw && !(max_keep > 0 && kept_total >= max_keep)) {
      if (tid < 32) {
        const int r0 = i0 + lane, r1 = i0 + 32 + lane;
        const unsigned long long d0 = (r0 < nv) ? mbase[static_cast<size_t>(r0) * words + blk] : 0ull;
        const unsigned long long d1 = (r1 < nv) ? mbase[static_cast<size_t>(r1) * words + blk] : 0ull;
        unsigned long long cur = remv[blk], keptbits = 0ull;
        int o0 = -1, o1 = -1;   // kOwner: owners of rows r0 and r1
        for (int tbit = 0; tbit < 64; ++tbit) {
          const unsigned long long dw = __shfl_sync(0xffffffffu, tbit < 32 ? d0 : d1, tbit & 31);
          if (i0 + tbit < nv && !((cur >> tbit) & 1ull)) {
            keptbits |= 1ull << tbit;
            if (kOwner) {
              const unsigned long long fresh = dw & ~cur;
              if ((fresh >> lane) & 1ull) o0 = i0 + tbit;
              if ((fresh >> (lane + 32)) & 1ull) o1 = i0 + tbit;
            }
            cur |= dw;
          }
        }
        if (lane == 0) kept_s = keptbits;
        if (kOwner) {
          if (o0 >= 0) owner[static_cast<size_t>(b) * n + r0] = o0;
          if (o1 >= 0) owner[static_cast<size_t>(b) * n + r1] = o1;
        }
      }
      __syncthreads();
      const unsigned long long keptbits = kept_s;
      kept_total += __popcll(keptbits);
      for (int w = blk + 1 + tid; w < nvw; w += blockDim.x) {
        unsigned long long acc = remv[w];
        unsigned long long kb = keptbits;
        while (kb) {
          unsigned long long v[8];
          int row[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            v[u] = 0ull;
            if (kb) {
              const int tbit = __ffsll(static_cast<long long>(kb)) - 1;
              kb &= kb - 1;
              v[u] = mbase[static_cast<size_t>(i0 + tbit) * words + w];
              if (kOwner) row[u] = i0 + tbit;
            }
          }
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            if (kOwner) {
              unsigned long long fresh = v[u] & ~acc;
              while (fresh) {
                const int j = __ffsll(static_cast<long long>(fresh)) - 1;
                fresh &= fresh - 1;
                owner[static_cast<size_t>(b) * n + w * 64 + j] = row[u];
              }
            }
            acc |= v[u];
          }
        }
        remv[w] = acc;
      }
      for (int tbit = tid; tbit < 64; tbit += blockDim.x)
        if (i0 + tbit < n) keep[static_cast<size_t>(b) * n + i0 + tbit] = (keptbits >> tbit) & 1ull;
      __syncthreads();
    } else {
      for (int tbit = tid; tbit < 64; tbit += blockDim.x)
        if (i0 + tbit < n) keep[static_cast<size_t>(b) * n + i0 + tbit] = 0;
    }
  }
}

int nms_batched(const float* boxes, const long long* ids, const int* nvalid, int B, int n, float thr,
                unsigned long long* mask_ws, float* max_coord_ws, unsigned char* keep, int max_keep,
                cudaStream_t stream) {
  RSP_CHECK_ARG(boxes && ids && nvalid && mask_ws && max_coord_ws && keep && B > 0 && n > 0, "nms: bad args");
  const int words = (n + 63) / 64;
  RSP_CHECK_ARG(words * 8 <= 48 * 1024, "nms: at most %d candidates per image", 48 * 1024 / 8 * 64);
  nms_max_coord_kernel<<<B, 256, 0, stream>>>(boxes, nvalid, n, max_coord_ws);
  RSP_CHECK_LAUNCH();
  dim3 grid(words, words, B);
  nms_mask_kernel<<<grid, 64, 0, stream>>>(boxes, ids, nvalid, max_coord_ws, n, thr, mask_ws);
  RSP_CHECK_LAUNCH();
  nms_scan_kernel<false><<<B, 128, words * 8, stream>>>(mask_ws, nvalid, n, max_keep, keep, nullptr);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

int nmm_batched(const float* boxes, const long long* labels, const int* nvalid, int B, int n, float thr, int metric,
                unsigned long long* mask_ws, unsigned char* keep, int* owner, cudaStream_t stream) {
  RSP_CHECK_ARG(boxes && labels && nvalid && mask_ws && keep && owner && B > 0 && n > 0, "nmm: bad args");
  RSP_CHECK_ARG(metric == 0 || metric == 1, "nmm: metric 0 (IoU) or 1 (IoS), got %d", metric);
  const int words = (n + 63) / 64;
  RSP_CHECK_ARG(words * 8 <= 48 * 1024, "nmm: at most %d candidates per image", 48 * 1024 / 8 * 64);
  dim3 grid(words, words, B);
  if (metric == 0) nmm_mask_kernel<0><<<grid, 64, 0, stream>>>(boxes, labels, nvalid, n, thr, mask_ws);
  else nmm_mask_kernel<1><<<grid, 64, 0, stream>>>(boxes, labels, nvalid, n, thr, mask_ws);
  RSP_CHECK_LAUNCH();
  nms_scan_kernel<true><<<B, 128, words * 8, stream>>>(mask_ws, nvalid, n, 0, keep, owner);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// first K kept candidates of each image, in order.  One warp per image (ballot prefix).
__global__ void compact_keep_kernel(const unsigned char* __restrict__ keep, const float* __restrict__ boxes,
                                    const float* __restrict__ scores, const long long* __restrict__ labels,
                                    int n, int K, float* __restrict__ out_boxes, float* __restrict__ out_scores,
                                    long long* __restrict__ out_labels, int* __restrict__ out_index,
                                    int* __restrict__ counts) {
  const int b = blockIdx.x, lane = threadIdx.x;
  int cnt = 0;
  for (int base = 0; base < n && cnt < K; base += 32) {
    const int i = base + lane;
    const bool k = (i < n) && keep[static_cast<size_t>(b) * n + i];
    const unsigned bal = __ballot_sync(0xffffffffu, k);
    const int pos = cnt + __popc(bal & ((1u << lane) - 1u));
    if (k && pos < K) {
      const size_t src = static_cast<size_t>(b) * n + i, dst = static_cast<size_t>(b) * K + pos;
#pragma unroll
      for (int c = 0; c < 4; ++c) out_boxes[dst * 4 + c] = boxes[src * 4 + c];
      out_scores[dst] = scores[src];
      if (labels) out_labels[dst] = labels[src];
      if (out_index) out_index[dst] = i;
    }
    cnt += __popc(bal);
  }
  cnt = min(cnt, K);
  for (int pos = cnt + lane; pos < K; pos += 32) {
    const size_t dst = static_cast<size_t>(b) * K + pos;
#pragma unroll
    for (int c = 0; c < 4; ++c) out_boxes[dst * 4 + c] = 0.f;
    out_scores[dst] = 0.f;
    if (labels) out_labels[dst] = 0;
    if (out_index) out_index[dst] = -1;
  }
  if (lane == 0) counts[b] = cnt;
}

int compact_keep(const unsigned char* keep, const float* boxes, const float* scores, const long long* labels,
                 int B, int n, int K, float* out_boxes, float* out_scores, long long* out_labels,
                 int* out_index, int* counts, cudaStream_t stream) {
  RSP_CHECK_ARG(keep && boxes && scores && out_boxes && out_scores && counts && B > 0 && n > 0 && K > 0,
                "compact_keep: bad args");
  compact_keep_kernel<<<B, 32, 0, stream>>>(keep, boxes, scores, labels, n, K, out_boxes, out_scores,
                                            out_labels, out_index, counts);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// Soft-NMS: mmcv.ops.batched_nms with nms_cfg type='soft_nms' (softnms_cpu of mmcv/ops/csrc/pytorch/cpu/nms.cpp).
// Candidates are taken in input order (ties go to the lower position, and the serial loop's swaps move positions,
// so the order is part of the answer).  Per image: boxes offset by id * (max + 1) as in nms_batched; below split_thr
// valid candidates one problem, otherwise one problem per id, merged by decayed score.  One CTA per (id, image)
// problem, state in the O(n) workspace: per candidate the offset box, area, running score and input index, plus a
// position -> candidate permutation.  A step is
//   argmax over positions [i, live) (larger score, then lower position; a NaN never replaces the running max, and a
//   NaN at i itself is selected, as the serial scan does) -> swap with i -> decay every position in (i, live) once
//   -> removal of the ones below min_score.
// The serial removal loop (the last live candidate moves into a removed one's slot, which is re-examined) leaves
// the m survivors of (i, live) as: survivors below i + 1 + m in place, and each removed slot below that end filled by
// a survivor from above it, lowest slot first, highest survivor first.  A step is therefore two block scans.
// A selection is final once made and selected scores do not increase, so K selections per problem suffice.
constexpr int SN_THREADS = 1024;
constexpr int SN_MAX_GROUPS = 1024;

struct SoftNmsWs {
  float *x1, *y1, *x2, *y2, *area, *score;   // [B, n] per candidate, segment-local order
  int *orig, *perm, *holes;                  // [B, n] input index, position -> candidate, removed slots
  float* sel_score;                          // [B, n] selections of segment g at seg_off[g]
  int* sel_idx;
  int *seg_off, *seg_cnt, *sel_cnt;          // [B, G]
  float* max_coord;                          // [B]
  int* per_class;                            // [B]
};

inline size_t sn_align(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }

inline SoftNmsWs sn_carve(void* base, int B, int n, int G, size_t* bytes) {
  char* p = static_cast<char*>(base);
  size_t off = 0;
  const size_t bn = static_cast<size_t>(B) * n * 4, bg = static_cast<size_t>(B) * G * 4, b1 = static_cast<size_t>(B) * 4;
  auto take = [&](size_t sz) { char* r = p + off; off += sn_align(sz); return r; };
  SoftNmsWs w;
  w.x1 = reinterpret_cast<float*>(take(bn)); w.y1 = reinterpret_cast<float*>(take(bn));
  w.x2 = reinterpret_cast<float*>(take(bn)); w.y2 = reinterpret_cast<float*>(take(bn));
  w.area = reinterpret_cast<float*>(take(bn)); w.score = reinterpret_cast<float*>(take(bn));
  w.orig = reinterpret_cast<int*>(take(bn)); w.perm = reinterpret_cast<int*>(take(bn));
  w.holes = reinterpret_cast<int*>(take(bn));
  w.sel_score = reinterpret_cast<float*>(take(bn)); w.sel_idx = reinterpret_cast<int*>(take(bn));
  w.seg_off = reinterpret_cast<int*>(take(bg)); w.seg_cnt = reinterpret_cast<int*>(take(bg));
  w.sel_cnt = reinterpret_cast<int*>(take(bg));
  w.max_coord = reinterpret_cast<float*>(take(b1)); w.per_class = reinterpret_cast<int*>(take(b1));
  if (bytes) *bytes = off;
  return w;
}

size_t soft_nms_workspace_bytes(int B, int n, int G) {
  size_t bytes = 0;
  sn_carve(nullptr, B, n, G, &bytes);
  return bytes;
}

// The three comparisons of softnms_cpu, in one place:
//   selection:  the running max is replaced only when  max < sc[pos]   (first position of the largest score wins)
//   decay:      naive / linear act when               ovr >= iou_threshold   (gaussian always)
//   removal:    a candidate is dropped when           sc[pos] < min_score
__device__ __forceinline__ bool sn_removed(float s, float min_score) { return s < min_score; }

__device__ __forceinline__ void sn_better(float& s, int& p, float s2, int p2) {
  if (s2 > s || (s2 == s && p2 < p)) { s = s2; p = p2; }
}

__device__ __forceinline__ float sn_weight(float ovr, float thr, float sigma, int method) {
  if (method == 0) return ovr >= thr ? 0.f : 1.f;
  if (method == 1) return ovr >= thr ? fsub(1.f, ovr) : 1.f;
  const float arg = __fdiv_rn(-fmul(ovr, ovr), sigma);       // -(ovr * ovr) / sigma in fp32
  return __double2float_rn(exp(static_cast<double>(arg)));   // exp in double, rounded once to fp32
}

// block-wide helpers for SN_THREADS threads; each ends with every thread holding the result
__device__ __forceinline__ void sn_block_argmax(float& s, int& p, float* rs, int* rp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const int p2 = __shfl_xor_sync(0xffffffffu, p, o);
    sn_better(s, p, s2, p2);
  }
  __syncthreads();
  if (lane == 0) { rs[warp] = s; rp[warp] = p; }
  __syncthreads();
  s = rs[0]; p = rp[0];
  for (int w = 1; w < SN_THREADS / 32; ++w) sn_better(s, p, rs[w], rp[w]);
}

// exclusive scan of two counters over the block; totals in ta / tb
__device__ __forceinline__ void sn_block_exscan2(int& a, int& b, int& ta, int& tb, int2* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int ia = a, ib = b;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int xa = __shfl_up_sync(0xffffffffu, ia, o), xb = __shfl_up_sync(0xffffffffu, ib, o);
    if (lane >= o) { ia += xa; ib += xb; }
  }
  __syncthreads();
  if (lane == 31) red[warp] = make_int2(ia, ib);
  __syncthreads();
  int pa = 0, pb = 0;
  ta = 0; tb = 0;
  for (int w = 0; w < SN_THREADS / 32; ++w) {
    const int2 v = red[w];
    if (w < warp) { pa += v.x; pb += v.y; }
    ta += v.x; tb += v.y;
  }
  a = pa + ia - a; b = pb + ib - b;
}

// per image: max coordinate of the valid boxes, the regime, and the per-id segments of the workspace
__global__ void __launch_bounds__(SN_THREADS)
soft_nms_prep_kernel(const float* __restrict__ boxes, const long long* __restrict__ ids, const int* __restrict__ nvalid,
                     int n, int G, int split_thr, SoftNmsWs ws) {
  __shared__ float red[SN_THREADS / 32];
  __shared__ int hist[SN_MAX_GROUPS];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int nv = min(max(nvalid[b], 0), n);
  const bool per_class = nv >= split_thr;
  float m = -INFINITY;
  for (int i = tid; i < nv * 4; i += SN_THREADS) m = fmaxf(m, boxes[static_cast<size_t>(b) * n * 4 + i]);
#pragma unroll
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  for (int g = tid; g < G; g += SN_THREADS) hist[g] = 0;
  if ((tid & 31) == 0) red[tid >> 5] = m;
  __syncthreads();
  if (per_class) {
    for (int i = tid; i < nv; i += SN_THREADS) {
      const long long id = ids[static_cast<size_t>(b) * n + i];
      if (id >= 0 && id < G) atomicAdd(&hist[id], 1);
    }
  } else if (tid == 0) {
    hist[0] = nv;
  }
  __syncthreads();
  if (tid == 0) {
    float mm = red[0];
    for (int w = 1; w < SN_THREADS / 32; ++w) mm = fmaxf(mm, red[w]);
    ws.max_coord[b] = mm;
    ws.per_class[b] = per_class ? 1 : 0;
    int off = 0;
    for (int g = 0; g < G; ++g) {
      ws.seg_off[b * G + g] = off;
      ws.seg_cnt[b * G + g] = hist[g];
      off += hist[g];
    }
  }
}

// one CTA per (id group, image): gather the group's candidates in input order, then run the serial loop's steps
__global__ void __launch_bounds__(SN_THREADS)
soft_nms_kernel(const float* __restrict__ boxes, const float* __restrict__ scores, const long long* __restrict__ ids,
                const int* __restrict__ nvalid, int n, int G, float thr, float sigma, float min_score, int method,
                int K, SoftNmsWs ws) {
  __shared__ float rs[SN_THREADS / 32];
  __shared__ int rp[SN_THREADS / 32];
  __shared__ int2 red2[SN_THREADS / 32];
  __shared__ int s_sel;
  const int g = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int cnt = ws.seg_cnt[b * G + g];
  if (cnt == 0) {
    if (tid == 0) ws.sel_cnt[b * G + g] = 0;
    return;
  }
  const size_t base = static_cast<size_t>(b) * n + ws.seg_off[b * G + g];
  float *x1 = ws.x1 + base, *y1 = ws.y1 + base, *x2 = ws.x2 + base, *y2 = ws.y2 + base;
  float *area = ws.area + base, *sc = ws.score + base;
  int *orig = ws.orig + base, *perm = ws.perm + base, *holes = ws.holes + base;
  const int nv = min(max(nvalid[b], 0), n);
  const bool per_class = ws.per_class[b] != 0;
  const float off1 = fadd(ws.max_coord[b], 1.0f);

  // gather (order-preserving compaction of this group's candidates)
  int run = 0;
  for (int j0 = 0; j0 < nv; j0 += SN_THREADS) {
    const int j = j0 + tid;
    const size_t gj = static_cast<size_t>(b) * n + j;
    const bool mine = j < nv && (!per_class || ids[gj] == g);
    int r = mine ? 1 : 0, z = 0, tot, tz;
    sn_block_exscan2(r, z, tot, tz, red2);
    if (mine) {
      const int k = run + r;
      const float off = fmul(static_cast<float>(ids[gj]), off1);
      const float a0 = fadd(boxes[gj * 4], off), a1 = fadd(boxes[gj * 4 + 1], off);
      const float a2 = fadd(boxes[gj * 4 + 2], off), a3 = fadd(boxes[gj * 4 + 3], off);
      x1[k] = a0; y1[k] = a1; x2[k] = a2; y2[k] = a3;
      area[k] = fmul(fsub(a2, a0), fsub(a3, a1));
      sc[k] = scores[gj];
      orig[k] = j;
      perm[k] = k;
    }
    run += tot;
  }
  __syncthreads();

  // first argmax over all positions
  float bs = -INFINITY;
  int bp = INT_MAX;
  for (int q = tid; q < cnt; q += SN_THREADS) sn_better(bs, bp, sc[q], q);
  sn_block_argmax(bs, bp, rs, rp);

  int live = cnt, i = 0;
  for (; i < live && i < K; ++i) {
    if (tid == 0) {
      const int p = isnan(sc[perm[i]]) ? i : bp;
      const int c = perm[p];
      perm[p] = perm[i];
      perm[i] = c;
      ws.sel_score[base + i] = sc[c];
      ws.sel_idx[base + i] = orig[c];
      s_sel = c;
    }
    __syncthreads();
    const int c = s_sel;
    const float ix1 = x1[c], iy1 = y1[c], ix2 = x2[c], iy2 = y2[c], iarea = area[c];
    const int lo0 = i + 1, len = live - lo0;
    if (len <= 0) { ++i; break; }
    const int L = (len + SN_THREADS - 1) / SN_THREADS;
    const int lo = min(lo0 + tid * L, live), hi = min(lo + L, live);
    // decay each of (i, live) once
    int alive = 0, zero = 0;
    for (int q = lo; q < hi; ++q) {
      const int d = perm[q];
      const float w = fmaxf(fsub(fminf(ix2, x2[d]), fmaxf(ix1, x1[d])), 0.f);
      const float h = fmaxf(fsub(fminf(iy2, y2[d]), fmaxf(iy1, y1[d])), 0.f);
      const float inter = fmul(w, h);
      const float ovr = __fdiv_rn(inter, fsub(fadd(iarea, area[d]), inter));
      const float s = fmul(sc[d], sn_weight(ovr, thr, sigma, method));
      sc[d] = s;
      alive += sn_removed(s, min_score) ? 0 : 1;
    }
    int m, unused;
    sn_block_exscan2(alive, zero, m, unused, red2);
    const int end = lo0 + m;
    // removed slots below the new end, survivors at or above it
    int nh = 0, ns = 0;
    for (int q = lo; q < hi; ++q) {
      const bool dead = sn_removed(sc[perm[q]], min_score);
      if (q < end) nh += dead ? 1 : 0;
      else ns += dead ? 0 : 1;
    }
    int th, ts;
    sn_block_exscan2(nh, ns, th, ts, red2);
    bs = -INFINITY; bp = INT_MAX;
    for (int q = lo; q < min(hi, end); ++q) {
      const float s = sc[perm[q]];
      if (sn_removed(s, min_score)) holes[nh++] = q;
      else sn_better(bs, bp, s, q);
    }
    __syncthreads();
    for (int q = max(lo, end); q < hi; ++q) {
      const int d = perm[q];
      const float s = sc[d];
      if (!sn_removed(s, min_score)) {
        const int dst = holes[ts - 1 - ns];   // highest survivor fills the lowest slot
        ++ns;
        perm[dst] = d;
        sn_better(bs, bp, s, dst);
      }
    }
    sn_block_argmax(bs, bp, rs, rp);
    live = end;
  }
  if (tid == 0) ws.sel_cnt[b * G + g] = i;
}

// entries of a non-increasing list before value s: v > s, or v >= s when ties rank first
__device__ __forceinline__ int sn_count_before(const float* v, int len, float s, bool ties_first) {
  int lo = 0, hi = len;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const float x = v[mid];
    if (ties_first ? x >= s : x > s) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// selections -> [B, K] outputs: entry k of group g goes to rank k + (entries of the other groups ranked before it);
// in the per-id regime that is a merge by decayed score (ties: lower id first), otherwise the selection order.
__global__ void soft_nms_finish_kernel(const float* __restrict__ boxes, const long long* __restrict__ ids, int n,
                                       int G, int K, SoftNmsWs ws, float* __restrict__ out_boxes,
                                       float* __restrict__ out_scores, long long* __restrict__ out_labels,
                                       int* __restrict__ out_index, int* __restrict__ counts) {
  const int b = blockIdx.y;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int* soff = ws.seg_off + b * G;
  const int* scnt = ws.seg_cnt + b * G;
  const int* selc = ws.sel_cnt + b * G;
  int total = 0;
  for (int h = 0; h < G; ++h) total += selc[h];
  const int kout = min(total, K);
  if (e < n) {
    int g = -1;
    for (int h = 0; h < G; ++h)
      if (scnt[h] > 0 && e >= soff[h] && e < soff[h] + scnt[h]) { g = h; break; }
    const int k = g >= 0 ? e - soff[g] : 0;
    if (g >= 0 && k < selc[g]) {
      const float* sel = ws.sel_score + static_cast<size_t>(b) * n;
      const float s = sel[e];
      int rank = k;
      for (int h = 0; h < G && rank < K; ++h)
        if (h != g && selc[h] > 0) rank += sn_count_before(sel + soff[h], selc[h], s, h < g);
      if (rank < K) {
        const int j = ws.sel_idx[static_cast<size_t>(b) * n + e];
        const size_t src = static_cast<size_t>(b) * n + j, dst = static_cast<size_t>(b) * K + rank;
#pragma unroll
        for (int c = 0; c < 4; ++c) out_boxes[dst * 4 + c] = boxes[src * 4 + c];
        out_scores[dst] = s;
        if (out_labels) out_labels[dst] = ids[src];
        if (out_index) out_index[dst] = j;
      }
    }
  }
  if (e >= kout && e < K) {
    const size_t dst = static_cast<size_t>(b) * K + e;
#pragma unroll
    for (int c = 0; c < 4; ++c) out_boxes[dst * 4 + c] = 0.f;
    out_scores[dst] = 0.f;
    if (out_labels) out_labels[dst] = 0;
    if (out_index) out_index[dst] = -1;
  }
  if (e == 0) counts[b] = kout;
}

int soft_nms_batched(const float* boxes, const float* scores, const long long* ids, const int* nvalid, int B, int n,
                     int G, float iou_thr, float sigma, float min_score, int method, int split_thr, int K, void* ws,
                     size_t ws_bytes, float* out_boxes, float* out_scores, long long* out_labels, int* out_index,
                     int* counts, cudaStream_t stream) {
  RSP_CHECK_ARG(boxes && scores && ids && nvalid && ws && out_boxes && out_scores && counts && B > 0 && B <= 65535 &&
                n > 0 && K > 0, "soft_nms_batched: bad args");
  RSP_CHECK_ARG(G >= 1 && G <= SN_MAX_GROUPS, "soft_nms_batched: 1 <= G <= %d id groups", SN_MAX_GROUPS);
  RSP_CHECK_ARG(method >= 0 && method <= 2, "soft_nms_batched: method 0 naive, 1 linear, 2 gaussian");
  RSP_CHECK_ARG(method != 2 || sigma > 0.f, "soft_nms_batched: gaussian needs sigma > 0");
  RSP_CHECK_ARG(static_cast<long long>(B) * n <= 0x7fffffffLL, "soft_nms_batched: B * n must fit in int32");
  size_t need = 0;
  SoftNmsWs w = sn_carve(ws, B, n, G, &need);
  RSP_CHECK_ARG(ws_bytes >= need, "soft_nms_batched: workspace of %zu bytes, %zu needed", ws_bytes, need);
  soft_nms_prep_kernel<<<B, SN_THREADS, 0, stream>>>(boxes, ids, nvalid, n, G, split_thr, w);
  RSP_CHECK_LAUNCH();
  soft_nms_kernel<<<dim3(G, B), SN_THREADS, 0, stream>>>(boxes, scores, ids, nvalid, n, G, iou_thr, sigma, min_score,
                                                         method, K, w);
  RSP_CHECK_LAUNCH();
  const int span = max(n, K);
  soft_nms_finish_kernel<<<dim3((span + 255) / 256, B), 256, 0, stream>>>(boxes, ids, n, G, K, w, out_boxes,
                                                                          out_scores, out_labels, out_index, counts);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
struct RoiLevels {
  const __nv_bfloat16* feat[4];
  const float* pe[4];   // fp32 [H, W, C] per level or null
  int H[4], W[4];
  float scale[4];
};

__device__ __forceinline__ void bilinear_setup(float y, float x, int H, int W, int& y0, int& x0, int& y1,
                                               int& x1, float& w00, float& w01, float& w10, float& w11,
                                               bool& inside) {
  inside = !(y < -1.0f || y > H || x < -1.0f || x > W);
  if (y <= 0.f) y = 0.f;
  if (x <= 0.f) x = 0.f;
  y0 = static_cast<int>(y); x0 = static_cast<int>(x);
  if (y0 >= H - 1) { y1 = y0 = H - 1; y = static_cast<float>(y0); } else { y1 = y0 + 1; }
  if (x0 >= W - 1) { x1 = x0 = W - 1; x = static_cast<float>(x0); } else { x1 = x0 + 1; }
  const float ly = y - y0, lx = x - x0, hy = 1.f - ly, hx = 1.f - lx;
  w00 = hy * hx; w01 = hy * lx; w10 = ly * hx; w11 = ly * lx;
}

// thread = 8 channels of one (roi, bin); out bf16 [n, P*P*C] in (ph, pw, c) order
__global__ void roi_align_nhwc_kernel(RoiLevels lv, const float* __restrict__ rois, int n, int C, int P,
                                      int num_levels, float finest_scale, __nv_bfloat16* __restrict__ out) {
  const int c8 = C / 8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(n) * P * P * c8;
  if (idx >= total) return;
  const int cc = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int pw = static_cast<int>(t % P); t /= P;
  const int ph = static_cast<int>(t % P);
  const int r = static_cast<int>(t / P);
  const float* roi = rois + static_cast<size_t>(r) * 5;
  const int b = static_cast<int>(roi[0]);
  // map_roi_levels: floor(log2(sqrt(w*h) / finest + 1e-6)) clamped
  const float sc = sqrtf((roi[3] - roi[1]) * (roi[4] - roi[2]));
  int l = static_cast<int>(floorf(log2f(sc / finest_scale + 1e-6f)));
  l = max(0, min(num_levels - 1, l));
  const int H = lv.H[l], W = lv.W[l];
  const float ss = lv.scale[l];
  const float x1 = roi[1] * ss - 0.5f, y1 = roi[2] * ss - 0.5f;
  const float rw = roi[3] * ss - 0.5f - x1, rh = roi[4] * ss - 0.5f - y1;
  const float bw = rw / P, bh = rh / P;
  const int gh = static_cast<int>(ceilf(rh / P)), gw = static_cast<int>(ceilf(rw / P));  // may be 0 (degenerate roi)
  const float cnt = static_cast<float>(max(gh * gw, 1));
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
  const __nv_bfloat16* fb = lv.feat[l] + static_cast<size_t>(b) * H * W * C + cc * 8;
  const float* pb = lv.pe[l] ? lv.pe[l] + cc * 8 : nullptr;
  for (int iy = 0; iy < gh; ++iy) {
    const float y = y1 + ph * bh + (iy + 0.5f) * bh / gh;
    for (int ix = 0; ix < gw; ++ix) {
      const float x = x1 + pw * bw + (ix + 0.5f) * bw / gw;
      int y0, x0, yy1, xx1;
      float w00, w01, w10, w11;
      bool inside;
      bilinear_setup(y, x, H, W, y0, x0, yy1, xx1, w00, w01, w10, w11, inside);
      if (!inside) continue;
      const size_t o00 = (static_cast<size_t>(y0) * W + x0) * C, o01 = (static_cast<size_t>(y0) * W + xx1) * C;
      const size_t o10 = (static_cast<size_t>(yy1) * W + x0) * C, o11 = (static_cast<size_t>(yy1) * W + xx1) * C;
      const uint4 u00 = *reinterpret_cast<const uint4*>(fb + o00), u01 = *reinterpret_cast<const uint4*>(fb + o01);
      const uint4 u10 = *reinterpret_cast<const uint4*>(fb + o10), u11 = *reinterpret_cast<const uint4*>(fb + o11);
      const uint32_t a00[4] = {u00.x, u00.y, u00.z, u00.w}, a01[4] = {u01.x, u01.y, u01.z, u01.w};
      const uint32_t a10[4] = {u10.x, u10.y, u10.z, u10.w}, a11[4] = {u11.x, u11.y, u11.z, u11.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const __nv_bfloat162 h00 = *reinterpret_cast<const __nv_bfloat162*>(&a00[j]);
        const __nv_bfloat162 h01 = *reinterpret_cast<const __nv_bfloat162*>(&a01[j]);
        const __nv_bfloat162 h10 = *reinterpret_cast<const __nv_bfloat162*>(&a10[j]);
        const __nv_bfloat162 h11 = *reinterpret_cast<const __nv_bfloat162*>(&a11[j]);
        acc[2 * j] += w00 * __bfloat162float(h00.x) + w01 * __bfloat162float(h01.x) +
                      w10 * __bfloat162float(h10.x) + w11 * __bfloat162float(h11.x);
        acc[2 * j + 1] += w00 * __bfloat162float(h00.y) + w01 * __bfloat162float(h01.y) +
                          w10 * __bfloat162float(h10.y) + w11 * __bfloat162float(h11.y);
      }
      if (pb) {
#pragma unroll
        for (int k = 0; k < 8; ++k)
          acc[k] += w00 * pb[o00 + k] + w01 * pb[o01 + k] + w10 * pb[o10 + k] + w11 * pb[o11 + k];
      }
    }
  }
  const float inv = 1.0f / cnt;
  __nv_bfloat16* o = out + (static_cast<size_t>(r) * P * P + ph * P + pw) * C + cc * 8;
  *reinterpret_cast<uint4*>(o) =
      make_uint4(pack_bf16x2(acc[0] * inv, acc[1] * inv), pack_bf16x2(acc[2] * inv, acc[3] * inv),
                 pack_bf16x2(acc[4] * inv, acc[5] * inv), pack_bf16x2(acc[6] * inv, acc[7] * inv));
}

int roi_align_nhwc(const void* const* feats, const float* const* pes, const int* Hs, const int* Ws,
                   const float* scales, int num_levels, const float* rois, int n, int C, int P,
                   float finest_scale, void* out, cudaStream_t stream) {
  RSP_CHECK_ARG(feats && Hs && Ws && scales && rois && out && n > 0 && C % 8 == 0 && num_levels >= 1 &&
                num_levels <= 4, "roi_align: bad args");
  RoiLevels lv;
  for (int i = 0; i < 4; ++i) {
    const int j = i < num_levels ? i : num_levels - 1;
    lv.feat[i] = static_cast<const __nv_bfloat16*>(feats[j]);
    lv.pe[i] = pes ? pes[j] : nullptr;
    lv.H[i] = Hs[j]; lv.W[i] = Ws[j]; lv.scale[i] = scales[j];
  }
  const long long total = static_cast<long long>(n) * P * P * (C / 8);
  roi_align_nhwc_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      lv, rois, n, C, P, num_levels, finest_scale, static_cast<__nv_bfloat16*>(out));
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// Mask paste: low-resolution maps [n, hm, wm] -> thresholded masks, bytes or bits.  Two kernel families: the x4 tile
// kernel below for the mask decoder's image / 4 logits, and mask_paste_px_kernel, which takes each pixel's value from
// a sampler (OneResize, TwoResizes, BoxSample).  MODE 1: v > thr; 0 and 2: v >= thr (mode 0 is OneResize<true>, which
// activates the taps; mode 2 takes maps that rsp_sigmoid_f32 activated once).

// x4 fast path (the mask decoder's logits are always image / 4): thread = 4 output rows x 16 columns
// PACKED: out holds W/8 bytes per row, pixel x = bit x%8 of byte x/8 (the result-record payload)
template <int MODE, bool PACKED>
__global__ void mask_paste_x4_kernel(const float* __restrict__ logits, unsigned char* __restrict__ out, int n, int hm,
                                     int wm, float thr) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int w4 = wm / 4;
  if (idx >= static_cast<long long>(n) * hm * w4) return;
  const int xb = static_cast<int>(idx % w4);
  long long t = idx / w4;
  const int yb = static_cast<int>(t % hm);
  const int m = static_cast<int>(t / hm);
  Up4Tile tile;
  up4_load(logits + static_cast<size_t>(m) * hm * wm, hm, wm, yb, xb, tile);
  const int W = 4 * wm;
  const int ldm = PACKED ? W / 8 : W;
  unsigned char* o = out + (static_cast<size_t>(m) * 4 * hm + 4 * yb) * ldm + (PACKED ? 2 : 16) * xb;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint32_t packed[4] = {0u, 0u, 0u, 0u};
    uint32_t bits = 0u;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float v = up4_value(tile, j, k);
      const uint32_t bit = (MODE == 1 ? (v > thr) : (v >= thr)) ? 1u : 0u;
      if (PACKED) bits |= bit << k;
      else packed[k >> 2] |= bit << ((k & 3) * 8);
    }
    if (PACKED) *reinterpret_cast<uint16_t*>(o + static_cast<size_t>(j) * ldm) = static_cast<uint16_t>(bits);
    else *reinterpret_cast<uint4*>(o + static_cast<size_t>(j) * W) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
  }
}

// FCNMaskHead paste (fcn_mask_head.py:_do_paste_mask + the threshold of _predict_by_feat_single :388-392): the
// activated RoI mask probs fp32 [n, hm, wm] of detection m are sampled bilinearly (F.grid_sample, align_corners=False,
// zero padding) at every image pixel centre mapped into its box, in the reference's rounding order.  row() reports
// rows whose taps all fall outside the RoI grid.
struct BoxSample {
  const float* probs;
  const float* boxes;
  int hm, wm;
  const float* p;
  float bx0, bx1, iy, fy;
  int yi0, yi1;
  bool vy0, vy1;

  __device__ __forceinline__ bool row(int m, int y) {
    const float by0 = boxes[m * 4 + 1], by1 = boxes[m * 4 + 3];
    bx0 = boxes[m * 4];
    bx1 = boxes[m * 4 + 2];
    // normalised grid coordinate in [-1, 1] (inf from a degenerate box becomes 0, as the reference does)
    float gy = __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn(y + 0.5f, by0), __fsub_rn(by1, by0)), 2.f), 1.f);
    if (isinf(gy)) gy = 0.f;
    iy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), static_cast<float>(hm)), 1.f), 0.5f);
    fy = floorf(iy);
    yi0 = static_cast<int>(fy);
    yi1 = yi0 + 1;
    vy0 = yi0 >= 0 && yi0 < hm;
    vy1 = yi1 >= 0 && yi1 < hm;
    p = probs + static_cast<size_t>(m) * hm * wm;
    return vy0 || vy1;
  }

  __device__ __forceinline__ float at(int x) const {
    float gx = __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn(x + 0.5f, bx0), __fsub_rn(bx1, bx0)), 2.f), 1.f);
    if (isinf(gx)) gx = 0.f;
    const float ix = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), static_cast<float>(wm)), 1.f), 0.5f);
    const float fx = floorf(ix);
    const int xi0 = static_cast<int>(fx), xi1 = xi0 + 1;
    const bool vx0 = xi0 >= 0 && xi0 < wm, vx1 = xi1 >= 0 && xi1 < wm;
    const float v00 = (vy0 && vx0) ? __ldg(p + yi0 * wm + xi0) : 0.f, v01 = (vy0 && vx1) ? __ldg(p + yi0 * wm + xi1) : 0.f;
    const float v10 = (vy1 && vx0) ? __ldg(p + yi1 * wm + xi0) : 0.f, v11 = (vy1 && vx1) ? __ldg(p + yi1 * wm + xi1) : 0.f;
    // grid_sample weights in ATen's form: (x_se - ix)(y_se - iy), (ix - x_nw)(y_se - iy), (x_se - ix)(iy - y_nw), ...
    const float wx0 = (fx + 1.f) - ix, wx1 = ix - fx, wy0 = (fy + 1.f) - iy, wy1 = iy - fy;
    return v00 * (wx0 * wy0) + v01 * (wx1 * wy0) + v10 * (wx0 * wy1) + v11 * (wx1 * wy1);
  }
};

// thread = 16 consecutive pixels of one output row.  BITS: record slots [n, Hr, Wr/8] (Wr % 16 == 0), pixel x = bit
// x % 8 of byte x / 8, one uint16 per thread, the (H, W) mask at the slot's top-left and 0 elsewhere.  Otherwise bytes
// [n, H, W] (Hr = H, Wr = W): one 16-byte store where the row segment is whole and 16-byte aligned, byte stores
// elsewhere.  Rows the sampler reports empty store zeros without loads.
template <class Sampler, int MODE, bool BITS>
__global__ void mask_paste_px_kernel(Sampler s, unsigned char* __restrict__ out, int n, int H, int W, int Hr, int Wr,
                                     float thr) {
  const int w16 = (Wr + 15) / 16;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(n) * Hr * w16) return;
  const int xb = static_cast<int>(idx % w16);
  const long long t = idx / w16;
  const int y = static_cast<int>(t % Hr);
  const int m = static_cast<int>(t / Hr);
  uint32_t packed[4] = {0u, 0u, 0u, 0u};
  uint32_t bits = 0u;
  if (y < H && s.row(m, y)) {
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int x = 16 * xb + k;
      if (x >= W) break;
      const float v = s.at(x);
      const uint32_t bit = (MODE == 1 ? (v > thr) : (v >= thr)) ? 1u : 0u;
      if (BITS) bits |= bit << k;
      else packed[k >> 2] |= bit << ((k & 3) * 8);
    }
  }
  if (BITS) {
    *reinterpret_cast<uint16_t*>(out + (static_cast<size_t>(m) * Hr + y) * (Wr / 8) + 2 * xb) = static_cast<uint16_t>(bits);
    return;
  }
  unsigned char* dst = out + (static_cast<size_t>(m) * H + y) * W + 16 * xb;
  if (16 * xb + 16 <= W && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    *reinterpret_cast<uint4*>(dst) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
  } else {
    for (int k = 0; k < 16 && 16 * xb + k < W; ++k) dst[k] = static_cast<unsigned char>((packed[k >> 2] >> ((k & 3) * 8)) & 1u);
  }
}

template <int MODE, bool BITS, class Sampler>
static int paste_px(const Sampler& s, unsigned char* out, int n, int H, int W, int Hr, int Wr, float thr,
                    cudaStream_t stream) {
  const long long total = static_cast<long long>(n) * Hr * ((Wr + 15) / 16);
  mask_paste_px_kernel<Sampler, MODE, BITS><<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      s, out, n, H, W, Hr, Wr, thr);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// MODE 1 for mode 1, MODE 2 otherwise
template <bool BITS, class Sampler>
static int paste_px12(const Sampler& s, unsigned char* out, int n, int H, int W, int Hr, int Wr, float thr, int mode,
                      cudaStream_t stream) {
  return mode == 1 ? paste_px<1, BITS>(s, out, n, H, W, Hr, Wr, thr, stream)
                   : paste_px<2, BITS>(s, out, n, H, W, Hr, Wr, thr, stream);
}

int mask_paste(const float* maps, unsigned char* out, int n, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w,
               int H, int W, int Hr, int Wr, int packed, float thr, int mode, cudaStream_t stream) {
  RSP_CHECK_ARG(maps && out && n > 0 &&
                (packed ? H <= Hr && W <= Wr && Wr % 16 == 0 && (reinterpret_cast<uintptr_t>(out) & 1) == 0
                        : Hr == H && Wr == W),
                "mask_paste: bad output (bytes: (Hr, Wr) = (H, W); bits: H <= Hr, W <= Wr, Wr % 16 == 0, 2-byte aligned)");
  if (Hb == 0) {   // one resize (hm, wm) -> (H, W)
    const bool x4 = H == 4 * hm && W == 4 * wm && wm % 4 == 0 && (reinterpret_cast<uintptr_t>(maps) & 15) == 0;
    RSP_CHECK_ARG(packed ? x4 && Hr == H && Wr == W && (mode == 1 || mode == 2) : W % 16 == 0,
                  "mask_paste: one resize needs W % 16 == 0; bit-packed, the x4 path only ((H, W) = (4hm, 4wm) = "
                  "(Hr, Wr), wm % 4 == 0, 16-byte aligned maps; mode 1: > thr on raw maps, 2: >= thr on activated maps)");
    if (x4 && mode != 0) {
      const long long tiles = static_cast<long long>(n) * hm * (wm / 4);
      const unsigned blocks = static_cast<unsigned>((tiles + 127) / 128);
      if (packed) {
        if (mode == 1) mask_paste_x4_kernel<1, true><<<blocks, 128, 0, stream>>>(maps, out, n, hm, wm, thr);
        else mask_paste_x4_kernel<2, true><<<blocks, 128, 0, stream>>>(maps, out, n, hm, wm, thr);
      } else {
        if (mode == 1) mask_paste_x4_kernel<1, false><<<blocks, 128, 0, stream>>>(maps, out, n, hm, wm, thr);
        else mask_paste_x4_kernel<2, false><<<blocks, 128, 0, stream>>>(maps, out, n, hm, wm, thr);
      }
      RSP_CHECK_LAUNCH();
      return RSP_OK;
    }
    if (mode == 0) return paste_px<0, false>(OneResize<true, false>{maps, hm, wm, H, W}, out, n, H, W, H, W, thr, stream);
    return paste_px12<false>(OneResize<false, false>{maps, hm, wm, H, W}, out, n, H, W, H, W, thr, mode, stream);
  }
  RSP_CHECK_ARG(hm > 0 && wm > 0 && Hb > 0 && Wb > 0 && crop_h > 0 && crop_w > 0 && crop_h <= Hb && crop_w <= Wb &&
                H > 0 && W > 0 && (mode == 1 || mode == 2),
                "mask_paste: bad args for two resizes (crop within (Hb, Wb); mode 1: > thr on raw maps, 2: >= thr on "
                "activated maps)");
  const TwoResizes s{maps, {hm, wm, Hb, Wb, crop_h, crop_w, H, W}};
  return packed ? paste_px12<true>(s, out, n, H, W, Hr, Wr, thr, mode, stream)
                : paste_px12<false>(s, out, n, H, W, H, W, thr, mode, stream);
}

int mask_paste_boxes(const float* probs, const float* boxes, unsigned char* out, int n, int hm, int wm, int H, int W,
                     float thr, int packed, cudaStream_t stream) {
  RSP_CHECK_ARG(probs && boxes && out && n > 0 && hm > 0 && wm > 0 && H > 0 && W > 0, "mask_paste_boxes: bad arguments");
  RSP_CHECK_ARG(!packed || W % 16 == 0, "mask_paste_boxes: bit-packed output needs W % 16 == 0");
  const BoxSample s{probs, boxes, hm, wm};
  return packed ? paste_px<2, true>(s, out, n, H, W, H, W, thr, stream)
                : paste_px<2, false>(s, out, n, H, W, H, W, thr, stream);
}

// ---------------------------------------------------------------------------------------
// SAM automatic mask generation, per candidate mask (HF SamImageProcessor.post_process_masks(binarize=False) followed
// by filter_masks' _compute_stability_score, > mask_threshold and _batched_mask_to_box): every pixel of the original-size
// mask comes from the TwoResizes sampler of mask_paste's two resizes, so its > thr decision is that kernel's bit, and
// only integers leave a block.  Block m * bands + band covers rows [band * SMS_ROWS, +SMS_ROWS) of mask m (the bands of
// a mask are consecutive blocks, so its low-res map is read while it is in L2); thread = 16 consecutive pixels of a
// row, as in mask_paste_px_kernel.  part: int32 [n, bands, 7] = (count > thr_hi,
// count > thr_lo, count > thr, x_min, y_min, x_max, y_max of > thr).
constexpr int SMS_ROWS = 16;
constexpr int SMS_THREADS = 256;
constexpr int SMS_FIELDS = 7;

__global__ void __launch_bounds__(SMS_THREADS, 4)   // 64 registers: 4 blocks per SM
sam_mask_stats_kernel(TwoResizes s, int H, int W, float thr, float thr_hi, float thr_lo, int bands,
                      int* __restrict__ part) {
  const int band = static_cast<int>(blockIdx.x % bands), m = static_cast<int>(blockIdx.x / bands);
  const int y0 = band * SMS_ROWS;
  const int rows = min(SMS_ROWS, H - y0);
  const int w16 = (W + 15) / 16;
  int n_hi = 0, n_lo = 0, n_mid = 0;
  int x_min = INT_MAX, y_min = INT_MAX, x_max = -1, y_max = -1;
  for (int it = threadIdx.x; it < rows * w16; it += SMS_THREADS) {
    const int y = y0 + it / w16, x0 = 16 * (it % w16);
    s.row(m, y);
    uint32_t bits = 0u;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int x = x0 + k;
      if (x >= W) break;
      const float v = s.at(x);
      n_hi += v > thr_hi;
      n_lo += v > thr_lo;
      if (v > thr) bits |= 1u << k;
    }
    if (bits) {
      n_mid += __popc(bits);
      x_min = min(x_min, x0 + __ffs(bits) - 1);
      x_max = max(x_max, x0 + 31 - __clz(bits));
      y_min = min(y_min, y);
      y_max = max(y_max, y);
    }
  }
  const unsigned all = 0xffffffffu;
  int v[SMS_FIELDS] = {__reduce_add_sync(all, n_hi), __reduce_add_sync(all, n_lo), __reduce_add_sync(all, n_mid),
                       __reduce_min_sync(all, x_min), __reduce_min_sync(all, y_min), __reduce_max_sync(all, x_max),
                       __reduce_max_sync(all, y_max)};
  __shared__ int red[SMS_THREADS / 32][SMS_FIELDS];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (lane == 0) {
#pragma unroll
    for (int f = 0; f < SMS_FIELDS; ++f) red[warp][f] = v[f];
  }
  __syncthreads();
  if (threadIdx.x < SMS_FIELDS) {
    const int f = threadIdx.x;
    int r = red[0][f];
    for (int w = 1; w < SMS_THREADS / 32; ++w) {
      const int o = red[w][f];
      r = f < 3 ? r + o : f < 5 ? min(r, o) : max(r, o);
    }
    part[(static_cast<size_t>(m) * bands + band) * SMS_FIELDS + f] = r;
  }
}

// The crop-edge rule of HF's filter_masks (image_processing_sam.py _is_box_near_crop_edge with atol 20, rtol 0): a
// mask's box, shifted by the crop's origin into the scene, is dropped when a side lies within 20 of the crop box's side
// and not within 20 of the scene's, in the fp32 arithmetic torch.isclose runs on (box + offset).float().
struct CropEdge {
  int x0, y0, x1, y1;   // the crop box in scene pixels, xyxy
  int H, W;             // the scene
};

__device__ __forceinline__ bool near_crop_edge(const int* box, const CropEdge& c) {
  const int off[4] = {c.x0, c.y0, c.x0, c.y0};
  const int crop[4] = {c.x0, c.y0, c.x1, c.y1};
  const int scene[4] = {0, 0, c.W, c.H};
  bool near = false;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float b = __int2float_rn(box[k] + off[k]);
    near = near || (fabsf(__fsub_rn(b, __int2float_rn(crop[k]))) <= 20.f &&
                    !(fabsf(__fsub_rn(b, __int2float_rn(scene[k]))) <= 20.f));
  }
  return near;
}

// one warp per mask: the band partials -> counts, the HF box ([0, 0, 0, 0] when nothing is > thr), the stability score
// (count > thr_hi) / (count > thr_lo) as torch's int32 / int32 true division (NaN for 0 / 0) and, with iou, the keep
// flag of filter_masks (a threshold > 0 enables its test; NaN fails every test).  kCrop adds the crop-edge rule to the
// keep flag.
template <bool kCrop>
__device__ __forceinline__ void sam_mask_stats_finish(const int* __restrict__ part, int n, int bands,
                                                      const float* __restrict__ iou, float pred_iou_thresh,
                                                      float stability_thresh, int* __restrict__ counts,
                                                      int* __restrict__ boxes, float* __restrict__ stability,
                                                      unsigned char* __restrict__ keep, const CropEdge& crop) {
  const int m = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (m >= n) return;
  int v[SMS_FIELDS] = {0, 0, 0, INT_MAX, INT_MAX, -1, -1};
  for (int b = lane; b < bands; b += 32) {
    const int* p = part + (static_cast<size_t>(m) * bands + b) * SMS_FIELDS;
#pragma unroll
    for (int f = 0; f < SMS_FIELDS; ++f) v[f] = f < 3 ? v[f] + p[f] : f < 5 ? min(v[f], p[f]) : max(v[f], p[f]);
  }
  const unsigned all = 0xffffffffu;
#pragma unroll
  for (int f = 0; f < SMS_FIELDS; ++f)
    v[f] = f < 3 ? __reduce_add_sync(all, v[f]) : f < 5 ? __reduce_min_sync(all, v[f]) : __reduce_max_sync(all, v[f]);
  if (lane != 0) return;
#pragma unroll
  for (int f = 0; f < 3; ++f) counts[m * 3 + f] = v[f];
  const bool empty = v[2] == 0;
  int box[4];
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    box[f] = empty ? 0 : v[3 + f];
    boxes[m * 4 + f] = box[f];
  }
  const float st = __fdiv_rn(__int2float_rn(v[0]), __int2float_rn(v[1]));
  stability[m] = st;
  if (iou != nullptr) {
    bool k = true;
    if (pred_iou_thresh > 0.f) k = k && iou[m] > pred_iou_thresh;
    if (stability_thresh > 0.f) k = k && st > stability_thresh;
    if (kCrop) k = k && !near_crop_edge(box, crop);
    keep[m] = k ? 1 : 0;
  }
}

__global__ void sam_mask_stats_finish_kernel(const int* __restrict__ part, int n, int bands,
                                             const float* __restrict__ iou, float pred_iou_thresh,
                                             float stability_thresh, int* __restrict__ counts, int* __restrict__ boxes,
                                             float* __restrict__ stability, unsigned char* __restrict__ keep) {
  sam_mask_stats_finish<false>(part, n, bands, iou, pred_iou_thresh, stability_thresh, counts, boxes, stability, keep,
                               CropEdge{});
}

__global__ void crop_mask_stats_finish_kernel(const int* __restrict__ part, int n, int bands,
                                              const float* __restrict__ iou, float pred_iou_thresh,
                                              float stability_thresh, int* __restrict__ counts,
                                              int* __restrict__ boxes, float* __restrict__ stability,
                                              unsigned char* __restrict__ keep, CropEdge crop) {
  sam_mask_stats_finish<true>(part, n, bands, iou, pred_iou_thresh, stability_thresh, counts, boxes, stability, keep,
                              crop);
}

int sam_mask_stats(const float* maps, int n, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w, int H, int W,
                   float thr, float thr_hi, float thr_lo, const float* iou, float pred_iou_thresh,
                   float stability_thresh, int crop_x0, int crop_y0, int crop_x1, int crop_y1, int scene_h,
                   int scene_w, int* part_ws, int* counts, int* boxes, float* stability, unsigned char* keep,
                   cudaStream_t stream) {
  const int bands = (H + SMS_ROWS - 1) / SMS_ROWS;
  const bool crop = scene_h != 0;
  RSP_CHECK_ARG(!crop || (iou && crop_x0 >= 0 && crop_y0 >= 0 && crop_x1 > crop_x0 && crop_y1 > crop_y0 &&
                          crop_x1 <= scene_w && crop_y1 <= scene_h && crop_x1 - crop_x0 == W && crop_y1 - crop_y0 == H),
                "sam_mask_stats: bad crop-edge args (iou needed; the crop box is the H x W mask's place in the scene)");
  RSP_CHECK_ARG(maps && part_ws && counts && boxes && stability && (!iou || keep) && n > 0 && hm > 0 && wm > 0 &&
                Hb > 0 && Wb > 0 && crop_h > 0 && crop_w > 0 && crop_h <= Hb && crop_w <= Wb && H > 0 && W > 0 &&
                static_cast<long long>(H) * W <= INT_MAX && static_cast<long long>(n) * bands <= INT_MAX,
                "sam_mask_stats: bad args (n > 0, crop within (Hb, Wb), H * W < 2^31, n * ceil(H / 16) < 2^31)");
  const TwoResizes s{maps, {hm, wm, Hb, Wb, crop_h, crop_w, H, W}};
  sam_mask_stats_kernel<<<static_cast<unsigned>(n) * bands, SMS_THREADS, 0, stream>>>(s, H, W, thr, thr_hi, thr_lo,
                                                                                     bands, part_ws);
  RSP_CHECK_LAUNCH();
  if (crop)
    crop_mask_stats_finish_kernel<<<(n + 7) / 8, 256, 0, stream>>>(
        part_ws, n, bands, iou, pred_iou_thresh, stability_thresh, counts, boxes, stability, keep,
        CropEdge{crop_x0, crop_y0, crop_x1, crop_y1, scene_h, scene_w});
  else
    sam_mask_stats_finish_kernel<<<(n + 7) / 8, 256, 0, stream>>>(part_ws, n, bands, iou, pred_iou_thresh,
                                                                   stability_thresh, counts, boxes, stability, keep);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

__global__ void sigmoid_f32_kernel(const float4* __restrict__ in, float4* __restrict__ out, long long n4) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 x = in[i];
  out[i] = make_float4(1.f / (1.f + expf(-x.x)), 1.f / (1.f + expf(-x.y)), 1.f / (1.f + expf(-x.z)),
                       1.f / (1.f + expf(-x.w)));
}

int sigmoid_f32(const float* in, float* out, long long n, cudaStream_t stream) {
  RSP_CHECK_ARG(in && out && n > 0 && n % 4 == 0, "sigmoid: n must be a positive multiple of 4");
  sigmoid_f32_kernel<<<static_cast<unsigned>((n / 4 + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const float4*>(in), reinterpret_cast<float4*>(out), n / 4);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// mode 0: 2x2 max pool stride 2; mode 1: stride-2 subsample (max_pool2d(k=1, s=2)).  bf16 NHWC.
__global__ void pool2_nhwc_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int B,
                                  int H, int W, int C, int mode) {
  const int Ho = mode == 0 ? H / 2 : (H + 1) / 2, Wo = mode == 0 ? W / 2 : (W + 1) / 2;
  const int c8 = C / 8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(B) * Ho * Wo * c8) return;
  const int cc = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int x = static_cast<int>(t % Wo); t /= Wo;
  const int y = static_cast<int>(t % Ho);
  const int b = static_cast<int>(t / Ho);
  const __nv_bfloat16* p = in + ((static_cast<size_t>(b) * H + 2 * y) * W + 2 * x) * C + cc * 8;
  uint4 v = *reinterpret_cast<const uint4*>(p);
  if (mode == 0) {
    const uint4 o[3] = {*reinterpret_cast<const uint4*>(p + C), *reinterpret_cast<const uint4*>(p + static_cast<size_t>(W) * C),
                        *reinterpret_cast<const uint4*>(p + static_cast<size_t>(W) * C + C)};
    __nv_bfloat162* a = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const __nv_bfloat162* bb = reinterpret_cast<const __nv_bfloat162*>(&o[k]);
#pragma unroll
      for (int j = 0; j < 4; ++j) a[j] = __hmax2(a[j], bb[j]);
    }
  }
  *reinterpret_cast<uint4*>(out + ((static_cast<size_t>(b) * Ho + y) * Wo + x) * C + cc * 8) = v;
}

int pool2_nhwc(const void* in, void* out, int B, int H, int W, int C, int mode, cudaStream_t stream) {
  RSP_CHECK_ARG(in && out && B > 0 && C % 8 == 0 && (mode == 0 || mode == 1), "pool2: bad args");
  const int Ho = mode == 0 ? H / 2 : (H + 1) / 2, Wo = mode == 0 ? W / 2 : (W + 1) / 2;
  const long long total = static_cast<long long>(B) * Ho * Wo * (C / 8);
  pool2_nhwc_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(in), static_cast<__nv_bfloat16*>(out), B, H, W, C, mode);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// Zero the 1-pixel border of bf16 NHWC maps in place.  FCNMaskHead runs its 3x3 convolutions on 14x14 RoI maps embedded
// in 16x16 canvases (128-pixel GEMM tiles are then boxes of the map, so the implicit-GEMM conv applies and no im2col
// matrix is built): the border must read as the convolution's zero padding again after every layer.
__global__ void zero_border_nhwc_kernel(__nv_bfloat16* __restrict__ x, int N, int H, int W, int C) {
  const int c8 = C / 8, ring = 2 * W + 2 * (H - 2);
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(N) * ring * c8) return;
  const int tc = static_cast<int>(idx % c8);
  const long long t = idx / c8;
  const int r = static_cast<int>(t % ring), n = static_cast<int>(t / ring);
  int y, xx;
  if (r < W) { y = 0; xx = r; }
  else if (r < 2 * W) { y = H - 1; xx = r - W; }
  else { const int k = r - 2 * W; y = 1 + (k >> 1); xx = (k & 1) ? W - 1 : 0; }
  *reinterpret_cast<uint4*>(x + ((static_cast<size_t>(n) * H + y) * W + xx) * C + tc * 8) = make_uint4(0u, 0u, 0u, 0u);
}

int zero_border_nhwc(void* x, int N, int H, int W, int C, cudaStream_t stream) {
  RSP_CHECK_ARG(x && N > 0 && H >= 3 && W >= 3 && C % 8 == 0, "zero_border_nhwc: bad args");
  const long long total = static_cast<long long>(N) * (2 * W + 2 * (H - 2)) * (C / 8);
  zero_border_nhwc_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<__nv_bfloat16*>(x), N, H, W, C);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
__global__ void sin_fold_kernel(const float* __restrict__ in, float* __restrict__ out, long long n_out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_out) return;
  const float2 v = *reinterpret_cast<const float2*>(in + 2 * i);
  out[i] = sinf(v.x) + v.y;
}

int sin_fold(const float* in, float* out, long long n_out, cudaStream_t stream) {
  RSP_CHECK_ARG(in && out && n_out > 0, "sin_fold: bad args");
  sin_fold_kernel<<<static_cast<unsigned>((n_out + 255) / 256), 256, 0, stream>>>(in, out, n_out);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace rsp
