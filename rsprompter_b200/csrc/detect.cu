// Detection-side kernels of the RSPrompter-anchor path: all batched over images with fixed-size
// padded candidate lists, so the whole RPN -> RoI -> mask pipeline runs without host syncs.
//
//   rpn_decode        top-k anchor indices -> sigmoid scores + delta2bbox boxes (rpn_head.py:188-226,
//                     anchor_generator.py:161-301, delta_xywh_bbox_coder.py:325-359)
//   bbox_cls_decode   softmax class scores + per-class delta2bbox (bbox_head.py:520-545)
//   nms_batched       mmcv.ops.batched_nms semantics: boxes offset by id * (max + 1), greedy NMS,
//                     suppress when IoU > thr (bbox_nms.py:95, rpn_head.py:285)
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

// one CTA (4 warps) per image: greedy scan in score order, 64 candidates at a time.  Warp 0 resolves a
// block serially in registers (the 64 diagonal mask words are held two per lane and broadcast by
// shuffle); then all 128 threads OR the kept rows' remaining words into the suppression bitmap,
// eight independent loads in flight per thread (the mask is L2-resident).
__global__ void __launch_bounds__(128)
nms_scan_kernel(const unsigned long long* __restrict__ mask, const int* __restrict__ nvalid, int n, int max_keep,
                unsigned char* __restrict__ keep) {
  extern __shared__ unsigned long long remv[];
  __shared__ unsigned long long kept_s;
  const int b = blockIdx.x;
  const int nv = nvalid[b];
  const int words = (n + 63) / 64;
  const int nvw = (nv + 63) / 64;
  const int tid = threadIdx.x, lane = tid & 31;
  for (int w = tid; w < words; w += blockDim.x) remv[w] = 0ull;
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
        for (int tbit = 0; tbit < 64; ++tbit) {
          const unsigned long long dw = __shfl_sync(0xffffffffu, tbit < 32 ? d0 : d1, tbit & 31);
          if (i0 + tbit < nv && !((cur >> tbit) & 1ull)) {
            keptbits |= 1ull << tbit;
            cur |= dw;
          }
        }
        if (lane == 0) kept_s = keptbits;
      }
      __syncthreads();
      const unsigned long long keptbits = kept_s;
      kept_total += __popcll(keptbits);
      for (int w = blk + 1 + tid; w < nvw; w += blockDim.x) {
        unsigned long long acc = remv[w];
        unsigned long long kb = keptbits;
        while (kb) {
          unsigned long long v[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            v[u] = 0ull;
            if (kb) {
              const int tbit = __ffsll(static_cast<long long>(kb)) - 1;
              kb &= kb - 1;
              v[u] = mbase[static_cast<size_t>(i0 + tbit) * words + w];
            }
          }
#pragma unroll
          for (int u = 0; u < 8; ++u) acc |= v[u];
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
  nms_scan_kernel<<<B, 128, words * 8, stream>>>(mask_ws, nvalid, n, max_keep, keep);
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
// logits fp32 [n, hm, wm] -> uint8 [n, H, W].  mode 0: (bilinear(sigmoid(x)) >= thr);
// mode 1: (bilinear(x) > thr).  PyTorch align_corners=False source index rule.
__global__ void mask_paste_kernel(const float* __restrict__ logits, unsigned char* __restrict__ out, int n,
                                  int hm, int wm, int H, int W, float thr, int mode) {
  // thread = 16 consecutive output pixels of one row (one 16-byte store)
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int w16 = W / 16;
  const long long total = static_cast<long long>(n) * H * w16;
  if (idx >= total) return;
  const int xb = static_cast<int>(idx % w16);
  long long t = idx / w16;
  const int y = static_cast<int>(t % H);
  const int m = static_cast<int>(t / H);
  const float sy = fmaxf((y + 0.5f) * (static_cast<float>(hm) / H) - 0.5f, 0.f);
  const int y0 = static_cast<int>(sy), y1 = min(y0 + 1, hm - 1);
  const float ly = sy - y0;
  const float* r0 = logits + (static_cast<size_t>(m) * hm + y0) * wm;
  const float* r1 = logits + (static_cast<size_t>(m) * hm + y1) * wm;
  const float sxs = static_cast<float>(wm) / W;
  uint32_t packed[4] = {0u, 0u, 0u, 0u};
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int x = xb * 16 + k;
    const float sx = fmaxf((x + 0.5f) * sxs - 0.5f, 0.f);
    const int x0 = static_cast<int>(sx), x1 = min(x0 + 1, wm - 1);
    const float lx = sx - x0;
    float v00 = __ldg(r0 + x0), v01 = __ldg(r0 + x1), v10 = __ldg(r1 + x0), v11 = __ldg(r1 + x1);
    if (mode == 0) {
      v00 = 1.f / (1.f + expf(-v00)); v01 = 1.f / (1.f + expf(-v01));
      v10 = 1.f / (1.f + expf(-v10)); v11 = 1.f / (1.f + expf(-v11));
    }
    const float v = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
    const uint32_t bit = (mode == 1 ? (v > thr) : (v >= thr)) ? 1u : 0u;   // mode 2: input already activated
    packed[k >> 2] |= bit << ((k & 3) * 8);
  }
  *reinterpret_cast<uint4*>(out + (static_cast<size_t>(m) * H + y) * W + xb * 16) =
      make_uint4(packed[0], packed[1], packed[2], packed[3]);
}

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

// general case: resized / padded images (two chained resizes with a crop); thread = 4 output pixels of one row
template <int MODE>
__global__ void mask_paste_rescale_kernel(const float* __restrict__ maps, unsigned char* __restrict__ out, int n,
                                          Resize2 g, float thr) {
  const int w4 = (g.W + 3) / 4;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(n) * g.H * w4) return;
  const int xb = static_cast<int>(idx % w4);
  long long t = idx / w4;
  const int y = static_cast<int>(t % g.H);
  const int m = static_cast<int>(t / g.H);
  const float* src = maps + static_cast<size_t>(m) * g.hm * g.wm;
  unsigned char* o = out + (static_cast<size_t>(m) * g.H + y) * g.W;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int x = 4 * xb + k;
    if (x >= g.W) break;
    const float v = resize2_at(src, g, y, x);
    o[x] = (MODE == 1 ? (v > thr) : (v >= thr)) ? 1 : 0;
  }
}

int mask_paste_rescale(const float* maps, unsigned char* out, int n, int hm, int wm, int Hb, int Wb, int crop_h,
                       int crop_w, int H, int W, float thr, int mode, cudaStream_t stream) {
  RSP_CHECK_ARG(maps && out && n > 0 && hm > 0 && wm > 0 && Hb > 0 && Wb > 0 && crop_h > 0 && crop_w > 0 &&
                crop_h <= Hb && crop_w <= Wb && H > 0 && W > 0 && (mode == 1 || mode == 2),
                "mask_paste_rescale: bad args (mode 1: > thr on raw maps, 2: >= thr on activated maps)");
  Resize2 g{hm, wm, Hb, Wb, crop_h, crop_w, H, W};
  const long long total = static_cast<long long>(n) * H * ((W + 3) / 4);
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  if (mode == 1) mask_paste_rescale_kernel<1><<<blocks, 256, 0, stream>>>(maps, out, n, g, thr);
  else mask_paste_rescale_kernel<2><<<blocks, 256, 0, stream>>>(maps, out, n, g, thr);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// FCNMaskHead paste (fcn_mask_head.py:_do_paste_mask + the threshold of _predict_by_feat_single :388-392): the
// activated RoI mask probs fp32 [n, hm, wm] of detection i are sampled bilinearly (F.grid_sample, align_corners=False,
// zero padding) at every image pixel centre mapped into its box, then compared with thr.  thread = 16 output pixels of
// one row (one 16-byte store); rows / columns whose taps all fall outside the RoI grid write zeros without loads.
__global__ void mask_paste_boxes_kernel(const float* __restrict__ probs, const float* __restrict__ boxes,
                                        unsigned char* __restrict__ out, int n, int hm, int wm, int H, int W, float thr,
                                        int packed) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int w16 = (W + 15) / 16;
  if (idx >= static_cast<long long>(n) * H * w16) return;
  const int xb = static_cast<int>(idx % w16);
  long long t = idx / w16;
  const int y = static_cast<int>(t % H);
  const int m = static_cast<int>(t / H);
  const float x0 = boxes[m * 4], y0 = boxes[m * 4 + 1], x1 = boxes[m * 4 + 2], y1 = boxes[m * 4 + 3];
  // normalised grid coordinate in [-1, 1] (inf from a degenerate box becomes 0, as the reference does)
  float gy = __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn(y + 0.5f, y0), __fsub_rn(y1, y0)), 2.f), 1.f);
  if (isinf(gy)) gy = 0.f;
  const float iy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), static_cast<float>(hm)), 1.f), 0.5f);
  const float fy = floorf(iy);
  const int yi0 = static_cast<int>(fy), yi1 = yi0 + 1;
  const bool vy0 = yi0 >= 0 && yi0 < hm, vy1 = yi1 >= 0 && yi1 < hm;
  const float* p = probs + static_cast<size_t>(m) * hm * wm;
  uint32_t pk[4] = {0u, 0u, 0u, 0u};
  if (vy0 || vy1) {
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int x = xb * 16 + k;
      float gx = __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn(x + 0.5f, x0), __fsub_rn(x1, x0)), 2.f), 1.f);
      if (isinf(gx)) gx = 0.f;
      const float ix = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), static_cast<float>(wm)), 1.f), 0.5f);
      const float fx = floorf(ix);
      const int xi0 = static_cast<int>(fx), xi1 = xi0 + 1;
      const bool vx0 = xi0 >= 0 && xi0 < wm, vx1 = xi1 >= 0 && xi1 < wm;
      const float v00 = (vy0 && vx0) ? __ldg(p + yi0 * wm + xi0) : 0.f, v01 = (vy0 && vx1) ? __ldg(p + yi0 * wm + xi1) : 0.f;
      const float v10 = (vy1 && vx0) ? __ldg(p + yi1 * wm + xi0) : 0.f, v11 = (vy1 && vx1) ? __ldg(p + yi1 * wm + xi1) : 0.f;
      // grid_sample weights in ATen's form: (x_se - ix)(y_se - iy), (ix - x_nw)(y_se - iy), (x_se - ix)(iy - y_nw), ...
      const float wx0 = (fx + 1.f) - ix, wx1 = ix - fx, wy0 = (fy + 1.f) - iy, wy1 = iy - fy;
      const float v = v00 * (wx0 * wy0) + v01 * (wx1 * wy0) + v10 * (wx0 * wy1) + v11 * (wx1 * wy1);
      pk[k >> 2] |= (v >= thr ? 1u : 0u) << ((k & 3) * 8);
    }
  }
  if (packed) {   // result-record layout: pixel x = bit x % 8 of byte x / 8 (W % 16 == 0)
    uint32_t bits = 0;
#pragma unroll
    for (int k = 0; k < 16; ++k) bits |= ((pk[k >> 2] >> ((k & 3) * 8)) & 1u) << k;
    *reinterpret_cast<unsigned short*>(out + (static_cast<size_t>(m) * H + y) * (W / 8) + xb * 2) =
        static_cast<unsigned short>(bits);
    return;
  }
  unsigned char* dst = out + (static_cast<size_t>(m) * H + y) * W + xb * 16;
  if ((W & 15) == 0) {
    *reinterpret_cast<uint4*>(dst) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
  } else {   // original-image canvases of any width: byte stores
    for (int k = 0; k < 16 && xb * 16 + k < W; ++k) dst[k] = static_cast<unsigned char>((pk[k >> 2] >> ((k & 3) * 8)) & 1u);
  }
}

int mask_paste_boxes(const float* probs, const float* boxes, unsigned char* out, int n, int hm, int wm, int H, int W,
                     float thr, int packed, cudaStream_t stream) {
  RSP_CHECK_ARG(probs && boxes && out && n > 0 && hm > 0 && wm > 0 && H > 0 && W > 0, "mask_paste_boxes: bad arguments");
  RSP_CHECK_ARG(!packed || W % 16 == 0, "mask_paste_boxes: bit-packed output needs W % 16 == 0");
  const long long total = static_cast<long long>(n) * H * ((W + 15) / 16);
  mask_paste_boxes_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(probs, boxes, out, n, hm, wm, H, W,
                                                                                         thr, packed);
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

int mask_paste_bits(const float* maps, unsigned char* bits, int n, int hm, int wm, float thr, int mode,
                    cudaStream_t stream) {
  RSP_CHECK_ARG(maps && bits && n > 0 && wm % 4 == 0 && (mode == 1 || mode == 2) &&
                (reinterpret_cast<uintptr_t>(maps) & 15) == 0 && (reinterpret_cast<uintptr_t>(bits) & 1) == 0,
                "mask_paste_bits: x4 path only (wm % 4 == 0, mode 1: > thr on raw maps, 2: >= thr on activated maps)");
  const long long tiles = static_cast<long long>(n) * hm * (wm / 4);
  const unsigned blocks = static_cast<unsigned>((tiles + 127) / 128);
  if (mode == 1) mask_paste_x4_kernel<1, true><<<blocks, 128, 0, stream>>>(maps, bits, n, hm, wm, thr);
  else mask_paste_x4_kernel<2, true><<<blocks, 128, 0, stream>>>(maps, bits, n, hm, wm, thr);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

int mask_paste(const float* logits, unsigned char* out, int n, int hm, int wm, int H, int W, float thr,
               int mode, cudaStream_t stream) {
  RSP_CHECK_ARG(logits && out && n > 0 && W % 16 == 0, "mask_paste: W must be a multiple of 16");
  if (mode != 0 && H == 4 * hm && W == 4 * wm && wm % 4 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0) {
    const long long tiles = static_cast<long long>(n) * hm * (wm / 4);
    const unsigned blocks = static_cast<unsigned>((tiles + 127) / 128);
    if (mode == 1) mask_paste_x4_kernel<1, false><<<blocks, 128, 0, stream>>>(logits, out, n, hm, wm, thr);
    else mask_paste_x4_kernel<2, false><<<blocks, 128, 0, stream>>>(logits, out, n, hm, wm, thr);
    RSP_CHECK_LAUNCH();
    return RSP_OK;
  }
  const long long total = static_cast<long long>(n) * H * (W / 16);
  mask_paste_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(logits, out, n, hm, wm, H, W,
                                                                                   thr, mode);
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
