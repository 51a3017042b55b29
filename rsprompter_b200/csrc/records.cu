// Byte-level kernels either side of the hot path (SURVEY 8(f1), 8(f2)); all HBM-bound, coalesced, no tensor cores.
//   pack_mask_bits / unpack_mask_bits   bool masks <-> the bit-packed payload of the per-image result record
//                                       (the device-side stand-in for encode_mask_results before collect_results,
//                                       mmdet/evaluation/metrics/coco_metric.py:346-400)
//   preprocess_u8                       DetDataPreprocessor.forward for one image: uint8 HWC -> channel flip ->
//                                       (x - mean) / std -> pad (data_preprocessor.py:110-148, BatchFixedSizePad :300)
//   patchify16_u8                       the same arithmetic fused into the patch-embed operand loader: uint8 HWC batch
//                                       -> bf16 [B*gh*gw, 768] patch rows (the fp32 NCHW image never exists)
#include "records.h"
#include "sm90.cuh"

namespace rsp {

// thread = 32 pixels of one row -> one uint32 of bits (pixel x = bit x % 8 of byte x / 8)
__global__ void pack_mask_bits_kernel(const unsigned char* __restrict__ masks, unsigned char* __restrict__ bits,
                                      long long rows, int W, int words) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= rows * words) return;
  const int wi = static_cast<int>(idx % words);
  const long long r = idx / words;
  const unsigned char* src = masks + r * W + wi * 32;
  const int nb = (W + 7) / 8;
  uint32_t v = 0u;
  const int n = min(32, W - wi * 32);
  if (n == 32 && ((reinterpret_cast<uintptr_t>(src) & 15) == 0)) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(src)), b = __ldg(reinterpret_cast<const uint4*>(src) + 1);
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int k = 0; k < 4; ++k) v |= (((w[i] >> (8 * k)) & 0xffu) ? 1u : 0u) << (4 * i + k);
    }
  } else {
    for (int k = 0; k < n; ++k) v |= (src[k] ? 1u : 0u) << k;
  }
  unsigned char* dst = bits + r * nb + wi * 4;
  const int bytes = min(4, nb - wi * 4);
  if (bytes == 4 && ((reinterpret_cast<uintptr_t>(dst) & 3) == 0)) *reinterpret_cast<uint32_t*>(dst) = v;
  else for (int k = 0; k < bytes; ++k) dst[k] = static_cast<unsigned char>(v >> (8 * k));
}

int pack_mask_bits(const unsigned char* masks, unsigned char* bits, long long rows, int W, cudaStream_t stream) {
  RSP_CHECK_ARG(masks && bits && rows > 0 && W > 0, "pack_mask_bits: bad args");
  const int words = (W + 31) / 32;
  const long long total = rows * words;
  pack_mask_bits_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(masks, bits, rows, W, words);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// thread = 8 pixels (one payload byte) -> 8 mask bytes
__global__ void unpack_mask_bits_kernel(const unsigned char* __restrict__ bits, unsigned char* __restrict__ masks,
                                        long long rows, int W, int nb) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= rows * nb) return;
  const int bi = static_cast<int>(idx % nb);
  const long long r = idx / nb;
  const uint32_t v = bits[idx];
  unsigned char* dst = masks + r * W + bi * 8;
  const int n = min(8, W - bi * 8);
  if (n == 8 && ((reinterpret_cast<uintptr_t>(dst) & 7) == 0)) {
    uint32_t lo = 0u, hi = 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      lo |= ((v >> k) & 1u) << (8 * k);
      hi |= ((v >> (4 + k)) & 1u) << (8 * k);
    }
    *reinterpret_cast<uint2*>(dst) = make_uint2(lo, hi);
  } else {
    for (int k = 0; k < n; ++k) dst[k] = (v >> k) & 1u;
  }
}

int unpack_mask_bits(const unsigned char* bits, unsigned char* masks, long long rows, int W, cudaStream_t stream) {
  RSP_CHECK_ARG(masks && bits && rows > 0 && W > 0, "unpack_mask_bits: bad args");
  const int nb = (W + 7) / 8;
  const long long total = rows * nb;
  unpack_mask_bits_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(bits, masks, rows, W, nb);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

struct Norm3 { float mean[3], stdv[3]; };

// thread = one output pixel (3 channel planes written; reads 3 bytes).  Division, not reciprocal multiply:
// torch computes (x - mean) / std in fp32 (data_preprocessor.py:118-119 via ImgDataPreprocessor.forward).
// Input addressing by byte strides: CHW planes (PackDetInputs' layout) = (h*w, w, 1), HWC = (1, 3w, 3).
__global__ void preprocess_u8_kernel(const unsigned char* __restrict__ img, int h, int w, long long sc, long long sy,
                                     long long sx, float* __restrict__ out, int H, int W, Norm3 nm, int swap_rb,
                                     float pad_value) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(H) * W) return;
  const int x = static_cast<int>(idx % W), y = static_cast<int>(idx / W);
  float v[3] = {pad_value, pad_value, pad_value};
  if (y < h && x < w) {
    const unsigned char* p = img + y * sy + x * sx;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float u = static_cast<float>(p[(swap_rb ? 2 - c : c) * sc]);
      v[c] = __fdiv_rn(__fsub_rn(u, nm.mean[c]), nm.stdv[c]);
    }
  }
  const size_t plane = static_cast<size_t>(H) * W;
  out[idx] = v[0]; out[plane + idx] = v[1]; out[2 * plane + idx] = v[2];
}

int preprocess_u8(const unsigned char* img, int h, int w, long long stride_c, long long stride_y, long long stride_x,
                  float* out, int H, int W, const float* mean3, const float* std3, int swap_rb, float pad_value,
                  cudaStream_t stream) {
  RSP_CHECK_ARG(img && out && mean3 && std3 && h > 0 && w > 0 && H >= h && W >= w && stride_c > 0 && stride_y > 0 &&
                stride_x > 0, "preprocess_u8: bad args (the padded size must cover the image)");
  Norm3 nm{{mean3[0], mean3[1], mean3[2]}, {std3[0], std3[1], std3[2]}};
  const long long total = static_cast<long long>(H) * W;
  preprocess_u8_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      img, h, w, stride_c, stride_y, stride_x, out, H, W, nm, swap_rb, pad_value);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// cv::resize INTER_LINEAR source tap of output index d along one axis (imgproc/src/resize.cpp, resizeGeneric's
// coefficient loop): f = (float)((d + 0.5) * scale - 0.5) with scale = 1 / (new / old) in double, i = floor(f),
// a = f - i; at either border the tap is clamped to (0, 0) / (old - 1, 0).  Explicit _rn intrinsics: no contraction.
__device__ __forceinline__ void cv_linear_tap(int d, int n_new, int n_old, int& i, float& a) {
  const double scale = __ddiv_rn(1.0, __ddiv_rn(static_cast<double>(n_new), static_cast<double>(n_old)));
  const float f = __double2float_rn(__dsub_rn(__dmul_rn(static_cast<double>(d) + 0.5, scale), 0.5));
  const float fl = floorf(f);
  i = static_cast<int>(fl);
  a = __fsub_rn(f, fl);
  if (i < 0) { i = 0; a = 0.f; }
  if (i >= n_old - 1) { i = n_old - 1; a = 0.f; }
}

// grid (pixels of the padded plane / 256, images); desc int64 [B, 8] per image = (source address, byte strides c, y,
// x, h, w, new_h, new_w).  thread = one output pixel, 3 channel planes written.  Horizontal pass then vertical pass,
// (1 - a) * p[i] + a * p[i + 1] in fp32, as cv2's HResizeLinear / VResizeLinear compute it for float images; then the
// normalisation of preprocess_u8.  Outside (new_h, new_w): pad3 (input channel order) normalised the same way.
__global__ void resize_pad_u8_kernel(const long long* __restrict__ desc, float* __restrict__ out, int Hp, int Wp,
                                     Norm3 nm, int swap_rb, Norm3 pad) {
  const long long plane = static_cast<long long>(Hp) * Wp;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= plane) return;
  const long long* d = desc + static_cast<size_t>(blockIdx.y) * 8;
  const int x = static_cast<int>(idx % Wp), y = static_cast<int>(idx / Wp);
  const int h = static_cast<int>(d[4]), w = static_cast<int>(d[5]), nh = static_cast<int>(d[6]),
            nw = static_cast<int>(d[7]);
  float v[3];
  if (y < nh && x < nw) {
    const unsigned char* img = reinterpret_cast<const unsigned char*>(d[0]);
    const long long sc = d[1], sy = d[2], sx = d[3];
    int ix, iy;
    float ax, ay;
    cv_linear_tap(x, nw, w, ix, ax);
    cv_linear_tap(y, nh, h, iy, ay);
    const int ix1 = min(ix + 1, w - 1), iy1 = min(iy + 1, h - 1);
    const float bx = __fsub_rn(1.f, ax), by = __fsub_rn(1.f, ay);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const unsigned char* p = img + (swap_rb ? 2 - c : c) * sc;
      const unsigned char* r0 = p + iy * sy;
      const unsigned char* r1 = p + iy1 * sy;
      const float h0 = __fadd_rn(__fmul_rn(static_cast<float>(r0[ix * sx]), bx), __fmul_rn(static_cast<float>(r0[ix1 * sx]), ax));
      const float h1 = __fadd_rn(__fmul_rn(static_cast<float>(r1[ix * sx]), bx), __fmul_rn(static_cast<float>(r1[ix1 * sx]), ax));
      const float u = __fadd_rn(__fmul_rn(h0, by), __fmul_rn(h1, ay));
      v[c] = __fdiv_rn(__fsub_rn(u, nm.mean[c]), nm.stdv[c]);
    }
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __fdiv_rn(__fsub_rn(pad.mean[swap_rb ? 2 - c : c], nm.mean[c]), nm.stdv[c]);
  }
  float* o = out + static_cast<size_t>(blockIdx.y) * 3 * plane + idx;
  o[0] = v[0]; o[plane] = v[1]; o[2 * plane] = v[2];
}

int resize_pad_u8(const long long* desc, const long long* desc_host, int B, float* out, int Hp, int Wp,
                  const float* mean3, const float* std3, int swap_rb, const float* pad3, cudaStream_t stream) {
  RSP_CHECK_ARG(desc && desc_host && out && mean3 && std3 && pad3 && B > 0 && B <= 65535 && Hp > 0 && Wp > 0,
                "resize_pad_u8: bad args");
  for (int b = 0; b < B; ++b) {
    const long long* d = desc_host + static_cast<size_t>(b) * 8;
    RSP_CHECK_ARG(d[0] != 0 && d[1] > 0 && d[2] > 0 && d[3] > 0 && d[4] > 0 && d[5] > 0 && d[6] > 0 && d[7] > 0 &&
                  d[6] <= Hp && d[7] <= Wp && d[4] < (1LL << 31) && d[5] < (1LL << 31),
                  "resize_pad_u8: bad descriptor (positive strides and sizes, the resized image inside the pad size)");
  }
  Norm3 nm{{mean3[0], mean3[1], mean3[2]}, {std3[0], std3[1], std3[2]}};
  Norm3 pad{{pad3[0], pad3[1], pad3[2]}, {0.f, 0.f, 0.f}};
  const long long plane = static_cast<long long>(Hp) * Wp;
  dim3 grid(static_cast<unsigned>((plane + 255) / 256), static_cast<unsigned>(B));
  resize_pad_u8_kernel<<<grid, 256, 0, stream>>>(desc, out, Hp, Wp, nm, swap_rb, pad);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// torchvision's antialiased uint8 bilinear resize (aten UpSampleKernel's separable int16-weight path), in two passes
// over host-built integer weight tables.  desc int64 [B, 16] per image = resize_pad_u8's 8 fields, then (workspace
// byte offset, x table offset, x row length, x precision, y table offset, y row length, y precision, 0); a table row
// (int32) = (first tap, tap count, weights...).  Integer MACs only: the result does not depend on device float.
__device__ __forceinline__ unsigned char aa_round(int acc, int prec) {
  return static_cast<unsigned char>(min(max((acc + (1 << (prec - 1))) >> prec, 0), 255));
}

// thread = one (source row, output column): 3 channels of the horizontal pass -> ws uint8 [3, h, new_w]
__global__ void resize_aa_h_kernel(const long long* __restrict__ desc, const int* __restrict__ tab,
                                   unsigned char* __restrict__ ws) {
  const long long* d = desc + static_cast<size_t>(blockIdx.y) * 16;
  const int h = static_cast<int>(d[4]), nw = static_cast<int>(d[7]);
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(h) * nw) return;
  const int x = static_cast<int>(idx % nw), y = static_cast<int>(idx / nw);
  const int* row = tab + d[9] + static_cast<long long>(x) * d[10];
  const int x0 = row[0], n = row[1], prec = static_cast<int>(d[11]);
  const long long sc = d[1], sx = d[3];
  const unsigned char* src = reinterpret_cast<const unsigned char*>(d[0]) + y * d[2] + x0 * sx;
  int acc0 = 0, acc1 = 0, acc2 = 0;
  for (int j = 0; j < n; ++j) {
    const int wj = __ldg(row + 2 + j);
    const unsigned char* p = src + j * sx;
    acc0 += wj * p[0];
    acc1 += wj * p[sc];
    acc2 += wj * p[2 * sc];
  }
  const long long plane = static_cast<long long>(h) * nw;
  unsigned char* o = ws + d[8] + idx;
  o[0] = aa_round(acc0, prec);
  o[plane] = aa_round(acc1, prec);
  o[2 * plane] = aa_round(acc2, prec);
}

// thread = one output pixel of the padded plane: the vertical pass over ws, then resize_pad_u8's normalisation
__global__ void resize_aa_v_pad_kernel(const long long* __restrict__ desc, const int* __restrict__ tab,
                                       const unsigned char* __restrict__ ws, float* __restrict__ out, int Hp, int Wp,
                                       Norm3 nm, int swap_rb, Norm3 pad) {
  const long long plane = static_cast<long long>(Hp) * Wp;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= plane) return;
  const long long* d = desc + static_cast<size_t>(blockIdx.y) * 16;
  const int x = static_cast<int>(idx % Wp), y = static_cast<int>(idx / Wp);
  const int h = static_cast<int>(d[4]), nh = static_cast<int>(d[6]), nw = static_cast<int>(d[7]);
  float v[3];
  if (y < nh && x < nw) {
    const int* row = tab + d[12] + static_cast<long long>(y) * d[13];
    const int y0 = row[0], n = row[1], prec = static_cast<int>(d[14]);
    const long long ip = static_cast<long long>(h) * nw;
    const unsigned char* src = ws + d[8] + static_cast<long long>(y0) * nw + x;
    int acc[3] = {0, 0, 0};
    for (int j = 0; j < n; ++j) {
      const int wj = __ldg(row + 2 + j);
      const unsigned char* p = src + static_cast<long long>(j) * nw;
      acc[0] += wj * p[0];
      acc[1] += wj * p[ip];
      acc[2] += wj * p[2 * ip];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float u = static_cast<float>(aa_round(acc[swap_rb ? 2 - c : c], prec));
      v[c] = __fdiv_rn(__fsub_rn(u, nm.mean[c]), nm.stdv[c]);
    }
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __fdiv_rn(__fsub_rn(pad.mean[swap_rb ? 2 - c : c], nm.mean[c]), nm.stdv[c]);
  }
  float* o = out + static_cast<size_t>(blockIdx.y) * 3 * plane + idx;
  o[0] = v[0]; o[plane] = v[1]; o[2 * plane] = v[2];
}

int resize_aa_pad_u8_ws_bytes(const long long* desc_host, int B, long long* bytes) {
  RSP_CHECK_ARG(desc_host && bytes && B > 0, "resize_aa_pad_u8_ws_bytes: bad args");
  long long n = 0;
  for (int b = 0; b < B; ++b) n += 3 * desc_host[static_cast<size_t>(b) * 16 + 4] * desc_host[static_cast<size_t>(b) * 16 + 7];
  *bytes = n;
  return RSP_OK;
}

// one table of n_out rows of length len: every row's taps inside [0, n_in), at most len - 2 of them
static bool aa_table_ok(const int* tab_host, long long n_tab, long long off, long long len, long long n_out,
                        long long n_in) {
  if (off < 0 || len < 3 || n_out <= 0 || off + n_out * len > n_tab) return false;
  for (long long i = 0; i < n_out; ++i) {
    const int* r = tab_host + off + i * len;
    if (r[0] < 0 || r[1] < 1 || r[1] > len - 2 || static_cast<long long>(r[0]) + r[1] > n_in) return false;
  }
  return true;
}

int resize_aa_pad_u8(const long long* desc, const long long* desc_host, const int* tab, const int* tab_host,
                     long long n_tab, int B, unsigned char* ws, long long ws_bytes, float* out, int Hp, int Wp,
                     const float* mean3, const float* std3, int swap_rb, const float* pad3, cudaStream_t stream) {
  RSP_CHECK_ARG(desc && desc_host && tab && tab_host && ws && out && mean3 && std3 && pad3 && B > 0 && B <= 65535 &&
                Hp > 0 && Wp > 0 && n_tab > 0, "resize_aa_pad_u8: bad args");
  long long ws_off = 0, max_h = 0;
  for (int b = 0; b < B; ++b) {
    const long long* d = desc_host + static_cast<size_t>(b) * 16;
    RSP_CHECK_ARG(d[0] != 0 && d[1] > 0 && d[2] > 0 && d[3] > 0 && d[4] > 0 && d[5] > 0 && d[6] > 0 && d[7] > 0 &&
                  d[6] <= Hp && d[7] <= Wp && d[4] < (1LL << 31) && d[5] < (1LL << 31) && d[8] == ws_off &&
                  d[11] >= 1 && d[11] <= 22 && d[14] >= 1 && d[14] <= 22,
                  "resize_aa_pad_u8: bad descriptor (positive strides and sizes, the resized image inside the pad "
                  "size, workspace offsets in image order, precisions in [1, 22])");
    RSP_CHECK_ARG(aa_table_ok(tab_host, n_tab, d[9], d[10], d[7], d[5]) &&
                  aa_table_ok(tab_host, n_tab, d[12], d[13], d[6], d[4]),
                  "resize_aa_pad_u8: a weight table row reads outside its source axis or the table");
    ws_off += 3 * d[4] * d[7];
    max_h = max(max_h, d[4] * d[7]);
  }
  RSP_CHECK_ARG(ws_off <= ws_bytes, "resize_aa_pad_u8: workspace too small (resize_aa_pad_u8_ws_bytes)");
  resize_aa_h_kernel<<<dim3(static_cast<unsigned>((max_h + 255) / 256), static_cast<unsigned>(B)), 256, 0, stream>>>(
      desc, tab, ws);
  RSP_CHECK_LAUNCH();
  Norm3 nm{{mean3[0], mean3[1], mean3[2]}, {std3[0], std3[1], std3[2]}};
  Norm3 pad{{pad3[0], pad3[1], pad3[2]}, {0.f, 0.f, 0.f}};
  const long long plane = static_cast<long long>(Hp) * Wp;
  resize_aa_v_pad_kernel<<<dim3(static_cast<unsigned>((plane + 255) / 256), static_cast<unsigned>(B)), 256, 0, stream>>>(
      desc, tab, ws, out, Hp, Wp, nm, swap_rb, pad);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

__device__ __forceinline__ void store_patch_seg(__nv_bfloat16* dst, const float f[16]) {
  reinterpret_cast<uint4*>(dst)[0] = make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]),
                                                pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
  reinterpret_cast<uint4*>(dst)[1] = make_uint4(pack_bf16x2(f[8], f[9]), pack_bf16x2(f[10], f[11]),
                                                pack_bf16x2(f[12], f[13]), pack_bf16x2(f[14], f[15]));
}

// HWC batch: thread = one (patch, ky): 16 pixels x 3 bytes = 48 contiguous bytes in, three 32-byte bf16 segments out
// (patch row layout [c][ky][kx], the flatten order of the patch-embed conv weight, HF:116,128)
__global__ void patchify16_u8_hwc_kernel(const unsigned char* __restrict__ img, __nv_bfloat16* __restrict__ out, int B,
                                         int Himg, int Wimg, Norm3 nm, int swap_rb) {
  const int gh = Himg / 16, gw = Wimg / 16;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(B) * gh * gw * 16) return;
  const int ky = static_cast<int>(idx & 15);
  const long long patch = idx >> 4;
  const int px = static_cast<int>(patch % gw);
  const int py = static_cast<int>((patch / gw) % gh);
  const int b = static_cast<int>(patch / (static_cast<long long>(gw) * gh));
  const unsigned char* src = img + ((static_cast<size_t>(b) * Himg + py * 16 + ky) * Wimg + px * 16) * 3;
  uint32_t raw[12];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const uint4 t = __ldg(reinterpret_cast<const uint4*>(src) + i);
    raw[4 * i] = t.x; raw[4 * i + 1] = t.y; raw[4 * i + 2] = t.z; raw[4 * i + 3] = t.w;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float f[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int b0 = 3 * k + c, b1 = 3 * k + 2 - c;
      const uint32_t u0 = (raw[b0 >> 2] >> (8 * (b0 & 3))) & 0xffu, u1 = (raw[b1 >> 2] >> (8 * (b1 & 3))) & 0xffu;
      f[k] = __fdiv_rn(__fsub_rn(static_cast<float>(swap_rb ? u1 : u0), nm.mean[c]), nm.stdv[c]);
    }
    store_patch_seg(out + patch * 768 + (c * 16 + ky) * 16, f);
  }
}

// CHW batch (the layout PackDetInputs hands to the data preprocessor): thread = one (patch, c, ky) segment of 16 bytes
__global__ void patchify16_u8_chw_kernel(const unsigned char* __restrict__ img, __nv_bfloat16* __restrict__ out, int B,
                                         int Himg, int Wimg, Norm3 nm, int swap_rb) {
  const int gh = Himg / 16, gw = Wimg / 16;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(B) * gh * gw * 48) return;
  const int seg = static_cast<int>(idx % 48);
  const long long patch = idx / 48;
  const int c = seg >> 4, ky = seg & 15;
  const int px = static_cast<int>(patch % gw);
  const int py = static_cast<int>((patch / gw) % gh);
  const int b = static_cast<int>(patch / (static_cast<long long>(gw) * gh));
  const int cs = swap_rb ? 2 - c : c;
  const unsigned char* src = img + ((static_cast<size_t>(b) * 3 + cs) * Himg + py * 16 + ky) * Wimg + px * 16;
  const uint4 t = __ldg(reinterpret_cast<const uint4*>(src));
  const uint32_t raw[4] = {t.x, t.y, t.z, t.w};
  const float mean = c == 0 ? nm.mean[0] : c == 1 ? nm.mean[1] : nm.mean[2];
  const float stdv = c == 0 ? nm.stdv[0] : c == 1 ? nm.stdv[1] : nm.stdv[2];
  float f[16];
#pragma unroll
  for (int k = 0; k < 16; ++k)
    f[k] = __fdiv_rn(__fsub_rn(static_cast<float>((raw[k >> 2] >> (8 * (k & 3))) & 0xffu), mean), stdv);
  store_patch_seg(out + patch * 768 + seg * 16, f);
}

int patchify16_u8(const unsigned char* img, int hwc, void* out, int B, int H, int W, const float* mean3,
                  const float* std3, int swap_rb, cudaStream_t stream) {
  RSP_CHECK_ARG(img && out && mean3 && std3 && B > 0 && H % 16 == 0 && W % 16 == 0 &&
                (reinterpret_cast<uintptr_t>(img) & 15) == 0, "patchify16_u8: bad shape / alignment");
  Norm3 nm{{mean3[0], mean3[1], mean3[2]}, {std3[0], std3[1], std3[2]}};
  const long long patches = static_cast<long long>(B) * (H / 16) * (W / 16);
  if (hwc)
    patchify16_u8_hwc_kernel<<<static_cast<unsigned>((patches * 16 + 255) / 256), 256, 0, stream>>>(
        img, static_cast<__nv_bfloat16*>(out), B, H, W, nm, swap_rb);
  else
    patchify16_u8_chw_kernel<<<static_cast<unsigned>((patches * 48 + 255) / 256), 256, 0, stream>>>(
        img, static_cast<__nv_bfloat16*>(out), B, H, W, nm, swap_rb);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace rsp
