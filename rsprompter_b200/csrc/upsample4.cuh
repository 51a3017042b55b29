// x4 bilinear up-sampling (F.interpolate(scale 4, mode='bilinear', align_corners=False)) of an fp32 map, one
// 4-row x 16-column output tile per call: 3 source rows x 6 source columns are loaded once (18 loads for 64
// outputs instead of 256) and the horizontal pass is shared by the 4 output rows.  The arithmetic keeps the
// per-pixel form  (1-ly) * ((1-lx) * v00 + lx * v01) + ly * ((1-lx) * v10 + lx * v11)  with the exact fractions
// 0.625 / 0.875 / 0.125 / 0.375 the source-index rule produces, and lx = ly = 0 on the clamped top / left border
// (M:652-656, M:1763-1777 use this resize for every predicted mask).
#pragma once
#include <cuda_runtime.h>

namespace rsp {

struct Up4Tile {
  float h[3][16];   // horizontally interpolated source rows yb-1, yb, yb+1 (clamped)
  bool edge_y;      // yb == 0: output rows 0, 1 take source row 0 with ly = 0
};

// src: one [hm, wm] map (wm % 4 == 0, 16-byte aligned rows); tile (yb, xb): output rows 4yb..4yb+3, cols 16xb..16xb+15
__device__ __forceinline__ void up4_load(const float* __restrict__ src, int hm, int wm, int yb, int xb, Up4Tile& t) {
  const bool edge_x = xb == 0;
  t.edge_y = yb == 0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int r = min(max(yb - 1 + i, 0), hm - 1);
    const float* rp = src + static_cast<size_t>(r) * wm;
    float a[6];
    a[0] = __ldg(rp + max(4 * xb - 1, 0));
    const float4 m = __ldg(reinterpret_cast<const float4*>(rp + 4 * xb));
    a[1] = m.x; a[2] = m.y; a[3] = m.z; a[4] = m.w;
    a[5] = __ldg(rp + min(4 * xb + 4, wm - 1));
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int q = k >> 2, f = k & 3;
      const int j = q + (f >= 2 ? 1 : 0);
      float lx = f == 0 ? 0.625f : f == 1 ? 0.875f : f == 2 ? 0.125f : 0.375f;
      float lo = a[j], hi = a[j + 1];
      if (k < 2) {   // left image border: source index clamps to 0 with lx = 0
        lo = edge_x ? a[1] : lo;
        hi = edge_x ? a[2] : hi;
        lx = edge_x ? 0.f : lx;
      }
      t.h[i][k] = (1.f - lx) * lo + lx * hi;
    }
  }
}

// value at output row 4yb + j (j compile-time after unrolling), column 16xb + k
__device__ __forceinline__ float up4_value(const Up4Tile& t, int j, int k) {
  float ly = j == 0 ? 0.625f : j == 1 ? 0.875f : j == 2 ? 0.125f : 0.375f;
  float top = j < 2 ? t.h[0][k] : t.h[1][k];
  float bot = j < 2 ? t.h[1][k] : t.h[2][k];
  if (j < 2) {
    top = t.edge_y ? t.h[1][k] : top;
    bot = t.edge_y ? t.h[2][k] : bot;
    ly = t.edge_y ? 0.f : ly;
  }
  return (1.f - ly) * top + ly * bot;
}

// Two chained F.interpolate(bilinear, align_corners=False) calls with a crop in between (the reference's mask
// path when the image was resized / padded: low-res map -> batch_input_shape -> crop to the resized image ->
// ori_shape; M:1763-1777, M:652-656 + 679-691), evaluated per output pixel without the intermediate map: the
// 4 intermediate taps are themselves bilinear samples of the source, with fp32 rounding at the same places.
struct Resize2 {
  int hm, wm;      // source map
  int Hb, Wb;      // intermediate (batch_input_shape)
  int ch, cw;      // crop of the intermediate that is resized (<= Hb, Wb)
  int H, W;        // output (ori_shape)
};

__device__ __forceinline__ float bilinear_at(const float* __restrict__ src, int h, int w, int H, int W, int y, int x) {
  const float sy = fmaxf((y + 0.5f) * (static_cast<float>(h) / H) - 0.5f, 0.f);
  const float sx = fmaxf((x + 0.5f) * (static_cast<float>(w) / W) - 0.5f, 0.f);
  const int y0 = min(static_cast<int>(sy), h - 1), x0 = min(static_cast<int>(sx), w - 1);
  const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
  const float ly = sy - y0, lx = sx - x0;
  return (1.f - ly) * ((1.f - lx) * __ldg(src + y0 * w + x0) + lx * __ldg(src + y0 * w + x1)) +
         ly * ((1.f - lx) * __ldg(src + y1 * w + x0) + lx * __ldg(src + y1 * w + x1));
}

// bilinear_at's resize (h, w) -> (H, W) of map m of maps [*, h, w] as a paste sampler: row() sets up an output row,
// at() returns the value at a column of it.  SIG applies the sigmoid to the 4 taps first.  The fused multiply-adds
// are explicit because where the blend rounds decides the pixels at the threshold: this is the rounding
// rsp_mask_paste and rsp_query_postprocess have always had, which differ in the top-row blend (FUSE_RIGHT: the right
// tap's product is the fused one).
template <bool SIG, bool FUSE_RIGHT>
struct OneResize {
  const float* maps;
  int h, w, H, W;
  const float* r0;
  const float* r1;
  float ly;

  __device__ __forceinline__ bool row(int m, int y) {
    const float sy = fmaxf(fmaf(y + 0.5f, static_cast<float>(h) / H, -0.5f), 0.f);
    const int y0 = min(static_cast<int>(sy), h - 1), y1 = min(y0 + 1, h - 1);
    ly = sy - y0;
    r0 = maps + (static_cast<size_t>(m) * h + y0) * w;
    r1 = maps + (static_cast<size_t>(m) * h + y1) * w;
    return true;
  }

  __device__ __forceinline__ float at(int x) const {
    const float sx = fmaxf(fmaf(x + 0.5f, static_cast<float>(w) / W, -0.5f), 0.f);
    const int x0 = min(static_cast<int>(sx), w - 1), x1 = min(x0 + 1, w - 1);
    const float lx = sx - x0;
    float v00 = __ldg(r0 + x0), v01 = __ldg(r0 + x1), v10 = __ldg(r1 + x0), v11 = __ldg(r1 + x1);
    if (SIG) {
      v00 = 1.f / (1.f + expf(-v00)); v01 = 1.f / (1.f + expf(-v01));
      v10 = 1.f / (1.f + expf(-v10)); v11 = 1.f / (1.f + expf(-v11));
    }
    const float top = FUSE_RIGHT ? fmaf(lx, v01, __fmul_rn(1.f - lx, v00)) : fmaf(1.f - lx, v00, __fmul_rn(lx, v01));
    const float bot = fmaf(1.f - lx, v10, __fmul_rn(lx, v11));
    return fmaf(1.f - ly, top, __fmul_rn(ly, bot));
  }
};

__device__ __forceinline__ float resize2_at(const float* __restrict__ src, const Resize2& g, int y, int x) {
  // second resize: (ch, cw) -> (H, W)
  const float sy = fmaxf((y + 0.5f) * (static_cast<float>(g.ch) / g.H) - 0.5f, 0.f);
  const float sx = fmaxf((x + 0.5f) * (static_cast<float>(g.cw) / g.W) - 0.5f, 0.f);
  const int y0 = min(static_cast<int>(sy), g.ch - 1), x0 = min(static_cast<int>(sx), g.cw - 1);
  const int y1 = min(y0 + 1, g.ch - 1), x1 = min(x0 + 1, g.cw - 1);
  const float ly = sy - y0, lx = sx - x0;
  // first resize (hm, wm) -> (Hb, Wb), sampled at the 4 taps
  const float v00 = bilinear_at(src, g.hm, g.wm, g.Hb, g.Wb, y0, x0), v01 = bilinear_at(src, g.hm, g.wm, g.Hb, g.Wb, y0, x1);
  const float v10 = bilinear_at(src, g.hm, g.wm, g.Hb, g.Wb, y1, x0), v11 = bilinear_at(src, g.hm, g.wm, g.Hb, g.Wb, y1, x1);
  return (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
}

// resize2_at of map m of maps [*, hm, wm], row by row as OneResize
struct TwoResizes {
  const float* maps;
  Resize2 g;
  const float* src;
  int y;

  __device__ __forceinline__ bool row(int m, int yy) {
    src = maps + static_cast<size_t>(m) * g.hm * g.wm;
    y = yy;
    return true;
  }

  __device__ __forceinline__ float at(int x) const { return resize2_at(src, g, y, x); }
};

}  // namespace rsp
