// COCO compressed RLE of binary masks on the device (SURVEY 8(f) rank 1, the RLE half): the encode CocoMetric.process
// runs on the host for every predicted mask (coco_metric.py:359-367 -> mask/utils.py:37-53 -> pycocotools maskApi.c
// rleEncode + rleToString).  HBM / L2 bound, no tensor cores.
//
// Format (results.mask_to_coco_rle restates it): runs in column-major order (flat index x*H + y), the first run counts
// zeros; count j is written in 5-bit groups with a continuation bit (0x20), offset 48, and for j > 2 as the
// sign-extended difference to count j - 2.
//
// Boundaries: P[0] = 0, then every flat index p whose pixel differs from pixel p - 1 (pixel -1 counts as 0), then
// H*W.  Count j = P[j+1] - P[j], so the chars of count j depend on P[j-2 .. j+1] only, and a scan with the
// associative "boundaries so far + last three boundary positions" operator gives every column the context its first
// counts need.
//
// One CTA per mask.  The mask is walked in tiles of kThreads columns; thread t owns column x0 + t and walks it top to
// bottom (consecutive lanes read consecutive bytes of a row).  Per tile:
//   walk 1  per column: boundary count, first and last three positions, and the chars of every count whose three
//           preceding boundaries lie in the same column;
//   scans   the context before each column -> the chars of its first (up to) three counts; an exclusive sum of the
//           column chars -> the column's offset in the mask's string;
//   walk 2  (write pass only) the column again, writing its chars there.
// The length pass stores each mask's char count, a one-CTA scan turns them into offsets, and the write pass repeats
// walk 1 + scans (same code, same result) before walk 2.  No atomics: the output is deterministic.  Every write is
// bounded by the mask's [offsets[i], offsets[i+1]) range.
#include <climits>

#include <cub/block/block_scan.cuh>

#include "rle.h"

namespace rsp {
namespace {

constexpr int kThreads = 256;
constexpr int kScanThreads = 256;

struct RleCtx {
  unsigned n;   // boundaries so far, P[0] included (<= H*W + 1 < 2^32)
  int p[3];     // the last three boundary positions, p[2] the latest
};

// context of a run of columns a followed by b
struct RleCtxOp {
  __device__ __forceinline__ RleCtx operator()(const RleCtx& a, const RleCtx& b) const {
    RleCtx r;
    r.n = a.n + b.n;
    r.p[2] = b.n >= 1 ? b.p[2] : a.p[2];
    r.p[1] = b.n >= 2 ? b.p[1] : (b.n == 1 ? a.p[2] : a.p[1]);
    r.p[0] = b.n >= 3 ? b.p[0] : (b.n == 2 ? a.p[2] : (b.n == 1 ? a.p[1] : a.p[0]));
    return r;
  }
};

// the value written for the count that ends at boundary `pos`, given the context before that boundary
__device__ __forceinline__ int rle_value(const RleCtx& c, int pos) {
  int v = pos - c.p[2];
  if (c.n >= 4) v -= c.p[1] - c.p[0];   // count index c.n - 1 > 2
  return v;
}

__device__ __forceinline__ void rle_push(RleCtx& c, int pos) {
  c.p[0] = c.p[1];
  c.p[1] = c.p[2];
  c.p[2] = pos;
  ++c.n;
}

__device__ __forceinline__ int rle_chars(int v) {
  int k = 0;
  bool more;
  do {
    const int ch = v & 0x1f;
    v >>= 5;   // arithmetic shift: negative differences
    more = (ch & 0x10) ? v != -1 : v != 0;
    ++k;
  } while (more);
  return k;
}

// writes the chars of v from dst on, none at or past `end`; returns the position after them
__device__ __forceinline__ char* rle_put(char* dst, const char* end, int v) {
  bool more;
  do {
    int ch = v & 0x1f;
    v >>= 5;
    more = (ch & 0x10) ? v != -1 : v != 0;
    if (more) ch |= 0x20;
    if (dst < end) *dst = static_cast<char>(ch + 48);
    ++dst;
  } while (more);
  return dst;
}

template <bool kPacked>
struct MaskView {
  const unsigned char* m;
  int ld;   // bytes per source row
  __device__ __forceinline__ unsigned at(int y, int x) const {
    const unsigned char* row = m + static_cast<long long>(y) * ld;
    if (kPacked) return (__ldg(row + (x >> 3)) >> (x & 7)) & 1u;
    return __ldg(row + x) != 0 ? 1u : 0u;
  }
  // rows y .. y + rows - 1 (rows <= 16) of column x, row y + k in bit k
  __device__ __forceinline__ unsigned chunk(int y, int x, int rows) const {
    unsigned w = 0u;
    if (rows == 16) {
#pragma unroll
      for (int k = 0; k < 16; ++k) w |= at(y + k, x) << k;
    } else {
      for (int k = 0; k < rows; ++k) w |= at(y + k, x) << k;
    }
    return w;
  }
};

// The OR of K placed parts, seen through the rectangle that bounds them (canvas rows ry0.., columns rx0..).  Part p is
// parts[7p .. 7p + 6] = (byte offset from src, row bytes, rows, visible h, w, canvas y0, x0).  A chunk ORs the bits of
// every part that covers its column and some of its rows; the canvas is never formed.
template <bool kPacked>
struct UnionView {
  const unsigned char* src;
  const long long* parts;
  int k;
  int ry0, rx0;
  __device__ __forceinline__ unsigned chunk(int y, int x, int rows) const {
    const int cy = ry0 + y, cx = rx0 + x;
    unsigned w = 0u;
#pragma unroll 1
    for (int p = 0; p < k; ++p) {
      const long long* d = parts + 7 * p;
      const int px0 = static_cast<int>(__ldg(d + 6)), pw = static_cast<int>(__ldg(d + 4));
      if (cx < px0 || cx >= px0 + pw) continue;
      const int py0 = static_cast<int>(__ldg(d + 5)), ph = static_cast<int>(__ldg(d + 3));
      const int a = max(cy, py0), e = min(cy + rows, py0 + ph);
      if (a >= e) continue;
      const MaskView<kPacked> mv{src + __ldg(d), static_cast<int>(__ldg(d + 1))};
#pragma unroll 4
      for (int r = a; r < e; ++r) w |= mv.at(r - py0, cx - px0) << (r - cy);
    }
    return w;
  }
  __device__ __forceinline__ unsigned at(int y, int x) const { return chunk(y, x, 1); }
};

// Where the h x w source mask lies in the H x W canvas whose runs are encoded: canvas[y0 + y, x0 + x] = mask[y, x],
// zero elsewhere.  The plain mode is h = H, w = W at the origin; the union mode's "mask" is the rectangle bounding
// its parts.  Only the w source columns are walked; the zero rows and columns around them enter through the boundary
// positions alone.
struct Placement {
  int h, w;     // visible extent
  int H, W;     // canvas
  int y0, x0;   // origin
};

// f(canvas flat position) for every boundary inside source column x, top to bottom; 16 rows are loaded before any
// is examined.  With the mask spanning the canvas height (y0 = 0, h = H) runs cross columns: the pixel before row 0
// is the previous source column's last one, and a run reaching the bottom ends in the next column's walk.
// Otherwise the pixels above and below the mask are zero: a run that reaches the mask's last row ends one past it
// (unless that is the end of the canvas, where the final count closes it).  A plain mask spans its canvas, so that
// last boundary exists only for placed ones.
template <bool kPlaced, typename V, typename F>
__device__ __forceinline__ void for_each_boundary(const V& mv, const Placement& pl, int x, F&& f) {
  const bool full_height = pl.y0 == 0 && pl.h == pl.H;
  unsigned prev = full_height && x > 0 ? mv.at(pl.h - 1, x - 1) : 0u;
  const int base = (pl.x0 + x) * pl.H + pl.y0;
  for (int y0 = 0; y0 < pl.h; y0 += 16) {
    const int rows = min(16, pl.h - y0);
    const unsigned w = mv.chunk(y0, x, rows);
    unsigned change = (w ^ ((w << 1) | prev)) & ((1u << rows) - 1u);
    prev = (w >> (rows - 1)) & 1u;
    while (change) {
      const int k = __ffs(change) - 1;
      change &= change - 1u;
      f(base + y0 + k);
    }
  }
  const int end = base + pl.h;   // canvas position after the mask's last row in this column
  if (kPlaced && prev && !(full_height && x + 1 < pl.w) && end < pl.H * pl.W) f(end);
}

// Descriptor of mask i: plain (kPlaced = false) int64 [3] = (byte offset, H, W), the canvas is the mask; placed
// int64 [9] = (byte offset, source row bytes, source rows, h, w, H, W, y0, x0).
template <bool kPacked, bool kPlaced>
__device__ __forceinline__ void load_desc(const long long* desc, int i, MaskView<kPacked>& mv, Placement& pl,
                                          const unsigned char* src) {
  if (kPlaced) {
    const long long* d = desc + 9 * i;
    mv = MaskView<kPacked>{src + d[0], static_cast<int>(d[1])};
    pl = Placement{static_cast<int>(d[3]), static_cast<int>(d[4]), static_cast<int>(d[5]), static_cast<int>(d[6]),
                   static_cast<int>(d[7]), static_cast<int>(d[8])};
  } else {
    const long long* d = desc + 3 * i;
    const int H = static_cast<int>(d[1]), W = static_cast<int>(d[2]);
    mv = MaskView<kPacked>{src + d[0], kPacked ? (W + 7) / 8 : W};
    pl = Placement{H, W, H, W, 0, 0};
  }
}

using CtxScan = cub::BlockScan<RleCtx, kThreads, cub::BLOCK_SCAN_WARP_SCANS>;
using SumScan = cub::BlockScan<long long, kThreads, cub::BLOCK_SCAN_WARP_SCANS>;
union RleTemp {
  typename CtxScan::TempStorage ctx;
  typename SumScan::TempStorage sum;
};

// The encode of canvas i, shared by every mode.  kWrite = false: offsets[i + 1] = its chars.  kWrite = true: the chars
// into pool[offsets[i], offsets[i+1]).
template <bool kWrite, bool kPlaced, typename V>
__device__ __forceinline__ void rle_encode(const V& mv, const Placement& pl, int i, long long* offsets, char* pool,
                                           int* lengths, RleTemp& tmp) {
  char* out = nullptr;
  const char* end = nullptr;
  if (kWrite) {
    out = pool + offsets[i];
    end = pool + offsets[i + 1];
  }
  RleCtx carry{1u, {0, 0, 0}};   // P[0] = 0
  long long chars = 0;           // chars of the tiles before this one
  for (int x0 = 0; x0 < pl.w; x0 += kThreads) {
    const int x = x0 + threadIdx.x;
    RleCtx local{0u, {0, 0, 0}};
    int first[3] = {0, 0, 0};
    long long len = 0;
    if (x < pl.w) {
      for_each_boundary<kPlaced>(mv, pl, x, [&](int pos) {
        if (local.n >= 3) len += rle_chars((pos - local.p[2]) - (local.p[1] - local.p[0]));
        else if (local.n == 0) first[0] = pos;
        else if (local.n == 1) first[1] = pos;
        else first[2] = pos;
        rle_push(local, pos);
      });
    }
    RleCtx pre, agg;
    CtxScan(tmp.ctx).ExclusiveScan(local, pre, RleCtxOp{}, agg);
    pre = threadIdx.x == 0 ? carry : RleCtxOp{}(carry, pre);
    RleCtx c = pre;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (k < static_cast<int>(local.n)) {
        len += rle_chars(rle_value(c, first[k]));
        rle_push(c, first[k]);
      }
    }
    __syncthreads();   // tmp is reused
    long long off, tile_chars;
    SumScan(tmp.sum).ExclusiveSum(len, off, tile_chars);
    if (kWrite && x < pl.w) {
      char* dst = out + chars + off;
      c = pre;
      for_each_boundary<kPlaced>(mv, pl, x, [&](int pos) {
        dst = rle_put(dst, end, rle_value(c, pos));
        rle_push(c, pos);
      });
    }
    carry = RleCtxOp{}(carry, agg);
    chars += tile_chars;
    __syncthreads();
  }
  if (threadIdx.x == 0) {   // the last count ends at H*W
    const int v = rle_value(carry, pl.H * pl.W);
    if (kWrite) {
      rle_put(out + chars, end, v);
      const long long len = offsets[i + 1] - offsets[i];
      lengths[i] = len <= INT_MAX ? static_cast<int>(len) : -1;
    } else {
      offsets[i + 1] = chars + rle_chars(v);
    }
  }
}

template <bool kPacked, bool kWrite, bool kPlaced>
__global__ void __launch_bounds__(kThreads) mask_rle_kernel(const unsigned char* __restrict__ src,
                                                            const long long* __restrict__ desc, long long* offsets,
                                                            char* __restrict__ pool, int* __restrict__ lengths) {
  __shared__ RleTemp tmp;
  const int i = blockIdx.x;
  MaskView<kPacked> mv;
  Placement pl;
  load_desc<kPacked, kPlaced>(desc, i, mv, pl, src);
  rle_encode<kWrite, kPlaced>(mv, pl, i, offsets, pool, lengths, tmp);
}

// Union mode: canvas i is desc[4i .. 4i + 3] = (H, W, first part, parts), its parts' rows of `parts` as UnionView
// reads them.  The rectangle bounding the parts is walked as one placed mask.
template <bool kPacked, bool kWrite>
__global__ void __launch_bounds__(kThreads) mask_rle_union_kernel(const unsigned char* __restrict__ src,
                                                                  const long long* __restrict__ desc,
                                                                  const long long* __restrict__ parts,
                                                                  long long* offsets, char* __restrict__ pool,
                                                                  int* __restrict__ lengths) {
  __shared__ RleTemp tmp;
  const int i = blockIdx.x;
  const long long* d = desc + 4 * i;
  const int H = static_cast<int>(d[0]), W = static_cast<int>(d[1]), k = static_cast<int>(d[3]);
  const long long* pp = parts + 7 * d[2];
  int y0 = INT_MAX, x0 = INT_MAX, y1 = 0, x1 = 0;
  for (int p = 0; p < k; ++p) {
    const long long* q = pp + 7 * p;
    y0 = min(y0, static_cast<int>(q[5]));
    x0 = min(x0, static_cast<int>(q[6]));
    y1 = max(y1, static_cast<int>(q[5] + q[3]));
    x1 = max(x1, static_cast<int>(q[6] + q[4]));
  }
  const UnionView<kPacked> uv{src, pp, k, y0, x0};
  const Placement pl{y1 - y0, x1 - x0, H, W, y0, x0};
  rle_encode<kWrite, true>(uv, pl, i, offsets, pool, lengths, tmp);
}

// offsets[1..n] = inclusive sum of the per-mask char counts stored there, offsets[0] = 0
__global__ void __launch_bounds__(kScanThreads) rle_offsets_kernel(long long* offsets, int n) {
  using Scan = cub::BlockScan<long long, kScanThreads, cub::BLOCK_SCAN_WARP_SCANS>;
  __shared__ typename Scan::TempStorage tmp;
  long long carry = 0;
  for (int i0 = 0; i0 < n; i0 += kScanThreads) {
    const int i = i0 + threadIdx.x;
    long long v = i < n ? offsets[i + 1] : 0, inc, agg;
    Scan(tmp).InclusiveSum(v, inc, agg);
    if (i < n) offsets[i + 1] = carry + inc;
    carry += agg;
    __syncthreads();
  }
  if (threadIdx.x == 0) offsets[0] = 0;
}

}  // namespace

namespace {

template <bool kPlaced>
int rle_lengths(const unsigned char* src, int packed, const long long* desc, int n, long long* offsets,
                cudaStream_t stream) {
  if (packed) mask_rle_kernel<true, false, kPlaced><<<n, kThreads, 0, stream>>>(src, desc, offsets, nullptr, nullptr);
  else mask_rle_kernel<false, false, kPlaced><<<n, kThreads, 0, stream>>>(src, desc, offsets, nullptr, nullptr);
  RSP_CHECK_LAUNCH();
  rle_offsets_kernel<<<1, kScanThreads, 0, stream>>>(offsets, n);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

template <bool kPlaced>
int rle_write(const unsigned char* src, int packed, const long long* desc, int n, const long long* offsets, char* pool,
              int* lengths, cudaStream_t stream) {
  long long* offs = const_cast<long long*>(offsets);   // only the length pass writes them
  if (packed) mask_rle_kernel<true, true, kPlaced><<<n, kThreads, 0, stream>>>(src, desc, offs, pool, lengths);
  else mask_rle_kernel<false, true, kPlaced><<<n, kThreads, 0, stream>>>(src, desc, offs, pool, lengths);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

template <bool kWrite>
void rle_union_launch(const unsigned char* src, int packed, const long long* desc, int n, const long long* parts,
                      long long* offsets, char* pool, int* lengths, cudaStream_t stream) {
  if (packed) mask_rle_union_kernel<true, kWrite><<<n, kThreads, 0, stream>>>(src, desc, parts, offsets, pool, lengths);
  else mask_rle_union_kernel<false, kWrite><<<n, kThreads, 0, stream>>>(src, desc, parts, offsets, pool, lengths);
}

}  // namespace

int mask_rle_lengths(const unsigned char* src, int packed, const long long* desc, const long long* desc_host, int n,
                     long long* offsets, cudaStream_t stream) {
  RSP_CHECK_ARG(src && desc && desc_host && offsets && n > 0 && (packed == 0 || packed == 1), "mask_rle_lengths: bad args");
  for (int i = 0; i < n; ++i) {
    const long long off = desc_host[3 * i], H = desc_host[3 * i + 1], W = desc_host[3 * i + 2];
    RSP_CHECK_ARG(off >= 0 && H >= 1 && W >= 1 && H <= INT_MAX && W <= INT_MAX && H * W <= INT_MAX,
                  "mask_rle_lengths: mask %d is %lld x %lld at offset %lld (1 .. 2^31 - 1 pixels)", i, H, W, off);
  }
  return rle_lengths<false>(src, packed, desc, n, offsets, stream);
}

int mask_rle_write(const unsigned char* src, int packed, const long long* desc, int n, const long long* offsets,
                   char* pool, int* lengths, cudaStream_t stream) {
  RSP_CHECK_ARG(src && desc && offsets && pool && lengths && n > 0 && (packed == 0 || packed == 1),
                "mask_rle_write: bad args");
  return rle_write<false>(src, packed, desc, n, offsets, pool, lengths, stream);
}

int mask_rle_placed_lengths(const unsigned char* src, int packed, const long long* desc, const long long* desc_host,
                            int n, long long* offsets, cudaStream_t stream) {
  RSP_CHECK_ARG(src && desc && desc_host && offsets && n > 0 && (packed == 0 || packed == 1),
                "mask_rle_placed_lengths: bad args");
  for (int i = 0; i < n; ++i) {
    const long long* d = desc_host + 9 * i;
    const long long off = d[0], ld = d[1], rows = d[2], h = d[3], w = d[4], H = d[5], W = d[6], y0 = d[7], x0 = d[8];
    RSP_CHECK_ARG(H >= 1 && W >= 1 && H <= INT_MAX && W <= INT_MAX && H * W <= INT_MAX,
                  "mask_rle_placed_lengths: mask %d: canvas %lld x %lld (1 .. 2^31 - 1 pixels)", i, H, W);
    RSP_CHECK_ARG(y0 >= 0 && x0 >= 0 && y0 < H && x0 < W,
                  "mask_rle_placed_lengths: mask %d: origin (%lld, %lld) outside the %lld x %lld canvas", i, y0, x0, H, W);
    RSP_CHECK_ARG(h >= 1 && w >= 1 && h <= H - y0 && w <= W - x0,
                  "mask_rle_placed_lengths: mask %d: %lld x %lld at (%lld, %lld) leaves the %lld x %lld canvas", i, h, w,
                  y0, x0, H, W);
    RSP_CHECK_ARG(off >= 0 && ld <= INT_MAX && h <= rows && w <= (packed ? 8 * ld : ld),
                  "mask_rle_placed_lengths: mask %d: visible %lld x %lld exceeds the source (%lld rows of %lld bytes, "
                  "offset %lld)", i, h, w, rows, ld, off);
  }
  return rle_lengths<true>(src, packed, desc, n, offsets, stream);
}

int mask_rle_placed_write(const unsigned char* src, int packed, const long long* desc, int n, const long long* offsets,
                          char* pool, int* lengths, cudaStream_t stream) {
  RSP_CHECK_ARG(src && desc && offsets && pool && lengths && n > 0 && (packed == 0 || packed == 1),
                "mask_rle_placed_write: bad args");
  return rle_write<true>(src, packed, desc, n, offsets, pool, lengths, stream);
}

int mask_rle_union_lengths(const unsigned char* src, int packed, const long long* desc, const long long* desc_host,
                           int n, const long long* parts, const long long* parts_host, int num_parts, long long* offsets,
                           cudaStream_t stream) {
  RSP_CHECK_ARG(src && desc && desc_host && parts && parts_host && offsets && n > 0 && num_parts > 0 &&
                (packed == 0 || packed == 1), "mask_rle_union_lengths: bad args");
  for (int i = 0; i < n; ++i) {
    const long long H = desc_host[4 * i], W = desc_host[4 * i + 1], first = desc_host[4 * i + 2],
                    k = desc_host[4 * i + 3];
    RSP_CHECK_ARG(H >= 1 && W >= 1 && H <= INT_MAX && W <= INT_MAX && H * W <= INT_MAX,
                  "mask_rle_union_lengths: mask %d: canvas %lld x %lld (1 .. 2^31 - 1 pixels)", i, H, W);
    RSP_CHECK_ARG(first >= 0 && k >= 1 && k <= num_parts - first,
                  "mask_rle_union_lengths: mask %d: parts [%lld, %lld + %lld) outside the %d parts", i, first, first, k,
                  num_parts);
    for (long long p = first; p < first + k; ++p) {
      const long long* d = parts_host + 7 * p;
      const long long off = d[0], ld = d[1], rows = d[2], h = d[3], w = d[4], y0 = d[5], x0 = d[6];
      RSP_CHECK_ARG(y0 >= 0 && x0 >= 0 && y0 < H && x0 < W,
                    "mask_rle_union_lengths: mask %d, part %lld: origin (%lld, %lld) outside the %lld x %lld canvas", i,
                    p, y0, x0, H, W);
      RSP_CHECK_ARG(h >= 1 && w >= 1 && h <= H - y0 && w <= W - x0,
                    "mask_rle_union_lengths: mask %d, part %lld: %lld x %lld at (%lld, %lld) leaves the %lld x %lld "
                    "canvas", i, p, h, w, y0, x0, H, W);
      RSP_CHECK_ARG(off >= 0 && ld <= INT_MAX && h <= rows && w <= (packed ? 8 * ld : ld),
                    "mask_rle_union_lengths: mask %d, part %lld: visible %lld x %lld exceeds the source (%lld rows of "
                    "%lld bytes, offset %lld)", i, p, h, w, rows, ld, off);
    }
  }
  rle_union_launch<false>(src, packed, desc, n, parts, offsets, nullptr, nullptr, stream);
  RSP_CHECK_LAUNCH();
  rle_offsets_kernel<<<1, kScanThreads, 0, stream>>>(offsets, n);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

int mask_rle_union_write(const unsigned char* src, int packed, const long long* desc, int n, const long long* parts,
                         const long long* offsets, char* pool, int* lengths, cudaStream_t stream) {
  RSP_CHECK_ARG(src && desc && parts && offsets && pool && lengths && n > 0 && (packed == 0 || packed == 1),
                "mask_rle_union_write: bad args");
  rle_union_launch<true>(src, packed, desc, n, parts, const_cast<long long*>(offsets), pool, lengths, stream);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace rsp
