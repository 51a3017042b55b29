// Small-region removal of SAM's automatic mask generator (segment_anything/utils/amg.py remove_small_regions, called
// per mask by SamAutomaticMaskGenerator.postprocess_small_regions) on bit-packed masks, for many masks at once.
//
// The working mask is ~mask (holes) or mask (islands).  Its 8-connected components come from a block-based union-find
// (Allegretti, Bolelli and Grana's BUF) over 2 x 2 pixel blocks: under 8-connectivity the four pixels of a block are
// mutually adjacent, so a block belongs to at most one component.  Unions go toward the smaller block index, so each
// component's root is its smallest block index (y / 2) * ceil(W / 2) + x / 2: the key by which cv2's default
// connectedComponentsWithStats (8-connectivity, Spaghetti) numbers its labels, which decides the islands fallback.
//
// merge, area and write: one thread covers a 2 x 32 pixel strip (16 blocks), rows 2 by and 2 by + 1, pixels
// [32 k, 32 k + 32), read as one 32-bit word per row (two 16-bit halves, since a row is only 2-byte aligned).  init,
// compress and decide touch labels only (init reads 2 bits per row): one thread per block, so a warp's label accesses
// are 32 consecutive ints.  A CTA covers a part of one mask.
// labels int32 [n, BH, BW] (BH = ceil(H / 2), BW = ceil(W / 2)) go through these values:
//   init      -1 for a block with no working pixel, else its own index
//   merge     parent pointers; a root points to itself
//   compress  every block points at its root; a root holds -1
//   area      a root holds -1 - (its component's pixel count)          (atomic adds: integers, order-free)
// then decide reduces, per mask, whether any component is small or large and the (area, -root) maximum, and write
// sets the output bits and reduces the output box.  Atomics race on intermediate labels only: every output is a
// function of the components, so two launches give identical bytes.
#include <climits>

#include "regions.h"

namespace rsp {
namespace {

constexpr int kThreads = 256;
constexpr int kBg = -1;
constexpr uint32_t kEven = 0x55555555u;

struct Geo {
  int H, W, ld, BH, BW, KW;
  int cpm;                         // CTAs per mask, one thread per strip (KW = ceil(W / 32) strips per row pair)
  int cpb;                         // CTAs per mask, one thread per block
};

struct MaskState {                  // 32 bytes per mask at the front of the workspace
  unsigned long long best;          // max of (area << 32 | ~root): the largest component, first label on ties
  int small, large;                 // some component has area < min_area / >= min_area
  int box[4];                       // x_min, y_min, x_max, y_max of the output
};

// one thread per 2 x 2 block: -> its mask m and index b, false past the mask's last block
__device__ __forceinline__ bool block(const Geo& g, int& m, int& b) {
  m = static_cast<int>(blockIdx.x / g.cpb);
  b = static_cast<int>(blockIdx.x % g.cpb) * kThreads + static_cast<int>(threadIdx.x);
  return b < g.BH * g.BW;
}

__device__ __forceinline__ bool strip(const Geo& g, int& m, int& by, int& k) {
  m = static_cast<int>(blockIdx.x / g.cpm);
  const int it = static_cast<int>(blockIdx.x % g.cpm) * kThreads + static_cast<int>(threadIdx.x);
  by = it / g.KW;
  k = it % g.KW;
  return by < g.BH;
}

// pixels [32 k, 32 k + 32) of row y as bits (pixel 32 k + i = bit i), x >= W cleared; 0 outside the image
__device__ __forceinline__ uint32_t raw_word(const unsigned char* mask, const Geo& g, int y, int k) {
  if (y < 0 || y >= g.H || k < 0 || k >= g.KW) return 0u;
  const uint16_t* r = reinterpret_cast<const uint16_t*>(mask + static_cast<size_t>(y) * g.ld) + 2 * k;
  uint32_t w = __ldg(r);
  if (4 * k + 2 < g.ld) w |= static_cast<uint32_t>(__ldg(r + 1)) << 16;
  const int rem = g.W - 32 * k;
  return rem >= 32 ? w : w & ((1u << rem) - 1u);
}

__device__ __forceinline__ uint32_t work_word(const unsigned char* mask, const Geo& g, int y, int k, bool holes) {
  if (y < 0 || y >= g.H || k < 0 || k >= g.KW) return 0u;
  const uint32_t w = raw_word(mask, g, y, k);
  if (!holes) return w;
  const int rem = g.W - 32 * k;
  return ~w & (rem >= 32 ? 0xffffffffu : (1u << rem) - 1u);
}

// bit 2 j set when pixel 2 j or 2 j + 1 of w is
__device__ __forceinline__ uint32_t pairs(uint32_t w) { return (w | (w >> 1)) & kEven; }

__device__ __forceinline__ int find_root(const int* L, int x) {
  int p = __ldcg(L + x);
  while (p != x) {
    x = p;
    p = __ldcg(L + x);
  }
  return x;
}

// link the components of blocks a and b under the smaller root
__device__ void unite(int* L, int a, int b) {
  while (true) {
    a = find_root(L, a);
    b = find_root(L, b);
    if (a == b) return;
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicMin(L + b, a);
    if (old == b) return;
    b = old;   // b got another parent meanwhile: link that one instead
  }
}

__global__ void __launch_bounds__(kThreads)
regions_init_kernel(const unsigned char* __restrict__ in, Geo g, int holes, int* __restrict__ labels,
                    MaskState* __restrict__ st) {
  int m, b;
  const bool ok = block(g, m, b);
  if (blockIdx.x % g.cpb == 0 && threadIdx.x == 0) {
    MaskState s;
    s.best = 0ull;
    s.small = s.large = 0;
    s.box[0] = s.box[1] = INT_MAX;
    s.box[2] = s.box[3] = -1;
    st[m] = s;
  }
  if (!ok) return;
  const int by = b / g.BW, x = 2 * (b % g.BW);
  const unsigned char* p = in + (static_cast<size_t>(m) * g.H + 2 * by) * g.ld + x / 8;
  // pixels x, x + 1 of rows 2 by (bits 0, 1) and 2 by + 1 (bits 2, 3), as the strip kernels' work_word sees them
  const unsigned valid = x + 1 < g.W ? 3u : 1u;
  const unsigned rows = 2 * by + 1 < g.H ? valid | valid << 2 : valid;
  unsigned px = (p[0] >> (x % 8)) & 3u;
  if (2 * by + 1 < g.H) px |= ((p[g.ld] >> (x % 8)) & 3u) << 2;
  px = (holes ? ~px : px) & rows;
  labels[static_cast<size_t>(m) * g.BH * g.BW + b] = px ? b : kBg;
}

// Each block joins its left, top-left, top and top-right neighbours when a pixel pair of the two is 8-adjacent.
__global__ void __launch_bounds__(kThreads)
regions_merge_kernel(const unsigned char* __restrict__ in, Geo g, int holes, int* __restrict__ labels) {
  int m, by, k;
  if (!strip(g, m, by, k)) return;
  const unsigned char* mask = in + static_cast<size_t>(m) * g.H * g.ld;
  const int y0 = 2 * by;
  const uint32_t w0 = work_word(mask, g, y0, k, holes), w1 = work_word(mask, g, y0 + 1, k, holes);
  const uint32_t col = w0 | w1;
  if (!col) return;
  const uint32_t wp = work_word(mask, g, y0 - 1, k, holes);
  const uint32_t lc = (work_word(mask, g, y0, k - 1, holes) | work_word(mask, g, y0 + 1, k - 1, holes)) >> 31;
  const uint32_t lp = work_word(mask, g, y0 - 1, k - 1, holes) >> 31;
  const uint32_t rp = work_word(mask, g, y0 - 1, k + 1, holes) & 1u;
  const uint32_t left = col & ((col << 1) | lc) & kEven;                 // (a | c) and the left block's (b | d)
  const uint32_t top = pairs(w0) & pairs(wp);                           // (a | b) and the top block's (c | d)
  const uint32_t top_left = w0 & ((wp << 1) | lp) & kEven;              // a and the top-left block's d
  const uint32_t top_right = (w0 >> 1) & ((wp >> 2) | (rp << 30)) & kEven;   // b and the top-right block's c
  uint32_t any = left | top | top_left | top_right;
  int* L = labels + static_cast<size_t>(m) * g.BH * g.BW;
  const int b0 = by * g.BW + 16 * k;
  while (any) {
    const int bit = __ffs(any) - 1;
    any &= any - 1;
    const int b = b0 + bit / 2;
    const uint32_t f = 1u << bit;
    if (left & f) unite(L, b, b - 1);
    if (top & f) unite(L, b, b - g.BW);
    if (top_left & f) unite(L, b, b - g.BW - 1);
    if (top_right & f) unite(L, b, b - g.BW + 1);
  }
}

// every block -> its root; roots -> -1.  A block's slot is written by its own thread only, and a chain that meets a
// negative slot has met a root, so finds running concurrently stay correct.
__global__ void __launch_bounds__(kThreads)
regions_compress_kernel(Geo g, int* __restrict__ labels) {
  int m, b;
  if (!block(g, m, b)) return;
  int* L = labels + static_cast<size_t>(m) * g.BH * g.BW;
  int x = __ldcg(L + b);
  if (x == kBg) return;
  if (x == b) {
    L[b] = -1;
    return;
  }
  int p = __ldcg(L + x);
  while (p >= 0 && p != x) {
    x = p;
    p = __ldcg(L + x);
  }
  L[b] = x;
}

// each root's slot -= the pixel count of every block of its component; consecutive blocks of one root add once
__global__ void __launch_bounds__(kThreads)
regions_area_kernel(const unsigned char* __restrict__ in, Geo g, int holes, int* __restrict__ labels) {
  int m, by, k;
  if (!strip(g, m, by, k)) return;
  const unsigned char* mask = in + static_cast<size_t>(m) * g.H * g.ld;
  const uint32_t w0 = work_word(mask, g, 2 * by, k, holes), w1 = work_word(mask, g, 2 * by + 1, k, holes);
  if (!(w0 | w1)) return;
  int* L = labels + static_cast<size_t>(m) * g.BH * g.BW;
  const int b0 = by * g.BW + 16 * k;
  int root = -1, sum = 0;
  for (int j = 0; j < 16; ++j) {
    const int p = __popc((w0 >> (2 * j)) & 3u) + __popc((w1 >> (2 * j)) & 3u);
    if (!p) continue;
    const int b = b0 + j;
    const int v = __ldcg(L + b);                   // a root's own slot is negative (and may be shrinking)
    const int r = v < 0 ? b : v;
    if (r != root) {
      if (sum) atomicSub(L + root, sum);
      root = r;
      sum = 0;
    }
    sum += p;
  }
  if (sum) atomicSub(L + root, sum);
}

__global__ void __launch_bounds__(kThreads)
regions_decide_kernel(Geo g, long long min_area, int islands, const int* __restrict__ labels,
                      MaskState* __restrict__ st) {
  int m, b;
  const bool ok = block(g, m, b);
  bool small = false, large = false;
  unsigned long long best = 0ull;
  const int v = ok ? labels[static_cast<size_t>(m) * g.BH * g.BW + b] : kBg;
  if (v <= -2) {                                   // a root (background is -1, other blocks >= 0)
    const long long area = -1ll - v;
    small = area < min_area;
    large = !small;
    best = static_cast<unsigned long long>(area) << 32 | (0xffffffffu - static_cast<unsigned>(b));
  }
  // a CTA covers one mask: one store / atomic per warp
  const unsigned all = 0xffffffffu;
  small = __any_sync(all, small);
  large = __any_sync(all, large);
#pragma unroll
  for (int o = 16; o > 0; o /= 2) {
    const unsigned long long t = __shfl_xor_sync(all, best, o);
    best = t > best ? t : best;
  }
  if (threadIdx.x % 32 != 0) return;
  MaskState& s = st[m];
  if (small) s.small = 1;                          // every writer stores the same value
  if (large) s.large = 1;
  if (islands && best > __ldcg(&s.best)) atomicMax(&s.best, best);
}

__global__ void __launch_bounds__(kThreads)
regions_write_kernel(const unsigned char* in, unsigned char* out, Geo g, long long min_area, int holes,
                     const int* __restrict__ labels, MaskState* __restrict__ st) {
  int m, by, k;
  const bool ok = strip(g, m, by, k);
  int x_min = INT_MAX, y_min = INT_MAX, x_max = -1, y_max = -1;
  if (ok) {
    const unsigned char* mask = in + static_cast<size_t>(m) * g.H * g.ld;
    const int y0 = 2 * by;
    const uint32_t r0 = raw_word(mask, g, y0, k), r1 = raw_word(mask, g, y0 + 1, k);
    const uint32_t w0 = work_word(mask, g, y0, k, holes), w1 = work_word(mask, g, y0 + 1, k, holes);
    uint32_t o0 = r0, o1 = r1;                     // no small component: the mask stays as it is
    const MaskState& s = st[m];
    if (s.small && (w0 | w1)) {
      const int* L = labels + static_cast<size_t>(m) * g.BH * g.BW;
      const int b0 = by * g.BW + 16 * k;
      const int best_root = static_cast<int>(0xffffffffu - static_cast<unsigned>(s.best & 0xffffffffull));
      const bool fallback = !holes && !s.large;
      uint32_t sel = 0u;
      uint32_t fg = pairs(w0 | w1);
      while (fg) {
        const int bit = __ffs(fg) - 1;
        fg &= fg - 1;
        const int b = b0 + bit / 2;
        const int v = L[b];
        const int r = v < 0 ? b : v;
        const long long area = -1ll - (r == b ? v : L[r]);
        const bool on = holes ? area < min_area : (area >= min_area || (fallback && r == best_root));
        if (on) sel |= 3u << bit;
      }
      o0 = (holes ? r0 : 0u) | (w0 & sel);
      o1 = (holes ? r1 : 0u) | (w1 & sel);
    }
    unsigned char* dst = out + static_cast<size_t>(m) * g.H * g.ld;
    for (int i = 0; i < 2 && y0 + i < g.H; ++i) {
      const uint32_t o = i ? o1 : o0;
      uint16_t* r = reinterpret_cast<uint16_t*>(dst + static_cast<size_t>(y0 + i) * g.ld) + 2 * k;
      r[0] = static_cast<uint16_t>(o);
      if (4 * k + 2 < g.ld) r[1] = static_cast<uint16_t>(o >> 16);
    }
    const uint32_t o = o0 | o1;
    if (o) {
      x_min = 32 * k + __ffs(o) - 1;
      x_max = 32 * k + 31 - __clz(o);
      y_min = o0 ? y0 : y0 + 1;
      y_max = o1 ? y0 + 1 : y0;
    }
  }
  // a CTA covers one mask: reduce per warp, then one atomic per warp and field
  const unsigned all = 0xffffffffu;
  x_min = __reduce_min_sync(all, x_min);
  y_min = __reduce_min_sync(all, y_min);
  x_max = __reduce_max_sync(all, x_max);
  y_max = __reduce_max_sync(all, y_max);
  if (threadIdx.x % 32 == 0 && x_max >= 0) {
    int* box = st[m].box;
    atomicMin(box + 0, x_min);
    atomicMin(box + 1, y_min);
    atomicMax(box + 2, x_max);
    atomicMax(box + 3, y_max);
  }
}

__global__ void regions_finish_kernel(const MaskState* __restrict__ st, int n, unsigned char* __restrict__ changed,
                                      int* __restrict__ boxes) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n) return;
  const MaskState& s = st[m];
  changed[m] = s.small ? 1 : 0;
  const bool empty = s.box[2] < 0;
#pragma unroll
  for (int f = 0; f < 4; ++f) boxes[m * 4 + f] = empty ? 0 : s.box[f];
}

}  // namespace

int mask_small_regions_bits(const unsigned char* in, unsigned char* out, int n, int H, int W, int ld,
                            long long min_area, int mode, void* ws, unsigned char* changed, int* boxes,
                            cudaStream_t stream) {
  RSP_CHECK_ARG(in && out && ws && changed && boxes && n > 0 && H > 0 && W > 0 &&
                static_cast<long long>(H) * W <= INT_MAX && (mode == 0 || mode == 1),
                "mask_small_regions_bits: bad args (n, H, W > 0, H * W < 2^31, mode 0 = holes or 1 = islands)");
  Geo g;
  g.H = H;
  g.W = W;
  g.ld = ld;
  g.BH = (H + 1) / 2;
  g.BW = (W + 1) / 2;
  g.KW = (W + 31) / 32;
  const long long strips = static_cast<long long>(g.BH) * g.KW;
  g.cpm = static_cast<int>((strips + kThreads - 1) / kThreads);
  const long long blocks = static_cast<long long>(g.BH) * g.BW;
  g.cpb = static_cast<int>((blocks + kThreads - 1) / kThreads);
  RSP_CHECK_ARG(ld % 2 == 0 && 8ll * ld >= W && ld <= 4 * g.KW, "mask_small_regions_bits: row bytes ld=%d for W=%d "
                "must be even, hold W bits and be at most 4 * ceil(W / 32)", ld, W);
  RSP_CHECK_ARG(reinterpret_cast<uintptr_t>(in) % 2 == 0 && reinterpret_cast<uintptr_t>(out) % 2 == 0 &&
                reinterpret_cast<uintptr_t>(ws) % 8 == 0,
                "mask_small_regions_bits: in / out must be 2-byte aligned, ws 8-byte aligned");
  RSP_CHECK_ARG(static_cast<long long>(n) * g.cpb <= INT_MAX, "mask_small_regions_bits: too many masks per launch");
  MaskState* st = static_cast<MaskState*>(ws);
  int* labels = reinterpret_cast<int*>(st + n);
  const unsigned grid = static_cast<unsigned>(n) * g.cpm, grid_b = static_cast<unsigned>(n) * g.cpb;
  const int holes = mode == 0;
  regions_init_kernel<<<grid_b, kThreads, 0, stream>>>(in, g, holes, labels, st);
  RSP_CHECK_LAUNCH();
  regions_merge_kernel<<<grid, kThreads, 0, stream>>>(in, g, holes, labels);
  RSP_CHECK_LAUNCH();
  regions_compress_kernel<<<grid_b, kThreads, 0, stream>>>(g, labels);
  RSP_CHECK_LAUNCH();
  regions_area_kernel<<<grid, kThreads, 0, stream>>>(in, g, holes, labels);
  RSP_CHECK_LAUNCH();
  regions_decide_kernel<<<grid_b, kThreads, 0, stream>>>(g, min_area, !holes, labels, st);
  RSP_CHECK_LAUNCH();
  regions_write_kernel<<<grid, kThreads, 0, stream>>>(in, out, g, min_area, holes, labels, st);
  RSP_CHECK_LAUNCH();
  regions_finish_kernel<<<(n + 255) / 256, 256, 0, stream>>>(st, n, changed, boxes);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace rsp
