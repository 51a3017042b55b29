// Mask borders as polygons on the device: cv2.findContours(mask, RETR_CCOMP, CHAIN_APPROX_NONE | CHAIN_APPROX_SIMPLE),
// the call mmdet.structures.mask.bitmap_to_polygon makes (mmdet/structures/mask/structures.py:1166-1194) per mask on
// the host.  oracle/restate_contours.py restates the same construction in Python and is checked against cv2.
//
// cv2 finds borders by a sequential raster scan (Suzuki and Abe).  Its result is a function of the connected
// components, which lets every border be found and followed independently:
//   - one outer border per 8-connected foreground component, starting at the component's first pixel in raster order;
//   - one hole border per 4-connected background component that does not reach the image edge (everything outside the
//     image is background), starting at the left neighbour of the hole's first pixel, whose outer border is its parent;
//   - list order: outer borders by descending start, each followed by its holes by descending start.
//
// Canvas i (the OR of its K placed parts, as rsp_mask_rle_union_* reads them) is formed only inside the rectangle
// bounding its parts, plus a one-pixel zero border: the "padded rectangle" of Hp x Wp pixels, indexed in raster order.
// Stages, all over the workspace:
//   form       bits = the union's pixels, labels = own index, aux = 0
//   merge      union-find toward the smaller index (foreground over 8 neighbours, background over 4), so every
//              component's root is its first pixel in raster order
//   compress   labels = root
//   enumerate  one CTA per canvas, in descending raster order: a hole's rank among its parent's holes goes to aux at
//              the hole's root and the parent's hole count accumulates in aux at the parent's root; at the parent's
//              root that count becomes the parent's list index (a scan of 1 + holes over the outer borders)
//   walk       one thread per border start: cv2's border following (icvFetchContour), counting its points; the count
//              and the start go to the canvas's contour slots, indexed by list position
//   scan       per canvas, the counts -> offsets in place and the canvas's point total; then the canvas totals
// The write pass follows each border again, one thread per contour.  Atomics touch intermediate values only (labels
// and hole counts, whose final values do not depend on the order of the updates): two calls give identical bytes.
#include <climits>
#include <vector>

#include <cub/block/block_scan.cuh>

#include "contours.h"

namespace rsp {
namespace {

constexpr int kThreads = 256;
constexpr int kEnumThreads = 512;
constexpr int kEnumWarps = kEnumThreads / 32;
constexpr int kMaxBlocksPerCanvas = 1024;

// per canvas, at the front of the workspace
struct CanvasHdr {
  long long pix;     // first pixel of its padded rectangle in the pixel arrays
  int Hp, Wp;        // padded rectangle
  int ry0, rx0;      // canvas position of the rectangle's first unpadded pixel
  int ncont;         // contours
  int pad_;
  long long npts;    // points
};
static_assert(sizeof(CanvasHdr) == 40, "header layout");

struct Ws {
  CanvasHdr* hdr;
  unsigned char* bits;   // [T] 0 / 1
  int* labels;           // [T]
  int* aux;              // [T]
  int* cnt;              // [T] per contour slot: point count, then offset within the canvas
  int* start;            // [T] per contour slot: start pixel, -1 - start for a hole
};

long long align256(long long v) { return (v + 255) / 256 * 256; }

// the workspace carved from its base for n canvases of T pixels in all (the same arithmetic on host and device)
__host__ __device__ Ws carve(void* base, int n, long long T) {
  char* p = static_cast<char*>(base);
  Ws w;
  w.hdr = reinterpret_cast<CanvasHdr*>(p);
  long long off = ((static_cast<long long>(n) * static_cast<long long>(sizeof(CanvasHdr))) + 255) / 256 * 256;
  w.bits = reinterpret_cast<unsigned char*>(p + off);
  off += (T + 255) / 256 * 256;
  w.labels = reinterpret_cast<int*>(p + off);
  off += 4 * T;
  w.aux = reinterpret_cast<int*>(p + off);
  off += 4 * T;
  w.cnt = reinterpret_cast<int*>(p + off);
  off += 4 * T;
  w.start = reinterpret_cast<int*>(p + off);
  return w;
}

long long ws_total(int n, long long T) {
  return align256(static_cast<long long>(n) * static_cast<long long>(sizeof(CanvasHdr))) + align256(T) + 16 * T;
}

// One pixel per thread over each canvas: blockIdx.x = canvas * bpc + block within it.
template <typename F>
__device__ __forceinline__ void for_each_pixel(const CanvasHdr* hdr, int bpc, F&& f) {
  const int i = static_cast<int>(blockIdx.x / bpc);
  const CanvasHdr h = hdr[i];
  const int np = h.Hp * h.Wp;
  for (int p = static_cast<int>(blockIdx.x % bpc) * kThreads + static_cast<int>(threadIdx.x); p < np;
       p += bpc * kThreads)
    f(h, p);
}

__global__ void __launch_bounds__(kThreads) contour_form_kernel(const unsigned char* __restrict__ src,
                                                                const long long* __restrict__ desc,
                                                                const long long* __restrict__ parts, Ws ws, int bpc) {
  const int i = static_cast<int>(blockIdx.x / bpc);
  const long long* pp = parts + 7 * __ldg(desc + 4 * i + 2);
  const int k = static_cast<int>(__ldg(desc + 4 * i + 3));
  for_each_pixel(ws.hdr, bpc, [&](const CanvasHdr& h, int p) {
    const int py = p / h.Wp, px = p - py * h.Wp;
    unsigned v = 0u;
    if (py > 0 && px > 0 && py < h.Hp - 1 && px < h.Wp - 1) {
      const int cy = h.ry0 + py - 1, cx = h.rx0 + px - 1;
#pragma unroll 1
      for (int q = 0; q < k && !v; ++q) {
        const long long* d = pp + 7 * q;
        const int y0 = static_cast<int>(__ldg(d + 5)), x0 = static_cast<int>(__ldg(d + 6));
        const int y = cy - y0, x = cx - x0;
        if (y < 0 || x < 0 || y >= static_cast<int>(__ldg(d + 3)) || x >= static_cast<int>(__ldg(d + 4))) continue;
        v = (__ldg(src + __ldg(d) + static_cast<long long>(y) * __ldg(d + 1) + (x >> 3)) >> (x & 7)) & 1u;
      }
    }
    ws.bits[h.pix + p] = static_cast<unsigned char>(v);
    ws.labels[h.pix + p] = p;
    ws.aux[h.pix + p] = 0;
  });
}

// The root of x, halving the path on the way (each visited pixel is pointed at its grandparent).  Labels only ever
// decrease and stay within the component, so the halving may race with unions; without it a one-pixel-wide path
// (a serpentine, a diagonal line) builds chains as long as itself and every union walks them.
__device__ __forceinline__ int find_root(int* L, int x) {
  for (;;) {
    const int y = L[x];
    if (y == x) return x;
    const int z = L[y];
    if (z == y) return y;
    atomicMin(L + x, z);
    x = z;
  }
}

// link the two roots, the larger to the smaller (Playne and Hawick's lock-free union)
__device__ __forceinline__ void unite(int* L, int a, int b) {
  for (;;) {
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
    b = old;
  }
}

__global__ void __launch_bounds__(kThreads) contour_merge_kernel(Ws ws, int bpc) {
  for_each_pixel(ws.hdr, bpc, [&](const CanvasHdr& h, int p) {
    const unsigned char* b = ws.bits + h.pix;
    int* L = ws.labels + h.pix;
    const int py = p / h.Wp, px = p - py * h.Wp;
    const unsigned char v = b[p];
    if (px > 0 && b[p - 1] == v) unite(L, p, p - 1);
    if (py > 0) {
      const int up = p - h.Wp;
      if (b[up] == v) unite(L, p, up);
      if (v) {   // foreground: the diagonal neighbours above too
        if (px > 0 && b[up - 1]) unite(L, p, up - 1);
        if (px < h.Wp - 1 && b[up + 1]) unite(L, p, up + 1);
      }
    }
  });
}

__global__ void __launch_bounds__(kThreads) contour_compress_kernel(Ws ws, int bpc) {
  for_each_pixel(ws.hdr, bpc, [&](const CanvasHdr& h, int p) {
    int* L = ws.labels + h.pix;
    L[p] = find_root(L, p);
  });
}

// hole root: a background pixel that is its component's first, except the outside's (pixel 0)
__device__ __forceinline__ bool is_hole_root(const unsigned char* b, const int* L, int p) {
  return p > 0 && !b[p] && L[p] == p;
}

__device__ __forceinline__ bool is_outer_root(const unsigned char* b, const int* L, int p) {
  return b[p] && L[p] == p;
}

// One CTA per canvas, tiles of kEnumThreads pixels in descending raster order (thread t takes pixel hi - t).  Every
// hole of an outer border lies after the border's start, so by the time the scan reaches the start its hole count is
// final.  Holes take their rank one warp at a time so that ranks follow descending order within the tile.
__global__ void __launch_bounds__(kEnumThreads) contour_enumerate_kernel(Ws ws) {
  using Scan = cub::BlockScan<int, kEnumThreads, cub::BLOCK_SCAN_WARP_SCANS>;
  __shared__ typename Scan::TempStorage tmp;
  CanvasHdr* hdr = ws.hdr + blockIdx.x;
  const long long pix = hdr->pix;
  const int np = hdr->Hp * hdr->Wp;
  const unsigned char* b = ws.bits + pix;
  const int* L = ws.labels + pix;
  int* aux = ws.aux + pix;
  const int warp = static_cast<int>(threadIdx.x) / 32, lane = static_cast<int>(threadIdx.x) % 32;
  int carry = 0;
  for (int hi = np - 1; hi >= 0; hi -= kEnumThreads) {
    const int p = hi - static_cast<int>(threadIdx.x);
    const bool hole = p >= 0 && is_hole_root(b, L, p);
    const bool outer = p >= 0 && is_outer_root(b, L, p);
    if (__syncthreads_or(hole)) {
      const int parent = hole ? L[p - 1] : -1;
      const unsigned same = __match_any_sync(0xffffffffu, parent);
      for (int w = 0; w < kEnumWarps; ++w) {
        if (w == warp && hole) {
          const int before = __popc(same & ((1u << lane) - 1u));
          aux[p] = aux[parent] + before;
          __syncwarp(same);
          if (before == 0) aux[parent] += __popc(same);   // the group's first lane updates the count
        }
        __syncthreads();
      }
    }
    const int v = outer ? 1 + aux[p] : 0;
    int pos, total;
    Scan(tmp).ExclusiveSum(v, pos, total);
    if (outer) aux[p] = carry + pos;
    carry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) hdr->ncont = carry;
}

// cv2's border following (imgproc contours.cpp icvFetchContour) from pixel p0 of a padded rectangle of width Wp,
// calling emit(x, y) (padded coordinates) for every point it outputs; returns the number of points.  Direction s =
// 0 .. 7 is right, up-right, up, up-left, left, down-left, down, down-right.  The first neighbour is searched
// clockwise from the background pixel (left of an outer border's start, right of a hole's), every later one
// counter-clockwise from the direction after the one the walk came in by.  CHAIN_APPROX_SIMPLE (simple = true) keeps
// a point only where the direction out of it differs from the previous move.
template <typename E>
__device__ __forceinline__ int follow(const unsigned char* __restrict__ b, int Wp, int p0, bool hole, bool simple,
                                      E&& emit) {
  // dx, dy + 1 of direction s in nibble s (no local arrays)
  const auto dx = [](int s) { return static_cast<int>((0x21000122u >> (4 * s)) & 0xfu) - 1; };
  const auto dy = [](int s) { return static_cast<int>((0x22210001u >> (4 * s)) & 0xfu) - 1; };
  const int y0 = p0 / Wp, x0 = p0 - y0 * Wp;
  const int s_end0 = hole ? 0 : 4;
  int s = s_end0, p1;
  do {
    s = (s - 1) & 7;
    p1 = p0 + dy(s) * Wp + dx(s);
  } while (!b[p1] && s != s_end0);
  if (s == s_end0) {   // an isolated pixel
    emit(x0, y0);
    return 1;
  }
  int n = 0, prev_s = s ^ 4, p3 = p0, x = x0, y = y0;
  for (;;) {
    int p4;
    do {
      s = (s + 1) & 7;
      p4 = p3 + dy(s) * Wp + dx(s);
    } while (!b[p4]);
    if (!simple || s != prev_s) {
      emit(x, y);
      ++n;
      prev_s = s;
    }
    x += dx(s);
    y += dy(s);
    if (p4 == p0 && p3 == p1) break;
    p3 = p4;
    s = (s + 4) & 7;
  }
  return n;
}

// One thread per pixel; border starts count their points into their list slot.
__global__ void __launch_bounds__(kThreads) contour_walk_length_kernel(Ws ws, int bpc, int simple) {
  for_each_pixel(ws.hdr, bpc, [&](const CanvasHdr& h, int p) {
    const unsigned char* b = ws.bits + h.pix;
    const int* L = ws.labels + h.pix;
    const int* aux = ws.aux + h.pix;
    int slot, p0;
    bool hole;
    if (is_outer_root(b, L, p)) {
      slot = aux[p];
      p0 = p;
      hole = false;
    } else if (is_hole_root(b, L, p)) {
      p0 = p - 1;
      slot = aux[L[p0]] + 1 + aux[p];
      hole = true;
    } else {
      return;
    }
    ws.cnt[h.pix + slot] = follow(b, h.Wp, p0, hole, simple != 0, [](int, int) {});
    ws.start[h.pix + slot] = hole ? -1 - p0 : p0;
  });
}

// One CTA per canvas: its contours' point counts -> exclusive offsets in place, the total into the header.
__global__ void __launch_bounds__(kEnumThreads) contour_canvas_scan_kernel(Ws ws) {
  using Scan = cub::BlockScan<long long, kEnumThreads, cub::BLOCK_SCAN_WARP_SCANS>;
  __shared__ typename Scan::TempStorage tmp;
  CanvasHdr* hdr = ws.hdr + blockIdx.x;
  int* cnt = ws.cnt + hdr->pix;
  const int nc = hdr->ncont;
  long long carry = 0;
  for (int k0 = 0; k0 < nc; k0 += kEnumThreads) {
    const int k = k0 + static_cast<int>(threadIdx.x);
    const long long v = k < nc ? cnt[k] : 0;
    long long off, total;
    Scan(tmp).ExclusiveSum(v, off, total);
    if (k < nc) cnt[k] = static_cast<int>(carry + off);   // wraps only past 2^31 - 1 points, rejected below
    carry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) hdr->npts = carry;
}

// contour_offsets / point_offsets [n + 1]: exclusive sums of the canvases' contour and point counts
__global__ void __launch_bounds__(kThreads) contour_offsets_kernel(const Ws ws, int n, long long* contour_offsets,
                                                                   long long* point_offsets) {
  using Scan = cub::BlockScan<long long, kThreads, cub::BLOCK_SCAN_WARP_SCANS>;
  __shared__ typename Scan::TempStorage tmp[2];
  long long cc = 0, pc = 0;
  for (int i0 = 0; i0 < n; i0 += kThreads) {
    const int i = i0 + static_cast<int>(threadIdx.x);
    const long long c = i < n ? ws.hdr[i].ncont : 0;
    // a canvas of 2^31 points or more (its offsets are int32) makes the total negative: the caller reports it
    const long long p = i >= n ? 0 : ws.hdr[i].npts <= INT_MAX ? ws.hdr[i].npts : LLONG_MIN / 4;
    long long co, ct, po, pt;
    Scan(tmp[0]).ExclusiveSum(c, co, ct);
    Scan(tmp[1]).ExclusiveSum(p, po, pt);
    if (i < n) {
      contour_offsets[i] = cc + co;
      point_offsets[i] = pc + po;
    }
    cc += ct;
    pc += pt;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    contour_offsets[n] = cc;
    point_offsets[n] = pc;
  }
}

// One thread per contour c of all canvases: its point offset, parent and points.
__global__ void __launch_bounds__(kThreads) contour_write_kernel(const Ws ws, int n, long long num_contours,
                                                                 const long long* __restrict__ contour_offsets,
                                                                 const long long* __restrict__ canvas_points,
                                                                 int* __restrict__ points,
                                                                 long long* __restrict__ point_offsets,
                                                                 int* __restrict__ parents, int simple) {
  const long long c = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x;
  if (c == 0) point_offsets[num_contours] = canvas_points[n];
  if (c >= num_contours) return;
  int lo = 0, hi = n - 1;   // the canvas: the last i with contour_offsets[i] <= c
  while (lo < hi) {
    const int mid = (lo + hi + 1) / 2;
    if (contour_offsets[mid] <= c) lo = mid;
    else hi = mid - 1;
  }
  const int i = lo;
  const CanvasHdr h = ws.hdr[i];
  const int k = static_cast<int>(c - contour_offsets[i]);
  const int* cnt = ws.cnt + h.pix;
  const long long first = canvas_points[i] + cnt[k];
  const long long end = k + 1 < h.ncont ? canvas_points[i] + cnt[k + 1] : canvas_points[i + 1];
  point_offsets[c] = first;
  const int s = ws.start[h.pix + k];
  const bool hole = s < 0;
  const int p0 = hole ? -1 - s : s;
  parents[c] = hole ? ws.aux[h.pix + ws.labels[h.pix + p0]] : -1;
  int2* out = reinterpret_cast<int2*>(points) + first;
  const int n_out = static_cast<int>(end - first);
  int j = 0;
  const int ox = h.rx0 - 1, oy = h.ry0 - 1;
  follow(ws.bits + h.pix, h.Wp, p0, hole, simple != 0, [&](int x, int y) {
    if (j < n_out) out[j] = make_int2(ox + x, oy + y);
    ++j;
  });
}

// The padded rectangle of canvas i from its parts' host descriptors, every descriptor checked as in
// mask_rle_union_lengths.  -> pixels, or -1 with the error set.
int canvas_rect(const char* what, const long long* desc_host, int i, const long long* parts_host, int num_parts,
                CanvasHdr* out) {
  const long long H = desc_host[4 * i], W = desc_host[4 * i + 1], first = desc_host[4 * i + 2], k = desc_host[4 * i + 3];
  RSP_CHECK_ARG(H >= 1 && W >= 1 && H <= INT_MAX && W <= INT_MAX && H * W <= INT_MAX,
                "%s: mask %d: canvas %lld x %lld (1 .. 2^31 - 1 pixels)", what, i, H, W);
  RSP_CHECK_ARG(first >= 0 && k >= 1 && k <= num_parts - first,
                "%s: mask %d: parts [%lld, %lld + %lld) outside the %d parts", what, i, first, first, k, num_parts);
  long long y0 = LLONG_MAX, x0 = LLONG_MAX, y1 = 0, x1 = 0;
  for (long long p = first; p < first + k; ++p) {
    const long long* d = parts_host + 7 * p;
    const long long off = d[0], ld = d[1], rows = d[2], h = d[3], w = d[4], py = d[5], px = d[6];
    RSP_CHECK_ARG(py >= 0 && px >= 0 && py < H && px < W,
                  "%s: mask %d, part %lld: origin (%lld, %lld) outside the %lld x %lld canvas", what, i, p, py, px, H,
                  W);
    RSP_CHECK_ARG(h >= 1 && w >= 1 && h <= H - py && w <= W - px,
                  "%s: mask %d, part %lld: %lld x %lld at (%lld, %lld) leaves the %lld x %lld canvas", what, i, p, h, w,
                  py, px, H, W);
    RSP_CHECK_ARG(off >= 0 && ld <= INT_MAX && h <= rows && w <= 8 * ld,
                  "%s: mask %d, part %lld: visible %lld x %lld exceeds the source (%lld rows of %lld bytes, offset "
                  "%lld)", what, i, p, h, w, rows, ld, off);
    y0 = py < y0 ? py : y0;
    x0 = px < x0 ? px : x0;
    y1 = py + h > y1 ? py + h : y1;
    x1 = px + w > x1 ? px + w : x1;
  }
  const long long Hp = y1 - y0 + 2, Wp = x1 - x0 + 2;
  RSP_CHECK_ARG(Hp * Wp <= INT_MAX, "%s: mask %d: the parts' rectangle %lld x %lld with its border exceeds 2^31 - 1 "
                "pixels", what, i, Hp - 2, Wp - 2);
  *out = CanvasHdr{0, static_cast<int>(Hp), static_cast<int>(Wp), static_cast<int>(y0), static_cast<int>(x0), 0, 0, 0};
  return RSP_OK;
}

// every canvas's header and the total pixel count; the largest rectangle sets the blocks per canvas
int layout(const char* what, const long long* desc_host, int n, const long long* parts_host, int num_parts,
           std::vector<CanvasHdr>& hdr, long long& T, int& bpc) {
  RSP_CHECK_ARG(desc_host && parts_host && n > 0 && num_parts > 0, "%s: bad args", what);
  hdr.resize(n);
  T = 0;
  long long most = 0;
  for (int i = 0; i < n; ++i) {
    RSP_TRY(canvas_rect(what, desc_host, i, parts_host, num_parts, &hdr[i]));
    hdr[i].pix = T;
    const long long np = static_cast<long long>(hdr[i].Hp) * hdr[i].Wp;
    T += np;
    most = np > most ? np : most;
  }
  const long long blocks = (most + kThreads - 1) / kThreads;
  bpc = static_cast<int>(blocks < kMaxBlocksPerCanvas ? blocks : kMaxBlocksPerCanvas);
  RSP_CHECK_ARG(static_cast<long long>(n) * bpc <= INT_MAX, "%s: %d canvases are too many for one call", what, n);
  return RSP_OK;
}

}  // namespace

int mask_contours_ws_bytes(const long long* desc_host, int n, const long long* parts_host, int num_parts,
                           long long* bytes) {
  RSP_CHECK_ARG(bytes, "mask_contours_ws_bytes: bad args");
  std::vector<CanvasHdr> hdr;
  long long T;
  int bpc;
  RSP_TRY(layout("mask_contours_ws_bytes", desc_host, n, parts_host, num_parts, hdr, T, bpc));
  *bytes = ws_total(n, T);
  return RSP_OK;
}

int mask_contours_lengths(const unsigned char* src, const long long* desc, const long long* desc_host, int n,
                          const long long* parts, const long long* parts_host, int num_parts, int approx, void* ws,
                          long long ws_bytes, long long* contour_offsets, long long* point_offsets,
                          cudaStream_t stream) {
  const char* what = "mask_contours_lengths";
  RSP_CHECK_ARG(src && desc && parts && ws && contour_offsets && point_offsets, "%s: bad args", what);
  RSP_CHECK_ARG(approx == kChainApproxNone || approx == kChainApproxSimple,
                "%s: approx %d (1 = CHAIN_APPROX_NONE, 2 = CHAIN_APPROX_SIMPLE)", what, approx);
  std::vector<CanvasHdr> hdr;
  long long T;
  int bpc;
  RSP_TRY(layout(what, desc_host, n, parts_host, num_parts, hdr, T, bpc));
  const long long need = ws_total(n, T);
  RSP_CHECK_ARG(ws_bytes >= need, "%s: workspace of %lld bytes, %lld needed", what, ws_bytes, need);
  const Ws w = carve(ws, n, T);
  RSP_CHECK_CUDA(cudaMemcpyAsync(w.hdr, hdr.data(), sizeof(CanvasHdr) * n, cudaMemcpyHostToDevice, stream));
  const int grid = n * bpc;
  contour_form_kernel<<<grid, kThreads, 0, stream>>>(src, desc, parts, w, bpc);
  RSP_CHECK_LAUNCH();
  contour_merge_kernel<<<grid, kThreads, 0, stream>>>(w, bpc);
  RSP_CHECK_LAUNCH();
  contour_compress_kernel<<<grid, kThreads, 0, stream>>>(w, bpc);
  RSP_CHECK_LAUNCH();
  contour_enumerate_kernel<<<n, kEnumThreads, 0, stream>>>(w);
  RSP_CHECK_LAUNCH();
  contour_walk_length_kernel<<<grid, kThreads, 0, stream>>>(w, bpc, approx == kChainApproxSimple);
  RSP_CHECK_LAUNCH();
  contour_canvas_scan_kernel<<<n, kEnumThreads, 0, stream>>>(w);
  RSP_CHECK_LAUNCH();
  contour_offsets_kernel<<<1, kThreads, 0, stream>>>(w, n, contour_offsets, point_offsets);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

int mask_contours_write(const long long* desc_host, int n, const long long* parts_host, int num_parts, int approx,
                        const void* ws, long long ws_bytes, const long long* contour_offsets,
                        const long long* canvas_points, long long num_contours, int* points, long long* point_offsets,
                        int* parents, cudaStream_t stream) {
  const char* what = "mask_contours_write";
  RSP_CHECK_ARG(ws && contour_offsets && canvas_points && point_offsets && num_contours >= 0 &&
                (num_contours == 0 || (points && parents)), "%s: bad args", what);
  RSP_CHECK_ARG(approx == kChainApproxNone || approx == kChainApproxSimple,
                "%s: approx %d (1 = CHAIN_APPROX_NONE, 2 = CHAIN_APPROX_SIMPLE)", what, approx);
  std::vector<CanvasHdr> hdr;
  long long T;
  int bpc;
  RSP_TRY(layout(what, desc_host, n, parts_host, num_parts, hdr, T, bpc));
  const long long need = ws_total(n, T);
  RSP_CHECK_ARG(ws_bytes >= need, "%s: workspace of %lld bytes, %lld needed", what, ws_bytes, need);
  const Ws w = carve(const_cast<void*>(ws), n, T);
  const long long blocks = num_contours / kThreads + 1;   // at least one: it writes point_offsets[num_contours]
  RSP_CHECK_ARG(blocks <= INT_MAX, "%s: %lld contours are too many for one call", what, num_contours);
  contour_write_kernel<<<static_cast<int>(blocks), kThreads, 0, stream>>>(
      w, n, num_contours, contour_offsets, canvas_points, points, point_offsets, parents,
      approx == kChainApproxSimple);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace rsp
