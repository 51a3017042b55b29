// Small-sequence attention pieces of SAM's two-way mask decoder (HF modeling_sam.py
// SamAttention :231-270 as used by SamTwoWayAttentionBlock :306-348).  The heavy image-token
// projections run on the wgmma GEMM; what is left has 10 prompt tokens on one side, far
// below a tensor-core tile, so these are CUDA-core kernels organised for coalesced HBM
// access (the image-token matrices they stream are the dominant cost).
//
//   token_self_attention   tokens attend to tokens            (T <= 16, 8 heads x 32)
//   t2i_attention          tokens (Tq <= 16) attend to the HW image tokens of their image
//   i2t_attention          every image token attends to the Tq prompt tokens
//   add_cast_bf16          out = bf16(a + b)  (query + point embedding before a projection)
#include "decoder.h"
#include "sm90.cuh"

namespace rsp {

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&w[j]);
    f[2 * j] = __bfloat162float(h.x);
    f[2 * j + 1] = __bfloat162float(h.y);
  }
}

// ---------------------------------------------------------------------------------------
__global__ void add_cast_bf16_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                     __nv_bfloat16* __restrict__ out, long long n, long long b_mod) {
  const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i >= n) return;
  float4 x = *reinterpret_cast<const float4*>(a + i);
  if (b) {
    const float4 y = *reinterpret_cast<const float4*>(b + (b_mod > 0 ? i % b_mod : i));
    x.x += y.x; x.y += y.y; x.z += y.z; x.w += y.w;
  }
  *reinterpret_cast<uint2*>(out + i) = make_uint2(pack_bf16x2(x.x, x.y), pack_bf16x2(x.z, x.w));
}

int add_cast_bf16(const float* a, const float* b, void* out, long long n, long long b_mod,
                  cudaStream_t stream) {
  RSP_CHECK_ARG(a && out && n > 0 && n % 4 == 0 && (b_mod == 0 || b_mod % 4 == 0), "add_cast: bad args");
  const long long n4 = n / 4;
  add_cast_bf16_kernel<<<static_cast<unsigned>((n4 + 255) / 256), 256, 0, stream>>>(
      a, b, static_cast<__nv_bfloat16*>(out), n, b_mod);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// One warp per (prompt, head); lane i < T owns query i.  q/k/v bf16 [N, T, heads*c].
template <int C>
__global__ void token_self_attention_kernel(const __nv_bfloat16* __restrict__ q,
                                            const __nv_bfloat16* __restrict__ k,
                                            const __nv_bfloat16* __restrict__ v,
                                            __nv_bfloat16* __restrict__ out, int N, int T, int heads,
                                            float scale) {
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= N * heads) return;
  const int n = gw / heads, h = gw % heads;
  const int D = heads * C;
  if (lane >= T) return;
  const __nv_bfloat16* qp = q + (static_cast<size_t>(n) * T + lane) * D + h * C;
  float qf[C];
#pragma unroll
  for (int d = 0; d < C; d += 8) {
    float t[8];
    unpack8(*reinterpret_cast<const uint4*>(qp + d), t);
#pragma unroll
    for (int j = 0; j < 8; ++j) qf[d + j] = t[j];
  }
  float s[16];
  float mx = -INFINITY;
  for (int j = 0; j < T; ++j) {
    const __nv_bfloat16* kp = k + (static_cast<size_t>(n) * T + j) * D + h * C;
    float acc = 0.f;
#pragma unroll
    for (int d = 0; d < C; d += 8) {
      float t[8];
      unpack8(*reinterpret_cast<const uint4*>(kp + d), t);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) acc += qf[d + jj] * t[jj];
    }
    s[j] = acc * scale;
    mx = fmaxf(mx, s[j]);
  }
  float l = 0.f;
  float o[C];
#pragma unroll
  for (int d = 0; d < C; ++d) o[d] = 0.f;
  for (int j = 0; j < T; ++j) {
    const float pj = __expf(s[j] - mx);
    l += pj;
    const __nv_bfloat16* vp = v + (static_cast<size_t>(n) * T + j) * D + h * C;
#pragma unroll
    for (int d = 0; d < C; d += 8) {
      float t[8];
      unpack8(*reinterpret_cast<const uint4*>(vp + d), t);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) o[d + jj] += pj * t[jj];
    }
  }
  const float inv = 1.0f / l;
  __nv_bfloat16* op = out + (static_cast<size_t>(n) * T + lane) * D + h * C;
#pragma unroll
  for (int d = 0; d < C; d += 8)
    *reinterpret_cast<uint4*>(op + d) =
        make_uint4(pack_bf16x2(o[d] * inv, o[d + 1] * inv), pack_bf16x2(o[d + 2] * inv, o[d + 3] * inv),
                   pack_bf16x2(o[d + 4] * inv, o[d + 5] * inv), pack_bf16x2(o[d + 6] * inv, o[d + 7] * inv));
}

int token_self_attention(const void* q, const void* k, const void* v, void* out, int N, int T,
                         int heads, int c, cudaStream_t stream) {
  RSP_CHECK_ARG(q && k && v && out && N > 0 && T > 0 && T <= 16 && heads > 0, "token_self_attention: bad args");
  RSP_CHECK_ARG(c == 32 || c == 16, "token_self_attention: per-head dim %d (16 or 32)", c);
  const int warps = N * heads;
  const int threads = 128;
  const int blocks = (warps * 32 + threads - 1) / threads;
  const float scale = 1.0f / sqrtf(static_cast<float>(c));
  if (c == 32)
    token_self_attention_kernel<32><<<blocks, threads, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k),
        static_cast<const __nv_bfloat16*>(v), static_cast<__nv_bfloat16*>(out), N, T, heads, scale);
  else
    token_self_attention_kernel<16><<<blocks, threads, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k),
        static_cast<const __nv_bfloat16*>(v), static_cast<__nv_bfloat16*>(out), N, T, heads, scale);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// t2i: CTA = one prompt, warp = one head.  K / V tiles of 64 image tokens x 128 channels are staged
// in smem with cp.async (double buffered, rows padded to 272 B so the fragment loads are
// conflict-free); S = Q K^T and O += P V run on mma.sync m16n8k16 (bf16 -> fp32): the 10 prompt
// tokens are the M dimension padded to 16, far too few rows for a wgmma tile, but enough to keep
// this kernel on the K / V byte stream (2 MB per prompt) instead of on CUDA-core FMAs.
constexpr int T2I_TILE = 64;
constexpr int T2I_ROWB = 272;  // bytes per staged row (256 + 16 pad)
constexpr int T2I_STAGE = 2 * T2I_TILE * T2I_ROWB;   // K + V of one tile

__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

// Per-warp state of one (prompt, head) of t2i: the pre-scaled Q fragment and the online-softmax accumulators of
// rows g and g + 8 (g = lane / 4).  t2i_attention and t2i_fused run the same three steps below, so for the same
// K / V bytes they produce the same output bytes.
struct T2iHead {
  uint32_t qa[4];
  float m0, m1, l0, l1;
  float o[2][4];
};

// Q fragment (A operand, rows = prompt tokens padded to 16, k = the head's 16 channels), pre-scaled
__device__ __forceinline__ void t2i_head_init(T2iHead& st, const __nv_bfloat16* __restrict__ q, int n, int Tq, int h,
                                              float scale) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  auto ldq = [&](int row, int col) -> uint32_t {
    if (row >= Tq) return 0u;
    const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(
        q + (static_cast<size_t>(n) * Tq + row) * 128 + h * 16 + col);
    return pack_bf16x2(__bfloat162float(v.x) * scale, __bfloat162float(v.y) * scale);
  };
  st.qa[0] = ldq(g, 2 * t); st.qa[1] = ldq(g + 8, 2 * t); st.qa[2] = ldq(g, 2 * t + 8); st.qa[3] = ldq(g + 8, 2 * t + 8);
  st.m0 = -INFINITY; st.m1 = -INFINITY; st.l0 = 0.f; st.l1 = 0.f;
#pragma unroll
  for (int d = 0; d < 2; ++d) st.o[d][0] = st.o[d][1] = st.o[d][2] = st.o[d][3] = 0.f;
}

// One tile of 64 keys: sK / sV = this head's 32-byte column slice of the staged K / V tiles (rows T2I_ROWB apart),
// valid = how many of the 64 keys exist (the rest are masked out of the softmax).
__device__ __forceinline__ void t2i_head_tile(T2iHead& st, uint32_t sK, uint32_t sV, int valid) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  float& m0 = st.m0; float& m1 = st.m1; float& l0 = st.l0; float& l1 = st.l1;
  float (&o)[2][4] = st.o;
  const uint32_t (&qa)[4] = st.qa;
  // ---- S = Q K^T for the 64 keys of the tile (8 n-tiles of 8 keys)
  float s[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    uint32_t b0, b1;
    const uint32_t addr = sK + (j * 8 + g) * T2I_ROWB + t * 4;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(b0) : "r"(addr));
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(b1) : "r"(addr + 16));
    s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
    mma_bf16_16816(s[j], qa, b0, b1);
    if (valid < T2I_TILE) {
      const int key = j * 8 + 2 * t;
      if (key >= valid) { s[j][0] = -INFINITY; s[j][2] = -INFINITY; }
      if (key + 1 >= valid) { s[j][1] = -INFINITY; s[j][3] = -INFINITY; }
    }
  }
  // ---- online softmax: rows g and g + 8; the 4 lanes of a quad hold the 64 keys of a row
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
    mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
  const float a0 = __expf(m0 - mn0), a1 = __expf(m1 - mn1);
  m0 = mn0; m1 = mn1;
  float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s[j][0] = __expf(s[j][0] - mn0); s[j][1] = __expf(s[j][1] - mn0);
    s[j][2] = __expf(s[j][2] - mn1); s[j][3] = __expf(s[j][3] - mn1);
    ps0 += s[j][0] + s[j][1];
    ps1 += s[j][2] + s[j][3];
  }
  l0 = l0 * a0 + ps0; l1 = l1 * a1 + ps1;
#pragma unroll
  for (int d = 0; d < 2; ++d) { o[d][0] *= a0; o[d][1] *= a0; o[d][2] *= a1; o[d][3] *= a1; }
  // ---- O += P V: 4 k-chunks of 16 keys, 2 n-tiles of 8 channels
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    uint32_t pa[4];
    pa[0] = pack_bf16x2(s[2 * c][0], s[2 * c][1]);
    pa[1] = pack_bf16x2(s[2 * c][2], s[2 * c][3]);
    pa[2] = pack_bf16x2(s[2 * c + 1][0], s[2 * c + 1][1]);
    pa[3] = pack_bf16x2(s[2 * c + 1][2], s[2 * c + 1][3]);
#pragma unroll
    for (int d = 0; d < 2; ++d) {
      // B[k = key][n = channel]: {V[key0][ch], V[key0+1][ch]} and keys + 8
      const uint32_t addr = sV + (c * 16 + 2 * t) * T2I_ROWB + (d * 8 + g) * 2;
      uint16_t v00, v01, v10, v11;
      asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v00) : "r"(addr));
      asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v01) : "r"(addr + T2I_ROWB));
      asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v10) : "r"(addr + 8 * T2I_ROWB));
      asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v11) : "r"(addr + 9 * T2I_ROWB));
      const uint32_t b0 = static_cast<uint32_t>(v00) | (static_cast<uint32_t>(v01) << 16);
      const uint32_t b1 = static_cast<uint32_t>(v10) | (static_cast<uint32_t>(v11) << 16);
      mma_bf16_16816(o[d], pa, b0, b1);
    }
  }
}

__device__ __forceinline__ void t2i_head_store(T2iHead& st, __nv_bfloat16* __restrict__ out, int n, int Tq, int h) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  // row sums live per lane: reduce across the quad
  float l0 = st.l0, l1 = st.l1;
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
  for (int d = 0; d < 2; ++d) {
    if (g < Tq)
      *reinterpret_cast<uint32_t*>(out + (static_cast<size_t>(n) * Tq + g) * 128 + h * 16 + d * 8 + 2 * t) =
          pack_bf16x2(st.o[d][0] * i0, st.o[d][1] * i0);
    if (g + 8 < Tq)
      *reinterpret_cast<uint32_t*>(out + (static_cast<size_t>(n) * Tq + g + 8) * 128 + h * 16 + d * 8 + 2 * t) =
          pack_bf16x2(st.o[d][2] * i1, st.o[d][3] * i1);
  }
}

__global__ void __launch_bounds__(256)
t2i_attention_kernel(const __nv_bfloat16* __restrict__ q,   // [N, Tq, 128]
                     const __nv_bfloat16* __restrict__ K,   // [blocks*HW, 128]
                     const __nv_bfloat16* __restrict__ V,
                     const int* __restrict__ kv_block,      // [N] or null
                     __nv_bfloat16* __restrict__ out,       // [N, Tq, 128]
                     int Tq, int HW, int ldkv, float scale) {
  extern __shared__ __align__(16) uint8_t t2i_smem[];
  const uint32_t s_base = smem_u32(t2i_smem);
  const int n = blockIdx.x;
  const int blk = kv_block ? kv_block[n] : n;
  const __nv_bfloat16* Kb = K + static_cast<size_t>(blk) * HW * ldkv;
  const __nv_bfloat16* Vb = V + static_cast<size_t>(blk) * HW * ldkv;
  const int tid = threadIdx.x, h = tid >> 5;
  const int n_tiles = (HW + T2I_TILE - 1) / T2I_TILE;

  auto issue_tile = [&](int tile, int stage) {
    // 64 rows x 16 chunks of 16 B for K and for V: 2048 chunks / 256 threads = 8 each
    const int t0 = tile * T2I_TILE;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + i * 256;
      const int which = idx >> 10, j = idx & 1023;
      const int row = j >> 4, ch = j & 15;
      const int grow = min(t0 + row, HW - 1);   // rows past the end are masked in the softmax
      const __nv_bfloat16* src = (which ? Vb : Kb) + static_cast<size_t>(grow) * ldkv + ch * 8;
      cp_async16(s_base + stage * T2I_STAGE + which * (T2I_TILE * T2I_ROWB) + row * T2I_ROWB + ch * 16, src);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  T2iHead st;
  t2i_head_init(st, q, n, Tq, h, scale);
  issue_tile(0, 0);
  for (int tile = 0; tile < n_tiles; ++tile) {
    const int stage = tile & 1;
    if (tile + 1 < n_tiles) {
      issue_tile(tile + 1, stage ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const uint32_t sK = s_base + stage * T2I_STAGE + h * 32;
    t2i_head_tile(st, sK, sK + T2I_TILE * T2I_ROWB, min(T2I_TILE, HW - tile * T2I_TILE));
    __syncthreads();   // everyone is done with this stage before it is refilled
  }
  t2i_head_store(st, out, n, Tq, h);
}

int t2i_attention(const void* q, const void* K, const void* V, int ldkv, const int* kv_block, void* out, int N,
                  int Tq, int HW, cudaStream_t stream) {
  RSP_CHECK_ARG(q && K && V && out && N > 0 && Tq > 0 && Tq <= 16 && HW > 0, "t2i_attention: bad args");
  RSP_CHECK_ARG(ldkv >= 128 && ldkv % 8 == 0 && (reinterpret_cast<uintptr_t>(K) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(V) & 15) == 0, "t2i_attention: K / V row stride / alignment");
  const int smem = 2 * T2I_STAGE;
  static bool attr_set_dev[kMaxDevices] = {};   // the attribute is per device (one flag per ordinal)
  bool& attr_set = attr_set_dev[current_device()];
  if (!attr_set) {
    RSP_CHECK_CUDA(cudaFuncSetAttribute(t2i_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set = true;
  }
  t2i_attention_kernel<<<N, 256, smem, stream>>>(
      static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(K),
      static_cast<const __nv_bfloat16*>(V), kv_block, static_cast<__nv_bfloat16*>(out), Tq, HW, ldkv, 0.25f);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// t2i with the k | v projection of the image tokens fused in front of it, for per-prompt keys: CTA = one prompt,
// which walks its HW keys in tiles of 64 rows in order (the softmax order of t2i_attention).  Per tile,
// KV = keys Wkv^T + kvb + pe_kv[row] is computed on wgmma and rounded to bf16 in registers exactly where the GEMM
// epilogue rounds it ((acc + bias) + residual), staged in shared memory in t2i_attention's layout, and consumed
// there by the same per-head step: K / V never reach HBM, the keys are read once.
//   warpgroups 0 / 1: the K / V halves of the projection (m64n128k16, same k order as the GEMM), then warp h runs
//     head h of the attention.  The wgmma of tile i + 1 and the loads of its positional rows are in flight while
//     the heads work on tile i.  Thread 0 loads Wkv once and the key tiles by TMA into a 2-stage ring, tile
//     i + 2 as soon as both warpgroups' wgmma have read tile i.
// Shared memory (226 KB, one CTA per SM), 1024-byte aligned:
//   [ Wkv: 4 k-blocks x 256 rows x 128 B (128 KB) | 2 x key tile: 4 k-blocks x 64 rows x 128 B (2 x 32 KB)
//   | K, V tile: 2 x 64 rows x 272 B (34 KB) | barriers ]
// Registers: 179 per thread (256 x 1 launch bound: a producer warpgroup would cap every thread at 168, too few to
// hold the positional rows next to the accumulator and the attention state).
constexpr int TF_THREADS = 256;
constexpr int TF_W_BYTES = 4 * 256 * 128;
constexpr int TF_A_BYTES = 4 * T2I_TILE * 128;
constexpr int TF_STAGES = 2;
constexpr int TF_BAR_OFF = TF_W_BYTES + TF_STAGES * TF_A_BYTES + T2I_STAGE;
constexpr int TF_SMEM = TF_BAR_OFF + 64;
static_assert(TF_SMEM <= 227 * 1024, "t2i_fused shared memory");

__global__ void __launch_bounds__(TF_THREADS, 1)
t2i_fused_kernel(const __grid_constant__ CUtensorMap tma_keys,   // keys bf16 [N*HW, 256], box 64 x 64
                 const __grid_constant__ CUtensorMap tma_w,      // Wkv bf16 [256, 256], box 256 x 64
                 const float* __restrict__ kvb,                  // [256]
                 const __nv_bfloat16* __restrict__ pe_kv,        // [HW, 256]
                 const __nv_bfloat16* __restrict__ q,            // [N, Tq, 128]
                 __nv_bfloat16* __restrict__ out,                // [N, Tq, 128]
                 int Tq, int HW, float scale) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t s_w = smem_u32(smem);
  const uint32_t s_a = s_w + TF_W_BYTES;
  const uint32_t s_kv = s_a + TF_STAGES * TF_A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + TF_BAR_OFF);
  const uint32_t bar_w = smem_u32(&bars[0]);
  auto bar_full = [&](int s) { return smem_u32(&bars[1 + s]); };
  const int n = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = (HW + T2I_TILE - 1) / T2I_TILE;
  // rows past the prompt's HW (a partial last tile) are masked in the softmax
  auto load_tile = [&](int tile) {
    const uint32_t full = bar_full(tile % TF_STAGES);
    mbar_expect_tx(full, TF_A_BYTES);
    for (int kb = 0; kb < 4; ++kb)
      tma_load_2d(s_a + (tile % TF_STAGES) * TF_A_BYTES + kb * (T2I_TILE * 128), &tma_keys, full, kb * 64,
                  n * HW + tile * T2I_TILE);
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_keys);
    tma_prefetch_desc(&tma_w);
    mbar_init(bar_w, 1);
    for (int s = 0; s < TF_STAGES; ++s) mbar_init(bar_full(s), 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar_w, TF_W_BYTES);
    for (int kb = 0; kb < 4; ++kb) tma_load_2d(s_w + kb * (256 * 128), &tma_w, bar_w, kb * 64, 0);
    for (int tile = 0; tile < TF_STAGES && tile < n_tiles; ++tile) load_tile(tile);
  }

  const int wg = warp >> 2;   // 0: K columns [0, 128), 1: V columns [128, 256)
  const int h = warp;         // head of the attention step
  const int tw = threadIdx.x & 127;
  const int g = lane >> 2, t = lane & 3;
  const int frow = (tw >> 5) * 16 + g;   // accumulator rows frow and frow + 8 of the 64-row tile
  T2iHead st;
  t2i_head_init(st, q, n, Tq, h, scale);
  const uint32_t sK = s_kv + h * 32, sV = sK + T2I_TILE * T2I_ROWB;
  const uint32_t s_dst = s_kv + wg * (T2I_TILE * T2I_ROWB) + frow * T2I_ROWB + t * 4;
  const float* bias = kvb + wg * 128 + 2 * t;
  const __nv_bfloat16* pe = pe_kv + wg * 128 + 2 * t;
  const uint32_t sb = s_w + wg * (128 * 128);
  mbar_wait(bar_w, 0);
  float acc[64];
#pragma unroll 1
  for (int tile = 0; tile < n_tiles; ++tile) {
    const int stage = tile % TF_STAGES;
    mbar_wait(bar_full(stage), (tile / TF_STAGES) & 1);
    const uint32_t sa = s_a + stage * TF_A_BYTES;
    acc_fence(acc);
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        Wgmma<128>::ss<0>(acc, make_gdesc(sa + kb * (T2I_TILE * 128) + k * 32, 16, 1024),
                          make_gdesc(sb + kb * (256 * 128) + k * 32, 16, 1024), (kb | k) != 0);
    }
    wgmma_commit();
    // positional residual of the tile's rows (bf16 pairs; rows past HW are masked keys, any finite value will do),
    // in flight while the heads work on the previous tile
    uint32_t r[2][16];
    {
      const int r0 = min(tile * T2I_TILE + frow, HW - 1), r1 = min(tile * T2I_TILE + frow + 8, HW - 1);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        r[0][j] = __ldg(reinterpret_cast<const unsigned int*>(pe + static_cast<size_t>(r0) * 256 + 8 * j));
        r[1][j] = __ldg(reinterpret_cast<const unsigned int*>(pe + static_cast<size_t>(r1) * 256 + 8 * j));
      }
    }
    if (tile > 0) t2i_head_tile(st, sK, sV, T2I_TILE);   // every tile but the last is whole
    wgmma_wait<0>();
    acc_fence(acc);
    // every head is done with the previous tile (the K / V buffer is free) and both warpgroups' wgmma have read
    // this tile's keys (their stage may be refilled)
    named_bar_sync(1, 256);
    if (threadIdx.x == 0 && tile + TF_STAGES < n_tiles) load_tile(tile + TF_STAGES);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float2 b = __ldg(reinterpret_cast<const float2*>(bias + 8 * j));
      const float v0 = (acc[4 * j] + b.x) + __uint_as_float(r[0][j] << 16);
      const float v1 = (acc[4 * j + 1] + b.y) + __uint_as_float(r[0][j] & 0xffff0000u);
      const float v2 = (acc[4 * j + 2] + b.x) + __uint_as_float(r[1][j] << 16);
      const float v3 = (acc[4 * j + 3] + b.y) + __uint_as_float(r[1][j] & 0xffff0000u);
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(s_dst + 16 * j), "r"(pack_bf16x2(v0, v1)) : "memory");
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(s_dst + 8 * T2I_ROWB + 16 * j), "r"(pack_bf16x2(v2, v3))
                   : "memory");
    }
    named_bar_sync(1, 256);   // K and V of this tile are staged
  }
  t2i_head_tile(st, sK, sV, HW - (n_tiles - 1) * T2I_TILE);
  t2i_head_store(st, out, n, Tq, h);
}

int t2i_fused(const void* keys, int ldk, const void* kvw, const float* kvb, const void* pe_kv, const void* q,
              void* out, int N, int Tq, int HW, cudaStream_t stream) {
  RSP_CHECK_ARG(keys && kvw && kvb && pe_kv && q && out, "t2i_fused: null pointer");
  RSP_CHECK_ARG(N > 0 && Tq > 0 && Tq <= 16 && HW > 0 && static_cast<long long>(N) * HW < (1ll << 31),
                "t2i_fused: N %d, Tq %d, HW %d (Tq <= 16, N * HW < 2^31)", N, Tq, HW);
  RSP_CHECK_ARG(ldk >= 256 && ldk % 8 == 0 && (reinterpret_cast<uintptr_t>(keys) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(kvw) & 15) == 0, "t2i_fused: keys / Wkv row stride or alignment");
  RSP_CHECK_ARG((reinterpret_cast<uintptr_t>(kvb) & 7) == 0 && (reinterpret_cast<uintptr_t>(pe_kv) & 3) == 0 &&
                (reinterpret_cast<uintptr_t>(q) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0,
                "t2i_fused: bias / positional term / q / out alignment");
  CUtensorMap ta, tw;
  RSP_TRY(make_tmap_bf16_2d(&ta, keys, static_cast<uint64_t>(N) * HW, 256, static_cast<uint64_t>(ldk) * 2,
                            T2I_TILE, 64));
  RSP_TRY(make_tmap_bf16_2d(&tw, kvw, 256, 256, 256 * 2, 256, 64));
  static bool attr_set_dev[kMaxDevices] = {};   // the attribute is per device (one flag per ordinal)
  bool& attr_set = attr_set_dev[current_device()];
  if (!attr_set) {
    RSP_CHECK_CUDA(cudaFuncSetAttribute(t2i_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TF_SMEM));
    attr_set = true;
  }
  t2i_fused_kernel<<<N, TF_THREADS, TF_SMEM, stream>>>(
      ta, tw, kvb, static_cast<const __nv_bfloat16*>(pe_kv), static_cast<const __nv_bfloat16*>(q),
      static_cast<__nv_bfloat16*>(out), Tq, HW, 0.25f);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// i2t: CTA = (prompt, 128 image tokens), warp = head.  The Q tile (128 x 256 B) is staged with
// cp.async, S = Q K_tok^T and O = P V_tok run on mma.sync m16n8k16 with the prompt's 10 token keys /
// values (padded to 16) held in registers as B fragments for the whole tile; the result overwrites
// the warp's own 32-byte column slice of the staged tile, which is then written out coalesced.
// HBM traffic = Q in + O out, 2 MB per prompt: the kernel's roofline.
constexpr int I2T_PIX = 128;
constexpr int I2T_ROWB = 272;

// Token K / V fragments of one (prompt, head) for i2t: kp / vp point at the head's 16 channels of token 0 (token rows
// 128 elements apart, in global or shared memory).  K (B[k = dim][n = token]) is pre-scaled; tokens >= Tq are 0.
__device__ __forceinline__ void i2t_token_frags(const __nv_bfloat16* kp, const __nv_bfloat16* vp, int Tq, float scale,
                                                uint32_t (&kb)[2][2], uint32_t (&vb)[2][2]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int tok = j * 8 + g;                       // B[k = dim][n = token]
    kb[j][0] = kb[j][1] = 0u;
    if (tok < Tq) {
      const __nv_bfloat162 k0 = *reinterpret_cast<const __nv_bfloat162*>(kp + tok * 128 + 2 * t);
      const __nv_bfloat162 k1 = *reinterpret_cast<const __nv_bfloat162*>(kp + tok * 128 + 2 * t + 8);
      kb[j][0] = pack_bf16x2(__bfloat162float(k0.x) * scale, __bfloat162float(k0.y) * scale);
      kb[j][1] = pack_bf16x2(__bfloat162float(k1.x) * scale, __bfloat162float(k1.y) * scale);
    }
    // B[k = token][n = dim]: dims j*8 + g, tokens (2t, 2t+1) and (2t+8, 2t+9)
    auto ldv = [&](int tok2) -> uint32_t {
      return tok2 < Tq ? static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(vp + tok2 * 128 + j * 8 + g)) : 0u;
    };
    vb[j][0] = ldv(2 * t) | (ldv(2 * t + 1) << 16);
    vb[j][1] = ldv(2 * t + 8) | (ldv(2 * t + 9) << 16);
  }
}

// 16 image tokens x one head: qa = their Q (m16n8k16 A fragment) -> o = bf16 attention output in the same fragment
// layout ({row g, dims 2t..}, {row g + 8, dims 2t..}, {row g, dims 8 + 2t..}, {row g + 8, dims 8 + 2t..}).
__device__ __forceinline__ void i2t_chunk(const uint32_t (&qa)[4], const uint32_t (&kb)[2][2], const uint32_t (&vb)[2][2],
                                          int Tq, uint32_t (&o)[4]) {
  const int t = threadIdx.x & 3;
  float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
  mma_bf16_16816(s0, qa, kb[0][0], kb[0][1]);
  mma_bf16_16816(s1, qa, kb[1][0], kb[1][1]);
  // mask padded tokens (columns 2t, 2t+1 of tile 0 and 8 + 2t, 9 + 2t of tile 1)
  if (2 * t >= Tq) { s0[0] = -INFINITY; s0[2] = -INFINITY; }
  if (2 * t + 1 >= Tq) { s0[1] = -INFINITY; s0[3] = -INFINITY; }
  if (8 + 2 * t >= Tq) { s1[0] = -INFINITY; s1[2] = -INFINITY; }
  if (9 + 2 * t >= Tq) { s1[1] = -INFINITY; s1[3] = -INFINITY; }
  float m0 = fmaxf(fmaxf(s0[0], s0[1]), fmaxf(s1[0], s1[1]));
  float m1 = fmaxf(fmaxf(s0[2], s0[3]), fmaxf(s1[2], s1[3]));
  m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
  m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
  s0[0] = __expf(s0[0] - m0); s0[1] = __expf(s0[1] - m0); s1[0] = __expf(s1[0] - m0); s1[1] = __expf(s1[1] - m0);
  s0[2] = __expf(s0[2] - m1); s0[3] = __expf(s0[3] - m1); s1[2] = __expf(s1[2] - m1); s1[3] = __expf(s1[3] - m1);
  float l0 = s0[0] + s0[1] + s1[0] + s1[1], l1 = s0[2] + s0[3] + s1[2] + s1[3];
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  uint32_t pa[4] = {pack_bf16x2(s0[0], s0[1]), pack_bf16x2(s0[2], s0[3]), pack_bf16x2(s1[0], s1[1]),
                    pack_bf16x2(s1[2], s1[3])};
  float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
  mma_bf16_16816(o0, pa, vb[0][0], vb[0][1]);
  mma_bf16_16816(o1, pa, vb[1][0], vb[1][1]);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
  o[0] = pack_bf16x2(o0[0] * i0, o0[1] * i0);
  o[1] = pack_bf16x2(o0[2] * i1, o0[3] * i1);
  o[2] = pack_bf16x2(o1[0] * i0, o1[1] * i0);
  o[3] = pack_bf16x2(o1[2] * i1, o1[3] * i1);
}

// i2t: CTA = (prompt, 128 image tokens), warp = head.  The Q tile (128 x 256 B) is staged with
// cp.async, S = Q K_tok^T and O = P V_tok run on mma.sync m16n8k16 with the prompt's 10 token keys /
// values (padded to 16) held in registers as B fragments for the whole tile; the result overwrites
// the warp's own 32-byte column slice of the staged tile, which is then written out coalesced.
// HBM traffic = Q in + O out, 2 MB per prompt: the kernel's roofline.
__global__ void __launch_bounds__(256)
i2t_attention_kernel(const __nv_bfloat16* __restrict__ Q,      // [blocks*HW, 128]
                     const int* __restrict__ q_block,          // [N] or null
                     const __nv_bfloat16* __restrict__ ktok,   // [N, Tq, 128]
                     const __nv_bfloat16* __restrict__ vtok,
                     __nv_bfloat16* __restrict__ out,          // [N*HW, 128]
                     int Tq, int HW, float scale) {
  __shared__ __align__(16) uint8_t tile[I2T_PIX * I2T_ROWB];
  const uint32_t s_tile = smem_u32(tile);
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * I2T_PIX;
  const int tid = threadIdx.x, lane = tid & 31, h = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int blk = q_block ? q_block[n] : n;
  const __nv_bfloat16* Qb = Q + (static_cast<size_t>(blk) * HW + p0) * 128;
  const int npix = min(I2T_PIX, HW - p0);
  // stage Q: 128 rows x 16 chunks of 16 B = 2048 chunks / 256 threads
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int idx = tid + i * 256;
    const int row = idx >> 4, ch = idx & 15;
    const int srow = min(row, npix - 1);
    cp_async16(s_tile + row * I2T_ROWB + ch * 16, Qb + static_cast<size_t>(srow) * 128 + ch * 8);
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  // token K / V fragments of this (prompt, head): constant for the tile
  uint32_t kb[2][2], vb[2][2];
  i2t_token_frags(ktok + static_cast<size_t>(n) * Tq * 128 + h * 16, vtok + static_cast<size_t>(n) * Tq * 128 + h * 16,
                  Tq, scale, kb, vb);
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  const uint32_t sq = s_tile + h * 32;
#pragma unroll 2
  for (int c = 0; c < I2T_PIX / 16; ++c) {
    uint32_t qa[4];
    const uint32_t a0 = sq + (c * 16 + g) * I2T_ROWB + t * 4;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(qa[0]) : "r"(a0));
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(qa[1]) : "r"(a0 + 8 * I2T_ROWB));
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(qa[2]) : "r"(a0 + 16));
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(qa[3]) : "r"(a0 + 8 * I2T_ROWB + 16));
    uint32_t o[4];
    i2t_chunk(qa, kb, vb, Tq, o);
    __syncwarp();   // all lanes have read this chunk's Q fragments before the slice is overwritten
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a0), "r"(o[0]) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a0 + 8 * I2T_ROWB), "r"(o[1]) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a0 + 16), "r"(o[2]) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a0 + 8 * I2T_ROWB + 16), "r"(o[3]) : "memory");
  }
  __syncthreads();
  __nv_bfloat16* Ob = out + (static_cast<size_t>(n) * HW + p0) * 128;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int idx = tid + i * 256;
    const int row = idx >> 4, ch = idx & 15;
    if (row < npix)
      *reinterpret_cast<uint4*>(Ob + static_cast<size_t>(row) * 128 + ch * 8) =
          *reinterpret_cast<const uint4*>(tile + row * I2T_ROWB + ch * 16);
  }
}

int i2t_attention(const void* Q, const int* q_block, const void* ktok, const void* vtok, void* out,
                  int N, int Tq, int HW, cudaStream_t stream) {
  RSP_CHECK_ARG(Q && ktok && vtok && out && N > 0 && Tq > 0 && Tq <= 16 && HW > 0, "i2t_attention: bad args");
  dim3 grid((HW + I2T_PIX - 1) / I2T_PIX, N);
  i2t_attention_kernel<<<grid, 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(Q), q_block, static_cast<const __nv_bfloat16*>(ktok),
      static_cast<const __nv_bfloat16*>(vtok), static_cast<__nv_bfloat16*>(out), Tq, HW, 0.25f);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// One image -> token step of a two-way layer for per-prompt keys, fused.  Per 64-row tile of keys (one prompt's rows):
//   Q   = bf16((keys Wq^T + qb) + pe_q[row])     wgmma m64n128k16: the Qimg GEMM's k order and rounding
//   att = i2t(Q, ktok, vtok)                      i2t_chunk per (16 rows, head), Q taken from the accumulators
//   out = LN4((att Wo^T + ob) + keys)             wgmma m64n256k16 with att as the register A operand
// The LayerNorm statistics are summed in the order of the EPI_LN_ROW GEMM epilogue: per half row (128 columns) in
// column order, shifted by the half row's first value, the halves merged by Chan's formula.  In the wgmma layout the
// 4 lanes of a quad share two rows; lane t gathers (row t & 1, half t >> 1) from the quad by shuffles and runs
// that chain.  So out has the bytes of gemm(Qimg) -> i2t_attention -> gemm(EPI_LN_ROW); Q and att never leave
// registers, the keys are read once (A operand and residual) and the normalised rows overwrite them in shared
// memory and leave by TMA store.
// Persistent: CTA c takes tiles c, c + grid, ...; warpgroup w of it takes every other one, so one warpgroup's
// tensor-core work overlaps the other's loads, stores and softmax.  Each warpgroup owns one key-tile buffer and loads
// its next tile by TMA as soon as the TMA store of the last one has read the buffer (warp = 16 rows of the tile).
// Shared memory: [ Wq 4 x 128 rows x 128 B (64 KB) | Wo 2 x 256 rows x 128 B (64 KB) | 2 x key tile 4 x 64 x 128 B
//   (64 KB) | 2 x token K, V 16 x 256 B (16 KB) | out_proj bias, LN gamma, beta (3 KB) | barriers ] = 211 KB, one CTA
//   per SM.
// Registers: 256 threads, so up to 255 each without setmaxnreg: the out_proj accumulator alone is 128.
constexpr int IF_THREADS = 256;
constexpr int IF_TILE = 64;
constexpr int IF_WQ_BYTES = 4 * 128 * 128;
constexpr int IF_WO_BYTES = 2 * 256 * 128;
constexpr int IF_A_BYTES = 4 * IF_TILE * 128;
constexpr int IF_TOK_BYTES = 2 * 16 * 256;
constexpr int IF_A_OFF = IF_WQ_BYTES + IF_WO_BYTES;
constexpr int IF_TOK_OFF = IF_A_OFF + 2 * IF_A_BYTES;
constexpr int IF_VEC_OFF = IF_TOK_OFF + 2 * IF_TOK_BYTES;   // ob, LN gamma, LN beta: fp32 [3][256]
constexpr int IF_BAR_OFF = IF_VEC_OFF + 3 * 256 * 4;
constexpr int IF_SMEM = IF_BAR_OFF + 64;
static_assert(IF_SMEM <= 227 * 1024, "i2t_fused shared memory");

__device__ __forceinline__ float sel4(int c, float a0, float a1, float a2, float a3) {
  const float lo = (c & 1) ? a1 : a0, hi = (c & 1) ? a3 : a2;
  return (c & 2) ? hi : lo;
}

__global__ void __launch_bounds__(IF_THREADS, 1)
i2t_fused_kernel(const __grid_constant__ CUtensorMap tma_keys,   // keys bf16 [M, 256], box 64 x 64
                 const __grid_constant__ CUtensorMap tma_out,    // out bf16 [M, 256], box 64 x 64
                 const __grid_constant__ CUtensorMap tma_wq,     // Wq bf16 [128, 256], box 128 x 64
                 const __grid_constant__ CUtensorMap tma_wo,     // Wo bf16 [256, 128], box 256 x 64
                 const float* __restrict__ qb,                   // [128]
                 const __nv_bfloat16* __restrict__ pe_q,         // [HW, 128]
                 const __nv_bfloat16* __restrict__ ktok,         // [N, Tq, 128]
                 const __nv_bfloat16* __restrict__ vtok,
                 const float* __restrict__ ob,                   // [256]
                 const float* __restrict__ ln_g, const float* __restrict__ ln_b, float eps,
                 int Tq, int HW, int num_tiles, float scale) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t s_wq = smem_u32(smem);
  const uint32_t s_wo = s_wq + IF_WQ_BYTES;
  const uint32_t s_a = s_wq + IF_A_OFF;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + IF_BAR_OFF);
  const uint32_t bar_w = smem_u32(&bars[0]);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int tw = threadIdx.x & 127;
  const uint32_t bar_full = smem_u32(&bars[1 + wg]);   // this warpgroup's key tile has landed
  const int stride = 2 * gridDim.x;
  auto load_tile = [&](int tile) {
    mbar_expect_tx(bar_full, IF_A_BYTES);
    for (int kb = 0; kb < 4; ++kb)
      tma_load_2d(s_a + wg * IF_A_BYTES + kb * (IF_TILE * 128), &tma_keys, bar_full, kb * 64, tile * IF_TILE);
  };

  float* vec = reinterpret_cast<float*>(smem + IF_VEC_OFF);
  for (int i = threadIdx.x; i < 256; i += IF_THREADS) {
    vec[i] = ob[i];
    vec[256 + i] = ln_g[i];
    vec[512 + i] = ln_b[i];
  }
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_keys);
    tma_prefetch_desc(&tma_out);
    for (int b = 0; b < 3; ++b) mbar_init(smem_u32(&bars[b]), 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar_w, IF_WQ_BYTES + IF_WO_BYTES);
    for (int kb = 0; kb < 4; ++kb) tma_load_2d(s_wq + kb * (128 * 128), &tma_wq, bar_w, kb * 64, 0);
    for (int kb = 0; kb < 2; ++kb) tma_load_2d(s_wo + kb * (256 * 128), &tma_wo, bar_w, kb * 64, 0);
  }
  const int first = blockIdx.x + wg * gridDim.x;
  if (tw == 0 && first < num_tiles) load_tile(first);
  const int g = lane >> 2, t = lane & 3;
  const int frow = (warp & 3) * 16 + g;   // accumulator rows frow and frow + 8 of the tile
  const uint32_t sa = s_a + wg * IF_A_BYTES;   // this warpgroup's ring stage
  uint8_t* tok = smem + IF_TOK_OFF + wg * IF_TOK_BYTES;   // token K [16][128], then V [16][128]
  const __nv_bfloat16* tok_k = reinterpret_cast<const __nv_bfloat16*>(tok);
  const __nv_bfloat16* tok_v = tok_k + 16 * 128;
  // byte offset of (row frow, columns 8 j + 2 t, + 1) inside a swizzled 64-row tile, j in [0, 8) of a k-block
  const uint32_t rs_off = frow * 128 + 4 * t;
  mbar_wait(bar_w, 0);
  uint32_t phase = 0;
#pragma unroll 1
  for (int tile = first; tile < num_tiles; tile += stride, phase ^= 1) {
    const int row0 = tile * IF_TILE;
    const int p = row0 / HW, prow = row0 - p * HW + frow;
    {   // the prompt's token keys / values -> shared memory (every reader of the last tile's is past its barrier)
      const __nv_bfloat16* kp = ktok + static_cast<size_t>(p) * Tq * 128;
      const __nv_bfloat16* vp = vtok + static_cast<size_t>(p) * Tq * 128;
      for (int i = tw; i < 2 * Tq * 16; i += 128) {
        const int which = i >= Tq * 16, j = i - which * Tq * 16;
        cp_async16(smem_u32(tok) + which * (16 * 256) + j * 16, (which ? vp : kp) + j * 8);
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
    mbar_wait(bar_full, phase);
    // ---- Q = keys Wq^T
    uint32_t qf[16][2];
    {
      float acc[64];
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          Wgmma<128>::ss<0>(acc, make_gdesc(sa + kb * (IF_TILE * 128) + k * 32, 16, 1024),
                            make_gdesc(s_wq + kb * (128 * 128) + k * 32, 16, 1024), (kb | k) != 0);
      }
      wgmma_commit();
      uint32_t r[2][16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        r[0][j] = __ldg(reinterpret_cast<const unsigned int*>(pe_q + static_cast<size_t>(prow) * 128 + 8 * j + 2 * t));
        r[1][j] = __ldg(reinterpret_cast<const unsigned int*>(pe_q + static_cast<size_t>(prow + 8) * 128 + 8 * j + 2 * t));
      }
      wgmma_wait<0>();
      acc_fence(acc);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(qb + 8 * j + 2 * t));
        qf[j][0] = pack_bf16x2((acc[4 * j] + b.x) + __uint_as_float(r[0][j] << 16),
                               (acc[4 * j + 1] + b.y) + __uint_as_float(r[0][j] & 0xffff0000u));
        qf[j][1] = pack_bf16x2((acc[4 * j + 2] + b.x) + __uint_as_float(r[1][j] << 16),
                               (acc[4 * j + 3] + b.y) + __uint_as_float(r[1][j] & 0xffff0000u));
      }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    named_bar_sync(1 + wg, 128);   // the tokens are staged
    // ---- att = i2t(Q): head h of these 16 rows is k-step h of the out_proj
    uint32_t af[8][4];
#pragma unroll
    for (int h = 0; h < 8; ++h) {
      uint32_t kb[2][2], vb[2][2];
      i2t_token_frags(tok_k + h * 16, tok_v + h * 16, Tq, scale, kb, vb);
      const uint32_t qa[4] = {qf[2 * h][0], qf[2 * h][1], qf[2 * h + 1][0], qf[2 * h + 1][1]};
      i2t_chunk(qa, kb, vb, Tq, af[h]);
    }
    // ---- out_proj
    float acc[128];
    wgmma_fence();
#pragma unroll
    for (int h = 0; h < 8; ++h)
      wgmma_rs_bf16_n256(acc, af[h], make_gdesc(s_wo + (h >> 2) * (256 * 128) + (h & 3) * 32, 16, 1024), h != 0);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc);
    // ---- v = (acc + ob) + keys, in place
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const uint32_t a0 = sa + (j >> 3) * (IF_TILE * 128) + rs_off + ((((j & 7) ^ g)) << 4);
      uint32_t w0, w1;
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w0) : "r"(a0));
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w1) : "r"(a0 + 8 * 128));
      const float2 b = *reinterpret_cast<const float2*>(vec + 8 * j + 2 * t);
      acc[4 * j] = (acc[4 * j] + b.x) + __uint_as_float(w0 << 16);
      acc[4 * j + 1] = (acc[4 * j + 1] + b.y) + __uint_as_float(w0 & 0xffff0000u);
      acc[4 * j + 2] = (acc[4 * j + 2] + b.x) + __uint_as_float(w1 << 16);
      acc[4 * j + 3] = (acc[4 * j + 3] + b.y) + __uint_as_float(w1 & 0xffff0000u);
    }
    // ---- LayerNorm statistics: lane t runs the chain of (row frow + 8 (t & 1), columns [128 (t >> 1), + 128))
    float sum = 0.f, sumsq = 0.f, piv = 0.f;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      float rc[4][2];   // rc[r]: what lane (t + r) & 3 holds of this lane's (row, half) at columns 8 jj' + 2 src + e
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int cs = (t - r) & 3;   // the combination this lane supplies to the lane reading it in round r
        const int src = (lane & ~3) | ((t + r) & 3);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float mine = sel4(cs, acc[4 * jj + e], acc[4 * jj + 2 + e], acc[4 * (16 + jj) + e],
                                  acc[4 * (16 + jj) + 2 + e]);
          rc[r][e] = __shfl_sync(0xffffffffu, mine, src);
        }
      }
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const int r = (s - t) & 3;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float v = sel4(r, rc[0][e], rc[1][e], rc[2][e], rc[3][e]);
          if (jj == 0 && s == 0 && e == 0) piv = v;
          const float d = v - piv;
          sum += d;
          sumsq = fmaf(d, d, sumsq);
        }
      }
    }
    const float mean_h = piv + sum * (1.0f / 128.0f);
    const float m2_h = fmaxf(sumsq - sum * sum * (1.0f / 128.0f), 0.f);
    const float ot_x = __shfl_xor_sync(0xffffffffu, mean_h, 2), ot_y = __shfl_xor_sync(0xffffffffu, m2_h, 2);
    const float mean = 0.5f * (mean_h + ot_x);
    const float dm = mean_h - ot_x;
    const float var = (m2_h + ot_y + dm * dm * 64.0f) * (1.0f / 256.0f);     // n0 n1 / (n0 + n1) = 64
    const float rstd = rsqrtf(var + eps);
    const float mean0 = __shfl_sync(0xffffffffu, mean, lane & ~3), rstd0 = __shfl_sync(0xffffffffu, rstd, lane & ~3);
    const float mean1 = __shfl_sync(0xffffffffu, mean, (lane & ~3) | 1);
    const float rstd1 = __shfl_sync(0xffffffffu, rstd, (lane & ~3) | 1);
    // ---- normalise, bf16 over the keys tile, TMA store
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const uint32_t a0 = sa + (j >> 3) * (IF_TILE * 128) + rs_off + ((((j & 7) ^ g)) << 4);
      const float2 gm = *reinterpret_cast<const float2*>(vec + 256 + 8 * j + 2 * t);
      const float2 bt = *reinterpret_cast<const float2*>(vec + 512 + 8 * j + 2 * t);
      const float y0 = fmaf((acc[4 * j] - mean0) * rstd0, gm.x, bt.x);
      const float y1 = fmaf((acc[4 * j + 1] - mean0) * rstd0, gm.y, bt.y);
      const float y2 = fmaf((acc[4 * j + 2] - mean1) * rstd1, gm.x, bt.x);
      const float y3 = fmaf((acc[4 * j + 3] - mean1) * rstd1, gm.y, bt.y);
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(a0), "r"(pack_bf16x2(y0, y1)) : "memory");
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(a0 + 8 * 128), "r"(pack_bf16x2(y2, y3)) : "memory");
    }
    fence_proxy_async_smem();
    named_bar_sync(1 + wg, 128);   // the tile is written (and every token read of this tile is done)
    if (tw == 0) {
      for (int kb = 0; kb < 4; ++kb) tma_store_2d(&tma_out, sa + kb * (IF_TILE * 128), kb * 64, row0);
      bulk_commit();
      bulk_wait_read0();   // the store has read the buffer: the next tile may land in it
      if (tile + stride < num_tiles) load_tile(tile + stride);
    }
  }
  if (tw == 0) bulk_wait0();   // every tile is in global memory before the CTA retires
}

int i2t_fused(const void* keys, int ldk, const void* wq, const float* qb, const void* pe_q, const void* ktok,
              const void* vtok, const void* wo, const float* ob, const float* ln_g, const float* ln_b, float eps,
              void* out, int N, int Tq, int HW, cudaStream_t stream) {
  RSP_CHECK_ARG(keys && wq && qb && pe_q && ktok && vtok && wo && ob && ln_g && ln_b && out, "i2t_fused: null pointer");
  RSP_CHECK_ARG(N > 0 && Tq > 0 && Tq <= 16 && HW > 0 && HW % IF_TILE == 0 && static_cast<long long>(N) * HW < (1ll << 31),
                "i2t_fused: N %d, Tq %d, HW %d (Tq <= 16, HW %% 64 == 0, N * HW < 2^31)", N, Tq, HW);
  RSP_CHECK_ARG(ldk >= 256 && ldk % 8 == 0, "i2t_fused: keys row stride %d", ldk);
  const uintptr_t a16 = reinterpret_cast<uintptr_t>(keys) | reinterpret_cast<uintptr_t>(wq) |
                        reinterpret_cast<uintptr_t>(wo) | reinterpret_cast<uintptr_t>(out) |
                        reinterpret_cast<uintptr_t>(ktok) | reinterpret_cast<uintptr_t>(vtok);
  const uintptr_t a8 = reinterpret_cast<uintptr_t>(qb) | reinterpret_cast<uintptr_t>(ob) |
                       reinterpret_cast<uintptr_t>(ln_g) | reinterpret_cast<uintptr_t>(ln_b);
  RSP_CHECK_ARG((a16 & 15) == 0 && (a8 & 7) == 0 && (reinterpret_cast<uintptr_t>(pe_q) & 3) == 0,
                "i2t_fused: operand alignment");
  const uint64_t M = static_cast<uint64_t>(N) * HW;
  CUtensorMap tk, to, tq, tw;
  RSP_TRY(make_tmap_bf16_2d(&tk, keys, M, 256, static_cast<uint64_t>(ldk) * 2, IF_TILE, 64));
  RSP_TRY(make_tmap_bf16_2d(&to, out, M, 256, 256 * 2, IF_TILE, 64));
  RSP_TRY(make_tmap_bf16_2d(&tq, wq, 128, 256, 256 * 2, 128, 64));
  RSP_TRY(make_tmap_bf16_2d(&tw, wo, 256, 128, 128 * 2, 256, 64));
  static bool attr_set_dev[kMaxDevices] = {};   // the attribute is per device (one flag per ordinal)
  bool& attr_set = attr_set_dev[current_device()];
  if (!attr_set) {
    RSP_CHECK_CUDA(cudaFuncSetAttribute(i2t_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, IF_SMEM));
    attr_set = true;
  }
  const int num_tiles = static_cast<int>(M / IF_TILE);
  const int grid = num_tiles < num_sms() ? num_tiles : num_sms();
  i2t_fused_kernel<<<grid, IF_THREADS, IF_SMEM, stream>>>(
      tk, to, tq, tw, qb, static_cast<const __nv_bfloat16*>(pe_q), static_cast<const __nv_bfloat16*>(ktok),
      static_cast<const __nv_bfloat16*>(vtok), ob, ln_g, ln_b, eps, Tq, HW, num_tiles, 0.25f);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace rsp
