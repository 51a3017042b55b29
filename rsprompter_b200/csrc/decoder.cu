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
  const int tid = threadIdx.x, lane = tid & 31, h = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
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

  // Q fragment (A operand, rows = prompt tokens padded to 16, k = the head's 16 channels), pre-scaled
  uint32_t qa[4];
  {
    auto ldq = [&](int row, int col) -> uint32_t {
      if (row >= Tq) return 0u;
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(
          q + (static_cast<size_t>(n) * Tq + row) * 128 + h * 16 + col);
      return pack_bf16x2(__bfloat162float(v.x) * scale, __bfloat162float(v.y) * scale);
    };
    qa[0] = ldq(g, 2 * t); qa[1] = ldq(g + 8, 2 * t); qa[2] = ldq(g, 2 * t + 8); qa[3] = ldq(g + 8, 2 * t + 8);
  }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float o[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};

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
    const uint32_t sV = sK + T2I_TILE * T2I_ROWB;
    const int valid = min(T2I_TILE, HW - tile * T2I_TILE);
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
    __syncthreads();   // everyone is done with this stage before it is refilled
  }
  // row sums live per lane: reduce across the quad
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
  for (int d = 0; d < 2; ++d) {
    if (g < Tq)
      *reinterpret_cast<uint32_t*>(out + (static_cast<size_t>(n) * Tq + g) * 128 + h * 16 + d * 8 + 2 * t) =
          pack_bf16x2(o[d][0] * i0, o[d][1] * i0);
    if (g + 8 < Tq)
      *reinterpret_cast<uint32_t*>(out + (static_cast<size_t>(n) * Tq + g + 8) * 128 + h * 16 + d * 8 + 2 * t) =
          pack_bf16x2(o[d][2] * i1, o[d][3] * i1);
  }
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
// i2t: CTA = (prompt, 128 image tokens), warp = head.  The Q tile (128 x 256 B) is staged with
// cp.async, S = Q K_tok^T and O = P V_tok run on mma.sync m16n8k16 with the prompt's 10 token keys /
// values (padded to 16) held in registers as B fragments for the whole tile; the result overwrites
// the warp's own 32-byte column slice of the staged tile, which is then written out coalesced.
// HBM traffic = Q in + O out, 2 MB per prompt: the kernel's roofline.
constexpr int I2T_PIX = 128;
constexpr int I2T_ROWB = 272;

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
  {
    const __nv_bfloat16* kp = ktok + static_cast<size_t>(n) * Tq * 128 + h * 16;
    const __nv_bfloat16* vp = vtok + static_cast<size_t>(n) * Tq * 128 + h * 16;
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
    __syncwarp();   // all lanes have read this chunk's Q fragments before the slice is overwritten
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a0), "r"(pack_bf16x2(o0[0] * i0, o0[1] * i0)) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a0 + 8 * I2T_ROWB), "r"(pack_bf16x2(o0[2] * i1, o0[3] * i1)) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a0 + 16), "r"(pack_bf16x2(o1[0] * i0, o1[1] * i0)) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a0 + 8 * I2T_ROWB + 16), "r"(pack_bf16x2(o1[2] * i1, o1[3] * i1)) : "memory");
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

}  // namespace rsp
