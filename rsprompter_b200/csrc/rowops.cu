// HBM-bound row kernels of the RSPrompter path (all coalesced, 16-byte vector accesses):
//   layernorm_rows   LayerNorm over the channel dim (+ optional GELU), with an optional
//                    gather map so window_partition's pad+permute (modeling_sam.py:900-922,
//                    vit_sam.py:17-44) is folded into the LN1 write; also SamLayerNorm /
//                    LayerNorm2d / LN2d in channels-last form (modeling_sam.py:147-170,
//                    mmpretrain norm.py:64-89, rsprompter models.py:33-50)
//   patchify16       NCHW fp32 image -> bf16 [B*gh*gw, 3*16*16] rows (patch-embed conv as GEMM;
//                    modeling_sam.py:116,128)
//   im2col_nhwc      NHWC bf16 -> [B*Ho*Wo, kh*kw*C] rows (3x3 convs of neck / FPN / RPN)
//   nhwc_to_nchw     layout change at module boundaries that must hand back NCHW tensors
#include "rowops.h"
#include "sm90.cuh"

namespace rsp {

static bool aligned(const void* ptr, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1)) == 0; }

template <typename T>
__device__ __forceinline__ float load_as_float(const T* p);
template <>
__device__ __forceinline__ float load_as_float<float>(const float* p) { return *p; }
template <>
__device__ __forceinline__ float load_as_float<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat162float(*p);
}

// One warp per output row.  C % 4 == 0.  Two passes over registers-cached data when the
// row fits (C <= 32 * 4 * MAXV), which covers every C on this path (<= 1280).
template <typename TIn, typename TOut, int MAXV>
__global__ void layernorm_rows_kernel(const TIn* __restrict__ in, TOut* __restrict__ out,
                                      const float* __restrict__ gamma,
                                      const float* __restrict__ beta,
                                      const int* __restrict__ src_map, int rows_out, int C,
                                      int ld_in, int ld_out, float eps, int act,
                                      __nv_bfloat16* __restrict__ copy_out, int ld_copy) {
  const int warps_per_block = blockDim.x >> 5;
  const int row = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows_out) return;
  const int src = src_map ? src_map[row] : row;
  TOut* o = out + static_cast<size_t>(row) * ld_out;
  if (src < 0) {
    for (int c = lane * 4; c < C; c += 128) {
#pragma unroll
      for (int k = 0; k < 4; ++k) o[c + k] = TOut(0.f);
    }
    return;
  }
  const TIn* x = in + static_cast<size_t>(src) * ld_in;
  float v[MAXV][4];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < C) {
      if (sizeof(TIn) == 4) {
        const float4 f = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x) + c);
        v[i][0] = f.x; v[i][1] = f.y; v[i][2] = f.z; v[i][3] = f.w;
      } else {
        const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(x) + c);
        const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(&u.x);
        const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(&u.y);
        v[i][0] = __bfloat162float(a.x); v[i][1] = __bfloat162float(a.y);
        v[i][2] = __bfloat162float(b.x); v[i][3] = __bfloat162float(b.y);
      }
      sum += v[i][0] + v[i][1] + v[i][2] + v[i][3];
    }
  }
  if (sizeof(TIn) == 4 && copy_out) {
    // bf16 copy of the un-normalised source row (every source row occurs once in a window map); after ALL loads
    // have been issued, so the stores do not break up the batch of outstanding loads
    __nv_bfloat16* cp = copy_out + static_cast<size_t>(src) * ld_copy;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int c = (i * 32 + lane) * 4;
      if (c < C) *reinterpret_cast<uint2*>(cp + c) = make_uint2(pack_bf16x2(v[i][0], v[i][1]), pack_bf16x2(v[i][2], v[i][3]));
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
  const float mean = sum / C;
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < C) {
#pragma unroll
      for (int k = 0; k < 4; ++k) { const float d = v[i][k] - mean; var += d * d; }
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) var += __shfl_xor_sync(0xffffffffu, var, s);
  const float rstd = rsqrtf(var / C + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < C) {
      const float4 g = *reinterpret_cast<const float4*>(gamma + c);
      const float4 b = *reinterpret_cast<const float4*>(beta + c);
      float y[4];
      y[0] = (v[i][0] - mean) * rstd * g.x + b.x;
      y[1] = (v[i][1] - mean) * rstd * g.y + b.y;
      y[2] = (v[i][2] - mean) * rstd * g.z + b.z;
      y[3] = (v[i][3] - mean) * rstd * g.w + b.w;
      if (act == 1) {
#pragma unroll
        for (int k = 0; k < 4; ++k) y[k] = gelu_erf(y[k]);
      }
      if (sizeof(TOut) == 4) {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(o) + c) = make_float4(y[0], y[1], y[2], y[3]);
      } else {
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(o) + c) =
            make_uint2(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]));
      }
    }
  }
}

template <typename TIn, typename TOut>
static int launch_ln(const LayerNormArgs& a, cudaStream_t stream) {
  const int warps = 8;
  const int blocks = (a.rows_out + warps - 1) / warps;
  if (a.C <= 32 * 4 * 2) {
    layernorm_rows_kernel<TIn, TOut, 2><<<blocks, warps * 32, 0, stream>>>(
        static_cast<const TIn*>(a.in), static_cast<TOut*>(a.out), a.gamma, a.beta, a.src_map,
        a.rows_out, a.C, a.ld_in, a.ld_out, a.eps, a.act, static_cast<__nv_bfloat16*>(a.copy_out), a.ld_copy);
  } else if (a.C <= 32 * 4 * 6) {
    layernorm_rows_kernel<TIn, TOut, 6><<<blocks, warps * 32, 0, stream>>>(
        static_cast<const TIn*>(a.in), static_cast<TOut*>(a.out), a.gamma, a.beta, a.src_map,
        a.rows_out, a.C, a.ld_in, a.ld_out, a.eps, a.act, static_cast<__nv_bfloat16*>(a.copy_out), a.ld_copy);
  } else {
    layernorm_rows_kernel<TIn, TOut, 10><<<blocks, warps * 32, 0, stream>>>(
        static_cast<const TIn*>(a.in), static_cast<TOut*>(a.out), a.gamma, a.beta, a.src_map,
        a.rows_out, a.C, a.ld_in, a.ld_out, a.eps, a.act, static_cast<__nv_bfloat16*>(a.copy_out), a.ld_copy);
  }
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

int layernorm_rows(const LayerNormArgs& a, cudaStream_t stream) {
  RSP_CHECK_ARG(a.in && a.out && a.gamma && a.beta, "layernorm: null pointer");
  RSP_CHECK_ARG(a.rows_out > 0 && a.C > 0 && a.C % 4 == 0 && a.C <= 1280, "layernorm: C=%d", a.C);
  RSP_CHECK_ARG(a.ld_in % 4 == 0 && a.ld_out % 4 == 0, "layernorm: ld must be multiple of 4");
  RSP_CHECK_ARG(!a.copy_out || (a.in_fp32 && a.ld_copy % 4 == 0 && a.ld_copy >= a.C), "layernorm: copy_out needs fp32 input");
  // 4 elements per access: float4 / uint2 loads and stores of in, out and copy_out, float4 loads of gamma and beta
  RSP_CHECK_ARG(aligned(a.in, a.in_fp32 ? 16 : 8), "layernorm: in must be %d-byte aligned", a.in_fp32 ? 16 : 8);
  RSP_CHECK_ARG(aligned(a.out, a.out_fp32 ? 16 : 8), "layernorm: out must be %d-byte aligned", a.out_fp32 ? 16 : 8);
  RSP_CHECK_ARG(aligned(a.gamma, 16) && aligned(a.beta, 16), "layernorm: gamma / beta must be 16-byte aligned");
  RSP_CHECK_ARG(aligned(a.copy_out, 8), "layernorm: copy_out must be 8-byte aligned");
  if (a.in_fp32 && !a.out_fp32) return launch_ln<float, __nv_bfloat16>(a, stream);
  if (a.in_fp32 && a.out_fp32) return launch_ln<float, float>(a, stream);
  if (!a.in_fp32 && !a.out_fp32) return launch_ln<__nv_bfloat16, __nv_bfloat16>(a, stream);
  return launch_ln<__nv_bfloat16, float>(a, stream);
}

// ---------------------------------------------------------------------------------------
// patchify: thread = one (patch row, channel, ky) segment of 16 pixels
__global__ void patchify16_kernel(const float* __restrict__ img, __nv_bfloat16* __restrict__ out,
                                  int B, int Himg, int Wimg) {
  const int gh = Himg / 16, gw = Wimg / 16;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * gh * gw * 48;
  if (idx >= total) return;
  const int seg = static_cast<int>(idx % 48);       // c * 16 + ky
  const long long patch = idx / 48;
  const int c = seg >> 4, ky = seg & 15;
  const int px = static_cast<int>(patch % gw);
  const int py = static_cast<int>((patch / gw) % gh);
  const int b = static_cast<int>(patch / (static_cast<long long>(gw) * gh));
  const float* src = img + ((static_cast<size_t>(b) * 3 + c) * Himg + py * 16 + ky) * Wimg + px * 16;
  __nv_bfloat16* dst = out + patch * 768 + seg * 16;
  float f[16];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 t = reinterpret_cast<const float4*>(src)[i];
    f[4 * i] = t.x; f[4 * i + 1] = t.y; f[4 * i + 2] = t.z; f[4 * i + 3] = t.w;
  }
  uint4 w0 = make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]),
                        pack_bf16x2(f[6], f[7]));
  uint4 w1 = make_uint4(pack_bf16x2(f[8], f[9]), pack_bf16x2(f[10], f[11]),
                        pack_bf16x2(f[12], f[13]), pack_bf16x2(f[14], f[15]));
  reinterpret_cast<uint4*>(dst)[0] = w0;
  reinterpret_cast<uint4*>(dst)[1] = w1;
}

int patchify16(const float* img, void* out, int B, int Himg, int Wimg, cudaStream_t stream) {
  RSP_CHECK_ARG(img && out, "patchify: null pointer");
  RSP_CHECK_ARG(B > 0 && Himg > 0 && Wimg > 0 && Himg % 16 == 0 && Wimg % 16 == 0,
                "patchify: shape B=%d H=%d W=%d (positive, H and W multiples of 16)", B, Himg, Wimg);
  // float4 image loads, uint4 patch-row stores
  RSP_CHECK_ARG(aligned(img, 16) && aligned(out, 16), "patchify: img / out must be 16-byte aligned");
  const long long total = static_cast<long long>(B) * (Himg / 16) * (Wimg / 16) * 48;
  const int threads = 256;
  patchify16_kernel<<<static_cast<unsigned>((total + threads - 1) / threads), threads, 0, stream>>>(
      img, static_cast<__nv_bfloat16*>(out), B, Himg, Wimg);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// im2col over NHWC bf16: thread = 8 channels (16 B) of one (output pixel, tap)
__global__ void im2col_nhwc_kernel(const __nv_bfloat16* __restrict__ in,
                                   __nv_bfloat16* __restrict__ out, int B, int H, int W, int C,
                                   int KH, int KW, int stride, int pad, int Ho, int Wo) {
  const int c8 = C / 8;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * Ho * Wo * KH * KW * c8;
  if (idx >= total) return;
  const int cc = static_cast<int>(idx % c8);
  long long t = idx / c8;
  const int tap = static_cast<int>(t % (KH * KW)); t /= (KH * KW);
  const int ox = static_cast<int>(t % Wo); t /= Wo;
  const int oy = static_cast<int>(t % Ho);
  const int b = static_cast<int>(t / Ho);
  const int ky = tap / KW, kx = tap % KW;
  const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (iy >= 0 && iy < H && ix >= 0 && ix < W)
    v = *reinterpret_cast<const uint4*>(in + ((static_cast<size_t>(b) * H + iy) * W + ix) * C + cc * 8);
  const size_t orow = (static_cast<size_t>(b) * Ho + oy) * Wo + ox;
  *reinterpret_cast<uint4*>(out + orow * (static_cast<size_t>(KH) * KW * C) + static_cast<size_t>(tap) * C +
                            cc * 8) = v;
}

int im2col_nhwc(const void* in, void* out, int B, int H, int W, int C, int KH, int KW, int stride,
                int pad, cudaStream_t stream) {
  RSP_CHECK_ARG(in && out, "im2col: null pointer");
  RSP_CHECK_ARG(C > 0 && C % 8 == 0 && B > 0 && H > 0 && W > 0,
                "im2col: shape B=%d H=%d W=%d C=%d (positive, C a multiple of 8)", B, H, W, C);
  RSP_CHECK_ARG(KH >= 1 && KW >= 1 && stride >= 1 && pad >= 0, "im2col: kernel %dx%d stride %d pad %d", KH, KW, stride,
                pad);
  // at least one output pixel per axis, checked before the division that would otherwise round a negative span to 0
  RSP_CHECK_ARG(H + 2 * pad >= KH && W + 2 * pad >= KW, "im2col: kernel %dx%d larger than the padded %dx%d input", KH,
                KW, H + 2 * pad, W + 2 * pad);
  // 8 channels (16 bytes) per access
  RSP_CHECK_ARG(aligned(in, 16) && aligned(out, 16), "im2col: in / out must be 16-byte aligned");
  const int Ho = (H + 2 * pad - KH) / stride + 1, Wo = (W + 2 * pad - KW) / stride + 1;
  const long long total = static_cast<long long>(B) * Ho * Wo * KH * KW * (C / 8);
  const int threads = 256;
  im2col_nhwc_kernel<<<static_cast<unsigned>((total + threads - 1) / threads), threads, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(in), static_cast<__nv_bfloat16*>(out), B, H, W, C, KH, KW,
      stride, pad, Ho, Wo);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// [B, HW, C] -> [B, C, HW] through a padded 32x32 smem tile; in bf16 or fp32, out fp32
template <typename TIn>
__global__ void nhwc_to_nchw_kernel(const TIn* __restrict__ in, float* __restrict__ out, int HW, int C) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const TIn* src = in + static_cast<size_t>(b) * HW * C;
  float* dst = out + static_cast<size_t>(b) * HW * C;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int p = p0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (p < HW && c < C) ? load_as_float(src + static_cast<size_t>(p) * C + c) : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, p = p0 + threadIdx.x;
    if (p < HW && c < C) dst[static_cast<size_t>(c) * HW + p] = tile[threadIdx.x][i];
  }
}

int nhwc_to_nchw(const void* in, int in_fp32, float* out, int B, int HW, int C, cudaStream_t stream) {
  RSP_CHECK_ARG(in && out && B > 0 && HW > 0 && C > 0, "nhwc_to_nchw: bad args");
  dim3 block(32, 8);
  dim3 grid((HW + 31) / 32, (C + 31) / 32, B);
  if (in_fp32) nhwc_to_nchw_kernel<float><<<grid, block, 0, stream>>>(static_cast<const float*>(in), out, HW, C);
  else nhwc_to_nchw_kernel<__nv_bfloat16><<<grid, block, 0, stream>>>(static_cast<const __nv_bfloat16*>(in), out, HW, C);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
__global__ void cast_f32_bf16_kernel(const float4* __restrict__ in, uint2* __restrict__ out, long long n4) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 f = in[i];
  out[i] = make_uint2(pack_bf16x2(f.x, f.y), pack_bf16x2(f.z, f.w));
}

int cast_f32_bf16(const float* in, void* out, long long n, cudaStream_t stream) {
  RSP_CHECK_ARG(in && out && n > 0 && n % 4 == 0, "cast: n must be a positive multiple of 4");
  RSP_CHECK_ARG(aligned(in, 16) && aligned(out, 8), "cast: in must be 16-byte and out 8-byte aligned");   // float4 / uint2
  const long long n4 = n / 4;
  cast_f32_bf16_kernel<<<static_cast<unsigned>((n4 + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const float4*>(in), static_cast<uint2*>(out), n4);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ---------------------------------------------------------------------------------------
// out = LayerNorm(x + residual) over rows of C <= 256 channels (warp per row, 8 channels per lane):
// the "keys = layer_norm4(keys + attn_out)" step of SamTwoWayAttentionBlock (HF:345-347) after a
// plain bf16 out_proj GEMM.  The residual row can be block-mapped (prompts sharing an image).
template <typename TRes>
__global__ void layernorm_add_kernel(const __nv_bfloat16* __restrict__ x, const TRes* __restrict__ res,
                                     const int* __restrict__ res_block_map, int res_block_rows,
                                     const float* __restrict__ gamma, const float* __restrict__ beta,
                                     __nv_bfloat16* __restrict__ out, const float* __restrict__ pos, int pos_mod,
                                     __nv_bfloat16* __restrict__ out_pe, long long rows, int C, float eps) {
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  long long rrow = row;
  if (res_block_map) {
    const long long blk = row / res_block_rows;
    rrow = static_cast<long long>(res_block_map[blk]) * res_block_rows + (row - blk * res_block_rows);
  }
  const int c = lane * 8;
  float v[8];
  const bool on = c < C;
  if (on) {
    const uint4 u = *reinterpret_cast<const uint4*>(x + row * C + c);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[2 * j] = __uint_as_float(w[j] << 16);
      v[2 * j + 1] = __uint_as_float(w[j] & 0xffff0000u);
    }
    if (sizeof(TRes) == 4) {
      const float4 a = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(res) + rrow * C + c);
      const float4 b = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(res) + rrow * C + c + 4);
      v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
    } else {
      const uint4 r = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(res) + rrow * C + c);
      const uint32_t rw[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        v[2 * j] += __uint_as_float(rw[j] << 16);
        v[2 * j + 1] += __uint_as_float(rw[j] & 0xffff0000u);
      }
    }
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.f;
  }
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) sum += v[j];
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
  const float mean = sum / C;
  float var = 0.f;
  if (on) {
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float d = v[j] - mean; var += d * d; }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) var += __shfl_xor_sync(0xffffffffu, var, s);
  const float rstd = rsqrtf(var / C + eps);
  if (on) {
    const float4 g0 = *reinterpret_cast<const float4*>(gamma + c), g1 = *reinterpret_cast<const float4*>(gamma + c + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(beta + c), b1 = *reinterpret_cast<const float4*>(beta + c + 4);
    const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    float y[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = (v[j] - mean) * rstd * g[j] + bb[j];
    *reinterpret_cast<uint4*>(out + row * C + c) =
        make_uint4(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]), pack_bf16x2(y[4], y[5]), pack_bf16x2(y[6], y[7]));
    if (out_pe) {   // second output: keys + positional embedding, the A operand of the next k / q projections
      const float* pp = pos + (row % pos_mod) * C + c;
      const float4 p0 = *reinterpret_cast<const float4*>(pp), p1 = *reinterpret_cast<const float4*>(pp + 4);
      *reinterpret_cast<uint4*>(out_pe + row * C + c) =
          make_uint4(pack_bf16x2(y[0] + p0.x, y[1] + p0.y), pack_bf16x2(y[2] + p0.z, y[3] + p0.w),
                     pack_bf16x2(y[4] + p1.x, y[5] + p1.y), pack_bf16x2(y[6] + p1.z, y[7] + p1.w));
    }
  }
}

int layernorm_add(const void* x, const void* res, int res_fp32, const int* res_block_map, int res_block_rows,
                  const float* gamma, const float* beta, void* out, const float* pos, int pos_mod, void* out_pe,
                  long long rows, int C, float eps, cudaStream_t stream) {
  RSP_CHECK_ARG(x && res && gamma && beta && out && rows > 0, "layernorm_add: null pointer");
  RSP_CHECK_ARG(!out_pe || (pos && pos_mod > 0), "layernorm_add: out_pe needs pos / pos_mod");
  RSP_CHECK_ARG(C % 8 == 0 && C <= 256, "layernorm_add: C=%d (multiple of 8, <= 256)", C);
  RSP_CHECK_ARG(!res_block_map || res_block_rows > 0, "layernorm_add: res_block_rows");
  const int warps = 8;
  const unsigned blocks = static_cast<unsigned>((rows + warps - 1) / warps);
  if (res_fp32)
    layernorm_add_kernel<float><<<blocks, warps * 32, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<const float*>(res), res_block_map, res_block_rows, gamma,
        beta, static_cast<__nv_bfloat16*>(out), pos, pos_mod, static_cast<__nv_bfloat16*>(out_pe), rows, C, eps);
  else
    layernorm_add_kernel<__nv_bfloat16><<<blocks, warps * 32, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(res), res_block_map, res_block_rows,
        gamma, beta, static_cast<__nv_bfloat16*>(out), pos, pos_mod, static_cast<__nv_bfloat16*>(out_pe), rows, C, eps);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// out = bf16(x + table[i % period]): the extra positional encoding of the RoI head added to a pyramid level once
// (M:1566-1574 computes x + pe before both RoI extractors), 8 elements per thread.
__global__ void add_table_bf16_kernel(const uint4* __restrict__ x, const float* __restrict__ table, uint4* __restrict__ out,
                                      long long n8, long long period) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const uint4 u = x[i];
  const float* t = table + (i * 8) % period;
  const float4 t0 = *reinterpret_cast<const float4*>(t), t1 = *reinterpret_cast<const float4*>(t + 4);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
  const float tv[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j)
    o[j] = pack_bf16x2(__uint_as_float(w[j] << 16) + tv[2 * j], __uint_as_float(w[j] & 0xffff0000u) + tv[2 * j + 1]);
  out[i] = make_uint4(o[0], o[1], o[2], o[3]);
}

int add_table_bf16(const void* x, const float* table, void* out, long long n, long long period, cudaStream_t stream) {
  RSP_CHECK_ARG(x && table && out && n > 0 && n % 8 == 0 && period > 0 && period % 8 == 0, "add_table: bad args");
  // uint4 loads and stores of 8 bf16, float4 table loads
  RSP_CHECK_ARG(aligned(x, 16) && aligned(table, 16) && aligned(out, 16), "add_table: x / table / out must be 16-byte aligned");
  const long long n8 = n / 8;
  add_table_bf16_kernel<<<static_cast<unsigned>((n8 + 255) / 256), 256, 0, stream>>>(
      static_cast<const uint4*>(x), table, static_cast<uint4*>(out), n8, period);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace rsp
