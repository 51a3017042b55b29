// Global attention for grids the flash kernel does not specialise (S = 48 / 80: 768^2 / 1280^2 inputs of the
// encoder-size sweep, VS:570-602 with img_size != 1024).  Three passes per (image, head), the two contractions on
// the wgmma GEMM:  scores = Q K^T (fp32 [T, T]) and tab = Q [Rh; Rw]^T (fp32 [T, 2*NT]) -> this file's row kernel
// P = softmax(scale * scores + rel_h + rel_w) (bf16) -> out = P V with V pre-transposed to [hd, T].
// Reference: HF:803-831 (SamVisionAttention.forward), HF:760-801 (decomposed rel-pos); VS:202-221, 117-157.
// HBM-bound on the T x T intermediates (12 bytes per score); the CUDA-core kernel it replaces took 108 ms (768^2) /
// 810 ms (1280^2) per ViT-H layer at batch 8.
#include "attention.h"
#include "sm90.cuh"

namespace rsp {

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// One block per query row of one (image, head); rows are stacked [n_rows = groups * T].  scores: fp32 [n_rows, lds];
// tab: fp32 [n_rows, ldt], columns [0, NT) = q . Rh[t], [NT, 2 NT) = q . Rw[t] (table index t = q_coord - k_coord +
// S - 1);  P: bf16 [n_rows, ldp].  A thread handles 4 consecutive keys per step (S % 4 == 0: they share the key row).
template <int NV>
__global__ void __launch_bounds__(256)
attn_softmax_bias_kernel(const float* __restrict__ scores, int lds, const float* __restrict__ tab, int ldt, int NT,
                         __nv_bfloat16* __restrict__ P, int ldp, int T, int S, float scale2) {
  __shared__ float bh[128], bw[128];
  __shared__ float red[8];
  const int row = blockIdx.x;
  const int q = row % T;
  const int qh = q / S, qw = q - qh * S;
  const float* trow = tab + static_cast<size_t>(row) * ldt;
  for (int i = threadIdx.x; i < S; i += 256) {        // pre-multiplied by log2 e: the softmax runs in base 2
    bh[i] = trow[qh - i + S - 1] * 1.4426950408889634f;
    bw[i] = trow[NT + qw - i + S - 1] * 1.4426950408889634f;
  }
  __syncthreads();
  const float4* srow = reinterpret_cast<const float4*>(scores + static_cast<size_t>(row) * lds);
  const float inv_s = 1.0f / static_cast<float>(S);
  float4 v[NV];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int k = 4 * (threadIdx.x + j * 256);
    if (k < T) {
      const int kh = static_cast<int>((static_cast<float>(k) + 0.5f) * inv_s);      // exact for k < 2^22
      const int kw = k - kh * S;
      const float4 s4 = __ldg(srow + (k >> 2));
      const float b = bh[kh];
      v[j].x = fmaf(s4.x, scale2, b + bw[kw]);
      v[j].y = fmaf(s4.y, scale2, b + bw[kw + 1]);
      v[j].z = fmaf(s4.z, scale2, b + bw[kw + 2]);
      v[j].w = fmaf(s4.w, scale2, b + bw[kw + 3]);
      mx = fmaxf(fmaxf(mx, fmaxf(v[j].x, v[j].y)), fmaxf(v[j].z, v[j].w));
    } else {
      v[j] = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    v[j].x = ex2f(v[j].x - mx); v[j].y = ex2f(v[j].y - mx); v[j].z = ex2f(v[j].z - mx); v[j].w = ex2f(v[j].w - mx);
    sum += (v[j].x + v[j].y) + (v[j].z + v[j].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) sum += red[w];
  const float inv = 1.0f / sum;
  uint2* prow = reinterpret_cast<uint2*>(P + static_cast<size_t>(row) * ldp);
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int k = 4 * (threadIdx.x + j * 256);
    if (k < T) prow[k >> 2] = make_uint2(pack_bf16x2(v[j].x * inv, v[j].y * inv), pack_bf16x2(v[j].z * inv, v[j].w * inv));
  }
}

int attn_softmax_bias(const float* scores, int lds, const float* tab, int ldt, int NT, void* P, int ldp, int n_rows,
                      int T, int S, float scale, cudaStream_t stream) {
  RSP_CHECK_ARG(scores && tab && P && T == S * S && S <= 128 && S % 4 == 0 && NT >= 2 * S - 1 && ldt >= 2 * NT &&
                lds >= T && ldp >= T && lds % 4 == 0 && ldp % 4 == 0 && n_rows > 0 && n_rows % T == 0 &&
                (reinterpret_cast<uintptr_t>(scores) & 15) == 0 && (reinterpret_cast<uintptr_t>(P) & 7) == 0,
                "attn_softmax_bias: bad args (S %% 4 == 0, 16-byte aligned rows)");
  auto* p = static_cast<__nv_bfloat16*>(P);
  const float scale2 = scale * 1.4426950408889634f;
  const unsigned grid = static_cast<unsigned>(n_rows);
  if (T <= 1024 * 3) attn_softmax_bias_kernel<3><<<grid, 256, 0, stream>>>(scores, lds, tab, ldt, NT, p, ldp, T, S, scale2);
  else if (T <= 1024 * 7) attn_softmax_bias_kernel<7><<<grid, 256, 0, stream>>>(scores, lds, tab, ldt, NT, p, ldp, T, S, scale2);
  else if (T <= 1024 * 16) attn_softmax_bias_kernel<16><<<grid, 256, 0, stream>>>(scores, lds, tab, ldt, NT, p, ldp, T, S, scale2);
  else { set_last_error("attn_softmax_bias: T = %d too large", T); return RSP_ERR_UNSUPPORTED; }
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// in: bf16 [n_seq * T, ld] columns [col0, col0 + C) -> out bf16 [n_seq, C, T] (V of every head as [hd, T] rows,
// the K-contiguous B operand of the P V contraction).  32 x 32 tiles through shared memory.
__global__ void transpose_cols_kernel(const __nv_bfloat16* __restrict__ in, int ld, int col0, int C, int T,
                                      __nv_bfloat16* __restrict__ out) {
  __shared__ __nv_bfloat16 tile[32][34];
  const int seq = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;     // 32 x 8
  for (int r = ty; r < 32; r += 8) {
    const int t = t0 + r, c = c0 + tx;
    tile[r][tx] = (t < T && c < C) ? in[(static_cast<size_t>(seq) * T + t) * ld + col0 + c] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r, t = t0 + tx;
    if (c < C && t < T) out[(static_cast<size_t>(seq) * C + c) * T + t] = tile[tx][r];
  }
}

int transpose_cols(const void* in, int ld, int col0, int C, int n_seq, int T, void* out, cudaStream_t stream) {
  RSP_CHECK_ARG(in && out && C > 0 && T > 0 && n_seq > 0 && ld >= col0 + C, "transpose_cols: bad args");
  dim3 grid((T + 31) / 32, (C + 31) / 32, n_seq);
  transpose_cols_kernel<<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(in), ld, col0, C, T,
                                                   static_cast<__nv_bfloat16*>(out));
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// in: bf16 [n_seq * T, ld], columns [col0 + h * hd, +hd) of head h  ->  out bf16 [n_seq, H, T, hd]: every (image, head)
// becomes a contiguous [T, hd] operand (stacked along rows: the grouped GEMM's A / W layout).  Thread = 16 bytes.
__global__ void split_heads_kernel(const __nv_bfloat16* __restrict__ in, int ld, int col0, int H, int hd, int T,
                                   long long total, __nv_bfloat16* __restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8 = hd / 8;
  const int cc = static_cast<int>(idx % c8);
  long long r = idx / c8;
  const int t = static_cast<int>(r % T); r /= T;
  const int h = static_cast<int>(r % H);
  const long long seq = r / H;
  const uint4 v = __ldg(reinterpret_cast<const uint4*>(in + (seq * T + t) * ld + col0 + h * hd + cc * 8));
  *reinterpret_cast<uint4*>(out + ((seq * H + h) * T + t) * hd + cc * 8) = v;
}

int split_heads(const void* in, int ld, int col0, int H, int hd, int n_seq, int T, void* out, cudaStream_t stream) {
  RSP_CHECK_ARG(in && out && H > 0 && hd % 8 == 0 && n_seq > 0 && T > 0 && ld % 8 == 0 && col0 % 8 == 0 &&
                ld >= col0 + H * hd, "split_heads: bad args");
  const long long total = static_cast<long long>(n_seq) * H * T * (hd / 8);
  split_heads_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(in), ld, col0, H, hd, T, total, static_cast<__nv_bfloat16*>(out));
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace rsp
