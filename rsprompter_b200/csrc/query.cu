// Kernels specific to the RSPrompter-query head (M:274-715): everything around the tensor-core GEMMs of
// MSDeformAttnPixelDecoder / Mask2Former decoder / RSMask2FormerHead._forward_head.
//
//   groupnorm_nhwc            GroupNorm(32) of the pixel decoder's ConvModules on channels-last maps, with the
//                             FPN top-down add (bilinear x2 of the coarser map) and ReLU fused into the apply pass
//                             (msdeformattn_pixel_decoder.py:94-109, 230-240)
//   ms_deform_attn_sample     mmcv MultiScaleDeformableAttention core: softmax over levels x points, bilinear
//                             sampling with zero padding (grid_sample, align_corners=False), weighted sum
//   mha_small                 nn.MultiheadAttention core for 100 queries (masked cross / self attention of
//                             Mask2FormerTransformerDecoderLayer, mask2former_layers.py:113-135)
//   attn_mask_build           attn_mask = sigmoid(bilinear(mask_pred_plus)) < 0.5, all-masked rows cleared
//                             (M:386-392, M:439-442)
//   mask_embed_src            SamMaskEmbedding (HF:569-593) + "image_embeddings + dense" (HF:499) + key PE:
//                             writes the decoder's two bf16 source tensors directly
//   query_postprocess         bilinear 256^2 -> S^2 + (> 0) + mask score + tight box per selected instance
//                             (M:652-656, maskformer_fusion_head.py:149-182, mask/utils.py:56-77), no S^2 fp32
//                             intermediate and no per-instance host sync
#include "query.h"
#include "sm90.cuh"
#include "upsample4.cuh"

namespace rsp {

__device__ __forceinline__ void unpack8f(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    f[2 * j] = __uint_as_float(w[j] << 16);
    f[2 * j + 1] = __uint_as_float(w[j] & 0xffff0000u);
  }
}

// ------------------------------------------------------------------------------------ GroupNorm
// Two-level, atomic-free (bit-reproducible) statistics: part[b][blk][g] = (sum, sumsq) of one 256-pixel block in
// fp32, then one thread per (b, g) folds the block partials in fp64 and emits (mean, rstd): the E[x^2] - mean^2
// cancellation happens in double precision, so large-mean inputs keep their variance.  CPG = C/G channels per group:
// 4 (E = 128, the RSPrompter-query head) or 8 (E = 256, the stock Mask2Former head).
template <int CPG>
__global__ void groupnorm_stats_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ part, int HW,
                                       int C, int G, int pix_per_block) {
  const int b = blockIdx.y;
  const int lanes_c = C / 8;                       // threads across channels (8 channels each)
  const int tc = threadIdx.x % lanes_c, tp = threadIdx.x / lanes_c;
  const int rows = blockDim.x / lanes_c;
  const int p0 = blockIdx.x * pix_per_block;
  constexpr int GPT = 8 / CPG;                     // groups per thread (a thread owns 8 channels)
  float s[2] = {0.f, 0.f}, q[2] = {0.f, 0.f};
  for (int p = p0 + tp; p < min(p0 + pix_per_block, HW); p += rows) {
    float f[8];
    unpack8f(*reinterpret_cast<const uint4*>(x + (static_cast<size_t>(b) * HW + p) * C + tc * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { s[j / CPG] += f[j]; q[j / CPG] += f[j] * f[j]; }
  }
  __shared__ float red[256 * 4];
  red[threadIdx.x * 4 + 0] = s[0]; red[threadIdx.x * 4 + 1] = q[0];
  red[threadIdx.x * 4 + 2] = s[1]; red[threadIdx.x * 4 + 3] = q[1];
  __syncthreads();
  if (tp == 0) {
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    for (int r = 0; r < rows; ++r)
#pragma unroll
      for (int k = 0; k < 4; ++k) a[k] += red[(r * lanes_c + tc) * 4 + k];
    float* st = part + ((static_cast<size_t>(b) * gridDim.x + blockIdx.x) * G + tc * GPT) * 2;
    st[0] = a[0]; st[1] = a[1];
    if (GPT == 2) { st[2] = a[2]; st[3] = a[3]; }
  }
}

__global__ void groupnorm_finalize_kernel(const float* __restrict__ part, float* __restrict__ stats, int B, int G,
                                          int nblk, double n, float eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * G) return;
  const int b = i / G, g = i - b * G;
  double s = 0.0, q = 0.0;
  for (int k = 0; k < nblk; ++k) {
    const float* st = part + ((static_cast<size_t>(b) * nblk + k) * G + g) * 2;
    s += st[0]; q += st[1];
  }
  const double mean = s / n;
  const double var = fmax(q / n - mean * mean, 0.0);
  stats[2 * i] = static_cast<float>(mean);
  stats[2 * i + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
}

// y = GN(x) (+ bilinear x2 upsample of `up` [B, H/2, W/2, C]) (ReLU)
template <int CPG>
__global__ void groupnorm_apply_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ stats,
                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                       const __nv_bfloat16* __restrict__ up, __nv_bfloat16* __restrict__ out, int B,
                                       int H, int W, int C, int G, float eps, int relu) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int c8 = C / 8;
  if (idx >= static_cast<long long>(B) * H * W * c8) return;
  const int tc = static_cast<int>(idx % c8);
  const long long pix = idx / c8;
  const int b = static_cast<int>(pix / (static_cast<long long>(H) * W));
  const int rem = static_cast<int>(pix - static_cast<long long>(b) * H * W);
  const int y = rem / W, xx = rem - y * W;
  float f[8];
  unpack8f(*reinterpret_cast<const uint4*>(x + pix * C + tc * 8), f);
  // (mean, rstd) of this thread's group(s): two groups of 4 channels (one 16-byte load) or one group of 8
  float4 mr;
  if (CPG == 4) {
    mr = __ldg(reinterpret_cast<const float4*>(stats + (static_cast<size_t>(b) * G + tc * 2) * 2));
  } else {
    const float2 m2 = __ldg(reinterpret_cast<const float2*>(stats + (static_cast<size_t>(b) * G + tc) * 2));
    mr = make_float4(m2.x, m2.y, m2.x, m2.y);
  }
  const float4 ga0 = __ldg(reinterpret_cast<const float4*>(gamma + tc * 8)), ga1 = __ldg(reinterpret_cast<const float4*>(gamma + tc * 8 + 4));
  const float4 be0 = __ldg(reinterpret_cast<const float4*>(beta + tc * 8)), be1 = __ldg(reinterpret_cast<const float4*>(beta + tc * 8 + 4));
  const float gam[8] = {ga0.x, ga0.y, ga0.z, ga0.w, ga1.x, ga1.y, ga1.z, ga1.w};
  const float bet[8] = {be0.x, be0.y, be0.z, be0.w, be1.x, be1.y, be1.z, be1.w};
  float o[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float mean = j < 4 ? mr.x : mr.z, rstd = j < 4 ? mr.y : mr.w;
    o[j] = (f[j] - mean) * rstd * gam[j] + bet[j];
  }
  if (up) {
    const int h2 = H / 2, w2 = W / 2;
    const float sy = fmaxf((y + 0.5f) * 0.5f - 0.5f, 0.f), sx = fmaxf((xx + 0.5f) * 0.5f - 0.5f, 0.f);
    const int y0 = static_cast<int>(sy), x0 = static_cast<int>(sx);
    const int y1 = min(y0 + 1, h2 - 1), x1 = min(x0 + 1, w2 - 1);
    const float ly = sy - y0, lx = sx - x0;
    const __nv_bfloat16* ub = up + static_cast<size_t>(b) * h2 * w2 * C + tc * 8;
    float a[8], c[8], d[8], e[8];
    unpack8f(*reinterpret_cast<const uint4*>(ub + (static_cast<size_t>(y0) * w2 + x0) * C), a);
    unpack8f(*reinterpret_cast<const uint4*>(ub + (static_cast<size_t>(y0) * w2 + x1) * C), c);
    unpack8f(*reinterpret_cast<const uint4*>(ub + (static_cast<size_t>(y1) * w2 + x0) * C), d);
    unpack8f(*reinterpret_cast<const uint4*>(ub + (static_cast<size_t>(y1) * w2 + x1) * C), e);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      o[j] += (1.f - ly) * ((1.f - lx) * a[j] + lx * c[j]) + ly * ((1.f - lx) * d[j] + lx * e[j]);
  }
  if (relu) {
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fmaxf(o[j], 0.f);
  }
  *reinterpret_cast<uint4*>(out + pix * C + tc * 8) =
      make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
}

int groupnorm_nhwc(const void* x, float* stats_ws, const float* gamma, const float* beta, const void* up, void* out,
                   int B, int H, int W, int C, int G, float eps, int relu, cudaStream_t stream) {
  RSP_CHECK_ARG(x && stats_ws && gamma && beta && out, "groupnorm: null pointer");
  RSP_CHECK_ARG(C % 8 == 0 && C % G == 0 && (C / G == 4 || C / G == 8) && C / 8 <= 32 && 256 % (C / 8) == 0,
                "groupnorm: C=%d G=%d unsupported", C, G);
  const bool cpg8 = C / G == 8;
  RSP_CHECK_ARG((reinterpret_cast<uintptr_t>(stats_ws) & 15) == 0, "groupnorm: stats_ws must be 16-byte aligned");
  const int HW = H * W;
  const int ppb = 256;
  const int nblk = (HW + ppb - 1) / ppb;
  dim3 grid(nblk, B);
  float* part = stats_ws + static_cast<size_t>(B) * G * 2;       // [B, nblk, G, 2] block partials behind the stats
  if (cpg8) groupnorm_stats_kernel<8><<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), part, HW, C, G, ppb);
  else groupnorm_stats_kernel<4><<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), part, HW, C, G, ppb);
  RSP_CHECK_LAUNCH();
  groupnorm_finalize_kernel<<<(B * G + 127) / 128, 128, 0, stream>>>(part, stats_ws, B, G, nblk,
                                                                   static_cast<double>(HW) * (C / G), eps);
  RSP_CHECK_LAUNCH();
  const long long total = static_cast<long long>(B) * HW * (C / 8);
  if (cpg8)
    groupnorm_apply_kernel<8><<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(x), stats_ws, gamma, beta, static_cast<const __nv_bfloat16*>(up),
        static_cast<__nv_bfloat16*>(out), B, H, W, C, G, eps, relu);
  else
    groupnorm_apply_kernel<4><<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(x), stats_ws, gamma, beta, static_cast<const __nv_bfloat16*>(up),
        static_cast<__nv_bfloat16*>(out), B, H, W, C, G, eps, relu);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ------------------------------------------------------------------------------------ MSDeformAttn
struct DeformLevels { int h[4], w[4], start[4]; };

// thread = 8 channels of one (batch, query, head); embed C = 8 heads x HD (HD = 16: RSPrompter-query, 32: Mask2Former)
template <int HD>
__global__ void ms_deform_attn_kernel(const __nv_bfloat16* __restrict__ value,   // [B, NQ, C]
                                      const float* __restrict__ ow, int ld_ow,    // [B*NQ, >= H*L*P*3]: offsets | logits
                                      DeformLevels lv, int B, int NQ, int L, int P,
                                      __nv_bfloat16* __restrict__ out) {          // [B*NQ, C]
  constexpr int PARTS = HD / 8, C = 8 * HD;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(B) * NQ * 8 * PARTS) return;
  const int half = static_cast<int>(idx % PARTS), h = static_cast<int>((idx / PARTS) & 7);
  const long long bq = idx / (8 * PARTS);
  const int b = static_cast<int>(bq / NQ), q = static_cast<int>(bq - static_cast<long long>(b) * NQ);
  // reference point: centre of the query's own cell, normalised
  int ql = 0;
  for (int l = 1; l < L; ++l) if (q >= lv.start[l]) ql = l;
  const int qp = q - lv.start[ql];
  const float rx = ((qp % lv.w[ql]) + 0.5f) / lv.w[ql], ry = ((qp / lv.w[ql]) + 0.5f) / lv.h[ql];
  const float* row = ow + bq * ld_ow;
  const float* offs = row + h * L * P * 2;
  const float* logit = row + 8 * L * P * 2 + h * L * P;
  float mx = -INFINITY;
  for (int i = 0; i < L * P; ++i) mx = fmaxf(mx, logit[i]);
  float den = 0.f;
  for (int i = 0; i < L * P; ++i) den += expf(logit[i] - mx);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int l = 0; l < L; ++l) {
    const int H = lv.h[l], W = lv.w[l];
    const __nv_bfloat16* vb = value + (static_cast<size_t>(b) * NQ + lv.start[l]) * C + h * HD + half * 8;
    for (int pt = 0; pt < P; ++pt) {
      const float wgt = expf(logit[l * P + pt] - mx) / den;
      const float lx = rx + offs[(l * P + pt) * 2] / W, ly = ry + offs[(l * P + pt) * 2 + 1] / H;
      const float x = lx * W - 0.5f, y = ly * H - 0.5f;      // grid_sample, align_corners=False
      const float xf = floorf(x), yf = floorf(y);
      const int x0 = static_cast<int>(xf), y0 = static_cast<int>(yf);
      const float ax = x - xf, ay = y - yf;
#pragma unroll
      for (int cy = 0; cy < 2; ++cy)
#pragma unroll
        for (int cx = 0; cx < 2; ++cx) {
          const int xi = x0 + cx, yi = y0 + cy;
          if (xi < 0 || xi >= W || yi < 0 || yi >= H) continue;   // zero padding
          const float cw = (cx ? ax : 1.f - ax) * (cy ? ay : 1.f - ay) * wgt;
          float f[8];
          unpack8f(*reinterpret_cast<const uint4*>(vb + (static_cast<size_t>(yi) * W + xi) * C), f);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] += cw * f[j];
        }
    }
  }
  *reinterpret_cast<uint4*>(out + bq * C + h * HD + half * 8) =
      make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]),
                 pack_bf16x2(acc[6], acc[7]));
}

int ms_deform_attn_sample(const void* value, const float* ow, int ld_ow, const int* hs, const int* ws, int L, int P,
                          int B, int NQ, void* out, int channels, cudaStream_t stream) {
  RSP_CHECK_ARG(value && ow && hs && ws && out && L >= 1 && L <= 4 && P >= 1, "ms_deform_attn: bad args");
  RSP_CHECK_ARG(channels == 128 || channels == 256, "ms_deform_attn: channels %d (8 heads x 16 or 32 supported)", channels);
  DeformLevels lv;
  int start = 0;
  for (int l = 0; l < 4; ++l) {
    lv.h[l] = l < L ? hs[l] : 1; lv.w[l] = l < L ? ws[l] : 1; lv.start[l] = start;
    if (l < L) start += hs[l] * ws[l];
  }
  RSP_CHECK_ARG(start == NQ, "ms_deform_attn: sum of level sizes %d != NQ %d", start, NQ);
  const long long total = static_cast<long long>(B) * NQ * (channels / 8);
  if (channels == 128)
    ms_deform_attn_kernel<16><<<static_cast<unsigned>((total + 127) / 128), 128, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(value), ow, ld_ow, lv, B, NQ, L, P, static_cast<__nv_bfloat16*>(out));
  else
    ms_deform_attn_kernel<32><<<static_cast<unsigned>((total + 127) / 128), 128, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(value), ow, ld_ow, lv, B, NQ, L, P, static_cast<__nv_bfloat16*>(out));
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ------------------------------------------------------------------------------------ small MHA
// nn.MultiheadAttention core, 8 heads x 16 channels, on mma.sync m16n8k16 (head_dim 16 = one k-step).
// CTA = (batch, head, 64 queries): 4 warps x one 16-query tile each; keys stream through shared memory in
// chunks of 64 (cp.async, double buffered).  S = Q K^T and O += P V keep P in registers (accumulator ->
// A-fragment reuse); V's B-fragment comes from ldmatrix.trans.  mask: bit words [B*nq][ceil(nk/64)],
// bit k%64 of word k/64 set = key k masked.
__device__ __forceinline__ void mma_bf16_16816q(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16q(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(src));
}

constexpr int MHA_KC = 64;     // keys per chunk
constexpr int MHA_WARPS = 4;

// HD = head channels (16: RSPrompter-query E = 128; 32: stock Mask2Former E = 256), 8 heads.  A staged key row is
// HD bf16 + 16 B pad (48 / 80 bytes: conflict-free fragment reads).
template <int HD>
__global__ void __launch_bounds__(MHA_WARPS * 32)
mha_kernel(const __nv_bfloat16* __restrict__ Q, int ldq, const __nv_bfloat16* __restrict__ K, int ldk,
           const __nv_bfloat16* __restrict__ V, int ldv, const unsigned long long* __restrict__ mask, int mask_words,
           int nq, int nk, __nv_bfloat16* __restrict__ out) {
  constexpr int KS = HD / 16;            // k-steps of Q K^T
  constexpr int PARTS = HD / 8;          // 16-byte pieces per staged row
  constexpr int ROWB = HD * 2 + 16;
  constexpr int E = 8 * HD;
  __shared__ __align__(16) unsigned char sK[2][MHA_KC * ROWB];
  __shared__ __align__(16) unsigned char sV[2][MHA_KC * ROWB];
  const int b = blockIdx.x >> 3, h = blockIdx.x & 7;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int q0 = (blockIdx.y * MHA_WARPS + warp) * 16;
  const bool active = q0 < nq;
  const int r0 = min(q0 + g, nq - 1), r1 = min(q0 + g + 8, nq - 1);

  // 1/sqrt(16) is exact in bf16 and is folded into Q; 1/sqrt(32) is not: it multiplies the fp32 scores instead
  constexpr float POST_SCALE = HD == 16 ? 1.0f : 0.17677669529663687f;
  uint32_t qa[KS][4];
  {
    const __nv_bfloat162 sc = __float2bfloat162_rn(HD == 16 ? 0.25f : 1.0f);
    const __nv_bfloat16* p0 = Q + (static_cast<size_t>(b) * nq + r0) * ldq + h * HD + 2 * t;
    const __nv_bfloat16* p1 = Q + (static_cast<size_t>(b) * nq + r1) * ldq + h * HD + 2 * t;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      __nv_bfloat162 v;
      v = __hmul2(*reinterpret_cast<const __nv_bfloat162*>(p0 + ks * 16), sc);     qa[ks][0] = *reinterpret_cast<uint32_t*>(&v);
      v = __hmul2(*reinterpret_cast<const __nv_bfloat162*>(p1 + ks * 16), sc);     qa[ks][1] = *reinterpret_cast<uint32_t*>(&v);
      v = __hmul2(*reinterpret_cast<const __nv_bfloat162*>(p0 + ks * 16 + 8), sc); qa[ks][2] = *reinterpret_cast<uint32_t*>(&v);
      v = __hmul2(*reinterpret_cast<const __nv_bfloat162*>(p1 + ks * 16 + 8), sc); qa[ks][3] = *reinterpret_cast<uint32_t*>(&v);
    }
  }
  const uint32_t sK0 = smem_u32(&sK[0][0]), sV0 = smem_u32(&sV[0][0]);
  constexpr uint32_t BUF = MHA_KC * ROWB;
  const int nchunks = (nk + MHA_KC - 1) / MHA_KC;
  auto issue = [&](int c, int buf) {
#pragma unroll
    for (int i = 0; i < PARTS; ++i) {
      const int piece = threadIdx.x + i * MHA_WARPS * 32;       // 2 * 64 * PARTS pieces of 16 B: K rows then V rows
      const int which = piece / (MHA_KC * PARTS), rem = piece % (MHA_KC * PARTS);
      const int row = rem / PARTS, part = rem % PARTS;
      const int key = min(c * MHA_KC + row, nk - 1);
      const __nv_bfloat16* src = (which ? V + (static_cast<size_t>(b) * nk + key) * ldv
                                        : K + (static_cast<size_t>(b) * nk + key) * ldk) + h * HD + part * 8;
      cp_async16q((which ? sV0 : sK0) + buf * BUF + row * ROWB + part * 16, src);
    }
    asm volatile("cp.async.commit_group;\n" ::);
  };
  issue(0, 0);
  const unsigned long long* mr0 = mask ? mask + (static_cast<size_t>(b) * nq + r0) * mask_words : nullptr;
  const unsigned long long* mr1 = mask ? mask + (static_cast<size_t>(b) * nq + r1) * mask_words : nullptr;
  unsigned long long w0n = mask ? mr0[0] : 0ull, w1n = mask ? mr1[0] : 0ull;

  constexpr float L2E = 1.4426950408889634f, NEG = -1e30f;
  float m0 = NEG, m1 = NEG, l0 = 0.f, l1 = 0.f;
  float o[HD / 8][4];
#pragma unroll
  for (int n = 0; n < HD / 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  for (int c = 0; c < nchunks; ++c) {
    const int buf = c & 1;
    asm volatile("cp.async.wait_all;\n" ::);
    __syncthreads();
    if (c + 1 < nchunks) issue(c + 1, buf ^ 1);
    const unsigned long long w0 = w0n, w1 = w1n;
    if (mask && c + 1 < nchunks) { w0n = mr0[c + 1]; w1n = mr1[c + 1]; }
    if (!active) continue;
    float s[8][4];
    const unsigned char* kb = sK[buf];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t* kr = reinterpret_cast<const uint32_t*>(kb + (8 * j + g) * ROWB);
      s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) mma_bf16_16816q(s[j], qa[ks], kr[ks * 8 + t], kr[ks * 8 + t + 4]);
      if (HD != 16) { s[j][0] *= POST_SCALE; s[j][1] *= POST_SCALE; s[j][2] *= POST_SCALE; s[j][3] *= POST_SCALE; }
    }
    const int kbase = c * MHA_KC;
    float mx0 = NEG, mx1 = NEG;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = 8 * j + 2 * t;
      const bool o0 = kbase + col >= nk, o1 = kbase + col + 1 >= nk;
      if (o0 || ((w0 >> col) & 1ull)) s[j][0] = NEG;
      if (o1 || ((w0 >> (col + 1)) & 1ull)) s[j][1] = NEG;
      if (o0 || ((w1 >> col) & 1ull)) s[j][2] = NEG;
      if (o1 || ((w1 >> (col + 1)) & 1ull)) s[j][3] = NEG;
      mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
      mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float a0 = exp2f((m0 - mn0) * L2E), a1 = exp2f((m1 - mn1) * L2E);
    m0 = mn0; m1 = mn1;
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {   // (s - m) first: exact 0 for the -1e30 sentinels (an fma against m * log2e is not)
      s[j][0] = exp2f((s[j][0] - mn0) * L2E); s[j][1] = exp2f((s[j][1] - mn0) * L2E);
      s[j][2] = exp2f((s[j][2] - mn1) * L2E); s[j][3] = exp2f((s[j][3] - mn1) * L2E);
      rs0 += s[j][0] + s[j][1];
      rs1 += s[j][2] + s[j][3];
    }
    l0 = l0 * a0 + rs0; l1 = l1 * a1 + rs1;
#pragma unroll
    for (int n = 0; n < HD / 8; ++n) { o[n][0] *= a0; o[n][1] *= a0; o[n][2] *= a1; o[n][3] *= a1; }
    const uint32_t vb = sV0 + buf * BUF;
    const int mi = lane >> 3, rr = lane & 7;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t pa[4];
      pa[0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
      pa[1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
      pa[2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      pa[3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int np = 0; np < KS; ++np) {        // 16 output channels per ldmatrix.x4.trans
        uint32_t v0, v1, v2, v3;
        const uint32_t addr = vb + (16 * kk + (mi & 1) * 8 + rr) * ROWB + (mi >> 1) * 16 + np * 32;
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                     : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3) : "r"(addr));
        mma_bf16_16816q(o[2 * np], pa, v0, v1);
        mma_bf16_16816q(o[2 * np + 1], pa, v2, v3);
      }
    }
  }
  if (!active) return;
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
  for (int n = 0; n < HD / 8; ++n) {
    if (q0 + g < nq)
      *reinterpret_cast<uint32_t*>(out + (static_cast<size_t>(b) * nq + q0 + g) * E + h * HD + 8 * n + 2 * t) =
          pack_bf16x2(o[n][0] * i0, o[n][1] * i0);
    if (q0 + g + 8 < nq)
      *reinterpret_cast<uint32_t*>(out + (static_cast<size_t>(b) * nq + q0 + g + 8) * E + h * HD + 8 * n + 2 * t) =
          pack_bf16x2(o[n][2] * i1, o[n][3] * i1);
  }
}

int mha_small(const void* Q, int ldq, const void* K, int ldk, const void* V, int ldv, const unsigned long long* mask,
              int B, int nq, int nk, void* out, int head_dim, cudaStream_t stream) {
  RSP_CHECK_ARG(Q && K && V && out && B > 0 && nq > 0 && nk > 0, "mha_small: bad args");
  RSP_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0, "mha_small: leading dims must be multiples of 8");
  RSP_CHECK_ARG(head_dim == 16 || head_dim == 32, "mha_small: head_dim %d (16 or 32 supported)", head_dim);
  dim3 grid(B * 8, (nq + MHA_WARPS * 16 - 1) / (MHA_WARPS * 16));
  if (head_dim == 16)
    mha_kernel<16><<<grid, MHA_WARPS * 32, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(Q), ldq, static_cast<const __nv_bfloat16*>(K), ldk,
        static_cast<const __nv_bfloat16*>(V), ldv, mask, (nk + 63) / 64, nq, nk, static_cast<__nv_bfloat16*>(out));
  else
    mha_kernel<32><<<grid, MHA_WARPS * 32, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(Q), ldq, static_cast<const __nv_bfloat16*>(K), ldk,
        static_cast<const __nv_bfloat16*>(V), ldv, mask, (nk + 63) / 64, nq, nk, static_cast<__nv_bfloat16*>(out));
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ------------------------------------------------------------------------------------ attention mask
// F.interpolate(mask_pred_plus, level size, bilinear) is linear in the mask features, so the level-sized
// logits are (mask_embed) x (bilinearly resized mask_feature)^T: resize_bilinear_nhwc produces the resized
// features once per step, a small GEMM produces logits [B*nq, nk], and this kernel turns a row into bit
// words: masked = sigmoid(x) < 0.5 = (x < 0); a row with every key masked is cleared (M:386-392, M:439-442).
__global__ void attn_mask_bits_kernel(const float* __restrict__ logits, int ld, int nk, int words,
                                      unsigned long long* __restrict__ out) {
  __shared__ unsigned long long sw[64];
  __shared__ int any_open;
  const int row = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* lr = logits + static_cast<size_t>(row) * ld;
  unsigned long long* orow = out + static_cast<size_t>(row) * words;
  int open = 0;
  for (int w0 = 0; w0 < words; w0 += 64) {
    if (threadIdx.x == 0) any_open = 0;
    __syncthreads();
    for (int w = w0 + warp; w < min(words, w0 + 64); w += blockDim.x >> 5) {
      const int k0 = 64 * w + lane, k1 = k0 + 32;
      const bool in0 = k0 < nk, in1 = k1 < nk;
      const bool m0 = in0 ? lr[k0] < 0.f : true, m1 = in1 ? lr[k1] < 0.f : true;
      const unsigned lo = __ballot_sync(0xffffffffu, m0), hi = __ballot_sync(0xffffffffu, m1);
      if ((in0 && !m0) || (in1 && !m1)) open = 1;
      if (lane == 0) sw[w - w0] = static_cast<unsigned long long>(lo) | (static_cast<unsigned long long>(hi) << 32);
    }
    __syncthreads();
    for (int w = w0 + threadIdx.x; w < min(words, w0 + 64); w += blockDim.x) orow[w] = sw[w - w0];
    __syncthreads();
  }
  if (open) any_open = 1;
  __syncthreads();
  if (!any_open)
    for (int w = threadIdx.x; w < words; w += blockDim.x) orow[w] = 0ull;
}

int attn_mask_bits(const float* logits, int ld, int rows, int nk, unsigned long long* out, cudaStream_t stream) {
  RSP_CHECK_ARG(logits && out && rows > 0 && nk > 0 && ld >= nk, "attn_mask_bits: bad args");
  attn_mask_bits_kernel<<<rows, 128, 0, stream>>>(logits, ld, nk, (nk + 63) / 64, out);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// x bf16 [B, H, W, C] -> out bf16 [B, h, w, C], F.interpolate(mode='bilinear', align_corners=False); thread = 8 channels
__global__ void resize_bilinear_nhwc_kernel(const __nv_bfloat16* __restrict__ x, int B, int H, int W, int C, int h, int w,
                                            __nv_bfloat16* __restrict__ out) {
  const int c8 = C >> 3;
  const size_t total = static_cast<size_t>(B) * h * w * c8;
  const float sy = static_cast<float>(H) / h, sx = static_cast<float>(W) / w;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % c8) * 8;
    size_t r = i / c8;
    const int ox = static_cast<int>(r % w); r /= w;
    const int oy = static_cast<int>(r % h);
    const int b = static_cast<int>(r / h);
    const float fy = fmaxf((oy + 0.5f) * sy - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * sx - 0.5f, 0.f);
    const int y0 = min(static_cast<int>(fy), H - 1), x0 = min(static_cast<int>(fx), W - 1);
    const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
    const float wy = fy - y0, wx = fx - x0;
    const float wt[4] = {(1.f - wy) * (1.f - wx), (1.f - wy) * wx, wy * (1.f - wx), wy * wx};
    const int ys[4] = {y0, y0, y1, y1}, xs[4] = {x0, x1, x0, x1};
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, v[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      unpack8f(*reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(b) * H + ys[k]) * W + xs[k]) * C + c), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += wt[k] * v[j];
    }
    *reinterpret_cast<uint4*>(out + i * 8) = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                                                        pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
  }
}

int resize_bilinear_nhwc(const void* x, int B, int H, int W, int C, int h, int w, void* out, cudaStream_t stream) {
  RSP_CHECK_ARG(x && out && B > 0 && H > 0 && W > 0 && h > 0 && w > 0 && C % 8 == 0, "resize_bilinear_nhwc: bad args");
  const size_t total = static_cast<size_t>(B) * h * w * (C / 8);
  const int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, static_cast<size_t>(num_sms()) * 16));
  resize_bilinear_nhwc_kernel<<<blocks, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), B, H, W, C, h, w,
                                                         static_cast<__nv_bfloat16*>(out));
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ------------------------------------------------------------------------------------ mask embedding -> src
struct MaskEmbedW {
  const float *w1, *b1, *g1, *be1;   // conv1 [4,1,2,2], LN(4)
  const float *w2, *b2, *g2, *be2;   // conv2 [16,4,2,2], LN(16)
  const float *w3, *b3;              // conv3 [256,16] (1x1), bias
};

// block = 128 threads x 2 output channels, 32 pixels of one prompt (hidden vector read as 4 x 128-bit LDS)
__global__ void mask_embed_src_kernel(const float* __restrict__ mpp, MaskEmbedW W, const float* __restrict__ emb,
                                      const float* __restrict__ pos, int n_per_img, int hm, int wm, int h, int w,
                                      float eps, __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ src_pe) {
  constexpr int PP = 32;
  __shared__ __align__(16) float hid[PP][16];
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * PP;
  const int HW = h * w;
  if (threadIdx.x < PP && p0 + threadIdx.x < HW) {
    const int pix = p0 + threadIdx.x, y = pix / w, x = pix - y * w;
    const float* in = mpp + (static_cast<size_t>(n) * hm + 4 * y) * wm + 4 * x;
    float h1[2][2][4];
#pragma unroll
    for (int py = 0; py < 2; ++py)
#pragma unroll
      for (int px = 0; px < 2; ++px) {
        float a[4], mean = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float s = W.b1[c];
#pragma unroll
          for (int ky = 0; ky < 2; ++ky)
#pragma unroll
            for (int kx = 0; kx < 2; ++kx) s += W.w1[c * 4 + ky * 2 + kx] * in[(2 * py + ky) * wm + 2 * px + kx];
          a[c] = s; mean += s;
        }
        mean *= 0.25f;
        float var = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) var += (a[c] - mean) * (a[c] - mean);
        const float rstd = rsqrtf(var * 0.25f + eps);
#pragma unroll
        for (int c = 0; c < 4; ++c) h1[py][px][c] = gelu_erf((a[c] - mean) * rstd * W.g1[c] + W.be1[c]);
      }
    float a2[16], mean = 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float s = W.b2[c];
#pragma unroll
      for (int ci = 0; ci < 4; ++ci)
#pragma unroll
        for (int ky = 0; ky < 2; ++ky)
#pragma unroll
          for (int kx = 0; kx < 2; ++kx) s += W.w2[((c * 4 + ci) * 2 + ky) * 2 + kx] * h1[ky][kx][ci];
      a2[c] = s; mean += s;
    }
    mean *= (1.0f / 16.0f);
    float var = 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) var += (a2[c] - mean) * (a2[c] - mean);
    const float rstd = rsqrtf(var * (1.0f / 16.0f) + eps);
#pragma unroll
    for (int c = 0; c < 16; ++c) hid[threadIdx.x][c] = gelu_erf((a2[c] - mean) * rstd * W.g2[c] + W.be2[c]);
  }
  __syncthreads();
  const int c = 2 * threadIdx.x;
  float wa[16], wb[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) { wa[k] = W.w3[c * 16 + k]; wb[k] = W.w3[(c + 1) * 16 + k]; }
  const float ba = W.b3[c], bb = W.b3[c + 1];
  const int img = n / n_per_img;
  const int npix = min(PP, HW - p0);
#pragma unroll 4
  for (int pp = 0; pp < npix; ++pp) {
    float hv[16];
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      const float4 v = *reinterpret_cast<const float4*>(&hid[pp][4 * k4]);
      hv[4 * k4] = v.x; hv[4 * k4 + 1] = v.y; hv[4 * k4 + 2] = v.z; hv[4 * k4 + 3] = v.w;
    }
    float sa = ba, sb = bb;
#pragma unroll
    for (int k = 0; k < 16; ++k) { sa = fmaf(wa[k], hv[k], sa); sb = fmaf(wb[k], hv[k], sb); }
    const int pix = p0 + pp;
    const float2 e = *reinterpret_cast<const float2*>(emb + (static_cast<size_t>(img) * HW + pix) * 256 + c);
    const float2 ps = *reinterpret_cast<const float2*>(pos + static_cast<size_t>(pix) * 256 + c);
    sa += e.x; sb += e.y;
    const size_t o = (static_cast<size_t>(n) * HW + pix) * 256 + c;
    *reinterpret_cast<uint32_t*>(src + o) = pack_bf16x2(sa, sb);
    if (src_pe) *reinterpret_cast<uint32_t*>(src_pe + o) = pack_bf16x2(sa + ps.x, sb + ps.y);
  }
}

// Tensor-core form of the same op for whole 128-pixel blocks (the shipped 64 x 64 embedding grid): thread = pixel for
// the two tiny stride-2 convs (coalesced float4 reads of the 4 x 4 logit patch), then the 16 -> 256 1x1 conv of the
// block runs as mma.sync m16n8k16 tiles (A = the block's 128 x 16 hidden vectors, bf16, from shared memory; B = conv3
// weight [256][16]), and  + bias + image embedding  happens on the accumulator fragments, stored as bf16x2.
// The round-1 kernel above spent 2.7 ms per step on fp32 FMAs with 25 % of the threads idle in the first phase.
__global__ void __launch_bounds__(128)
mask_embed_src_mma_kernel(const float* __restrict__ mpp, MaskEmbedW W, const float* __restrict__ emb, int n_per_img,
                          int hm, int wm, int h, int w, float eps, __nv_bfloat16* __restrict__ src) {
  __shared__ __align__(16) __nv_bfloat16 hid[128][24];      // 16 used + 8 pad: conflict-free fragment reads
  __shared__ __align__(16) __nv_bfloat16 w3s[256][24];
  __shared__ float b3s[256];
  __shared__ __align__(16) float stage[4][16][72];           // per warp: one 16-row x 64-channel fp32 quarter tile (+8 pad)
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * 128;
  const int HW = h * w;
  for (int i = threadIdx.x; i < 256 * 16; i += 128) w3s[i >> 4][i & 15] = __float2bfloat16(W.w3[i]);
  for (int i = threadIdx.x; i < 256; i += 128) b3s[i] = W.b3[i];
  {
    const int pix = p0 + threadIdx.x, y = pix / w, x = pix - y * w;
    const float* in = mpp + (static_cast<size_t>(n) * hm + 4 * y) * wm + 4 * x;
    float v[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(in + static_cast<size_t>(r) * wm));
      v[r][0] = t.x; v[r][1] = t.y; v[r][2] = t.z; v[r][3] = t.w;
    }
    float h1[2][2][4];
#pragma unroll
    for (int py = 0; py < 2; ++py)
#pragma unroll
      for (int px = 0; px < 2; ++px) {
        float a[4], mean = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float s = W.b1[c];
#pragma unroll
          for (int ky = 0; ky < 2; ++ky)
#pragma unroll
            for (int kx = 0; kx < 2; ++kx) s += W.w1[c * 4 + ky * 2 + kx] * v[2 * py + ky][2 * px + kx];
          a[c] = s; mean += s;
        }
        mean *= 0.25f;
        float var = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) var += (a[c] - mean) * (a[c] - mean);
        const float rstd = rsqrtf(var * 0.25f + eps);
#pragma unroll
        for (int c = 0; c < 4; ++c) h1[py][px][c] = gelu_erf((a[c] - mean) * rstd * W.g1[c] + W.be1[c]);
      }
    float a2[16], mean = 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float s = W.b2[c];
#pragma unroll
      for (int ci = 0; ci < 4; ++ci)
#pragma unroll
        for (int ky = 0; ky < 2; ++ky)
#pragma unroll
          for (int kx = 0; kx < 2; ++kx) s += W.w2[((c * 4 + ci) * 2 + ky) * 2 + kx] * h1[ky][kx][ci];
      a2[c] = s; mean += s;
    }
    mean *= (1.0f / 16.0f);
    float var = 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) var += (a2[c] - mean) * (a2[c] - mean);
    const float rstd = rsqrtf(var * (1.0f / 16.0f) + eps);
    uint32_t pk[8];
#pragma unroll
    for (int c = 0; c < 8; ++c)
      pk[c] = pack_bf16x2(gelu_erf((a2[2 * c] - mean) * rstd * W.g2[2 * c] + W.be2[2 * c]),
                          gelu_erf((a2[2 * c + 1] - mean) * rstd * W.g2[2 * c + 1] + W.be2[2 * c + 1]));
    uint4* hp = reinterpret_cast<uint4*>(&hid[threadIdx.x][0]);
    hp[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    hp[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, q = lane & 3;
  const int img = n / n_per_img;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
    const int r0 = warp * 32 + mt * 16;              // first pixel (row) of this 16-row tile inside the block
    uint32_t a[4];                                   // A fragment: rows g / g+8, k = 2q..2q+1 and 2q+8..2q+9
    a[0] = *reinterpret_cast<const uint32_t*>(&hid[r0 + g][2 * q]);
    a[1] = *reinterpret_cast<const uint32_t*>(&hid[r0 + g + 8][2 * q]);
    a[2] = *reinterpret_cast<const uint32_t*>(&hid[r0 + g][2 * q + 8]);
    a[3] = *reinterpret_cast<const uint32_t*>(&hid[r0 + g + 8][2 * q + 8]);
    // The accumulator fragments give a lane 2 channels of rows g / g + 8: stored from there, one warp store touches 8
    // pixel rows x 16 bytes (8 LSU wavefronts per 128 bytes; the kernel ran at 1.4 TB/s, LSU-bound).  Instead the 16 x 64
    // fp32 quarter tiles go through a per-warp staging buffer and leave as whole rows: lane = 2 channels, one wavefront
    // per 128-byte bf16 store and two per 256-byte embedding load.  Same arithmetic order ((acc + bias) + embedding).
    float (*st)[72] = stage[warp];
#pragma unroll 1
    for (int qt = 0; qt < 4; ++qt) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int c0 = qt * 64 + nt * 8;
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&w3s[c0 + g][2 * q]);        // B(k, n) = w3[c0 + n][k]
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&w3s[c0 + g][2 * q + 8]);
        float d[4] = {0.f, 0.f, 0.f, 0.f};
        mma_bf16_16816q(d, a, b0, b1);
        *reinterpret_cast<float2*>(&st[g][nt * 8 + 2 * q]) = make_float2(d[0], d[1]);
        *reinterpret_cast<float2*>(&st[g + 8][nt * 8 + 2 * q]) = make_float2(d[2], d[3]);
      }
      __syncwarp();
      const int c = qt * 64 + 2 * lane;                 // this lane's two output channels
      const float ba = b3s[c], bb = b3s[c + 1];
      const float* e0 = emb + (static_cast<size_t>(img) * HW + p0 + r0) * 256 + c;
      __nv_bfloat16* o0 = src + (static_cast<size_t>(n) * HW + p0 + r0) * 256 + c;
#pragma unroll 8
      for (int r = 0; r < 16; ++r) {
        const float2 v = *reinterpret_cast<const float2*>(&st[r][2 * lane]);
        const float2 e = __ldg(reinterpret_cast<const float2*>(e0 + static_cast<size_t>(r) * 256));
        *reinterpret_cast<uint32_t*>(o0 + static_cast<size_t>(r) * 256) = pack_bf16x2(v.x + ba + e.x, v.y + bb + e.y);
      }
      __syncwarp();
    }
  }
}

int mask_embed_src(const float* mpp, const float* const* wts, const float* emb, const float* pos, int N, int n_per_img,
                   int hm, int wm, int h, int w, float eps, void* src, void* src_pe, cudaStream_t stream) {
  RSP_CHECK_ARG(mpp && wts && emb && pos && src && N > 0 && hm == 4 * h && wm == 4 * w, "mask_embed_src: bad args");
  MaskEmbedW W{wts[0], wts[1], wts[2], wts[3], wts[4], wts[5], wts[6], wts[7], wts[8], wts[9]};
  // whole 128-pixel blocks without src_pe take the tensor-core kernel, every other shape the fp32 one
  if (!src_pe && (h * w) % 128 == 0 && w % 4 == 0 && (reinterpret_cast<uintptr_t>(mpp) & 15) == 0) {
    dim3 grid(h * w / 128, N);
    mask_embed_src_mma_kernel<<<grid, 128, 0, stream>>>(mpp, W, emb, n_per_img, hm, wm, h, w, eps,
                                                        static_cast<__nv_bfloat16*>(src));
    RSP_CHECK_LAUNCH();
    return RSP_OK;
  }
  dim3 grid((h * w + 31) / 32, N);
  mask_embed_src_kernel<<<grid, 128, 0, stream>>>(mpp, W, emb, pos, n_per_img, hm, wm, h, w, eps,
                                                  static_cast<__nv_bfloat16*>(src), static_cast<__nv_bfloat16*>(src_pe));
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// SamMaskEmbedding alone, fp32 out: the dense prompt embedding of HF SamPromptEncoder.forward (HF:691-692) as
// channels-last rows [B*h*w, 256].  A kernel of its own (the two above feed the query head and stay as they are):
// block = 32 pixels of one mask; thread = pixel for the two stride-2 convs, then thread = 2 output channels for the 1x1.
__global__ void sam_mask_embed_kernel(const float* __restrict__ masks, MaskEmbedW W, int hm, int wm, int h, int w,
                                      float eps, float* __restrict__ dense) {
  constexpr int PP = 32;
  __shared__ __align__(16) float hid[PP][16];
  const int b = blockIdx.y;
  const int p0 = blockIdx.x * PP;
  const int HW = h * w;
  if (threadIdx.x < PP && p0 + threadIdx.x < HW) {
    const int pix = p0 + threadIdx.x, y = pix / w, x = pix - y * w;
    const float* in = masks + (static_cast<size_t>(b) * hm + 4 * y) * wm + 4 * x;
    float h1[2][2][4];
#pragma unroll
    for (int py = 0; py < 2; ++py)
#pragma unroll
      for (int px = 0; px < 2; ++px) {
        float a[4], mean = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float s = W.b1[c];
#pragma unroll
          for (int ky = 0; ky < 2; ++ky)
#pragma unroll
            for (int kx = 0; kx < 2; ++kx) s += W.w1[c * 4 + ky * 2 + kx] * in[(2 * py + ky) * wm + 2 * px + kx];
          a[c] = s; mean += s;
        }
        mean *= 0.25f;
        float var = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) var += (a[c] - mean) * (a[c] - mean);
        const float rstd = rsqrtf(var * 0.25f + eps);
#pragma unroll
        for (int c = 0; c < 4; ++c) h1[py][px][c] = gelu_erf((a[c] - mean) * rstd * W.g1[c] + W.be1[c]);
      }
    float a2[16], mean = 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float s = W.b2[c];
#pragma unroll
      for (int ci = 0; ci < 4; ++ci)
#pragma unroll
        for (int ky = 0; ky < 2; ++ky)
#pragma unroll
          for (int kx = 0; kx < 2; ++kx) s += W.w2[((c * 4 + ci) * 2 + ky) * 2 + kx] * h1[ky][kx][ci];
      a2[c] = s; mean += s;
    }
    mean *= (1.0f / 16.0f);
    float var = 0.f;
#pragma unroll
    for (int c = 0; c < 16; ++c) var += (a2[c] - mean) * (a2[c] - mean);
    const float rstd = rsqrtf(var * (1.0f / 16.0f) + eps);
#pragma unroll
    for (int c = 0; c < 16; ++c) hid[threadIdx.x][c] = gelu_erf((a2[c] - mean) * rstd * W.g2[c] + W.be2[c]);
  }
  __syncthreads();
  const int c = 2 * threadIdx.x;
  float wa[16], wb[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) { wa[k] = W.w3[c * 16 + k]; wb[k] = W.w3[(c + 1) * 16 + k]; }
  const float ba = W.b3[c], bb = W.b3[c + 1];
  const int npix = min(PP, HW - p0);
#pragma unroll 4
  for (int pp = 0; pp < npix; ++pp) {
    float hv[16];
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      const float4 v = *reinterpret_cast<const float4*>(&hid[pp][4 * k4]);
      hv[4 * k4] = v.x; hv[4 * k4 + 1] = v.y; hv[4 * k4 + 2] = v.z; hv[4 * k4 + 3] = v.w;
    }
    float sa = ba, sb = bb;
#pragma unroll
    for (int k = 0; k < 16; ++k) { sa = fmaf(wa[k], hv[k], sa); sb = fmaf(wb[k], hv[k], sb); }
    *reinterpret_cast<float2*>(dense + (static_cast<size_t>(b) * HW + p0 + pp) * 256 + c) = make_float2(sa, sb);
  }
}

int sam_mask_embed(const float* masks, const float* const* wts, int B, int hm, int wm, int h, int w, float eps,
                   float* dense, cudaStream_t stream) {
  RSP_CHECK_ARG(masks && wts && dense && B > 0 && h > 0 && w > 0 && hm == 4 * h && wm == 4 * w,
                "sam_mask_embed: bad args");
  RSP_CHECK_ARG((reinterpret_cast<uintptr_t>(dense) & 7) == 0, "sam_mask_embed: dense must be 8-byte aligned");
  MaskEmbedW W{wts[0], wts[1], wts[2], wts[3], wts[4], wts[5], wts[6], wts[7], wts[8], wts[9]};
  dim3 grid((h * w + 31) / 32, B);
  sam_mask_embed_kernel<<<grid, 128, 0, stream>>>(masks, W, hm, wm, h, w, eps, dense);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

// ------------------------------------------------------------------------------------ query post-process
// grid (rows / QP_ROWS, instances); logits fp32 [n_maps, hm, wm]; sel int32 [n_inst] map index of each instance.
// The mask kernels write the boolean mask and per-block partials (sum sigmoid over positives, count, bbox) reduced by
// query_finalize_kernel in a fixed order (deterministic).  Two families: the x4 tile kernel for the mask decoder's
// image / 4 logits, and query_mask_px_kernel, which takes each pixel's value from OneResize or TwoResizes.
constexpr int QP_ROWS = 16;

// The block's (sum, count, min / max x, min / max y) over a fixed tree (deterministic) -> its 6-float partial.  Every
// thread of the block calls it; blockDim.x <= 256.
__device__ __forceinline__ void qp_block_partial(float sum, int cnt, int minx, int maxx, int miny, int maxy,
                                                 float* __restrict__ part) {
  __shared__ float s_sum[256];
  __shared__ int s_i[256][5];
  s_sum[threadIdx.x] = sum;
  s_i[threadIdx.x][0] = cnt; s_i[threadIdx.x][1] = minx; s_i[threadIdx.x][2] = maxx;
  s_i[threadIdx.x][3] = miny; s_i[threadIdx.x][4] = maxy;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      s_sum[threadIdx.x] += s_sum[threadIdx.x + s];
      s_i[threadIdx.x][0] += s_i[threadIdx.x + s][0];
      s_i[threadIdx.x][1] = min(s_i[threadIdx.x][1], s_i[threadIdx.x + s][1]);
      s_i[threadIdx.x][2] = max(s_i[threadIdx.x][2], s_i[threadIdx.x + s][2]);
      s_i[threadIdx.x][3] = min(s_i[threadIdx.x][3], s_i[threadIdx.x + s][3]);
      s_i[threadIdx.x][4] = max(s_i[threadIdx.x][4], s_i[threadIdx.x + s][4]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float* o = part + (static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x) * 6;
    o[0] = s_sum[0]; o[1] = static_cast<float>(s_i[0][0]); o[2] = static_cast<float>(s_i[0][1]);
    o[3] = static_cast<float>(s_i[0][2]); o[4] = static_cast<float>(s_i[0][3]); o[5] = static_cast<float>(s_i[0][4]);
  }
}

// Block = QP_ROWS rows of the (H, W) mask of instance blockIdx.y; a thread takes PX consecutive pixels of a row per
// step (PX = 4: one uchar4 store, W % 4 == 0).  The pixel -> thread order fixes each thread's fast-sigmoid sum, so
// it decides the scores' bits.  BITS: the mask goes bit-packed into record slots [n, Hr, Wr/8] (Wr % 16 == 0), the
// (H, W) mask at the slot's top-left and 0 elsewhere: the block's rows collect in a shared bitmap (QP_ROWS x Wr/32
// words) and leave as one uint16 store per 16 pixels.  Otherwise bytes [n, H, W] (Hr = H, Wr = W).
template <class Sampler, int PX, bool BITS>
__global__ void query_mask_px_kernel(Sampler s, const int* __restrict__ sel, int H, int W, int Hr, int Wr,
                                     unsigned char* __restrict__ out, float* __restrict__ part) {
  extern __shared__ uint32_t s_bits[];
  const int words = (Wr + 31) / 32;
  if (BITS) {
    for (int i = threadIdx.x; i < QP_ROWS * words; i += blockDim.x) s_bits[i] = 0u;
    __syncthreads();
  }
  const int inst = blockIdx.y, m = sel[inst];
  float sum = 0.f;
  int cnt = 0, minx = W, maxx = -1, miny = H, maxy = -1;
  const int y_base = blockIdx.x * QP_ROWS, wp = W / PX;
  for (int i = threadIdx.x; i < QP_ROWS * wp; i += blockDim.x) {
    const int y = y_base + i / wp, xp = i % wp;
    if (y >= H) break;
    s.row(m, y);
    unsigned char r[4];
#pragma unroll
    for (int k = 0; k < PX; ++k) {
      const int x = PX * xp + k;
      const float v = s.at(x);
      const bool on = v > 0.f;
      r[k] = on;
      if (on) {
        if (BITS) atomicOr(&s_bits[(y - y_base) * words + (x >> 5)], 1u << (x & 31));
        sum += __fdividef(1.f, 1.f + __expf(-v));   // fast sigmoid: ~2 ulp, the sum is an average over >= 1e3 pixels
        ++cnt;
        minx = min(minx, x); maxx = max(maxx, x); miny = min(miny, y); maxy = max(maxy, y);
      }
    }
    if (!BITS) {
      unsigned char* o = out + (static_cast<size_t>(inst) * H + y) * W + PX * xp;
      if (PX == 4) *reinterpret_cast<uchar4*>(o) = make_uchar4(r[0], r[1], r[2], r[3]);
      else *o = r[0];
    }
  }
  if (BITS) {
    __syncthreads();
    for (int i = threadIdx.x; i < QP_ROWS * (Wr / 16); i += blockDim.x) {
      const int rr = i / (Wr / 16), k = i % (Wr / 16);
      const int y = y_base + rr;
      if (y >= Hr) break;
      const uint32_t w = s_bits[rr * words + (k >> 1)];
      *reinterpret_cast<uint16_t*>(out + (static_cast<size_t>(inst) * Hr + y) * (Wr / 8) + 2 * k) =
          static_cast<uint16_t>(k & 1 ? w >> 16 : w);
    }
  }
  qp_block_partial(sum, cnt, minx, maxx, miny, maxy, part);
}

// x4 fast path: block = 16 output rows of one instance (see query_mask_px_kernel for the partials); thread = 4 x 16 tile
// PACKED: masks is the bit-packed record payload (H rows of W/8 bytes, pixel x = bit x%8 of byte x/8, i.e.
// numpy packbits(bitorder='little')); a thread writes its 16 pixels of a row as one uint16.
template <bool PACKED>
__global__ void query_mask_x4_kernel(const float* __restrict__ logits, const int* __restrict__ sel, int hm, int wm,
                                     unsigned char* __restrict__ masks, float* __restrict__ part) {
  const int inst = blockIdx.y;
  const float* src = logits + static_cast<size_t>(sel[inst]) * hm * wm;
  const int H = 4 * hm, W = 4 * wm, w4 = wm / 4;
  float sum = 0.f;
  int cnt = 0, minx = W, maxx = -1, miny = H, maxy = -1;
  for (int t = threadIdx.x; t < 4 * w4; t += blockDim.x) {
    const int yb = blockIdx.x * 4 + t / w4, xb = t % w4;
    if (yb >= hm) break;
    Up4Tile tile;
    up4_load(src, hm, wm, yb, xb, tile);
    const int ldm = PACKED ? W / 8 : W;       // bytes per mask row
    unsigned char* o = masks + (static_cast<size_t>(inst) * H + 4 * yb) * ldm + (PACKED ? 2 : 16) * xb;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint32_t packed[4] = {0u, 0u, 0u, 0u};
      uint32_t bits = 0u;
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const float v = up4_value(tile, j, k);
        if (v > 0.f) {
          sum += __fdividef(1.f, 1.f + __expf(-v));   // fast sigmoid: ~2 ulp, the sum is an average over >= 1e3 pixels
          bits |= 1u << k;
          if (!PACKED) packed[k >> 2] |= 1u << ((k & 3) * 8);
        }
      }
      if (PACKED) *reinterpret_cast<uint16_t*>(o + static_cast<size_t>(j) * ldm) = static_cast<uint16_t>(bits);
      else *reinterpret_cast<uint4*>(o + static_cast<size_t>(j) * W) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
      if (bits) {
        cnt += __popc(bits);
        minx = min(minx, 16 * xb + __ffs(bits) - 1);
        maxx = max(maxx, 16 * xb + 31 - __clz(bits));
        miny = min(miny, 4 * yb + j);
        maxy = max(maxy, 4 * yb + j);
      }
    }
  }
  qp_block_partial(sum, cnt, minx, maxx, miny, maxy, part);
}

__global__ void query_finalize_kernel(const float* __restrict__ part, int nblk, const float* __restrict__ cls_scores,
                                      int n_inst, int W, int H, float* __restrict__ scores, float* __restrict__ boxes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_inst) return;
  float sum = 0.f, cnt = 0.f, minx = static_cast<float>(W), maxx = -1.f, miny = static_cast<float>(H), maxy = -1.f;
  for (int b = 0; b < nblk; ++b) {
    const float* o = part + (static_cast<size_t>(i) * nblk + b) * 6;
    sum += o[0]; cnt += o[1];
    minx = fminf(minx, o[2]); maxx = fmaxf(maxx, o[3]); miny = fminf(miny, o[4]); maxy = fmaxf(maxy, o[5]);
  }
  scores[i] = cls_scores[i] * (sum / (cnt + 1e-6f));
  const bool any = cnt > 0.f;
  boxes[i * 4 + 0] = any ? minx : 0.f; boxes[i * 4 + 1] = any ? miny : 0.f;
  boxes[i * 4 + 2] = any ? maxx + 1.f : 0.f; boxes[i * 4 + 3] = any ? maxy + 1.f : 0.f;
}

// checks the mask kernel's launch, then reduces its partials of grid (nblk, n_inst) into scores and boxes
static int query_finalize(const float* part_ws, int nblk, const float* cls_scores, int n_inst, int H, int W,
                          float* scores, float* boxes, cudaStream_t stream) {
  RSP_CHECK_LAUNCH();
  query_finalize_kernel<<<(n_inst + 127) / 128, 128, 0, stream>>>(part_ws, nblk, cls_scores, n_inst, W, H, scores, boxes);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

template <int PX, bool BITS, class Sampler>
static int query_px(const Sampler& s, const int* sel, const float* cls_scores, int n_inst, int H, int W, int Hr, int Wr,
                    unsigned char* out, float* part_ws, float* scores, float* boxes, cudaStream_t stream) {
  // BITS: blocks past row H contribute empty partials (+0 to the sums), so scores equal the byte path's
  const int nblk = (Hr + QP_ROWS - 1) / QP_ROWS;
  const size_t smem = BITS ? QP_ROWS * ((Wr + 31) / 32) * sizeof(uint32_t) : 0;
  query_mask_px_kernel<Sampler, PX, BITS><<<dim3(nblk, n_inst), 256, smem, stream>>>(s, sel, H, W, Hr, Wr, out, part_ws);
  return query_finalize(part_ws, nblk, cls_scores, n_inst, H, W, scores, boxes, stream);
}

int query_postprocess(const float* logits, const int* sel, const float* cls_scores, int n_inst, int hm, int wm, int H,
                      int W, unsigned char* masks, float* part_ws, float* scores, float* boxes, cudaStream_t stream) {
  RSP_CHECK_ARG(logits && sel && cls_scores && masks && part_ws && scores && boxes && n_inst > 0 && W % 4 == 0,
                "query_postprocess: bad args");
  if (H == 4 * hm && W == 4 * wm && wm % 4 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0) {
    const int nblk = (H + QP_ROWS - 1) / QP_ROWS;
    query_mask_x4_kernel<false><<<dim3(nblk, n_inst), 256, 0, stream>>>(logits, sel, hm, wm, masks, part_ws);
    return query_finalize(part_ws, nblk, cls_scores, n_inst, H, W, scores, boxes, stream);
  }
  return query_px<4, false>(OneResize<false, true>{logits, hm, wm, H, W}, sel, cls_scores, n_inst, H, W, H, W, masks, part_ws,
                            scores, boxes, stream);
}

int query_postprocess_bits(const float* logits, const int* sel, const float* cls_scores, int n_inst, int hm, int wm,
                           unsigned char* bits, float* part_ws, float* scores, float* boxes, cudaStream_t stream) {
  RSP_CHECK_ARG(logits && sel && cls_scores && bits && part_ws && scores && boxes && n_inst > 0 && wm % 4 == 0 &&
                (reinterpret_cast<uintptr_t>(logits) & 15) == 0 && (reinterpret_cast<uintptr_t>(bits) & 1) == 0,
                "query_postprocess_bits: needs wm % 4 == 0 and 16-byte aligned logits (x4 path only)");
  const int H = 4 * hm, W = 4 * wm;
  const int nblk = (H + QP_ROWS - 1) / QP_ROWS;
  query_mask_x4_kernel<true><<<dim3(nblk, n_inst), 256, 0, stream>>>(logits, sel, hm, wm, bits, part_ws);
  return query_finalize(part_ws, nblk, cls_scores, n_inst, H, W, scores, boxes, stream);
}

int query_postprocess_rescale(const float* logits, const int* sel, const float* cls_scores, int n_inst, int hm, int wm,
                              int Hb, int Wb, int crop_h, int crop_w, int H, int W, unsigned char* masks, float* part_ws,
                              float* scores, float* boxes, cudaStream_t stream) {
  RSP_CHECK_ARG(logits && sel && cls_scores && masks && part_ws && scores && boxes && n_inst > 0 && crop_h > 0 &&
                crop_w > 0 && crop_h <= Hb && crop_w <= Wb && H > 0 && W > 0, "query_postprocess_rescale: bad args");
  const TwoResizes s{logits, {hm, wm, Hb, Wb, crop_h, crop_w, H, W}};
  return query_px<1, false>(s, sel, cls_scores, n_inst, H, W, H, W, masks, part_ws, scores, boxes, stream);
}

int query_postprocess_rescale_bits(const float* logits, const int* sel, const float* cls_scores, int n_inst, int hm,
                                   int wm, int Hb, int Wb, int crop_h, int crop_w, int H, int W, int Hr, int Wr,
                                   unsigned char* bits, float* part_ws, float* scores, float* boxes,
                                   cudaStream_t stream) {
  RSP_CHECK_ARG(logits && sel && cls_scores && bits && part_ws && scores && boxes && n_inst > 0 && crop_h > 0 &&
                crop_w > 0 && crop_h <= Hb && crop_w <= Wb && H > 0 && W > 0 && H <= Hr && W <= Wr &&
                Wr % 16 == 0 && Wr <= 16384 && (reinterpret_cast<uintptr_t>(bits) & 1) == 0,
                "query_postprocess_rescale_bits: bad args (H <= Hr, W <= Wr, Wr % 16 == 0, Wr <= 16384, 2-byte "
                "aligned bits)");
  const TwoResizes s{logits, {hm, wm, Hb, Wb, crop_h, crop_w, H, W}};
  return query_px<1, true>(s, sel, cls_scores, n_inst, H, W, Hr, Wr, bits, part_ws, scores, boxes, stream);
}

// ------------------------------------------------------------------------------------ panoptic post-process
// MaskFormerFusionHead.panoptic_postprocess (maskformer_fusion_head.py:41-106) for every image of a batch, in three
// passes with no host read between them (the reference reads two counts per kept query back to the host):
//   argmax  per pixel, argmax over the kept queries of score * sigmoid(logit) (first query on ties, as torch.argmax),
//           the query index as uint16 (PAN_NONE: nothing kept), one bit for sigmoid(best) >= 0.5, and per query the
//           integer counts original_area (sigmoid >= 0.5) and mask_area (argmax == q)
//   decide  per image, the kept queries in order: skip, or the segment id (instance ids advance on written things)
//   write   the int32 map from the index map, the bit and the segment ids
// Queries are addressed by their index: the kept queries in kept order are the kept indices in ascending order.
constexpr int PAN_THREADS = 256, PAN_PPT = 8;
constexpr int PAN_TILE = PAN_THREADS * PAN_PPT;   // a block's pixels: PAN_TILE consecutive pixels in raster order
constexpr int PAN_CHUNK = 2048;                   // queries per round of block-local counts
constexpr int PAN_NONE = 0xffff;
constexpr int PAN_INSTANCE_OFFSET = 1000;         // mmdet.evaluation.functional.INSTANCE_OFFSET

// adds `one` of the calling lane to counter s_cnt[key - c0] for keys in [c0, c1), one shared atomic per distinct key
__device__ __forceinline__ void pan_count(int* s_cnt, int key, int c0, int c1) {
  const bool in = key >= c0 && key < c1;
  const unsigned act = __ballot_sync(0xffffffffu, in);
  if (!in) return;
  const unsigned peers = __match_any_sync(act, key);
  if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&s_cnt[key - c0], __popc(peers));
}

// grid (ceil(H*W / PAN_TILE), images); sampler map index = image * nq + query.  areas: mask_area [images, nq] then
// original_area [images, nq], zeroed by the caller; the integer sums do not depend on the order of the atomics.
template <class Sampler>
__global__ void __launch_bounds__(PAN_THREADS)
panoptic_argmax_kernel(Sampler s, const uint8_t* __restrict__ keep, const float* __restrict__ scores, int nq, int H,
                       int W, uint16_t* __restrict__ idx, uint32_t* __restrict__ bits, int* __restrict__ mask_area,
                       int* __restrict__ orig_area) {
  __shared__ int s_cnt[PAN_CHUNK];
  const int img = blockIdx.y, lane = threadIdx.x & 31;
  const int HW = H * W;
  const int p0 = blockIdx.x * PAN_TILE;
  int py[PAN_PPT], px[PAN_PPT], bi[PAN_PPT];
  float best[PAN_PPT];
#pragma unroll
  for (int j = 0; j < PAN_PPT; ++j) {
    const int p = p0 + j * PAN_THREADS + threadIdx.x;
    py[j] = p < HW ? p / W : -1;
    px[j] = p - (p / W) * W;
    best[j] = -1.f;                 // every prob is >= 0: the first kept query takes the pixel
    bi[j] = PAN_NONE;               // bit 16: sigmoid(best) >= 0.5
  }
  const uint8_t* kp = keep + static_cast<size_t>(img) * nq;
  const float* sp = scores + static_cast<size_t>(img) * nq;
  for (int c0 = 0; c0 < nq; c0 += PAN_CHUNK) {
    const int c1 = min(nq, c0 + PAN_CHUNK);
    for (int i = threadIdx.x; i < c1 - c0; i += PAN_THREADS) s_cnt[i] = 0;
    __syncthreads();
    for (int q = c0; q < c1; ++q) {
      if (!kp[q]) continue;
      const float sc = sp[q];
      const int m = img * nq + q;
      int cnt = 0;
#pragma unroll
      for (int j = 0; j < PAN_PPT; ++j) {
        if (py[j] < 0) continue;
        s.row(m, py[j]);
        const float sig = 1.f / (1.f + expf(-s.at(px[j])));      // torch's CUDA sigmoid
        const float prob = __fmul_rn(sc, sig);
        const bool on = sig >= 0.5f;
        cnt += on;
        if (prob > best[j]) { best[j] = prob; bi[j] = q | (on ? 0x10000 : 0); }
      }
      cnt = __reduce_add_sync(0xffffffffu, cnt);
      if (lane == 0 && cnt) atomicAdd(&s_cnt[q - c0], cnt);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < c1 - c0; i += PAN_THREADS)
      if (s_cnt[i]) atomicAdd(&orig_area[static_cast<size_t>(img) * nq + c0 + i], s_cnt[i]);
    __syncthreads();
  }
  for (int c0 = 0; c0 < nq; c0 += PAN_CHUNK) {
    const int c1 = min(nq, c0 + PAN_CHUNK);
    for (int i = threadIdx.x; i < c1 - c0; i += PAN_THREADS) s_cnt[i] = 0;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < PAN_PPT; ++j) pan_count(s_cnt, py[j] < 0 ? -1 : bi[j] & 0xffff, c0, c1);
    __syncthreads();
    for (int i = threadIdx.x; i < c1 - c0; i += PAN_THREADS)
      if (s_cnt[i]) atomicAdd(&mask_area[static_cast<size_t>(img) * nq + c0 + i], s_cnt[i]);
    __syncthreads();
  }
  const size_t base = static_cast<size_t>(img) * HW;
  const size_t wbase = static_cast<size_t>(img) * ((HW + 31) / 32);
#pragma unroll
  for (int j = 0; j < PAN_PPT; ++j) {
    const int p = p0 + j * PAN_THREADS + threadIdx.x;
    if (p < HW) idx[base + p] = static_cast<uint16_t>(bi[j] & 0xffff);
    const unsigned word = __ballot_sync(0xffffffffu, p < HW && (bi[j] >> 16));
    if (lane == 0 && p < HW) bits[wbase + p / 32] = word;     // p % 32 == 0: the warp's 32 pixels are one word
  }
}

// one thread per image: maskformer_fusion_head.py:83-104 over the kept queries in order.  seg[q]: the segment id
// written where the argmax is q, or -1 (skipped or not kept: those pixels keep num_classes).
__global__ void panoptic_decide_kernel(const uint8_t* __restrict__ keep, const int* __restrict__ labels,
                                       const int* __restrict__ mask_area, const int* __restrict__ orig_area, int n_img,
                                       int nq, int num_things, double iou_thr, int* __restrict__ seg) {
  const int img = blockIdx.x * blockDim.x + threadIdx.x;
  if (img >= n_img) return;
  int instance_id = 1;
  for (int q = 0; q < nq; ++q) {
    const size_t i = static_cast<size_t>(img) * nq + q;
    int v = -1;
    const int ma = mask_area[i], oa = orig_area[i];
    // Python's true division of the two counts (correctly rounded double) against the float threshold
    if (keep[i] && ma > 0 && oa > 0 && !(static_cast<double>(ma) / static_cast<double>(oa) < iou_thr)) {
      const int label = labels[i];
      v = label < num_things ? label + instance_id++ * PAN_INSTANCE_OFFSET : label;
    }
    seg[i] = v;
  }
}

// grid (ceil(H*W / 256), images): pan = seg[argmax] where it is not -1 (and, with filter_low_score, where
// sigmoid(best) >= 0.5), num_classes everywhere else
__global__ void panoptic_write_kernel(const uint16_t* __restrict__ idx, const uint32_t* __restrict__ bits,
                                      const int* __restrict__ seg, int nq, int HW, int num_classes, int filter_low_score,
                                      int* __restrict__ pan) {
  const int img = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const size_t o = static_cast<size_t>(img) * HW + p;
  const int k = idx[o];
  int v = num_classes;
  if (k != PAN_NONE) {
    const int sv = seg[static_cast<size_t>(img) * nq + k];
    const bool on = (bits[static_cast<size_t>(img) * ((HW + 31) / 32) + p / 32] >> (p & 31)) & 1u;
    if (sv >= 0 && (!filter_low_score || on)) v = sv;
  }
  pan[o] = v;
}

template <class Sampler>
static int panoptic_run(const Sampler& s, const uint8_t* keep, const float* scores, const int* labels, int n_img,
                        int nq, int H, int W, int num_things, int num_classes, double iou_thr, int filter_low_score,
                        uint16_t* idx_ws, uint32_t* bits_ws, int* areas, int* seg, int* pan, cudaStream_t stream) {
  const int HW = H * W;
  const size_t n = static_cast<size_t>(n_img) * nq;
  RSP_CHECK_CUDA(cudaMemsetAsync(areas, 0, 2 * n * sizeof(int), stream));
  panoptic_argmax_kernel<Sampler><<<dim3((HW + PAN_TILE - 1) / PAN_TILE, n_img), PAN_THREADS, 0, stream>>>(
      s, keep, scores, nq, H, W, idx_ws, bits_ws, areas, areas + n);
  RSP_CHECK_LAUNCH();
  panoptic_decide_kernel<<<(n_img + 31) / 32, 32, 0, stream>>>(keep, labels, areas, areas + n, n_img, nq, num_things,
                                                              iou_thr, seg);
  RSP_CHECK_LAUNCH();
  panoptic_write_kernel<<<dim3((HW + 255) / 256, n_img), 256, 0, stream>>>(idx_ws, bits_ws, seg, nq, HW, num_classes,
                                                                          filter_low_score, pan);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

#define RSP_PANOPTIC_ARGS_OK                                                                                          \
  (logits && keep && scores && labels && idx_ws && bits_ws && areas && seg && pan && n_img > 0 && n_img <= 65535 &&     \
   nq > 0 && nq < PAN_NONE && hm > 0 && wm > 0 && H > 0 && W > 0 &&                                                     \
   static_cast<long long>(H) * W <= 0x7fffffffLL - PAN_TILE && num_things >= 0 && num_things <= num_classes &&      \
   num_classes < PAN_INSTANCE_OFFSET &&                                                                              \
   static_cast<long long>(nq) * PAN_INSTANCE_OFFSET + num_classes <= 0x7fffffffLL && iou_thr)

int panoptic_postprocess(const float* logits, const uint8_t* keep, const float* scores, const int* labels, int n_img,
                         int nq, int hm, int wm, int H, int W, int num_things, int num_classes, const double* iou_thr,
                         int filter_low_score, uint16_t* idx_ws, uint32_t* bits_ws, int* areas, int* seg, int* pan,
                         cudaStream_t stream) {
  RSP_CHECK_ARG(RSP_PANOPTIC_ARGS_OK, "panoptic_postprocess: bad args (nq < 65535, num_classes < 1000)");
  return panoptic_run(OneResize<false, true>{logits, hm, wm, H, W}, keep, scores, labels, n_img, nq, H, W, num_things,
                      num_classes, *iou_thr, filter_low_score, idx_ws, bits_ws, areas, seg, pan, stream);
}

int panoptic_postprocess_rescale(const float* logits, const uint8_t* keep, const float* scores, const int* labels,
                                 int n_img, int nq, int hm, int wm, int Hb, int Wb, int crop_h, int crop_w, int H, int W,
                                 int num_things, int num_classes, const double* iou_thr, int filter_low_score,
                                 uint16_t* idx_ws, uint32_t* bits_ws, int* areas, int* seg, int* pan,
                                 cudaStream_t stream) {
  RSP_CHECK_ARG(RSP_PANOPTIC_ARGS_OK && crop_h > 0 && crop_w > 0 && crop_h <= Hb && crop_w <= Wb,
                "panoptic_postprocess_rescale: bad args (nq < 65535, num_classes < 1000, crop within the batch shape)");
  const TwoResizes s{logits, {hm, wm, Hb, Wb, crop_h, crop_w, H, W}};
  return panoptic_run(s, keep, scores, labels, n_img, nq, H, W, num_things, num_classes, *iou_thr, filter_low_score,
                      idx_ws, bits_ws, areas, seg, pan, stream);
}
#undef RSP_PANOPTIC_ARGS_OK

}  // namespace rsp
