// Persistent, warp-specialised bf16 GEMM for sm_90a:  out = epilogue(A[M,K] * W[N,K]^T)
//
//   warp 0 (1 lane)  TMA producer: A and W tiles -> 128B-swizzled smem ring (mbarrier tx);
//                    runs ahead into the next tile while the consumers are in their epilogue
//   warps 4-11       two consumer warpgroups: wgmma 64 x BN x 16 (rows 64 wg ..), fp32
//                    accumulators in registers, then through a shared-memory tile to
//   warps 4-7        the epilogue (thread = output row): bias / GELU / ReLU /
//                    residual add / row scatter, bf16 or fp32 stores
//
// This one kernel is every dense contraction on the RSPrompter inference path:
// ViT qkv / proj / MLP linears (reference: transformers modeling_sam.py SamVisionAttention
// .qkv/.proj, SamMLPBlock; mmpretrain vit_sam.py:189-190,282), patch-embed and neck convs
// after re-layout, FPN / RPN / RoI-head convs and FCs, and the mask decoder's image-token
// projections.  window_unpartition (modeling_sam.py:925-952) is the `row_map` scatter in
// the epilogue, the residual adds of SamVisionLayer.forward (:966-971) are `residual`.
#include "gemm.h"
#include "sm90.cuh"

#include <stdlib.h>

namespace rsp {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = one 128-byte swizzle row
constexpr int GEMM_THREADS = 384;
constexpr int A_STAGE_BYTES = BM * BK * 2;

template <int BN>
struct GemmCfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int ACC_LD = BN + 4;                       // fp32 accumulator tile row stride
  static constexpr int ACC_BYTES = BM * ACC_LD * 4;
  static constexpr int STAGES = (BN == 256) ? 1 : (BN == 128) ? 4 : (BN == 64) ? 6 : 8;   // 227 KB per block
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + 1024;  // + alignment slack
};

enum { EPI_STD = 0, EPI_LN_ROW = 1, EPI_LN64_GELU = 2, EPI_GELU_HYPER = 3 };

struct GemmDev {
  int M, N, K;
  const float* bias;
  const void* residual;
  void* out;
  const int* row_map;
  int res_mod;
  int ldo, ldr;
  int act;
  int out_fp32;
  int res_fp32;
  int num_n_blocks;
  int num_tiles;
  // --- epilogue variants (mask decoder) ---
  int epi_mode;               // EPI_STD / EPI_LN_ROW / EPI_LN64_GELU / EPI_GELU_HYPER
  const float* ln_gamma;      // [N] (row LN) or [64] (grouped LN)
  const float* ln_beta;
  float ln_eps;
  const int* res_block_map;   // residual row = res_block_map[row / res_block_rows] * res_block_rows + row % res_block_rows
  int res_block_rows;
  const float* hyper;         // [n_prompts, 32]
  float* mask_out;            // [n_prompts, 4*grid_h, 4*grid_w]
  int grid_h, grid_w;
};

__device__ __forceinline__ int residual_row(const GemmDev& p, int orow) {
  if (p.res_block_map) {
    const int blk = orow / p.res_block_rows;
    return p.res_block_map[blk] * p.res_block_rows + (orow - blk * p.res_block_rows);
  }
  return p.res_mod > 0 ? (orow % p.res_mod) : orow;
}

// v[0..31] += bias[col0..] ; v += residual[rrow, col0..]   (col0 + 32 <= N, 16-byte aligned)
__device__ __forceinline__ void add_bias_residual32(const GemmDev& p, float (&v)[32], int rrow, int col0) {
  if (p.bias) {
    const float4* b4 = reinterpret_cast<const float4*>(p.bias + col0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 b = __ldg(b4 + i);
      v[4 * i + 0] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
    }
  }
  if (p.residual) {
    if (p.res_fp32) {
      const float4* r4 = reinterpret_cast<const float4*>(
          static_cast<const float*>(p.residual) + static_cast<size_t>(rrow) * p.ldr + col0);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 x = r4[i];
        v[4 * i + 0] += x.x; v[4 * i + 1] += x.y; v[4 * i + 2] += x.z; v[4 * i + 3] += x.w;
      }
    } else {
      const uint4* r4 = reinterpret_cast<const uint4*>(
          static_cast<const __nv_bfloat16*>(p.residual) + static_cast<size_t>(rrow) * p.ldr + col0);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint4 x = r4[i];
        const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&w[j]);
          v[8 * i + 2 * j + 0] += __bfloat162float(h.x);
          v[8 * i + 2 * j + 1] += __bfloat162float(h.y);
        }
      }
    }
  }
}

__device__ __forceinline__ void store32(const GemmDev& p, const float (&v)[32], int orow, int col0) {
  if (p.out_fp32) {
    float4* o4 = reinterpret_cast<float4*>(static_cast<float*>(p.out) + static_cast<size_t>(orow) * p.ldo + col0);
#pragma unroll
    for (int i = 0; i < 8; ++i) o4[i] = make_float4(v[4 * i + 0], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
  } else {
    uint4* o4 = reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(p.out) + static_cast<size_t>(orow) * p.ldo + col0);
#pragma unroll
    for (int i = 0; i < 4; ++i)
      o4[i] = make_uint4(pack_bf16x2(v[8 * i + 0], v[8 * i + 1]), pack_bf16x2(v[8 * i + 2], v[8 * i + 3]),
                         pack_bf16x2(v[8 * i + 4], v[8 * i + 5]), pack_bf16x2(v[8 * i + 6], v[8 * i + 7]));
  }
}

// EPI_LN_ROW: out = LayerNorm_N(acc + bias + residual) (N <= BN, one n-block: the thread owns the
// whole row in the accumulator tile; two passes over it, statistics in fp32).  SamTwoWayAttentionBlock
// layer_norm4 fused into cross_attn_image_to_token.out_proj (HF:341-347).
template <int BN>
__device__ __forceinline__ void epilogue_ln_row(const GemmDev& p, uint32_t t_row, int orow, int rrow) {
  // shifted sums (pivot = the row's first value): no E[x^2] - E[x]^2 cancellation for rows with a large mean
  float sum = 0.f, sq = 0.f, piv = 0.f;
  const int nch = p.N / 32;
  for (int c = 0; c < nch; ++c) {
    uint32_t r[32];
    acc_ld32(t_row + (c * 32) * 4, r);
    if (orow < 0) continue;
    float v[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]);
    add_bias_residual32(p, v, rrow, c * 32);
    if (c == 0) piv = v[0];
#pragma unroll
    for (int i = 0; i < 32; ++i) { const float d = v[i] - piv; sum += d; sq += d * d; }
  }
  const float dmean = sum / p.N;
  const float mean = piv + dmean;
  const float rstd = rsqrtf(fmaxf(sq / p.N - dmean * dmean, 0.f) + p.ln_eps);
  for (int c = 0; c < nch; ++c) {
    uint32_t r[32];
    acc_ld32(t_row + (c * 32) * 4, r);
    if (orow < 0) continue;
    float v[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]);
    add_bias_residual32(p, v, rrow, c * 32);
    const float4* g4 = reinterpret_cast<const float4*>(p.ln_gamma + c * 32);
    const float4* b4 = reinterpret_cast<const float4*>(p.ln_beta + c * 32);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 g = __ldg(g4 + i), b = __ldg(b4 + i);
      v[4 * i + 0] = (v[4 * i + 0] - mean) * rstd * g.x + b.x;
      v[4 * i + 1] = (v[4 * i + 1] - mean) * rstd * g.y + b.y;
      v[4 * i + 2] = (v[4 * i + 2] - mean) * rstd * g.z + b.z;
      v[4 * i + 3] = (v[4 * i + 3] - mean) * rstd * g.w + b.w;
    }
    store32(p, v, orow, c * 32);
  }
}

// EPI_LN64_GELU: columns are (tap, 64 channels); out = GELU(LN_64(acc + bias)) per tap:
// upscale_conv1 (ConvTranspose2d k2 s2 as a GEMM over taps) + upscale_layer_norm + GELU (HF:519-521).
template <int BN>
__device__ __forceinline__ void epilogue_ln64_gelu(const GemmDev& p, uint32_t t_row, int orow, int n_blk) {
  for (int gi = 0; gi < BN / 64; ++gi) {
    const int col0 = n_blk * BN + gi * 64;
    uint32_t r0[32], r1[32];
    acc_ld32(t_row + (gi * 64) * 4, r0);
    acc_ld32(t_row + (gi * 64 + 32) * 4, r1);
    if (orow < 0 || col0 >= p.N) continue;
    float v[64];
#pragma unroll
    for (int i = 0; i < 32; ++i) { v[i] = __uint_as_float(r0[i]); v[32 + i] = __uint_as_float(r1[i]); }
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) { v[i] += __ldg(p.bias + col0 + i); sum += v[i]; }
    const float mean = sum * (1.0f / 64.0f);
    float var = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) { const float d = v[i] - mean; var += d * d; }
    const float rstd = rsqrtf(var * (1.0f / 64.0f) + p.ln_eps);
    uint4* o4 = reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(p.out) + static_cast<size_t>(orow) * p.ldo + col0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float y[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 8 * i + j;
        y[j] = gelu_erf((v[c] - mean) * rstd * __ldg(p.ln_gamma + c) + __ldg(p.ln_beta + c));
      }
      o4[i] = make_uint4(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]), pack_bf16x2(y[4], y[5]),
                         pack_bf16x2(y[6], y[7]));
    }
  }
}

// EPI_GELU_HYPER: rows are (prompt, y, x, tap1) of the first upscale, columns (tap2, 32 channels) of
// upscale_conv2; mask[prompt, 4y+2ty1+ty2, 4x+2tx1+tx2] = sum_c GELU(acc + bias)[tap2, c] * hyper[prompt, c]
// (HF:521-531): the 32 x 4h x 4w upscaled embedding never leaves the SM.
template <int BN>
__device__ __forceinline__ void epilogue_gelu_hyper(const GemmDev& p, uint32_t t_row, int row) {
  const bool valid = row < p.M;
  const int rows_per_prompt = p.grid_h * p.grid_w * 4;
  const int n = valid ? row / rows_per_prompt : 0;
  const int rem = row - n * rows_per_prompt;
  const int tap1 = rem & 3, pix = rem >> 2;
  const int y = pix / p.grid_w, x = pix - y * p.grid_w;
  float hyp[32];
  if (valid) {
    const float4* h4 = reinterpret_cast<const float4*>(p.hyper + static_cast<size_t>(n) * 32);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 h = __ldg(h4 + i);
      hyp[4 * i] = h.x; hyp[4 * i + 1] = h.y; hyp[4 * i + 2] = h.z; hyp[4 * i + 3] = h.w;
    }
  }
  float m[4];
#pragma unroll
  for (int t2 = 0; t2 < 4; ++t2) {
    uint32_t r[32];
    acc_ld32(t_row + (t2 * 32) * 4, r);
    float acc = 0.f;
    if (valid) {
#pragma unroll
      for (int i = 0; i < 32; ++i)
        acc += gelu_erf(__uint_as_float(r[i]) + __ldg(p.bias + t2 * 32 + i)) * hyp[i];
    }
    m[t2] = acc;
  }
  if (valid) {
    const int W4 = 4 * p.grid_w;
    const int Y = 4 * y + 2 * (tap1 >> 1), X = 4 * x + 2 * (tap1 & 1);
    float* o = p.mask_out + (static_cast<size_t>(n) * 4 * p.grid_h + Y) * W4 + X;
    *reinterpret_cast<float2*>(o) = make_float2(m[0], m[1]);
    *reinterpret_cast<float2*>(o + W4) = make_float2(m[2], m[3]);
  }
}

template <int BN, bool B_MN_MAJOR>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tma_a,
                       const __grid_constant__ CUtensorMap tma_b, const GemmDev p) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[STAGES];
  __shared__ __align__(8) uint64_t bar_empty[STAGES];

  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t acc_base = smem_base + STAGES * Cfg::STAGE_BYTES;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_kb = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0 && lane == 0) {
    // ------------------------------------------------------------ TMA producer
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int m_blk = tile / p.num_n_blocks;
      const int n_blk = tile % p.num_n_blocks;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(smem_u32(&bar_empty[stage]), phase ^ 1);
        const uint32_t full = smem_u32(&bar_full[stage]);
        const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES;
        const uint32_t sb = sa + A_STAGE_BYTES;
        mbar_expect_tx(full, Cfg::STAGE_BYTES);
        tma_load_2d(sa, &tma_a, full, kb * BK, m_blk * BM);
        if (!B_MN_MAJOR) {
          tma_load_2d(sb, &tma_b, full, kb * BK, n_blk * BN);
        } else {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j)
            tma_load_2d(sb + j * (BK * 128), &tma_b, full, n_blk * BN + j * 64, kb * BK);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    for (int i = 0; i < STAGES; ++i) {   // tail: leave no "empty" completion without a waiter (see gemm_v2.cu)
      mbar_wait(smem_u32(&bar_empty[stage]), phase ^ 1);
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------ consumers: wgmma, then epilogue (warps 4-7)
    const int wg = (warp - 4) >> 2;
    const int ew = warp - 4;
    int stage = 0;
    uint32_t phase = 0;
    const bool vec_ok = (p.ldo % 8 == 0) && (p.residual == nullptr || p.ldr % 8 == 0) &&
                        ((reinterpret_cast<uintptr_t>(p.out) & 15) == 0) &&
                        ((reinterpret_cast<uintptr_t>(p.residual) & 15) == 0) &&
                        ((reinterpret_cast<uintptr_t>(p.bias) & 15) == 0);
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int m_blk = tile / p.num_n_blocks;
      const int n_blk = tile % p.num_n_blocks;
      float acc[BN / 2];
      wg_mainloop<BN, B_MN_MAJOR, STAGES>(acc, smem_base, Cfg::STAGE_BYTES, A_STAGE_BYTES, num_kb, wg, stage, phase,
                                          bar_full, bar_empty);
      named_bar_sync(1, 256);   // the previous tile's epilogue has read the accumulator tile
      acc_store<BN>(acc, acc_base, Cfg::ACC_LD, wg, threadIdx.x & 127);
      named_bar_sync(1, 256);
      if (ew >= 4) continue;
      const int row = m_blk * BM + ew * 32 + lane;
      int orow = -1;
      if (row < p.M) orow = p.row_map ? p.row_map[row] : row;
      const int rrow = (orow >= 0 && p.residual) ? residual_row(p, orow) : orow;
      const uint32_t t_row = acc_row(acc_base, Cfg::ACC_LD, ew * 32 + lane);
      if (p.epi_mode == EPI_LN_ROW) {
        epilogue_ln_row<BN>(p, t_row, orow, rrow);
      } else if (p.epi_mode == EPI_LN64_GELU) {
        if constexpr (BN >= 64) epilogue_ln64_gelu<BN>(p, t_row, orow, n_blk);
      } else if (p.epi_mode == EPI_GELU_HYPER) {
        if constexpr (BN == 128) epilogue_gelu_hyper<BN>(p, t_row, row);
      } else
#pragma unroll 1
      for (int c = 0; c < BN / 32; ++c) {
        uint32_t r[32];
        acc_ld32(t_row + (c * 32) * 4, r);
        const int col0 = n_blk * BN + c * 32;
        if (orow < 0 || col0 >= p.N) continue;
        float v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]);
        const bool full_chunk = (col0 + 32 <= p.N) && vec_ok;
        if (full_chunk) {
          if (p.bias) {
            const float4* b4 = reinterpret_cast<const float4*>(p.bias + col0);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float4 b = __ldg(b4 + i);
              v[4 * i + 0] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
            }
          }
          if (p.act == 1) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = gelu_erf(v[i]);
          } else if (p.act == 2) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.0f);
          }
          if (p.residual) {
            if (p.res_fp32) {
              const float4* r4 = reinterpret_cast<const float4*>(
                  static_cast<const float*>(p.residual) + static_cast<size_t>(rrow) * p.ldr + col0);
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float4 x = r4[i];
                v[4 * i + 0] += x.x; v[4 * i + 1] += x.y; v[4 * i + 2] += x.z; v[4 * i + 3] += x.w;
              }
            } else {
              const uint4* r4 = reinterpret_cast<const uint4*>(
                  static_cast<const __nv_bfloat16*>(p.residual) + static_cast<size_t>(rrow) * p.ldr +
                  col0);
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const uint4 x = r4[i];
                const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&w[j]);
                  v[8 * i + 2 * j + 0] += __bfloat162float(h.x);
                  v[8 * i + 2 * j + 1] += __bfloat162float(h.y);
                }
              }
            }
          }
          if (p.out_fp32) {
            float4* o4 = reinterpret_cast<float4*>(static_cast<float*>(p.out) +
                                                   static_cast<size_t>(orow) * p.ldo + col0);
#pragma unroll
            for (int i = 0; i < 8; ++i)
              o4[i] = make_float4(v[4 * i + 0], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
          } else {
            uint4* o4 = reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(p.out) +
                                                 static_cast<size_t>(orow) * p.ldo + col0);
#pragma unroll
            for (int i = 0; i < 4; ++i)
              o4[i] = make_uint4(pack_bf16x2(v[8 * i + 0], v[8 * i + 1]),
                                 pack_bf16x2(v[8 * i + 2], v[8 * i + 3]),
                                 pack_bf16x2(v[8 * i + 4], v[8 * i + 5]),
                                 pack_bf16x2(v[8 * i + 6], v[8 * i + 7]));
          }
        } else {
          // ragged / unaligned tail: scalar path
          for (int i = 0; i < 32; ++i) {
            const int col = col0 + i;
            if (col >= p.N) break;
            float x = v[i];
            if (p.bias) x += p.bias[col];
            if (p.act == 1) x = gelu_erf(x);
            else if (p.act == 2) x = fmaxf(x, 0.0f);
            if (p.residual) {
              const size_t ri = static_cast<size_t>(rrow) * p.ldr + col;
              x += p.res_fp32 ? static_cast<const float*>(p.residual)[ri]
                              : __bfloat162float(static_cast<const __nv_bfloat16*>(p.residual)[ri]);
            }
            const size_t oi = static_cast<size_t>(orow) * p.ldo + col;
            if (p.out_fp32) static_cast<float*>(p.out)[oi] = x;
            else static_cast<__nv_bfloat16*>(p.out)[oi] = __float2bfloat16_rn(x);
          }
        }
      }
    }
  }
}

static void fill_dev(GemmDev& p, const GemmArgs& a) {
  p.M = a.M; p.N = a.N; p.K = a.K;
  p.bias = a.bias; p.residual = a.residual; p.out = a.out; p.row_map = a.row_map;
  p.res_mod = a.res_mod; p.ldo = a.ldo; p.ldr = a.ldr; p.act = a.act;
  p.out_fp32 = a.out_fp32; p.res_fp32 = a.res_fp32;
  p.epi_mode = a.epi_mode; p.ln_gamma = a.ln_gamma; p.ln_beta = a.ln_beta; p.ln_eps = a.ln_eps;
  p.res_block_map = a.res_block_map; p.res_block_rows = a.res_block_rows;
  p.hyper = a.hyper; p.mask_out = a.mask_out; p.grid_h = a.grid_h; p.grid_w = a.grid_w;
  p.num_n_blocks = 0; p.num_tiles = 0;
}

template <int BN, bool B_MN>
static int launch_gemm(const GemmArgs& a, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  CUtensorMap ta, tb;
  RSP_TRY(make_tmap_bf16_2d(&ta, a.A, a.M, a.K, static_cast<uint64_t>(a.lda) * 2, BM, BK));
  if (!B_MN) {
    RSP_TRY(make_tmap_bf16_2d(&tb, a.W, a.N, a.K, static_cast<uint64_t>(a.ldw) * 2, BN, BK));
  } else {
    // W given as [K, N] row-major (N contiguous): boxes of 64 N-elements x 64 K-rows
    RSP_TRY(make_tmap_bf16_2d(&tb, a.W, a.K, a.N, static_cast<uint64_t>(a.ldw) * 2, BK, 64));
  }
  GemmDev p;
  fill_dev(p, a);
  const int num_m_blocks = (a.M + BM - 1) / BM;
  p.num_n_blocks = (a.N + BN - 1) / BN;
  p.num_tiles = num_m_blocks * p.num_n_blocks;
  auto kern = gemm_bf16_wgmma_kernel<BN, B_MN>;
  static bool attr_set_dev[kMaxDevices] = {};   // the attribute is per device (one flag per ordinal)
  bool& attr_set = attr_set_dev[current_device()];
  if (!attr_set) {
    RSP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        Cfg::SMEM_BYTES));
    attr_set = true;
  }
  int grid = p.num_tiles < num_sms() ? p.num_tiles : num_sms();
  if (a.max_ctas > 0 && grid > a.max_ctas) grid = a.max_ctas;
  kern<<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(ta, tb, p);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

int gemm_upscale_masks(const GemmArgs& a, int n_out, cudaStream_t stream) {
  RSP_CHECK_ARG(a.A && a.W && a.bias && a.hyper && a.mask_out, "gemm_upscale_masks: null pointer");
  RSP_CHECK_ARG(n_out >= 1 && n_out <= 3, "gemm_upscale_masks: n_out %d (1 to 3)", n_out);
  RSP_CHECK_ARG(a.M > 0 && a.K > 0 && a.N == 128 && a.lda % 8 == 0 && a.ldw % 8 == 0 && a.grid_h > 0 &&
                a.grid_w > 0 && a.grid_w % 2 == 0 && a.M % (4 * a.grid_h * a.grid_w) == 0,
                "gemm_upscale_masks: needs N == 128, an even grid_w and M = prompts * 4 * h * w");
  auto al = [](const void* ptr, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1)) == 0; };
  // float4 hyper and bias loads, float2 mask stores
  RSP_CHECK_ARG(al(a.hyper, 16) && al(a.bias, 16) && al(a.mask_out, 8), "gemm_upscale_masks: alignment");
  return gemm_bf16_v2_gelu_hyper_multi(a, n_out, stream);
}

int gemm_bf16(const GemmArgs& a, cudaStream_t stream) {
  RSP_CHECK_ARG(a.A && a.W && (a.out || a.mask_out), "gemm: null pointer");
  RSP_CHECK_ARG(a.M > 0 && a.N > 0 && a.K > 0, "gemm: bad shape %d %d %d", a.M, a.N, a.K);
  RSP_CHECK_ARG(a.lda % 8 == 0 && a.ldw % 8 == 0, "gemm: lda/ldw must be multiples of 8 bf16");
  RSP_CHECK_ARG(a.act >= 0 && a.act <= 2, "gemm: act %d", a.act);
  if (a.res_block_map) RSP_CHECK_ARG(a.res_block_rows > 0, "gemm: res_block_rows");
  auto al = [](const void* ptr, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1)) == 0; };
  // The fused epilogues make vector accesses (16-byte rows, float4 / float2 loads and stores) whose alignment is
  // checked here, before any kernel is chosen: a misaligned pointer is rejected, never handed to a fallback.
  if (a.epi_mode == EPI_LN_ROW) {
    RSP_CHECK_ARG(a.N % 32 == 0 && a.N <= 256 && a.ln_gamma && a.ln_beta && !a.w_is_kn && !a.row_map,
                  "gemm: row-LN epilogue needs N %% 32 == 0, N <= 256, gamma/beta");
    // both kernels move 16 bytes at a time through out, residual, bias, gamma and beta
    RSP_CHECK_ARG(a.ldo % 8 == 0 && (!a.residual || a.ldr % 8 == 0) && al(a.out, 16) && al(a.residual, 16) &&
                  al(a.bias, 16) && al(a.ln_gamma, 16) && al(a.ln_beta, 16), "gemm: row-LN epilogue alignment");
    if (gemm_v2_ln_row_eligible(a)) return gemm_bf16_v2_ln_row(a, stream);
    if (a.N > 128) return launch_gemm<256, false>(a, stream);
    if (a.N > 64) return launch_gemm<128, false>(a, stream);
    return launch_gemm<64, false>(a, stream);
  }
  if (a.epi_mode == EPI_LN64_GELU) {
    RSP_CHECK_ARG(a.N % 64 == 0 && a.bias && a.ln_gamma && a.ln_beta && !a.out_fp32 && !a.w_is_kn && !a.row_map,
                  "gemm: LN64+GELU epilogue needs N %% 64 == 0, bias, bf16 out");
    static const bool v1 = getenv("RSP_GEMM_V1") != nullptr;
    if (!v1 && a.N % 128 == 0 && al(a.out, 8) && a.ldo % 4 == 0) {
      // float4 bias / gamma / beta loads; out is a TMA store (16-byte aligned rows) or 8-byte stores
      RSP_CHECK_ARG(al(a.bias, 16) && al(a.ln_gamma, 16) && al(a.ln_beta, 16), "gemm: LN64+GELU epilogue alignment");
      return gemm_bf16_v2_ln64_gelu(a, stream);
    }
    // 16-byte stores of 8 bf16 per row
    RSP_CHECK_ARG(al(a.out, 16) && a.ldo % 8 == 0, "gemm: LN64+GELU epilogue output alignment");
    if (a.N % 128 == 0) return launch_gemm<128, false>(a, stream);
    return launch_gemm<64, false>(a, stream);
  }
  if (a.epi_mode == EPI_GELU_HYPER) {
    RSP_CHECK_ARG(a.N == 128 && a.bias && a.hyper && a.mask_out && a.grid_h > 0 && a.grid_w > 0 &&
                  a.M % (4 * a.grid_h * a.grid_w) == 0 && !a.w_is_kn,
                  "gemm: GELU+hyper epilogue needs N == 128 and M = prompts * 4 * h * w");
    // float4 hyper loads, float2 mask stores (at even columns of rows 4 * grid_w wide)
    RSP_CHECK_ARG(al(a.hyper, 16) && al(a.mask_out, 8), "gemm: GELU+hyper epilogue alignment");
    static const bool v1h = getenv("RSP_GEMM_V1") != nullptr;
    if (!v1h && a.grid_w % 2 == 0) {
      RSP_CHECK_ARG(al(a.bias, 16), "gemm: GELU+hyper epilogue bias alignment");   // float4 bias loads
      return gemm_bf16_v2_gelu_hyper(a, stream);
    }
    return launch_gemm<128, false>(a, stream);
  }
  RSP_CHECK_ARG(a.epi_mode == EPI_STD, "gemm: epi_mode %d", a.epi_mode);
  if (a.m_group_rows > 0)
    RSP_CHECK_ARG(a.m_group_rows % BM == 0 && a.M % a.m_group_rows == 0 && a.w_group_rows > 0 && !a.w_is_kn &&
                  a.conv_c == 0 && gemm_v2_eligible(a), "gemm: grouped weights need m_group_rows %% 128 == 0 and the v2 kernel");
  if (a.w_is_kn) {
    RSP_CHECK_ARG(a.N % 64 == 0, "gemm: [K,N] weights need N %% 64 == 0");
    if (a.N % 128 == 0) return launch_gemm<128, true>(a, stream);
    return launch_gemm<64, true>(a, stream);
  }
  int bn = a.force_bn;
  if (bn == 0) {
    // 128 at most: a 256-wide tile's fp32 accumulator tile leaves shared memory for a single pipeline stage
    if (a.N > 64) bn = 128;
    else if (a.N > 32) bn = 64;
    else bn = 32;
  }
  {
    static const bool force_v1 = getenv("RSP_GEMM_V1") != nullptr;
    // the v2 kernel's standard epilogue runs tiles up to 128 wide; an explicit 256 stays on this one
    if ((!force_v1 || a.m_group_rows > 0) && (bn <= 128 || a.m_group_rows > 0) && gemm_v2_eligible(a))
      return gemm_bf16_v2(a, bn, stream);
  }
  switch (bn) {
    case 256: return launch_gemm<256, false>(a, stream);
    case 128: return launch_gemm<128, false>(a, stream);
    case 64: return launch_gemm<64, false>(a, stream);
    case 32: return launch_gemm<32, false>(a, stream);
    default: set_last_error("gemm: unsupported BN %d", bn); return RSP_ERR_INVALID;
  }
}

// ---------------------------------------------------------------------------------------
// 3x3 / stride 1 / pad 1 convolution as an implicit GEMM (no im2col buffer): the A tile of tap (ky, kx) is the
// output-pixel box shifted by (ky - 1, kx - 1), fetched by one 4-D TMA load whose out-of-range rows / columns
// come back as zeros.  A 128-pixel tile must be a whole box of the [B, H, W] pixel grid.
bool conv3x3_geometry_ok(int B, int H, int W, int C) {
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || C % BK != 0) return false;
  const int tw = W < BM ? W : BM;
  if (BM % tw != 0 || W % tw != 0) return false;
  const int th = (BM / tw) < H ? BM / tw : H;
  if (th > 1 && tw != W) return false;
  if (H % th != 0 || BM % (tw * th) != 0) return false;
  const int tb = BM / (tw * th);
  if (tb > 1 && th != H) return false;
  return tw <= 256 && th <= 256 && tb <= 256;
}

int conv3x3_bf16(const GemmArgs& a, cudaStream_t stream) {
  RSP_CHECK_ARG(a.A && a.W && a.out, "conv3x3: null pointer");
  RSP_CHECK_ARG(conv3x3_geometry_ok(a.conv_b, a.conv_h, a.conv_w, a.conv_c),
                "conv3x3: unsupported geometry B=%d H=%d W=%d C=%d (C %% 64, 128-pixel tiles must be boxes)",
                a.conv_b, a.conv_h, a.conv_w, a.conv_c);
  RSP_CHECK_ARG(a.M == a.conv_b * a.conv_h * a.conv_w && a.K == 9 * a.conv_c && a.ldw % 8 == 0 && a.N > 0,
                "conv3x3: M / K do not match the map");
  RSP_CHECK_ARG(a.epi_mode == EPI_STD && !a.w_is_kn && !a.row_map && a.act >= 0 && a.act <= 2, "conv3x3: epilogue");
  RSP_CHECK_ARG(gemm_v2_eligible(a), "conv3x3: output / residual alignment");
  const int bn = a.N > 64 ? 128 : a.N > 32 ? 64 : 32;
  return gemm_bf16_v2(a, bn, stream);
}

// ---------------------------------------------------------------------------------------
// Plain SIMT GEMM with the same epilogue contract.  Used (a) by the device self-test as an
// independent check of the wgmma path and (b) for contractions too small to fill one
// 128-row tile (hypernetwork / IoU MLPs on a handful of tokens).
__global__ void gemm_bf16_simt_kernel(const __nv_bfloat16* __restrict__ A, int lda,
                                      const __nv_bfloat16* __restrict__ W, int ldw, int w_is_kn,
                                      GemmDev p) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = blockIdx.y;
  if (col >= p.N || row >= p.M) return;
  float acc = 0.f;
  if (!w_is_kn) {
    for (int k = 0; k < p.K; ++k)
      acc += __bfloat162float(A[static_cast<size_t>(row) * lda + k]) *
             __bfloat162float(W[static_cast<size_t>(col) * ldw + k]);
  } else {
    for (int k = 0; k < p.K; ++k)
      acc += __bfloat162float(A[static_cast<size_t>(row) * lda + k]) *
             __bfloat162float(W[static_cast<size_t>(k) * ldw + col]);
  }
  const int orow = p.row_map ? p.row_map[row] : row;
  if (orow < 0) return;
  const int rrow = residual_row(p, orow);
  if (p.bias) acc += p.bias[col];
  if (p.act == 1) acc = gelu_erf(acc);
  else if (p.act == 2) acc = fmaxf(acc, 0.f);
  if (p.residual) {
    const size_t ri = static_cast<size_t>(rrow) * p.ldr + col;
    acc += p.res_fp32 ? static_cast<const float*>(p.residual)[ri]
                      : __bfloat162float(static_cast<const __nv_bfloat16*>(p.residual)[ri]);
  }
  const size_t oi = static_cast<size_t>(orow) * p.ldo + col;
  if (p.out_fp32) static_cast<float*>(p.out)[oi] = acc;
  else static_cast<__nv_bfloat16*>(p.out)[oi] = __float2bfloat16_rn(acc);
}

int gemm_bf16_simt(const GemmArgs& a, cudaStream_t stream) {
  RSP_CHECK_ARG(a.A && a.W && a.out, "gemm_simt: null pointer");
  RSP_CHECK_ARG(a.M > 0 && a.N > 0 && a.K > 0, "gemm_simt: bad shape");
  RSP_CHECK_ARG(a.epi_mode == EPI_STD, "gemm_simt: only the standard epilogue");
  GemmDev p;
  fill_dev(p, a);
  dim3 block(128);
  dim3 grid((a.N + 127) / 128, a.M);
  gemm_bf16_simt_kernel<<<grid, block, 0, stream>>>(static_cast<const __nv_bfloat16*>(a.A), a.lda,
                                                    static_cast<const __nv_bfloat16*>(a.W), a.ldw,
                                                    a.w_is_kn, p);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace rsp
