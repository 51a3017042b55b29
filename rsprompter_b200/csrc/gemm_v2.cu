// Persistent, warp-specialised bf16 GEMM for sm_90a:  out = epilogue(A[M,K] * W[N,K]^T), every dense contraction
// of the inference path (gemm_bf16, conv3x3_bf16 and gemm_upscale_masks in gemm.cu check the arguments and call in
// here).  Warp 0 is the TMA producer (A and W tiles -> 128B-swizzled smem ring), two warpgroups run the wgmma
// mainloop (sm90.cuh wg_mainloop) and write the fp32 accumulators into a padded tile in shared memory, from which the
// epilogue (bias, GELU / ReLU, residual, row scatter, bf16 / fp32 out, and the fused LayerNorm / upscaler epilogues)
// takes them:
//   * the epilogue runs on warps of its own (below), each owning 32 rows of the accumulator tile, or on the 8 MMA
//     warps (2 per 32-row quarter, each owning half of the tile's columns);
//   * every warp transposes its 32-row x 128-byte slab through a private, bank-conflict-free smem
//     staging buffer, so global traffic is fully coalesced: each half-warp reads (residual) and
//     writes one whole 128-byte line per instruction instead of 32 lanes touching 32 different
//     lines (a thread-per-row epilogue leaves K = 768 GEMMs epilogue-bound at ~35-55 % of the large-K rate).
//     Rows that are not 8-byte aligned (odd N or ldo, fp32 rows at 4-byte alignment) go through the same staging
//     buffer one element per store.  Only the row LayerNorm of the rows EPI_LN_ROW does not take reads its row per
//     thread (EPI_LN_ROW_T).
// Three schedules share the kernel template:
//   * EPI_STD (plain, implicit-conv3x3 and grouped-weight GEMMs), 512 threads: warp 0 is the TMA producer, warpgroups
//     1-2 only run the wgmma mainloop and write the accumulator tile, warpgroup 3 runs the epilogue from that tile.
//     The tile changes hands through a "tile full" / "tile empty" mbarrier pair, so the MMA warpgroups start the next
//     tile's k-loop while the epilogue of the last one is still running; at BN <= 64 the tile is double-buffered.
//     setmaxnreg moves the producer warpgroup's registers to the MMA and epilogue warpgroups.
//   * the fused epilogues (row LayerNorm, LN64 + GELU, GELU + hypernetwork), 384 threads: the two MMA warpgroups run
//     the epilogue themselves after each tile.
//   * EPI_STD_WIDE (bf16-output plain GEMMs with long k-loops and many tiles), 384 threads, 128 x 256 tiles: the MMA
//     warpgroups run the epilogue from their accumulator registers, with no accumulator tile (epilogue_wide).
// All shared memory is dynamic (1024-byte aligned by declaration), barriers live at its end:
//   [ STAGES x (A 16 KB + B BN*128 B) | epilogue warps x 32 x 136 B staging | ACC_BUFS x 128 x (BN + 4) fp32 | barriers ]
#include "gemm.h"
#include "sm90.cuh"

namespace rsp {

namespace v2 {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_BYTES = BM * BK * 2;
constexpr int STG_ROW = 136;          // 128-byte payload + 8 pad: conflict-free 8-byte accesses
constexpr int STG_WARP = 32 * STG_ROW;
constexpr int BAR_BYTES = 256;
constexpr int SMEM_MAX = 227 * 1024;

// EPI_GELU_HYPER2 / 3: EPI_GELU_HYPER with 2 / 3 hypernetwork vectors per prompt (multimask_output); the output count
// is part of the instantiation, so the single-output kernel is compiled exactly as before.
// EPI_LN_ROW and EPI_LN_ROW_T are the two row-LayerNorm epilogues of epi_mode 1 (see gemm_bf16_v2).
// EPI_STD_WIDE is the standard epilogue (bias, GELU / ReLU, bf16 out by TMA; no residual, no scatter) on 128 x 256
// tiles, run by the MMA warpgroups straight from their accumulator registers (see gemm_bf16_v2 for when it is used).
enum { EPI_STD = 0, EPI_LN_ROW = 1, EPI_LN64_GELU = 2, EPI_GELU_HYPER = 3, EPI_GELU_HYPER2 = 4, EPI_GELU_HYPER3 = 5,
       EPI_LN_ROW_T = 6, EPI_STD_WIDE = 7 };

__host__ __device__ constexpr int hyper_outputs(int epi) { return epi == EPI_GELU_HYPER3 ? 3 : epi == EPI_GELU_HYPER2 ? 2 : 1; }

template <int BN, int EPI>
struct Cfg {
  static constexpr bool SPLIT = EPI == EPI_STD;   // epilogue on its own warpgroup (BN <= 128)
  static_assert(!SPLIT || BN <= 128, "a 64 x 256 wgmma needs more registers than a 512-thread block has per thread");
  // accumulators never leave the registers: no accumulator tile, and 16-row output slabs (one warp's rows)
  static constexpr bool WIDE = EPI == EPI_STD_WIDE;
  static_assert(!WIDE || BN == 256, "the register epilogue is written for the 64 x 256 fragment");
  static constexpr int THREADS = SPLIT ? 512 : 384;
  static constexpr int EPI_WARPS = SPLIT ? 4 : 8;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_LD = BN + 4;
  static constexpr int ACC_BYTES = BM * ACC_LD * 4;
  static constexpr int ACC_BUFS = WIDE ? 0 : (SPLIT && BN <= 64) ? 2 : 1;
  static constexpr int STG_BYTES = EPI_WARPS * STG_WARP;
  static constexpr int STAGES =
      WIDE ? 4 : SPLIT ? ((BN == 128) ? 4 : (BN == 64) ? 5 : 8) : ((BN == 256) ? 1 : 3);   // 227 KB
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STG_BYTES + ACC_BUFS * ACC_BYTES + BAR_BYTES;
  static_assert(SMEM_BYTES <= SMEM_MAX, "shared memory");
  static_assert(2 * STAGES + 8 + 2 * ACC_BUFS <= BAR_BYTES / 8, "barrier area");
  // warps per 32-row quarter of the tile, each owning BN / NHALF columns: two halves when the MMA warpgroups run the
  // epilogue of a wide tile, whole rows for the epilogue warpgroup of the split schedule and for EPI_LN_ROW_T
  // (warps 4-7, thread = row)
  static constexpr int NHALF = (!SPLIT && BN >= 128 && EPI != EPI_LN_ROW_T) ? 2 : 1;
  static constexpr int COLS_PER_WARP = BN / NHALF;
  // setmaxnreg budgets of the split schedule (launched at 128 per thread: producer + 2 x MMA + epilogue <= 4 x 128)
  // and of the wide one (launched at 168: producer + 2 x MMA <= 3 x 168; 128 of the MMA registers are accumulators)
  static constexpr int REG_PRODUCER = 40;
  static constexpr int REG_MMA = WIDE ? 232 : 168;
  static_assert(!WIDE || REG_PRODUCER + 2 * REG_MMA <= 3 * 168, "wide schedule register budget");
  static constexpr int REG_EPI = SPLIT ? 512 - REG_PRODUCER - 2 * REG_MMA : 0;
  static_assert(!SPLIT || (REG_EPI >= 128 && REG_EPI % 8 == 0), "the epilogue warpgroup takes registers, never gives them up");
};

struct Dev {
  int M, N, K;
  const float* bias;
  const void* residual;
  void* out;
  const int* row_map;
  const int* res_block_map;
  int res_block_rows;
  int res_mod;
  int ldo, ldr;
  int act;
  int out_fp32;
  int res_fp32;
  int num_n_blocks;
  int num_tiles;
  // EPI 1 - 3 (the mask decoder's fused epilogues, see rsp_gemm_bf16 in rsp_b200.h for the maths)
  const float* ln_gamma;
  const float* ln_beta;
  float ln_eps;
  const float* hyper;
  float* mask_out;
  int grid_h, grid_w;
  int conv_kb, conv_h, conv_w;   // conv_kb = Cin / 64 k-blocks per tap (0 = plain GEMM)
  int mblk_per_group, w_group_rows;   // grouped weights (0 = one W for every row)
  int tma_store;                 // output leaves through tma_c (no scatter, BN >= 64)
  int tma_res;                   // residual slabs arrive through tma_r into the staging buffer (added in place)
  int scalar_rows;               // standard epilogue: out / residual / bias rows read and written one element at a time
};

__device__ __forceinline__ int num_kblocks(const Dev& p) { return p.conv_kb > 0 ? 9 * p.conv_kb : (p.K + BK - 1) / BK; }

__device__ __forceinline__ int residual_row(const Dev& p, int orow) {
  if (p.res_block_map) {
    const int blk = orow / p.res_block_rows;
    return p.res_block_map[blk] * p.res_block_rows + (orow - blk * p.res_block_rows);
  }
  return p.res_mod > 0 ? (orow % p.res_mod) : orow;
}

// EPI_LN_ROW_T: v[0..31] += bias[col0..] ; v += residual[rrow, col0..]   (col0 + 32 <= N, 16-byte aligned)
__device__ __forceinline__ void add_bias_residual32(const Dev& p, float (&v)[32], int rrow, int col0) {
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

// EPI_LN_ROW_T: out[orow, col0 .. col0 + 31] = v   (16-byte aligned)
__device__ __forceinline__ void store32(const Dev& p, const float (&v)[32], int orow, int col0) {
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

// scalar rows of the standard epilogue: one element of the residual / output
__device__ __forceinline__ float residual_at(const Dev& p, int rrow, int col) {
  const size_t i = static_cast<size_t>(rrow) * p.ldr + col;
  return p.res_fp32 ? static_cast<const float*>(p.residual)[i]
                    : __bfloat162float(static_cast<const __nv_bfloat16*>(p.residual)[i]);
}
__device__ __forceinline__ void store_at(const Dev& p, int orow, int col, float x) {
  const size_t i = static_cast<size_t>(orow) * p.ldo + col;
  if (p.out_fp32) static_cast<float*>(p.out)[i] = x;
  else static_cast<__nv_bfloat16*>(p.out)[i] = __float2bfloat16_rn(x);
}

// Output path of the standard epilogue: chosen per tile, or fixed for a whole loop of tiles
enum { OUT_ANY = 0, OUT_TMA = 1, OUT_SCATTER = 2 };

// One epilogue warp's share of a 128 x BN accumulator tile at acc_base: rows [32 q, 32 q + 32) with q = e & 3,
// columns [hf COLS_PER_WARP, (hf + 1) COLS_PER_WARP).  e also selects the warp's staging buffer and residual barrier.
template <int BN, int EPI, int OUT = OUT_ANY>
__device__ __forceinline__ void epilogue_tile(const Dev& p, const CUtensorMap& tma_c, const CUtensorMap& tma_r,
                                              int m_blk, int n_blk, int e, int hf, uint32_t acc_base,
                                              uint8_t* stg_all, uint64_t* bar_res, uint32_t& rphase) {
  using C = Cfg<BN, EPI>;
  const int lane = threadIdx.x & 31;
  const int q = e & 3;
  uint8_t* stg = stg_all + e * STG_WARP;
  const uint32_t stg_s = smem_u32(stg);
  const bool stage_f32 = p.out_fp32 || (p.residual != nullptr) || p.scalar_rows;
  const int W = stage_f32 ? 32 : (C::COLS_PER_WARP < 64 ? C::COLS_PER_WARP : 64);   // columns per pass
  const int n_pass = C::COLS_PER_WARP / W;
  const int lpr = stage_f32 ? 16 : (W * 2) / 8;     // lanes per row at 8 bytes each
  const int rpi = 32 / lpr;                          // rows per write-out iteration
  const int epl = stage_f32 ? 2 : 4;                 // elements per lane (8 bytes)
  if constexpr (EPI == EPI_GELU_HYPER) {
    // rows = (prompt, y, x, tap1); this warp owns tap2 in {2hf, 2hf+1} = output row 4y + 2ty1 + hf.
    // 16 consecutive lanes (4 x-positions... 8 with both tx1) write one contiguous 128-byte run.
    const int row = m_blk * BM + q * 32 + lane;
    const bool valid = row < p.M;
    const int rows_per_prompt = p.grid_h * p.grid_w * 4;
    const int n = valid ? row / rows_per_prompt : 0;
    const int rem = row - n * rows_per_prompt;
    const int tap1 = rem & 3, pix = rem >> 2;
    const int y = pix / p.grid_w, x = pix - y * p.grid_w;
    float hyp[32];
    {
      const float4* h4 = reinterpret_cast<const float4*>(p.hyper + static_cast<size_t>(n) * 32);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 h = __ldg(h4 + i);
        hyp[4 * i] = h.x; hyp[4 * i + 1] = h.y; hyp[4 * i + 2] = h.z; hyp[4 * i + 3] = h.w;
      }
    }
    const uint32_t t_row = acc_row(acc_base, C::ACC_LD, q * 32 + lane) + 4 * hf * 64;
    float m2[2];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      uint32_t r[32];
      acc_ld32(t_row + (t * 32) * 4, r);
      const float4* b4 = reinterpret_cast<const float4*>(p.bias + hf * 64 + t * 32);
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 b = __ldg(b4 + i);
        acc += gelu_fast(__uint_as_float(r[4 * i]) + b.x) * hyp[4 * i];
        acc += gelu_fast(__uint_as_float(r[4 * i + 1]) + b.y) * hyp[4 * i + 1];
        acc += gelu_fast(__uint_as_float(r[4 * i + 2]) + b.z) * hyp[4 * i + 2];
        acc += gelu_fast(__uint_as_float(r[4 * i + 3]) + b.w) * hyp[4 * i + 3];
      }
      m2[t] = acc;
    }
    if (valid) {
      const int W4 = 4 * p.grid_w;
      const int Y = 4 * y + 2 * (tap1 >> 1) + hf, X = 4 * x + 2 * (tap1 & 1);
      *reinterpret_cast<float2*>(p.mask_out + (static_cast<size_t>(n) * 4 * p.grid_h + Y) * W4 + X) =
          make_float2(m2[0], m2[1]);
    }
  } else if constexpr (EPI == EPI_GELU_HYPER2 || EPI == EPI_GELU_HYPER3) {
    // the EPI_GELU_HYPER tile for NO outputs: hyper [prompt, NO, 32], mask_out [prompt, NO, 4h, 4w].  GELU(acc + bias)
    // is evaluated once per element and feeds NO sums; each sum takes its terms in the single-output order, so output
    // o has the bytes of an EPI_GELU_HYPER launch with hyper[:, o], and the up1 rows are read once instead of NO times
    constexpr int NO = hyper_outputs(EPI);
    const int row = m_blk * BM + q * 32 + lane;
    const bool valid = row < p.M;
    const int rows_per_prompt = p.grid_h * p.grid_w * 4;
    const int n = valid ? row / rows_per_prompt : 0;
    const int rem = row - n * rows_per_prompt;
    const int tap1 = rem & 3, pix = rem >> 2;
    const int y = pix / p.grid_w, x = pix - y * p.grid_w;
    float hyp[NO][32];
#pragma unroll
    for (int o = 0; o < NO; ++o) {
      const float4* h4 = reinterpret_cast<const float4*>(p.hyper + (static_cast<size_t>(n) * NO + o) * 32);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 h = __ldg(h4 + i);
        hyp[o][4 * i] = h.x; hyp[o][4 * i + 1] = h.y; hyp[o][4 * i + 2] = h.z; hyp[o][4 * i + 3] = h.w;
      }
    }
    const uint32_t t_row = acc_row(acc_base, C::ACC_LD, q * 32 + lane) + 4 * hf * 64;
    float m2[NO][2];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      uint32_t r[32];
      acc_ld32(t_row + (t * 32) * 4, r);
      const float4* b4 = reinterpret_cast<const float4*>(p.bias + hf * 64 + t * 32);
      float acc[NO];
#pragma unroll
      for (int o = 0; o < NO; ++o) acc[o] = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 b = __ldg(b4 + i);
        const float g0 = gelu_fast(__uint_as_float(r[4 * i]) + b.x);
        const float g1 = gelu_fast(__uint_as_float(r[4 * i + 1]) + b.y);
        const float g2 = gelu_fast(__uint_as_float(r[4 * i + 2]) + b.z);
        const float g3 = gelu_fast(__uint_as_float(r[4 * i + 3]) + b.w);
#pragma unroll
        for (int o = 0; o < NO; ++o) {
          acc[o] += g0 * hyp[o][4 * i];
          acc[o] += g1 * hyp[o][4 * i + 1];
          acc[o] += g2 * hyp[o][4 * i + 2];
          acc[o] += g3 * hyp[o][4 * i + 3];
        }
      }
#pragma unroll
      for (int o = 0; o < NO; ++o) m2[o][t] = acc[o];
    }
    if (valid) {
      const int W4 = 4 * p.grid_w;
      const int Y = 4 * y + 2 * (tap1 >> 1) + hf, X = 4 * x + 2 * (tap1 & 1);
#pragma unroll
      for (int o = 0; o < NO; ++o)
        *reinterpret_cast<float2*>(p.mask_out + ((static_cast<size_t>(n) * NO + o) * 4 * p.grid_h + Y) * W4 + X) =
            make_float2(m2[o][0], m2[o][1]);
    }
  } else if constexpr (EPI == EPI_LN_ROW_T) {
    // out = LayerNorm_N(acc + bias + residual) for N % 32 == 0, N <= BN (one n-block; BN 128 for N <= 128, 256
    // above): the lane owns the whole row in
    // the accumulator tile, two passes over it, statistics in fp32 taken sequentially over the N / 32 chunks in
    // column order.  Shifted sums (pivot = the row's first value): no E[x^2] - E[x]^2 cancellation for rows with a
    // large mean.  fp32 or bf16 residual and output, res_mod / res_block_map, or no residual: the mask decoder's token
    // norms (SamTwoWayAttentionBlock layer_norm1-3, layer_norm_final_attn, HF:316-338, 398-404) and layer_norm4 where
    // the block map's rows are not whole 32-row slabs.
    const int row = m_blk * BM + q * 32 + lane;
    const int orow = row < p.M ? row : -1;
    const int rrow = (orow >= 0 && p.residual) ? residual_row(p, orow) : orow;
    const uint32_t t_row = acc_row(acc_base, C::ACC_LD, q * 32 + lane);
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
    // sq / N - dmean^2: one rounding at BN 256, two at BN 128, the rounding each tile width has always had.  Written
    // out, because whether ptxas fuses a multiply and a subtract depends on its schedule.
    const float var = BN == 256 ? fmaf(-dmean, dmean, sq / p.N) : __fsub_rn(sq / p.N, __fmul_rn(dmean, dmean));
    const float rstd = rsqrtf(fmaxf(var, 0.f) + p.ln_eps);
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
  } else if constexpr (EPI == EPI_LN_ROW) {
    // out = LayerNorm_256(acc + bias + residual), bf16 (N == BN == 256: the tile holds whole rows).  Two warps
    // share a row (128 columns each).  Pass 1: v = acc + bias + residual (residual slabs arrive by TMA in the
    // staging buffer) is written back over the accumulator tile while sum / sum of squares accumulate;
    // the pair exchanges its partial statistics through shared memory; pass 2 re-reads v from the tile
    // in shared memory, normalises, and leaves through the same staging buffer as TMA stores.
    const uint32_t t_row = acc_row(acc_base, C::ACC_LD, q * 32 + lane) + 4 * hf * 128;
    const int col_warp = hf * 128;
    const int row0 = m_blk * BM + q * 32;
    const uint32_t sbuf = smem_u32(stg_all) + e * 4096;
    const uint32_t srow = sbuf + lane * 128;
    const int sw = lane & 7;
    float2* xchg = reinterpret_cast<float2*>(stg_all + 8 * 4096);   // [2][128] (mean, M2) of each half row
    const bool valid = row0 < p.M;
    const uint32_t rbar = smem_u32(&bar_res[e]);
    int rrow0 = row0;
    if (valid && p.res_block_map) {
      const int blk = row0 / p.res_block_rows;
      rrow0 = __ldg(p.res_block_map + blk) * p.res_block_rows + (row0 - blk * p.res_block_rows);
    }
    auto issue_res = [&](int col0) {
      if (lane == 0) {
        bulk_wait_read0();
        mbar_expect_tx(rbar, 4096);
        tma_load_2d(sbuf, &tma_r, rbar, col0, rrow0);
      }
    };
    if (valid) issue_res(col_warp);
    // shifted sums: d = v - pivot with the pivot = this half row's first value, so a large common offset of the
    // row (keys with a big mean) does not cancel in E[d^2] - E[d]^2; the halves are merged with Chan's formula
    float sum = 0.f, sumsq = 0.f, piv = 0.f;
    bool have_piv = false;
    if (valid) {
#pragma unroll 1
      for (int ps = 0; ps < 2; ++ps) {
        const int col0 = col_warp + ps * 64;
        mbar_wait(rbar, rphase);
        rphase ^= 1;
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          uint32_t r[32];
          acc_ld32(t_row + (ps * 64 + c * 32) * 4, r);
          const float4* b4 = reinterpret_cast<const float4*>(p.bias + col0 + c * 32);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            uint32_t w0, w1, w2, w3;
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                         : "=r"(w0), "=r"(w1), "=r"(w2), "=r"(w3) : "r"(srow + (((c * 4 + j) ^ sw) << 4)));
            const float4 ba = __ldg(b4 + 2 * j), bb = __ldg(b4 + 2 * j + 1);
            float v[8];
            v[0] = __uint_as_float(r[8 * j]) + ba.x + __uint_as_float(w0 << 16);
            v[1] = __uint_as_float(r[8 * j + 1]) + ba.y + __uint_as_float(w0 & 0xffff0000u);
            v[2] = __uint_as_float(r[8 * j + 2]) + ba.z + __uint_as_float(w1 << 16);
            v[3] = __uint_as_float(r[8 * j + 3]) + ba.w + __uint_as_float(w1 & 0xffff0000u);
            v[4] = __uint_as_float(r[8 * j + 4]) + bb.x + __uint_as_float(w2 << 16);
            v[5] = __uint_as_float(r[8 * j + 5]) + bb.y + __uint_as_float(w2 & 0xffff0000u);
            v[6] = __uint_as_float(r[8 * j + 6]) + bb.z + __uint_as_float(w3 << 16);
            v[7] = __uint_as_float(r[8 * j + 7]) + bb.w + __uint_as_float(w3 & 0xffff0000u);
            if (!have_piv) { piv = v[0]; have_piv = true; }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              const float d = v[k] - piv;
              sum += d;
              sumsq = fmaf(d, d, sumsq);
              r[8 * j + k] = __float_as_uint(v[k]);
            }
          }
          acc_st32(t_row + (ps * 64 + c * 32) * 4, r);
        }
        __syncwarp();                         // every lane has read its residual row: the buffer is free
        if (ps == 0) issue_res(col0 + 64);
      }
    }
    const float mean_h = piv + sum * (1.0f / 128.0f);
    const float m2_h = fmaxf(sumsq - sum * sum * (1.0f / 128.0f), 0.f);
    xchg[hf * 128 + q * 32 + lane] = make_float2(mean_h, m2_h);
    asm volatile("bar.sync %0, 64;" ::"r"(1 + q) : "memory");
    const float2 ot = xchg[(hf ^ 1) * 128 + q * 32 + lane];
    const float mean = 0.5f * (mean_h + ot.x);
    const float dm = mean_h - ot.x;
    const float var = (m2_h + ot.y + dm * dm * 64.0f) * (1.0f / 256.0f);     // n0 n1 / (n0 + n1) = 64
    const float rstd = rsqrtf(var + p.ln_eps);
    asm volatile("bar.sync %0, 64;" ::"r"(1 + q) : "memory");   // xchg may be rewritten by the next tile
    if (valid) {
#pragma unroll 1
      for (int ps = 0; ps < 2; ++ps) {
        const int col0 = col_warp + ps * 64;
        uint32_t pk[32];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          uint32_t r[32];
          acc_ld32(t_row + (ps * 64 + c * 32) * 4, r);
          const float4* g4 = reinterpret_cast<const float4*>(p.ln_gamma + col0 + c * 32);
          const float4* e4 = reinterpret_cast<const float4*>(p.ln_beta + col0 + c * 32);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 g = __ldg(g4 + j), bt = __ldg(e4 + j);
            const float y0 = fmaf((__uint_as_float(r[4 * j]) - mean) * rstd, g.x, bt.x);
            const float y1 = fmaf((__uint_as_float(r[4 * j + 1]) - mean) * rstd, g.y, bt.y);
            const float y2 = fmaf((__uint_as_float(r[4 * j + 2]) - mean) * rstd, g.z, bt.z);
            const float y3 = fmaf((__uint_as_float(r[4 * j + 3]) - mean) * rstd, g.w, bt.w);
            pk[c * 16 + 2 * j] = pack_bf16x2(y0, y1);
            pk[c * 16 + 2 * j + 1] = pack_bf16x2(y2, y3);
          }
        }
        if (lane == 0) bulk_wait_read0();
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 8; ++j)
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(srow + ((j ^ sw) << 4)), "r"(pk[4 * j]),
                       "r"(pk[4 * j + 1]), "r"(pk[4 * j + 2]), "r"(pk[4 * j + 3])
                       : "memory");
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) { tma_store_2d(&tma_c, sbuf, col0, row0); bulk_commit(); }
      }
    }
  } else if constexpr (EPI == EPI_LN64_GELU) {
    // this warp owns two 64-column groups (taps); per group: bias, LayerNorm over the 64
    // channels, GELU, bf16 -> staging -> coalesced 128-byte rows
    const int my_row = m_blk * BM + q * 32 + lane;
    const int my_orow = my_row < p.M ? my_row : -1;
    const uint32_t t_row = acc_row(acc_base, C::ACC_LD, q * 32 + lane) + 4 * hf * C::COLS_PER_WARP;
    const int col_warp = n_blk * BN + hf * C::COLS_PER_WARP;
    const int sub = lane >> 4, cl = lane & 15;
#pragma unroll 1
    for (int gi = 0; gi < C::COLS_PER_WARP / 64; ++gi) {
      const int col0 = col_warp + gi * 64;
      if (col0 >= p.N) break;
      float v[64];
      {
        uint32_t r0[32], r1[32];
        acc_ld32(t_row + (gi * 64) * 4, r0);
        acc_ld32(t_row + (gi * 64 + 32) * 4, r1);
#pragma unroll
        for (int i = 0; i < 32; ++i) { v[i] = __uint_as_float(r0[i]); v[32 + i] = __uint_as_float(r1[i]); }
      }
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + col0) + i);
        v[4 * i] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
        sum += v[4 * i] + v[4 * i + 1] + v[4 * i + 2] + v[4 * i + 3];
      }
      const float mean = sum * (1.0f / 64.0f);
      float var = 0.f;
#pragma unroll
      for (int i = 0; i < 64; ++i) { const float d = v[i] - mean; var += d * d; }
      const float rstd = rsqrtf(var * (1.0f / 64.0f) + p.ln_eps);
      if (p.tma_store) {
        // swizzled 32 x 128 B slab -> one TMA store (rows >= M are clipped by the tensor map)
        const uint32_t sbuf = smem_u32(stg_all) + e * 4096;
        const uint32_t srow = sbuf + lane * 128;
        const int sw = lane & 7;
        uint32_t pk[32];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const float4 g = __ldg(reinterpret_cast<const float4*>(p.ln_gamma) + i);
          const float4 bt = __ldg(reinterpret_cast<const float4*>(p.ln_beta) + i);
          const float y0 = gelu_fast((v[4 * i] - mean) * rstd * g.x + bt.x);
          const float y1 = gelu_fast((v[4 * i + 1] - mean) * rstd * g.y + bt.y);
          const float y2 = gelu_fast((v[4 * i + 2] - mean) * rstd * g.z + bt.z);
          const float y3 = gelu_fast((v[4 * i + 3] - mean) * rstd * g.w + bt.w);
          pk[2 * i] = pack_bf16x2(y0, y1);
          pk[2 * i + 1] = pack_bf16x2(y2, y3);
        }
        if (lane == 0) bulk_wait_read0();
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 8; ++j)
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(srow + ((j ^ sw) << 4)), "r"(pk[4 * j]),
                       "r"(pk[4 * j + 1]), "r"(pk[4 * j + 2]), "r"(pk[4 * j + 3])
                       : "memory");
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) { tma_store_2d(&tma_c, sbuf, col0, m_blk * BM + q * 32); bulk_commit(); }
        continue;
      }
      const uint32_t a = stg_s + lane * STG_ROW;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(p.ln_gamma) + i);
        const float4 bt = __ldg(reinterpret_cast<const float4*>(p.ln_beta) + i);
        const float y0 = gelu_fast((v[4 * i] - mean) * rstd * g.x + bt.x);
        const float y1 = gelu_fast((v[4 * i + 1] - mean) * rstd * g.y + bt.y);
        const float y2 = gelu_fast((v[4 * i + 2] - mean) * rstd * g.z + bt.z);
        const float y3 = gelu_fast((v[4 * i + 3] - mean) * rstd * g.w + bt.w);
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a + i * 8), "r"(pack_bf16x2(y0, y1)),
                     "r"(pack_bf16x2(y2, y3))
                     : "memory");
      }
      __syncwarp();
      const int col = col0 + cl * 4;
#pragma unroll 4
      for (int k = 0; k < 16; ++k) {
        const int rr = 2 * k + sub;
        const int orow = __shfl_sync(0xffffffffu, my_orow, rr);
        if (orow < 0) continue;
        uint32_t w0, w1;
        asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(w0), "=r"(w1) : "r"(stg_s + rr * STG_ROW + cl * 8));
        *reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(p.out) + static_cast<size_t>(orow) * p.ldo + col) =
            make_uint2(w0, w1);
      }
      __syncwarp();
    }
  } else if (OUT == OUT_TMA || (OUT == OUT_ANY && p.tma_store)) {
    // ---- lean path: accumulator tile -> registers -> bias / activation -> 128-byte-swizzled staging -> one TMA store per
    // 32 x 128 B slab.  No per-element address or bounds arithmetic: the tensor map clips rows >= M / cols >= N.
    // With a residual, its slab is TMA-loaded into the same staging buffer (issued as soon as the previous
    // store has drained it), added in place by the lane that owns the row, and stored from there.
    const uint32_t t_row = acc_row(acc_base, C::ACC_LD, q * 32 + lane) + 4 * hf * C::COLS_PER_WARP;
    const int col_warp = n_blk * BN + hf * C::COLS_PER_WARP;
    const int row0 = m_blk * BM + q * 32;
    const uint32_t sbuf = smem_u32(stg_all) + e * 4096;
    const uint32_t srow = sbuf + lane * 128;
    const int sw = lane & 7;
    const bool has_res = p.tma_res != 0 && row0 < p.M;
    const uint32_t rbar = smem_u32(&bar_res[e]);
    int rrow0 = row0;
    if (has_res) {
      if (p.res_block_map) {
        const int blk = row0 / p.res_block_rows;
        rrow0 = __ldg(p.res_block_map + blk) * p.res_block_rows + (row0 - blk * p.res_block_rows);
      } else if (p.res_mod > 0) {
        rrow0 = row0 % p.res_mod;
      }
    }
    auto issue_res = [&](int col0) {
      if (lane == 0) {
        bulk_wait_read0();
        mbar_expect_tx(rbar, 4096);
        tma_load_2d(sbuf, &tma_r, rbar, col0, rrow0);
      }
    };
    if (has_res && col_warp < p.N) issue_res(col_warp);
    const int act = p.act;
    const float* bias = p.bias;
    const int N = p.N;
    auto bias_act = [&](float (&v)[32], int col0) {
      if (bias) {
        if (col0 + 32 <= N) {
          const float4* b4 = reinterpret_cast<const float4*>(bias + col0);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 b = __ldg(b4 + i);
            v[4 * i] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
          }
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] += (col0 + i < N) ? __ldg(bias + col0 + i) : 0.f;
        }
      }
      if (act == 1) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = gelu_fast(v[i]);
      } else if (act == 2) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.f);
      }
    };
    if (p.out_fp32) {
#pragma unroll 1
      for (int ps = 0; ps < C::COLS_PER_WARP / 32; ++ps) {
        const int col0 = col_warp + ps * 32;
        if (col0 >= N) break;
        uint32_t r[32];
        acc_ld32(t_row + (ps * 32) * 4, r);
        float v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]);
        bias_act(v, col0);
        if (has_res) {
          mbar_wait(rbar, rphase);
          rphase ^= 1;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float x0, x1, x2, x3;
            asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                         : "=f"(x0), "=f"(x1), "=f"(x2), "=f"(x3) : "r"(srow + ((j ^ sw) << 4)));
            v[4 * j] += x0; v[4 * j + 1] += x1; v[4 * j + 2] += x2; v[4 * j + 3] += x3;
          }
        } else {
          if (lane == 0) bulk_wait_read0();      // the previous slab has left the staging buffer
          __syncwarp();
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
          asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(srow + ((j ^ sw) << 4)), "f"(v[4 * j]),
                       "f"(v[4 * j + 1]), "f"(v[4 * j + 2]), "f"(v[4 * j + 3])
                       : "memory");
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) { tma_store_2d(&tma_c, sbuf, col0, row0); bulk_commit(); }
        if (has_res && ps + 1 < C::COLS_PER_WARP / 32 && col0 + 32 < N) issue_res(col0 + 32);
      }
    } else {
#pragma unroll 1
      for (int ps = 0; ps < C::COLS_PER_WARP / 64; ++ps) {
        const int col0 = col_warp + ps * 64;
        if (col0 >= N) break;
        uint32_t r0[32], r1[32];
        acc_ld32(t_row + (ps * 64) * 4, r0);
        acc_ld32(t_row + (ps * 64 + 32) * 4, r1);
        float v0[32], v1[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) { v0[i] = __uint_as_float(r0[i]); v1[i] = __uint_as_float(r1[i]); }
        bias_act(v0, col0);
        if (col0 + 32 < N) bias_act(v1, col0 + 32);
        if (has_res) {
          mbar_wait(rbar, rphase);
          rphase ^= 1;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            uint32_t w0, w1, w2, w3;
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                         : "=r"(w0), "=r"(w1), "=r"(w2), "=r"(w3) : "r"(srow + ((j ^ sw) << 4)));
            float* vv = j < 4 ? &v0[8 * j] : &v1[8 * (j - 4)];
            vv[0] += __uint_as_float(w0 << 16); vv[1] += __uint_as_float(w0 & 0xffff0000u);
            vv[2] += __uint_as_float(w1 << 16); vv[3] += __uint_as_float(w1 & 0xffff0000u);
            vv[4] += __uint_as_float(w2 << 16); vv[5] += __uint_as_float(w2 & 0xffff0000u);
            vv[6] += __uint_as_float(w3 << 16); vv[7] += __uint_as_float(w3 & 0xffff0000u);
          }
        } else {
          if (lane == 0) bulk_wait_read0();
          __syncwarp();
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(srow + ((j ^ sw) << 4)),
                       "r"(pack_bf16x2(v0[8 * j], v0[8 * j + 1])), "r"(pack_bf16x2(v0[8 * j + 2], v0[8 * j + 3])),
                       "r"(pack_bf16x2(v0[8 * j + 4], v0[8 * j + 5])), "r"(pack_bf16x2(v0[8 * j + 6], v0[8 * j + 7]))
                       : "memory");
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(srow + (((j + 4) ^ sw) << 4)),
                       "r"(pack_bf16x2(v1[8 * j], v1[8 * j + 1])), "r"(pack_bf16x2(v1[8 * j + 2], v1[8 * j + 3])),
                       "r"(pack_bf16x2(v1[8 * j + 4], v1[8 * j + 5])), "r"(pack_bf16x2(v1[8 * j + 6], v1[8 * j + 7]))
                       : "memory");
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) { tma_store_2d(&tma_c, sbuf, col0, row0); bulk_commit(); }
        if (has_res && ps + 1 < C::COLS_PER_WARP / 64 && col0 + 64 < N) issue_res(col0 + 64);
      }
    }
  } else {
    const int my_row = m_blk * BM + q * 32 + lane;
    int my_orow = -1;
    if (my_row < p.M) my_orow = p.row_map ? p.row_map[my_row] : my_row;
    const int my_rrow = (my_orow >= 0 && p.residual) ? residual_row(p, my_orow) : 0;
    const uint32_t t_row = acc_row(acc_base, C::ACC_LD, q * 32 + lane) + 4 * hf * C::COLS_PER_WARP;
    const int col_warp = n_blk * BN + hf * C::COLS_PER_WARP;
    const int sub = lane / lpr, cl = lane - sub * lpr;
    // destination / residual row of tile-local row rr: plain arithmetic when there is no scatter map
    // (warp-uniform choice), otherwise a shuffle from the lane that owns the row
    const bool simple_rows = (p.row_map == nullptr) && (p.res_block_map == nullptr) && (p.res_mod % 32 == 0);
    const int tile_row0 = m_blk * BM + q * 32;
    const int res_row0 = p.res_mod > 0 ? tile_row0 % p.res_mod : tile_row0;   // tiles never straddle res_mod
    auto get_orow = [&](int rr) -> int {
      if (simple_rows) return (tile_row0 + rr < p.M) ? tile_row0 + rr : -1;
      return __shfl_sync(0xffffffffu, my_orow, rr);
    };
    auto get_rrow = [&](int rr) -> int {
      if (simple_rows) return res_row0 + rr;
      return __shfl_sync(0xffffffffu, my_rrow, rr);
    };
    // residual prefetch (fp32-staged path: 16 lanes x 8 B per row, 2 rows per instruction): the 16
    // loads of a pass are issued back to back before the accumulator is touched, so ~4 KB per warp
    // is in flight while the accumulator read / activation of the same pass runs
    float2 resv[16];
    auto load_residual = [&](int col_pass) {
      const int col = col_pass + cl * 2;
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const int rr = 2 * k + sub;
        const int orow = get_orow(rr);
        const int rrow = get_rrow(rr);
        resv[k] = make_float2(0.f, 0.f);
        if (orow >= 0 && col < p.N) {
          if (p.scalar_rows) {
            resv[k].x = residual_at(p, rrow, col);
            if (col + 1 < p.N) resv[k].y = residual_at(p, rrow, col + 1);
          } else if (p.res_fp32) {
            resv[k] = *reinterpret_cast<const float2*>(static_cast<const float*>(p.residual) +
                                                       static_cast<size_t>(rrow) * p.ldr + col);
          } else {
            // keep the raw bits: converting here would make every load wait for its own data
            // before the next one can issue (in-order issue) and serialise the 16 latencies
            resv[k].x = __uint_as_float(*reinterpret_cast<const uint32_t*>(
                static_cast<const __nv_bfloat16*>(p.residual) + static_cast<size_t>(rrow) * p.ldr + col));
          }
        }
      }
    };
    if (p.residual && col_warp < p.N) load_residual(col_warp);
#pragma unroll 1
    for (int ps = 0; ps < n_pass; ++ps) {
      const int col_pass = col_warp + ps * W;
      if (col_pass < p.N) {
        if (p.residual && ps > 0) load_residual(col_pass);
        // ---- phase 1: accumulator tile -> registers -> bias / activation -> staging row `lane`
#pragma unroll 1
        for (int c = 0; c < W / 32; ++c) {
          uint32_t r[32];
          acc_ld32(t_row + (ps * W + c * 32) * 4, r);
          const int col0 = col_pass + c * 32;
          float v[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]);
          if (p.bias) {
            if (col0 + 32 <= p.N && !p.scalar_rows) {
              const float4* b4 = reinterpret_cast<const float4*>(p.bias + col0);
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float4 b = __ldg(b4 + i);
                v[4 * i] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
              }
            } else {
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] += (col0 + i < p.N) ? __ldg(p.bias + col0 + i) : 0.f;
            }
          }
          if (p.act == 1) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = gelu_fast(v[i]);
          } else if (p.act == 2) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.f);
          }
          if (stage_f32) {
            const uint32_t a = stg_s + lane * STG_ROW;
#pragma unroll
            for (int i = 0; i < 16; ++i)
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a + i * 8), "f"(v[2 * i]), "f"(v[2 * i + 1])
                           : "memory");
          } else {
            const uint32_t a = stg_s + lane * STG_ROW + c * 64;
#pragma unroll
            for (int i = 0; i < 8; ++i)
              asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a + i * 8),
                           "r"(pack_bf16x2(v[4 * i], v[4 * i + 1])), "r"(pack_bf16x2(v[4 * i + 2], v[4 * i + 3]))
                           : "memory");
          }
        }
        __syncwarp();
        // ---- phase 2: coalesced write-out, 8 bytes per lane, whole 128-byte lines per half-warp
        const int col = col_pass + cl * epl;
        if (stage_f32) {
#pragma unroll
          for (int k = 0; k < 16; ++k) {
            const int rr = 2 * k + sub;
            const int orow = get_orow(rr);
            if (orow < 0 || col >= p.N) continue;
            float x0, x1;
            asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(x0), "=f"(x1) : "r"(stg_s + rr * STG_ROW + cl * 8));
            if (p.residual) {
              if (p.res_fp32 || p.scalar_rows) {
                x0 += resv[k].x; x1 += resv[k].y;
              } else {
                const uint32_t raw = __float_as_uint(resv[k].x);
                x0 += __uint_as_float(raw << 16); x1 += __uint_as_float(raw & 0xffff0000u);
              }
            }
            if (p.scalar_rows) {
              store_at(p, orow, col, x0);
              if (col + 1 < p.N) store_at(p, orow, col + 1, x1);
            } else if (p.out_fp32)
              *reinterpret_cast<float2*>(static_cast<float*>(p.out) + static_cast<size_t>(orow) * p.ldo + col) =
                  make_float2(x0, x1);
            else
              *reinterpret_cast<uint32_t*>(static_cast<__nv_bfloat16*>(p.out) + static_cast<size_t>(orow) * p.ldo +
                                           col) = pack_bf16x2(x0, x1);
          }
        } else {
#pragma unroll 4
          for (int r0 = 0; r0 < 32; r0 += rpi) {
            const int rr = r0 + sub;
            const int orow = get_orow(rr);
            if (orow < 0 || col >= p.N) continue;
            uint32_t w0, w1;
            asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(w0), "=r"(w1) : "r"(stg_s + rr * STG_ROW + cl * 8));
            *reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(p.out) + static_cast<size_t>(orow) * p.ldo + col) =
                make_uint2(w0, w1);
          }
        }
        __syncwarp();
      }
    }
  }
}

// Epilogue warpgroup of the split schedule: the CTA's tiles in order, each taken from accumulator buffer it % ACC_BUFS
// once the MMA warpgroups have filled it ("tile full") and handed back ("tile empty") when its reads are done.
template <int BN, int EPI, int OUT>
__device__ __forceinline__ void epilogue_loop(const Dev& p, const CUtensorMap& tma_c, const CUtensorMap& tma_r, int e,
                                              uint32_t acc_base, uint8_t* stg_all, uint64_t* bar_res,
                                              uint64_t* bar_tfull, uint64_t* bar_tempty) {
  using C = Cfg<BN, EPI>;
  uint32_t rphase = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int m_blk = tile / p.num_n_blocks;
    const int n_blk = tile % p.num_n_blocks;
    const int it = (tile - blockIdx.x) / gridDim.x;   // tiles this CTA has run before this one
    const int buf = C::ACC_BUFS == 2 ? (it & 1) : 0;
    const uint32_t use = C::ACC_BUFS == 2 ? (it >> 1) : it;
    mbar_wait(smem_u32(&bar_tfull[buf]), use & 1);
    epilogue_tile<BN, EPI, OUT>(p, tma_c, tma_r, m_blk, n_blk, e, 0, acc_base + buf * C::ACC_BYTES, stg_all, bar_res,
                                rphase);
    mbar_arrive(smem_u32(&bar_tempty[buf]));
  }
}

// Epilogue of the wide schedule, run by each MMA warp on its own accumulator fragment.  Warp e holds rows
// [64 wg + 16 (e & 3), + 16) of the 128 x 256 tile; its lane l holds rows l / 4 and l / 4 + 8 of those, and in every
// 8-column group c the columns 8 c + 2 (l % 4) + {0, 1} (acc[4 c + {0, 1}] and acc[4 c + {2, 3}]).  Bias, activation
// and bf16 rounding are the split epilogue's, in its order, so both schedules write the same bytes.  The warp's four
// 16 x 64 slabs leave through the two 2 KB halves of its staging buffer (128-byte swizzled, as the 64 x 16 box of
// tma_c expects) as TMA stores; a store is waited for only before its half is rewritten, so the stores of one tile
// drain while the next tile's k-loop runs.
__device__ __forceinline__ void epilogue_wide(const Dev& p, const CUtensorMap& tma_c, const float (&acc)[128],
                                              int m_blk, int n_blk, int wg, int e, uint8_t* stg_all) {
  const int lane = threadIdx.x & 31;
  const int r = lane >> 2;                           // rows r and r + 8 of the warp's 16; (r + 8) & 7 == r
  const int row0 = m_blk * BM + wg * 64 + (e & 3) * 16;
  const uint32_t slab = smem_u32(stg_all) + e * 4096;
  const float* bias = p.bias;
  const int act = p.act;
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    const int col0 = n_blk * 256 + s * 64;
    const uint32_t half = slab + (s & 1) * 2048;
    if (lane == 0) bulk_wait_read1();                // the store that last read this half is done with it
    __syncwarp();
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float v[4] = {acc[32 * s + 4 * c], acc[32 * s + 4 * c + 1], acc[32 * s + 4 * c + 2], acc[32 * s + 4 * c + 3]};
      if (bias) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(bias + col0 + 8 * c + 2 * (lane & 3)));
        v[0] += b.x; v[1] += b.y; v[2] += b.x; v[3] += b.y;
      }
      if (act == 1) {
#pragma unroll
        for (int i = 0; i < 4; ++i) v[i] = gelu_fast(v[i]);
      } else if (act == 2) {
#pragma unroll
        for (int i = 0; i < 4; ++i) v[i] = fmaxf(v[i], 0.f);
      }
      const uint32_t a = half + r * 128 + ((c ^ r) << 4) + 4 * (lane & 3);
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(pack_bf16x2(v[0], v[1])) : "memory");
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + 8 * 128), "r"(pack_bf16x2(v[2], v[3])) : "memory");
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) { tma_store_2d(&tma_c, half, col0, row0); bulk_commit(); }
  }
}

template <int BN, int EPI>
__global__ void __launch_bounds__(Cfg<BN, EPI>::THREADS, 1)
gemm_bf16_wgmma_v2_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                            const __grid_constant__ CUtensorMap tma_c, const __grid_constant__ CUtensorMap tma_r,
                            const Dev p) {
  using C = Cfg<BN, EPI>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t smem_base = smem_u32(smem);
  uint8_t* stg_all = smem + STAGES * C::STAGE_BYTES;
  const uint32_t acc_base = smem_u32(stg_all + C::STG_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(stg_all + C::STG_BYTES + C::ACC_BUFS * C::ACC_BYTES);
  uint64_t* bar_full = bars;
  uint64_t* bar_empty = bars + STAGES;
  uint64_t* bar_res = bars + 2 * STAGES;           // one per epilogue warp: residual slab landed
  uint64_t* bar_tfull = bar_res + 8;               // per accumulator buffer: the MMA warps have written the tile
  uint64_t* bar_tempty = bar_tfull + C::ACC_BUFS;  // per accumulator buffer: the epilogue has read it

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), 8);
    }
    for (int s = 0; s < 8; ++s) mbar_init(smem_u32(&bar_res[s]), 1);
    for (int b = 0; b < C::ACC_BUFS; ++b) {
      mbar_init(smem_u32(&bar_tfull[b]), 256);
      mbar_init(smem_u32(&bar_tempty[b]), 32 * C::EPI_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // each role's setmaxnreg comes first in its branch: ptxas allocates the branch's registers under that budget
  if (warp < 4) {
    if constexpr (C::SPLIT || C::WIDE) setmaxnreg_dec<C::REG_PRODUCER>();
    if (warp == 0 && lane == 0) {
      const int num_kb = num_kblocks(p);
      // ---------------------------------------------------------- TMA producer
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int m_blk = tile / p.num_n_blocks;
        const int n_blk = tile % p.num_n_blocks;
        int cb = 0, cy = 0, cx = 0, tap = 0, ckb = 0;
        const int w_row0 = p.mblk_per_group > 0 ? (m_blk / p.mblk_per_group) * p.w_group_rows : 0;
        if (p.conv_kb > 0) {   // the tile's 128 output pixels are a (images x rows x cols) box of the NHWC map
          const int hw = p.conv_h * p.conv_w, p0 = m_blk * BM;
          cb = p0 / hw;
          const int rem = p0 - cb * hw;
          cy = rem / p.conv_w;
          cx = rem - cy * p.conv_w;
        }
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(smem_u32(&bar_empty[stage]), phase ^ 1);
          const uint32_t full = smem_u32(&bar_full[stage]);
          const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
          mbar_expect_tx(full, C::STAGE_BYTES);
          if (p.conv_kb > 0) {
            const int ky = tap / 3, kx = tap - 3 * ky;
            tma_load_4d(sa, &tma_a, full, ckb * BK, cx + kx - 1, cy + ky - 1, cb);   // halo -> zero fill
            if (++ckb == p.conv_kb) { ckb = 0; ++tap; }
          } else {
            tma_load_2d(sa, &tma_a, full, kb * BK, m_blk * BM);
          }
          tma_load_2d(sa + A_BYTES, &tma_b, full, kb * BK, n_blk * BN + w_row0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
      // tail: consume the ring's last "empty" completions, so that no consumer arrive is left without a waiter when the
      // CTA retires; never-used slots pass at once
      for (int i = 0; i < STAGES; ++i) {
        mbar_wait(smem_u32(&bar_empty[stage]), phase ^ 1);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp < 12) {
    // ------------------------------------------------------------ MMA warpgroups: rows [64 wg, 64 wg + 64) of each tile
    if constexpr (C::SPLIT || C::WIDE) setmaxnreg_inc<C::REG_MMA>();
    const int wg = (warp - 4) >> 2;
    const int num_kb = num_kblocks(p);   // computed per role: a value live across setmaxnreg goes to local memory
    int kstage = 0;
    uint32_t kphase = 0;
    if constexpr (C::WIDE) {
      // the producer refills the ring for the next tile while these warps run the epilogue
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        float acc[BN / 2];
        wg_mainloop<BN, STAGES>(acc, smem_base, C::STAGE_BYTES, A_BYTES, num_kb, wg, kstage, kphase, bar_full,
                                bar_empty);
        epilogue_wide(p, tma_c, acc, tile / p.num_n_blocks, tile % p.num_n_blocks, wg, warp - 4, stg_all);
      }
      if (lane == 0) bulk_wait0();   // every slab is in global memory before the CTA retires
    } else if constexpr (C::SPLIT) {
      int it = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
        float acc[BN / 2];
        wg_mainloop<BN, STAGES>(acc, smem_base, C::STAGE_BYTES, A_BYTES, num_kb, wg, kstage, kphase, bar_full,
                                bar_empty);
        const int buf = C::ACC_BUFS == 2 ? (it & 1) : 0;
        const uint32_t use = C::ACC_BUFS == 2 ? (it >> 1) : it;   // earlier tiles through this buffer
        mbar_wait(smem_u32(&bar_tempty[buf]), (use & 1) ^ 1);   // the epilogue is done with its previous tile
        acc_store<BN>(acc, acc_base + buf * C::ACC_BYTES, C::ACC_LD, wg, threadIdx.x & 127);
        mbar_arrive(smem_u32(&bar_tfull[buf]));
      }
    } else {
      // the same warps run the epilogue: 8 warps, warp e = rows [32 (e & 3), + 32), column half wg
      const int e = warp - 4;
      uint32_t rphase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int m_blk = tile / p.num_n_blocks;
        const int n_blk = tile % p.num_n_blocks;
        {
          float acc[BN / 2];
          wg_mainloop<BN, STAGES>(acc, smem_base, C::STAGE_BYTES, A_BYTES, num_kb, wg, kstage, kphase, bar_full,
                                  bar_empty);
          named_bar_sync(5, 256);   // the previous tile's epilogue has read the accumulator tile
          acc_store<BN>(acc, acc_base, C::ACC_LD, wg, threadIdx.x & 127);
          named_bar_sync(5, 256);
        }
        if (wg < C::NHALF)
          epilogue_tile<BN, EPI>(p, tma_c, tma_r, m_blk, n_blk, e, wg, acc_base, stg_all, bar_res, rphase);
      }
      if (p.tma_store && lane == 0) bulk_wait0();   // every slab is in global memory before the CTA retires
    }
  } else if constexpr (C::SPLIT) {
    // ------------------------------------------------------------ epilogue warpgroup: warp e = rows [32 e, 32 e + 32)
    setmaxnreg_inc<C::REG_EPI>();
    const int e = warp - 12;
    // one tile loop per output path: each is register-allocated on its own (together in one loop they spill)
    if (p.tma_store) {
      epilogue_loop<BN, EPI, OUT_TMA>(p, tma_c, tma_r, e, acc_base, stg_all, bar_res, bar_tfull, bar_tempty);
      if (lane == 0) bulk_wait0();   // every slab is in global memory before the CTA retires
    } else {
      epilogue_loop<BN, EPI, OUT_SCATTER>(p, tma_c, tma_r, e, acc_base, stg_all, bar_res, bar_tfull, bar_tempty);
    }
  }
}

template <int BN, int EPI>
static int launch(const GemmArgs& a, cudaStream_t stream) {
  using C = Cfg<BN, EPI>;
  CUtensorMap ta, tb;
  Dev p;
  p.conv_kb = 0; p.conv_h = a.conv_h; p.conv_w = a.conv_w;
  if (a.conv_c > 0) {
    const uint64_t C_ = a.conv_c, W_ = a.conv_w, H_ = a.conv_h, B_ = a.conv_b;
    const uint32_t tw = a.conv_w < BM ? a.conv_w : BM;
    const uint32_t th = (BM / tw) < static_cast<uint32_t>(a.conv_h) ? BM / tw : a.conv_h;
    const uint32_t tb = BM / (tw * th);
    uint64_t dims[4] = {C_, W_, H_, B_};
    uint64_t strides[3] = {C_ * 2, W_ * C_ * 2, H_ * W_ * C_ * 2};
    uint32_t box[4] = {static_cast<uint32_t>(BK), tw, th, tb};
    RSP_TRY(make_tmap_bf16(&ta, a.A, 4, dims, strides, box));
    p.conv_kb = a.conv_c / BK;
  } else {
    RSP_TRY(make_tmap_bf16_2d(&ta, a.A, a.M, a.K, static_cast<uint64_t>(a.lda) * 2, BM, BK));
  }
  const int n_groups = a.m_group_rows > 0 ? (a.M + a.m_group_rows - 1) / a.m_group_rows : 1;
  const uint64_t w_rows = a.m_group_rows > 0 ? static_cast<uint64_t>(n_groups - 1) * a.w_group_rows + a.N : a.N;
  RSP_TRY(make_tmap_bf16_2d(&tb, a.W, w_rows, a.K, static_cast<uint64_t>(a.ldw) * 2, BN, BK));
  CUtensorMap tc = tb, tr = tb;
  p.tma_store = 0;
  p.tma_res = 0;
  p.scalar_rows = EPI == EPI_STD && !gemm_vector_rows(a);
  {
    const uint64_t esz = a.out_fp32 ? 4 : 2;
    bool res_ok = true;
    if (a.residual) {
      res_ok = (a.res_fp32 != 0) == (a.out_fp32 != 0) &&
               (reinterpret_cast<uintptr_t>(a.residual) & 15) == 0 && (static_cast<uint64_t>(a.ldr) * esz) % 16 == 0 &&
               (a.res_block_map ? (a.res_block_rows % 32 == 0 && a.M % 32 == 0) : (a.res_mod == 0 || a.res_mod % 32 == 0));
    }
    if ((EPI == EPI_STD || EPI == EPI_STD_WIDE || EPI == EPI_LN_ROW || EPI == EPI_LN64_GELU) && BN >= 64 && res_ok &&
        !a.row_map && !p.scalar_rows && a.out &&
        (reinterpret_cast<uintptr_t>(a.out) & 15) == 0 && (static_cast<uint64_t>(a.ldo) * esz) % 16 == 0) {
      uint64_t dims[2] = {static_cast<uint64_t>(a.N), static_cast<uint64_t>(a.M)};
      uint64_t strides[1] = {static_cast<uint64_t>(a.ldo) * esz};
      uint32_t box[2] = {a.out_fp32 ? 32u : 64u, C::WIDE ? 16u : 32u};
      RSP_TRY(make_tmap(&tc, a.out, 2, dims, strides, box, a.out_fp32));
      p.tma_store = 1;
      if (a.residual) {
        // rows the map may address: the whole destination (identity), one period (res_mod) or an open bound
        // (block map: the host guarantees map[blk] * res_block_rows + 31 stays inside the residual tensor)
        const uint64_t rrows = a.res_block_map ? (1ull << 31) : (a.res_mod > 0 ? a.res_mod : a.M);
        uint64_t rdims[2] = {static_cast<uint64_t>(a.N), rrows};
        uint64_t rstrides[1] = {static_cast<uint64_t>(a.ldr) * esz};
        RSP_TRY(make_tmap(&tr, a.residual, 2, rdims, rstrides, box, a.out_fp32));
        p.tma_res = 1;
      }
    }
  }
  if (EPI == EPI_LN_ROW && !(p.tma_store && p.tma_res)) {
    set_last_error("gemm_v2: fused row LayerNorm needs TMA-eligible bf16 output and residual");
    return RSP_ERR_INVALID;
  }
  if (C::WIDE && !(p.tma_store && !a.residual && !a.out_fp32 && a.N % BN == 0 && a.conv_c == 0 && a.m_group_rows == 0)) {
    set_last_error("gemm_v2: the wide schedule needs a plain GEMM with TMA-eligible bf16 output, no residual, N %% 256 == 0");
    return RSP_ERR_INVALID;
  }
  p.M = a.M; p.N = a.N; p.K = a.K;
  p.bias = a.bias; p.residual = a.residual; p.out = a.out; p.row_map = a.row_map;
  p.res_block_map = a.res_block_map; p.res_block_rows = a.res_block_rows;
  p.res_mod = a.res_mod; p.ldo = a.ldo; p.ldr = a.ldr; p.act = a.act;
  p.out_fp32 = a.out_fp32; p.res_fp32 = a.res_fp32;
  p.mblk_per_group = a.m_group_rows > 0 ? a.m_group_rows / BM : 0;
  p.w_group_rows = a.w_group_rows;
  p.num_n_blocks = (a.N + BN - 1) / BN;
  p.num_tiles = ((a.M + BM - 1) / BM) * p.num_n_blocks;
  p.ln_gamma = a.ln_gamma; p.ln_beta = a.ln_beta; p.ln_eps = a.ln_eps;
  p.hyper = a.hyper; p.mask_out = a.mask_out; p.grid_h = a.grid_h; p.grid_w = a.grid_w;
  auto kern = gemm_bf16_wgmma_v2_kernel<BN, EPI>;
  static bool attr_set_dev[kMaxDevices] = {};   // the attribute is per device (one flag per ordinal)
  bool& attr_set = attr_set_dev[current_device()];
  if (!attr_set) {
    RSP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    attr_set = true;
  }
  const int grid = p.num_tiles < num_sms() ? p.num_tiles : num_sms();
  kern<<<grid, C::THREADS, C::SMEM_BYTES, stream>>>(ta, tb, tc, tr, p);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace v2

// Rows the standard epilogue moves 8 bytes (and bias 16 bytes) at a time: N, ldo, ldr and the out / residual / bias
// pointers aligned for it.  Other rows take its scalar path.
bool gemm_vector_rows(const GemmArgs& a) {
  const bool stage_f32 = a.out_fp32 || a.residual;
  const uintptr_t po = reinterpret_cast<uintptr_t>(a.out), pr = reinterpret_cast<uintptr_t>(a.residual);
  if (stage_f32) {
    if (a.N % 2 != 0 || a.ldo % 2 != 0 || (po & (a.out_fp32 ? 7 : 3)) != 0) return false;
  } else {
    if (a.N % 4 != 0 || a.ldo % 4 != 0 || (po & 7) != 0) return false;
  }
  if (a.residual && (a.ldr % 2 != 0 || (pr & (a.res_fp32 ? 7 : 3)) != 0)) return false;
  if (a.bias && (reinterpret_cast<uintptr_t>(a.bias) & 15) != 0) return false;
  return true;
}

// Row LayerNorms that EPI_LN_ROW takes (two warps per row, residual slabs and output by TMA): N == 256, bf16 residual
// and output, residual rows in whole 32-row slabs (mask decoder: LN4(keys + attn)).  gemm_bf16 has checked the
// 16-byte alignment of every row.  The others run EPI_LN_ROW_T.
static bool ln_row_tma(const GemmArgs& a) {
  return a.N == 256 && !a.out_fp32 && a.residual && !a.res_fp32 && a.bias && a.res_mod == 0 && a.act == 0 &&
         (a.res_block_map ? (a.res_block_rows % 32 == 0 && a.M % 32 == 0) : true);
}

// Standard-epilogue GEMMs the wide schedule can take: plain 2-D A, bf16 output through TMA, no residual or row scatter,
// whole 256-wide n-blocks and 64-deep k-blocks.
static bool std_wide_shape(const GemmArgs& a) {
  return a.epi_mode == v2::EPI_STD && !a.residual && !a.row_map && !a.out_fp32 && a.conv_c == 0 &&
         a.m_group_rows == 0 && a.N % 256 == 0 && a.K % 64 == 0 && gemm_vector_rows(a) && a.out &&
         (reinterpret_cast<uintptr_t>(a.out) & 15) == 0 && a.ldo % 8 == 0;
}

int gemm_bf16_v2_std(const GemmArgs& a, bool wide, cudaStream_t stream) {
  if (wide) return v2::launch<256, v2::EPI_STD_WIDE>(a, stream);
  if (a.N > 64) return v2::launch<128, v2::EPI_STD>(a, stream);
  if (a.N > 32) return v2::launch<64, v2::EPI_STD>(a, stream);
  return v2::launch<32, v2::EPI_STD>(a, stream);
}

int gemm_bf16_v2(const GemmArgs& a, cudaStream_t stream) {
  if (a.epi_mode == v2::EPI_STD) {
    // 128 x 256 tiles with the epilogue in registers where they pay.  The epilogue stalls the tensor cores once per
    // tile, so the k-loop must be long enough to amortise it, and a wide tile is twice the work of the split
    // schedule's, so the last partial wave costs twice as much.  `rsp_selftest gemm bench` (H100 SXM, 700 W):
    // K = 1280 at 29 - 39 waves of wide tiles (ViT-H qkv / lin1, 32 768 - 39 200 rows) runs 1.06 - 1.16x faster;
    // K = 768 (ViT-B qkv / lin1, same rows) 0.94 - 0.99x, K = 512 0.82x, and K = 1280 at 7 - 10 waves 0.86 - 0.91x.
    // Every other call takes 128-wide tiles or narrower with the epilogue on its own warpgroup: the fp32 accumulator
    // tile of a 256-wide one would leave shared memory for a single stage.
    const long long wide_tiles = static_cast<long long>((a.M + v2::BM - 1) / v2::BM) * (a.N / 256);
    const bool wide = std_wide_shape(a) && a.K >= 1024 && wide_tiles >= 16ll * num_sms();
    return gemm_bf16_v2_std(a, wide, stream);
  }
  if (a.epi_mode == v2::EPI_LN_ROW) {
    if (ln_row_tma(a)) return v2::launch<256, v2::EPI_LN_ROW>(a, stream);
    return a.N > 128 ? v2::launch<256, v2::EPI_LN_ROW_T>(a, stream) : v2::launch<128, v2::EPI_LN_ROW_T>(a, stream);
  }
  if (a.epi_mode == v2::EPI_LN64_GELU) return v2::launch<128, v2::EPI_LN64_GELU>(a, stream);
  return v2::launch<128, v2::EPI_GELU_HYPER>(a, stream);
}

int gemm_bf16_v2_gelu_hyper_multi(const GemmArgs& a, int n_out, cudaStream_t stream) {
  switch (n_out) {
    case 1: return v2::launch<128, v2::EPI_GELU_HYPER>(a, stream);
    case 2: return v2::launch<128, v2::EPI_GELU_HYPER2>(a, stream);
    case 3: return v2::launch<128, v2::EPI_GELU_HYPER3>(a, stream);
    default: set_last_error("gemm_v2: %d hypernetwork outputs (1 to 3)", n_out); return RSP_ERR_INVALID;
  }
}

}  // namespace rsp
