// ViT-SAM attention core for sm_90a: softmax(scale * q k^T + rel_h + rel_w) v per
// (sequence, head), sequences being 14x14 windows (T = 196) or whole 32x32 / 64x64 images
// (T = 1024 / 4096).  Reference: transformers modeling_sam.py SamVisionAttention.forward
// (:803-831), get_rel_pos / get_decomposed_rel_pos (:729-801); mmpretrain vit_sam.py
// Attention.forward (:202-221), add_decomposed_rel_pos (:117-157).
//
// Flash-style on wgmma.  Persistent: one CTA per SM works through query tiles of 128 rows of one (sequence, head),
// 384 threads in three warpgroups:
//   * warpgroup 0 gives its registers up (setmaxnreg).  Warp 0 is the TMA producer: the layer's two rel-pos tables
//     once, then per query tile its Q (double-buffered where shared memory allows, so the next tile's Q lands during
//     this one) and its 64-key K / V tiles through a four-stage mbarrier ring that runs on across query tiles.
//     Warps 1-3 convert each landed V tile bf16 -> fp16 in place (exact for |v| in fp16's normal range), off the
//     consumers' critical path.
//   * warpgroups 1 and 2 own 64 query rows each.  S = Q K^T is an SS wgmma (bf16, fp32 accumulators); the online
//     softmax runs on the accumulator fragment; P (fp16, which keeps 11 mantissa bits of a value in [0, 1] where bf16
//     keeps 8) goes straight from those registers into the A operand of an RS wgmma against the fp16 V tile.
//     Scores stay fp32 until the exp (reference: softmax in fp32).
// Shared-memory layout of a [rows x hd] bf16 tile: columns 0-63 in the 128-byte-swizzled layout (rows of 128 bytes),
// then, for hd = 80, columns 64-79 in the 32-byte-swizzled layout (rows of 32 bytes).  A head is 160 bytes, not a
// multiple of one 128-byte swizzle row, so each tile is two TMA boxes (64 and 16 columns wide) from two tensor maps.
// Q K^T is four k16 steps in the first part and one in the second; P V is an N = 64 wgmma on the first part plus an
// N = 16 one on the second (both MN-major).  The fp16 V conversion keeps every element in place, so it needs no
// layout of its own.
// The decomposed relative-position bias is never materialised as a T x T tensor: a prologue runs Q x table^T for both
// tables on the same wgmma path (the reference's two einsums) and scatters each row's S + S values (pre-multiplied by
// log2 e) into shared memory.  For S = 32 / 64 the key tile is a multiple of S, so each register of a thread's score
// fragment always meets the same key column kw: the thread keeps its rel_w terms in registers and reads one rel_h
// value per row and S-key block per tile.  For S = 14 both terms are read from shared memory per score.
#include <cstdlib>

#include "attention.h"
#include "sm90.cuh"

namespace rsp {

constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t bf16x2_to_f16x2(uint32_t w) {
  return pack_f16x2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
}

template <int HD, int S>
struct AttCfg {
  static constexpr int T = S * S;
  static constexpr int BM = 128;                        // query rows per CTA: two consumer warpgroups of 64
  static constexpr int BN = 64;                         // keys per K / V tile
  static constexpr int NQT = (T + BM - 1) / BM;
  static constexpr int NKT = (T + BN - 1) / BN;
  static constexpr int NREL = 2 * S - 1;                // rel-pos table rows
  static constexpr int NTAB = NREL <= 32 ? 32 : (NREL <= 64 ? 64 : 128);   // table rows loaded (N of the prologue)
  static constexpr int TAIL = HD - 64;                  // columns in the 32-byte-swizzled part: 0 or 16
  static constexpr int STAGES = 4;
  static constexpr int SP = S + 4;                      // row stride of the gathered bias (floats)
  __host__ __device__ static constexpr int tile_bytes(int rows) { return rows * (128 + 2 * TAIL); }
  static constexpr int STAGE_BYTES = 2 * tile_bytes(BN);   // K, then V
  static constexpr int smem_bytes(int qbuf) {                 // + 1024 bytes of slack to align the base
    return qbuf * tile_bytes(BM) + STAGES * STAGE_BYTES + 2 * tile_bytes(NTAB) + 2 * BM * SP * 4 + 8 * 64 + 1024;
  }
  static constexpr int QBUF = smem_bytes(2) <= 227 * 1024 ? 2 : 1;   // Q buffers: the next tile's Q lands early
  static constexpr int Q_OFF = 0;
  static constexpr int KV_OFF = Q_OFF + QBUF * tile_bytes(BM);
  static constexpr int TAB_OFF = KV_OFF + STAGES * STAGE_BYTES;
  static constexpr int BIAS_OFF = TAB_OFF + 2 * tile_bytes(NTAB);
  static constexpr int BAR_OFF = BIAS_OFF + 2 * BM * SP * 4;
  static constexpr int SMEM_BYTES = smem_bytes(QBUF);
  static constexpr int REG_PRODUCER = 40, REG_CONSUMER = 232;    // 128 x 40 + 256 x 232 <= 64K registers
  static_assert(HD == 64 || HD == 80, "head dim");
  static_assert(NREL <= 128, "table rows");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory");
};

struct AttDev {
  __nv_bfloat16* out;  // [M_tok, D]
  const int* out_row_map;   // window_unpartition + crop fused into the store (HF:925-952), or null
  int H;
  int D;
  int n_items;         // query tiles in all: n_seq * H * NQT
  float scale2;        // hd^-0.5 * log2(e)
};

// acc[64 x N] = (this warpgroup's 64 rows of Q) x B^T, B = the first N rows of a K-like tile of b_rows rows at b
template <int N, int TAIL>
__device__ __forceinline__ void qk_wgmma(float (&acc)[N / 2], uint32_t qa, uint32_t qtail, uint32_t b, int b_rows) {
  acc_fence(acc);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k)
    Wgmma<N>::template ss<0>(acc, make_gdesc(qa + 32 * k, 16, 1024), make_gdesc(b + 32 * k, 16, 1024), k);
  if constexpr (TAIL > 0)
    Wgmma<N>::template ss<0>(acc, make_gdesc_sw32(qtail, 16, 256), make_gdesc_sw32(b + b_rows * 128, 16, 256), 1);
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(acc);
}

// one [rows x HD] tile of a 3-D (column, token, sequence) tensor map pair: 64 columns 128B-swizzled, then the tail
template <int TAIL>
__device__ __forceinline__ void load_tile(uint32_t dst, int rows, const CUtensorMap* m, const CUtensorMap* mt,
                                          uint32_t bar, int col, int row, int seq) {
  tma_load_3d(dst, m, bar, col, row, seq);
  if constexpr (TAIL > 0) tma_load_3d(dst + rows * 128, mt, bar, col + 64, row, seq);
}

template <int HD, int S>
__global__ void __launch_bounds__(384, 1)
vit_attention_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_q_t,
                     const __grid_constant__ CUtensorMap tm_kv, const __grid_constant__ CUtensorMap tm_kv_t,
                     const __grid_constant__ CUtensorMap tm_rh, const __grid_constant__ CUtensorMap tm_rh_t,
                     const __grid_constant__ CUtensorMap tm_rw, const __grid_constant__ CUtensorMap tm_rw_t,
                     const AttDev p) {
  using C = AttCfg<HD, S>;
  constexpr int T = C::T, BM = C::BM, BN = C::BN, NKT = C::NKT, SP = C::SP, STAGES = C::STAGES, TAIL = C::TAIL;
  constexpr int QBUF = C::QBUF;
  constexpr uint32_t TILE_KV = C::tile_bytes(BN), TILE_TAB = C::tile_bytes(C::NTAB);
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(smem);
  float* relh = reinterpret_cast<float*>(smem + C::BIAS_OFF);   // [BM][SP]: rel_h term of (row, key row kh)
  float* relw = relh + BM * SP;                                 // [BM][SP]: rel_w term of (row, key column kw)
  uint64_t* bar_tab = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);   // both tables landed
  uint64_t* bar_q = bar_tab + 1;            // per Q buffer: Q tile landed
  uint64_t* bar_qe = bar_q + QBUF;          // per Q buffer: both consumer warpgroups are done with it
  uint64_t* bar_k = bar_qe + QBUF;          // per stage: K tile landed
  uint64_t* bar_v = bar_k + STAGES;         // per stage: V tile landed (bf16)
  uint64_t* bar_vc = bar_v + STAGES;        // per stage: V tile converted to fp16 (one arrive per converter warp)
  uint64_t* bar_e = bar_vc + STAGES;        // per stage: both consumer warpgroups are done with K and V

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // Persistent: CTA b runs query tiles b, b + gridDim.x, ...  The query tiles of one (sequence, head) are adjacent
  // numbers, so CTAs running at the same time share K / V through L2.
  auto decode = [&](int item, int& q0, int& head, int& seq) {
    q0 = (item % C::NQT) * BM;
    item /= C::NQT;
    head = item % p.H;
    seq = item / p.H;
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_kv);
    mbar_init(smem_u32(bar_tab), 1);
    for (int b = 0; b < QBUF; ++b) {
      mbar_init(smem_u32(&bar_q[b]), 1);
      mbar_init(smem_u32(&bar_qe[b]), 8);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bar_k[s]), 1);
      mbar_init(smem_u32(&bar_v[s]), 1);
      mbar_init(smem_u32(&bar_vc[s]), 3);
      mbar_init(smem_u32(&bar_e[s]), 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<C::REG_PRODUCER>();
    if (warp == 0) {
      if (lane == 0) {
        // ------------------------------------------------------------ TMA producer
        const uint32_t bq = smem_u32(bar_tab);   // the tables are the layer's: loaded once
        mbar_expect_tx(bq, 2 * TILE_TAB);
        tma_load_2d(sbase + C::TAB_OFF, &tm_rh, bq, 0, 0);
        tma_load_2d(sbase + C::TAB_OFF + TILE_TAB, &tm_rw, bq, 0, 0);
        if constexpr (TAIL > 0) {
          tma_load_2d(sbase + C::TAB_OFF + C::NTAB * 128, &tm_rh_t, bq, 64, 0);
          tma_load_2d(sbase + C::TAB_OFF + TILE_TAB + C::NTAB * 128, &tm_rw_t, bq, 64, 0);
        }
        int g = 0;   // K / V tiles issued so far: ring position
#pragma unroll 1
        for (int item = blockIdx.x, it = 0; item < p.n_items; item += gridDim.x, ++it) {
          int q0, head, seq;
          decode(item, q0, head, seq);
          const int colq = head * HD, colk = p.D + colq, colv = 2 * p.D + colq;
          const int qb = it % QBUF;
          mbar_wait(smem_u32(&bar_qe[qb]), ((it / QBUF) & 1) ^ 1);
          mbar_expect_tx(smem_u32(&bar_q[qb]), C::tile_bytes(BM));
          load_tile<TAIL>(sbase + C::Q_OFF + qb * C::tile_bytes(BM), BM, &tm_q, &tm_q_t, smem_u32(&bar_q[qb]),
                          colq, q0, seq);
#pragma unroll 1
          for (int j = 0; j < NKT; ++j, ++g) {
            const int s = g % STAGES;
            mbar_wait(smem_u32(&bar_e[s]), ((g / STAGES) & 1) ^ 1);
            const uint32_t kb = sbase + C::KV_OFF + s * C::STAGE_BYTES;
            mbar_expect_tx(smem_u32(&bar_k[s]), TILE_KV);
            load_tile<TAIL>(kb, BN, &tm_kv, &tm_kv_t, smem_u32(&bar_k[s]), colk, j * BN, seq);
            mbar_expect_tx(smem_u32(&bar_v[s]), TILE_KV);
            load_tile<TAIL>(kb + TILE_KV, BN, &tm_kv, &tm_kv_t, smem_u32(&bar_v[s]), colv, j * BN, seq);
          }
        }
      }
    } else {
      // ------------------------------------------------------------ V converters: bf16 -> fp16 in place
      const int t = threadIdx.x - 32;
      const int n_tiles = ((p.n_items - static_cast<int>(blockIdx.x) + gridDim.x - 1) / gridDim.x) * NKT;
#pragma unroll 1
      for (int g = 0; g < n_tiles; ++g) {
        const int s = g % STAGES;
        mbar_wait(smem_u32(&bar_v[s]), (g / STAGES) & 1);
        uint4* v = reinterpret_cast<uint4*>(smem + C::KV_OFF + s * C::STAGE_BYTES + TILE_KV);
#pragma unroll 2
        for (int i = t; i < static_cast<int>(TILE_KV / 16); i += 96) {
          uint4 w = v[i];
          w.x = bf16x2_to_f16x2(w.x);
          w.y = bf16x2_to_f16x2(w.y);
          w.z = bf16x2_to_f16x2(w.z);
          w.w = bf16x2_to_f16x2(w.w);
          v[i] = w;
        }
        fence_proxy_async_smem();   // the generic-proxy writes become visible to wgmma
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bar_vc[s]));
      }
    }
    return;
  }

  // -------------------------------------------------------------- consumers: rows [64 wg, 64 wg + 64) of the tile
  setmaxnreg_inc<C::REG_CONSUMER>();
  const int wg = (warp >> 2) - 1;
  // this thread's fragment coordinates: rows r0 + 8 i (i = 0, 1) of the tile, columns 8 b + cq + {0, 1}
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  constexpr bool REG_W = BN % S == 0;
  constexpr int CPS = REG_W ? S / 8 : 1;   // 8-column blocks per S keys
  mbar_wait(smem_u32(bar_tab), 0);
  int g = 0;   // K / V tiles consumed so far: ring position
#pragma unroll 1
  for (int item = blockIdx.x, it = 0; item < p.n_items; item += gridDim.x, ++it) {
    int q0, head, seq;
    decode(item, q0, head, seq);
    const int qb = it % QBUF;
    const uint32_t qbase = sbase + C::Q_OFF + qb * C::tile_bytes(BM);
    const uint32_t qa = qbase + wg * 64 * 128;                 // this warpgroup's Q rows, columns 0-63
    const uint32_t qtail = qbase + BM * 128 + wg * 64 * 32;    // columns 64-79

    // ---- prologue: Q x table^T for both tables, gathered into relh / relw (this warpgroup's 64 rows only)
    mbar_wait(smem_u32(&bar_q[qb]), (it / QBUF) & 1);
    named_bar_sync(1 + wg, 128);   // the warpgroup is done reading the previous tile's bias
#pragma unroll 1
    for (int tab = 0; tab < 2; ++tab) {
      float acc[C::NTAB / 2];
      qk_wgmma<C::NTAB, TAIL>(acc, qa, qtail, sbase + C::TAB_OFF + tab * TILE_TAB, C::NTAB);
      float* dst = tab ? relw : relh;
#pragma unroll
      for (int x = 0; x < C::NTAB / 2; ++x) {
        const int r = r0 + 8 * ((x >> 1) & 1);
        const int tq = q0 + r;
        const int qc = tab ? tq % S : tq / S;          // query coordinate along the table's axis
        const int t = 8 * (x >> 2) + cq + (x & 1);     // table index t = q - k + S - 1
        const int k = qc + S - 1 - t;
        if (t < C::NREL && k >= 0 && k < S) dst[r * SP + k] = acc[x] * LOG2E;
      }
    }
    named_bar_sync(1 + wg, 128);

    // S = 32 / 64: register x of the score fragment is key column kw = 8 ((x / 4) % CPS) + cq + x % 2 of every S-key
    // block; the thread keeps those rel_w terms of its two rows in registers
    float rw[2][2 * CPS];
    if constexpr (REG_W) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int m = 0; m < 2 * CPS; ++m) rw[i][m] = relw[(r0 + 8 * i) * SP + 8 * (m >> 1) + cq + (m & 1)];
    }

    float om[32], ot[8];
#pragma unroll
    for (int y = 0; y < 32; ++y) om[y] = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) ot[y] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const float scale2 = p.scale2;

#pragma unroll(REG_W ? 1 : NKT)
    for (int j = 0; j < NKT; ++j, ++g) {
      const int s = g % STAGES;
      const uint32_t ph = (g / STAGES) & 1;
      const uint32_t kb = sbase + C::KV_OFF + s * C::STAGE_BYTES, vb = kb + TILE_KV;
      mbar_wait(smem_u32(&bar_k[s]), ph);
      float sc[BN / 2];
      qk_wgmma<BN, TAIL>(sc, qa, qtail, kb, BN);
      if (j == NKT - 1) {   // the last Q K^T of this query tile has retired: its Q buffer may be refilled
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bar_qe[qb]));
      }

      // scores in the log2 domain with the bias; keys past T (last window tile) drop out
      float mx[2] = {-INFINITY, -INFINITY};
      if constexpr (REG_W) {
        constexpr int NB = BN / S;   // S-key blocks per tile: one rel_h value per row and block
        float bh[2][NB];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int b = 0; b < NB; ++b) bh[i][b] = relh[(r0 + 8 * i) * SP + j * NB + b];
#pragma unroll
        for (int x = 0; x < BN / 2; ++x) {
          const int i = (x >> 1) & 1;
          const float t = fmaf(sc[x], scale2, bh[i][(x >> 2) / CPS] + rw[i][((x >> 2) % CPS) * 2 + (x & 1)]);
          sc[x] = t;
          mx[i] = fmaxf(mx[i], t);
        }
      } else {
#pragma unroll
        for (int x = 0; x < BN / 2; ++x) {
          const int i = (x >> 1) & 1;
          const int key = j * BN + 8 * (x >> 2) + cq + (x & 1);
          float t = -INFINITY;
          if (T % BN == 0 || key < T) {
            const int kh = key / S, kw = key - kh * S;
            const int r = r0 + 8 * i;
            t = fmaf(sc[x], scale2, relh[r * SP + kh] + relw[r * SP + kw]);
          }
          sc[x] = t;
          mx[i] = fmaxf(mx[i], t);
        }
      }
      float alpha[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
        mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
        const float m_new = fmaxf(m_run[i], mx[i]);
        alpha[i] = fast_exp2(m_run[i] - m_new);
        m_run[i] = m_new;
        l_run[i] *= alpha[i];
      }
#pragma unroll
      for (int y = 0; y < 32; ++y) om[y] *= alpha[(y >> 1) & 1];
#pragma unroll
      for (int y = 0; y < 8; ++y) ot[y] *= alpha[(y >> 1) & 1];
      // P = exp2(t - m) -> fp16 A fragments of P V: k16 step kk holds score registers 8 kk .. 8 kk + 7
      uint32_t pa[BN / 16][4];
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk) {
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          const int x = 8 * kk + 2 * h, i = h & 1;
          const float p0 = fast_exp2(sc[x] - m_run[i]), p1 = fast_exp2(sc[x + 1] - m_run[i]);
          l_run[i] += p0 + p1;
          pa[kk][h] = pack_f16x2(p0, p1);
        }
      }
      mbar_wait(smem_u32(&bar_vc[s]), ph);
      acc_fence(om);
      acc_fence(ot);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk) {
        WgmmaRsF16<64>::rs(om, pa[kk], make_gdesc(vb + kk * 2048, BN * 128, 1024));
        if constexpr (TAIL > 0) WgmmaRsF16<16>::rs(ot, pa[kk], make_gdesc_sw32(vb + BN * 128 + kk * 512, 256, 256));
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(om);
      acc_fence(ot);
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&bar_e[s]));
    }

    // ---- epilogue: O / l -> out[token, head*HD .. ]
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float l = l_run[i];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const float inv = 1.0f / l;
      const int tq = q0 + r0 + 8 * i;
      if (tq >= T) continue;
      int dst = seq * T + tq;
      if (p.out_row_map) dst = __ldg(p.out_row_map + dst);
      if (dst < 0) continue;
      __nv_bfloat16* orow = p.out + static_cast<size_t>(dst) * p.D + head * HD + cq;
#pragma unroll
      for (int nb = 0; nb < 8; ++nb)
        *reinterpret_cast<uint32_t*>(orow + nb * 8) = pack_bf16x2(om[4 * nb + 2 * i] * inv, om[4 * nb + 2 * i + 1] * inv);
      if constexpr (TAIL > 0) {
#pragma unroll
        for (int nb = 0; nb < 2; ++nb)
          *reinterpret_cast<uint32_t*>(orow + 64 + nb * 8) =
              pack_bf16x2(ot[4 * nb + 2 * i] * inv, ot[4 * nb + 2 * i + 1] * inv);
      }
    }
  }
}

template <int HD, int S>
static int launch_att(const AttentionArgs& a, cudaStream_t stream) {
  using C = AttCfg<HD, S>;
  RSP_CHECK_ARG((reinterpret_cast<uintptr_t>(a.qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.rel_h) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(a.rel_w) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.out) & 3) == 0,
                "attention: qkv / tables must be 16-byte aligned");
  AttDev p;
  p.out = static_cast<__nv_bfloat16*>(a.out);
  p.out_row_map = a.out_row_map;
  p.H = a.H; p.D = a.H * HD;
  p.scale2 = (1.0f / sqrtf(static_cast<float>(HD))) * LOG2E;
  // qkv as (column, token, sequence): a box never reads past its sequence (rows >= T of the last tile are zero)
  const uint64_t ld = 3ull * p.D;
  const uint64_t qdims[3] = {ld, static_cast<uint64_t>(C::T), static_cast<uint64_t>(a.n_seq)};
  const uint64_t qstr[2] = {ld * 2, ld * 2 * C::T};
  const uint64_t tdims[2] = {static_cast<uint64_t>(HD), static_cast<uint64_t>(C::NREL)};
  const uint64_t tstr[1] = {static_cast<uint64_t>(HD) * 2};
  // boxes: Q tiles of BM rows, K / V tiles of BN rows (the box is what each load's transaction bytes count)
  const uint32_t qbox[3] = {64, C::BM, 1}, qbox_t[3] = {16, C::BM, 1};
  const uint32_t kvbox[3] = {64, C::BN, 1}, kvbox_t[3] = {16, C::BN, 1};
  const uint32_t tbox[2] = {64, static_cast<uint32_t>(C::NTAB)}, tbox_t[2] = {16, static_cast<uint32_t>(C::NTAB)};
  CUtensorMap tq, tkv, th, tw, tq_t, tkv_t, th_t, tw_t;
  RSP_TRY(make_tmap_swizzled(&tq, a.qkv, 3, qdims, qstr, qbox, 0, 128));
  RSP_TRY(make_tmap_swizzled(&tkv, a.qkv, 3, qdims, qstr, kvbox, 0, 128));
  RSP_TRY(make_tmap_swizzled(&th, a.rel_h, 2, tdims, tstr, tbox, 0, 128));
  RSP_TRY(make_tmap_swizzled(&tw, a.rel_w, 2, tdims, tstr, tbox, 0, 128));
  if (C::TAIL > 0) {
    RSP_TRY(make_tmap_swizzled(&tq_t, a.qkv, 3, qdims, qstr, qbox_t, 0, 32));
    RSP_TRY(make_tmap_swizzled(&tkv_t, a.qkv, 3, qdims, qstr, kvbox_t, 0, 32));
    RSP_TRY(make_tmap_swizzled(&th_t, a.rel_h, 2, tdims, tstr, tbox_t, 0, 32));
    RSP_TRY(make_tmap_swizzled(&tw_t, a.rel_w, 2, tdims, tstr, tbox_t, 0, 32));
  } else {   // hd = 64 has no tail; the kernel never reads these
    tq_t = tq; tkv_t = tkv; th_t = th; tw_t = tw;
  }
  auto kern = vit_attention_kernel<HD, S>;
  static bool attr_set_dev[kMaxDevices] = {};   // the attribute is per device (one flag per ordinal)
  bool& attr_set = attr_set_dev[current_device()];
  if (!attr_set) {
    RSP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    attr_set = true;
  }
  const long long items = static_cast<long long>(a.n_seq) * a.H * C::NQT;
  RSP_CHECK_ARG(items > 0 && items < (1ll << 31), "attention: %lld query tiles", items);
  p.n_items = static_cast<int>(items);
  const int grid = static_cast<int>(items < num_sms() ? items : num_sms());   // one CTA per SM
  kern<<<grid, 384, C::SMEM_BYTES, stream>>>(tq, tq_t, tkv, tkv_t, th, th_t, tw, tw_t, p);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

int vit_attention(const AttentionArgs& a, cudaStream_t stream) {
  RSP_CHECK_ARG(a.qkv && a.rel_h && a.rel_w && a.out, "attention: null pointer");
  RSP_CHECK_ARG(a.T == a.S * a.S, "attention: T=%d is not S^2 (S=%d)", a.T, a.S);
  RSP_CHECK_ARG(a.n_seq > 0 && a.H > 0, "attention: bad n_seq/H");
  if (a.S != 14 && a.S != 32 && a.S != 64)   // other grids (768^2 / 1280^2 inputs): CUDA-core kernel
    return vit_attention_simt(a, stream);
  if (a.hd == 64) {
    if (a.S == 64) return launch_att<64, 64>(a, stream);
    if (a.S == 32) return launch_att<64, 32>(a, stream);
    return launch_att<64, 14>(a, stream);
  }
  if (a.hd == 80) {
    if (a.S == 64) return launch_att<80, 64>(a, stream);
    if (a.S == 32) return launch_att<80, 32>(a, stream);
    return launch_att<80, 14>(a, stream);
  }
  set_last_error("attention: head dim %d unsupported (64, 80)", a.hd);
  return RSP_ERR_UNSUPPORTED;
}

// ---------------------------------------------------------------------------------------
// SIMT restatement (one thread per query row, fp32 throughout): the device-side check of
// the tensor-core kernel in the native self-test, and the path for grid sizes the tensor-core
// kernel does not specialise (S other than 14 / 64).
__global__ void vit_attention_simt_kernel(const __nv_bfloat16* __restrict__ qkv,
                                          const __nv_bfloat16* __restrict__ rel_h,
                                          const __nv_bfloat16* __restrict__ rel_w,
                                          __nv_bfloat16* __restrict__ out, int T, int S, int H,
                                          int hd, float scale, const int* __restrict__ out_row_map) {
  const int D = H * hd;
  const int tq = blockIdx.x * blockDim.x + threadIdx.x;
  const int head = blockIdx.y;
  const int seq = blockIdx.z;
  if (tq >= T) return;
  const int qh = tq / S, qw = tq % S;
  const __nv_bfloat16* qp = qkv + (static_cast<size_t>(seq) * T + tq) * 3 * D + head * hd;
  float q[128];
  for (int d = 0; d < hd; ++d) q[d] = __bfloat162float(qp[d]);
  float rh[128], rw[128];  // S <= 128
  for (int k = 0; k < S; ++k) {
    float ah = 0.f, aw = 0.f;
    const __nv_bfloat16* th = rel_h + static_cast<size_t>(qh - k + S - 1) * hd;
    const __nv_bfloat16* tw = rel_w + static_cast<size_t>(qw - k + S - 1) * hd;
    for (int d = 0; d < hd; ++d) {
      ah += q[d] * __bfloat162float(th[d]);
      aw += q[d] * __bfloat162float(tw[d]);
    }
    rh[k] = ah; rw[k] = aw;
  }
  float m = -INFINITY, l = 0.f;
  float o[128];
  for (int d = 0; d < hd; ++d) o[d] = 0.f;
  for (int k = 0; k < T; ++k) {
    const __nv_bfloat16* kp = qkv + (static_cast<size_t>(seq) * T + k) * 3 * D + D + head * hd;
    const __nv_bfloat16* vp = kp + D;
    float s = 0.f;
    for (int d = 0; d < hd; ++d) s += q[d] * __bfloat162float(kp[d]);
    s = s * scale + rh[k / S] + rw[k % S];
    const float mn = fmaxf(m, s);
    const float a = expf(m - mn), pe = expf(s - mn);
    l = l * a + pe;
    for (int d = 0; d < hd; ++d) o[d] = o[d] * a + pe * __bfloat162float(vp[d]);
    m = mn;
  }
  int dst = seq * T + tq;
  if (out_row_map) dst = out_row_map[dst];
  if (dst < 0) return;
  __nv_bfloat16* op = out + static_cast<size_t>(dst) * D + head * hd;
  for (int d = 0; d < hd; ++d) op[d] = __float2bfloat16_rn(o[d] / l);
}

int vit_attention_simt(const AttentionArgs& a, cudaStream_t stream) {
  RSP_CHECK_ARG(a.qkv && a.rel_h && a.rel_w && a.out, "attention_simt: null pointer");
  RSP_CHECK_ARG(a.T == a.S * a.S && a.S <= 128 && a.hd <= 128, "attention_simt: bad T/S/hd");
  dim3 block(64);
  dim3 grid((a.T + 63) / 64, a.H, a.n_seq);
  vit_attention_simt_kernel<<<grid, block, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(a.qkv), static_cast<const __nv_bfloat16*>(a.rel_h),
      static_cast<const __nv_bfloat16*>(a.rel_w), static_cast<__nv_bfloat16*>(a.out), a.T, a.S, a.H,
      a.hd, 1.0f / sqrtf(static_cast<float>(a.hd)), a.out_row_map);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace rsp
