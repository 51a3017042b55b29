// ViT-SAM attention core for sm_90a: softmax(scale * q k^T + rel_h + rel_w) v per
// (sequence, head), sequences being 14x14 windows (T = 196) or whole 32x32 / 64x64 images
// (T = 1024 / 4096).  Reference: transformers modeling_sam.py SamVisionAttention.forward
// (:803-831), get_rel_pos / get_decomposed_rel_pos (:729-801); mmpretrain vit_sam.py
// Attention.forward (:202-221), add_decomposed_rel_pos (:117-157).
//
// Flash-style, everything in registers: one CTA = 64 query rows of one (sequence, head), 4 warps of 16 rows each.
// Scores and the output accumulator are bf16 mma.sync m16n8k16 fragments with fp32 accumulation; the score fragment
// of a 64-key tile becomes, after the online softmax, the A operand of P V without leaving the registers.  P V runs in
// fp16 (P in [0, 1] keeps 11 mantissa bits instead of bf16's 8; each V tile is converted in shared memory, exactly for
// |v| in fp16's normal range).  K / V tiles stream through a two-stage cp.async ring (rows padded by 16 bytes:
// conflict-free ldmatrix).
// The decomposed relative-position bias is never materialised as a T x T tensor: a prologue runs Q x table^T for both
// tables on the same tensor-core path (the reference's two einsums), scatters each row's S + S values (pre-multiplied
// by log2 e) into shared memory, and the bias is added to the scores before the exp.  Scores stay fp32 until the exp
// (reference: softmax in fp32).
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
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
// d (+)= a[16 x 16] * b[16 x 8], bf16 (or fp16) in, fp32 accumulators (row.col)
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_f16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

template <int HD, int S>
struct AttCfg {
  static constexpr int T = S * S;
  static constexpr int HDP = HD + 8;                  // padded smem row (bf16): 16-byte rows shift banks
  static constexpr int CH = HD / 8;                   // 16-byte chunks per row
  static constexpr int NKT = (T + 63) / 64;           // 64-key tiles
  static constexpr int NREL = 2 * S - 1;              // rel-pos table rows
  static constexpr int NTG = (NREL + 63) / 64;        // 64-row groups of a table
  static constexpr int SP = S + 4;                    // row stride of the gathered bias (floats)
  static constexpr int Q_ELEMS = 64 * HDP;
  static constexpr int KV_ELEMS = 128 * HDP;          // two 64-key stages (in the prologue: one whole table)
  static constexpr int SMEM_BYTES = (Q_ELEMS + 2 * KV_ELEMS) * 2 + 2 * 64 * SP * 4;
  static_assert(NREL <= 128, "table rows");
};

struct AttDev {
  const __nv_bfloat16* qkv;
  const __nv_bfloat16* rel_h;
  const __nv_bfloat16* rel_w;
  __nv_bfloat16* out;  // [M_tok, D]
  int H;
  int D;
  int n_qt;            // 64-query tiles per sequence
  float scale2;        // hd^-0.5 * log2(e)
  const int* out_row_map;   // window_unpartition + crop fused into the store (HF:925-952), or null
};

template <int HD, int S>
__global__ void __launch_bounds__(128)
vit_attention_kernel(const AttDev p) {
  using C = AttCfg<HD, S>;
  constexpr int T = C::T, HDP = C::HDP, CH = C::CH, SP = C::SP;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* sK = sQ + C::Q_ELEMS;
  __nv_bfloat16* sV = sK + C::KV_ELEMS;
  float* relh = reinterpret_cast<float*>(sV + C::KV_ELEMS);   // [64][SP]: rel_h term of (row, key row kh)
  float* relw = relh + 64 * SP;                               // [64][SP]: rel_w term of (row, key column kw)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int bid = blockIdx.x;
  const int qt = bid % p.n_qt; bid /= p.n_qt;
  const int head = bid % p.H;
  const int seq = bid / p.H;
  const int q0 = qt * 64;
  const size_t ld = static_cast<size_t>(3) * p.D;
  const __nv_bfloat16* base = p.qkv + static_cast<size_t>(seq) * T * ld;
  const int colq = head * HD, colk = p.D + head * HD, colv = 2 * p.D + head * HD;

  // rows [r0, r0 + nrows) of a [*, ldr] bf16 matrix (columns col0 .. col0 + HD) -> padded smem; rows >= nvalid -> 0
  auto load_rows = [&](__nv_bfloat16* dst, const __nv_bfloat16* src, size_t ldr, int col0, int r0, int nrows,
                       int nvalid) {
    for (int i = tid; i < nrows * CH; i += 128) {
      const int r = i / CH, c = i - (i / CH) * CH;
      const bool ok = r0 + r < nvalid;
      const __nv_bfloat16* g = src + static_cast<size_t>(ok ? r0 + r : 0) * ldr + col0 + c * 8;
      cp_async16(smem_u32(dst + r * HDP + c * 8), g, ok);
    }
  };
  load_rows(sQ, base, ld, colq, q0, 64, T);
  load_rows(sK, p.rel_h, HD, 0, 0, C::NTG * 64, C::NREL);
  load_rows(sV, p.rel_w, HD, 0, 0, C::NTG * 64, C::NREL);
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();

  // this thread's fragment coordinates: rows rl + 8 i (i = 0, 1) of the warp's 16, columns 2 (lane % 4) + {0, 1}
  const int rl = warp * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  uint32_t qf[HD / 16][4];
#pragma unroll
  for (int kk = 0; kk < HD / 16; ++kk)
    ldsm_x4(smem_u32(sQ + (warp * 16 + (lane & 15)) * HDP + kk * 16 + (lane >> 4) * 8), qf[kk][0], qf[kk][1],
            qf[kk][2], qf[kk][3]);
  // B operand (x4: two 8-row blocks of K-like [rows][HD] smem at k-step kk)
  const int b_row = (lane & 7) + ((lane >> 4) << 3), b_col = ((lane >> 3) & 1) * 8;

  // ---- prologue: Q x table^T for both tables, gathered into relh / relw (this warp's 16 rows only)
#pragma unroll 1
  for (int tab = 0; tab < 2; ++tab) {
    const __nv_bfloat16* tb = tab ? sV : sK;
    float* dst = tab ? relw : relh;
#pragma unroll 1
    for (int g = 0; g < C::NTG; ++g) {
      float acc[8][4];
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) acc[nb][0] = acc[nb][1] = acc[nb][2] = acc[nb][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) {
#pragma unroll
        for (int np = 0; np < 4; ++np) {
          uint32_t b0, b1, b2, b3;
          ldsm_x4(smem_u32(tb + (g * 64 + np * 16 + b_row) * HDP + kk * 16 + b_col), b0, b1, b2, b3);
          mma_bf16(acc[2 * np], qf[kk], b0, b1);
          mma_bf16(acc[2 * np + 1], qf[kk], b2, b3);
        }
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = rl + 8 * i;
        const int tq = q0 + r;
        const int qc = tab ? tq % S : tq / S;   // query coordinate along the table's axis
#pragma unroll
        for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int t = g * 64 + nb * 8 + cq + e;   // table index t = q - k + S - 1
            const int k = qc + S - 1 - t;
            if (t < C::NREL && k >= 0 && k < S) dst[r * SP + k] = acc[nb][2 * i + e] * LOG2E;
          }
        }
      }
    }
  }
  __syncthreads();   // the tables' smem becomes the K / V ring

  auto load_kv = [&](int j) {
    const int st = j & 1;
    load_rows(sK + st * 64 * HDP, base, ld, colk, j * 64, 64, T);
    load_rows(sV + st * 64 * HDP, base, ld, colv, j * 64, 64, T);
    cp_async_commit();
  };
  load_kv(0);

  float o[HD / 8][4];
#pragma unroll
  for (int nb = 0; nb < HD / 8; ++nb) o[nb][0] = o[nb][1] = o[nb][2] = o[nb][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float scale2 = p.scale2;
  const float* bh[2] = {relh + rl * SP, relh + (rl + 8) * SP};
  const float* bw[2] = {relw + rl * SP, relw + (rl + 8) * SP};
  // V operand (x4 trans: two 8-key halves of a 16-key step, two 8-column blocks)
  const int v_row = (lane & 7) + ((lane >> 3) & 1) * 8, v_col = (lane >> 4) * 8;

#pragma unroll 1
  for (int j = 0; j < C::NKT; ++j) {
    if (j + 1 < C::NKT) {
      load_kv(j + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const __nv_bfloat16* Ks = sK + (j & 1) * 64 * HDP;
    const __nv_bfloat16* Vs = sV + (j & 1) * 64 * HDP;
    {   // V tile bf16 -> fp16 in place
      uint32_t* v32 = reinterpret_cast<uint32_t*>(sV + (j & 1) * 64 * HDP);
      for (int i = tid; i < 64 * HDP / 2; i += 128) {
        const uint32_t w = v32[i];
        v32[i] = pack_f16x2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
      }
    }

    float sc[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) sc[nb][0] = sc[nb][1] = sc[nb][2] = sc[nb][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4(smem_u32(Ks + (np * 16 + b_row) * HDP + kk * 16 + b_col), b0, b1, b2, b3);
        mma_bf16(sc[2 * np], qf[kk], b0, b1);
        mma_bf16(sc[2 * np + 1], qf[kk], b2, b3);
      }
    }
    // scores in the log2 domain with the bias; keys past T (last window tile) drop out
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = j * 64 + nb * 8 + cq + (e & 1);
        const int i = e >> 1;
        float t = -INFINITY;
        if (T % 64 == 0 || key < T) {
          const int kh = key / S, kw = key - kh * S;
          t = fmaf(sc[nb][e], scale2, bh[i][kh] + bw[i][kw]);
        }
        sc[nb][e] = t;
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
    for (int nb = 0; nb < HD / 8; ++nb) {
      o[nb][0] *= alpha[0]; o[nb][1] *= alpha[0];
      o[nb][2] *= alpha[1]; o[nb][3] *= alpha[1];
    }
    // P = exp2(t - m) -> fp16 A fragments of P V
    uint32_t pa[4][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      const float p0 = fast_exp2(sc[nb][0] - m_run[0]), p1 = fast_exp2(sc[nb][1] - m_run[0]);
      const float p2 = fast_exp2(sc[nb][2] - m_run[1]), p3 = fast_exp2(sc[nb][3] - m_run[1]);
      l_run[0] += p0 + p1;
      l_run[1] += p2 + p3;
      pa[nb >> 1][(nb & 1) * 2 + 0] = pack_f16x2(p0, p1);
      pa[nb >> 1][(nb & 1) * 2 + 1] = pack_f16x2(p2, p3);
    }
    __syncthreads();   // the whole V tile is fp16
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int np = 0; np < HD / 16; ++np) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(smem_u32(Vs + (kk * 16 + v_row) * HDP + np * 16 + v_col), b0, b1, b2, b3);
        mma_f16(o[2 * np], pa[kk], b0, b1);
        mma_f16(o[2 * np + 1], pa[kk], b2, b3);
      }
    }
    __syncthreads();   // this stage may be refilled by the next iteration's load
  }

  // ---- epilogue: O / l -> out[token, head*HD .. ]
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_run[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const int tq = q0 + rl + 8 * i;
    if (tq >= T) continue;
    int dst = seq * T + tq;
    if (p.out_row_map) dst = __ldg(p.out_row_map + dst);
    if (dst < 0) continue;
    __nv_bfloat16* orow = p.out + static_cast<size_t>(dst) * p.D + colq + cq;
#pragma unroll
    for (int nb = 0; nb < HD / 8; ++nb)
      *reinterpret_cast<uint32_t*>(orow + nb * 8) = pack_bf16x2(o[nb][2 * i] * inv, o[nb][2 * i + 1] * inv);
  }
}

template <int HD, int S>
static int launch_att(const AttentionArgs& a, cudaStream_t stream) {
  using C = AttCfg<HD, S>;
  AttDev p;
  p.qkv = static_cast<const __nv_bfloat16*>(a.qkv);
  p.rel_h = static_cast<const __nv_bfloat16*>(a.rel_h);
  p.rel_w = static_cast<const __nv_bfloat16*>(a.rel_w);
  p.out = static_cast<__nv_bfloat16*>(a.out);
  p.H = a.H; p.D = a.H * HD;
  p.n_qt = (C::T + 63) / 64;
  p.scale2 = (1.0f / sqrtf(static_cast<float>(HD))) * LOG2E;
  p.out_row_map = a.out_row_map;
  RSP_CHECK_ARG((reinterpret_cast<uintptr_t>(a.qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.rel_h) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(a.rel_w) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.out) & 3) == 0,
                "attention: qkv / tables must be 16-byte aligned");
  auto kern = vit_attention_kernel<HD, S>;
  static bool attr_set_dev[kMaxDevices] = {};   // the attribute is per device (one flag per ordinal)
  bool& attr_set = attr_set_dev[current_device()];
  if (!attr_set) {
    RSP_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    attr_set = true;
  }
  const long long grid = static_cast<long long>(a.n_seq) * a.H * p.n_qt;
  RSP_CHECK_ARG(grid > 0 && grid < (1ll << 31), "attention: grid %lld", grid);
  kern<<<static_cast<unsigned>(grid), 128, C::SMEM_BYTES, stream>>>(p);
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
