// Checked entry points of the bf16 GEMM: out = epilogue(A[M,K] * W[N,K]^T).  Every argument the tensor-core kernel
// (gemm_v2.cu) relies on, alignment included, is checked here before any launch: a call that breaks one returns
// RSP_ERR_INVALID.
//
// gemm_bf16 is every dense contraction on the RSPrompter inference path: ViT qkv / proj / MLP linears (reference:
// transformers modeling_sam.py SamVisionAttention .qkv/.proj, SamMLPBlock; mmpretrain vit_sam.py:189-190,282),
// patch-embed and neck convs after re-layout, FPN / RPN / RoI-head convs and FCs, and the mask decoder's projections.
// window_unpartition (modeling_sam.py:925-952) is the `row_map` scatter in the epilogue, the residual adds of
// SamVisionLayer.forward (:966-971) are `residual`.
#include "gemm.h"
#include "sm90.cuh"

namespace rsp {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = one 128-byte swizzle row

enum { EPI_STD = 0, EPI_LN_ROW = 1, EPI_LN64_GELU = 2, EPI_GELU_HYPER = 3 };

static bool aligned(const void* ptr, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1)) == 0; }

int gemm_upscale_masks(const GemmArgs& a, int n_out, cudaStream_t stream) {
  RSP_CHECK_ARG(a.A && a.W && a.bias && a.hyper && a.mask_out, "gemm_upscale_masks: null pointer");
  RSP_CHECK_ARG(n_out >= 1 && n_out <= 3, "gemm_upscale_masks: n_out %d (1 to 3)", n_out);
  RSP_CHECK_ARG(a.M > 0 && a.K > 0 && a.N == 128 && a.lda % 8 == 0 && a.ldw % 8 == 0 && a.grid_h > 0 &&
                a.grid_w > 0 && a.M % (4 * a.grid_h * a.grid_w) == 0,
                "gemm_upscale_masks: needs N == 128 and M = prompts * 4 * h * w");
  // float4 hyper and bias loads, float2 mask stores (at even columns of rows 4 * grid_w wide)
  RSP_CHECK_ARG(aligned(a.hyper, 16) && aligned(a.bias, 16) && aligned(a.mask_out, 8), "gemm_upscale_masks: alignment");
  return gemm_bf16_v2_gelu_hyper_multi(a, n_out, stream);
}

int gemm_bf16(const GemmArgs& a, cudaStream_t stream) {
  RSP_CHECK_ARG(a.A && a.W && (a.epi_mode == EPI_GELU_HYPER ? a.mask_out != nullptr : a.out != nullptr),
                "gemm: null pointer");
  RSP_CHECK_ARG(a.M > 0 && a.N > 0 && a.K > 0, "gemm: bad shape %d %d %d", a.M, a.N, a.K);
  RSP_CHECK_ARG(a.lda % 8 == 0 && a.ldw % 8 == 0, "gemm: lda/ldw must be multiples of 8 bf16");
  RSP_CHECK_ARG(a.act >= 0 && a.act <= 2, "gemm: act %d", a.act);
  if (a.res_block_map) RSP_CHECK_ARG(a.res_block_rows > 0, "gemm: res_block_rows");
  // The fused epilogues make vector accesses (16-byte rows, float4 / float2 loads and stores) whose alignment is
  // checked here: a misaligned pointer is rejected before launch.
  if (a.epi_mode == EPI_LN_ROW) {
    RSP_CHECK_ARG(a.N % 32 == 0 && a.N <= 256 && a.ln_gamma && a.ln_beta && !a.row_map,
                  "gemm: row-LN epilogue needs N %% 32 == 0, N <= 256, gamma/beta");
    // both row-LN epilogues move 16 bytes at a time through out, residual, bias, gamma and beta
    RSP_CHECK_ARG(a.ldo % 8 == 0 && (!a.residual || a.ldr % 8 == 0) && aligned(a.out, 16) && aligned(a.residual, 16) &&
                  aligned(a.bias, 16) && aligned(a.ln_gamma, 16) && aligned(a.ln_beta, 16),
                  "gemm: row-LN epilogue alignment");
  } else if (a.epi_mode == EPI_LN64_GELU) {
    RSP_CHECK_ARG(a.N % 128 == 0 && a.bias && a.ln_gamma && a.ln_beta && !a.out_fp32 && !a.row_map,
                  "gemm: LN64+GELU epilogue needs N %% 128 == 0, bias, bf16 out");
    // float4 bias / gamma / beta loads; out is a TMA store (16-byte aligned rows) or 8-byte stores
    RSP_CHECK_ARG(aligned(a.out, 8) && a.ldo % 4 == 0 && aligned(a.bias, 16) && aligned(a.ln_gamma, 16) &&
                  aligned(a.ln_beta, 16), "gemm: LN64+GELU epilogue alignment");
  } else if (a.epi_mode == EPI_GELU_HYPER) {
    RSP_CHECK_ARG(a.N == 128 && a.bias && a.hyper && a.mask_out && a.grid_h > 0 && a.grid_w > 0 &&
                  a.M % (4 * a.grid_h * a.grid_w) == 0,
                  "gemm: GELU+hyper epilogue needs N == 128 and M = prompts * 4 * h * w");
    // float4 hyper and bias loads, float2 mask stores (at even columns of rows 4 * grid_w wide)
    RSP_CHECK_ARG(aligned(a.hyper, 16) && aligned(a.bias, 16) && aligned(a.mask_out, 8),
                  "gemm: GELU+hyper epilogue alignment");
  } else {
    RSP_CHECK_ARG(a.epi_mode == EPI_STD, "gemm: epi_mode %d", a.epi_mode);
    if (a.m_group_rows > 0)
      RSP_CHECK_ARG(a.m_group_rows % BM == 0 && a.M % a.m_group_rows == 0 && a.w_group_rows > 0 && a.conv_c == 0 &&
                    gemm_vector_rows(a), "gemm: grouped weights need m_group_rows %% 128 == 0 and aligned output rows");
  }
  return gemm_bf16_v2(a, stream);
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
  RSP_CHECK_ARG(a.epi_mode == EPI_STD && !a.row_map && a.act >= 0 && a.act <= 2, "conv3x3: epilogue");
  RSP_CHECK_ARG(gemm_vector_rows(a), "conv3x3: output / residual alignment");
  return gemm_bf16_v2(a, stream);
}

// ---------------------------------------------------------------------------------------
// Plain SIMT GEMM with the standard epilogue contract: the independent check of the tensor-core kernel in the device
// self-test and the tests.
__global__ void gemm_bf16_simt_kernel(const GemmArgs p) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = blockIdx.y;
  if (col >= p.N || row >= p.M) return;
  const __nv_bfloat16* A = static_cast<const __nv_bfloat16*>(p.A);
  const __nv_bfloat16* W = static_cast<const __nv_bfloat16*>(p.W);
  float acc = 0.f;
  for (int k = 0; k < p.K; ++k)
    acc += __bfloat162float(A[static_cast<size_t>(row) * p.lda + k]) *
           __bfloat162float(W[static_cast<size_t>(col) * p.ldw + k]);
  const int orow = p.row_map ? p.row_map[row] : row;
  if (orow < 0) return;
  const int blk = p.res_block_map ? orow / p.res_block_rows : 0;
  const int rrow = p.res_block_map ? p.res_block_map[blk] * p.res_block_rows + (orow - blk * p.res_block_rows)
                                   : p.res_mod > 0 ? (orow % p.res_mod) : orow;
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
  dim3 block(128);
  dim3 grid((a.N + 127) / 128, a.M);
  gemm_bf16_simt_kernel<<<grid, block, 0, stream>>>(a);
  RSP_CHECK_LAUNCH();
  return RSP_OK;
}

}  // namespace rsp
