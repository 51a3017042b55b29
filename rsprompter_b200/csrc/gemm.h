#pragma once
#include "host_util.h"

namespace rsp {

// out[row_map[m], n] = act(sum_k A[m,k] * W[n,k] + bias[n]) + residual[row_map[m] % res_mod, n]
struct GemmArgs {
  const void* A = nullptr;   // bf16 [M, K], row stride lda
  const void* W = nullptr;   // bf16 [N, K] (nn.Linear layout), row stride ldw
  void* out = nullptr;       // bf16 or fp32 [*, ldo]
  const float* bias = nullptr;     // fp32 [N] or null
  const void* residual = nullptr;  // fp32 or bf16 [*, ldr] or null (may alias out)
  const int* row_map = nullptr;    // int32 [M] destination row (-1 = drop) or null = identity
  int M = 0, N = 0, K = 0;
  int lda = 0, ldw = 0, ldo = 0, ldr = 0;
  int res_mod = 0;    // if > 0 the residual row is (destination row % res_mod)
  int act = 0;        // 0 none, 1 GELU (erf; gelu_fast on the wgmma kernel), 2 ReLU   (applied before the residual add)
  int out_fp32 = 0;
  int res_fp32 = 1;
  // epilogue variants used by the mask decoder (see rsp_gemm_bf16 in rsp_b200.h)
  int epi_mode = 0;                   // 0 standard, 1 row LayerNorm, 2 LN over 64-column groups + GELU,
                                      // 3 GELU + hypernetwork dot + 2x2 mask scatter
  const float* ln_gamma = nullptr;
  const float* ln_beta = nullptr;
  float ln_eps = 1e-6f;
  const int* res_block_map = nullptr; // residual row = map[row / res_block_rows] * res_block_rows + row % res_block_rows
  int res_block_rows = 0;
  const float* hyper = nullptr;       // fp32 [prompts, 32]
  float* mask_out = nullptr;          // fp32 [prompts, 4*grid_h, 4*grid_w]
  int grid_h = 0, grid_w = 0;
  // implicit 3x3 / stride 1 / pad 1 convolution: A = bf16 NHWC [conv_b, conv_h, conv_w, conv_c], M = b*h*w,
  // K = 9 * conv_c, W = [N, (ky, kx, c)]; the im2col matrix is never built (TMA zero-fills the halo)
  int conv_b = 0, conv_h = 0, conv_w = 0, conv_c = 0;
  // grouped weights: rows [g * m_group_rows, (g+1) * m_group_rows) of A multiply W rows [g * w_group_rows, +N)
  // (every group has its own [N, K] operand; batched Q K^T / P V of the three-pass attention).  m_group_rows % 128 == 0.
  int m_group_rows = 0, w_group_rows = 0;
};

// checked entry points (gemm.cu): every argument the kernels rely on is checked here, before any launch
int gemm_bf16(const GemmArgs& a, cudaStream_t stream);
int gemm_bf16_simt(const GemmArgs& a, cudaStream_t stream);   // CUDA cores, standard epilogue: the tests' reference
bool conv3x3_geometry_ok(int B, int H, int W, int C);
int conv3x3_bf16(const GemmArgs& a, cudaStream_t stream);   // conv_* set; standard epilogue only
// the multi-output upscale: epi_mode 3 arguments + n_out
int gemm_upscale_masks(const GemmArgs& a, int n_out, cudaStream_t stream);

// the wgmma kernel (gemm_v2.cu), called by the entry points above with checked arguments
bool gemm_vector_rows(const GemmArgs& a);   // out / residual / bias rows the standard epilogue moves 8 bytes at a time
int gemm_bf16_v2(const GemmArgs& a, cudaStream_t stream);   // any epi_mode
// epi_mode 0 on the schedule given (wide: 128 x 256 tiles, epilogue in registers; else the split schedule), without
// gemm_bf16_v2's choice between them: the self-test's A/B of the two
int gemm_bf16_v2_std(const GemmArgs& a, bool wide, cudaStream_t stream);
// N == 128, hyper [prompts, n_out, 32], mask_out [prompts, n_out, 4*grid_h, 4*grid_w], 1 <= n_out <= 3
int gemm_bf16_v2_gelu_hyper_multi(const GemmArgs& a, int n_out, cudaStream_t stream);

}  // namespace rsp
