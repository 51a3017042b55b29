#pragma once
#include "host_util.h"

namespace rsp {

// qkv: bf16 [n_seq * T, 3 * H * hd], columns ordered [q | k | v], each split into H heads
// (the layout nn.Linear(dim, 3 * dim) produces; reference modeling_sam.py:806-812).
// rel_h / rel_w: bf16 [2S-1, hd] tables of this layer.  out: bf16 [n_seq * T, H * hd].
struct AttentionArgs {
  const void* qkv = nullptr;
  const void* rel_h = nullptr;
  const void* rel_w = nullptr;
  void* out = nullptr;
  int n_seq = 0;  // windows (B * 25) or images (B)
  int T = 0;      // tokens per sequence = S * S
  int S = 0;      // 14 (window) or 64 (global, 1024^2 input)
  int H = 0;
  int hd = 0;     // 64 (ViT-B/L) or 80 (ViT-H)
  const int* out_row_map = nullptr;   // int32 [n_seq * T]: destination row of each output row (-1 = drop), or null
};

int vit_attention(const AttentionArgs& a, cudaStream_t stream);
int vit_attention_simt(const AttentionArgs& a, cudaStream_t stream);
// pieces of the three-pass path for other grids (attention_generic.cu)
int attn_softmax_bias(const float* scores, int lds, const float* tab, int ldt, int NT, void* P, int ldp, int n_rows,
                      int T, int S, float scale, cudaStream_t stream);
int transpose_cols(const void* in, int ld, int col0, int C, int n_seq, int T, void* out, cudaStream_t stream);
int split_heads(const void* in, int ld, int col0, int H, int hd, int n_seq, int T, void* out, cudaStream_t stream);

}  // namespace rsp
