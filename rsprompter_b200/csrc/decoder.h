#pragma once
#include "host_util.h"

namespace rsp {

int add_cast_bf16(const float* a, const float* b, void* out, long long n, long long b_mod,
                  cudaStream_t stream);
int token_self_attention(const void* q, const void* k, const void* v, void* out, int N, int T,
                         int heads, int c, cudaStream_t stream);
int t2i_attention(const void* q, const void* K, const void* V, int ldkv, const int* kv_block, void* out, int N,
                  int Tq, int HW, cudaStream_t stream);
int t2i_fused(const void* keys, int ldk, const void* kvw, const float* kvb, const void* pe_kv, const void* q,
              void* out, int N, int Tq, int HW, cudaStream_t stream);
int i2t_attention(const void* Q, const int* q_block, const void* ktok, const void* vtok, void* out,
                  int N, int Tq, int HW, cudaStream_t stream);
int i2t_fused(const void* keys, int ldk, const void* wq, const float* qb, const void* pe_q, const void* ktok,
              const void* vtok, const void* wo, const float* ob, const float* ln_g, const float* ln_b, float eps,
              void* out, int N, int Tq, int HW, cudaStream_t stream);

}  // namespace rsp
