// Native self-test of the tensor-core ViT attention kernel against the SIMT restatement.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "attention.h"

namespace rsp { const char* last_error(); }
using namespace rsp;

#define CK(x)                                                                        \
  do {                                                                               \
    cudaError_t e = (x);                                                             \
    if (e != cudaSuccess) {                                                          \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      exit(2);                                                                       \
    }                                                                                \
  } while (0)

static uint32_t a_seed = 777;
static float arand() {
  a_seed = a_seed * 1664525u + 1013904223u;
  return ((a_seed >> 8) & 0xffff) / 65536.0f - 0.5f;
}
static uint16_t f2bf(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  uint32_t r = ((u >> 16) & 1) + 0x7fff;
  return (uint16_t)((u + r) >> 16);
}
static float bf2f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

static int attn_case(const char* name, int n_seq, int S, int H, int hd, float qk_mag, float tab_mag,
                     int bench) {
  const int T = S * S, D = H * hd;
  const size_t m_tok = (size_t)n_seq * T;
  std::vector<uint16_t> hqkv(m_tok * 3 * D), hrh((size_t)(2 * S - 1) * hd), hrw((size_t)(2 * S - 1) * hd);
  for (auto& x : hqkv) x = f2bf(arand() * qk_mag);
  for (auto& x : hrh) x = f2bf(arand() * tab_mag);
  for (auto& x : hrw) x = f2bf(arand() * tab_mag);
  void *dqkv, *drh, *drw, *do1, *do2;
  CK(cudaMalloc(&dqkv, hqkv.size() * 2));
  CK(cudaMalloc(&drh, hrh.size() * 2));
  CK(cudaMalloc(&drw, hrw.size() * 2));
  CK(cudaMalloc(&do1, m_tok * D * 2));
  CK(cudaMalloc(&do2, m_tok * D * 2));
  CK(cudaMemcpy(dqkv, hqkv.data(), hqkv.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(drh, hrh.data(), hrh.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(drw, hrw.data(), hrw.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemset(do1, 0xff, m_tok * D * 2));
  CK(cudaMemset(do2, 0xff, m_tok * D * 2));
  AttentionArgs a;
  a.qkv = dqkv; a.rel_h = drh; a.rel_w = drw; a.n_seq = n_seq; a.T = T; a.S = S; a.H = H; a.hd = hd;
  a.out = do1;
  int s = vit_attention(a, 0);
  if (s) { printf("[%s] vit_attention failed: %s\n", name, last_error()); return 1; }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("[%s] kernel error: %s\n", name, cudaGetErrorString(e)); exit(3); }
  int fail = 0;
  if (!bench) {
    a.out = do2;
    s = vit_attention_simt(a, 0);
    if (s) { printf("[%s] simt failed: %s\n", name, last_error()); return 1; }
    CK(cudaDeviceSynchronize());
    std::vector<uint16_t> h1(m_tok * D), h2(m_tok * D);
    CK(cudaMemcpy(h1.data(), do1, h1.size() * 2, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(h2.data(), do2, h2.size() * 2, cudaMemcpyDeviceToHost));
    double maxerr = 0, maxref = 0;
    size_t nbad = 0, first_bad = (size_t)-1;
    for (size_t i = 0; i < h2.size(); ++i) if (fabs(bf2f(h2[i])) > maxref) maxref = fabs(bf2f(h2[i]));
    // P is rounded to bf16 and the rel-pos row term to fp16 before the exp: judge the error
    // against the output scale (norm-wise), 1.5 % of max|ref|.
    for (size_t i = 0; i < h1.size(); ++i) {
      const float x = bf2f(h1[i]), y = bf2f(h2[i]);
      const double d = fabs((double)x - (double)y);
      if (!(d <= 1.5e-2 * maxref)) { if (!nbad) first_bad = i; ++nbad; }
      if (d > maxerr || d != d) maxerr = d;
      if (fabs(y) > maxref) maxref = fabs(y);
    }
    printf("[%s] n_seq=%d S=%d H=%d hd=%d  max|diff|=%.3e max|ref|=%.3e bad=%zu/%zu %s\n", name,
           n_seq, S, H, hd, maxerr, maxref, nbad, h1.size(), nbad ? "FAIL" : "PASS");
    if (nbad) {
      const size_t row = first_bad / D, col = first_bad % D;
      printf("   first bad at token %zu (seq %zu, t %zu) col %zu: got %.4f want %.4f\n", row, row / T,
             row % T, col, bf2f(h1[first_bad]), bf2f(h2[first_bad]));
      for (int rr = 0; rr < 3; ++rr) {
        printf("   tok %d:", rr * 77);
        for (int j = 0; j < 6; ++j)
          printf(" %.4f/%.4f", bf2f(h1[(size_t)rr * 77 * D + j]), bf2f(h2[(size_t)rr * 77 * D + j]));
        printf("\n");
      }
      fail = 1;
    }
  } else {
    for (int i = 0; i < 3; ++i) vit_attention(a, 0);
    CK(cudaDeviceSynchronize());
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int iters = 10;
    cudaEventRecord(e0);
    for (int i = 0; i < iters; ++i) vit_attention(a, 0);
    cudaEventRecord(e1);
    CK(cudaDeviceSynchronize());
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    ms /= iters;
    const double flops = 4.0 * n_seq * H * (double)T * T * hd;
    printf("bench attn [%s] n_seq=%d S=%d H=%d hd=%d: %.3f ms  %.1f TFLOP/s (QK^T+PV)\n", name, n_seq,
           S, H, hd, ms, flops / ms * 1e-9);
  }
  cudaFree(dqkv); cudaFree(drh); cudaFree(drw); cudaFree(do1); cudaFree(do2);
  return fail;
}

int selftest_attention(int bench) {
  int fails = 0;
  fails += attn_case("win-hd64", 3, 14, 2, 64, 2.0f, 1.0f, 0);
  fails += attn_case("win-hd80", 3, 14, 2, 80, 2.0f, 1.0f, 0);
  fails += attn_case("win-hd64-many", 50, 14, 12, 64, 3.0f, 2.0f, 0);
  fails += attn_case("glob-hd64", 1, 64, 2, 64, 2.0f, 1.0f, 0);
  fails += attn_case("glob-hd80", 1, 64, 2, 80, 2.0f, 1.0f, 0);
  fails += attn_case("glob-hd64-sharp", 2, 64, 3, 64, 6.0f, 3.0f, 0);
  if (bench) {
    attn_case("vitb-window", 200, 14, 12, 64, 2.0f, 1.0f, 1);
    attn_case("vitb-global", 8, 64, 12, 64, 2.0f, 1.0f, 1);
    attn_case("vith-window", 200, 14, 16, 80, 2.0f, 1.0f, 1);
    attn_case("vith-global", 8, 64, 16, 80, 2.0f, 1.0f, 1);
  }
  return fails;
}
