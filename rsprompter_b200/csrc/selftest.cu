// Native device self-test / micro-benchmark (no Python, no torch): fast to run on a GPU box.
//   ./rsp_selftest [gemm|attn|all] [bench]
// Every tensor-core kernel is compared with a plain SIMT implementation of the same contract.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "gemm.h"
#include "sm90.cuh"

namespace rsp { const char* last_error(); }
using namespace rsp;

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e = (x);                                                           \
    if (e != cudaSuccess) {                                                        \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      exit(2);                                                                     \
    }                                                                              \
  } while (0)

static uint32_t g_seed = 12345;
static float frand() {
  g_seed = g_seed * 1664525u + 1013904223u;
  return ((g_seed >> 8) & 0xffff) / 65536.0f - 0.5f;
}
static uint16_t f2bf(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  uint32_t r = ((u >> 16) & 1) + 0x7fff;
  return (uint16_t)((u + r) >> 16);
}

struct Case {
  const char* name;
  int M, N, K;
  int bias, act, residual, res_fp32, out_fp32, row_map, res_mod, w_is_kn, force_bn;
};

static int run_case(const Case& c) {
  const int M = c.M, N = c.N, K = c.K;
  std::vector<uint16_t> hA((size_t)M * K), hW((size_t)N * K);
  for (auto& x : hA) x = f2bf(frand());
  for (auto& x : hW) x = f2bf(frand() * 0.25f);
  std::vector<float> hb(N);
  for (auto& x : hb) x = frand();
  int out_rows = M;
  std::vector<int> hmap;
  if (c.row_map) {
    hmap.resize(M);
    // reversed order with every 7th row dropped
    int o = 0;
    for (int i = M - 1; i >= 0; --i) hmap[i] = (i % 7 == 3) ? -1 : o++;
    out_rows = o;
  }
  const int res_rows = c.res_mod > 0 ? c.res_mod : out_rows;
  std::vector<float> hres((size_t)res_rows * N);
  for (auto& x : hres) x = frand();
  std::vector<uint16_t> hres_bf((size_t)res_rows * N);
  for (size_t i = 0; i < hres.size(); ++i) hres_bf[i] = f2bf(hres[i]);

  void *dA, *dW, *dO1, *dO2, *dres;
  float* db;
  int* dmap = nullptr;
  const size_t osz = (size_t)out_rows * N * (c.out_fp32 ? 4 : 2);
  CK(cudaMalloc(&dA, hA.size() * 2));
  CK(cudaMalloc(&dW, hW.size() * 2));
  CK(cudaMalloc(&db, N * 4));
  CK(cudaMalloc(&dO1, osz));
  CK(cudaMalloc(&dO2, osz));
  CK(cudaMalloc(&dres, hres.size() * 4));
  CK(cudaMemcpy(dA, hA.data(), hA.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dW, hW.data(), hW.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(db, hb.data(), N * 4, cudaMemcpyHostToDevice));
  if (c.res_fp32) CK(cudaMemcpy(dres, hres.data(), hres.size() * 4, cudaMemcpyHostToDevice));
  else CK(cudaMemcpy(dres, hres_bf.data(), hres_bf.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemset(dO1, 0xff, osz));
  CK(cudaMemset(dO2, 0xff, osz));
  if (c.row_map) {
    CK(cudaMalloc(&dmap, M * 4));
    CK(cudaMemcpy(dmap, hmap.data(), M * 4, cudaMemcpyHostToDevice));
  }
  GemmArgs a;
  a.A = dA; a.W = dW; a.M = M; a.N = N; a.K = K;
  a.lda = K; a.ldw = c.w_is_kn ? N : K; a.ldo = N; a.ldr = N;
  a.bias = c.bias ? db : nullptr;
  a.residual = c.residual ? dres : nullptr;
  a.res_fp32 = c.res_fp32; a.out_fp32 = c.out_fp32; a.act = c.act;
  a.row_map = dmap; a.res_mod = c.res_mod; a.w_is_kn = c.w_is_kn; a.force_bn = c.force_bn;
  a.out = dO1;
  int s = gemm_bf16(a, 0);
  if (s) { printf("[%s] gemm_bf16 failed: %s\n", c.name, last_error()); return 1; }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("[%s] kernel error: %s\n", c.name, cudaGetErrorString(e)); exit(3); }
  a.out = dO2;
  s = gemm_bf16_simt(a, 0);
  if (s) { printf("[%s] simt failed: %s\n", c.name, last_error()); return 1; }
  CK(cudaDeviceSynchronize());
  std::vector<uint8_t> h1(osz), h2(osz);
  CK(cudaMemcpy(h1.data(), dO1, osz, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(h2.data(), dO2, osz, cudaMemcpyDeviceToHost));
  double maxerr = 0, maxref = 0;
  size_t nbad = 0;
  const size_t n = (size_t)out_rows * N;
  for (size_t i = 0; i < n; ++i) {
    float x, y;
    if (c.out_fp32) { x = ((float*)h1.data())[i]; y = ((float*)h2.data())[i]; }
    else {
      uint32_t ux = (uint32_t)((uint16_t*)h1.data())[i] << 16, uy = (uint32_t)((uint16_t*)h2.data())[i] << 16;
      memcpy(&x, &ux, 4); memcpy(&y, &uy, 4);
    }
    const double d = fabs((double)x - (double)y);
    if (!(d <= 1e-2 * (1.0 + fabs(y)))) ++nbad;
    if (d > maxerr || d != d) maxerr = d;
    if (fabs(y) > maxref) maxref = fabs(y);
  }
  printf("[%s] M=%d N=%d K=%d  max|diff|=%.3e  max|ref|=%.3e  bad=%zu/%zu  %s\n", c.name, M, N, K,
         maxerr, maxref, nbad, n, nbad == 0 ? "PASS" : "FAIL");
  if (nbad) {
    // dump a small corner for diagnosis
    for (int r = 0; r < 4 && r < out_rows; ++r) {
      printf("   row %d:", r);
      for (int j = 0; j < 8 && j < N; ++j) {
        float x, y;
        size_t i = (size_t)r * N + j;
        if (c.out_fp32) { x = ((float*)h1.data())[i]; y = ((float*)h2.data())[i]; }
        else {
          uint32_t ux = (uint32_t)((uint16_t*)h1.data())[i] << 16, uy = (uint32_t)((uint16_t*)h2.data())[i] << 16;
          memcpy(&x, &ux, 4); memcpy(&y, &uy, 4);
        }
        printf(" %.3f/%.3f", x, y);
      }
      printf("\n");
    }
  }
  cudaFree(dA); cudaFree(dW); cudaFree(db); cudaFree(dO1); cudaFree(dO2); cudaFree(dres);
  if (dmap) cudaFree(dmap);
  return nbad ? 1 : 0;
}

static void bench_gemm(int M, int N, int K, int bn, int act, int out_fp32, int residual, int res_bf16 = 0, int iters = 20, int res_mod = 0) {
  void *dA, *dW, *dO, *dR = nullptr;
  float* db;
  CK(cudaMalloc(&dA, (size_t)M * K * 2));
  CK(cudaMalloc(&dW, (size_t)N * K * 2));
  CK(cudaMalloc(&dO, (size_t)M * N * 4));
  CK(cudaMalloc(&db, N * 4));
  CK(cudaMemset(dA, 0x11, (size_t)M * K * 2));
  CK(cudaMemset(dW, 0x11, (size_t)N * K * 2));
  CK(cudaMemset(db, 0, N * 4));
  if (residual) { CK(cudaMalloc(&dR, (size_t)M * N * 4)); CK(cudaMemset(dR, 0, (size_t)M * N * 4)); }
  (void)res_bf16;
  GemmArgs a;
  a.A = dA; a.W = dW; a.out = dO; a.bias = db; a.M = M; a.N = N; a.K = K;
  a.lda = K; a.ldw = K; a.ldo = N; a.ldr = N; a.act = act; a.out_fp32 = out_fp32; a.force_bn = bn;
  a.residual = dR; a.res_fp32 = res_bf16 ? 0 : 1; a.res_mod = res_mod;
  for (int i = 0; i < 3; ++i) gemm_bf16(a, 0);
  CK(cudaDeviceSynchronize());
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  for (int i = 0; i < iters; ++i) gemm_bf16(a, 0);
  cudaEventRecord(e1);
  CK(cudaDeviceSynchronize());
  float ms;
  cudaEventElapsedTime(&ms, e0, e1);
  ms /= iters;
  const double bytes = (double)M * K * 2 + (double)N * K * 2 + (double)M * N * (out_fp32 ? 4 : 2) +
                       (residual ? (double)M * N * (res_bf16 ? 2 : 4) : 0.0);
  printf("bench gemm M=%d N=%d K=%d bn=%d act=%d outf32=%d res=%d%s: %.3f ms  %.1f TFLOP/s  %.0f GB/s\n", M, N, K,
         bn, act, out_fp32, residual, res_bf16 ? "(bf16)" : "", ms, 2.0 * M * N * K / ms * 1e-9, bytes / ms * 1e-6);
  cudaFree(dA); cudaFree(dW); cudaFree(dO); cudaFree(db);
  if (dR) cudaFree(dR);
}

int selftest_attention(int bench);


int main(int argc, char** argv) {
  const char* what = argc > 1 ? argv[1] : "all";
  const int bench = argc > 2 && !strcmp(argv[2], "bench");
  int fails = 0;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  printf("device: %s sm_%d%d, %d SMs\n", prop.name, prop.major, prop.minor, prop.multiProcessorCount);
  if (!strcmp(what, "gemm") || !strcmp(what, "all")) {
    const Case cases[] = {
        //            name        M     N     K   bias act res rf32 of32 map mod kn  bn
        {"tiny-f32",            128,  128,   64,  0, 0, 0, 1, 1, 0, 0, 0, 128},
        {"k128-f32",            256,  256,  128,  0, 0, 0, 1, 1, 0, 0, 0, 0},
        {"bn256",               384,  512,  256,  1, 0, 0, 1, 1, 0, 0, 0, 256},
        {"bn64",                200,   64,  192,  1, 2, 0, 1, 0, 0, 0, 0, 64},
        {"bn32",                200,   32,  192,  1, 2, 0, 1, 0, 0, 0, 0, 32},
        {"ragged-n",            300,   40,  128,  1, 0, 0, 1, 1, 0, 0, 0, 0},
        {"bias-gelu-bf16",     1000,  768,  768,  1, 1, 0, 1, 0, 0, 0, 0, 0},
        {"resid-f32",          1000,  768, 3072,  1, 0, 1, 1, 1, 0, 0, 0, 0},
        {"resid-bf16",          777,  256,  320,  1, 2, 1, 0, 0, 0, 0, 0, 0},
        {"rowmap-resid",       4000, 2304,  768,  1, 0, 1, 1, 1, 1, 0, 0, 256},
        {"posembed-mod",       2048,  768,  768,  1, 0, 1, 1, 1, 0, 512, 0, 0},
        {"multi-tile-per-cta", 40000, 256,  128,  1, 0, 0, 1, 0, 0, 0, 0, 0},
        {"w-kn-128",            512,  128,  256,  0, 0, 0, 1, 1, 0, 0, 1, 0},
        {"w-kn-64",             300,   64,  192,  1, 0, 0, 1, 1, 0, 0, 1, 0},
        {"w-kn-256n",           512,  256,  128,  0, 0, 0, 1, 1, 0, 0, 1, 0},
    };
    for (const Case& c : cases) fails += run_case(c);
    if (bench) {
      bench_gemm(32768, 2304, 768, 256, 0, 0, 0);
      bench_gemm(32768, 768, 768, 256, 0, 1, 1);
      bench_gemm(32768, 3072, 768, 256, 1, 0, 0);
      bench_gemm(32768, 768, 3072, 256, 0, 1, 1);
      bench_gemm(32768, 768, 3072, 128, 0, 1, 1);
      bench_gemm(8192, 8192, 8192, 256, 0, 0, 0);
      bench_gemm(8192, 8192, 8192, 128, 0, 0, 0);
    }
  }
  if (!strcmp(what, "gemmprof")) {
    // mask-decoder shapes (N prompts * 4096 image tokens rows)
    bench_gemm(1 << 20, 256, 128, 0, 0, 1, 1, 1, 3);   // i2t out_proj + bf16 residual -> fp32
    bench_gemm(1 << 20, 128, 256, 0, 0, 0, 0, 0, 3);   // k / v / q projections
    bench_gemm(1 << 20, 256, 128, 0, 0, 0, 0, 0, 3);
    bench_gemm(1 << 20, 128, 256, 0, 0, 0, 1, 0, 3, 4096);   // k-proj + broadcast fp32 residual (k_proj(pe))
  }
  if (!strcmp(what, "attn") || !strcmp(what, "all")) fails += selftest_attention(bench);
  printf("selftest: %d failing case(s)\n", fails);
  return fails ? 1 : 0;
}
