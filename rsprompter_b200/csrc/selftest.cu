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
  int bias, act, residual, res_fp32, out_fp32, row_map, res_mod;
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
  a.lda = K; a.ldw = K; a.ldo = N; a.ldr = N;
  a.bias = c.bias ? db : nullptr;
  a.residual = c.residual ? dres : nullptr;
  a.res_fp32 = c.res_fp32; a.out_fp32 = c.out_fp32; a.act = c.act;
  a.row_map = dmap; a.res_mod = c.res_mod;
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

static void bench_gemm(int M, int N, int K, int act, int out_fp32, int residual, int res_bf16 = 0, int iters = 20, int res_mod = 0) {
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
  a.lda = K; a.ldw = K; a.ldo = N; a.ldr = N; a.act = act; a.out_fp32 = out_fp32;
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
  printf("bench gemm M=%d N=%d K=%d act=%d outf32=%d res=%d%s: %.3f ms  %.1f TFLOP/s  %.0f GB/s\n", M, N, K,
         act, out_fp32, residual, res_bf16 ? "(bf16)" : "", ms, 2.0 * M * N * K / ms * 1e-9, bytes / ms * 1e-6);
  cudaFree(dA); cudaFree(dW); cudaFree(dO); cudaFree(db);
  if (dR) cudaFree(dR);
}

// A/B of the two standard-epilogue schedules on one bf16-output shape: 128 x 128 tiles with the epilogue on its own
// warpgroup, and 128 x 256 tiles with the epilogue in registers.  Seeded random operands; the two outputs must be
// byte-identical.  The schedules are timed alternately (rounds x iters launches each, after a warm-up) so that clock
// and co-tenant drift hits both alike.  Returns 1 if the outputs differ.
static int bench_gemm_ab(const char* name, int M, int N, int K, int act, int rounds = 5, int iters = 10) {
  std::vector<uint16_t> hA((size_t)M * K), hW((size_t)N * K);
  for (auto& x : hA) x = f2bf(frand());
  for (auto& x : hW) x = f2bf(frand() * 0.25f);
  std::vector<float> hb(N);
  for (auto& x : hb) x = frand();
  void *dA, *dW, *dO[2];
  float* db;
  const size_t osz = (size_t)M * N * 2;
  CK(cudaMalloc(&dA, hA.size() * 2));
  CK(cudaMalloc(&dW, hW.size() * 2));
  CK(cudaMalloc(&db, N * 4));
  CK(cudaMalloc(&dO[0], osz));
  CK(cudaMalloc(&dO[1], osz));
  CK(cudaMemcpy(dA, hA.data(), hA.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dW, hW.data(), hW.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(db, hb.data(), N * 4, cudaMemcpyHostToDevice));
  CK(cudaMemset(dO[0], 0xff, osz));
  CK(cudaMemset(dO[1], 0x7f, osz));
  GemmArgs a;
  a.A = dA; a.W = dW; a.bias = db; a.M = M; a.N = N; a.K = K;
  a.lda = K; a.ldw = K; a.ldo = N; a.act = act;
  for (int w = 0; w < 2; ++w) {
    a.out = dO[w];
    for (int i = 0; i < 3; ++i)
      if (gemm_bf16_v2_std(a, w == 1, 0)) { printf("[%s] launch failed: %s\n", name, last_error()); exit(3); }
  }
  CK(cudaDeviceSynchronize());
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  float ms[2] = {0.f, 0.f};
  for (int r = 0; r < rounds; ++r) {
    for (int w = 0; w < 2; ++w) {
      a.out = dO[w];
      cudaEventRecord(e0);
      for (int i = 0; i < iters; ++i) gemm_bf16_v2_std(a, w == 1, 0);
      cudaEventRecord(e1);
      CK(cudaEventSynchronize(e1));
      float t;
      cudaEventElapsedTime(&t, e0, e1);
      ms[w] += t;
    }
  }
  std::vector<uint8_t> h0(osz), h1(osz);
  CK(cudaMemcpy(h0.data(), dO[0], osz, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(h1.data(), dO[1], osz, cudaMemcpyDeviceToHost));
  size_t ndiff = 0;
  for (size_t i = 0; i < osz; i += 2) ndiff += memcmp(&h0[i], &h1[i], 2) != 0;
  const double flop = 2.0 * M * N * K;
  const double t128 = ms[0] / (rounds * iters), t256 = ms[1] / (rounds * iters);
  printf("ab gemm %-10s M=%d N=%d K=%d act=%d: 128x128 %.3f ms %.1f TFLOP/s | 128x256 %.3f ms %.1f TFLOP/s | "
         "speed-up %.3f | outputs %s (%zu of %zu differ)\n",
         name, M, N, K, act, t128, flop / t128 * 1e-9, t256, flop / t256 * 1e-9, t128 / t256,
         ndiff ? "DIFFER" : "identical", ndiff, osz / 2);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  cudaFree(dA); cudaFree(dW); cudaFree(db); cudaFree(dO[0]); cudaFree(dO[1]);
  return ndiff ? 1 : 0;
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
        //            name        M     N     K   bias act res rf32 of32 map mod
        {"tiny-f32",            128,  128,   64,  0, 0, 0, 1, 1, 0, 0},
        {"k128-f32",            256,  256,  128,  0, 0, 0, 1, 1, 0, 0},
        {"n512-f32",            384,  512,  256,  1, 0, 0, 1, 1, 0, 0},
        {"bn64",                200,   64,  192,  1, 2, 0, 1, 0, 0, 0},
        {"bn32",                200,   32,  192,  1, 2, 0, 1, 0, 0, 0},
        {"ragged-n",            300,   40,  128,  1, 0, 0, 1, 1, 0, 0},
        {"bias-gelu-bf16",     1000,  768,  768,  1, 1, 0, 1, 0, 0, 0},
        {"resid-f32",          1000,  768, 3072,  1, 0, 1, 1, 1, 0, 0},
        {"resid-bf16",          777,  256,  320,  1, 2, 1, 0, 0, 0, 0},
        {"rowmap-resid",       4000, 2304,  768,  1, 0, 1, 1, 1, 1, 0},
        {"posembed-mod",       2048,  768,  768,  1, 0, 1, 1, 1, 0, 512},
        {"multi-tile-per-cta", 40000, 256,  128,  1, 0, 0, 1, 0, 0, 0},
        {"wide-bias-gelu",    65000, 1280, 1024,  1, 1, 0, 1, 0, 0, 0},   // 128 x 256 schedule
    };
    for (const Case& c : cases) fails += run_case(c);
    if (bench) {
      // ViT-H encoder linears at 1024^2, batch 8 (default tile width): qkv over 25 padded 14 x 14 windows per image,
      // proj / lin1 / lin2 over 64 x 64 tokens per image
      bench_gemm(39200, 3840, 1280, 0, 0, 0);   // qkv: bias -> bf16
      bench_gemm(32768, 1280, 1280, 0, 1, 1);   // proj: bias + fp32 residual -> fp32
      bench_gemm(32768, 5120, 1280, 1, 0, 0);   // lin1: bias + GELU -> bf16
      bench_gemm(32768, 1280, 5120, 0, 1, 1);   // lin2: bias + fp32 residual -> fp32
      bench_gemm(32768, 768, 3072, 0, 1, 1);
      bench_gemm(8192, 8192, 8192, 0, 0, 0);
      // the bf16-output encoder linears on both schedules (ViT-H: 1280 wide, ViT-B: 768; qkv over 25 windows of
      // 14 x 14 or over 64 x 64 global tokens per image, batch 8), then qkv / lin1 at fewer tokens around the number
      // of 128 x 256 tiles and the depth K where gemm_bf16_v2 starts to take the wide schedule
      fails += bench_gemm_ab("vith-qkv", 39200, 3840, 1280, 0);
      fails += bench_gemm_ab("vith-qkv", 32768, 3840, 1280, 0);
      fails += bench_gemm_ab("vith-lin1", 32768, 5120, 1280, 1);
      fails += bench_gemm_ab("vitb-qkv", 39200, 2304, 768, 0);
      fails += bench_gemm_ab("vitb-qkv", 32768, 2304, 768, 0);
      fails += bench_gemm_ab("vitb-lin1", 32768, 3072, 768, 1);
      for (int m : {1024, 2048, 4096, 8192}) {
        fails += bench_gemm_ab("vith-qkv", m, 3840, 1280, 0);
        fails += bench_gemm_ab("vith-lin1", m, 5120, 1280, 1);
      }
      for (int k : {256, 512}) fails += bench_gemm_ab("k-sweep", 32768, 1280, k, 0);
    }
  }
  if (!strcmp(what, "gemmprof")) {
    // mask-decoder shapes (N prompts * 4096 image tokens rows)
    bench_gemm(1 << 20, 256, 128, 0, 1, 1, 1, 3);   // i2t out_proj + bf16 residual -> fp32
    bench_gemm(1 << 20, 128, 256, 0, 0, 0, 0, 3);   // k / v / q projections
    bench_gemm(1 << 20, 256, 128, 0, 0, 0, 0, 3);
    bench_gemm(1 << 20, 128, 256, 0, 0, 1, 0, 3, 4096);   // k-proj + broadcast fp32 residual (k_proj(pe))
  }
  if (!strcmp(what, "attn") || !strcmp(what, "all")) fails += selftest_attention(bench);
  printf("selftest: %d failing case(s)\n", fails);
  return fails ? 1 : 0;
}
