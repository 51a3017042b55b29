// sm_90a primitives used by every kernel in this library: mbarrier, TMA
// (cp.async.bulk.tensor), wgmma (warpgroup MMA from shared-memory descriptors) and the
// GEMM mainloop / accumulator-tile helpers built on them.
//
// Everything here is inline PTX; nothing comes from CUTLASS.  Layout conventions:
//   * operand tiles live in shared memory in the canonical 128-byte-swizzled layout
//     (what TMA writes with CU_TENSOR_MAP_SWIZZLE_128B): one "row" = 128 bytes, eight
//     rows = one 1024-byte swizzle atom, the 16-byte chunk index of a row is XOR-ed with
//     (row & 7).  Tile bases must be 1024-byte aligned.
//   * a 128-row GEMM tile is computed by two warpgroups (64 rows each, accumulators in
//     registers) and handed to the epilogue through an fp32 tile in shared memory.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rsp {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .b32 rx;\n"
      ".reg .pred px;\n"
      "elect.sync rx|px, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, px;\n"
      "}\n"
      : "=r"(pred));
  return pred;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok;
}
// Bounded wait: a protocol bug must trap (launch error) instead of hanging the GPU box.
// ~2^31 cycles (about a second) is far beyond any legitimate wait in this library.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3ff) == 0 && clock64() - t0 > (1ll << 31)) {
      printf("rsp: mbarrier timeout block %d thread %d bar 0x%x parity %u\n", (int)blockIdx.x,
             (int)threadIdx.x, bar, parity);
      __trap();
    }
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(m), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// TMA store (shared -> global, bulk async group), used by the GEMM epilogue
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(m), "r"(src),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor (sm_90 GMMA), 128-byte swizzle.
//   bits  0-13  start address >> 4
//   bits 16-29  leading-dimension byte offset >> 4
//   bits 32-45  stride-dimension byte offset >> 4
//   bits 62-63  layout type: 1 = SWIZZLE_128B
// K-major operand  (rows = M or N, 64 bf16 of K per 128-byte row):
//   SBO = 1024 (distance between 8-row groups); LBO unused (one atom along K per
//   descriptor; the K offset inside the atom is folded into the start address, +32 B per
//   k16 step).
// MN-major operand (rows = K, 64 bf16 of M/N per 128-byte row):
//   SBO = 1024 (distance between 8-row groups along K); LBO = distance between 64-wide
//   atoms along M/N; one k16 step = 16 rows = +2048 B on the start address.
__device__ __forceinline__ uint64_t make_gdesc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3ffff) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3fff) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3fff) << 32;
  d |= 1ull << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across wgmma_fence / wgmma_wait
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 in, fp32 accumulators in registers of the issuing warpgroup.
// A is K-major; TB = 1 takes B MN-major.  Register i of thread t holds row 16 (t / 32) + (t % 32) / 4 + 8 ((i / 2) % 2),
// column 8 (i / 4) + 2 (t % 4) + i % 2.
template <int N>
struct Wgmma;
template <> struct Wgmma<32> {
  template <int TB>
  __device__ __forceinline__ static void ss(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\n"
        "setp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{" 
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
        "}, %16, %17, p, 1, 1, 0, %19;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(acc), "n"(TB));
  }
};
template <> struct Wgmma<64> {
  template <int TB>
  __device__ __forceinline__ static void ss(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{" 
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, 0, %35;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(acc), "n"(TB));
  }
};
template <> struct Wgmma<128> {
  template <int TB>
  __device__ __forceinline__ static void ss(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{" 
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, 0, %67;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(acc), "n"(TB));
  }
};
template <> struct Wgmma<256> {
  template <int TB>
  __device__ __forceinline__ static void ss(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\n"
        "setp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{" 
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
        "}, %128, %129, p, 1, 1, 0, %131;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a), "l"(b), "r"(acc), "n"(TB));
  }
};

// ---------------------------------------------------------------- accumulator tile in shared memory
// A GEMM tile's fp32 accumulators leave the two consumer warpgroups through a [128][BN + 4] fp32 tile in shared memory,
// from which the epilogue reads whole row segments (thread = row; the 4-float pad keeps those 16-byte reads
// conflict-free).  acc_row(base, ld, row) is the byte address of a row, columns are 4 bytes apart.
__device__ __forceinline__ uint32_t acc_row(uint32_t base, int ld, int row) {
  return base + static_cast<uint32_t>(row * ld) * 4u;
}
// 32 consecutive fp32 of one row (addr 16-byte aligned)
__device__ __forceinline__ void acc_ld32(uint32_t addr, uint32_t (&r)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[4 * i]), "=r"(r[4 * i + 1]), "=r"(r[4 * i + 2]), "=r"(r[4 * i + 3])
                 : "r"(addr + 16 * i));
}
__device__ __forceinline__ void acc_st32(uint32_t addr, const uint32_t (&r)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr + 16 * i), "r"(r[4 * i]), "r"(r[4 * i + 1]),
                 "r"(r[4 * i + 2]), "r"(r[4 * i + 3])
                 : "memory");
}
// warpgroup wg (0 / 1) writes its 64 x BN accumulator fragment into rows [64 wg, 64 wg + 64) of the tile
template <int BN>
__device__ __forceinline__ void acc_store(const float (&d)[BN / 2], uint32_t base, int ld, int wg, int t) {
  const int row = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);
  const int col = 2 * (t & 3);
  const uint32_t a0 = acc_row(base, ld, row) + col * 4, a1 = acc_row(base, ld, row + 8) + col * 4;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a0 + 32 * j), "f"(d[4 * j]), "f"(d[4 * j + 1]) : "memory");
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a1 + 32 * j), "f"(d[4 * j + 2]), "f"(d[4 * j + 3]) : "memory");
  }
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Consumer side of the GEMM ring: warpgroup wg accumulates rows [64 wg, 64 wg + 64) of a 128 x BN tile over num_kb
// 64-deep k-blocks.  Stage s holds A (128 rows x 128 B, K-major) at base + s * stage_bytes and B at + a_bytes
// (K-major BN rows, or MN-major: BN / 64 atoms of 64 K-rows x 128 B).  Each of the warpgroup's warps arrives once on
// the stage's "empty" barrier (count 8 for two warpgroups) when its reads are done.
template <int BN, bool B_MN>
__device__ __forceinline__ void wg_mainloop(float (&d)[BN / 2], uint32_t base, int stage_bytes, int a_bytes, int stages,
                                            int num_kb, int wg, int& stage, uint32_t& phase, uint64_t* bar_full,
                                            uint64_t* bar_empty) {
  const int lane = threadIdx.x & 31;
#pragma unroll 1
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(smem_u32(&bar_full[stage]), phase);
    const uint32_t sa = base + stage * stage_bytes + wg * 8192;
    const uint32_t sb = base + stage * stage_bytes + a_bytes;
    acc_fence(d);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t adesc = make_gdesc(sa + k * 32, 16, 1024);
      const uint64_t bdesc = B_MN ? make_gdesc(sb + k * 2048, 64 * 128, 1024) : make_gdesc(sb + k * 32, 16, 1024);
      Wgmma<BN>::template ss<B_MN ? 1 : 0>(d, adesc, bdesc, (kb | k) != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(d);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&bar_empty[stage]));
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
}

// ---------------------------------------------------------------- small math helpers
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}

// GELU(erf) as x * sigmoid(x * P(x^2)): the logit of the normal CDF is an odd, smooth function; a degree-9 odd
// polynomial (minimax fit on [-9, 9], coefficients pre-multiplied by log2 e, positive beyond the fit range so the
// tails saturate to 0 / x) gives |error| <= 3.6e-6 absolute against 0.5 x (1 + erf(x / sqrt 2)) evaluated in fp32 -
// three orders below the bf16 resolution of the values it produces.  10 instructions (2 MUFU) instead of the ~17
// of an erf built from Abramowitz-Stegun 7.1.26 or the ~30 of libdevice erff: the GELU epilogues are
// instruction-issue bound.
__device__ __forceinline__ float gelu_fast(float x) {
  const float x2 = x * x;
  float p = fmaf(3.229002131292087e-06f, x2, -8.823835998556129e-05f);
  p = fmaf(p, x2, -0.0003602734064506858f);
  p = fmaf(p, x2, 0.10522668605353103f);
  p = fmaf(p, x2, 2.302045390974673f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-p * x));
  return __fdividef(x, 1.0f + e);
}

}  // namespace rsp
