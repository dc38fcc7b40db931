// PTX wrappers of the tensor-core GEMM kernels (gemm_tc3.cu): mbarrier, TMA, wgmma and the fast epilogue activation.
// sm_90a.
#pragma once
#include <cuda.h>
#include <stdint.h>

#include "common.cuh"

namespace gib {
namespace tcptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded wait: ~10 s of wall clock, then trap (surfaces as a CUDA error instead of hanging the box)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > 20000000000LL) __trap();   // ~10 s: a dead-lock, not contention
}

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      :
      : "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ---- warpgroup MMA (wgmma) ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// shared-memory descriptor of a K-major operand tile that TMA wrote with the 128-byte swizzle (rows of 32 fp32,
// 1024-byte aligned tile base): 8-row groups 1024 B apart (stride byte offset); the leading byte offset is unused
// because the k extent of one instruction (8 tf32 = 32 B) stays inside a 128-byte row.  The k-step within the row is
// selected by advancing the start address in 32-byte steps: the hardware applies the swizzle to the full address.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// d[64] += A[64 x 8] * B[8 x 128], tf32 in, fp32 accumulate.  A from registers: this thread's fragment a[4] in the
// m16n8k8 layout of its warp's 16 rows (rows g, g+8 x cols t, t+4); B from shared memory through `desc`.
// d: per warp 16 rows x 128 columns, the m16n8 C-fragment layout repeated over 16 column blocks of 8.
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float* d, const uint32_t* a, uint64_t desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
      "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "n"(1));
}

// ---- 16-bit operands (H16 = 1: bf16, 2: fp16) ----
// shared-memory descriptor of a K-major tile of 16-bit values that TMA wrote with the 64-byte swizzle (rows of 32
// values = 64 B, 512-byte aligned tile base): 8-row groups 512 B apart; one instruction's k extent (16 values = 32 B)
// stays inside a row, and the second k16 step of a row is selected by advancing the start address by 32 B.
__device__ __forceinline__ uint64_t wgmma_desc_sw64(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(512 >> 4) << 32) | ((uint64_t)2 << 62);
}

// two fp32 values rounded to nearest-even into one register of 16-bit values, `lo` in the low half (the lower column
// of an MMA fragment pair) -- the rounding of torch's tensor.to(torch.bfloat16 / torch.float16); an fp16 value beyond
// +-65504 becomes +-inf as there
template <int H16>
__device__ __forceinline__ uint32_t pack16(float lo, float hi) {
  uint32_t r;
  if constexpr (H16 == 1) asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

#define GIB_WGMMA_D64                                                                                                 \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),         \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),          \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),         \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),         \
      "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),         \
      "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),         \
      "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),         \
      "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define GIB_WGMMA_K16(TYPE)                                                                                          \
  "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"                                                                  \
  "wgmma.mma_async.sync.aligned.m64n128k16.f32." TYPE "." TYPE " "                                                    \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "  \
  "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "    \
  "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "                      \
  "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"

// d[64] += A[64 x 16] * B[16 x 128], bf16 / fp16 in, fp32 accumulate.  A from registers: this thread's fragment a[4]
// in the m16n8k16 layout of its warp's 16 rows (a[0] row g, a[1] row g+8 at columns 2t, 2t+1; a[2], a[3] the same
// rows at columns 2t+8, 2t+9; lower column in the low half); B K-major from shared memory through `desc`.
template <int H16>
__device__ __forceinline__ void wgmma_m64n128k16_h16(float* d, const uint32_t* a, uint64_t desc) {
  if constexpr (H16 == 1)
    asm volatile(GIB_WGMMA_K16("bf16") : GIB_WGMMA_D64 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "n"(1));
  else
    asm volatile(GIB_WGMMA_K16("f16") : GIB_WGMMA_D64 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "n"(1));
}
#undef GIB_WGMMA_K16
#undef GIB_WGMMA_D64

// epilogue activation: SELU through the hardware exp2 path (MUFU), |abs err| <~ 2e-7, instead of expm1f's
// ~30-instruction software path.  Branch-free: ex2.approx.ftz of a large positive argument is +inf: not selected.
__device__ __forceinline__ float selu_fast(float x) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * 1.4426950408889634f));
  const float neg = fmaf(e, GIB_SELU_SCALE * GIB_SELU_ALPHA, -(GIB_SELU_SCALE * GIB_SELU_ALPHA));
  const float pos = GIB_SELU_SCALE * x;
  return x > 0.f ? pos : neg;
}
__device__ __forceinline__ float act_fast(float x, int act) {
  if (act == ACT_SELU) return selu_fast(x);
  if (act == ACT_TANH) return tanhf(x);
  return x;
}

}  // namespace tcptx
}  // namespace gib
