// Shared helpers for the GraphINVENT hot-path kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace gib {

constexpr int kTileRows = 128;  // row granularity of a bond-type segment (GEMM M tile)

__host__ __device__ inline int pad16(int x) { return (x + 15) & ~15; }
__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

// SELU constants (torch.nn.SELU; reference gnn/modules.py:127, SURVEY Appendix D)
#define GIB_SELU_SCALE 1.0507009873554804934193349852946f
#define GIB_SELU_ALPHA 1.6732632423543772848170429916717f

enum Act : int { ACT_NONE = 0, ACT_SELU = 1, ACT_TANH = 2 };

__device__ __forceinline__ float selu_f(float x) {
  return x > 0.f ? GIB_SELU_SCALE * x : (GIB_SELU_SCALE * GIB_SELU_ALPHA) * expm1f(x);
}
// derivative of SELU expressed through its OUTPUT y (y > 0 <=> x > 0)
__device__ __forceinline__ float dselu_from_out(float y) {
  return y > 0.f ? GIB_SELU_SCALE : y + GIB_SELU_SCALE * GIB_SELU_ALPHA;
}
__device__ __forceinline__ float act_f(float x, int act) {
  if (act == ACT_SELU) return selu_f(x);
  if (act == ACT_TANH) return tanhf(x);
  return x;
}
__device__ __forceinline__ float dact_from_out(float y, int act) {
  if (act == ACT_SELU) return dselu_from_out(y);
  if (act == ACT_TANH) return 1.f - y * y;
  return 1.f;
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

// CTA-wide max / sum of one float per thread (NT threads, sm >= NT / 32 floats of shared memory); every thread
// gets the result.  Fixed order: deterministic.
template <int NT>
__device__ __forceinline__ float block_reduce(float v, float* sm, bool is_max) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float t = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, t) : v + t;
  }
  __syncthreads();
  if (lane == 0) sm[wid] = v;
  __syncthreads();
  float r = sm[0];
  for (int i = 1; i < NT / 32; ++i) r = is_max ? fmaxf(r, sm[i]) : r + sm[i];
  return r;
}

// Unaligned int8 rows through aligned 16-byte loads (the loader's gather and the route fill): every aligned word
// load_span reads holds at least one byte of the span, so no load leaves a 16-byte aligned allocation.
typedef unsigned __int128 u128;

__device__ __forceinline__ u128 ld16(const uint8_t* p) {
  const uint4 w = __ldg(reinterpret_cast<const uint4*>(p));
  return (u128)w.x | ((u128)w.y << 32) | ((u128)w.z << 64) | ((u128)w.w << 96);
}

// bytes p[0, len) in the low bytes of the result, 1 <= len <= 16; the bytes above len are unspecified
__device__ __forceinline__ u128 load_span(const uint8_t* p, int len) {
  const int off = (int)(reinterpret_cast<uintptr_t>(p) & 15);
  const uint8_t* a = p - off;
  const u128 lo = ld16(a);
  if (off == 0) return lo;
  const u128 hi = off + len > 16 ? ld16(a + 16) : (u128)0;
  return (lo >> (8 * off)) | (hi << (128 - 8 * off));
}

__device__ __forceinline__ void st16(void* p, u128 v) {
  *reinterpret_cast<uint4*>(p) = make_uint4((unsigned)v, (unsigned)(v >> 32), (unsigned)(v >> 64), (unsigned)(v >> 96));
}

// error plumbing: kernels are launched through GIB_LAUNCH_CHECK so that a bad launch
// configuration is reported at the C-ABI boundary as a cudaError_t (>0).
#define GIB_CUDA_TRY(expr)                                   \
  do {                                                       \
    cudaError_t _e = (expr);                                 \
    if (_e != cudaSuccess) return (int)_e;                   \
  } while (0)
extern long long g_launch_count;  // kernels launched by this library (bench.py reports it)
#define GIB_LAUNCH_CHECK()                 \
  do {                                     \
    ++::gib::g_launch_count;               \
    GIB_CUDA_TRY(cudaGetLastError());      \
  } while (0)
#define GIB_TRY(expr)                                        \
  do {                                                       \
    int _r = (expr);                                         \
    if (_r != 0) return _r;                                  \
  } while (0)

void set_error(const char* fmt, ...);

}  // namespace gib
