// Flat-bucket Adam step (SURVEY.md 8f rank 2): one launch over the contiguous parameter / gradient /
// moment buffers, replacing the per-tensor update of torch.optim.Adam at Workflow.py:191,221,245
// (stepped at Workflow.py:795-796).  HBM-bound: 4 streams read, 3 written, 28 B per parameter.
#include <math.h>

#include "../../include/gib200.h"
#include "common.cuh"
#include "gemm.cuh"

namespace gib {

struct AdamScalars {
  float beta1, beta2, one_minus_beta1, one_minus_beta2, eps, weight_decay;
  float step_size;      // lr / (1 - beta1^t)
  float bc2_sqrt;       // sqrt(1 - beta2^t)
  float grad_scale;     // applied to the gradient first (1 / world size when the bucket holds an all-reduce SUM)
};

// same operation order as torch/optim/adam.py::_single_tensor_adam (non-amsgrad, L2 weight decay):
//   g += wd * p;  m += (g - m) * (1 - b1);  v = v * b2 + (1 - b2) * g * g;
//   p -= step_size * m / (sqrt(v) / sqrt(bc2) + eps)
__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, const AdamScalars& s) {
  g *= s.grad_scale;
  g = fmaf(s.weight_decay, p, g);
  m = fmaf(g - m, s.one_minus_beta1, m);
  v = fmaf(s.one_minus_beta2 * g, g, v * s.beta2);
  const float denom = sqrtf(v) / s.bc2_sqrt + s.eps;
  p = fmaf(-s.step_size, m / denom, p);
}

__global__ void __launch_bounds__(256, 6) adam_flat_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                        float* __restrict__ m, float* __restrict__ v, long long n,
                                                        long long head, AdamScalars s) {
  // [0, head) scalar prologue up to 16-byte alignment, then float4 body, then scalar tail
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  const long long nvec = (n - head) >> 2;
  float4* p4 = reinterpret_cast<float4*>(p + head);
  const float4* g4 = reinterpret_cast<const float4*>(g + head);
  float4* m4 = reinterpret_cast<float4*>(m + head);
  float4* v4 = reinterpret_cast<float4*>(v + head);
  for (long long i = tid; i < nvec; i += nthreads) {
    float4 pp = p4[i], mm = m4[i], vv = v4[i];
    const float4 gg = __ldg(g4 + i);
    adam_one(pp.x, gg.x, mm.x, vv.x, s);
    adam_one(pp.y, gg.y, mm.y, vv.y, s);
    adam_one(pp.z, gg.z, mm.z, vv.z, s);
    adam_one(pp.w, gg.w, mm.w, vv.w, s);
    p4[i] = pp; m4[i] = mm; v4[i] = vv;
  }
  const long long tail0 = head + (nvec << 2);
  const long long nscalar = head + (n - tail0);
  for (long long i = tid; i < nscalar; i += nthreads) {
    const long long j = i < head ? i : tail0 + (i - head);
    float pp = p[j], mm = m[j], vv = v[j];
    adam_one(pp, g[j], mm, vv, s);
    p[j] = pp; m[j] = mm; v[j] = vv;
  }
}

}  // namespace gib

extern "C" int gib_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                             long long step, double lr, double beta1, double beta2, double eps,
                             double weight_decay, double grad_scale, gib_stream stream) {
  using namespace gib;
  if (n < 0 || step < 1) { set_error("gib_adam_step: n >= 0 and step >= 1 required (n=%lld step=%lld)", n, step); return -2; }
  if (n == 0) return 0;
  if (!params || !grads || !exp_avg || !exp_avg_sq) { set_error("gib_adam_step: null buffer"); return -2; }
  const uintptr_t a = reinterpret_cast<uintptr_t>(params);
  if ((a & 3) || ((reinterpret_cast<uintptr_t>(grads) ^ a) & 15) || ((reinterpret_cast<uintptr_t>(exp_avg) ^ a) & 15) ||
      ((reinterpret_cast<uintptr_t>(exp_avg_sq) ^ a) & 15)) {
    set_error("gib_adam_step: the four buffers must share their alignment modulo 16 bytes");
    return -2;
  }
  AdamScalars s;
  // bias corrections in double on the host, as the reference optimizer computes them in Python floats
  const double bc1 = 1.0 - pow(beta1, (double)step);
  const double bc2 = 1.0 - pow(beta2, (double)step);
  s.beta1 = (float)beta1; s.beta2 = (float)beta2;
  s.one_minus_beta1 = (float)(1.0 - beta1);
  s.one_minus_beta2 = (float)(1.0 - beta2);
  s.eps = (float)eps; s.weight_decay = (float)weight_decay;
  s.step_size = (float)(lr / bc1);
  s.bc2_sqrt = (float)sqrt(bc2);
  s.grad_scale = (float)grad_scale;
  long long head = ((16 - (a & 15)) & 15) >> 2;
  if (head > n) head = n;
  const long long work = (n + 3) / 4;
  long long blocks = (work + 255) / 256;
  const long long cap = (long long)gib::device_sm_count() * 6;   // one wave: 6 resident CTAs of 256 threads per SM (40 registers)
  if (blocks > cap) blocks = cap;
  adam_flat_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(params, grads, exp_avg,
                                                                                         exp_avg_sq, n, head, s);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ---- dynamic loss scaling on the device (torch.amp.GradScaler's step / update without a host round trip) ----------
namespace gib {

__device__ __forceinline__ bool nonfinite(float x) { return (__float_as_uint(x) & 0x7f800000u) == 0x7f800000u; }

// found_inf = 1 if any of x[0, n) is inf or NaN; never cleared here.  Same split as adam_flat_kernel.
__global__ void __launch_bounds__(256) nonfinite_check_kernel(const float* __restrict__ x, long long n, long long head,
                                                              float* __restrict__ found_inf) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  const long long nvec = (n - head) >> 2;
  const float4* x4 = reinterpret_cast<const float4*>(x + head);
  bool bad = false;
  for (long long i = tid; i < nvec; i += nthreads) {
    const float4 v = __ldg(x4 + i);
    bad |= nonfinite(v.x) | nonfinite(v.y) | nonfinite(v.z) | nonfinite(v.w);
  }
  const long long tail0 = head + (nvec << 2);
  const long long nscalar = head + (n - tail0);
  for (long long i = tid; i < nscalar; i += nthreads) bad |= nonfinite(x[i < head ? i : tail0 + (i - head)]);
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) *found_inf = 1.f;
}

// adam_flat_kernel behind the scaler: nothing is written when *found_inf is set; otherwise every gradient is first
// multiplied by inv_scale = (float)(1 / (double)*scale) (GradScaler.unscale_), and the bias corrections come from the
// device count (*step_count + 1), in double as gib_adam_step computes them on the host.  The count itself is advanced
// by gib_amp_update_scale, a later launch, so no CTA of this one can see it change.
__global__ void __launch_bounds__(256, 6) adam_scaled_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                          float* __restrict__ m, float* __restrict__ v, long long n,
                                                          long long head, const long long* __restrict__ step_count,
                                                          const float* __restrict__ found_inf,
                                                          const float* __restrict__ scale, double lr, double beta1,
                                                          double beta2, double eps, double weight_decay,
                                                          double grad_scale) {
  __shared__ AdamScalars ss;
  __shared__ float inv_s;
  if (*found_inf != 0.f) return;
  if (threadIdx.x == 0) {
    const double t = (double)(*step_count + 1);
    const double bc1 = 1.0 - pow(beta1, t);
    const double bc2 = 1.0 - pow(beta2, t);
    AdamScalars s;
    s.beta1 = (float)beta1; s.beta2 = (float)beta2;
    s.one_minus_beta1 = (float)(1.0 - beta1);
    s.one_minus_beta2 = (float)(1.0 - beta2);
    s.eps = (float)eps; s.weight_decay = (float)weight_decay;
    s.step_size = (float)(lr / bc1);
    s.bc2_sqrt = (float)sqrt(bc2);
    s.grad_scale = (float)grad_scale;
    ss = s;
    inv_s = (float)(1.0 / (double)*scale);
  }
  __syncthreads();
  const AdamScalars s = ss;
  const float inv = inv_s;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  const long long nvec = (n - head) >> 2;
  float4* p4 = reinterpret_cast<float4*>(p + head);
  const float4* g4 = reinterpret_cast<const float4*>(g + head);
  float4* m4 = reinterpret_cast<float4*>(m + head);
  float4* v4 = reinterpret_cast<float4*>(v + head);
  for (long long i = tid; i < nvec; i += nthreads) {
    float4 pp = p4[i], mm = m4[i], vv = v4[i];
    const float4 gg = __ldg(g4 + i);
    adam_one(pp.x, gg.x * inv, mm.x, vv.x, s);
    adam_one(pp.y, gg.y * inv, mm.y, vv.y, s);
    adam_one(pp.z, gg.z * inv, mm.z, vv.z, s);
    adam_one(pp.w, gg.w * inv, mm.w, vv.w, s);
    p4[i] = pp; m4[i] = mm; v4[i] = vv;
  }
  const long long tail0 = head + (nvec << 2);
  const long long nscalar = head + (n - tail0);
  for (long long i = tid; i < nscalar; i += nthreads) {
    const long long j = i < head ? i : tail0 + (i - head);
    float pp = p[j], mm = m[j], vv = v[j];
    adam_one(pp, g[j] * inv, mm, vv, s);
    p[j] = pp; m[j] = mm; v[j] = vv;
  }
}

// torch._amp_update_scale_ (one thread), and the step counts of the optimizer that was gated on the same found_inf
__global__ void amp_update_scale_kernel(float* scale, int* growth_tracker, const float* found_inf,
                                        double growth_factor, double backoff_factor, int growth_interval,
                                        long long* step_counts, int n_counts) {
  const bool skipped = *found_inf != 0.f;
  if (!skipped)
    for (int i = threadIdx.x; i < n_counts; i += blockDim.x) step_counts[i] += 1;
  if (threadIdx.x != 0) return;
  if (skipped) {
    *scale = (float)((double)*scale * backoff_factor);
    *growth_tracker = 0;
  } else {
    const int successful = *growth_tracker + 1;
    if (successful == growth_interval) {
      const float grown = (float)((double)*scale * growth_factor);
      if (!nonfinite(grown)) *scale = grown;
      *growth_tracker = 0;
    } else {
      *growth_tracker = successful;
    }
  }
}

static long long grid_for(long long n, int per_sm) {
  long long blocks = ((n + 3) / 4 + 255) / 256;
  const long long cap = (long long)device_sm_count() * per_sm;
  if (blocks > cap) blocks = cap;
  return blocks < 1 ? 1 : blocks;
}

}  // namespace gib

extern "C" int gib_nonfinite_check(const float* x, long long n, float* found_inf, gib_stream stream) {
  using namespace gib;
  if (n < 0) { set_error("gib_nonfinite_check: n >= 0 required (n=%lld)", n); return -2; }
  if (!found_inf || (n > 0 && !x)) { set_error("gib_nonfinite_check: null buffer"); return -2; }
  if ((reinterpret_cast<uintptr_t>(x) & 3)) { set_error("gib_nonfinite_check: x must be 4-byte aligned"); return -2; }
  if (n == 0) return 0;
  long long head = ((16 - (reinterpret_cast<uintptr_t>(x) & 15)) & 15) >> 2;
  if (head > n) head = n;
  nonfinite_check_kernel<<<(unsigned)grid_for(n, 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, n, head,
                                                                                                       found_inf);
  GIB_LAUNCH_CHECK();
  return 0;
}

extern "C" int gib_adam_step_scaled(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                                    const long long* step_count, const float* found_inf, const float* scale,
                                    double lr, double beta1, double beta2, double eps, double weight_decay,
                                    double grad_scale, gib_stream stream) {
  using namespace gib;
  if (n < 0) { set_error("gib_adam_step_scaled: n >= 0 required (n=%lld)", n); return -2; }
  if (!step_count || !found_inf || !scale) { set_error("gib_adam_step_scaled: null device scalar"); return -2; }
  if (n == 0) return 0;
  if (!params || !grads || !exp_avg || !exp_avg_sq) { set_error("gib_adam_step_scaled: null buffer"); return -2; }
  const uintptr_t a = reinterpret_cast<uintptr_t>(params);
  if ((a & 3) || ((reinterpret_cast<uintptr_t>(grads) ^ a) & 15) || ((reinterpret_cast<uintptr_t>(exp_avg) ^ a) & 15) ||
      ((reinterpret_cast<uintptr_t>(exp_avg_sq) ^ a) & 15)) {
    set_error("gib_adam_step_scaled: the four buffers must share their alignment modulo 16 bytes");
    return -2;
  }
  long long head = ((16 - (a & 15)) & 15) >> 2;
  if (head > n) head = n;
  adam_scaled_kernel<<<(unsigned)grid_for(n, 6), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      params, grads, exp_avg, exp_avg_sq, n, head, step_count, found_inf, scale, lr, beta1, beta2, eps, weight_decay,
      grad_scale);
  GIB_LAUNCH_CHECK();
  return 0;
}

extern "C" int gib_amp_update_scale(float* scale, int* growth_tracker, const float* found_inf, double growth_factor,
                                    double backoff_factor, int growth_interval, long long* step_counts, int n_counts,
                                    gib_stream stream) {
  using namespace gib;
  if (!scale || !growth_tracker || !found_inf || (n_counts > 0 && !step_counts)) {
    set_error("gib_amp_update_scale: null device scalar");
    return -2;
  }
  if (n_counts < 0 || growth_interval < 1) {
    set_error("gib_amp_update_scale: n_counts >= 0 and growth_interval >= 1 required (n_counts=%d interval=%d)",
              n_counts, growth_interval);
    return -2;
  }
  amp_update_scale_kernel<<<1, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      scale, growth_tracker, found_inf, growth_factor, backoff_factor, growth_interval, step_counts, n_counts);
  GIB_LAUNCH_CHECK();
  return 0;
}
