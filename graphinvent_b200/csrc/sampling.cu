// The sampling policy of the generators: temperature, top-k and nucleus (top-p) sampling on the device
// (include/gib200.h: gib_sampling_policy, gib_sample_actions_policy, gib_*_sample_round_policy).
//
// One CTA of 256 threads per row, as sample_actions_kernel (api.cu).  The row is staged in shared memory when it fits
// (apd <= kStageMax = 11264 floats, 44 KiB: with the 3.2 KiB of static shared memory inside the 48 KiB a launch may
// use without opting in); longer rows are read from global memory, where the up to 11 passes below hit L2.  The same
// code serves both: only the row pointer differs.
//
//  1. the row maximum m and the model's softmax denominator, by the reduction and the fixed-order chunk prefix of
//     sample_actions_kernel: the recorded likelihood is the model's probability, bit for bit gib_sample_actions' value;
//  2. the kept set, a prefix of the ranking (o descending, ties to the lower index).  Its boundary is a (key, count)
//     pair: every finite entry whose order key exceeds `key`, and the first `count` entries in index order whose key
//     equals it (tied entries have equal weights).  It is found by MSB radix select over the 32-bit order keys of o
//     (4 passes of 8 bits, 256-bin shared histograms), not by sorting:
//       top-k  counts (one per finite entry) until k;
//       top-p  weight mass of the entries top-k kept, until ceil(top_p * their total).  The masses are fixed point
//              (w * 2^(62 - ceil(log2 apd)), truncated), so the histogram atomics are exact integer sums and the
//              selection does not depend on their order;
//  3. the draw: inverse CDF over the kept weights (fp32) in index order with sample_actions_kernel's chunk prefix and
//     owner rule.  With the policy off the kept set is every finite entry and its weights are the model's, so the
//     draw is gib_sample_actions' draw.
// Every reduction runs in a fixed order or on integers: the same logits and uniforms give the same outputs on every
// launch and replay.
#include "../../include/gib200.h"
#include "common.cuh"
#include "ops.cuh"

namespace gib {
namespace {

constexpr int kThreads = 256;
constexpr int kStageMax = 11264;       // floats of a row staged in shared memory (44 KiB)

// larger key = larger value; -0 and +0 share one key (they tie in the ranking)
__device__ __forceinline__ unsigned order_key(float x) {
  const unsigned u = __float_as_uint(x + 0.f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct Policy {
  float t;                              // temperature; 0 = greedy
  int k;                                // top-k (0: off)
  float p;                              // top-p (1: off)
  __device__ bool valid() const { return t >= 0.f && t < INFINITY && k >= 0 && p > 0.f && p <= 1.f; }
  __device__ float weight(float x, float m) const { return t > 0.f ? expf((x - m) / t) : 1.f; }
};

struct Smem {
  float pre[kThreads + 1];
  float red[kThreads / 32];
  unsigned long long hist[256];
  unsigned long long total;
  int wsum[kThreads / 32];
  int count;
  unsigned sel_key;
  unsigned long long sel_above;
};

// the largest order key t such that the contributions of the finite entries with key >= t reach `need` (sum over the
// entries with key > t: `above`).  contrib(x, key) is the contribution of one entry; `extra` is added for the key
// `extra_key` (the top-k ties, which the top-p pass counts as one group).  need <= the total is the caller's rule.
template <class Contrib>
__device__ void radix_select(const float* o, int apd, unsigned long long need, Contrib contrib, unsigned extra_key,
                             unsigned long long extra, Smem& s, unsigned& key, unsigned long long& above) {
  unsigned prefix = 0, mask = 0;
  unsigned long long done = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    s.hist[threadIdx.x] = 0;
    __syncthreads();
    for (int k = threadIdx.x; k < apd; k += kThreads) {
      const float x = o[k];
      if (!isfinite(x)) continue;
      const unsigned kk = order_key(x);
      if ((kk & mask) != prefix) continue;
      const unsigned long long c = contrib(x, kk);
      if (c) atomicAdd(&s.hist[(kk >> shift) & 255u], c);
    }
    if (threadIdx.x == 0 && extra && (extra_key & mask) == prefix) atomicAdd(&s.hist[(extra_key >> shift) & 255u], extra);
    __syncthreads();
    if (threadIdx.x < 32) {             // warp 0: bins from the top, 8 per lane, integer scan
      const int lane = threadIdx.x;
      unsigned long long v = 0;
      for (int i = 0; i < 8; ++i) v += s.hist[255 - 8 * lane - i];
      unsigned long long incl = v;
      for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
      }
      const unsigned long long rem = need - done;
      const unsigned hit = __ballot_sync(0xffffffffu, incl >= rem);
      const int owner = hit ? __ffs(hit) - 1 : 31;
      if (lane == owner) {
        unsigned long long run = incl - v;
        int bin = 255 - 8 * lane;
        for (int i = 0; i < 8; ++i) {
          bin = 255 - 8 * lane - i;
          if (run + s.hist[bin] >= rem) break;
          if (i < 7) run += s.hist[bin];
        }
        s.sel_key = (unsigned)bin;
        s.sel_above = done + run;
      }
    }
    __syncthreads();
    prefix |= s.sel_key << shift;
    mask |= 255u << shift;
    done = s.sel_above;
    __syncthreads();
  }
  key = prefix;
  above = done;
}

// exclusive prefix of one int per thread over the CTA, in thread order (integers: exact)
__device__ __forceinline__ int block_excl_scan(int v, Smem& s) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = v;
  for (int d = 1; d < 32; d <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) s.wsum[wid] = incl;
  __syncthreads();
  int base = 0;
  for (int w = 0; w < wid; ++w) base += s.wsum[w];
  __syncthreads();
  return base + incl - v;
}

__global__ void __launch_bounds__(kThreads) policy_sample_kernel(const float* __restrict__ out, int apd,
                                                                 const float* __restrict__ uniforms,
                                                                 const gib_sampling_policy* __restrict__ policy,
                                                                 int* __restrict__ action, float* __restrict__ lik,
                                                                 float* __restrict__ q_out, RoundGate g) {
  extern __shared__ float staged[];
  __shared__ Smem s;
  const int b = blockIdx.x;
  if (g.state) {
    const int r = gate_round(g), B = gridDim.x;
    if (r < 0) return;
    uniforms += (size_t)r * B;
  }
  const float* o = out + (size_t)b * apd;
  if (apd <= kStageMax) {
    for (int k = threadIdx.x; k < apd; k += kThreads) staged[k] = o[k];
    o = staged;                         // made visible by the reduction's barriers below
  }
  const Policy P{policy->temperature, policy->top_k, policy->top_p};

  // 1. m and the model's denominator: sample_actions_kernel's reduction and chunk prefix
  float mx = -INFINITY;
  for (int k = threadIdx.x; k < apd; k += kThreads) mx = fmaxf(mx, o[k]);
  mx = block_reduce<kThreads>(mx, s.red, true);
  const int L = ceil_div(apd, kThreads);
  const int lo = min(apd, (int)threadIdx.x * L), hi = min(apd, lo + L);
  float sum = 0.f;
  int finite = 0;
  for (int k = lo; k < hi; ++k) {
    sum += expf(o[k] - mx);
    finite += isfinite(o[k]) ? 1 : 0;
  }
  s.pre[threadIdx.x + 1] = sum;
  if (threadIdx.x == 0) { s.pre[0] = 0.f; s.count = 0; s.total = 0; }
  __syncthreads();
  atomicAdd(&s.count, finite);
  if (threadIdx.x == 0)
    for (int i = 1; i <= kThreads; ++i) s.pre[i] += s.pre[i - 1];
  __syncthreads();
  const float model_total = s.pre[kThreads];
  const int nf = s.count;
  const float u = uniforms[b];
  // a row without a finite entry, with NaN / +inf, a NaN uniform or an invalid policy: gib_sample_actions' outputs
  if (!(model_total == model_total && model_total > 0.f && model_total < INFINITY && u == u && P.valid())) {
    if (threadIdx.x == 0) {
      action[b] = apd - 1;
      lik[b] = NAN;
      if (q_out) q_out[b] = NAN;
    }
    return;
  }
  __syncthreads();                      // every thread has read pre[] before it is reused

  // 2. the kept set: finite entries with key > cut_key, and the first cut_n (index order) with key == cut_key
  const int k_eff = P.t > 0.f ? P.k : 1;                  // greedy = the first entry of the ranking
  unsigned cut_key = 0;                                   // below every finite key: every finite entry is kept
  long long cut_n = 0;
  if (k_eff > 0 && k_eff < nf) {
    unsigned long long above;
    radix_select(o, apd, (unsigned long long)k_eff, [](float, unsigned) { return 1ull; }, 0u, 0ull, s, cut_key,
                 above);
    cut_n = k_eff - (long long)above;
  }
  if (P.t > 0.f && P.p < 1.f) {
    const int lg = apd > 1 ? 32 - __clz(apd - 1) : 0;    // ceil(log2 apd): the fixed-point total stays below 2^62
    const double scale = ldexp(1.0, 62 - lg);
    const float tie_w = cut_key ? P.weight(key_value(cut_key), mx) : 0.f;
    const unsigned long long tie_mass = (unsigned long long)(tie_w * scale) * (unsigned long long)cut_n;
    auto mass = [&](float x, unsigned kk) -> unsigned long long {
      return kk > cut_key ? (unsigned long long)(P.weight(x, mx) * scale) : 0ull;
    };
    unsigned long long part = 0;
    for (int k = threadIdx.x; k < apd; k += kThreads)
      if (isfinite(o[k])) part += mass(o[k], order_key(o[k]));
    atomicAdd(&s.total, part);
    __syncthreads();
    const unsigned long long total = s.total + tie_mass;
    unsigned long long need = (unsigned long long)ceil((double)P.p * (double)total);
    need = min(max(need, 1ull), total);
    unsigned key;
    unsigned long long above;
    radix_select(o, apd, need, mass, cut_key, tie_mass, s, key, above);
    // the entries tied at `key` share one weight > 0 (the cumulative mass reached `need` there)
    const unsigned long long w_key = (unsigned long long)(P.weight(key_value(key), mx) * scale);
    cut_n = w_key ? (long long)((need - above + w_key - 1) / w_key) : 1;
    cut_key = key;
  }

  // 3. the draw over the kept weights in index order: tie ranks by an exact scan, weights by the fixed-order prefix
  int ties = 0;
  for (int k = lo; k < hi; ++k)
    if (isfinite(o[k]) && order_key(o[k]) == cut_key) ++ties;
  const long long tie0 = block_excl_scan(ties, s);
  auto kept_weight = [&](int k, long long& rank) -> float {
    const float x = o[k];
    if (!isfinite(x)) return 0.f;
    const unsigned kk = order_key(x);
    bool keep = kk > cut_key;
    if (kk == cut_key) keep = rank++ < cut_n;
    return keep ? P.weight(x, mx) : 0.f;
  };
  float wsum = 0.f;
  long long rank = tie0;
  for (int k = lo; k < hi; ++k) wsum += kept_weight(k, rank);
  s.pre[threadIdx.x + 1] = wsum;
  if (threadIdx.x == 0) s.pre[0] = 0.f;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int i = 1; i <= kThreads; ++i) s.pre[i] += s.pre[i - 1];
  __syncthreads();
  const float total = s.pre[kThreads];
  float target = u * total;
  if (target >= total) target = nextafterf(total, 0.f);
  // the owner chunk (its bracket holds the target, so it holds an entry of weight > 0); the running sum can end a few
  // ulps short of pre[t + 1]: then the chunk's last entry of non-zero weight, as in sample_actions_kernel
  if (s.pre[threadIdx.x] <= target && target < s.pre[threadIdx.x + 1] && hi > lo) {
    float run = s.pre[threadIdx.x];
    int pick = -1, last = lo;
    float w_pick = 0.f, w_last = 0.f;
    rank = tie0;
    for (int k = lo; k < hi; ++k) {
      const float w = kept_weight(k, rank);
      run += w;
      if (w > 0.f) { last = k; w_last = w; }
      if (target < run) { pick = k; w_pick = w; break; }
    }
    if (pick < 0) { pick = last; w_pick = w_last; }
    action[b] = pick;
    lik[b] = expf(o[pick] - mx) / model_total;
    if (q_out) q_out[b] = w_pick / total;
  }
}

}  // namespace

int policy_sample_launch(const float* out, int B, int apd, const float* uniforms, const gib_sampling_policy* policy,
                         int* action, float* lik, float* q, const RoundGate* gate, cudaStream_t st) {
  if (B <= 0) return 0;
  const size_t smem = apd <= kStageMax ? (size_t)apd * sizeof(float) : 0;
  policy_sample_kernel<<<B, kThreads, smem, st>>>(out, apd, uniforms, policy, action, lik, q,
                                                  gate ? *gate : RoundGate{});
  GIB_LAUNCH_CHECK();
  return 0;
}

}  // namespace gib

using namespace gib;

extern "C" int gib_sampling_policy_set(gib_sampling_policy* policy, float temperature, int top_k, float top_p,
                                       gib_stream stream) {
  if (!policy || !(temperature >= 0.f && temperature < INFINITY) || top_k < 0 || !(top_p > 0.f && top_p <= 1.f)) {
    set_error("gib_sampling_policy_set: refused (policy %s, temperature=%g must be finite and >= 0, top_k=%d must be "
              ">= 0, top_p=%g must lie in (0, 1])", policy ? "given" : "null", temperature, top_k, top_p);
    return -1;
  }
  const gib_sampling_policy v{temperature, top_k, top_p, 0};
  // pageable source: the call returns once the value is staged, so the stack copy may go out of scope
  GIB_CUDA_TRY(cudaMemcpyAsync(policy, &v, sizeof(v), cudaMemcpyHostToDevice, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

extern "C" int gib_sample_actions_policy(const float* out, int B, int apd, const float* uniforms,
                                         const gib_sampling_policy* policy, int* action, float* likelihood, float* q,
                                         gib_stream stream) {
  if (B < 0 || apd < 1 || !out || !uniforms || !action || !likelihood || (!policy && q)) {
    set_error("gib_sample_actions_policy: bad arguments (B=%d apd=%d; logits, uniforms, action and likelihood must be "
              "given, and q needs a policy)", B, apd);
    return -1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!policy) return sample_actions_launch(out, B, apd, uniforms, action, likelihood, nullptr, st);
  return policy_sample_launch(out, B, apd, uniforms, policy, action, likelihood, q, nullptr, st);
}
