// The RL rollout of GraphGeneratorRL (GraphGeneratorRL.py:109-172, Workflow.learning_step :569-612) as captured rounds,
// and its backward by recomputation.
//
// Rollout round (graphed.GraphedGeneratorRL):  gib_rl_snapshot -> K0 -> forward(agent) -> forward(prior) ->
// gib_rl_sample_round (generate.cu: sample from the agent, rl_probs_kernel, the round kernels with slot tags).  A round
// keeps only its INPUT: the 0/1 generation state as int8 in a [2N, B, ...] record.  After the last round
// gib_rl_gather maps the per-round probabilities p[r, b] through the (molecule, round) -> slot map the round kernels
// wrote into generated_likelihoods.
//
// Backward: gib_rl_scatter_grad inverts that map (dL/d generated likelihoods -> dL/dp[r, b]); then per model and round
// gib_rl_restore -> K0 -> forward -> gib_rl_dlogits -> gib_model_backward -> gib_rl_next_round, the round index in
// device memory.  The kernels are deterministic and int8 inputs give the float inputs' logits bit for bit, so the
// recomputed probabilities equal the rollout's.
#include <algorithm>

#include "../../include/gib200.h"
#include "common.cuh"
#include "ops.cuh"

namespace gib {

constexpr int kRowThreads = 256;

// softmax statistics of one APD row in a fixed order (max, then sum of exp(x - max)); every thread gets both.  The
// rollout and the backward both go through here, which makes their probabilities identical.
__device__ __forceinline__ void row_softmax(const float* __restrict__ o, int apd, float* sm, float& mx, float& se) {
  float m = -INFINITY;
  for (int k = threadIdx.x; k < apd; k += kRowThreads) m = fmaxf(m, o[k]);
  m = block_reduce<kRowThreads>(m, sm, true);
  float s = 0.f;
  for (int k = threadIdx.x; k < apd; k += kRowThreads) s += expf(o[k] - m);
  se = block_reduce<kRowThreads>(s, sm, false);
  mx = m;
}

// probability of action a (0 for an index outside the APD: such a slot terminates as invalid and is never read back)
__device__ __forceinline__ float row_prob(const float* __restrict__ o, int apd, int a, float mx, float se) {
  return (a >= 0 && a < apd) ? expf(o[a] - mx) / se : 0.f;
}

__global__ void __launch_bounds__(kRowThreads) rl_probs_kernel(const float* __restrict__ la,
                                                               const float* __restrict__ lb, int apd,
                                                               const int* __restrict__ action,
                                                               const int* __restrict__ ctl, int* __restrict__ act_rec,
                                                               float* __restrict__ p_a, float* __restrict__ p_b,
                                                               float* __restrict__ tags) {
  __shared__ float sm[kRowThreads / 32];
  const int r = ctl[0];
  if (r < 0) return;
  const int b = blockIdx.x, B = gridDim.x;
  const int a = action[b];
  float mx, se;
  row_softmax(la + (size_t)b * apd, apd, sm, mx, se);
  const float pa = row_prob(la + (size_t)b * apd, apd, a, mx, se);
  row_softmax(lb + (size_t)b * apd, apd, sm, mx, se);
  const float pb = row_prob(lb + (size_t)b * apd, apd, a, mx, se);
  if (threadIdx.x == 0) {
    const size_t i = (size_t)r * B + b;
    act_rec[i] = a;
    p_a[i] = pa;
    p_b[i] = pb;
    tags[b] = (float)(b + 1);
  }
}

int rl_probs_launch(const float* logits_a, const float* logits_b, int B, int apd, const int* action, const int* ctl,
                    int* act_rec, float* p_a, float* p_b, float* tags, cudaStream_t st) {
  rl_probs_kernel<<<B, kRowThreads, 0, st>>>(logits_a, logits_b, apd, action, ctl, act_rec, p_a, p_b, tags);
  GIB_LAUNCH_CHECK();
  return 0;
}

// the route scorer's probability of each slot's route action (graphed.RouteScorer): p = softmax(logits[b])[a] by
// rl_probs_kernel's reduction, written at the state's place dst; slots [2B] = {action[B], dst[B]}, dst < 0: padding
__global__ void __launch_bounds__(kRowThreads) route_probs_kernel(const float* __restrict__ logits, int apd,
                                                                  const int* __restrict__ slots,
                                                                  float* __restrict__ lik) {
  __shared__ float sm[kRowThreads / 32];
  const int b = blockIdx.x, B = gridDim.x;
  const int dst = slots[B + b];
  if (dst < 0) return;
  const float* o = logits + (size_t)b * apd;
  float mx, se;
  row_softmax(o, apd, sm, mx, se);
  const float p = row_prob(o, apd, slots[b], mx, se);
  if (threadIdx.x == 0) lik[dst] = p;
}

// one CTA per slot: float 0/1 state -> int8 model input and, for a running round, the record row state[0]
__global__ void __launch_bounds__(128) rl_snapshot_kernel(int N, int F, int Ef, int att_view,
                                                          const float* __restrict__ nodes,
                                                          const float* __restrict__ edges,
                                                          const int* __restrict__ state,
                                                          const int* __restrict__ counters,
                                                          signed char* __restrict__ rec_nodes,
                                                          signed char* __restrict__ rec_edges,
                                                          signed char* __restrict__ in_nodes,
                                                          signed char* __restrict__ in_edges) {
  const int b = blockIdx.x, B = gridDim.x;
  const int r = state[0];
  // the sampler's gate (api.cu): this round runs and will be back-propagated through
  const bool live = counters[0] < B && state[1] == 0 && r >= 0 && r < 2 * N;
  const int NF = N * F, NNE = N * N * Ef;
  const float* nb = nodes + (size_t)b * NF;
  const float* eb = edges + (size_t)b * NNE;
  signed char* rn = rec_nodes + ((size_t)(live ? r : 0) * B + b) * NF;
  signed char* re = rec_edges + ((size_t)(live ? r : 0) * B + b) * NNE;
  for (int i = threadIdx.x; i < NF; i += 128) {
    const signed char v = (signed char)__float2int_rz(nb[i]);
    in_nodes[(size_t)b * NF + i] = v;
    if (live) rn[i] = v;
  }
  for (int i = threadIdx.x; i < NNE; i += 128) {
    float x = eb[i];
    if (att_view && b == 0 && x != 0.f) {
      // GraphGenerator._model_inputs: the dummy graph keeps the first non-zero type of each bond only
      const int t = i % Ef;
      for (int u = 0; u < t; ++u)
        if (eb[i - t + u] != 0.f) x = 0.f;
    }
    const signed char v = (signed char)__float2int_rz(x);
    in_edges[(size_t)b * NNE + i] = v;
    if (live) re[i] = v;
  }
}

__global__ void rl_restore_kernel(const signed char* __restrict__ rec, signed char* __restrict__ in, long long n,
                                  const int* __restrict__ ctl) {
  const signed char* src = rec + (long long)ctl[0] * n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    in[i] = src[i];
}

// out[g, t] = p[t, owner[g, t] - 1], 0 where owner[g, t] == 0
__global__ void rl_gather_kernel(int B, long long n, int Lw, const float* __restrict__ owner,
                                 const float* __restrict__ p_a, const float* __restrict__ p_b,
                                 float* __restrict__ out_a, float* __restrict__ out_b) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int t = (int)(i % Lw);
  const int s = (int)owner[i] - 1;
  const bool hit = s >= 0 && s < B;
  out_a[i] = hit ? p_a[(size_t)t * B + s] : 0.f;
  out_b[i] = hit ? p_b[(size_t)t * B + s] : 0.f;
}

// the inverse map: dp[t, owner[g, t] - 1] = d[g, t].  A slot's round-t action belongs to at most one molecule and
// slot 0 (the dummy graph) to none, so every dp element is written at most once: no atomics, deterministic
__global__ void rl_scatter_grad_kernel(int B, long long n, int Lw, const float* __restrict__ owner,
                                       const float* __restrict__ d_a, const float* __restrict__ d_b,
                                       float* __restrict__ dp_a, float* __restrict__ dp_b) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int t = (int)(i % Lw);
  const int s = (int)owner[i] - 1;
  if (s < 0 || s >= B) return;
  if (d_a) dp_a[(size_t)t * B + s] = d_a[i];
  if (d_b) dp_b[(size_t)t * B + s] = d_b[i];
}

// dlogits[b, :] = dp[r, b] * p * (onehot(a) - softmax(logits[b])), p = softmax(logits[b])[a], a = act[r, b]
__global__ void __launch_bounds__(kRowThreads) rl_dlogits_kernel(int apd, const float* __restrict__ logits,
                                                                 const int* __restrict__ act,
                                                                 const float* __restrict__ dp,
                                                                 const int* __restrict__ ctl,
                                                                 float* __restrict__ dlogits, float* __restrict__ p_out) {
  __shared__ float sm[kRowThreads / 32];
  const int b = blockIdx.x, B = gridDim.x;
  const size_t i = (size_t)(ctl ? ctl[0] : 0) * B + b;
  const int a = act[i];
  const float* o = logits + (size_t)b * apd;
  float mx, se;
  row_softmax(o, apd, sm, mx, se);
  const float p = row_prob(o, apd, a, mx, se);
  const float g = dp[i] * p;
  float* dl = dlogits + (size_t)b * apd;
  for (int k = threadIdx.x; k < apd; k += kRowThreads) dl[k] = g * ((k == a ? 1.f : 0.f) - expf(o[k] - mx) / se);
  if (threadIdx.x == 0 && p_out) p_out[i] = p;
}

__global__ void rl_next_round_kernel(int* ctl) { ctl[0] += 1; }

}  // namespace gib

using namespace gib;

#define ST(s) reinterpret_cast<cudaStream_t>(s)

static int check_state_dims(const char* who, int B, int N, int F, int Ef) {
  if (B <= 0 || N <= 0 || N > 127 || F <= 0 || Ef <= 0 || (long long)B * N * N * Ef >= (1ll << 31)) {
    set_error("%s: unsupported dims B=%d N=%d F=%d Ef=%d", who, B, N, F, Ef);
    return -1;
  }
  return 0;
}

static unsigned grid_for(long long n, int threads) { return (unsigned)std::min<long long>(ceil_div_ll(n, threads), 1 << 16); }

extern "C" {

int gib_rl_snapshot(int B, int N, int F, int Ef, int att_view, const float* nodes, const float* edges,
                    const int* state, const int* counters, signed char* rec_nodes, signed char* rec_edges,
                    signed char* in_nodes, signed char* in_edges, gib_stream stream) {
  GIB_TRY(check_state_dims("gib_rl_snapshot", B, N, F, Ef));
  if (!nodes || !edges || !state || !counters || !rec_nodes || !rec_edges || !in_nodes || !in_edges) {
    set_error("gib_rl_snapshot: null buffer");
    return -1;
  }
  rl_snapshot_kernel<<<B, 128, 0, ST(stream)>>>(N, F, Ef, att_view, nodes, edges, state, counters, rec_nodes,
                                                rec_edges, in_nodes, in_edges);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gib_rl_restore(int B, int N, int F, int Ef, const signed char* rec_nodes, const signed char* rec_edges,
                   const int* ctl, signed char* in_nodes, signed char* in_edges, gib_stream stream) {
  GIB_TRY(check_state_dims("gib_rl_restore", B, N, F, Ef));
  if (!rec_nodes || !rec_edges || !ctl || !in_nodes || !in_edges) {
    set_error("gib_rl_restore: null buffer");
    return -1;
  }
  const long long nn = (long long)B * N * F, ne = (long long)B * N * N * Ef;
  rl_restore_kernel<<<grid_for(nn, 256), 256, 0, ST(stream)>>>(rec_nodes, in_nodes, nn, ctl);
  GIB_LAUNCH_CHECK();
  rl_restore_kernel<<<grid_for(ne, 256), 256, 0, ST(stream)>>>(rec_edges, in_edges, ne, ctl);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gib_rl_gather(int B, int rows, int Lw, const float* owner, const float* p_a, const float* p_b, float* out_a,
                  float* out_b, gib_stream stream) {
  if (B <= 0 || rows <= 0 || Lw <= 0 || !owner || !p_a || !p_b || !out_a || !out_b) {
    set_error("gib_rl_gather: bad arguments (B=%d rows=%d Lw=%d, every table must be given)", B, rows, Lw);
    return -1;
  }
  const long long n = (long long)rows * Lw;
  rl_gather_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, ST(stream)>>>(B, n, Lw, owner, p_a, p_b, out_a, out_b);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gib_rl_scatter_grad(int B, int rows, int Lw, const float* owner, const float* d_a, const float* d_b, float* dp_a,
                        float* dp_b, gib_stream stream) {
  if (B <= 0 || rows <= 0 || Lw <= 0 || !owner || (d_a && !dp_a) || (d_b && !dp_b)) {
    set_error("gib_rl_scatter_grad: bad arguments (B=%d rows=%d Lw=%d; an output table for every input)", B, rows,
              Lw);
    return -1;
  }
  cudaStream_t st = ST(stream);
  if (d_a) GIB_CUDA_TRY(cudaMemsetAsync(dp_a, 0, (size_t)Lw * B * sizeof(float), st));
  if (d_b) GIB_CUDA_TRY(cudaMemsetAsync(dp_b, 0, (size_t)Lw * B * sizeof(float), st));
  const long long n = (long long)rows * Lw;
  rl_scatter_grad_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(B, n, Lw, owner, d_a, d_b, dp_a, dp_b);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gib_rl_dlogits(int B, int apd, const float* logits, const int* act, const float* dp, const int* ctl,
                   float* dlogits, float* p, gib_stream stream) {
  if (B <= 0 || apd <= 0 || !logits || !act || !dp || !dlogits) {
    set_error("gib_rl_dlogits: bad arguments (B=%d apd=%d; logits, act, dp and dlogits must be given)", B, apd);
    return -1;
  }
  rl_dlogits_kernel<<<B, kRowThreads, 0, ST(stream)>>>(apd, logits, act, dp, ctl, dlogits, p);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gib_route_probs(int B, int apd, const float* logits, const int* slots, float* likelihoods, gib_stream stream) {
  if (B <= 0 || apd <= 0 || !logits || !slots || !likelihoods) {
    set_error("gib_route_probs: bad arguments (B=%d apd=%d; logits, slots and likelihoods must be given)", B, apd);
    return -1;
  }
  route_probs_kernel<<<B, kRowThreads, 0, ST(stream)>>>(logits, apd, slots, likelihoods);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gib_rl_next_round(int* ctl, gib_stream stream) {
  if (!ctl) {
    set_error("gib_rl_next_round: null counter");
    return -1;
  }
  rl_next_round_kernel<<<1, 1, 0, ST(stream)>>>(ctl);
  GIB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
