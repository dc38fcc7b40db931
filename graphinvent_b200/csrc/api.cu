// extern "C" boundary of libgib200.so (see include/gib200.h for the contract).
#include <stdarg.h>
#include <string.h>

#include <algorithm>

#include "../../include/gib200.h"
#include "gemm.cuh"
#include "model.cuh"
#include "ops.cuh"

namespace gib {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// ---- KL-divergence loss + gradient (Workflow.py:833-860), one CTA per molecule ---------
__global__ void __launch_bounds__(256) kl_loss_kernel(const float* __restrict__ out, const float* __restrict__ target,
                                                      int apd, float grad_scale, const gib_batch_ctl* ctl,
                                                      const float* __restrict__ loss_scale,
                                                      float* __restrict__ loss_rows, float* __restrict__ dout) {
  __shared__ float sm[8];
  const int b = blockIdx.x;
  if (ctl) {                                    // a partial batch: rows past the live count are padding
    if (b >= ctl->live) {
      if (dout)
        for (int k = threadIdx.x; k < apd; k += 256) dout[(size_t)b * apd + k] = 0.f;
      if (threadIdx.x == 0 && loss_rows) loss_rows[b] = 0.f;
      return;
    }
    grad_scale = ctl->scale;
  }
  const float* o = out + (size_t)b * apd;
  const float* t = target + (size_t)b * apd;
  float mx = -INFINITY, ts = 0.f;
  for (int k = threadIdx.x; k < apd; k += 256) { mx = fmaxf(mx, o[k]); ts += t[k]; }
  mx = block_reduce<256>(mx, sm, true);
  ts = block_reduce<256>(ts, sm, false);
  float se = 0.f;
  for (int k = threadIdx.x; k < apd; k += 256) se += expf(o[k] - mx);
  se = block_reduce<256>(se, sm, false);
  const float lse = mx + logf(se);
  float acc = 0.f;
  for (int k = threadIdx.x; k < apd; k += 256) {
    const float th = t[k] / ts;                 // Workflow.py:854 (NaN for an all-zero target row, as in the reference)
    const float logp = o[k] - lse;
    acc += (th > 0.f ? th * logf(th) : (th == 0.f ? 0.f : th)) - th * logp;   // xlogy(t,t) - t*logp
    if (dout) {
      float d = (expf(logp) - th) * grad_scale;
      if (loss_scale) d *= *loss_scale;         // autograd's dout * g for g = the GradScaler's scale
      dout[(size_t)b * apd + k] = d;
    }
  }
  acc = block_reduce<256>(acc, sm, false);
  if (threadIdx.x == 0 && loss_rows) loss_rows[b] = acc;
}

// ---- validation NLL per sub-graph (Analyzer.get_validation_likelihood, Analyzer.py:744-758):
//      nll[b] = -log( sum_k softmax(out[b])_k * target[b,k] / sum(target[b]) );  an all-zero target row gives NaN,
//      which the reference filters out afterwards (Analyzer.py:756) -----------------------------------------------
__global__ void __launch_bounds__(256) validation_nll_kernel(const float* __restrict__ out,
                                                             const float* __restrict__ target, int apd,
                                                             const gib_batch_ctl* ctl, float* __restrict__ nll) {
  __shared__ float sm[8];
  const int b = blockIdx.x;
  if (ctl && b >= ctl->live) {
    if (threadIdx.x == 0) nll[b] = 0.f;
    return;
  }
  const float* o = out + (size_t)b * apd;
  const float* t = target + (size_t)b * apd;
  float mx = -INFINITY, ts = 0.f;
  for (int k = threadIdx.x; k < apd; k += 256) { mx = fmaxf(mx, o[k]); ts += t[k]; }
  mx = block_reduce<256>(mx, sm, true);
  ts = block_reduce<256>(ts, sm, false);
  float se = 0.f, dot = 0.f;
  for (int k = threadIdx.x; k < apd; k += 256) {
    const float e = expf(o[k] - mx);
    se += e;
    dot += e * t[k];
  }
  se = block_reduce<256>(se, sm, false);
  dot = block_reduce<256>(dot, sm, false);
  if (threadIdx.x == 0) nll[b] = -logf((dot / se) / ts);     // ts == 0 -> 0/0 = NaN like target/sum(target)
}

// ---- categorical sampling of one action per molecule (GraphGenerator.py:121, 535-542) ----
// g.state != null: the round-gated form of gib_generation_sample_round (ops.cuh: RoundGate)
__global__ void __launch_bounds__(256) sample_actions_kernel(const float* __restrict__ out, int apd,
                                                             const float* __restrict__ uniforms,
                                                             int* __restrict__ action, float* __restrict__ lik,
                                                             RoundGate g) {
  __shared__ float sm[8];
  __shared__ float pre[257];
  const int b = blockIdx.x;
  if (g.state) {
    // every CTA reads the same words before any of them is written (state[0] / counters advance in gen_scan_kernel,
    // which runs after this kernel); only CTA 0 writes, and a status it sets cannot change another CTA's decision
    const int r = g.state[0], B = gridDim.x;
    const bool live = g.counters[0] < B && g.state[1] == 0;
    const bool go = live && r >= 0 && r < g.rounds;
    if (b == 0 && threadIdx.x == 0) {
      g.ctl[0] = go ? r : -1;
      if (live && !go) g.state[1] = 1;
    }
    if (!go) return;
    if (g.actions) {                  // recorded actions: row r is the draw, the caller computes the likelihoods
      if (threadIdx.x == 0) action[b] = g.actions[(size_t)r * B + b];
      return;
    }
    uniforms += (size_t)r * B;
  }
  const float* o = out + (size_t)b * apd;
  float mx = -INFINITY;
  for (int k = threadIdx.x; k < apd; k += 256) mx = fmaxf(mx, o[k]);
  mx = block_reduce<256>(mx, sm, true);
  const int L = ceil_div(apd, 256);
  const int lo = min(apd, (int)threadIdx.x * L), hi = min(apd, lo + L);
  float s = 0.f;
  for (int k = lo; k < hi; ++k) s += expf(o[k] - mx);
  pre[threadIdx.x + 1] = s;
  if (threadIdx.x == 0) pre[0] = 0.f;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int i = 1; i <= 256; ++i) pre[i] += pre[i - 1];   // fixed-order prefix: deterministic
  __syncthreads();
  const float total = pre[256];
  float target = uniforms[b] * total;
  // u * total may round up to the total: keep the target inside [0, total) so that it always has an owner chunk
  if (target >= total) target = nextafterf(total, 0.f);
  // the owner thread is the chunk whose prefix bracket [pre[t], pre[t+1]) holds the target: its sum is > 0, so it holds
  // an action of non-zero probability
  const bool owner = pre[threadIdx.x] <= target && target < pre[threadIdx.x + 1];
  if (owner && hi > lo) {
    float run = pre[threadIdx.x];
    int pick = -1, last = lo;
    for (int k = lo; k < hi; ++k) {
      const float e = expf(o[k] - mx);
      run += e;
      if (e > 0.f) last = k;
      if (target < run) { pick = k; break; }
    }
    // the running sum can end a few ulps below pre[t+1] (other rounding order): the last action of the chunk with
    // non-zero probability, never one of probability 0
    if (pick < 0) pick = last;
    action[b] = pick;
    lik[b] = expf(o[pick] - mx) / total;
  }
  // a row with NaN / Inf logits has no owner (every comparison with NaN is false): defined outputs instead of the
  // caller's uninitialised memory -- "terminate" with a NaN likelihood, which the caller can detect
  if (threadIdx.x == 0 && !(total == total && total > 0.f && total < INFINITY && target == target)) {
    action[b] = apd - 1;
    lik[b] = NAN;
  }
}

int sample_actions_launch(const float* out, int B, int apd, const float* uniforms, int* action, float* lik,
                          const RoundGate* gate, cudaStream_t st) {
  if (B <= 0) return 0;
  sample_actions_kernel<<<B, 256, 0, st>>>(out, apd, uniforms, action, lik, gate ? *gate : RoundGate{});
  GIB_LAUNCH_CHECK();
  return 0;
}

// ---- the per-batch tail of a validation pass (include/gib200.h: gib_eval_collect), one CTA --------------------------
constexpr int kEvalThreads = 1024;
__global__ void __launch_bounds__(kEvalThreads) eval_collect_kernel(const float* __restrict__ kl_rows,
                                                                    const float* __restrict__ nll_rows,
                                                                    const float* __restrict__ target, int B, int apd,
                                                                    const gib_batch_ctl* __restrict__ ctl,
                                                                    const int* __restrict__ count_ws,
                                                                    gib_eval_pass* pass) {
  __shared__ float sm[kEvalThreads / 32];
  __shared__ int warp_kept[kEvalThreads / 32];
  const int live = max(0, min(B, ctl->live));
  const int idx = pass->idx;     // read by every thread before the first barrier; thread 0 advances it at the end
  float kl = 0.f, ns = 0.f;
  for (int b = threadIdx.x; b < live; b += kEvalThreads) {
    kl += kl_rows[b];
    ns += target[(size_t)b * apd + apd - 1];      // the unnormalised target: its last column counts the sub-graphs
  }
  kl = block_reduce<kEvalThreads>(kl, sm, false);
  ns = block_reduce<kEvalThreads>(ns, sm, false);
  // likelihood[~isnan(likelihood)] written from idx * B: an order-preserving compaction, one CTA-wide scan per chunk
  float* lik = pass->lik;
  const long long base = (long long)idx * B;
  int kept = 0;                  // uniform across the CTA
  if (lik) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long len = pass->lik_len;
    for (int c = 0; c < live; c += kEvalThreads) {
      const int b = c + threadIdx.x;
      const float v = b < live ? nll_rows[b] : NAN;
      const bool keep = !isnan(v);
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) warp_kept[wid] = __popc(m);
      __syncthreads();
      int before = __popc(m & ((1u << lane) - 1u)), total = 0;
      for (int w = 0; w < kEvalThreads / 32; ++w) {
        const int x = warp_kept[w];
        before += w < wid ? x : 0;
        total += x;
      }
      const long long pos = base + kept + before;
      if (keep && pos < len) lik[pos] = v;
      kept += total;
      __syncthreads();           // warp_kept is rewritten by the next chunk
    }
  }
  if (threadIdx.x == 0) {
    if (pass->batch_loss && idx >= 0 && idx < pass->n_slots) pass->batch_loss[idx] = kl / (float)live;
    if (lik) {
      const long long past = base + kept - pass->lik_len;     // kept rows at positions >= lik_len
      pass->clipped += (int)(past <= 0 ? 0 : past < kept ? past : kept);
    }
    pass->n_structures += ns;
    pass->flags |= count_ws[HDR_FLAGS];
    pass->idx = idx + 1;
  }
}

}  // namespace gib

using namespace gib;

#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

const char* gib_last_error(void) { return g_err; }
// 200: capacity mode, int8 inputs, grouped dW; 201: 5 profile classes; 202: test hooks; 203: forward / glue test hooks;
// 204: gib_generation_round_layout (implicit-H / chirality action layouts); 205: gib_generation_sample_round;
// 206: the matmul precision is gib_dims.tf32, no longer a thread-local setting
int gib_version(void) { return 206; }
void gib_set_tensor_cores(int on) { g_use_tc = on != 0; }
int gib_get_tensor_cores(void) { return g_use_tc ? 1 : 0; }
void gib_tc_debug(int mode) { g_tc_debug = mode; }
int gib_device_sm_count(void) { return device_sm_count(); }
void gib_scatter_variant(int v) { g_scatter_variant = v; }
void gib_tc_trace(long long* device_buf, int tiles) { tc3_set_trace(device_buf, tiles); }

static int groups_of(const gib_dims* d) { return d->model == GIB_EMN ? 1 : d->Ef; }
static bool is_cap(const int* hdr) { return hdr[HDR_CAPACITY] != 0; }

size_t gib_graph_count_ws_bytes(const gib_dims* d) {
  return graph_count_ws_ints(d->B, groups_of(d)) * sizeof(int);
}
int gib_graph_count(const gib_dims* d, const void* edges, void* count_ws, gib_stream stream) {
  return graph_count(edges, d->in_dtype, d->B, d->N, d->Ef, d->model != GIB_EMN, reinterpret_cast<int*>(count_ws),
                     ST(stream));
}
int gib_graph_header_capacity(const gib_dims* d, int entry_capacity, const void* count_ws, int* hdr) {
  if (entry_capacity < 1 || !count_ws) { set_error("gib_graph_header_capacity: bad capacity / workspace"); return -1; }
  const int G = groups_of(d);
  memset(hdr, 0, HDR_INTS * sizeof(int));
  hdr[HDR_E] = entry_capacity;
  // every type group is padded to a multiple of 128 rows: at most 127 pad rows per group
  hdr[HDR_P] = ceil_div(entry_capacity, kTileRows) * kTileRows + G * kTileRows;
  hdr[HDR_CAPACITY] = 1;
  const unsigned long long a = reinterpret_cast<unsigned long long>(count_ws);
  hdr[HDR_DEV_LO] = (int)(unsigned)(a & 0xffffffffull);
  hdr[HDR_DEV_HI] = (int)(unsigned)(a >> 32);
  return 0;
}
size_t gib_graph_bytes(const gib_dims* d, const int* hdr) {
  return graph_buf_ints((long long)d->B * d->N, hdr[HDR_E], hdr[HDR_P]) * sizeof(int);
}
int gib_graph_fill(const gib_dims* d, const void* edges, void* count_ws, const int* hdr, void* graph_buf,
                   gib_stream stream) {
  GraphArrays ga = graph_arrays(graph_buf, (long long)d->B * d->N, hdr[HDR_E], hdr[HDR_P]);
  return graph_fill(edges, d->in_dtype, d->B, d->N, d->Ef, d->model != GIB_EMN, reinterpret_cast<int*>(count_ws), ga,
                    is_cap(hdr) ? hdr[HDR_E] : 0, is_cap(hdr) ? hdr[HDR_P] : 0, ST(stream));
}
void* gib_graph_array(const gib_dims* d, const int* hdr, void* graph_buf, int which) {
  GraphArrays ga = graph_arrays(graph_buf, (long long)d->B * d->N, hdr[HDR_E], hdr[HDR_P]);
  switch (which) {
    case 0: return ga.ent_src;
    case 1: return ga.ent_dst;
    case 2: return ga.ent_w;
    case 3: return ga.dst_ptr;
    case 4: return ga.dst_ent;
    case 5: return ga.src_ptr;
    case 6: return ga.src_ent;
  }
  return nullptr;
}

int gib_model_num_params(const gib_dims* d) {
  Plan pl;
  if (build_plan(*d, pl)) return -1;
  return (int)pl.param_numel.size();
}
long long gib_model_param_numel(const gib_dims* d, int index) {
  Plan pl;
  if (build_plan(*d, pl) || index < 0 || index >= (int)pl.param_numel.size()) return -1;
  return pl.param_numel[index];
}
size_t gib_model_packed_bytes(const gib_dims* d) {
  Plan pl;
  if (build_plan(*d, pl)) return 0;
  return pl.packed_floats * sizeof(float);
}
int gib_model_pack(const gib_dims* d, const float* const* params, void* packed, gib_stream stream) {
  Plan pl;
  GIB_TRY(build_plan(*d, pl));
  return pack_params(pl, params, reinterpret_cast<float*>(packed), d->tf32, ST(stream));
}

size_t gib_model_workspace_bytes(const gib_dims* d, const int* hdr) {
  Run r;
  if (make_run(*d, hdr, r)) return 0;
  return r.L.total * sizeof(float) + 256;
}
int gib_model_forward(const gib_dims* d, const int* hdr, const void* nodes, const void* edges, const void* graph_buf,
                      const void* packed, void* workspace, float* out, gib_stream stream) {
  Run r;
  GIB_TRY(make_run(*d, hdr, r));
  GIB_TRY(check_precision(r.tf32, "gib_model_forward"));
  r.nodes = nodes; r.edges = edges;
  r.ga = graph_arrays(const_cast<void*>(graph_buf), r.S, r.E, r.P);
  r.packed = reinterpret_cast<const float*>(packed);
  r.ws = reinterpret_cast<float*>(workspace);
  r.st = ST(stream);
  return model_forward(r, out);
}
void* gib_model_msg_rows(const gib_dims* d, const int* hdr, void* workspace, int which) {
  Run r;
  if (make_run(*d, hdr, r) || d->model == GIB_EMN || d->model == GIB_ATTGGNN) return nullptr;
  const size_t offs[10] = {r.L.mr_src, r.L.mr_w, r.L.mr_ptr, r.L.mr_dst, r.L.mr_ent, r.L.mr_dst_u, r.L.mr_sptr,
                           r.L.mr_su, r.L.mr_meta, r.L.mr_tmp};
  if (which < 0 || which >= 10) return nullptr;
  return reinterpret_cast<float*>(workspace) + offs[which];
}
size_t gib_model_bwd_scratch_bytes(const gib_dims* d, const int* hdr) {
  Run r;
  if (make_run(*d, hdr, r)) return 0;
  BwdBufs bb;
  make_bwd(r, bb);
  return bb.total * sizeof(float) + 256;
}
int gib_model_backward(const gib_dims* d, const int* hdr, const void* nodes, const void* edges, const void* graph_buf,
                       const void* packed, const void* workspace, const float* out, const float* dout,
                       float* const* grads, void* scratch, gib_stream stream) {
  return gib_model_backward_part(d, hdr, nodes, edges, graph_buf, packed, workspace, out, dout, grads, scratch, 0,
                                 stream);
}
int gib_model_backward_part(const gib_dims* d, const int* hdr, const void* nodes, const void* edges,
                            const void* graph_buf, const void* packed, const void* workspace, const float* out,
                            const float* dout, float* const* grads, void* scratch, int part, gib_stream stream) {
  Run r;
  GIB_TRY(make_run(*d, hdr, r));
  GIB_TRY(check_precision(r.tf32, "gib_model_backward"));
  r.nodes = nodes; r.edges = edges;
  r.ga = graph_arrays(const_cast<void*>(graph_buf), r.S, r.E, r.P);
  r.packed = reinterpret_cast<const float*>(packed);
  r.ws = reinterpret_cast<float*>(const_cast<void*>(workspace));
  r.scratch = reinterpret_cast<float*>(scratch);
  r.grads = grads;
  r.st = ST(stream);
  BwdBufs bb;
  make_bwd(r, bb);
  return model_backward(r, bb, out, dout, part);
}

int gib_kl_loss_fwd_bwd(const float* out, const float* target, int B, int apd, float grad_scale, float* loss_rows,
                        float* dout, gib_stream stream) {
  if (B <= 0) return 0;
  kl_loss_kernel<<<B, 256, 0, ST(stream)>>>(out, target, apd, grad_scale, nullptr, nullptr, loss_rows, dout);
  GIB_LAUNCH_CHECK();
  return 0;
}
int gib_kl_loss_fwd_bwd_ctl(const float* out, const float* target, int B, int apd, const gib_batch_ctl* ctl,
                            float* loss_rows, float* dout, gib_stream stream) {
  if (!ctl) { set_error("gib_kl_loss_fwd_bwd_ctl: ctl is null"); return -1; }
  if (B <= 0) return 0;
  kl_loss_kernel<<<B, 256, 0, ST(stream)>>>(out, target, apd, 0.f, ctl, nullptr, loss_rows, dout);
  GIB_LAUNCH_CHECK();
  return 0;
}
int gib_kl_loss_fwd_bwd_ctl_scaled(const float* out, const float* target, int B, int apd, const gib_batch_ctl* ctl,
                                   const float* loss_scale, float* loss_rows, float* dout, gib_stream stream) {
  if (!ctl || !loss_scale) { set_error("gib_kl_loss_fwd_bwd_ctl_scaled: ctl and loss_scale must be non-null"); return -1; }
  if (B <= 0) return 0;
  kl_loss_kernel<<<B, 256, 0, ST(stream)>>>(out, target, apd, 0.f, ctl, loss_scale, loss_rows, dout);
  GIB_LAUNCH_CHECK();
  return 0;
}

// out[0] = scale * sum_b rows[b], fixed order (one CTA): the batch-mean of the per-molecule losses without an ATen
// reduction inside a captured step
// ctl != null: the first min(n, ctl->live) rows, scaled by ctl->scale
__global__ void __launch_bounds__(256) sum_scaled_kernel(const float* __restrict__ rows, int n, float scale,
                                                         const gib_batch_ctl* ctl, float* __restrict__ out) {
  __shared__ float sm[8];
  if (ctl) {
    n = min(n, ctl->live);
    scale = ctl->scale;
  }
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) s += rows[i];
  s = block_reduce<256>(s, sm, false);
  if (threadIdx.x == 0) out[0] = s * scale;
}
int gib_sum_scaled(const float* rows, int n, float scale, float* out, gib_stream stream) {
  sum_scaled_kernel<<<1, 256, 0, ST(stream)>>>(rows, n, scale, nullptr, out);
  GIB_LAUNCH_CHECK();
  return 0;
}
int gib_sum_scaled_ctl(const float* rows, int n, const gib_batch_ctl* ctl, float* out, gib_stream stream) {
  if (!ctl) { set_error("gib_sum_scaled_ctl: ctl is null"); return -1; }
  sum_scaled_kernel<<<1, 256, 0, ST(stream)>>>(rows, n, 0.f, ctl, out);
  GIB_LAUNCH_CHECK();
  return 0;
}
int gib_fill_zero(void* ptr, size_t bytes, gib_stream stream) {
  if (bytes == 0) return 0;
  GIB_CUDA_TRY(cudaMemsetAsync(ptr, 0, bytes, ST(stream)));
  return 0;
}

int gib_validation_nll(const float* out, const float* target, int B, int apd, float* nll, gib_stream stream) {
  if (B <= 0) return 0;
  validation_nll_kernel<<<B, 256, 0, ST(stream)>>>(out, target, apd, nullptr, nll);
  GIB_LAUNCH_CHECK();
  return 0;
}
int gib_validation_nll_ctl(const float* out, const float* target, int B, int apd, const gib_batch_ctl* ctl, float* nll,
                           gib_stream stream) {
  if (!ctl) { set_error("gib_validation_nll_ctl: ctl is null"); return -1; }
  if (B <= 0) return 0;
  validation_nll_kernel<<<B, 256, 0, ST(stream)>>>(out, target, apd, ctl, nll);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gib_eval_collect(const float* kl_rows, const float* nll_rows, const float* target, int B, int apd,
                     const gib_batch_ctl* ctl, const void* count_ws, gib_eval_pass* pass, gib_stream stream) {
  if (B <= 0 || apd <= 0 || !kl_rows || !nll_rows || !target || !ctl || !count_ws || !pass) {
    set_error("gib_eval_collect: B = %d, apd = %d (both > 0) and every pointer non-null", B, apd);
    return -1;
  }
  eval_collect_kernel<<<1, kEvalThreads, 0, ST(stream)>>>(kl_rows, nll_rows, target, B, apd, ctl,
                                                          reinterpret_cast<const int*>(count_ws), pass);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gib_sample_actions(const float* out, int B, int apd, const float* uniforms, int* action, float* likelihood,
                       gib_stream stream) {
  return sample_actions_launch(out, B, apd, uniforms, action, likelihood, nullptr, ST(stream));
}

int gib_linear_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias, float* Y, int ldy, int M,
                   int N, int K, int act, gib_stream stream) {
  GemmNT p;
  p.A = X; p.lda = ldx; p.B = W; p.ldb = ldw; p.C = Y; p.ldc = ldy; p.M = M; p.N = N; p.K = K; p.bias = bias;
  p.act = act; p.mode = EPI_ACT; p.n_store = N; p.n_valid = N;
  return gemm_nt(p, ST(stream));
}
int gib_linear_fwd_tc(const float* X, int ldx, const float* W, int ldw, const float* bias, float* Y, int ldy, int M,
                      int N, int K, int act, gib_stream stream) {
  GemmNT p;
  p.A = X; p.lda = ldx; p.B = W; p.ldb = ldw; p.C = Y; p.ldc = ldy; p.M = M; p.N = N; p.K = K; p.bias = bias;
  p.act = act; p.mode = EPI_ACT; p.n_store = N; p.n_valid = N;
  return gemm_nt_tc(p, ST(stream));
}
int gib_linear_fwd_tc_planes(const float* X, int ldx, const float* W_hi, const float* W_lo, int ldw, const float* bias,
                             float* Y, int ldy, int M, int N, int K, int act, const int* m_dev, const int* base_dev,
                             gib_stream stream) {
  GemmNT p;
  p.A = X; p.lda = ldx; p.B = W_hi; p.B_hi = W_hi; p.B_lo = W_lo; p.ldb = ldw; p.C = Y; p.ldc = ldy;
  p.M = M; p.N = N; p.K = K; p.bias = bias; p.act = act; p.mode = EPI_ACT; p.n_store = N; p.n_valid = N;
  p.m_dev = m_dev; p.base_dev = base_dev;
  if (g_tc_debug & 1) {
    if (m_dev) { set_error("device-side row counts need the second-generation kernel"); return -2; }
    return gemm_nt_tc(p, ST(stream));
  }
  return gemm_nt_tc3_group(&p, 1, ST(stream));
}
__global__ void split_planes_kernel(const float* __restrict__ W, float* __restrict__ hi, float* __restrict__ lo,
                                    long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = W[i];
  unsigned h, l;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(x - __uint_as_float(h)));
  hi[i] = __uint_as_float(h);
  lo[i] = __uint_as_float(l);
}
int gib_split_planes(const float* W, float* W_hi, float* W_lo, long long n, gib_stream stream) {
  if (n <= 0) return 0;
  split_planes_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, ST(stream)>>>(W, W_hi, W_lo, n);
  GIB_LAUNCH_CHECK();
  return 0;
}
__global__ void round_plane16_kernel(const float* __restrict__ W, uint16_t* __restrict__ out, long long n, int kind) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint16_t u;
  if (kind == 2) asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(u) : "f"(W[i]));
  else asm("cvt.rn.f16.f32 %0, %1;" : "=h"(u) : "f"(W[i]));
  out[i] = u;
}
int gib_round_plane16(const float* W, void* out, long long n, int kind, gib_stream stream) {
  if (kind != 2 && kind != 3) { set_error("gib_round_plane16: kind %d (2 = bf16, 3 = fp16)", kind); return -2; }
  if (n <= 0) return 0;
  round_plane16_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, ST(stream)>>>(W, reinterpret_cast<uint16_t*>(out), n, kind);
  GIB_LAUNCH_CHECK();
  return 0;
}
size_t gib_dw_scratch_bytes(int M, int Nn, int Kk) { return gemm_dw_scratch_floats(M, Nn, Kk) * sizeof(float); }
int gib_linear_bwd_dw(const float* G, int ldg, int Nn, const float* X, int ldx, int Kk, int M, float* dW, float* dbias,
                      int R, int C, void* scratch, const int* m_dev, const int* base_dev, gib_stream stream) {
  GemmDW q;
  q.G = G; q.ldg = ldg; q.Nn = Nn; q.X = X; q.ldx = ldx; q.Kk = Kk; q.M = M; q.dW = dW; q.dbias = dbias;
  q.R = R; q.C = C; q.Rb = R; q.Rbp = Nn; q.rs = C; q.cs = 1; q.scratch = reinterpret_cast<float*>(scratch);
  q.half_floats = gemm_dw_half_floats(M, Nn, Kk);
  q.m_dev = m_dev; q.base_dev = base_dev;
  GIB_TRY(dw_begin());
  const int rc = gemm_dw(q, ST(stream));
  const int rj = dw_join(ST(stream));
  return rc ? rc : rj;
}
int gib_scatter_sum(float* out, const float* msg, int ld, const int* ptr, const int* ent, const float* w, long long S,
                    gib_stream stream) {
  if (ld & 3) { set_error("gib_scatter_sum: ld must be a multiple of 4"); return -2; }
  return scatter_sum(out, msg, ld, ptr, ent, w, 0, S, ST(stream));
}
int gib_seg_softmax(float* out, const float* EM, const float* EN, int ld, const int* ptr, const int* ent,
                    const float* w, long long S, gib_stream stream) {
  return seg_softmax_fwd(out, EM, EN, ld, ptr, ent, w, S, ST(stream));
}
int gib_gru_gates(float* hn, const float* gi, const float* gh, const float* h, int Hp, const int* ptr, long long S,
                  gib_stream stream) {
  return gru_fwd(hn, gi, gh, h, Hp, ptr, S, nullptr, ST(stream));
}
int gib_graph_gather(float* g, float* att, const float* en, const float* em, int ld, const int* ptr, int N, int B,
                     float big, gib_stream stream) {
  return graph_gather_fwd(g, att, en, em, ld, ptr, N, B, big, ST(stream));
}

}  // extern "C"

// ---- test hooks (include/gib200.h): C-ABI mirrors -> the internal structs, nothing else ----------------------------
static GemmNT to_gemm_nt(const gib_gemm_problem& s) {
  GemmNT p;
  p.A = s.A; p.lda = s.lda; p.B = s.W; p.ldb = s.ldw; p.B_hi = s.W_hi; p.B_lo = s.W_lo;
  p.C = s.C; p.ldc = s.ldc; p.M = s.M; p.N = s.N; p.K = s.K; p.bias = s.bias; p.act = s.act; p.mode = s.mode;
  p.aux = s.aux; p.ldaux = s.ldaux; p.n_store = s.n_store; p.n_valid = s.n_valid;
  p.m_dev = s.m_dev; p.base_dev = s.base_dev; p.tf32 = s.tf32;
  if (s.tf32 >= 2) p.B_lo = nullptr;        // W_hi: the 16-bit plane; W_lo is not read
  return p;
}
static GemmDW to_gemm_dw(const gib_dw_problem& s) {
  GemmDW q;
  q.G = s.G; q.ldg = s.ldg; q.Nn = s.Nn; q.X = s.X; q.ldx = s.ldx; q.Kk = s.Kk; q.M = s.M; q.dW = s.dW;
  q.dbias = s.dbias; q.R = s.R; q.C = s.C; q.Rb = s.Rb; q.Rbp = s.Rbp; q.rs = s.rs; q.cs = s.cs;
  q.m_dev = s.m_dev; q.base_dev = s.base_dev; q.tf32 = s.tf32;
  return q;
}
// both scratch halves, sized as make_bwd sizes them: the largest group (with the same plan rows) and member
static size_t test_dw_scratch_floats(const gib_dw_problem* qs, const int* group_sizes, int n_groups,
                                     long long plan_rows) {
  size_t f = 0;
  int k = 0;
  for (int g = 0; g < n_groups; ++g) {
    GemmDW grp[kTc3MaxProblems];
    const int n = group_sizes[g];
    if (n < 1 || n > kTc3MaxProblems) return 0;
    for (int i = 0; i < n; ++i) grp[i] = to_gemm_dw(qs[k + i]);
    f = std::max(f, 2 * gemm_dw_group_half_floats(grp, n, plan_rows));
    k += n;
  }
  return f;
}

extern "C" {

size_t gib_test_chain_flag_bytes(const gib_gemm_problem* ps, int n) {
  if (n < 1 || n > kTc3MaxProblems) return 0;
  GemmNT p[kTc3MaxProblems];
  for (int i = 0; i < n; ++i) p[i] = to_gemm_nt(ps[i]);
  return tc3_chain_flag_ints(p, n) * sizeof(int);
}
int gib_test_gemm_nt(const gib_gemm_problem* ps, int n, const int* dep, int* flags, gib_stream stream) {
  if (n < 1 || n > kTc3MaxProblems) { set_error("gib_test_gemm_nt: %d problems (1..%d)", n, kTc3MaxProblems); return -2; }
  GemmNT p[kTc3MaxProblems];
  for (int i = 0; i < n; ++i) {
    if (ps[i].tf32 >= 2 && !ps[i].W_hi) {
      set_error("gib_test_gemm_nt: problem %d is bf16 / fp16 but has no 16-bit plane (W_hi, gib_round_plane16)", i);
      return -2;
    }
    p[i] = to_gemm_nt(ps[i]);
  }
  if (!dep) return n == 1 ? gemm_nt(p[0], ST(stream)) : gemm_nt_group(p, n, ST(stream));
  if (!gemm_nt_chain_ok(p, n)) { set_error("gib_test_gemm_nt: the problems do not qualify for a chain"); return -3; }
  return gemm_nt_chain(p, dep, n, flags, ST(stream));
}
size_t gib_test_dw_scratch_bytes(const gib_dw_problem* qs, const int* group_sizes, int n_groups, long long plan_rows) {
  return test_dw_scratch_floats(qs, group_sizes, n_groups, plan_rows) * sizeof(float);
}
int gib_test_dw_groups(const gib_dw_problem* qs, const int* group_sizes, int n_groups, long long plan_rows,
                       void* scratch, gib_stream stream) {
  const size_t floats = test_dw_scratch_floats(qs, group_sizes, n_groups, plan_rows);
  if (n_groups < 1 || floats == 0) { set_error("gib_test_dw_groups: bad group sizes"); return -2; }
  GIB_TRY(dw_begin());
  int rc = 0;
  for (int g = 0, k = 0; g < n_groups && rc == 0; k += group_sizes[g++]) {
    GemmDW grp[kTc3MaxProblems];
    for (int i = 0; i < group_sizes[g]; ++i) {
      grp[i] = to_gemm_dw(qs[k + i]);
      grp[i].scratch = reinterpret_cast<float*>(scratch);
      grp[i].half_floats = floats / 2;
    }
    rc = group_sizes[g] == 1 ? gemm_dw(grp[0], ST(stream)) : gemm_dw_group(grp, group_sizes[g], plan_rows, ST(stream));
  }
  const int rj = dw_join(ST(stream));
  return rc ? rc : rj;
}
int gib_test_scatter_bwd(float* G, const float* dM, const float* Y, int ld, const int* dst, const float* w, int act,
                         long long P, gib_stream stream) {
  return scatter_bwd(G, dM, Y, ld, dst, w, act, P, ST(stream));
}
int gib_test_seg_reduce_dact(float* G, const float* dM, const float* Y, int ld, const int* ptr, const int* ent,
                             const float* row_w, int act, long long rows, gib_stream stream) {
  return seg_reduce_dact(G, dM, Y, ld, ptr, ent, row_w, act, rows, ST(stream));
}
int gib_test_seg_softmax_bwd(float* GM, float* GN, const float* dM, const float* EM, const float* EN, int ld,
                             const int* ptr, const int* ent, const float* w, long long S, gib_stream stream) {
  return seg_softmax_bwd(GM, GN, dM, EM, EN, ld, ptr, ent, w, S, ST(stream));
}
int gib_test_gru_bwd(float* dgi, float* dgh, float* dh, const float* dhn, const float* gi, const float* gh,
                     const float* h, int Hp, const int* ptr, long long S, const int* live, gib_stream stream) {
  return gru_bwd(dgi, dgh, dh, dhn, gi, gh, h, Hp, ptr, S, live, ST(stream));
}
int gib_test_colsum_add(float* out, const float* G, int ldg, long long M, int R, int Rb, int Rbp, const int* live,
                        gib_stream stream) {
  return colsum_add(out, G, ldg, M, R, Rb, Rbp, live, ST(stream));
}
int gib_test_graph_gather_bwd(float* Gen, float* Gem, const float* dg, const float* att, const float* en,
                              const float* em, int ld, int N, int B, gib_stream stream) {
  return graph_gather_bwd(Gen, Gem, dg, att, en, em, ld, N, B, ST(stream));
}
int gib_test_emn_aggregate_fwd(float* msg, const float* EMx, const float* ENx, const float* EMm, const float* ENm,
                               int ld, const int* ent_dst, const int* ent_src, const int* dst_ptr, long long E,
                               const int* live, gib_stream stream) {
  return emn_aggregate_fwd(msg, EMx, ENx, EMm, ENm, ld, ent_dst, ent_src, dst_ptr, E, live, ST(stream));
}
int gib_test_emn_aggregate_bwd(float* dEMx, float* dENx, float* dEMm, float* dENm, float* st3, const float* dmsg,
                               const float* EMx, const float* ENx, const float* EMm, const float* ENm, int ld,
                               const int* ent_dst, const int* ent_src, const int* dst_ptr, const int* src_ptr,
                               const int* src_ent, long long E, const int* live, gib_stream stream) {
  GraphArrays ga{};
  ga.ent_dst = const_cast<int*>(ent_dst); ga.ent_src = const_cast<int*>(ent_src); ga.dst_ptr = const_cast<int*>(dst_ptr);
  ga.src_ptr = const_cast<int*>(src_ptr); ga.src_ent = const_cast<int*>(src_ent);
  return emn_aggregate_bwd(dEMx, dENx, dEMm, dENm, st3, dmsg, EMx, ENx, EMm, ENm, ld, ga, E, live, ST(stream));
}
int gib_test_scatter_sum(float* out, const float* msg, int ld, const int* ptr, const int* ent, const float* w,
                         int accumulate, long long S, gib_stream stream) {
  return scatter_sum(out, msg, ld, ptr, ent, w, accumulate, S, ST(stream));
}
int gib_test_gru_fwd(float* hn, const float* gi, const float* gh, const float* h, int Hp, const int* ptr, long long S,
                     const int* live, gib_stream stream) {
  return gru_fwd(hn, gi, gh, h, Hp, ptr, S, live, ST(stream));
}
int gib_test_gather_rows(float* dst, const float* h, int ld, const int* src, const float* w, int scale, long long P,
                         const int* live, gib_stream stream) {
  return gather_rows(dst, h, ld, src, w, scale, P, live, ST(stream));
}
int gib_test_sum_nodes_fwd(float* g, const float* h, int ld, int N, int B, gib_stream stream) {
  return sum_nodes_fwd(g, h, ld, N, B, ST(stream));
}
int gib_test_bcast_nodes_add(float* dh, const float* dg, int ld, int N, long long S, gib_stream stream) {
  return bcast_nodes_add(dh, dg, ld, N, S, ST(stream));
}
int gib_test_concat2_in(float* dst, int ldd, const void* a, int lda, int wa, int a_i8, const void* b, int ldb, int wb,
                        int b_i8, long long rows, gib_stream stream) {
  return concat2_in(dst, ldd, a, lda, wa, a_i8, b, ldb, wb, b_i8, rows, ST(stream));
}
int gib_test_concat_flat(float* dst, int ldd, const float* f1, int ldf, int N, int fa, const float* g, int ldg, int W,
                         int B, gib_stream stream) {
  return concat_flat(dst, ldd, f1, ldf, N, fa, g, ldg, W, B, ST(stream));
}
int gib_test_unflatten_dact(float* G, int ldf, const float* dcat, int ldd, const float* f1, int N, int fa, long long S,
                            gib_stream stream) {
  return unflatten_dact(G, ldf, dcat, ldd, f1, N, fa, S, ST(stream));
}
int gib_test_dact_slice(float* G, int ldg, const float* dout, const float* out, int ldo, int off, int width, int act,
                        int rows, gib_stream stream) {
  return dact_slice(G, ldg, dout, out, ldo, off, width, act, rows, ST(stream));
}
int gib_test_sum3_cols(float* dst, int ldd, int W, const float* a, int lda, int offa, const float* b2, int ldb,
                       int offb, const float* c3, int ldc, int rows, gib_stream stream) {
  return sum3_cols(dst, ldd, W, a, lda, offa, b2, ldb, offb, c3, ldc, rows, ST(stream));
}
int gib_test_tanh_fwd(float* y, const float* x, long long rows, int ld, const int* live, gib_stream stream) {
  return tanh_fwd(y, x, rows, ld, live, ST(stream));
}
int gib_test_tanh_selu_bwd(float* G, const float* dy, const float* y, const float* pre, long long rows, int ld,
                           const int* live, gib_stream stream) {
  return tanh_selu_bwd(G, dy, y, pre, rows, ld, live, ST(stream));
}
int gib_test_mul_dselu(float* G, const float* d, const float* y, long long rows, int ld, const int* live,
                       gib_stream stream) {
  return mul_dselu(G, d, y, rows, ld, live, ST(stream));
}
int gib_test_emn_input(float* X, int ld, const void* nodes, const void* edges, int i8, const int* ent_dst,
                       const int* ent_src, int N, int F, int Ef, long long P, gib_stream stream) {
  return emn_input(X, ld, nodes, edges, i8, ent_dst, ent_src, N, F, Ef, P, ST(stream));
}
int gib_test_plan_linear(const gib_dims* d, int i, long long* out) {
  Plan pl;
  GIB_TRY(build_plan(*d, pl));
  const int n = (int)pl.lins.size();
  if (i < 0 || i >= n) { set_error("gib_test_plan_linear: Linear %d of %d", i, n); return -2; }
  const Lin& l = pl.lins[i];
  const long long v[GIB_PLAN_LINEAR_FIELDS] = {l.pw, l.pb, l.src_off, l.rs, l.cs, l.nblk, l.Rb, l.Rbp, l.C, l.Cp, l.Ct,
                                               l.Ctp, (long long)l.ow, (long long)l.owt, (long long)l.ob,
                                               (long long)l.ow_hi, (long long)l.ow_lo, (long long)l.owt_hi,
                                               (long long)l.owt_lo};
  memcpy(out, v, sizeof(v));
  return n;
}

}  // extern "C"
