// Host launch wrappers of the HBM-bound kernels (graph_ops.cu).  All return 0 / cudaError_t.
#pragma once
#include "common.cuh"
#include "graph.cuh"

namespace gib {

constexpr int kMaxPackEntries = 96;
struct PackEntry {   // one reference weight (+bias) -> its padded / transposed copies in the packed arena
  const float* W; const float* bias;
  long long rs, cs, ow, owt, ob, ow_hi, ow_lo, owt_hi, owt_lo;
  int nblk, Rb, Rbp, C, Cp, Ct, Ctp;
  unsigned blk_begin;
};
// h16: 0 = the TF32 (hi, lo) planes of Wp / WTp; 1 / 2 = their hi planes and, over the bytes of each lo plane, the
// bf16 / fp16 plane (Wp / WTp rounded to nearest-even, same shape, ld in 16-bit elements) of the 16-bit matmul modes
struct PackTable { int n; unsigned total_blocks; int h16; PackEntry e[kMaxPackEntries]; };
int pack_all(const PackTable& T, float* packed, cudaStream_t st);

int concat2(float* dst, int ldd, const float* a, int lda, int wa, const float* b, int ldb, int wb, long long rows, cudaStream_t st);
int concat2_in(float* dst, int ldd, const void* a, int lda, int wa, int a_i8, const void* b, int ldb, int wb, int b_i8, long long rows, cudaStream_t st);
int concat_flat(float* dst, int ldd, const float* f1, int ldf, int N, int fa, const float* g, int ldg, int W, int B, cudaStream_t st);
int unflatten_dact(float* G, int ldf, const float* dcat, int ldd, const float* f1, int N, int fa, long long S, cudaStream_t st);
int dact_slice(float* G, int ldg, const float* dout, const float* out, int ldo, int off, int width, int act, int rows, cudaStream_t st);
int sum3_cols(float* dst, int ldd, int W, const float* a, int lda, int offa, const float* b2, int ldb, int offb, const float* c3, int ldc, int rows, cudaStream_t st);
// live (may be null): device-side count of the live rows among the `rows` / P / S / E / M rows (EMN bond rows in
// capacity mode, see graph_ops.cu: live_rows); the grid is sized from the capacity, rows past the count are untouched
int tanh_fwd(float* y, const float* x, long long rows, int ld, const int* live, cudaStream_t st);
int tanh_selu_bwd(float* G, const float* dy, const float* y, const float* pre, long long rows, int ld, const int* live, cudaStream_t st);
int gather_rows(float* dst, const float* h, int ld, const int* src, const float* w, int scale, long long P, const int* live, cudaStream_t st);
// bytes: algorithmic bytes of the launch for the profile hooks (0 = unknown)
int scatter_sum(float* out, const float* msg, int ld, const int* ptr, const int* ent, const float* w, int accumulate, long long S, cudaStream_t st, double bytes = 0.0);
extern int g_scatter_variant;
int scatter_bwd(float* G, const float* dM, const float* Y, int ld, const int* dst, const float* w, int act, long long P, cudaStream_t st);
// backward of the message rows (K2 with a fused epilogue): G[u] = row_w[u] * act'(Y[u]) * sum_{q in [ptr[u], ptr[u+1])}
// dM[ent[q]] for rows u < rows (row_w may be null: 1); an empty segment gives exact 0 and Y is not read there
int seg_reduce_dact(float* G, const float* dM, const float* Y, int ld, const int* ptr, const int* ent, const float* row_w, int act, long long rows, cudaStream_t st);
int seg_softmax_fwd(float* out, const float* EM, const float* EN, int ld, const int* ptr, const int* ent, const float* w, long long S, cudaStream_t st);
int seg_softmax_bwd(float* GM, float* GN, const float* dM, const float* EM, const float* EN, int ld, const int* ptr, const int* ent, const float* w, long long S, cudaStream_t st);
int gru_fwd(float* hn, const float* gi, const float* gh, const float* h, int Hp, const int* ptr, long long S, const int* live, cudaStream_t st);
int gru_bwd(float* dgi, float* dgh, float* dh_direct, const float* dhn, const float* gi, const float* gh, const float* h, int Hp, const int* ptr, long long S, const int* live, cudaStream_t st);
int colsum_add(float* out, const float* G, int ldg, long long M, int R, int Rb, int Rbp, const int* live, cudaStream_t st);
int graph_gather_fwd(float* g, float* att, const float* en, const float* em, int ld, const int* ptr, int N, int B, float big, cudaStream_t st);
int graph_gather_bwd(float* Gen, float* Gem, const float* dg, const float* att, const float* en, const float* em, int ld, int N, int B, cudaStream_t st);
int sum_nodes_fwd(float* g, const float* h, int ld, int N, int B, cudaStream_t st);
int bcast_nodes_add(float* dh, const float* dg, int ld, int N, long long S, cudaStream_t st);
int emn_input(float* X, int ld, const void* nodes, const void* edges, int i8, const int* ent_dst, const int* ent_src, int N, int F, int Ef, long long P, cudaStream_t st);
int emn_aggregate_fwd(float* msg, const float* EMx, const float* ENx, const float* EMm, const float* ENm, int ld, const int* ent_dst, const int* ent_src, const int* dst_ptr, long long E, const int* live, cudaStream_t st);
int emn_aggregate_bwd(float* dEMx, float* dENx, float* dEMm, float* dENm, float* st3, const float* dmsg, const float* EMx, const float* ENx, const float* EMm, const float* ENm, int ld, const GraphArrays& ga, long long E, const int* live, cudaStream_t st);
int mul_dselu(float* G, const float* d, const float* y, long long rows, int ld, const int* live, cudaStream_t st);
int pack_weight(float* Wp, float* WTp, float* bp, const float* W, const float* bias, long long rs, long long cs, int nblk, int Rb, int Rbp, int C, int Cp, int Ct, int Ctp, cudaStream_t st);

// The categorical sampler (api.cu).  gate != null (gib_generation_sample_round, generate.cu): the round index and the
// loop condition are read from device memory.  state = {next round, status}; a call runs when counters[0] < B,
// status == 0 and state[0] < rounds, samples row state[0] of uniforms [rounds, B] and leaves state[0] in ctl[0]
// (-1 when it does not run: the round kernels then do nothing).  A call that finds state[0] >= rounds while
// counters[0] < B sets status 1.  actions != null ([rounds, B]): a running call takes row state[0] of it as the
// draw instead of sampling, and leaves `lik` untouched.
struct RoundGate { int* state; const int* counters; int* ctl; int rounds; const int* actions; };
int sample_actions_launch(const float* out, int B, int apd, const float* uniforms, int* action, float* lik,
                          const RoundGate* gate, cudaStream_t st);

// RL rollout (rl.cu): for every slot b of a running round r = ctl[0] (ctl[0] < 0: nothing), the softmax
// probability of action[b] under logits_a / logits_b [B, apd] into p_a / p_b[r, b], action[b] into act_rec[r, b], and
// the slot tag b + 1 into tags[b] (the "likelihood" the round kernels store: the (molecule, round) -> slot map)
int rl_probs_launch(const float* logits_a, const float* logits_b, int B, int apd, const int* action, const int* ctl,
                    int* act_rec, float* p_a, float* p_b, float* tags, cudaStream_t st);

}  // namespace gib
