/*
 * gib200 -- C-ABI of the H100-native GraphINVENT MPNN hot path (libgib200.so).
 *
 * The reference has no FFI layer: its boundary for this path is the Python
 * `torch.nn.Module` protocol (`gnn.mpnn.{MNN,GGNN,AttentionGGNN,EMN}(constants)`,
 * `forward(nodes, edges) -> logits`, SURVEY.md §8b).  The drop-in modules in
 * `graphinvent_b200/gnn/` keep that protocol and bind the entry points below through
 * ctypes (INTEGRATION.md shows the stub).  Each entry point names the reference code
 * it replaces (paths relative to /root/reference/graphinvent/).
 *
 * Conventions
 *  - every pointer except `hdr_host`, `params` / `grads` (host arrays of device pointers)
 *    and `dims` is a DEVICE pointer owned by the caller (PyTorch caching allocator:
 *    `tensor.data_ptr()`); the library never allocates or frees device memory -- sizes come
 *    from the *_bytes() queries;
 *  - `stream` is a cudaStream_t (`torch.cuda.current_stream().cuda_stream`); every call is
 *    asynchronous on it and performs no host synchronisation (the exact-size mode needs ONE 64-byte header read
 *    by the caller between gib_graph_count and gib_graph_fill; capacity mode needs none);
 *  - return value: 0 ok, < 0 invalid argument (see gib_last_error()), > 0 a cudaError_t;
 *  - nothing is thrown across the boundary.  Library state: the thread-local error string, a per-device helper
 *    stream for the split reductions (joined back into `stream` before a call returns) and per-device caches of
 *    function attributes / TMA descriptors (mutex-guarded).  One host thread drives one device's model at a time
 *    (the reference's threading model, SURVEY.md 8b); different devices are independent;
 *  - all reductions run in a fixed order (no float atomics): results are bit-stable.
 *
 * Tensor layouts (reference `BlockDatasetLoader.py:135-143`, SURVEY.md §8b):
 *    nodes  float32 [B, N, F]        dense, zero padded
 *    edges  float32 [B, N, N, Ef]    dense, zero padded, dst = row i, src = column j
 *    out    float32 [B, N*f_add + N*f_conn + 1]   un-normalised (SELU-activated) APD logits
 */
#ifndef GIB200_H
#define GIB200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* gib_stream; /* cudaStream_t */

enum { GIB_GGNN = 0, GIB_MNN = 1, GIB_ATTGGNN = 2, GIB_EMN = 3 };

/* Hyper-parameters the reference reads from `constants` (SURVEY.md §5 config row). */
typedef struct gib_dims {
  int model;                       /* GIB_* */
  int B, N, F, Ef;                 /* batch, max_n_nodes, n_node_features, n_edge_features */
  int H, M, T;                     /* hidden_node_features, message_size, message_passes
                                      (EMN: H = M = edge_emb_size) */
  int msg_hidden, msg_depth;       /* GGNN: enn_*;  AttGGNN / EMN: msg_* */
  int att_hidden, att_depth;       /* AttGGNN / EMN: att_* */
  int eemb_hidden, eemb_depth;     /* EMN: edge_emb_* */
  int gather_width, gatt_hidden, gatt_depth, gemb_hidden, gemb_depth;
  int mlp1_hidden, mlp1_depth, mlp2_hidden, mlp2_depth;
  int f_add, f_conn;               /* len_f_add_per_node, len_f_conn_per_node */
  float big;                       /* constants.big_positive (1e6) */
  int in_dtype;                    /* element type of `nodes` / `edges`: 0 = float32 (BlockDatasetLoader.py:139-143),
                                      1 = int8, the reference's on-disk type (DataProcesser.py:157-161), read
                                      directly by K0 and the first-layer kernels */
  /* tf32: precision of the tensor-core GEMMs that gib_model_forward, gib_model_backward and gib_model_backward_part
   * launch: 0 = 3xTF32, fp32-accurate; 1 = single-pass TF32, the hi*hi term of the 3xTF32 split alone (both operands
   * rounded to TF32 to nearest, fp32 accumulation): the precision torch gives a CUDA fp32 matmul when its fp32_precision
   * is "tf32".  The fp32 SIMT GEMMs (narrow APD output layers, small exact-mode problems) and every non-GEMM kernel are
   * fp32 in both modes.  2 = bf16, 3 = fp16 (torch.autocast): every tensor-core GEMM operand (activations, output
   * gradients, inputs, weights) rounded to nearest-even to 16 bits, as tensor.to(torch.bfloat16 / torch.float16)
   * rounds, fp32 accumulation; an fp16 operand beyond +-65504 becomes +-inf as torch's cast makes it.  The SIMT GEMMs,
   * the bias-gradient sums, every other kernel and every buffer stay fp32.  gib_model_pack also reads it: in the 16-bit
   * modes it writes the 16-bit planes of the weights over the bytes of their TF32 lo planes (the arena size is the
   * same), so an arena packed in a 16-bit mode serves that mode only.  Other codes are refused, and so is a 16-bit code
   * when the tensor cores are off (gib_set_tensor_cores) or gib_tc_debug bit 0 is set.  K0 and every size query ignore
   * it: no size, workspace or packed-weight layout depends on it. */
  int tf32;
} gib_dims;

/* Graph header: 16 ints written on the device by gib_graph_count() at the start of its workspace.
 * Exact mode: the caller copies them to the host (the one D2H read of a forward) and passes them back as `hdr_host`;
 * buffers are then sized exactly.  Capacity mode: the caller never reads them -- gib_graph_header_capacity() builds a
 * host header that carries static capacities and the ADDRESS of the device header, every kernel whose extent depends
 * on the batch content (the per-bond-type GEMM row ranges, the split counts of the weight-gradient reductions, and for
 * the EMN every kernel over bond rows) reads the live counts from device memory, and no launch parameter depends on
 * the batch: a step has no host synchronisation and is capturable in a CUDA graph.  All four models support it.
 * Index meaning: */
enum {
  GIB_HDR_E = 0,          /* bond entries (non-zero elements of `edges`) */
  GIB_HDR_P = 1,          /* rows of the type-grouped entry arrays (groups padded to 128) */
  GIB_HDR_TYPE_COUNT = 2, /* [4] */
  GIB_HDR_TYPE_BASE = 6,  /* [5] */
  GIB_HDR_FLAGS = 11,     /* bit0: a bond with >1 non-zero type; bit1: a bond value != 1; bit2: the batch exceeds the
                             capacity (capacity mode; results of that step are invalid, nothing is written out of bounds) */
  GIB_HDR_CAPACITY = 12,  /* host header only: != 0 = capacity header (E, P are capacities) */
  GIB_HDR_DEV_LO = 13,    /* host header only: address of the device header, low / high 32 bits */
  GIB_HDR_DEV_HI = 14,
  GIB_HDR_INTS = 16
};

const char* gib_last_error(void);
int gib_version(void);
/* tensor-core 3xTF32 GEMM path on (default) / off (fp32 SIMT GEMMs only); process-wide switch */
void gib_set_tensor_cores(int on);
int gib_get_tensor_cores(void);
/* bit 3: GGNN / MNN message MLPs on one row per bond entry (the AttentionGGNN's layout) instead of one per message row.
 * bit 2: narrow outputs (N < 48, the APD heads) on the tensor-core kernel too (default: fp32 SIMT, see gemm_simt.cu).
 * bit 1: no dependent-chain launches (every MLP layer its own launch).
 * bit 0: per-problem call pattern: no grouped or chained tensor-core launches, raw weights split inside the kernel,
 * single-problem weight gradients with the bias column sums on the side stream; process-wide, A/B measurements only.
 * Capacity mode needs the default. */
void gib_tc_debug(int mode);
/* K2 scatter-aggregate variant (A/B measurements): bit 0 = two slots per thread, bit 1 = streaming cache hints;
 * default 2 (the fastest at the C4 shape).  Results are identical across variants. */
void gib_scatter_variant(int v);
/* diagnosis: while device_buf != NULL, CTA 0 of every tensor-core GEMM launch writes clock64 stamps of its first
 * `tiles` work items into device_buf[tile][16] (int64): 0 work item started, 6 tile stored (tools/tc3_trace.py) */
void gib_tc_trace(long long* device_buf, int tiles);
/* streaming multiprocessors of the current device (grid sizing of the persistent kernels) */
int gib_device_sm_count(void);

/* ---- K0: edges -> bond entries + CSR.  Replaces summation_mpnn.py:102-118,
 *      aggregation_mpnn.py:105-148, edge_mpnn.py:104-173. ------------------------------- */
size_t gib_graph_count_ws_bytes(const gib_dims* d);
int gib_graph_count(const gib_dims* d, const void* edges, void* count_ws, gib_stream stream);
/* capacity mode: host header for `entry_capacity` bond entries (no device access; valid as long as count_ws lives) */
int gib_graph_header_capacity(const gib_dims* d, int entry_capacity, const void* count_ws, int* hdr_host_out);
size_t gib_graph_bytes(const gib_dims* d, const int* hdr_host);
int gib_graph_fill(const gib_dims* d, const void* edges, void* count_ws, const int* hdr_host, void* graph_buf,
                   gib_stream stream);
/* device addresses of the arrays inside graph_buf, for tests / standalone kernel calls:
 * which = 0 ent_src, 1 ent_dst, 2 ent_w, 3 dst_ptr, 4 dst_ent, 5 src_ptr, 6 src_ent */
void* gib_graph_array(const gib_dims* d, const int* hdr_host, void* graph_buf, int which);

/* ---- parameters: state_dict order of the reference (SURVEY.md Appendix A) ------------- */
int gib_model_num_params(const gib_dims* d);
long long gib_model_param_numel(const gib_dims* d, int index);
size_t gib_model_packed_bytes(const gib_dims* d);
/* zero-padded + transposed copies of every weight (and 3xTF32 splits when enabled) */
int gib_model_pack(const gib_dims* d, const float* const* params, void* packed, gib_stream stream);

/* ---- whole-model forward / backward.  Replaces SummationMPNN.forward
 *      (summation_mpnn.py:80-149), AggregationMPNN.forward (aggregation_mpnn.py:83-168),
 *      EdgeMPNN.forward (edge_mpnn.py:82-192), the model bodies in mpnn.py and
 *      GraphGather / GlobalReadout (modules.py:39-52, 237-281), and their autograd. ------- */
size_t gib_model_workspace_bytes(const gib_dims* d, const int* hdr_host);
int gib_model_forward(const gib_dims* d, const int* hdr_host, const void* nodes, const void* edges,
                      const void* graph_buf, const void* packed, void* workspace, float* out,
                      gib_stream stream);
/* GGNN / MNN: device addresses of the message-row table the forward builds in `workspace` (one message row per
 * (molecule, source atom, bond type) for the bond entries of value 1, one per other entry; layout in
 * graphinvent_b200/csrc/graph.cuh, MsgRows), for tests: which = 0 u_src [P], 1 u_w [P] (float), 2 u_ptr [P+1],
 * 3 u_dst [E], 4 ent_u [P], 5 dst_u [E], 6 s_ptr [S+1], 7 s_u [E], 8 meta [16], 9 build scratch.  NULL for the other
 * models or a bad `which`. */
void* gib_model_msg_rows(const gib_dims* d, const int* hdr_host, void* workspace, int which);
size_t gib_model_bwd_scratch_bytes(const gib_dims* d, const int* hdr_host);
/* The backward in two parts on the same scratch: part 1 = readout only -- afterwards the gradients of the gather.* and
 * APDReadout.* parameters (the tail of the parameter order, 79 % of the bytes) are final and a data-parallel caller
 * can start their all-reduce; part 2 = the message passes; part 0 = both (== gib_model_backward). */
int gib_model_backward_part(const gib_dims* d, const int* hdr_host, const void* nodes, const void* edges,
                            const void* graph_buf, const void* packed, const void* workspace, const float* out,
                            const float* dout, float* const* grads, void* scratch, int part, gib_stream stream);
/* grads[i] (same order / shapes as params) are ACCUMULATED into (+=). */
int gib_model_backward(const gib_dims* d, const int* hdr_host, const void* nodes, const void* edges,
                       const void* graph_buf, const void* packed, const void* workspace,
                       const float* out, const float* dout, float* const* grads, void* scratch,
                       gib_stream stream);

/* ---- call-site post-ops (Workflow.py:833-860): KLDivLoss(batchmean)(log_softmax(out),
 *      target / sum(target)) and its gradient w.r.t. `out`, one kernel.
 *      loss_rows[b] = per-molecule KL (sum and divide by B on the caller side or pass
 *      inv_scale); dout = (softmax(out) - t_hat) * grad_scale. ---------------------------- */
int gib_kl_loss_fwd_bwd(const float* out, const float* target, int B, int apd, float grad_scale,
                        float* loss_rows, float* dout, gib_stream stream);

/* out[0] = scale * sum(rows[0..n)) in a fixed order (the batch mean of loss_rows), and a plain asynchronous memset:
 * the two non-model operations of a captured training step (graphinvent_b200/graphed.py) */
int gib_sum_scaled(const float* rows, int n, float scale, float* out, gib_stream stream);
int gib_fill_zero(void* ptr, size_t bytes, gib_stream stream);

/* ---- validation NLL of the "correct" actions (Analyzer.get_validation_likelihood, Analyzer.py:744-758), one kernel:
 *      nll[b] = -log( sum_k softmax(out[b])_k * target[b,k] / sum_k target[b,k] ).  Rows with an all-zero target
 *      give NaN (the reference drops them afterwards, Analyzer.py:756). -------------------------------------- */
int gib_validation_nll(const float* out, const float* target, int B, int apd, float* nll, gib_stream stream);

/* ---- partial batches of a captured step: the live molecule count and the loss scale of the batch in the static
 *      buffers, in DEVICE memory, written by the host before each replay.  The _ctl forms below take `ctl` instead of
 *      a host scale; rows b >= ctl->live are padding: their loss / NLL row is +0 and their dout row is zero.  On a
 *      batch with live == B they compute exactly what the host-argument forms compute with scale == ctl->scale. */
typedef struct gib_batch_ctl {
  int live;       /* molecules [0, live) of the B rows are real */
  float scale;    /* gradient and sum scale (1 / the batch-mean's denominator) */
} gib_batch_ctl;
int gib_kl_loss_fwd_bwd_ctl(const float* out, const float* target, int B, int apd, const gib_batch_ctl* ctl,
                            float* loss_rows, float* dout, gib_stream stream);   /* dout may be NULL */
/* gib_kl_loss_fwd_bwd_ctl with dynamic loss scaling: every dout value it writes is multiplied once more, by the
 * DEVICE float *loss_scale (a torch.amp.GradScaler's scale; autograd's `dout * scale` of scaler.scale(loss)).  The
 * loss rows are not scaled.  ctl and loss_scale must be non-NULL. */
int gib_kl_loss_fwd_bwd_ctl_scaled(const float* out, const float* target, int B, int apd, const gib_batch_ctl* ctl,
                                   const float* loss_scale, float* loss_rows, float* dout, gib_stream stream);
/* out[0] = ctl->scale * sum(rows[0..min(n, ctl->live))), the order gib_sum_scaled uses for those rows */
int gib_sum_scaled_ctl(const float* rows, int n, const gib_batch_ctl* ctl, float* out, gib_stream stream);
int gib_validation_nll_ctl(const float* out, const float* target, int B, int apd, const gib_batch_ctl* ctl,
                           float* nll, gib_stream stream);

/* ---- the per-batch tail of a validation pass (Workflow.validation_epoch, Workflow.py:813-831, and
 *      Analyzer.get_validation_likelihood, Analyzer.py:734-778), one CTA.  `pass` is DEVICE memory; with
 *      i = pass->idx (the batch cursor) and L = ctl->live:
 *        batch_loss[i] = sum_{b<L} kl_rows[b] / L      when batch_loss != NULL and 0 <= i < n_slots (KLDivLoss batchmean)
 *        lik[i*B + j] = j-th non-NaN nll_rows[b], b < L, in order   when lik != NULL; positions >= lik_len are not
 *                       written and counted in `clipped` (the reference's slice assignment raises there)
 *        n_structures += sum_{b<L} target[b, apd-1]
 *        flags |= count_ws[GIB_HDR_FLAGS]              (the batch's K0 header)
 *        idx += 1
 *      Every sum runs in a fixed order. */
typedef struct gib_eval_pass {
  float* batch_loss;
  float* lik;
  long long lik_len;
  int n_slots;
  int idx;
  float n_structures;
  int flags;
  int clipped;
  int reserved;
} gib_eval_pass;
int gib_eval_collect(const float* kl_rows, const float* nll_rows, const float* target, int B, int apd,
                     const gib_batch_ctl* ctl, const void* count_ws, gib_eval_pass* pass, gib_stream stream);

/* ---- one batch from a device-resident block of int8 rows (graphinvent_b200/loader.py, DeviceBlockLoader; replaces
 *      BlockDatasetLoader.py's ShuffleBlockWrapper indexing, default collate and the three host-to-device copies of
 *      Workflow.train_epoch, Workflow.py:781-783).  nodes [*, row_nodes], edges [*, row_edges], apds [*, apd]: the
 *      block, row-major int8.  For r < b, output row r is block row rows[r]: out_nodes / out_edges as int8
 *      (out_dtype 1) or widened to float32 (out_dtype 0), out_target always float32 widened from signed int8 (as
 *      HDFDataset.__getitem__'s .type(torch.float32)).  Rows b <= r < B are zero (empty molecules).  ctl, when not
 *      NULL, is set to {b, b > 0 ? float32(1.0 / b) : 0}.  One launch; rows[] must index the block (the loader makes
 *      them).  Block and output pointers must be 16-byte aligned; b > B, non-positive dims, null pointers and an
 *      unknown out_dtype are refused. */
int gib_gather_rows(const signed char* nodes, const signed char* edges, const signed char* apds, const int* rows,
                    int b, int B, int row_nodes, int row_edges, int apd, void* out_nodes, void* out_edges,
                    int out_dtype, float* out_target, gib_batch_ctl* ctl, gib_stream stream);   /* ctl may be NULL */

/* ---- flat-bucket Adam step: replaces torch.optim.Adam.step() on the model parameters (constructed at
 *      Workflow.py:191,221,245, stepped at Workflow.py:795-796; same update rule, L2 weight decay, no amsgrad)
 *      with ONE launch over contiguous params / grads / exp_avg / exp_avg_sq of n floats.  `step` is the
 *      1-based update count (bias corrections are evaluated in double on the host, as the reference does in
 *      Python floats); grads are multiplied by grad_scale first (1/world when the bucket holds an all-reduce
 *      sum).  The four buffers must share their address modulo 16 bytes. ------------------------------------ */
int gib_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                  long long step, double lr, double beta1, double beta2, double eps, double weight_decay,
                  double grad_scale, gib_stream stream);

/* ---- dynamic loss scaling on the device: torch.amp.GradScaler's `step(optimizer); update()` without a host read.
 *      All scalars are DEVICE memory.
 *      gib_nonfinite_check: *found_inf = 1.0f if any of x[0, n) is inf or NaN (the check of
 *        torch._amp_foreach_non_finite_check_and_unscale_); it never clears *found_inf.
 *      gib_adam_step_scaled: gib_adam_step gated on *found_inf -- nothing is written when it is non-zero -- with the
 *        gradients multiplied by (float)(1 / (double)*scale) before grad_scale (GradScaler.unscale_) and the step
 *        taken as *step_count + 1 (bias corrections in double on the device).  It does not advance *step_count.
 *      gib_amp_update_scale: torch._amp_update_scale_ on (*scale, *growth_tracker) from *found_inf, and, when
 *        *found_inf is zero, step_counts[0, n_counts) += 1 (the counts of the optimizer gated on it). */
int gib_nonfinite_check(const float* x, long long n, float* found_inf, gib_stream stream);
int gib_adam_step_scaled(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                         const long long* step_count, const float* found_inf, const float* scale, double lr,
                         double beta1, double beta2, double eps, double weight_decay, double grad_scale,
                         gib_stream stream);
int gib_amp_update_scale(float* scale, int* growth_tracker, const float* found_inf, double growth_factor,
                         double backoff_factor, int growth_interval, long long* step_counts, int n_counts,
                         gib_stream stream);

/* ---- single kernels (unit tests, ncu evidence, reuse) --------------------------------- */
/* Y = act(X W^T + b); X [M, ldx], W packed [Np, Kp] (ldw), Y [M, ldy]; act 0 none / 1 selu / 2 tanh */
int gib_linear_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias, float* Y, int ldy,
                   int M, int N, int K, int act, gib_stream stream);
/* same contract, forced onto the tensor-core 3xTF32 kernel regardless of the size heuristics */
int gib_linear_fwd_tc(const float* X, int ldx, const float* W, int ldw, const float* bias, float* Y, int ldy,
                      int M, int N, int K, int act, gib_stream stream);
/* the model's own call pattern: W arrives as its TF32 hi / lo planes (hi = rna(W), lo = rna(W - hi), as
 * gib_model_pack lays them out), only X is split in the kernel.  m_dev / base_dev (device ints, may be NULL): the live
 * row range [*base_dev, *base_dev + *m_dev) inside buffers of M rows (capacity mode). */
int gib_linear_fwd_tc_planes(const float* X, int ldx, const float* W_hi, const float* W_lo, int ldw,
                             const float* bias, float* Y, int ldy, int M, int N, int K, int act,
                             const int* m_dev, const int* base_dev, gib_stream stream);
/* TF32 hi / lo planes of a row-major matrix (round-to-nearest split), for callers of the entry above */
int gib_split_planes(const float* W, float* W_hi, float* W_lo, long long n, gib_stream stream);
/* the 16-bit plane of n fp32 values (kind 2 = bf16, 3 = fp16: the gib_dims.tf32 codes), rounded to nearest-even
 * as gib_model_pack rounds them, into n 16-bit values at out -- the W_hi of a 16-bit test-hook problem */
int gib_round_plane16(const float* W, void* out, long long n, int kind, gib_stream stream);
/* dW[R,C] += G^T X, dbias[R] += colsum(G); G [M, ldg], X [M, ldx]; scratch from gib_dw_scratch_bytes */
size_t gib_dw_scratch_bytes(int M, int Nn, int Kk);
int gib_linear_bwd_dw(const float* G, int ldg, int Nn, const float* X, int ldx, int Kk, int M, float* dW,
                      float* dbias, int R, int C, void* scratch, const int* m_dev, const int* base_dev,
                      gib_stream stream);
/* K2 scatter-aggregate: out[s,:] = sum_{q in [ptr[s],ptr[s+1])} w[ent[q]] * msg[ent[q],:]   (w may be NULL) */
int gib_scatter_sum(float* out, const float* msg, int ld, const int* ptr, const int* ent, const float* w,
                    long long S, gib_stream stream);
/* K2' segmented softmax-aggregate (AttentionGGNN) */
int gib_seg_softmax(float* out, const float* EM, const float* EN, int ld, const int* ptr, const int* ent,
                    const float* w, long long S, gib_stream stream);
/* GRU gates: hn = GRU(gi, gh, h) on rows whose CSR segment is non-empty (ptr may be NULL) */
int gib_gru_gates(float* hn, const float* gi, const float* gh, const float* h, int Hp, const int* ptr,
                  long long S, gib_stream stream);
/* GraphGather softmax readout */
int gib_graph_gather(float* g, float* att, const float* en, const float* em, int ld, const int* ptr, int N,
                     int B, float big, gib_stream stream);

/* ---- test hooks: thin entries into the GEMM dispatchers and the backward / EMN kernels the model calls, so that each
 *      can be checked on its own against a float64 reference (tests/test_gpu_gemm_patterns.py,
 *      tests/test_gpu_graph_kernels.py, tests/test_gpu_forward_kernels.py).  Each entry calls the internal function the model calls and adds no path of its
 *      own.  `ps`, `dep`, `qs` and `group_sizes` are HOST arrays; everything they point to lives on the device. ---- */
/* one NT problem: C[M, :n_store] = epi(A[M,K] W[N,K]^T) with A, W row-major, K % 16 == 0, lda / ldb % 4 == 0;
 * epi (mode): 0 act(acc + bias), 1 acc * act'(aux) (aux = the activation OUTPUT), 2 acc + aux (aux may alias C);
 * act 0 none / 1 selu / 2 tanh.  Columns [n_valid, n_store) are stored as zeros, columns >= n_store are not touched.
 * W_hi / W_lo (may be NULL): its TF32 planes (gib_split_planes).  m_dev / base_dev (may be NULL): the live row range
 * [*base_dev, *base_dev + *m_dev) inside buffers of M rows.  tf32: precision of the tensor-core kernels (0 = 3xTF32,
 * 1 = single-pass TF32, as gib_dims.tf32; W then read from W_hi only, or raw W rounded in the kernel; 2 / 3 =
 * bf16 / fp16: W_hi then points at the 16-bit plane (gib_round_plane16, ldw in its elements, a multiple of 8 for the
 * tensor-core path) and W_lo is ignored; a 16-bit problem without W_hi is refused); the problems of one call must
 * agree. */
typedef struct gib_gemm_problem {
  const float* A; int lda;
  const float* W; int ldw;
  const float* W_hi; const float* W_lo;
  float* C; int ldc;
  int M, N, K;
  const float* bias;
  int act, mode;
  const float* aux; int ldaux;
  int n_store, n_valid;
  const int* m_dev; const int* base_dev;
  int tf32;
} gib_gemm_problem;
/* dep == NULL: the n problems as the model launches independent siblings (one problem: the single-GEMM dispatcher,
 * n <= 4: one grouped tensor-core launch when they qualify, else problem by problem).  dep != NULL: ONE dependent-chain
 * launch in which problem i reads as its A operand what problem dep[i] < i stores (-1: independent); returns < 0
 * without launching when the problems do not qualify for a chain.  flags: >= gib_test_chain_flag_bytes(ps, n). */
size_t gib_test_chain_flag_bytes(const gib_gemm_problem* ps, int n);
int gib_test_gemm_nt(const gib_gemm_problem* ps, int n, const int* dep, int* flags, gib_stream stream);
/* one weight-gradient problem: dW[r*rs + c*cs] += sum_m G[m, prow(r)] X[m, c], dbias[r] += sum_m G[m, prow(r)]
 * (either may be NULL) for r < R, c < C, prow(r) = (r / Rb) * Rbp + r % Rb; G [M, Nn] (ldg), X [M, Kk] (ldx); tf32 as in
 * gib_gemm_problem (the bias sums stay fp32 sums of G); the members of one group must agree */
typedef struct gib_dw_problem {
  const float* G; int ldg; int Nn;
  const float* X; int ldx; int Kk;
  int M;
  float* dW; float* dbias;
  int R, C, Rb, Rbp;
  long long rs, cs;
  const int* m_dev; const int* base_dev;
  int tf32;
} gib_dw_problem;
/* n_groups consecutive groups of group_sizes[g] (<= 16) problems, each run as the model runs the weight gradients of one
 * layer (one grouped tensor-core launch + one side-stream reduction when it qualifies), all on ONE scratch whose two
 * halves alternate between groups; plan_rows: the expected reduction rows of a group (0: the sum of its M).  The
 * members of one group write disjoint destinations; different groups may add into the same ones. */
size_t gib_test_dw_scratch_bytes(const gib_dw_problem* qs, const int* group_sizes, int n_groups, long long plan_rows);
int gib_test_dw_groups(const gib_dw_problem* qs, const int* group_sizes, int n_groups, long long plan_rows,
                       void* scratch, gib_stream stream);
/* G[p] = w[p] * dM[dst[p]] * act'(Y[p]) (rows with dst[p] < 0: zeros) */
int gib_test_scatter_bwd(float* G, const float* dM, const float* Y, int ld, const int* dst, const float* w, int act,
                         long long P, gib_stream stream);
/* backward of the message rows: G[u] = row_w[u] * act'(Y[u]) * sum_{q in [ptr[u], ptr[u+1])} dM[ent[q]] (row_w may be
 * NULL: 1; rows with an empty segment: zeros, Y not read), with the variant gib_scatter_variant selects; ld % 4 == 0 */
int gib_test_seg_reduce_dact(float* G, const float* dM, const float* Y, int ld, const int* ptr, const int* ent,
                             const float* row_w, int act, long long rows, gib_stream stream);
/* backward of gib_seg_softmax with SELU outputs EM / EN; GM / GN rows in no segment are not written */
int gib_test_seg_softmax_bwd(float* GM, float* GN, const float* dM, const float* EM, const float* EN, int ld,
                             const int* ptr, const int* ent, const float* w, long long S, gib_stream stream);
/* backward of gib_gru_gates; h == NULL: h = 0 and gh is one bias row (the EMN form); live (may be NULL): device count
 * of the rows to process, rows past it are not touched */
int gib_test_gru_bwd(float* dgi, float* dgh, float* dh, const float* dhn, const float* gi, const float* gh,
                     const float* h, int Hp, const int* ptr, long long S, const int* live, gib_stream stream);
/* out[r] += sum over the first min(*live, M) rows m of G[m, prow(r)] (live may be NULL: all M rows) */
int gib_test_colsum_add(float* out, const float* G, int ldg, long long M, int R, int Rb, int Rbp, const int* live,
                        gib_stream stream);
/* backward of gib_graph_gather at its stored attention `att`, SELU outputs en / em */
int gib_test_graph_gather_bwd(float* Gen, float* Gem, const float* dg, const float* att, const float* en,
                              const float* em, int ld, int N, int B, gib_stream stream);
/* EMN line-graph aggregation over the bond entries (ordered by destination: ent_dst ascending) and its two-pass
 * backward: dEMx / dENx are accumulated (+=), dEMm / dENm stored; st3 is a [3, E, ld] stash; rows >= *live untouched */
int gib_test_emn_aggregate_fwd(float* msg, const float* EMx, const float* ENx, const float* EMm, const float* ENm,
                               int ld, const int* ent_dst, const int* ent_src, const int* dst_ptr, long long E,
                               const int* live, gib_stream stream);
int gib_test_emn_aggregate_bwd(float* dEMx, float* dENx, float* dEMm, float* dENm, float* st3, const float* dmsg,
                               const float* EMx, const float* ENx, const float* EMm, const float* ENm, int ld,
                               const int* ent_dst, const int* ent_src, const int* dst_ptr, const int* src_ptr,
                               const int* src_ent, long long E, const int* live, gib_stream stream);
/* forward and glue kernels (tests/test_gpu_forward_kernels.py).  live (may be NULL): device count of the rows to
 * process, clamped to the row count; rows past it are not touched.
 * scatter_sum: out[s] (+= when accumulate) sum_{q in [ptr[s], ptr[s+1])} w[ent[q]] msg[ent[q]] (w may be NULL: 1),
 * with the variant gib_scatter_variant selects; ld % 4 == 0 */
int gib_test_scatter_sum(float* out, const float* msg, int ld, const int* ptr, const int* ent, const float* w,
                         int accumulate, long long S, gib_stream stream);
/* gib_gru_gates with a live count (h == NULL: h = 0 and gh is one bias row, the EMN form) */
int gib_test_gru_fwd(float* hn, const float* gi, const float* gh, const float* h, int Hp, const int* ptr, long long S,
                     const int* live, gib_stream stream);
/* dst[p] = (scale && w ? w[p] : 1) * h[src[p]] (src[p] < 0: zeros); ld % 4 == 0 */
int gib_test_gather_rows(float* dst, const float* h, int ld, const int* src, const float* w, int scale, long long P,
                         const int* live, gib_stream stream);
/* g[b] = sum_i h[b*N + i] (MNN readout) and its backward dh[s] += dg[s / N] */
int gib_test_sum_nodes_fwd(float* g, const float* h, int ld, int N, int B, gib_stream stream);
int gib_test_bcast_nodes_add(float* dh, const float* dg, int ld, int N, long long S, gib_stream stream);
/* dst[r] = [a[r, :wa] | b[r, :wb] | 0] over ldd columns; a / b int8 when a_i8 / b_i8 */
int gib_test_concat2_in(float* dst, int ldd, const void* a, int lda, int wa, int a_i8, const void* b, int ldb, int wb,
                        int b_i8, long long rows, gib_stream stream);
/* dst[b] = [f1[b*N + 0, :fa] | ... | f1[b*N + N-1, :fa] | g[b, :W] | 0] over ldd columns */
int gib_test_concat_flat(float* dst, int ldd, const float* f1, int ldf, int N, int fa, const float* g, int ldg, int W,
                         int B, gib_stream stream);
/* G[s, a] = dcat[s / N, (s % N)*fa + a] * selu'(f1[s, a]) for a < fa, 0 up to ldf */
int gib_test_unflatten_dact(float* G, int ldf, const float* dcat, int ldd, const float* f1, int N, int fa, long long S,
                            gib_stream stream);
/* G[m, n] = dout[m, off + n] * act'(out[m, off + n]) for n < width, 0 up to ldg (act: the activation OUTPUT) */
int gib_test_dact_slice(float* G, int ldg, const float* dout, const float* out, int ldo, int off, int width, int act,
                        int rows, gib_stream stream);
/* dst[r, c] = a[r, offa + c] + b2[r, offb + c] + c3[r, c] for c < W, 0 up to ldd; any operand may be NULL, c3 may be dst */
int gib_test_sum3_cols(float* dst, int ldd, int W, const float* a, int lda, int offa, const float* b2, int ldb,
                       int offb, const float* c3, int ldc, int rows, gib_stream stream);
/* EMN elementwise kernels over rows x ld: y = tanh(x);  G = dy (1 - y^2) selu'(pre);  G = d selu'(y) */
int gib_test_tanh_fwd(float* y, const float* x, long long rows, int ld, const int* live, gib_stream stream);
int gib_test_tanh_selu_bwd(float* G, const float* dy, const float* y, const float* pre, long long rows, int ld,
                           const int* live, gib_stream stream);
int gib_test_mul_dselu(float* G, const float* d, const float* y, long long rows, int ld, const int* live,
                       gib_stream stream);
/* EMN input rows X[r] = [nodes[i, :F] | nodes[j, :F] | edges[i, j % N, :Ef] | 0], i = ent_dst[r], j = ent_src[r]
 * (i < 0: zeros); nodes / edges int8 when i8 */
int gib_test_emn_input(float* X, int ld, const void* nodes, const void* edges, int i8, const int* ent_dst,
                       const int* ent_src, int N, int F, int Ef, long long P, gib_stream stream);
/* host only: the plan's descriptor of Linear i -- out[GIB_PLAN_LINEAR_FIELDS] = {pw, pb, src_off, rs, cs, nblk, Rb, Rbp,
 * C, Cp, Ct, Ctp, ow, owt, ob, ow_hi, ow_lo, owt_hi, owt_lo}: parameter indices (pb = -1: no bias), source offset and
 * strides, extents, and the float offsets of Wp, WTp, bp and the TF32 planes in gib_model_pack's output.  Returns the
 * number of Linears of the plan, < 0 when i is out of range or the dims are unsupported. */
#define GIB_PLAN_LINEAR_FIELDS 19
int gib_test_plan_linear(const gib_dims* d, int i, long long* out);

/* ---- generation round post-processing (SURVEY §8f #1): softmax + categorical sample of one
 *      action per molecule from the APD logits, inverse-CDF on a caller-provided uniform. ---- */
int gib_sample_actions(const float* out, int B, int apd, const float* uniforms, int* action,
                       float* likelihood, gib_stream stream);

/* ---- one round of batched graph generation on the device (SURVEY.md §8f rank 1): decode the sampled flat APD
 *      index per slot, validity rules, copy terminated graphs out (pre-action state; terminate-sampled first, then
 *      invalid, ascending), apply add / connect, reset, re-stamp the dummy graph in slot 0.  Replaces
 *      GraphGenerator.get_actions / get_invalid_actions / copy_terminated_graphs / apply_actions / reset_graphs
 *      (GraphGenerator.py:467-657, 340-385, 211-338, 425-465).
 *      Action layout: f_add[bond_to, atom, charge, (imp_h,) (chirality,) bond_type] | f_conn[bond_to, bond_type] |
 *      term, node features atom type + formal charge (+ implicit H) (+ chirality); n_imp_H / n_chirality = 0 means
 *      the segment is absent, so F must equal n_atom_types + n_charges + n_imp_H + n_chirality.  Every index count is
 *      <= 255.  The reference's `f_add_idc[5]` quirk is kept in every layout (its chirality reset makes the first
 *      atom's chirality index 0 when both segments are present); an add into a full graph terminates as invalid.
 *      gib_generation_round is this entry point with n_imp_H = n_chirality = 0 (the gdb13 layout).
 *      State: nodes [B,N,F] f32, edges [B,N,N,Ef] f32, n_nodes [B] i32, likelihoods [B,2N] f32; outputs
 *      gen_* with `capacity` rows; counters[0] = n_generated (in/out), counters[1] = graphs written this round.
 *      An action index outside [0, apd) terminates its slot as invalid and edits nothing.  Output rows at or past
 *      `capacity` are counted in n_generated but not written.  `scratch` and the gen_* rows may hold anything;
 *      `properly_terminated` must be zeroed by the caller before the first round (the rounds only set flags to 1). ---- */
size_t gib_generation_scratch_bytes(int B);
int gib_generation_round(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int round,
                         const int* action, const float* likelihood, float* nodes, float* edges, int* n_nodes,
                         float* likelihoods, float* gen_nodes, float* gen_edges, signed char* gen_n_nodes,
                         float* gen_likelihoods, signed char* properly_terminated, int capacity, int* counters,
                         void* scratch, gib_stream stream);
int gib_generation_round_layout(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                int n_chirality, int round, const int* action, const float* likelihood,
                                float* nodes, float* edges, int* n_nodes, float* likelihoods, float* gen_nodes,
                                float* gen_edges, signed char* gen_n_nodes, float* gen_likelihoods,
                                signed char* properly_terminated, int capacity, int* counters, void* scratch,
                                gib_stream stream);
/* One sample-and-round step with the round index, the stop rule and the uniforms read on the device (a CUDA-graph
 * capturable round: the launch parameters never change between rounds).
 * state (device, int[2]): [0] = index of the next round, [1] = status: 0 running, 1 round limit
 * (a round 2N would be needed while counters[0] < B).  A call whose start finds counters[0] >= B or
 * status != 0 changes nothing (an "inert" round); otherwise it samples row state[0] of `uniforms`
 * ([2N, B], inverse CDF as gib_sample_actions) from `logits` [B, apd] into action / likelihood [B], runs the round at
 * that index exactly as gib_generation_round_layout does, and increments state[0].  apd must be the layout's action
 * count; the other arguments are validated as gib_generation_round_layout validates them. */
int gib_generation_sample_round(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                int n_chirality, const float* logits, int apd, const float* uniforms, int* state,
                                int* action, float* likelihood, float* nodes, float* edges, int* n_nodes,
                                float* likelihoods, float* gen_nodes, float* gen_edges, signed char* gen_n_nodes,
                                float* gen_likelihoods, signed char* properly_terminated, int capacity,
                                int* counters, void* scratch, gib_stream stream);

/* ---- the RL rollout (GraphGeneratorRL.py:109-172) as captured rounds, and its backward by recomputation
 *      (graphinvent_b200.graphed.GraphedGeneratorRL).  Tables indexed [round, slot] have 2N rows of B. ----
 * gib_rl_sample_round: gib_generation_sample_round with two models.  The draw comes from logits_a (row state[0] of
 * `uniforms`), or, when `actions` is given, is row state[0] of `actions` [2N, B].  A running round stores the draw in
 * act_rec[r, b] and its softmax probability under logits_a / logits_b [B, apd] in p_a / p_b[r, b], then runs the round
 * with the slot tag b + 1 as every slot's likelihood (written to `tags` [B]): gen_likelihoods becomes the map from
 * (finished molecule, round) to slot + 1.  B < 2^24 - 1; the other arguments are validated as for
 * gib_generation_sample_round. */
int gib_rl_sample_round(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H, int n_chirality,
                        const float* logits_a, const float* logits_b, int apd, const float* uniforms,
                        const int* actions, int* state, int* act_rec, float* p_a, float* p_b, int* action,
                        float* tags, float* nodes, float* edges, int* n_nodes, float* likelihoods, float* gen_nodes,
                        float* gen_edges, signed char* gen_n_nodes, float* gen_likelihoods,
                        signed char* properly_terminated, int capacity, int* counters, void* scratch,
                        gib_stream stream);
/* the model input of a round: nodes [B,N,F] / edges [B,N,N,Ef] (float 0/1) as int8 into in_nodes / in_edges and, when
 * the round runs (gib_generation_sample_round's state / counters: 0 <= state[0] < 2N, state[1] == 0,
 * counters[0] < B), into row state[0] of rec_nodes [2N,B,N,F] / rec_edges [2N,B,N,N,Ef].  att_view != 0: slot 0's
 * bonds keep their first non-zero type only (the AttentionGGNN view of the dummy graph, GraphGenerator._model_inputs) */
int gib_rl_snapshot(int B, int N, int F, int Ef, int att_view, const float* nodes, const float* edges,
                    const int* state, const int* counters, signed char* rec_nodes, signed char* rec_edges,
                    signed char* in_nodes, signed char* in_edges, gib_stream stream);
/* row ctl[0] (device int) of rec_nodes / rec_edges into in_nodes / in_edges */
int gib_rl_restore(int B, int N, int F, int Ef, const signed char* rec_nodes, const signed char* rec_edges,
                   const int* ctl, signed char* in_nodes, signed char* in_edges, gib_stream stream);
/* out[g, t] = p[t, owner[g, t] - 1] for owner[g, t] in 1..B, else 0; owner / out [rows, Lw], p [Lw, B] */
int gib_rl_gather(int B, int rows, int Lw, const float* owner, const float* p_a, const float* p_b, float* out_a,
                  float* out_b, gib_stream stream);
/* the gradient of gib_rl_gather: dp [Lw, B] = 0, then dp[t, owner[g, t] - 1] = d[g, t].  d_a or d_b may be null
 * (that table is then not written).  Each (round, slot) belongs to at most one molecule. */
int gib_rl_scatter_grad(int B, int rows, int Lw, const float* owner, const float* d_a, const float* d_b, float* dp_a,
                        float* dp_b, gib_stream stream);
/* dlogits[b, :] = dp[r, b] * p * (onehot(a) - softmax(logits[b])) with a = act[r, b], p = softmax(logits[b])[a] (0 for
 * an a outside [0, apd)), and p into p_out[r, b] when p_out is given; r = ctl[0] (device int), or 0 when ctl is null.
 * The softmax is computed exactly as gib_rl_sample_round computes p_a / p_b. */
int gib_rl_dlogits(int B, int apd, const float* logits, const int* act, const float* dp, const int* ctl,
                   float* dlogits, float* p_out, gib_stream stream);
/* ctl[0] += 1 on the device (the round counter of a captured backward round) */
int gib_rl_next_round(int* ctl, gib_stream stream);

/* ---- generated molecules: the host table of graph_to_graph (GraphGenerator.py:659-804) and the histograms of
 *      Analyzer.get_molecular_properties (Analyzer.py:311-599), from generated_nodes [B,N,F] f32, generated_edges
 *      [B,N,N,Ef] f32 and generated_n_nodes [B] int8 (graphinvent_b200.molecules).  1 <= N <= 255, 1 <= F <= 32767,
 *      1 <= Ef <= 16.
 * Table (int32 words, gib_molecule_table_bytes from the dims; only the first GIB_MOL_HDR_WORDS + GIB_MOL_WORDS * B
 * words plus the used records are written):
 *   [0] atom records, [1] bonds, [2] first molecule whose statistics raise in the reference (-1: none; written by
 *   gib_graph_statistics), [3] its GIB_MOL_ERR_*, [4] its atom, [5] OR of the molecules' key-error / duplicate flags.
 *   Molecule m at GIB_MOL_HDR_WORDS + GIB_MOL_WORDS * m: n_nodes, atom records (min(max(n_nodes, 0), N)), bonds,
 *   atom offset, bond offset, GIB_MOL_* flags.
 *   Atom records from word GIB_MOL_HDR_WORDS + GIB_MOL_WORDS * B, GIB_MOL_ATOM_WORDS words = int16 [nnz, first,
 *   second, third, last non-zero feature index, 0] (-1 where absent); non-zero as torch.nonzero (NaN counts).
 *   Bonds right after the atom records, one word each = uint8 [i, j, type, 0], in the order of
 *   torch.nonzero(edges * triu(ones(N, N), 1)) over the padded N x N x Ef (NaN / inf on or below the diagonal is listed).
 * GIB_MOL_DECODES: every row _features_to_atom reads decodes (enough non-zeros, every list index inside [-len, len))
 * and n_nodes <= N; GIB_MOL_KEY_ERROR: a bond to an atom >= n_nodes; GIB_MOL_DUPLICATE_BOND: an unordered pair listed
 * twice, or a self bond (RDKit's AddBond raises). */
#define GIB_MOL_HDR_WORDS 8
#define GIB_MOL_WORDS 6
#define GIB_MOL_ATOM_WORDS 3
enum { GIB_MOL_DECODES = 1, GIB_MOL_KEY_ERROR = 2, GIB_MOL_DUPLICATE_BOND = 4 };
enum { GIB_MOL_ERR_VALUE = 1, GIB_MOL_ERR_OVERFLOW = 2, GIB_MOL_ERR_INDEX = 3 };
typedef struct gib_mol_layout {
  int n_atom_types, n_formal_charge, n_imp_H;  /* constants.n_* (feature segment widths) */
  int use_imp_H;                               /* not use_explicit_H and not ignore_H */
  int use_chirality;
  int len_atom_types, len_formal_charge, len_imp_H, len_chirality;  /* len() of the constants' lists */
} gib_mol_layout;
size_t gib_molecule_table_bytes(int B, int N, int F, int Ef);
int gib_molecule_table(int B, int N, int F, int Ef, const gib_mol_layout* layout, const float* nodes,
                       const float* edges, const signed char* n_nodes, int* table, gib_stream stream);
/* Statistics of the molecules of a table built from the same tensors, with n_nodes = 0 for a molecule that does not
 * decode.  out (f32): n_nodes_hist [N+1] | column sums of the nodes [F] | n_edges_hist [10] | edge_feature_hist [Ef] |
 * sum_k k * n_nodes_hist[k] | sum_k (k+1) * n_edges_hist[k].  Sums run in molecule order, as the reference's loops do
 * (exact for integer-valued features); a per-(atom, type) row sum beyond +-1e12 is clamped before it is summed.
 * Writes words [2..4] of the table.  ws: gib_graph_statistics_ws_bytes, may hold anything. */
size_t gib_graph_statistics_bytes(int N, int F, int Ef);
size_t gib_graph_statistics_ws_bytes(int B, int N, int F, int Ef);
int gib_graph_statistics(int B, int N, int F, int Ef, const float* nodes, const float* edges, int* table, float* out,
                         void* ws, gib_stream stream);

/* ---- training-set construction: DataProcesser.get_subgraphs (DataProcesser.py:167-271) over the decoding routes of
 *      PreprocessingGraph (MolecularGraph.py:463-555, 635-732), for one chunk of molecules (graphinvent_b200.preprocess).
 * Input: `nodes` int8 [n, N, F] and `edges` int8 [n, N, N, Ef], padded one-hot graphs in decoding order: node rows
 * [0, n_atoms) one-hot per segment with 0 / 1 entries, zero rows after; edges symmetric, 0 / 1, one bond type per
 * atom pair, no self bond; every route connected.  A chunk holding any other molecule produces no group; status[3]
 * then holds GIB_PP_* bits and status[4] the first such molecule (a route that disconnects only flags that molecule
 * when it is reached, see status[3]).
 * Groups start at molecule 0 of the chunk and follow each other as the reference's do: a group reads at most
 * batch_size molecules, appends rows by the reference's rule (a state matching no row, or whose first match is the
 * last row) and ends when it reaches batch_size rows (the rest of that molecule's route is dropped) or runs out of
 * its molecules.  A group that runs out of the chunk's molecules before either, when last_chunk == 0, is not
 * written: the caller starts the next chunk at its first molecule (status[1]).  No group starts once fewer than
 * batch_size rows of max_rows are left.
 * Output: rows [0, status[2]) of out_nodes [max_rows, N, F] int8, out_edges [max_rows, N, N, Ef] int8 and out_apds
 * [max_rows, apd] int32 (APD counts, apd = gib_preprocess_apd_length); groups [max_molecules, 4] int32 per group:
 * first molecule, molecule after the last one it visited, first row, rows.  status int32 [GIB_PP_STATUS_INTS]:
 * [0] groups, [1] first molecule not yet in a group, [2] rows, [3] GIB_PP_* flags, [4] first bad molecule
 * (INT_MAX: none), [5] route states of the chunk.  The workspace may hold anything; results are deterministic.
 * Limits: N*N*Ef <= 32768, N*F <= 8192, n_atom_types and n_formal_charge >= 1, n_imp_H and n_chirality >= 0 (0: the
 * segment is absent: the four action layouts), F their sum, batch_size >= 1, max_rows >= batch_size,
 * max_molecules * (N*(N-1)/2 + 2) < 2^30. */
#define GIB_PP_STATUS_INTS 8
enum { GIB_PP_BAD_NODES = 1, GIB_PP_BAD_EDGES = 2, GIB_PP_EMPTY = 4, GIB_PP_DISCONNECTED = 8 };
typedef struct gib_pp_dims {
  int N, F, Ef;                                             /* max_n_nodes, n_node_features, n_edge_features */
  int n_atom_types, n_formal_charge, n_imp_H, n_chirality;  /* node-feature segment widths, in order */
  int batch_size;                                           /* rows per group (constants.batch_size) */
} gib_pp_dims;
int gib_preprocess_apd_length(const gib_pp_dims* d);        /* N * (f_add + Ef) + 1, < 0 for unsupported dims */
size_t gib_preprocess_ws_bytes(const gib_pp_dims* d, int max_molecules, int max_rows);
int gib_preprocess_chunk(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int n_molecules,
                         int last_chunk, int max_molecules, int max_rows, void* ws, signed char* out_nodes,
                         signed char* out_edges, int* out_apds, int* groups, int* status, gib_stream stream);
/* The training-set properties of the groups a gib_preprocess_chunk call completed (Analyzer.get_molecular_properties,
 * Analyzer.py:311-599, as DataProcesser.get_ts_properties runs it per group), on the same stream after that call, from
 * the same `nodes` / `edges`, `n_molecules`, `max_molecules`, `groups` and `status` (the group count is read on the
 * device).  Row g of `out` (int32, gib_preprocess_group_statistics_bytes(d, max_molecules) bytes; rows past status[0]
 * are not written) is group g's 4 words of `groups` followed by integer sums over its molecules [first, after last):
 *   n_nodes_hist [N+1]     molecules per atom count (the rows up to the last non-zero one)
 *   node sums [F]          column sums of the node features
 *   n_edges_hist [10]      atoms per bond count, as _get_n_edges_distribution bins them: a count above 10 goes to bin
 *                          9, and so does an atom without bonds (bin n_edges - 1 = -1)
 *   bonds [Ef]             bonds per type (half the sum of the symmetric edge entries)
 * Each molecule's partials come from the per-molecule pass of gib_graph_statistics; each group is summed by one CTA
 * in molecule order: the results are deterministic.  Besides gib_preprocess_chunk's limits: N <= 255, Ef <= 16.
 * ws: gib_preprocess_group_statistics_ws_bytes(d, max_molecules), may hold anything. */
size_t gib_preprocess_group_statistics_bytes(const gib_pp_dims* d, int max_groups);
size_t gib_preprocess_group_statistics_ws_bytes(const gib_pp_dims* d, int max_molecules);
int gib_preprocess_group_statistics(const gib_pp_dims* d, const signed char* nodes, const signed char* edges,
                                    int n_molecules, int max_molecules, const int* groups, const int* status,
                                    void* ws, int* out, gib_stream stream);

/* ---- the likelihood of a molecule's decoding route (graphinvent_b200.graphed.RouteScorer): for every route state,
 *      p(action | state) = softmax(model(state))[action], one chunk of molecules at a time.
 * gib_route_plan: the decoding routes of a chunk, by the count / scan / route kernels of gib_preprocess_chunk (same
 * input contract, dims and limits; d->batch_size is the scorer's batch B).  Writes offsets [n_molecules + 1] (the
 * molecules' first state; offsets[n] = S, the chunk's states) and the per-state plan in ws, and status int32
 * [GIB_PP_STATUS_INTS]: [3] GIB_PP_* flags, [4] first bad molecule (INT_MAX: none), [5] S, [6] = 0, the fill cursor;
 * the other words are 0.  A chunk with a bad molecule has no valid plan.  ws: gib_route_plan_ws_bytes, may hold
 * anything.  gib_route_max_states: the most states a chunk of max_molecules molecules can have (< 0: bad dims).
 * gib_route_fill: states [c*B, c*B + B) of the chunk, c = status[6], into out_nodes [B, N, F] / out_edges [B, N, N, Ef]
 * int8 (state k of a molecule: node rows below its node count, the bonds the route still holds at step k), zero rows
 * past S; ctl->live = the states it wrote; slots int32 [2B]: each slot's action, then its place in the chunk's
 * likelihood buffer (-1 / -1 for a zero row).  A molecule's places run offsets[m] .. offsets[m+1]-1 in BUILD order:
 * the empty graph first, the full graph with the terminate action last.  Advance the cursor with
 * gib_rl_next_round(status + 6).  Reads only what gib_route_plan wrote for this chunk, from the same nodes / edges;
 * nodes, edges and both outputs 16-byte aligned.
 * gib_route_probs: likelihoods[slots[B+b]] = softmax(logits[b])[slots[b]] for every slot with slots[B+b] >= 0, by
 * the softmax reduction of the RL sampler (bit for bit the probability gib_rl_sample_round records for that row).
 * gib_route_reduce: per molecule m < n_molecules, over likelihoods[offsets[m] .. offsets[m+1]) in order, in fp64:
 * nll[m] = -sum log p and final[m] = log(sum p), each rounded once to fp32. */
size_t gib_route_plan_ws_bytes(const gib_pp_dims* d, int max_molecules);
long long gib_route_max_states(const gib_pp_dims* d, int max_molecules);
int gib_route_plan(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int n_molecules,
                   int max_molecules, void* ws, int* offsets, int* status, gib_stream stream);
int gib_route_fill(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int max_molecules,
                   const void* ws, const int* offsets, const int* status, gib_batch_ctl* ctl, int* slots,
                   signed char* out_nodes, signed char* out_edges, gib_stream stream);
int gib_route_probs(int B, int apd, const float* logits, const int* slots, float* likelihoods, gib_stream stream);
int gib_route_reduce(int n_molecules, const int* offsets, const float* likelihoods, float* nll, float* final_,
                     gib_stream stream);

/* ---- measurement hooks: CUDA-event timing per kernel class on the launching stream.
 *      class 0 = forward/dX launches of the tensor-core kernel, 1 = its weight-gradient launches, 2 = scatter-aggregate (K2),
 *      3 / 4 = forward/dX and weight-gradient GEMMs on the fp32 SIMT kernels.  GIB_PROFILE_CLASSES entries per array.
 *      work = algorithmic FLOPs (GEMM classes) or bytes (class 2).  Collect after a stream sync. -- */
#define GIB_PROFILE_CLASSES 5
void gib_profile_enable(int on);
long long gib_launch_count(void); /* kernels launched by this library since load */
int gib_profile_collect(double* ms, double* work, long long* count);
/* per-launch records in launch order (before gib_profile_collect, which clears them): returns their number */
int gib_profile_records(double* ms, double* work, int* cls, int cap);

#ifdef __cplusplus
}
#endif
#endif /* GIB200_H */
