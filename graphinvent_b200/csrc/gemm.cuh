// Internal GEMM interfaces shared by the SIMT (gemm_simt.cu) and tensor-core (gemm_tc3.cu) paths.
#pragma once
#include "common.cuh"
#include "prof.cuh"

namespace gib {

enum Epi : int {
  EPI_ACT = 0,       // C = act(acc + bias)
  EPI_MUL_DACT = 1,  // C = acc * act'(aux)      (aux = activation OUTPUT of the layer below)
  EPI_ADD = 2        // C = acc + aux
};

// C[M, :N] = epi( A[M,K] * B[N,K]^T ).  A, B row-major, K-contiguous, K % 16 == 0,
// lda/ldb % 4 == 0.  Columns [n_valid, n_store) are written as zeros; columns >= n_store
// are not touched.
struct GemmNT {
  const float* A = nullptr; int lda = 0;
  const float* B = nullptr; int ldb = 0;
  const float* B_hi = nullptr;      // optional TF32 hi / lo planes of B (same shape and ldb): the tensor-core kernel
  const float* B_lo = nullptr;      // then loads them directly and only splits A on the fly
  float* C = nullptr; int ldc = 0;
  int M = 0, N = 0, K = 0;
  const float* bias = nullptr;
  int act = ACT_NONE;
  int mode = EPI_ACT;
  const float* aux = nullptr; int ldaux = 0;
  int n_store = 0;
  int n_valid = 0;
  double work = 0;   // algorithmic FLOPs of this launch (0: derive from the padded extents)
  // Device-side row range (capacity mode, tensor-core path only): when m_dev is set, A / C / aux point at row 0 of buffers
  // of M rows (the capacity) and the problem covers rows [*base_dev, *base_dev + *m_dev) of them -- the bond-type
  // group sizes K0 leaves in device memory, so no launch parameter depends on the batch content.
  const int* m_dev = nullptr;
  const int* base_dev = nullptr;
  // Precision of the tensor-core kernels: 0 = 3xTF32 (fp32-accurate), 1 = single-pass TF32 (the hi*hi term only),
  // 2 = bf16, 3 = fp16 operands (fp32 accumulation; B_hi then points at the 16-bit plane of B, ldb in elements, and
  // B_lo is not read).  The fp32 SIMT kernel ignores it.
  int tf32 = 0;
};

struct GemmTN {  // kernel-level args of the split-K dW kernel
  const float* G; int ldg;
  const float* X; int ldx;
  int M, Nn, Kk, chunk_rows;
  float* ws; float* ws_bias;
};

// dW[r, c] += sum_m G[m, prow(r)] * X[m, c];  dbias[r] += sum_m G[m, prow(r)]
// prow(r) = (r / Rb) * Rbp + r % Rb maps a real output row to its padded (gate-blocked) row.
// Destination element (r, c) lives at dW[r * rs + c * cs] (handles MNN's strided weights).
struct GemmDW {
  const float* G = nullptr; int ldg = 0; int Nn = 0;  // G: [M, Nn] padded width
  const float* X = nullptr; int ldx = 0; int Kk = 0;  // X: [M, Kk] padded width
  int M = 0;
  float* dW = nullptr; float* dbias = nullptr;        // either may be null
  int R = 0, C = 0, Rb = 0, Rbp = 0;
  long long rs = 0, cs = 1;
  float* scratch = nullptr;                           // >= gemm_dw_scratch_floats(...) of the largest call: two halves
  size_t half_floats = 0;                             // size of one half (same value for every call on this scratch)
  double work = 0;                                    // algorithmic FLOPs (0: derive)
  const int* m_dev = nullptr;                         // device-side row range inside buffers of M rows (see GemmNT)
  const int* base_dev = nullptr;
  int tf32 = 0;                                       // tensor-core precision (see GemmNT)
};

constexpr int kTc3MaxProblems = 16;   // problems per launch of the tensor-core kernel

// scratch layout of one grouped weight-gradient launch of the tensor-core kernel (gemm_tc3.cu)
struct Dw3Layout {
  int chunk_rows;                          // reduction rows per work item
  int cap_splits[kTc3MaxProblems];         // split capacity per problem (the live count may be smaller: device-side row counts)
  size_t part_off[kTc3MaxProblems];        // float offsets of [cap_splits][Nn][Kk] partial products
  size_t bias_off[kTc3MaxProblems];        // float offsets of [cap_splits][Nn] partial column sums
  size_t floats;                           // total
};

int gemm_nt(const GemmNT& p, cudaStream_t st);      // dispatches to the tensor-core path when enabled and eligible
int gemm_nt_simt(const GemmNT& p, cudaStream_t st);
int gemm_nt_tc(const GemmNT& p, cudaStream_t st);
int gemm_nt_tc_group(const GemmNT* ps, int n, cudaStream_t st);   // n <= 4 independent problems, raw or pre-split W
int gemm_nt_group(const GemmNT* ps, int n, cudaStream_t st);      // dispatcher: grouped tensor-core launch or per-problem
bool gemm_nt_chain_ok(const GemmNT* ps, int n);                   // can these run as one dependent-chain launch?
int gemm_nt_chain(const GemmNT* ps, const int* dep, int n, int* flags, cudaStream_t st);
bool tc_eligible(const GemmNT& p);
// pre-split weight planes (the model's call pattern); the activation operand is split in registers
bool tc3_eligible(const GemmNT& p);
int gemm_nt_tc3_group(const GemmNT* ps, int n, cudaStream_t st);
// Dependent chain in ONE persistent launch: problem i consumes (A operand) what problem dep[i] produces (dep[i] < i,
// -1 = independent) with the same row range; work flows from layer to layer row block by row block through counters in
// `flags` (device ints, >= tc3_chain_flag_ints(ps, n), zeroed here).  No per-layer launch, prologue, tail or wave
// quantisation.
size_t tc3_chain_flag_ints(const GemmNT* ps, int n);
int gemm_nt_tc3_chain(const GemmNT* ps, const int* dep, int n, int* flags, cudaStream_t st);
bool tc3_dw_eligible(const GemmDW& q);
int tc3_dw_chunk_rows(const GemmDW* qs, int n, long long plan_rows);   // from ALL members of a group (sizing == run time)
void tc3_dw_layout(const GemmDW* qs, int n, int chunk_rows, Dw3Layout* L);
int gemm_dw_tc3_partials(const GemmDW* qs, int n, const Dw3Layout& L, float* scratch, cudaStream_t st);
int gemm_dw_tc3_reduce(const GemmDW* qs, int n, const Dw3Layout& L, const float* scratch, cudaStream_t st);
int device_sm_count();     // SMs of the current device (cached per device)
void tc3_set_trace(long long* buf, int tiles);   // diagnosis: per-tile clock64 stamps of CTA 0
extern bool g_use_tc;
extern int g_tc_debug;
// 0 when a GEMM of precision `prec` can run as asked (a known code; 16-bit codes need the tensor-core path), else the
// error code with the message set
int check_precision(int prec, const char* who);

int gemm_dw(const GemmDW& q, cudaStream_t st);
// n <= 16 weight-gradient problems that may run as ONE grouped tensor-core launch + ONE reduction launch (siblings of a
// layer: the per-bond-type message MLPs, the readout heads, the two GRU projections).  plan_rows: expected total
// reduction rows of the group (0: the sum of q.M), used to size the split so that the group fills the machine once.
int gemm_dw_group(const GemmDW* qs, int n, long long plan_rows, cudaStream_t st);
size_t gemm_dw_group_half_floats(const GemmDW* qs, int n, long long plan_rows);
int dw_begin();            // start of a C-ABI call that uses gemm_dw: forget the previous call's side-stream jobs
void gemm_dw_plan(int M, int Nn, int Kk, int* splits, int* chunk);
void tc_dw_plan(int M, int Nn, int Kk, int* splits, int* chunk);
bool tc_dw_eligible(const GemmDW& q);
int gemm_dw_tc_partials(const GemmDW& q, int* splits_out, cudaStream_t st);
size_t gemm_dw_scratch_floats(int M, int Nn, int Kk);   // both halves
size_t gemm_dw_half_floats(int M, int Nn, int Kk);
int dw_join(cudaStream_t st);                            // drain the helper side stream into `st`

}  // namespace gib
