// fp32 SIMT GEMMs for the dense blocks of the hot path (edge-MLP, GRU, gather, APD readout).
//
// Why fp32 FMA and not plain TF32/BF16 tensor-core math: the parity bar is 1e-4 on the
// logits and single-pass TF32 operand rounding alone gives 1.8e-2 (SURVEY.md §7 "hard
// parts").  This file is the fp32-exact baseline path; the tensor-core 3xTF32 path
// (gemm_tc3.cu) replaces it where enabled and is validated against it.
//
// Layout contract (DESIGN.md "data layout"): every operand is row-major with a leading
// dimension that is a multiple of 16 floats, pad columns hold exact zeros, the reduction
// extent K is a multiple of 16.  Replaces the ATen `addmm`/`mm` call sites of
// reference gnn/modules.py:162-170 (MLP), gnn/mpnn.py:296 (GRUCell) and their autograd.
#include <algorithm>
#include <mutex>

#include "gemm.cuh"
#include "ops.cuh"

namespace gib {

constexpr int BK = 16;

// Epilogue of the fp32 SIMT NT kernels: the sums v of row m, columns [n, n + 4) -> C (columns >= n_store untouched).
// vec_c / vec_x: C / aux rows may be read and written as float4.
__device__ __forceinline__ void sgemm_nt_epilogue4(const GemmNT& p, int m, int n, const float (&acc)[4], bool vec_c,
                                                   bool vec_x) {
  float v[4] = {acc[0], acc[1], acc[2], acc[3]};
  float x[4] = {0.f, 0.f, 0.f, 0.f};
  if (p.mode != EPI_ACT) {
    if (vec_x && n + 3 < p.n_store) {
      float4 t4 = *reinterpret_cast<const float4*>(p.aux + (size_t)m * p.ldaux + n);
      x[0] = t4.x; x[1] = t4.y; x[2] = t4.z; x[3] = t4.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (n + j < p.n_store) x[j] = p.aux[(size_t)m * p.ldaux + n + j];
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (p.mode == EPI_ACT) {
      float bj = (p.bias && n + j < p.N) ? p.bias[n + j] : 0.f;
      v[j] = act_f(v[j] + bj, p.act);
    } else if (p.mode == EPI_MUL_DACT) {
      v[j] = v[j] * dact_from_out(x[j], p.act);
    } else {
      v[j] = v[j] + x[j];
    }
    if (n + j >= p.n_valid) v[j] = 0.f;
  }
  float* dst = p.C + (size_t)m * p.ldc + n;
  if (vec_c && n + 3 < p.n_store) {
    *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (n + j < p.n_store) dst[j] = v[j];
  }
}

__device__ __forceinline__ bool sgemm_vec_c(const GemmNT& p) {
  return (p.ldc & 3) == 0 && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0);
}
__device__ __forceinline__ bool sgemm_vec_x(const GemmNT& p) {
  return p.aux && (p.ldaux & 3) == 0 && ((reinterpret_cast<uintptr_t>(p.aux) & 15) == 0);
}

// ------------------------------------------------------------------------------------
// C[M,N] = epilogue( A[M,K] * B[N,K]^T )       (both operands K-contiguous)
// ------------------------------------------------------------------------------------
template <int BM, int BN, int RM, int RN>
__global__ void __launch_bounds__(256, 2) sgemm_nt_kernel(const GemmNT p) {
  static_assert((BM / (4 * RM)) * (BN / (4 * RN)) == 256, "256 threads");
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];

  const int tid = threadIdx.x;
  const int w = tid >> 5, l = tid & 31;
  const int ty = (w >> 1) * 4 + (l >> 3);  // 0..15 along M
  const int tx = (w & 1) * 8 + (l & 7);    // 0..15 along N
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

  constexpr int LA = BM / 64, LB = BN / 64;  // float4 loads per thread per tile
  float4 ra[LA], rb[LB];
  const float* a_ptr[LA];
  const float* b_ptr[LB];
  bool a_ok[LA], b_ok[LB];
#pragma unroll
  for (int i = 0; i < LA; ++i) {
    int q = tid + i * 256, row = q >> 2, kq = q & 3;
    a_ok[i] = (m0 + row) < p.M;
    a_ptr[i] = p.A + (size_t)(m0 + row) * p.lda + kq * 4;
  }
#pragma unroll
  for (int i = 0; i < LB; ++i) {
    int q = tid + i * 256, row = q >> 2, kq = q & 3;
    b_ok[i] = (n0 + row) < p.N;
    b_ptr[i] = p.B + (size_t)(n0 + row) * p.ldb + kq * 4;
  }
  auto gload = [&](int k0) {
#pragma unroll
    for (int i = 0; i < LA; ++i)
      ra[i] = a_ok[i] ? __ldg(reinterpret_cast<const float4*>(a_ptr[i] + k0)) : make_float4(0, 0, 0, 0);
#pragma unroll
    for (int i = 0; i < LB; ++i)
      rb[i] = b_ok[i] ? __ldg(reinterpret_cast<const float4*>(b_ptr[i] + k0)) : make_float4(0, 0, 0, 0);
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      int q = tid + i * 256, row = q >> 2, kq = (q & 3) * 4;
      As[buf][kq + 0][row] = ra[i].x; As[buf][kq + 1][row] = ra[i].y;
      As[buf][kq + 2][row] = ra[i].z; As[buf][kq + 3][row] = ra[i].w;
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      int q = tid + i * 256, row = q >> 2, kq = (q & 3) * 4;
      Bs[buf][kq + 0][row] = rb[i].x; Bs[buf][kq + 1][row] = rb[i].y;
      Bs[buf][kq + 2][row] = rb[i].z; Bs[buf][kq + 3][row] = rb[i].w;
    }
  };

  float acc[RM][4][RN][4];
#pragma unroll
  for (int a = 0; a < RM; ++a)
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int b = 0; b < RN; ++b)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[a][i][b][j] = 0.f;

  const int ntiles = p.K / BK;
  gload(0);
  sstore(0);
  __syncthreads();
  for (int t = 0; t < ntiles; ++t) {
    const int buf = t & 1;
    if (t + 1 < ntiles) gload((t + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float4 fa[RM], fb[RN];
#pragma unroll
      for (int a = 0; a < RM; ++a)
        fa[a] = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4 + a * (BM / RM)]);
#pragma unroll
      for (int b = 0; b < RN; ++b)
        fb[b] = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4 + b * (BN / RN)]);
#pragma unroll
      for (int a = 0; a < RM; ++a) {
        const float av[4] = {fa[a].x, fa[a].y, fa[a].z, fa[a].w};
#pragma unroll
        for (int b = 0; b < RN; ++b) {
          const float bv[4] = {fb[b].x, fb[b].y, fb[b].z, fb[b].w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[a][i][b][j] = fmaf(av[i], bv[j], acc[a][i][b][j]);
        }
      }
    }
    if (t + 1 < ntiles) sstore(buf ^ 1);
    __syncthreads();
  }

  // ---- epilogue -------------------------------------------------------------------
  const bool vec_c = sgemm_vec_c(p), vec_x = sgemm_vec_x(p);
#pragma unroll
  for (int a = 0; a < RM; ++a)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + ty * 4 + a * (BM / RM) + i;
      if (m >= p.M) continue;
#pragma unroll
      for (int b = 0; b < RN; ++b) {
        const int n = n0 + tx * 4 + b * (BN / RN);
        if (n >= p.n_store) continue;
        const float v[4] = {acc[a][i][b][0], acc[a][i][b][1], acc[a][i][b][2], acc[a][i][b][3]};
        sgemm_nt_epilogue4(p, m, n, v, vec_c, vec_x);
      }
    }
}

// ------------------------------------------------------------------------------------
// Narrow outputs (max(N, n_store) <= 48: the APD heads' output layers), up to kNarrowMax independent problems per
// launch.  One column tile per problem, 16, 32 or 48 wide; 192 threads, each owning TM rows x 4 columns, so a CTA covers
// (192 / (bn / 4)) * TM rows.  Every output is the same fmaf chain over k = 0 .. K-1 as in sgemm_nt_kernel and goes
// through the same epilogue: the results are bit-identical to it.
// ------------------------------------------------------------------------------------
constexpr int kNarrowThreads = 192;
constexpr int kNarrowMaxN = 48;
constexpr int kNarrowMax = 4;
struct NarrowGroup {
  GemmNT p[kNarrowMax];
  int bn[kNarrowMax];          // column tile of each problem
  int cta0[kNarrowMax + 1];    // first CTA of each problem
  int n;
};

template <int TM>
__global__ void __launch_bounds__(kNarrowThreads) sgemm_nt_narrow_kernel(const __grid_constant__ NarrowGroup g) {
  __shared__ __align__(16) float As[2][BK][kNarrowThreads / 4 * TM + 4];   // rows of a 16-wide tile, the tallest
  __shared__ __align__(16) float Bs[2][BK][kNarrowMaxN + 4];
  int pi = 0;
  while (pi + 1 < g.n && (int)blockIdx.x >= g.cta0[pi + 1]) ++pi;
  const GemmNT& p = g.p[pi];
  const int bn = g.bn[pi], nt = bn / 4;
  const int tid = threadIdx.x;
  const int cg = tid % nt, rg = tid / nt;
  const int bm = (kNarrowThreads / nt) * TM;
  const int m0 = ((int)blockIdx.x - g.cta0[pi]) * bm;

  float4 ra[TM], rb;
  const float* a_ptr[TM];
  bool a_ok[TM];
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int q = tid + i * kNarrowThreads, row = q >> 2;
    a_ok[i] = q < bm * 4 && (m0 + row) < p.M;
    a_ptr[i] = p.A + (size_t)(m0 + row) * p.lda + (q & 3) * 4;
  }
  const bool b_ok = tid < bn * 4 && (tid >> 2) < p.N;
  const float* b_ptr = p.B + (size_t)(tid >> 2) * p.ldb + (tid & 3) * 4;
  auto gload = [&](int k0) {
#pragma unroll
    for (int i = 0; i < TM; ++i)
      ra[i] = a_ok[i] ? __ldg(reinterpret_cast<const float4*>(a_ptr[i] + k0)) : make_float4(0, 0, 0, 0);
    rb = b_ok ? __ldg(reinterpret_cast<const float4*>(b_ptr + k0)) : make_float4(0, 0, 0, 0);
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int q = tid + i * kNarrowThreads, row = q >> 2, kq = (q & 3) * 4;
      if (q < bm * 4) {
        As[buf][kq + 0][row] = ra[i].x; As[buf][kq + 1][row] = ra[i].y;
        As[buf][kq + 2][row] = ra[i].z; As[buf][kq + 3][row] = ra[i].w;
      }
    }
    if (tid < bn * 4) {
      const int row = tid >> 2, kq = (tid & 3) * 4;
      Bs[buf][kq + 0][row] = rb.x; Bs[buf][kq + 1][row] = rb.y;
      Bs[buf][kq + 2][row] = rb.z; Bs[buf][kq + 3][row] = rb.w;
    }
  };

  float acc[TM][4];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int ntiles = p.K / BK;
  gload(0);
  sstore(0);
  __syncthreads();
  for (int t = 0; t < ntiles; ++t) {
    const int buf = t & 1;
    if (t + 1 < ntiles) gload((t + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float av[TM];
      if constexpr (TM == 4) {
        const float4 f = *reinterpret_cast<const float4*>(&As[buf][kk][rg * 4]);
        av[0] = f.x; av[1] = f.y; av[2] = f.z; av[3] = f.w;
      } else if constexpr (TM == 2) {
        const float2 f = *reinterpret_cast<const float2*>(&As[buf][kk][rg * 2]);
        av[0] = f.x; av[1] = f.y;
      } else {
        av[0] = As[buf][kk][rg];
      }
      const float4 fb = *reinterpret_cast<const float4*>(&Bs[buf][kk][cg * 4]);
      const float bv[4] = {fb.x, fb.y, fb.z, fb.w};
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (t + 1 < ntiles) sstore(buf ^ 1);
    __syncthreads();
  }

  const bool vec_c = sgemm_vec_c(p), vec_x = sgemm_vec_x(p);
  const int n = cg * 4;
  if (n >= p.n_store) return;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + rg * TM + i;
    if (m < p.M) sgemm_nt_epilogue4(p, m, n, acc[i], vec_c, vec_x);
  }
}

// gib_tc_debug bit 0: the per-problem call pattern (no grouped / chained launches, W split in the kernel)
static inline bool use_tc3() { return (g_tc_debug & 1) == 0; }

// bf16 / fp16 operands (precision 2 / 3) exist on the wgmma kernels only: with tensor cores off or debug bit 0 a
// 16-bit call is refused rather than run in another precision
int check_precision(int prec, const char* who) {
  if (prec < 0 || prec > 3) { set_error("%s: unknown matmul precision %d", who, prec); return -2; }
  if (prec >= 2 && (!g_use_tc || !use_tc3())) {
    set_error("%s: bf16 / fp16 GEMMs need the tensor-core path (tensor cores on, gib_tc_debug bit 0 clear)", who);
    return -2;
  }
  return 0;
}

// gib_tc_debug bit 4: the dispatch before the narrow kernel -- narrow problems on sgemm_nt_kernel, mixed groups and the
// first-layer input gradients of sibling MLPs problem by problem (A/B comparisons, and the reference of the tests)
static inline bool narrow_dispatch() { return (g_tc_debug & 16) == 0; }

// Where gemm_nt sends one problem
enum NtRoute { NT_TC3, NT_TC, NT_NARROW, NT_SIMT };
static NtRoute nt_route(const GemmNT& p) {
  // tensor-core path for all but the tiny / skinny GEMMs (those stay on the SIMT kernels); a problem whose row count
  // lives on the device (capacity mode) runs there only (gemm_nt refuses it when that path is off or not eligible)
  if (p.m_dev) return NT_TC3;
  if (g_use_tc && p.N >= 48 && p.K >= 32) {
    if (use_tc3() && p.M >= 256 && tc3_eligible(p)) return NT_TC3;
    if (p.M >= 1024 && tc_eligible(p)) return NT_TC;
  }
  // Narrow outputs (the APD heads: 1024 x 500 -> 39 / 3 / 1) stay on the fp32 SIMT kernels unless debug bit 2 is set:
  // a handful of tensor-core tiles would be faster, but the output layer's 3xTF32 error lands on the logits
  // unattenuated, and on the shipped checkpoint x 256 gdb13 rows the logit error is already close to the 1e-4 contract
  // with this layer in fp32 (tests/test_gpu_parity.py::test_pretrained_checkpoint_on_real_gdb13_rows).
  if (g_use_tc && use_tc3() && (g_tc_debug & 4) && p.N < 48 && p.K >= 128 && p.M >= 256 && tc3_eligible(p))
    return NT_TC3;
  if (narrow_dispatch() && std::max(p.N, p.n_store) <= kNarrowMaxN) return NT_NARROW;
  return NT_SIMT;
}

int gemm_nt(const GemmNT& p, cudaStream_t st) {
  GIB_TRY(check_precision(p.tf32, "gemm_nt"));
  if (p.m_dev && (!g_use_tc || !use_tc3() || !tc3_eligible(p))) {
    set_error("gemm_nt: device-side row counts need the tensor-core path (tensor cores on, pre-split weights)");
    return -2;
  }
  switch (nt_route(p)) {
    case NT_TC3: return gemm_nt_tc3_group(&p, 1, st);
    case NT_TC: return gemm_nt_tc(p, st);
    case NT_NARROW: return gemm_nt_narrow(&p, 1, st);
    default: return gemm_nt_simt(p, st);
  }
}

// n <= 4 independent problems that write disjoint outputs, with the results gemm_nt gives each of them: the members
// gemm_nt sends to the wgmma kernel as one grouped launch, the narrow ones as one narrow launch, the rest one by one
int gemm_nt_batch(const GemmNT* ps, int n, cudaStream_t st) {
  if (n > kNarrowMax) { set_error("gemm_nt_batch: %d problems (max %d)", n, kNarrowMax); return -2; }
  if (n == 1 || !narrow_dispatch()) {
    for (int i = 0; i < n; ++i) GIB_TRY(gemm_nt(ps[i], st));
    return 0;
  }
  GemmNT tc3[kNarrowMax], narrow[kNarrowMax];
  int n3 = 0, nn = 0;
  for (int i = 0; i < n; ++i) {
    const GemmNT& p = ps[i];
    const NtRoute rt = nt_route(p);
    const bool refused = p.m_dev && (!g_use_tc || !use_tc3() || !tc3_eligible(p));
    if (refused || (rt != NT_TC3 && rt != NT_NARROW)) { GIB_TRY(gemm_nt(p, st)); continue; }
    GIB_TRY(check_precision(p.tf32, "gemm_nt_batch"));
    if (p.M <= 0 || p.N <= 0) continue;
    if (rt == NT_TC3) tc3[n3++] = p; else narrow[nn++] = p;
  }
  if (n3) GIB_TRY(gemm_nt_tc3_group(tc3, n3, st));
  if (nn) GIB_TRY(gemm_nt_narrow(narrow, nn, st));
  return 0;
}

// Several independent problems (sibling MLPs, the per-bond-type message MLPs): one grouped tensor-core launch when
// together they fill the machine reasonably, else as gemm_nt_batch
int gemm_nt_group(const GemmNT* ps, int n, cudaStream_t st) {
  if (n == 1) return gemm_nt(ps[0], st);
  for (int i = 0; i < n; ++i) GIB_TRY(check_precision(ps[i].tf32, "gemm_nt_group"));
  bool ok = g_use_tc && n <= 4, ok3 = ok && use_tc3(), dyn = false;
  long long tiles = 0;
  for (int i = 0; i < n && ok; ++i) {
    if (ps[i].m_dev) dyn = true;
    if (ps[i].M <= 0 || ps[i].N <= 0) continue;
    ok = tc_eligible(ps[i]) && ps[i].K >= 32 && ps[i].N >= 48;
    ok3 = ok3 && ok && tc3_eligible(ps[i]);
    tiles += (long long)ceil_div(ps[i].M, 128) * ceil_div(ps[i].N, 128);
  }
  if (ok3 && (tiles >= 4 || dyn)) return gemm_nt_tc3_group(ps, n, st);
  if (ok && !dyn && tiles >= 16) return gemm_nt_tc_group(ps, n, st);
  return gemm_nt_batch(ps, n, st);
}

// Dependent chain (the layers of sibling MLPs): ONE persistent tensor-core launch when every member qualifies,
// else layer by layer through gemm_nt_group (members of one layer = consecutive problems with equal `layer`).
bool gemm_nt_chain_ok(const GemmNT* ps, int n) {
  if (!g_use_tc || !use_tc3() || n < 2 || n > kTc3MaxProblems || (g_tc_debug & 2)) return false;
  long long tiles = 0;
  bool dyn = false;
  for (int i = 0; i < n; ++i) {
    const GemmNT& p = ps[i];
    if (p.M <= 0 || p.N <= 0) continue;
    if (!tc3_eligible(p) || p.N < 48 || p.K < 32) return false;
    if (p.m_dev) dyn = true;
    tiles += (long long)ceil_div(p.M, 128) * ceil_div(p.N, 128);
  }
  return dyn || tiles >= 16;      // small members ride along; a tiny chain is not worth a persistent launch over every SM
}
int gemm_nt_chain(const GemmNT* ps, const int* dep, int n, int* flags, cudaStream_t st) {
  return gemm_nt_tc3_chain(ps, dep, n, flags, st);
}

int gemm_nt_simt(const GemmNT& p, cudaStream_t st) {
  if (p.M <= 0 || p.N <= 0) return 0;
  if (p.K % BK != 0 || (p.lda & 3) || (p.ldb & 3) || p.K <= 0) {
    set_error("gemm_nt: K=%d lda=%d ldb=%d violate the padded-layout contract", p.K, p.lda, p.ldb);
    return -2;
  }
  ProfScope prof(PROF_GEMM_NT_SIMT, p.work > 0 ? p.work : 2.0 * p.M * (double)p.N * p.K, st);
  const int ncols = std::max(p.N, p.n_store);     // columns [N, n_store) are stored too (zeros / epi(0))
  const long long ctas_big = (long long)ceil_div(p.M, 128) * ceil_div(ncols, 128);
  const int num_sms = device_sm_count();
  if (ctas_big >= num_sms && ncols > 64) {
    dim3 grid(ceil_div(ncols, 128), ceil_div(p.M, 128));
    sgemm_nt_kernel<128, 128, 2, 2><<<grid, 256, 0, st>>>(p);
  } else if (ncols <= 64 && (long long)ceil_div(p.M, 128) >= num_sms) {
    dim3 grid(ceil_div(ncols, 64), ceil_div(p.M, 128));
    sgemm_nt_kernel<128, 64, 2, 1><<<grid, 256, 0, st>>>(p);
  } else {
    dim3 grid(ceil_div(ncols, 64), ceil_div(p.M, 64));
    sgemm_nt_kernel<64, 64, 1, 1><<<grid, 256, 0, st>>>(p);
  }
  GIB_LAUNCH_CHECK();
  return 0;
}

int gemm_nt_narrow(const GemmNT* ps, int n, cudaStream_t st) {
  NarrowGroup g;
  g.n = 0;
  double work = 0;
  for (int i = 0; i < n; ++i) {
    const GemmNT& p = ps[i];
    if (p.M <= 0 || p.N <= 0) continue;
    if (p.K % BK != 0 || (p.lda & 3) || (p.ldb & 3) || p.K <= 0 || p.m_dev || std::max(p.N, p.n_store) > kNarrowMaxN ||
        g.n == kNarrowMax) {
      set_error("gemm_nt_narrow: K=%d lda=%d ldb=%d N=%d n_store=%d (problem %d of %d) violate the narrow-kernel "
                "contract", p.K, p.lda, p.ldb, p.N, p.n_store, i, n);
      return -2;
    }
    g.p[g.n] = p;
    g.bn[g.n] = ceil_div(std::max(p.N, p.n_store), 16) * 16;
    ++g.n;
    work += p.work > 0 ? p.work : 2.0 * p.M * (double)p.N * p.K;
  }
  if (g.n == 0) return 0;
  // the most rows per thread that still gives every SM a CTA
  const int num_sms = device_sm_count();
  int tm = 4;
  for (;; tm >>= 1) {
    g.cta0[0] = 0;
    for (int i = 0; i < g.n; ++i) g.cta0[i + 1] = g.cta0[i] + ceil_div(g.p[i].M, kNarrowThreads / (g.bn[i] / 4) * tm);
    if (tm == 1 || g.cta0[g.n] >= num_sms) break;
  }
  ProfScope prof(PROF_GEMM_NT_SIMT, work, st);
  const int grid = g.cta0[g.n];
  if (tm == 4) sgemm_nt_narrow_kernel<4><<<grid, kNarrowThreads, 0, st>>>(g);
  else if (tm == 2) sgemm_nt_narrow_kernel<2><<<grid, kNarrowThreads, 0, st>>>(g);
  else sgemm_nt_narrow_kernel<1><<<grid, kNarrowThreads, 0, st>>>(g);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------
// dW partials:  P[z][n][k] = sum_{m in chunk z} G[m,n] * X[m,k]     (reduction over rows)
// bias partials: Pb[z][n]  = sum_{m in chunk z} G[m,n]
// ------------------------------------------------------------------------------------
template <int BM, int BN, int RM, int RN>
__global__ void __launch_bounds__(256, 2) sgemm_tn_splitk_kernel(const GemmTN p) {
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];
  const int tid = threadIdx.x;
  const int w = tid >> 5, l = tid & 31;
  const int ty = (w >> 1) * 4 + (l >> 3);
  const int tx = (w & 1) * 8 + (l & 7);
  const int n0 = blockIdx.y * BM;  // output row block (columns of G)
  const int k0 = blockIdx.x * BN;  // output col block (columns of X)
  const int z = blockIdx.z;
  const int m_begin = z * p.chunk_rows;
  const int m_end = min(p.M, m_begin + p.chunk_rows);

  constexpr int LA = BM / 64, LB = BN / 64;
  float4 ra[LA], rb[LB];
  auto gload = [&](int m0) {
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      int q = tid + i * 256, kk = q / (BM / 4), c = (q % (BM / 4)) * 4;
      bool ok = (m0 + kk) < m_end && (n0 + c) < p.Nn;
      ra[i] = ok ? __ldg(reinterpret_cast<const float4*>(p.G + (size_t)(m0 + kk) * p.ldg + n0 + c))
                 : make_float4(0, 0, 0, 0);
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      int q = tid + i * 256, kk = q / (BN / 4), c = (q % (BN / 4)) * 4;
      bool ok = (m0 + kk) < m_end && (k0 + c) < p.Kk;
      rb[i] = ok ? __ldg(reinterpret_cast<const float4*>(p.X + (size_t)(m0 + kk) * p.ldx + k0 + c))
                 : make_float4(0, 0, 0, 0);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      int q = tid + i * 256, kk = q / (BM / 4), c = (q % (BM / 4)) * 4;
      *reinterpret_cast<float4*>(&As[buf][kk][c]) = ra[i];
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      int q = tid + i * 256, kk = q / (BN / 4), c = (q % (BN / 4)) * 4;
      *reinterpret_cast<float4*>(&Bs[buf][kk][c]) = rb[i];
    }
  };

  float acc[RM][4][RN][4];
  float bacc[RM][4];
#pragma unroll
  for (int a = 0; a < RM; ++a)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      bacc[a][i] = 0.f;
#pragma unroll
      for (int b = 0; b < RN; ++b)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[a][i][b][j] = 0.f;
    }
  const bool do_bias = p.ws_bias != nullptr && blockIdx.x == 0 && (w & 1) == 0;  // warp-uniform

  const int ntiles = (m_end > m_begin) ? ceil_div(m_end - m_begin, BK) : 0;
  if (ntiles > 0) {
    gload(m_begin);
    sstore(0);
  }
  __syncthreads();
  for (int t = 0; t < ntiles; ++t) {
    const int buf = t & 1;
    if (t + 1 < ntiles) gload(m_begin + (t + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float4 fa[RM], fb[RN];
#pragma unroll
      for (int a = 0; a < RM; ++a)
        fa[a] = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4 + a * (BM / RM)]);
#pragma unroll
      for (int b = 0; b < RN; ++b)
        fb[b] = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4 + b * (BN / RN)]);
#pragma unroll
      for (int a = 0; a < RM; ++a) {
        const float av[4] = {fa[a].x, fa[a].y, fa[a].z, fa[a].w};
        if (do_bias) {
#pragma unroll
          for (int i = 0; i < 4; ++i) bacc[a][i] += av[i];
        }
#pragma unroll
        for (int b = 0; b < RN; ++b) {
          const float bv[4] = {fb[b].x, fb[b].y, fb[b].z, fb[b].w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[a][i][b][j] = fmaf(av[i], bv[j], acc[a][i][b][j]);
        }
      }
    }
    if (t + 1 < ntiles) sstore(buf ^ 1);
    __syncthreads();
  }

  float* out = p.ws + (size_t)z * p.Nn * p.Kk;
#pragma unroll
  for (int a = 0; a < RM; ++a)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int n = n0 + ty * 4 + a * (BM / RM) + i;
      if (n >= p.Nn) continue;
#pragma unroll
      for (int b = 0; b < RN; ++b) {
        const int k = k0 + tx * 4 + b * (BN / RN);
        if (k >= p.Kk) continue;
        *reinterpret_cast<float4*>(out + (size_t)n * p.Kk + k) =
            make_float4(acc[a][i][b][0], acc[a][i][b][1], acc[a][i][b][2], acc[a][i][b][3]);
      }
      if (do_bias && (l & 7) == 0) p.ws_bias[(size_t)z * p.Nn + n] = bacc[a][i];
    }
}

// Fixed-order reduction of the split partials into the gradient tensors, one launch for weight AND bias:
//   blocks [0, nblk_w):  dW[r*rs + c*cs] += sum_z ws[z][prow(r)][c]      (one thread per element, z ascending)
//   blocks [nblk_w, ..): db[r]           += sum_z wsb[z][prow(r)]        (32 rows per block, 8 partial chains)
// prow(r) = (r / Rb) * Rbp + r % Rb maps a real row to its padded (gate-blocked) row.
__global__ void __launch_bounds__(256) reduce_grads_kernel(const float* __restrict__ ws, int splits, int Nn, int Kk,
                                                           float* __restrict__ dW, int R, int C, int Rb, int Rbp,
                                                           long long rs, long long cs, int nblk_w,
                                                           const float* __restrict__ wsb, int bsplits,
                                                           float* __restrict__ db) {
  if ((int)blockIdx.x < nblk_w) {
    const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
    if (idx >= (long long)R * C) return;
    const int r = (int)(idx / C), c = (int)(idx % C);
    const int prow = (r / Rb) * Rbp + (r % Rb);
    const float* src = ws + (size_t)prow * Kk + c;
    const size_t stride = (size_t)Nn * Kk;
    float s = 0.f;
    int zi = 0;
    for (; zi + 8 <= splits; zi += 8) {      // 8 independent loads in flight, summed in ascending z
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = src[(size_t)(zi + u) * stride];
#pragma unroll
      for (int u = 0; u < 8; ++u) s += v[u];
    }
    for (; zi < splits; ++zi) s += src[(size_t)zi * stride];
    dW[r * rs + c * cs] += s;
  } else {
    __shared__ float sm[8][33];
    const int r = ((int)blockIdx.x - nblk_w) * 32 + (threadIdx.x & 31);
    const int wy = threadIdx.x >> 5;
    float s = 0.f;
    if (r < R) {
      const int prow = (r / Rb) * Rbp + (r % Rb);
      for (int zi = wy; zi < bsplits; zi += 8) s += wsb[(size_t)zi * Nn + prow];
    }
    sm[wy][threadIdx.x & 31] = s;
    __syncthreads();
    if (wy == 0 && r < R) {
      float t = 0.f;
      for (int k = 0; k < 8; ++k) t += sm[k][threadIdx.x];
      db[r] += t;
    }
  }
}

static int launch_reduce(const float* ws, int splits, const GemmDW& q, const float* wsb, int bsplits, cudaStream_t st) {
  const int nblk_w = q.dW ? (int)ceil_div_ll((long long)q.R * q.C, 256) : 0;
  const int nblk_b = q.dbias ? ceil_div(q.R, 32) : 0;
  if (nblk_w + nblk_b == 0) return 0;
  reduce_grads_kernel<<<nblk_w + nblk_b, 256, 0, st>>>(ws, splits, q.Nn, q.Kk, q.dW, q.R, q.C, q.Rb, q.Rbp, q.rs, q.cs,
                                                      nblk_w, wsb, bsplits, q.dbias);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ---- helper side stream ------------------------------------------------------------------------------------
// A tensor-core GEMM CTA leaves ~16K registers and some shared memory free on every SM -- room for a 256-thread block
// of the split reduction.  The reductions therefore run on a library-owned side stream (one per device),
// concurrently with the NEXT tensor-core launches of the main stream, instead of serialising ~10 us per layer:
//   job i (scratch half i&1):  main: [wait done(i-2)] partial products (+ bias partials) -> record tn(i)
//                              side: wait tn(i); fixed-order reduction into the gradients; record done(i)
// The side job reads only the scratch half (bias column sums come out of the GEMM), so the only hazard is the reuse
// of that half by job i+2.  dw_join() drains the side stream
// into the caller's stream; every C-ABI entry that uses gemm_dw calls dw_begin() first and dw_join() before
// returning, so the pattern is self-contained per call (fork / join: capturable in a CUDA graph).
// One thread per device at a time (the C-ABI contract: one host thread drives a device's model).
struct DwSide {
  cudaStream_t side = nullptr;
  cudaEvent_t ev_tn[2], ev_done[2];
  bool done_valid[2] = {false, false};
  long long calls = 0;
  int last = -1;         // half of the most recent job
};
static DwSide g_dw[64];
static std::mutex g_dw_mu;

static int dw_side(DwSide** out) {
  int dev = 0;
  GIB_CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) { set_error("device index %d out of range", dev); return -4; }
  std::lock_guard<std::mutex> lk(g_dw_mu);
  DwSide& d = g_dw[dev];
  if (!d.side) {
    GIB_CUDA_TRY(cudaStreamCreateWithFlags(&d.side, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
      GIB_CUDA_TRY(cudaEventCreateWithFlags(&d.ev_tn[i], cudaEventDisableTiming));
      GIB_CUDA_TRY(cudaEventCreateWithFlags(&d.ev_done[i], cudaEventDisableTiming));
    }
  }
  *out = &d;
  return 0;
}

int dw_begin() {
  DwSide* d;
  GIB_TRY(dw_side(&d));
  d->done_valid[0] = d->done_valid[1] = false;   // the previous call joined its jobs into its stream
  d->calls = 0; d->last = -1;
  return 0;
}

int dw_join(cudaStream_t st) {
  DwSide* d;
  GIB_TRY(dw_side(&d));
  if (d->last >= 0) {       // the side stream is in order: the last job's event covers all of them
    GIB_CUDA_TRY(cudaStreamWaitEvent(st, d->ev_done[d->last], 0));
    d->last = -1;
  }
  return 0;
}

size_t gemm_dw_half_floats(int M, int Nn, int Kk) {
  int splits, chunk;
  gemm_dw_plan(M, Nn, Kk, &splits, &chunk);
  const size_t f = ((size_t)splits * Nn * Kk + (size_t)splits * Nn + 63) & ~(size_t)63;
  GemmDW q; q.M = M; q.Nn = Nn; q.Kk = Kk;
  Dw3Layout L;
  tc3_dw_layout(&q, 1, &L);
  return std::max(f, (L.floats + 63) & ~(size_t)63);
}

size_t gemm_dw_scratch_floats(int M, int Nn, int Kk) {
  // two halves: the side stream may still be reducing job i while job i+1 writes its partials
  return 2 * gemm_dw_half_floats(M, Nn, Kk);
}

size_t gemm_dw_group_half_floats(const GemmDW* qs, int n) {
  size_t f = 0;
  for (int i = 0; i < n; ++i) f = std::max(f, gemm_dw_half_floats(qs[i].M, qs[i].Nn, qs[i].Kk));
  Dw3Layout L;
  tc3_dw_layout(qs, n, &L);
  return std::max(f, (L.floats + 63) & ~(size_t)63);
}

void gemm_dw_plan(int M, int Nn, int Kk, int* splits, int* chunk) {
  const int tiles = ceil_div(Nn, 128) * ceil_div(Kk, 128);
  int s = ceil_div(2 * device_sm_count(), tiles);
  const int max_s = ceil_div(M, 64) > 0 ? ceil_div(M, 64) : 1;  // >= 64 rows per split
  if (s > max_s) s = max_s;
  if (s < 1) s = 1;
  int c = ceil_div(ceil_div(M, s), BK) * BK;
  if (c < BK) c = BK;
  s = ceil_div(M, c);
  if (s < 1) s = 1;
  *splits = s;
  *chunk = c;
}

// one tensor-core launch (partials + bias partials of every member) on the caller's stream and one fixed-order
// reduction launch on the side stream
static int dw_tc_launch(const GemmDW* live, int nl, double work, const ProfRows* dyn_rows, int ndyn, cudaStream_t st) {
  ProfScope prof(PROF_GEMM_DW, work, st, dyn_rows, ndyn);
  DwSide* d;
  GIB_TRY(dw_side(&d));
  const int half = (int)(d->calls++ & 1);
  float* const scratch = live[0].scratch + (size_t)half * live[0].half_floats;
  Dw3Layout L;
  tc3_dw_layout(live, nl, &L);
  if (L.floats > live[0].half_floats) {
    set_error("gemm_dw_group: scratch half of %zu floats is too small for %zu", live[0].half_floats, L.floats);
    return -2;
  }
  if (d->done_valid[half]) GIB_CUDA_TRY(cudaStreamWaitEvent(st, d->ev_done[half], 0));   // job i-2 released this half
  GIB_TRY(gemm_dw_tc3_partials(live, nl, L, scratch, st));
  GIB_CUDA_TRY(cudaEventRecord(d->ev_tn[half], st));
  GIB_CUDA_TRY(cudaStreamWaitEvent(d->side, d->ev_tn[half], 0));
  GIB_TRY(gemm_dw_tc3_reduce(live, nl, L, scratch, d->side));
  GIB_CUDA_TRY(cudaEventRecord(d->ev_done[half], d->side));
  d->done_valid[half] = true;
  d->last = half;
  return 0;
}

// grouped weight gradients: one tensor-core launch + one reduction for the members that qualify, the others one by one
int gemm_dw_group(const GemmDW* qs, int n, cudaStream_t st) {
  if (n < 1) return 0;
  if (n > kDwMaxProblems) { set_error("gemm_dw_group: %d problems (max %d)", n, kDwMaxProblems); return -2; }
  for (int i = 0; i < n; ++i) GIB_TRY(check_precision(qs[i].tf32, "gemm_dw_group"));
  const bool tc3 = g_use_tc && use_tc3();
  bool dyn = false;
  long long rows = 0;
  double work = 0;
  ProfRows dyn_rows[kDwMaxProblems];
  int ndyn = 0;
  GemmDW live[kDwMaxProblems];       // members that run in the grouped tensor-core launch
  GemmDW rest[kDwMaxProblems];       // too small / unaligned for it: one by one
  int nl = 0, nr = 0;
  for (int i = 0; i < n; ++i) {
    const GemmDW& q = qs[i];
    if (q.M <= 0) continue;
    // (16-wide operands are eligible; narrower than 32 is only worth the launch when the row count is on the device)
    const bool good = tc3 && tc3_dw_eligible(q) && ((q.Nn >= 32 && q.Kk >= 32) || q.m_dev) &&
                      q.scratch == qs[0].scratch && q.half_floats == qs[0].half_floats;
    if (q.m_dev) {
      dyn = true;
      if (!good) {
        set_error("gemm_dw_group: device-side row counts need the tensor-core path (tensor cores on, aligned operands)");
        return -2;
      }
    }
    if (good) {
      rows += (long long)q.M * q.passes;
      const double qw = q.work > 0 ? q.work : 2.0 * q.M * (double)q.R * q.C * q.passes;
      if (q.m_dev) dyn_rows[ndyn++] = ProfRows{q.m_dev, q.base_dev, q.M, qw / q.M};   // the rows launched
      else work += qw;
      live[nl++] = q;
    } else {
      rest[nr++] = q;
    }
  }
  if (nl && !dyn && rows < 2048) {           // not worth a tensor-core launch
    for (int i = 0; i < nl; ++i) rest[nr++] = live[i];
    nl = 0;
  }
  for (int i = 0; i < nr; ++i) GIB_TRY(gemm_dw(rest[i], st));
  if (nl == 0) return 0;
  return dw_tc_launch(live, nl, work, dyn_rows, ndyn, st);
}

int dw_check_operands(const GemmDW& q, const char* who) {
  const char* bad = nullptr;
  if (reinterpret_cast<uintptr_t>(q.G) & 15) bad = "G is not 16-byte aligned";
  else if (reinterpret_cast<uintptr_t>(q.X) & 15) bad = "X is not 16-byte aligned";
  else if (q.passes > 1 && (q.pass_g & 3)) bad = "pass_g is not a multiple of 4";
  else if (q.passes > 1 && (q.pass_x & 3)) bad = "pass_x is not a multiple of 4";
  if (!bad) return 0;
  set_error("%s: %s", who, bad);
  return -2;
}

int gemm_dw(const GemmDW& q, cudaStream_t st) {
  if (q.M <= 0) return 0;  // nothing to add
  GIB_TRY(check_precision(q.tf32, "gemm_dw"));
  if ((q.ldg & 3) || (q.ldx & 3) || (q.Nn & 3) || (q.Kk & 3)) {
    set_error("gemm_dw: ldg=%d ldx=%d Nn=%d Kk=%d violate the padded-layout contract", q.ldg, q.ldx, q.Nn, q.Kk);
    return -2;
  }
  GIB_TRY(dw_check_operands(q, "gemm_dw"));
  if (q.m_dev) return gemm_dw_group(&q, 1, st);
  // the tensor-core launch as a group of one (also under gib_tc_debug bit 0, which groups no weight gradients)
  const double work = q.work > 0 ? q.work : 2.0 * q.M * (double)q.R * q.C * q.passes;
  if (g_use_tc && q.dW && (long long)q.M * q.passes >= 2048 && q.Nn >= 32 && q.Kk >= 32 && tc3_dw_eligible(q) &&
      q.half_floats > 0)
    return dw_tc_launch(&q, 1, work, nullptr, 0, st);
  if (q.passes > 1) {   // the SIMT kernel has no pass extent: one call per pass, last pass first as the backward runs
    for (int t = q.passes - 1; t >= 0; --t) {
      GemmDW s = q;
      s.passes = 1;
      s.G += t * q.pass_g; s.X += t * q.pass_x;
      s.work = work / q.passes;
      GIB_TRY(gemm_dw(s, st));
    }
    return 0;
  }
  ProfScope prof(PROF_GEMM_DW_SIMT, work, st);
  DwSide* d;
  GIB_TRY(dw_side(&d));
  const int half = (int)(d->calls++ & 1);
  float* const scratch = q.scratch + (size_t)half * q.half_floats;
  if (d->done_valid[half]) GIB_CUDA_TRY(cudaStreamWaitEvent(st, d->ev_done[half], 0));   // job i-2 released this half
  GIB_TRY(dw_join(st));               // fp32 SIMT path: everything on the caller's stream, nothing left pending
  int splits, chunk;
  gemm_dw_plan(q.M, q.Nn, q.Kk, &splits, &chunk);
  GemmTN p;
  p.G = q.G; p.ldg = q.ldg; p.X = q.X; p.ldx = q.ldx; p.M = q.M; p.Nn = q.Nn; p.Kk = q.Kk;
  p.chunk_rows = chunk;
  p.ws = scratch;
  p.ws_bias = q.dbias ? scratch + (size_t)splits * q.Nn * q.Kk : nullptr;
  if (q.dW) {
    dim3 grid(ceil_div(q.Kk, 128), ceil_div(q.Nn, 128), splits);
    sgemm_tn_splitk_kernel<128, 128, 2, 2><<<grid, 256, 0, st>>>(p);
    GIB_LAUNCH_CHECK();
  } else if (q.dbias) {  // bias only: run one k-tile column
    GemmTN pb = p;
    pb.Kk = 4;  // minimal X extent; acc discarded (the ws slab holds >= Nn*4 floats per split: Kk >= 16 everywhere)
    dim3 grid(1, ceil_div(q.Nn, 128), splits);
    sgemm_tn_splitk_kernel<128, 128, 2, 2><<<grid, 256, 0, st>>>(pb);
    GIB_LAUNCH_CHECK();
  }
  GIB_TRY(launch_reduce(p.ws, splits, q, p.ws_bias, splits, st));
  return 0;
}

}  // namespace gib
