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
constexpr int kColsumSplits = 296;  // row chunks (one block each) of the two-stage bias-gradient column sum

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
  const bool vec_c = (p.ldc & 3) == 0 && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0);
  const bool vec_x = p.aux && (p.ldaux & 3) == 0 && ((reinterpret_cast<uintptr_t>(p.aux) & 15) == 0);
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
        float v[4] = {acc[a][i][b][0], acc[a][i][b][1], acc[a][i][b][2], acc[a][i][b][3]};
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

int gemm_nt(const GemmNT& p, cudaStream_t st) {
  GIB_TRY(check_precision(p.tf32, "gemm_nt"));
  // tensor-core path for all but the tiny / skinny GEMMs (those stay on the SIMT kernel); a problem whose row count
  // lives on the device (capacity mode) needs the grouped call pattern
  if (p.m_dev) {
    if (!g_use_tc || !use_tc3() || !tc3_eligible(p)) {
      set_error("gemm_nt: device-side row counts need the tensor-core path (tensor cores on, pre-split weights)");
      return -2;
    }
    return gemm_nt_tc3_group(&p, 1, st);
  }
  if (g_use_tc && p.N >= 48 && p.K >= 32) {
    if (use_tc3() && p.M >= 256 && tc3_eligible(p)) return gemm_nt_tc3_group(&p, 1, st);
    if (p.M >= 1024 && tc_eligible(p)) return gemm_nt_tc(p, st);
  }
  // Narrow outputs (the APD heads: 1024 x 500 -> 39 / 3 / 1) stay on the fp32 SIMT kernel unless debug bit 2 is set:
  // a handful of tensor-core tiles would be faster, but the output layer's 3xTF32 error lands on the logits
  // unattenuated, and on the shipped checkpoint x 256 gdb13 rows the logit error is already close to the 1e-4 contract
  // with this layer in fp32 (tests/test_gpu_parity.py::test_pretrained_checkpoint_on_real_gdb13_rows).
  if (g_use_tc && use_tc3() && (g_tc_debug & 4) && p.N < 48 && p.K >= 128 && p.M >= 256 && tc3_eligible(p))
    return gemm_nt_tc3_group(&p, 1, st);
  return gemm_nt_simt(p, st);
}

// Several independent problems (sibling MLPs, the per-bond-type message MLPs): one grouped tensor-core launch when
// together they fill the machine reasonably, else problem by problem.
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
  for (int i = 0; i < n; ++i) GIB_TRY(gemm_nt(ps[i], st));
  return 0;
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

// part[z][n] = sum over the z-th row chunk of G[m, n]  (fixed order inside the chunk; chunks reduced in order).
// One block per row chunk, whole rows read with float4 (fully coalesced); thread t owns float4 column t % (Nn/4) and
// every (256 / (Nn/4))-th row of the chunk, partial sums meet in shared memory in a fixed order.
__global__ void __launch_bounds__(256) colsum_partial_kernel(float* __restrict__ part, const float* __restrict__ G,
                                                             int ldg, int M, int Nn) {
  __shared__ float4 sm[256];
  const int n4 = Nn >> 2;                       // float4 columns per row (Nn is a multiple of 16)
  const int rows = ceil_div(M, (int)gridDim.x);
  const int m0 = blockIdx.x * rows, m1 = min(M, m0 + rows);
  for (int c0 = 0; c0 < n4; c0 += 256) {        // Nn <= 1024 handled in one sweep per 256 float4 columns
    const int width = min(256, n4 - c0);        // active float4 columns in this sweep
    const int lanes = 256 / width;              // row lanes sharing the sweep
    const int col = threadIdx.x % width, rl = threadIdx.x / width;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (rl < lanes) {
      int m = m0 + rl;
      for (; m + 3 * lanes < m1; m += 4 * lanes) {      // four row loads in flight, summed in ascending row order
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u)
          v[u] = __ldg(reinterpret_cast<const float4*>(G + (size_t)(m + u * lanes) * ldg) + c0 + col);
#pragma unroll
        for (int u = 0; u < 4; ++u) { acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w; }
      }
      for (; m < m1; m += lanes) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(G + (size_t)m * ldg) + c0 + col);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    }
    sm[threadIdx.x] = acc;
    __syncthreads();
    if (rl == 0) {
      float4 t = sm[col];
      for (int k = 1; k < lanes; ++k) {
        const float4 u = sm[k * width + col];
        t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
      }
      reinterpret_cast<float4*>(part + (size_t)blockIdx.x * Nn)[c0 + col] = t;
    }
    __syncthreads();
  }
}

// ---- helper side stream ------------------------------------------------------------------------------------
// A tensor-core GEMM CTA leaves ~16K registers and some shared memory free on every SM -- room for a 256-thread block
// of the split reduction.  The reductions therefore run on a library-owned side stream (one per device),
// concurrently with the NEXT tensor-core launches of the main stream, instead of serialising ~10 us per layer:
//   job i (scratch half i&1):  main: [wait done(i-2)] partial products (+ bias partials) -> record tn(i)
//                              side: wait tn(i); fixed-order reduction into the gradients; record done(i)
// Second-generation kernel: the side job reads only the scratch half (bias column sums come out of the GEMM), so the
// only hazard is the reuse of that half by job i+2.  First-generation kernel: the side job also reads the G operand
// (column sums), hence the extra wait before the caller's next dX GEMM (g_pending).  dw_join() drains the side stream
// into the caller's stream; every C-ABI entry that uses gemm_dw calls dw_begin() first and dw_join() before
// returning, so the pattern is self-contained per call (fork / join: capturable in a CUDA graph).
// One thread per device at a time (the C-ABI contract: one host thread drives a device's model).
struct DwSide {
  cudaStream_t side = nullptr;
  cudaEvent_t ev_tn[2], ev_done[2];
  bool done_valid[2] = {false, false};
  long long calls = 0;
  int pending = -1;      // first generation: job whose completion the main stream has not waited for yet
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
  d->calls = 0; d->pending = -1; d->last = -1;
  return 0;
}

int dw_join(cudaStream_t st) {
  DwSide* d;
  GIB_TRY(dw_side(&d));
  if (d->last >= 0) {       // the side stream is in order: the last job's event covers all of them
    GIB_CUDA_TRY(cudaStreamWaitEvent(st, d->ev_done[d->last], 0));
    d->last = -1; d->pending = -1;
  }
  return 0;
}

size_t gemm_dw_half_floats(int M, int Nn, int Kk) {
  int splits, chunk, s2, c2;
  gemm_dw_plan(M, Nn, Kk, &splits, &chunk);
  tc_dw_plan(M, Nn, Kk, &s2, &c2);       // the tensor-core path may pick a different split count
  if (s2 > splits) splits = s2;
  size_t f = (((size_t)splits * Nn * Kk + (size_t)(splits > kColsumSplits ? splits : kColsumSplits) * Nn) + 63) & ~(size_t)63;
  GemmDW q; q.M = M; q.Nn = Nn; q.Kk = Kk;
  Dw3Layout L;
  tc3_dw_layout(&q, 1, tc3_dw_chunk_rows(&q, 1, 0), &L);
  return std::max(f, (L.floats + 63) & ~(size_t)63);
}

size_t gemm_dw_scratch_floats(int M, int Nn, int Kk) {
  // two halves: the side stream may still be reducing job i while job i+1 writes its partials
  return 2 * gemm_dw_half_floats(M, Nn, Kk);
}

size_t gemm_dw_group_half_floats(const GemmDW* qs, int n, long long plan_rows) {
  size_t f = 0;
  for (int i = 0; i < n; ++i) f = std::max(f, gemm_dw_half_floats(qs[i].M, qs[i].Nn, qs[i].Kk));
  Dw3Layout L;
  tc3_dw_layout(qs, n, tc3_dw_chunk_rows(qs, n, plan_rows), &L);
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

// grouped weight gradients: one tensor-core launch (partials + bias partials of every member) on the caller's stream and
// one fixed-order reduction launch on the side stream; falls back to member-by-member when the group is not eligible
int gemm_dw_group(const GemmDW* qs, int n, long long plan_rows, cudaStream_t st) {
  if (n < 1) return 0;
  if (n > kTc3MaxProblems) { set_error("gemm_dw_group: %d problems (max %d)", n, kTc3MaxProblems); return -2; }
  for (int i = 0; i < n; ++i) GIB_TRY(check_precision(qs[i].tf32, "gemm_dw_group"));
  const bool tc3 = g_use_tc && use_tc3();
  bool dyn = false;
  long long rows = 0;
  double work = 0;
  ProfRows dyn_rows[kTc3MaxProblems];
  int ndyn = 0;
  GemmDW live[kTc3MaxProblems];      // members that run in the grouped tensor-core launch
  GemmDW rest[kTc3MaxProblems];      // too small / unaligned for it: one by one
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
      rows += q.M;
      const double qw = q.work > 0 ? q.work : 2.0 * q.M * (double)q.R * q.C;
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
  ProfScope prof(PROF_GEMM_DW, work, st, dyn_rows, ndyn);
  DwSide* d;
  GIB_TRY(dw_side(&d));
  const int half = (int)(d->calls++ & 1);
  float* const scratch = live[0].scratch + (size_t)half * live[0].half_floats;
  Dw3Layout L;       // chunk from ALL members (as the scratch was sized), offsets for the grouped ones
  tc3_dw_layout(live, nl, tc3_dw_chunk_rows(qs, n, plan_rows), &L);
  if (L.floats > live[0].half_floats) {
    set_error("gemm_dw_group: scratch half of %zu floats is too small for %zu", live[0].half_floats, L.floats);
    return -2;
  }
  if (d->pending >= 0) {      // a first-generation job still reads its G operand: finish it first
    GIB_CUDA_TRY(cudaStreamWaitEvent(st, d->ev_done[d->pending], 0));
    d->pending = -1;
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

int gemm_dw(const GemmDW& q, cudaStream_t st) {
  if (q.M <= 0) return 0;  // nothing to add
  GIB_TRY(check_precision(q.tf32, "gemm_dw"));
  if ((q.ldg & 3) || (q.ldx & 3) || (q.Nn & 3) || (q.Kk & 3)) {
    set_error("gemm_dw: ldg=%d ldx=%d Nn=%d Kk=%d violate the padded-layout contract", q.ldg, q.ldx, q.Nn, q.Kk);
    return -2;
  }
  if (q.m_dev || (g_use_tc && use_tc3() && q.dW && q.M >= 2048 && q.Nn >= 32 && q.Kk >= 32 && tc3_dw_eligible(q) &&
                  q.half_floats > 0))
    return gemm_dw_group(&q, 1, 0, st);
  const bool tc = g_use_tc && q.dW && tc_dw_eligible(q);
  ProfScope prof(tc ? PROF_GEMM_DW : PROF_GEMM_DW_SIMT, q.work > 0 ? q.work : 2.0 * q.M * (double)q.R * q.C, st);
  DwSide* d;
  GIB_TRY(dw_side(&d));
  const int half = (int)(d->calls++ & 1);
  float* const scratch = q.scratch + (size_t)half * q.half_floats;
  if (d->done_valid[half]) GIB_CUDA_TRY(cudaStreamWaitEvent(st, d->ev_done[half], 0));   // job i-2 released this half
  if (tc) {
    // per-problem tensor-core partials (MN-major operands straight from the row-major activations) on the main
    // stream; bias column sums + the fixed-order split reduction on the side stream
    int tsplits = 0;
    GemmDW q2 = q;
    q2.scratch = scratch;
    GIB_TRY(gemm_dw_tc_partials(q2, &tsplits, st));
    GIB_CUDA_TRY(cudaEventRecord(d->ev_tn[half], st));
    GIB_CUDA_TRY(cudaStreamWaitEvent(d->side, d->ev_tn[half], 0));
    float* part = scratch + (size_t)tsplits * q.Nn * q.Kk;         // [kColsumSplits][Nn] partial column sums
    if (q.dbias) {
      colsum_partial_kernel<<<kColsumSplits, 256, 0, d->side>>>(part, q.G, q.ldg, q.M, q.Nn);
      GIB_LAUNCH_CHECK();
    }
    GIB_TRY(launch_reduce(scratch, tsplits, q, part, kColsumSplits, d->side));
    GIB_CUDA_TRY(cudaEventRecord(d->ev_done[half], d->side));
    d->done_valid[half] = true;
    const int prev = d->pending;      // the job before this one must be complete before the caller's next dX GEMM
    d->pending = half;
    d->last = half;
    if (prev >= 0 && prev != half) GIB_CUDA_TRY(cudaStreamWaitEvent(st, d->ev_done[prev], 0));
    return 0;
  }
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
