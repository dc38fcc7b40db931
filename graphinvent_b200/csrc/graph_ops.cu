// HBM-bound kernels of the hot path: bond-entry gather, segmented scatter-aggregate (K2),
// segmented softmax-aggregate (K2'), GRU gates, graph-gather readout, concat/flatten glue,
// parameter packing.  All index reads are coalesced int32, all row traffic is float4, every
// reduction runs in a fixed order (no float atomics) so results are run-to-run bit-stable.
#include "ops.cuh"
#include "prof.cuh"

namespace gib {

#define GIB_1D(total, threads) (unsigned)ceil_div_ll((long long)(total), (threads)), (threads)

// Live rows of a buffer of `rows` bond rows.  Capacity mode passes the device int K0 wrote (the entry count of the
// one untyped EMN group): the grid is sized from the capacity, and the threads at or past the live count exit before
// any index load.  A count above the capacity (an overflowing batch) is clamped to it.  live == nullptr (exact mode):
// every row is live.
__device__ __forceinline__ long long live_rows(const int* live, long long rows) {
  if (!live) return rows;
  const long long n = __ldg(live);
  return n < 0 ? 0 : (n < rows ? n : rows);
}

// ------------------------------------------------------------------------------------
// concat2: dst[r, :] = [ a[r, :wa] | b[r, :wb] | 0 ... ]      (dst width = ldd)
// reference: summation_mpnn.py:121-125 (zero-pad node features), modules.py:46 (cat(hidden, input))
// ------------------------------------------------------------------------------------
// Either source may be the int8 input tensor of the reference's on-disk format (i8 flags): it is widened here, in the
// first kernel that touches it, instead of by a host-side cast (BlockDatasetLoader.py:139-143).
__device__ __forceinline__ float ld_in(const void* p, size_t i, int i8) {
  return i8 ? (float)__ldg(reinterpret_cast<const signed char*>(p) + i) : __ldg(reinterpret_cast<const float*>(p) + i);
}
__global__ void concat2_kernel(float* __restrict__ dst, int ldd, const void* __restrict__ a, int lda, int wa, int a_i8,
                               const void* __restrict__ b, int ldb, int wb, int b_i8, long long rows) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * ldd) return;
  const long long r = idx / ldd;
  const int c = (int)(idx % ldd);
  float v = 0.f;
  if (c < wa) v = ld_in(a, (size_t)r * lda + c, a_i8);
  else if (c < wa + wb) v = ld_in(b, (size_t)r * ldb + (c - wa), b_i8);
  dst[idx] = v;
}
int concat2_in(float* dst, int ldd, const void* a, int lda, int wa, int a_i8, const void* b, int ldb, int wb, int b_i8,
               long long rows, cudaStream_t st) {
  if (rows <= 0) return 0;
  concat2_kernel<<<GIB_1D(rows * ldd, 256), 0, st>>>(dst, ldd, a, lda, wa, a_i8, b, ldb, wb, b_i8, rows);
  GIB_LAUNCH_CHECK();
  return 0;
}
int concat2(float* dst, int ldd, const float* a, int lda, int wa, const float* b, int ldb, int wb, long long rows,
            cudaStream_t st) {
  return concat2_in(dst, ldd, a, lda, wa, 0, b, ldb, wb, 0, rows, st);
}

// dst[b, :] = [ flatten_i( f1[b*N + i, :fa] ) | g[b, :W] | 0 ]      (modules.py:257-268)
__global__ void concat_flat_kernel(float* __restrict__ dst, int ldd, const float* __restrict__ f1, int ldf, int N,
                                   int fa, const float* __restrict__ g, int ldg, int W, int B) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * ldd) return;
  const int b = (int)(idx / ldd), c = (int)(idx % ldd);
  float v = 0.f;
  if (c < N * fa) v = f1[((size_t)b * N + c / fa) * ldf + c % fa];
  else if (c < N * fa + W) v = g[(size_t)b * ldg + (c - N * fa)];
  dst[idx] = v;
}
int concat_flat(float* dst, int ldd, const float* f1, int ldf, int N, int fa, const float* g, int ldg, int W, int B,
                cudaStream_t st) {
  concat_flat_kernel<<<GIB_1D((long long)B * ldd, 256), 0, st>>>(dst, ldd, f1, ldf, N, fa, g, ldg, W, B);
  GIB_LAUNCH_CHECK();
  return 0;
}

// G1[(b,i), a] = dcat[b, i*fa + a] * selu'(f1[(b,i), a])   (a < fa; pad columns 0)
__global__ void unflatten_dact_kernel(float* __restrict__ G, int ldf, const float* __restrict__ dcat, int ldd,
                                      const float* __restrict__ f1, int N, int fa, long long S) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= S * ldf) return;
  const long long s = idx / ldf;
  const int a = (int)(idx % ldf);
  float v = 0.f;
  if (a < fa) {
    const long long b = s / N;
    const int i = (int)(s % N);
    v = dcat[b * ldd + i * fa + a] * dselu_from_out(f1[idx]);
  }
  G[idx] = v;
}
int unflatten_dact(float* G, int ldf, const float* dcat, int ldd, const float* f1, int N, int fa, long long S,
                   cudaStream_t st) {
  unflatten_dact_kernel<<<GIB_1D(S * ldf, 256), 0, st>>>(G, ldf, dcat, ldd, f1, N, fa, S);
  GIB_LAUNCH_CHECK();
  return 0;
}

// G[m, n] = dOut[m, off + n] * act'(out[m, off + n])  (n < width; pad columns 0)
__global__ void dact_slice_kernel(float* __restrict__ G, int ldg, const float* __restrict__ dout,
                                  const float* __restrict__ out, int ldo, int off, int width, int act, int rows) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)rows * ldg) return;
  const int m = (int)(idx / ldg), n = (int)(idx % ldg);
  float v = 0.f;
  if (n < width) {
    const size_t o = (size_t)m * ldo + off + n;
    v = dout[o] * dact_from_out(out[o], act);
  }
  G[idx] = v;
}
int dact_slice(float* G, int ldg, const float* dout, const float* out, int ldo, int off, int width, int act, int rows,
               cudaStream_t st) {
  dact_slice_kernel<<<GIB_1D((long long)rows * ldg, 256), 0, st>>>(G, ldg, dout, out, ldo, off, width, act, rows);
  GIB_LAUNCH_CHECK();
  return 0;
}

// dg[b, c] = a[b, offa + c] + b2[b, offb + c] + c3[b, c]   (c < W, pad 0)
__global__ void sum3_cols_kernel(float* __restrict__ dst, int ldd, int W, const float* __restrict__ a, int lda,
                                 int offa, const float* __restrict__ b2, int ldb, int offb,
                                 const float* __restrict__ c3, int ldc, int rows) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)rows * ldd) return;
  const int r = (int)(idx / ldd), c = (int)(idx % ldd);
  float v = 0.f;
  if (c < W) {
    if (a) v += a[(size_t)r * lda + offa + c];
    if (b2) v += b2[(size_t)r * ldb + offb + c];
    if (c3) v += c3[(size_t)r * ldc + c];
  }
  dst[idx] = v;
}
int sum3_cols(float* dst, int ldd, int W, const float* a, int lda, int offa, const float* b2, int ldb, int offb,
              const float* c3, int ldc, int rows, cudaStream_t st) {
  sum3_cols_kernel<<<GIB_1D((long long)rows * ldd, 256), 0, st>>>(dst, ldd, W, a, lda, offa, b2, ldb, offb, c3, ldc,
                                                                  rows);
  GIB_LAUNCH_CHECK();
  return 0;
}

// y = tanh(x) elementwise over rows x ld (EMN edge embedding, mpnn.py:469), and its backward
__global__ void tanh_fwd_kernel(float* __restrict__ y, const float* __restrict__ x, long long rows, int ld,
                                const int* __restrict__ live) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < live_rows(live, rows) * ld) y[i] = tanhf(x[i]);
}
int tanh_fwd(float* y, const float* x, long long rows, int ld, const int* live, cudaStream_t st) {
  if (rows <= 0) return 0;
  tanh_fwd_kernel<<<GIB_1D(rows * ld, 256), 0, st>>>(y, x, rows, ld, live);
  GIB_LAUNCH_CHECK();
  return 0;
}
// G = dy * (1 - y^2) * selu'(pre)   where pre is the SELU output that fed tanh
__global__ void tanh_selu_bwd_kernel(float* __restrict__ G, const float* __restrict__ dy, const float* __restrict__ y,
                                     const float* __restrict__ pre, long long rows, int ld,
                                     const int* __restrict__ live) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < live_rows(live, rows) * ld) G[i] = dy[i] * (1.f - y[i] * y[i]) * dselu_from_out(pre[i]);
}
int tanh_selu_bwd(float* G, const float* dy, const float* y, const float* pre, long long rows, int ld,
                  const int* live, cudaStream_t st) {
  if (rows <= 0) return 0;
  tanh_selu_bwd_kernel<<<GIB_1D(rows * ld, 256), 0, st>>>(G, dy, y, pre, rows, ld, live);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------
// gather_rows: X0[p, :] = (scale ? w_p : 1) * h[src_p, :]      (pad rows -> 0; rows at or past *live are not written)
// reference: summation_mpnn.py:131 (`hidden_nodes[b, nghb]`) + mpnn.py:286-288 (edge-value scaling)
// ------------------------------------------------------------------------------------
__global__ void gather_rows_kernel(float4* __restrict__ dst, const float4* __restrict__ h, int ld4,
                                   const int* __restrict__ src, const float* __restrict__ w, int scale, long long P,
                                   const int* __restrict__ live) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= live_rows(live, P) * ld4) return;
  const long long p = idx / ld4;
  const int c = (int)(idx % ld4);
  const int s = __ldg(src + p);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (s >= 0) {
    v = __ldg(h + (size_t)s * ld4 + c);
    if (scale && w) {
      const float ww = __ldg(w + p);
      v.x *= ww; v.y *= ww; v.z *= ww; v.w *= ww;
    }
  }
  dst[idx] = v;
}
int gather_rows(float* dst, const float* h, int ld, const int* src, const float* w, int scale, long long P,
                const int* live, cudaStream_t st) {
  if (P <= 0) return 0;
  gather_rows_kernel<<<GIB_1D(P * (ld / 4), 256), 0, st>>>(reinterpret_cast<float4*>(dst),
                                                          reinterpret_cast<const float4*>(h), ld / 4, src, w, scale, P,
                                                          live);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------
// K2  segmented scatter-aggregate:  out[s, :] (+)= sum_{q in [ptr[s], ptr[s+1])} w[ent[q]] * msg[ent[q], :]
// Replaces the dense [V,E] x [E,msg] matmul of summation_mpnn.py:141.  One thread per
// (slot, float4 column); the threads of a row share the index reads (warp broadcast), each
// entry row is one contiguous 16*ld4-byte read, each output row one contiguous write.
// Algorithmic bytes per launch: E*ld*4 (messages) + S*ld*4 (aggregates) + (S+1)*4 + E*8 (indices, w).
// ------------------------------------------------------------------------------------
// Streaming access hints: message rows are read exactly once and aggregates written exactly once per launch, so they
// should not displace the (re-used) index arrays in L2: ld.global.cs / st.global.cs (evict-first).
template <int HINT> __device__ __forceinline__ float4 ld_row(const float4* p) {
  if (HINT) return __ldcs(p);
  return __ldg(p);
}
template <int HINT> __device__ __forceinline__ void st_row(float4* p, const float4& v) {
  if (HINT) __stcs(p, v);
  else *p = v;
}

// SLOTS slots per thread, interleaved level by level (row pointers of all slots, then their entry indices, then their
// message rows) so that a thread has SLOTS x 4 row reads in flight instead of 4: the kernel is latency-bound (ncu:
// 77 % of the warps resident, DRAM 51 % busy), each extra independent load chain hides one more round trip.
// Y != null: the backward of the message rows (seg_reduce_dact) instead of an aggregate -- out[s] = row_w[s] * acc *
// act'(Y[s]), and an empty segment (a pad row) is written as exact 0 without reading Y.
template <int SLOTS, int HINT>
__global__ void __launch_bounds__(256) scatter_sum_kernel(float4* __restrict__ out, const float4* __restrict__ msg,
                                                          int ld4, const int* __restrict__ ptr,
                                                          const int* __restrict__ ent, const float* __restrict__ w,
                                                          int accumulate, long long S, long long slots_per_pass,
                                                          const float* __restrict__ row_w,
                                                          const float4* __restrict__ Y, int act) {
  const long long idx0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx0 >= slots_per_pass * ld4) return;
  const long long s0 = idx0 / ld4;
  const int c = (int)(idx0 % ld4);
  long long s[SLOTS];
  int q0[SLOTS], q1[SLOTS];
  float4 acc[SLOTS];
#pragma unroll
  for (int k = 0; k < SLOTS; ++k) {
    s[k] = s0 + (long long)k * slots_per_pass;       // slot k of this thread: one "pass" further down
    const bool live = s[k] < S;
    q0[k] = live ? __ldg(ptr + s[k]) : 0;
    q1[k] = live ? __ldg(ptr + s[k] + 1) : 0;
  }
#pragma unroll
  for (int k = 0; k < SLOTS; ++k)
    acc[k] = (accumulate && s[k] < S) ? out[s[k] * ld4 + c] : make_float4(0.f, 0.f, 0.f, 0.f);
  // 4 entries per slot and trip: the index loads, then the row loads, are issued back to back (molecular graphs:
  // degree <= 4 almost always -> one trip).  Accumulation stays ascending in q: bit-stable results.
  bool more = true;
  for (int trip = 0; more; ++trip) {
    int p[SLOTS][4];
    float ww[SLOTS][4];
    float4 v[SLOTS][4];
    more = false;
#pragma unroll
    for (int k = 0; k < SLOTS; ++k)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int q = q0[k] + trip * 4 + u;
        p[k][u] = (q < q1[k]) ? __ldg(ent + q) : -1;
      }
#pragma unroll
    for (int k = 0; k < SLOTS; ++k)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        ww[k][u] = (p[k][u] >= 0 && w) ? __ldg(w + p[k][u]) : 1.f;
        v[k][u] = (p[k][u] >= 0) ? ld_row<HINT>(msg + (size_t)p[k][u] * ld4 + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
    for (int k = 0; k < SLOTS; ++k) {
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (p[k][u] >= 0) {
          acc[k].x = fmaf(ww[k][u], v[k][u].x, acc[k].x); acc[k].y = fmaf(ww[k][u], v[k][u].y, acc[k].y);
          acc[k].z = fmaf(ww[k][u], v[k][u].z, acc[k].z); acc[k].w = fmaf(ww[k][u], v[k][u].w, acc[k].w);
        }
      if (q0[k] + (trip + 1) * 4 < q1[k]) more = true;
    }
  }
#pragma unroll
  for (int k = 0; k < SLOTS; ++k)
    if (s[k] < S) {
      if (Y) {
        float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
        if (q1[k] > q0[k]) {
          const float ww = row_w ? __ldg(row_w + s[k]) : 1.f;
          const float4 y = __ldg(Y + s[k] * ld4 + c);
          g.x = ww * acc[k].x * dact_from_out(y.x, act); g.y = ww * acc[k].y * dact_from_out(y.y, act);
          g.z = ww * acc[k].z * dact_from_out(y.z, act); g.w = ww * acc[k].w * dact_from_out(y.w, act);
        }
        acc[k] = g;
      }
      st_row<HINT>(out + s[k] * ld4 + c, acc[k]);
    }
}

// tools/k2_variants.py times the variants at the C4 shape
int g_scatter_variant = 2;     // 0: 1 slot / thread, default caching   1: 2 slots   2: 1 slot + streaming hints   3: 2 slots + hints

static int scatter_launch(float* out, const float* msg, int ld, const int* ptr, const int* ent, const float* w,
                          int accumulate, long long S, const float* row_w, const float* Y, int act, cudaStream_t st) {
  float4* o = reinterpret_cast<float4*>(out);
  const float4* m = reinterpret_cast<const float4*>(msg);
  const float4* y = reinterpret_cast<const float4*>(Y);
  const int ld4 = ld / 4;
  const int slots = (g_scatter_variant & 1) ? 2 : 1;
  const long long per_pass = ceil_div_ll(S, slots);
  const unsigned grid = (unsigned)ceil_div_ll(per_pass * ld4, 256);
  switch (g_scatter_variant & 3) {
    case 0: scatter_sum_kernel<1, 0><<<grid, 256, 0, st>>>(o, m, ld4, ptr, ent, w, accumulate, S, per_pass, row_w, y, act); break;
    case 1: scatter_sum_kernel<2, 0><<<grid, 256, 0, st>>>(o, m, ld4, ptr, ent, w, accumulate, S, per_pass, row_w, y, act); break;
    case 2: scatter_sum_kernel<1, 1><<<grid, 256, 0, st>>>(o, m, ld4, ptr, ent, w, accumulate, S, per_pass, row_w, y, act); break;
    default: scatter_sum_kernel<2, 1><<<grid, 256, 0, st>>>(o, m, ld4, ptr, ent, w, accumulate, S, per_pass, row_w, y, act); break;
  }
  GIB_LAUNCH_CHECK();
  return 0;
}

int scatter_sum(float* out, const float* msg, int ld, const int* ptr, const int* ent, const float* w, int accumulate,
                long long S, cudaStream_t st, double bytes) {
  if (S <= 0) return 0;
  ProfScope prof(PROF_SCATTER, bytes, st);   // algorithmic bytes (SURVEY.md 8d) when the caller knows the entry count
  return scatter_launch(out, msg, ld, ptr, ent, w, accumulate, S, nullptr, nullptr, ACT_NONE, st);
}

int seg_reduce_dact(float* G, const float* dM, const float* Y, int ld, const int* ptr, const int* ent,
                    const float* row_w, int act, long long rows, cudaStream_t st) {
  if (rows <= 0) return 0;
  return scatter_launch(G, dM, ld, ptr, ent, nullptr, 0, rows, row_w, Y, act, st);
}

// backward of K2 (gather-broadcast) fused with the activation derivative of the message MLP's
// last layer:  G[p, :] = w_p * dM[dst_p, :] * act'(Y[p, :])     (pad rows -> 0)
__global__ void scatter_bwd_kernel(float4* __restrict__ G, const float4* __restrict__ dM, const float4* __restrict__ Y,
                                   int ld4, const int* __restrict__ dst, const float* __restrict__ w, int act,
                                   long long P) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P * ld4) return;
  const long long p = idx / ld4;
  const int c = (int)(idx % ld4);
  const int s = __ldg(dst + p);
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  if (s >= 0) {
    const float ww = w ? __ldg(w + p) : 1.f;
    const float4 d = __ldg(dM + (size_t)s * ld4 + c);
    const float4 y = __ldg(Y + idx);
    g.x = ww * d.x * dact_from_out(y.x, act); g.y = ww * d.y * dact_from_out(y.y, act);
    g.z = ww * d.z * dact_from_out(y.z, act); g.w = ww * d.w * dact_from_out(y.w, act);
  }
  G[idx] = g;
}
int scatter_bwd(float* G, const float* dM, const float* Y, int ld, const int* dst, const float* w, int act,
                long long P, cudaStream_t st) {
  if (P <= 0) return 0;
  scatter_bwd_kernel<<<GIB_1D(P * (ld / 4), 256), 0, st>>>(reinterpret_cast<float4*>(G),
                                                          reinterpret_cast<const float4*>(dM),
                                                          reinterpret_cast<const float4*>(Y), ld / 4, dst, w, act, P);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------
// K2'  segmented softmax-aggregate (AttentionGGNN, mpnn.py:370-389): per destination slot and
// per channel, softmax over the incoming entries of  w*EN  applied to  w*EM.
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) seg_softmax_fwd_kernel(float* __restrict__ out, const float* __restrict__ EM,
                                                              const float* __restrict__ EN, int ld,
                                                              const int* __restrict__ ptr, const int* __restrict__ ent,
                                                              const float* __restrict__ w, long long S) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= S * ld) return;
  const long long s = idx / ld;
  const int c = (int)(idx % ld);
  const int q0 = __ldg(ptr + s), q1 = __ldg(ptr + s + 1);
  float res = 0.f;
  if (q1 > q0) {
    float mx = -INFINITY;
    for (int q = q0; q < q1; ++q) {
      const int p = __ldg(ent + q);
      mx = fmaxf(mx, (w ? __ldg(w + p) : 1.f) * __ldg(EN + (size_t)p * ld + c));
    }
    float den = 0.f, num = 0.f;
    for (int q = q0; q < q1; ++q) {
      const int p = __ldg(ent + q);
      const float ww = w ? __ldg(w + p) : 1.f;
      const float e = expf(ww * __ldg(EN + (size_t)p * ld + c) - mx);
      den += e;
      num = fmaf(e, ww * __ldg(EM + (size_t)p * ld + c), num);
    }
    res = num / den;
  }
  out[idx] = res;
}
int seg_softmax_fwd(float* out, const float* EM, const float* EN, int ld, const int* ptr, const int* ent,
                    const float* w, long long S, cudaStream_t st) {
  if (S <= 0) return 0;
  seg_softmax_fwd_kernel<<<GIB_1D(S * ld, 256), 0, st>>>(out, EM, EN, ld, ptr, ent, w, S);
  GIB_LAUNCH_CHECK();
  return 0;
}

// backward: GM[p,c] = w a_p dM selu'(EM);  GN[p,c] = w a_p (da_p - sum_q a_q da_q) selu'(EN), da_p = w EM dM
// (GM / GN must be zero-initialised: pad rows are never visited)
__global__ void __launch_bounds__(256) seg_softmax_bwd_kernel(float* __restrict__ GM, float* __restrict__ GN,
                                                              const float* __restrict__ dM,
                                                              const float* __restrict__ EM,
                                                              const float* __restrict__ EN, int ld,
                                                              const int* __restrict__ ptr, const int* __restrict__ ent,
                                                              const float* __restrict__ w, long long S) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= S * ld) return;
  const long long s = idx / ld;
  const int c = (int)(idx % ld);
  const int q0 = __ldg(ptr + s), q1 = __ldg(ptr + s + 1);
  if (q1 <= q0) return;
  const float d = dM[idx];
  float mx = -INFINITY;
  for (int q = q0; q < q1; ++q) {
    const int p = __ldg(ent + q);
    mx = fmaxf(mx, (w ? __ldg(w + p) : 1.f) * __ldg(EN + (size_t)p * ld + c));
  }
  float den = 0.f, dot = 0.f;
  for (int q = q0; q < q1; ++q) {
    const int p = __ldg(ent + q);
    const float ww = w ? __ldg(w + p) : 1.f;
    const float e = expf(ww * __ldg(EN + (size_t)p * ld + c) - mx);
    den += e;
    dot = fmaf(e, ww * __ldg(EM + (size_t)p * ld + c) * d, dot);
  }
  const float inv = 1.f / den;
  dot *= inv;
  for (int q = q0; q < q1; ++q) {
    const int p = __ldg(ent + q);
    const float ww = w ? __ldg(w + p) : 1.f;
    const float en = __ldg(EN + (size_t)p * ld + c), em = __ldg(EM + (size_t)p * ld + c);
    const float a = expf(ww * en - mx) * inv;
    GM[(size_t)p * ld + c] = ww * a * d * dselu_from_out(em);
    GN[(size_t)p * ld + c] = ww * a * (ww * em * d - dot) * dselu_from_out(en);
  }
}
int seg_softmax_bwd(float* GM, float* GN, const float* dM, const float* EM, const float* EN, int ld, const int* ptr,
                    const int* ent, const float* w, long long S, cudaStream_t st) {
  if (S <= 0) return 0;
  seg_softmax_bwd_kernel<<<GIB_1D(S * ld, 256), 0, st>>>(GM, GN, dM, EM, EN, ld, ptr, ent, w, S);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------
// GRU gates (torch.nn.GRUCell, mpnn.py:296-297; gate order r,z,n; SURVEY Appendix D)
// gi, gh: [S, 3*Hp] gate-blocked (gate g at columns g*Hp..).  h == nullptr means h = 0 and
// gh is a single bias row (EMN: `self.gru(message)` with hx=None, mpnn.py:488).
// Slots whose CSR row is empty keep their state (summation_mpnn.py:143-144 updates only
// the nodes that have a bond).  ptr == nullptr: every row is active.  live (EMN bond rows, capacity mode): rows at or
// past *live are neither read nor written.
// ------------------------------------------------------------------------------------
__global__ void gru_fwd_kernel(float* __restrict__ hn, const float* __restrict__ gi, const float* __restrict__ gh,
                               const float* __restrict__ h, int Hp, const int* __restrict__ ptr, long long S,
                               const int* __restrict__ live) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= live_rows(live, S) * Hp) return;
  const long long s = idx / Hp;
  const int c = (int)(idx % Hp);
  const float hv = h ? h[idx] : 0.f;
  const bool active = !ptr || (__ldg(ptr + s + 1) > __ldg(ptr + s));
  float res = hv;
  if (active) {
    const float* gi_r = gi + (size_t)s * 3 * Hp;
    const float* gh_r = h ? gh + (size_t)s * 3 * Hp : gh;
    const float r = sigmoid_f(gi_r[c] + gh_r[c]);
    const float z = sigmoid_f(gi_r[Hp + c] + gh_r[Hp + c]);
    const float n = tanhf(gi_r[2 * Hp + c] + r * gh_r[2 * Hp + c]);
    res = (1.f - z) * n + z * hv;
  }
  hn[idx] = res;
}
int gru_fwd(float* hn, const float* gi, const float* gh, const float* h, int Hp, const int* ptr, long long S,
            const int* live, cudaStream_t st) {
  if (S <= 0) return 0;
  gru_fwd_kernel<<<GIB_1D(S * Hp, 256), 0, st>>>(hn, gi, gh, h, Hp, ptr, S, live);
  GIB_LAUNCH_CHECK();
  return 0;
}

__global__ void gru_bwd_kernel(float* __restrict__ dgi, float* __restrict__ dgh, float* __restrict__ dh_direct,
                               const float* __restrict__ dhn, const float* __restrict__ gi,
                               const float* __restrict__ gh, const float* __restrict__ h, int Hp,
                               const int* __restrict__ ptr, long long S, const int* __restrict__ live) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= live_rows(live, S) * Hp) return;
  const long long s = idx / Hp;
  const int c = (int)(idx % Hp);
  const float d = dhn[idx];
  const float hv = h ? h[idx] : 0.f;
  const bool active = !ptr || (__ldg(ptr + s + 1) > __ldg(ptr + s));
  float gir = 0.f, giz = 0.f, gin = 0.f, ghn = 0.f, dd = d;
  if (active) {
    const float* gi_r = gi + (size_t)s * 3 * Hp;
    const float* gh_r = h ? gh + (size_t)s * 3 * Hp : gh;
    const float hn_pre = gh_r[2 * Hp + c];
    const float r = sigmoid_f(gi_r[c] + gh_r[c]);
    const float z = sigmoid_f(gi_r[Hp + c] + gh_r[Hp + c]);
    const float n = tanhf(gi_r[2 * Hp + c] + r * hn_pre);
    const float dn = d * (1.f - z);
    const float dz = d * (hv - n);
    const float dpre_n = dn * (1.f - n * n);
    const float dr = dpre_n * hn_pre;
    gir = dr * r * (1.f - r);
    giz = dz * z * (1.f - z);
    gin = dpre_n;
    ghn = dpre_n * r;
    dd = d * z;
  }
  float* o = dgi + (size_t)s * 3 * Hp;
  o[c] = gir; o[Hp + c] = giz; o[2 * Hp + c] = gin;
  float* o2 = dgh + (size_t)s * 3 * Hp;
  o2[c] = gir; o2[Hp + c] = giz; o2[2 * Hp + c] = ghn;
  if (dh_direct) dh_direct[idx] = dd;
}
int gru_bwd(float* dgi, float* dgh, float* dh_direct, const float* dhn, const float* gi, const float* gh,
            const float* h, int Hp, const int* ptr, long long S, const int* live, cudaStream_t st) {
  if (S <= 0) return 0;
  gru_bwd_kernel<<<GIB_1D(S * Hp, 256), 0, st>>>(dgi, dgh, dh_direct, dhn, gi, gh, h, Hp, ptr, S, live);
  GIB_LAUNCH_CHECK();
  return 0;
}

// column sums: out[r] += sum_m G[m, prow(r)]  (bias gradient when no dW GEMM runs alongside).  live: sum over the
// first *live of the M rows only, in the same order as an exact-size launch over those rows
__global__ void colsum_kernel(float* __restrict__ out, const float* __restrict__ G, int ldg, long long M, int R,
                              int Rb, int Rbp, const int* __restrict__ live) {
  // one CTA per 32 columns, 8 warps stride over rows; fixed-order tree at the end
  __shared__ float sm[8][33];
  const int r = blockIdx.x * 32 + (threadIdx.x & 31);
  const int wy = threadIdx.x >> 5;
  M = live_rows(live, M);
  float s = 0.f;
  if (r < R) {
    const int prow = (r / Rb) * Rbp + (r % Rb);
    for (long long m = wy; m < M; m += 8) s += G[m * ldg + prow];
  }
  sm[wy][threadIdx.x & 31] = s;
  __syncthreads();
  if (wy == 0 && r < R) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += sm[k][threadIdx.x];
    out[r] += t;
  }
}
int colsum_add(float* out, const float* G, int ldg, long long M, int R, int Rb, int Rbp, const int* live,
               cudaStream_t st) {
  if (M <= 0 || R <= 0) return 0;
  colsum_kernel<<<ceil_div(R, 32), 256, 0, st>>>(out, G, ldg, M, R, Rb, Rbp, live);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------
// GraphGather readout (modules.py:39-52): per molecule and per channel a masked softmax over
// the atom axis.  The mask arithmetic is the reference's: energies - 1e6 * (mask == 0) in
// fp32 (for molecules with no bonded atom every energy is quantised to 1/16 by that
// subtraction, and the result depends on it -- SURVEY §7 hard parts).
// active atom <=> its dst-CSR row is non-empty (summation_mpnn.py:146 `adjacency.sum(-1) != 0`).
// ------------------------------------------------------------------------------------
__global__ void graph_gather_fwd_kernel(float* __restrict__ g, float* __restrict__ att, const float* __restrict__ en,
                                        const float* __restrict__ em, int ld, const int* __restrict__ ptr, int N,
                                        int B, float big) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * ld) return;
  const int b = (int)(idx / ld), c = (int)(idx % ld);
  const size_t base = (size_t)b * N;
  float mx = -INFINITY;
  for (int i = 0; i < N; ++i) {
    const bool active = __ldg(ptr + base + i + 1) > __ldg(ptr + base + i);
    const float e = en[(base + i) * ld + c] - (active ? 0.f : big);
    mx = fmaxf(mx, e);
  }
  float den = 0.f;
  for (int i = 0; i < N; ++i) {
    const bool active = __ldg(ptr + base + i + 1) > __ldg(ptr + base + i);
    const float e = en[(base + i) * ld + c] - (active ? 0.f : big);
    den += expf(e - mx);
  }
  float acc = 0.f;
  for (int i = 0; i < N; ++i) {
    const bool active = __ldg(ptr + base + i + 1) > __ldg(ptr + base + i);
    const float e = en[(base + i) * ld + c] - (active ? 0.f : big);
    const float a = expf(e - mx) / den;
    att[(base + i) * ld + c] = a;
    acc = fmaf(a, em[(base + i) * ld + c], acc);
  }
  g[idx] = acc;
}
int graph_gather_fwd(float* g, float* att, const float* en, const float* em, int ld, const int* ptr, int N, int B,
                     float big, cudaStream_t st) {
  graph_gather_fwd_kernel<<<GIB_1D((long long)B * ld, 128), 0, st>>>(g, att, en, em, ld, ptr, N, B, big);
  GIB_LAUNCH_CHECK();
  return 0;
}

// Gen[s,c] = a (da - sum a da) selu'(en);  Gem[s,c] = a dg selu'(em);   da = dg * em
__global__ void graph_gather_bwd_kernel(float* __restrict__ Gen, float* __restrict__ Gem, const float* __restrict__ dg,
                                        const float* __restrict__ att, const float* __restrict__ en,
                                        const float* __restrict__ em, int ld, int N, int B) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * ld) return;
  const int b = (int)(idx / ld), c = (int)(idx % ld);
  const size_t base = (size_t)b * N;
  const float d = dg[idx];
  float dot = 0.f;
  for (int i = 0; i < N; ++i) dot = fmaf(att[(base + i) * ld + c], d * em[(base + i) * ld + c], dot);
  for (int i = 0; i < N; ++i) {
    const size_t o = (base + i) * ld + c;
    const float a = att[o], emv = em[o];
    Gen[o] = a * (d * emv - dot) * dselu_from_out(en[o]);
    Gem[o] = a * d * dselu_from_out(emv);
  }
}
int graph_gather_bwd(float* Gen, float* Gem, const float* dg, const float* att, const float* en, const float* em,
                     int ld, int N, int B, cudaStream_t st) {
  graph_gather_bwd_kernel<<<GIB_1D((long long)B * ld, 128), 0, st>>>(Gen, Gem, dg, att, en, em, ld, N, B);
  GIB_LAUNCH_CHECK();
  return 0;
}

// MNN readout (mpnn.py:70-74): graph embedding = plain sum over the atom axis
__global__ void sum_nodes_fwd_kernel(float* __restrict__ g, const float* __restrict__ h, int ld, int N, int B) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * ld) return;
  const int b = (int)(idx / ld), c = (int)(idx % ld);
  float acc = 0.f;
  for (int i = 0; i < N; ++i) acc += h[((size_t)b * N + i) * ld + c];
  g[idx] = acc;
}
int sum_nodes_fwd(float* g, const float* h, int ld, int N, int B, cudaStream_t st) {
  sum_nodes_fwd_kernel<<<GIB_1D((long long)B * ld, 128), 0, st>>>(g, h, ld, N, B);
  GIB_LAUNCH_CHECK();
  return 0;
}
// dh[s, c] += dg[b(s), c]
__global__ void bcast_nodes_add_kernel(float* __restrict__ dh, const float* __restrict__ dg, int ld, int N,
                                       long long S) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= S * ld) return;
  const long long s = idx / ld;
  const int c = (int)(idx % ld);
  dh[idx] += dg[(s / N) * ld + c];
}
int bcast_nodes_add(float* dh, const float* dg, int ld, int N, long long S, cudaStream_t st) {
  bcast_nodes_add_kernel<<<GIB_1D(S * ld, 256), 0, st>>>(dh, dg, ld, N, S);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------
// EMN (edge memory network) kernels: edge_mpnn.py:104-192, mpnn.py:466-488
// bond r = (b, i, j): ent_dst = slot of i, ent_src = slot of j.  Entries are untyped (one
// group) and in reference order, so entry row == bond index r and dst_ent is the identity.
// Capacity mode: E is the capacity and `live` the device-side bond count; rows [live, E) are pad rows (ent_src =
// ent_dst = -1) or, after an overflow, bonds past the capacity.  The aggregation kernels skip them: the live rows
// never read a row at or past the live count (K0 clamps dst_ptr / src_ptr to the capacity).
// ------------------------------------------------------------------------------------
// X[r, :] = [ nodes[i, :F] | nodes[j, :F] | edges[i, j, :Ef] | 0 ]
__global__ void emn_input_kernel(float* __restrict__ X, int ld, const void* __restrict__ nodes,
                                 const void* __restrict__ edges, int i8, const int* __restrict__ ent_dst,
                                 const int* __restrict__ ent_src, int N, int F, int Ef, long long P) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P * ld) return;
  const long long r = idx / ld;
  const int c = (int)(idx % ld);
  const int si = __ldg(ent_dst + r), sj = __ldg(ent_src + r);
  float v = 0.f;
  if (si >= 0) {
    if (c < F) v = ld_in(nodes, (size_t)si * F + c, i8);
    else if (c < 2 * F) v = ld_in(nodes, (size_t)sj * F + (c - F), i8);
    else if (c < 2 * F + Ef) v = ld_in(edges, ((size_t)si * N + (sj % N)) * Ef + (c - 2 * F), i8);
  }
  X[idx] = v;
}
int emn_input(float* X, int ld, const void* nodes, const void* edges, int i8, const int* ent_dst, const int* ent_src,
              int N, int F, int Ef, long long P, cudaStream_t st) {
  if (P <= 0) return 0;
  emn_input_kernel<<<GIB_1D(P * ld, 256), 0, st>>>(X, ld, nodes, edges, i8, ent_dst, ent_src, N, F, Ef, P);
  GIB_LAUNCH_CHECK();
  return 0;
}

// message[r, c] = softmax-weighted sum over { (ENx[r], EMx[r]) } U { (ENm[s], EMm[s]) : s in row(head j of r),
// head(s) != tail i of r }.  Reference slot order: self first, then the bonds of j in ascending k.
__global__ void __launch_bounds__(256) emn_aggregate_fwd_kernel(float* __restrict__ msg, const float* __restrict__ EMx,
                                                                const float* __restrict__ ENx,
                                                                const float* __restrict__ EMm,
                                                                const float* __restrict__ ENm, int ld,
                                                                const int* __restrict__ ent_dst,
                                                                const int* __restrict__ ent_src,
                                                                const int* __restrict__ dst_ptr, long long E,
                                                                const int* __restrict__ live) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= live_rows(live, E) * ld) return;
  const long long r = idx / ld;
  const int c = (int)(idx % ld);
  const int si = __ldg(ent_dst + r), sj = __ldg(ent_src + r);
  const int q0 = __ldg(dst_ptr + sj), q1 = __ldg(dst_ptr + sj + 1);
  const float e_self = ENx[idx];
  float mx = e_self;
  for (int s = q0; s < q1; ++s)
    if (__ldg(ent_src + s) != si) mx = fmaxf(mx, ENm[(size_t)s * ld + c]);
  float den = expf(e_self - mx);
  float num = den * EMx[idx];
  for (int s = q0; s < q1; ++s)
    if (__ldg(ent_src + s) != si) {
      const float e = expf(ENm[(size_t)s * ld + c] - mx);
      den += e;
      num = fmaf(e, EMm[(size_t)s * ld + c], num);
    }
  msg[idx] = num / den;
}
int emn_aggregate_fwd(float* msg, const float* EMx, const float* ENx, const float* EMm, const float* ENm, int ld,
                      const int* ent_dst, const int* ent_src, const int* dst_ptr, long long E, const int* live,
                      cudaStream_t st) {
  if (E <= 0) return 0;
  emn_aggregate_fwd_kernel<<<GIB_1D(E * ld, 256), 0, st>>>(msg, EMx, ENx, EMm, ENm, ld, ent_dst, ent_src, dst_ptr, E,
                                                           live);
  GIB_LAUNCH_CHECK();
  return 0;
}

// backward, receiver-side pass: per (r, c) recompute the softmax, write the self-term gradients
//   dEMx[r] += a_self * d ;  dENx[r] += a_self * (EMx*d - dot)
// and stash per-receiver (mx, 1/den, dot) so the sender-side pass can form its terms without atomics.
__global__ void __launch_bounds__(256) emn_aggregate_bwd_recv_kernel(
    float* __restrict__ dEMx, float* __restrict__ dENx, float* __restrict__ st_mx, float* __restrict__ st_inv,
    float* __restrict__ st_dot, const float* __restrict__ dmsg, const float* __restrict__ EMx,
    const float* __restrict__ ENx, const float* __restrict__ EMm, const float* __restrict__ ENm, int ld,
    const int* __restrict__ ent_dst, const int* __restrict__ ent_src, const int* __restrict__ dst_ptr, long long E,
    const int* __restrict__ live) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= live_rows(live, E) * ld) return;
  const long long r = idx / ld;
  const int c = (int)(idx % ld);
  const int si = __ldg(ent_dst + r), sj = __ldg(ent_src + r);
  const int q0 = __ldg(dst_ptr + sj), q1 = __ldg(dst_ptr + sj + 1);
  const float d = dmsg[idx];
  const float e_self = ENx[idx];
  float mx = e_self;
  for (int s = q0; s < q1; ++s)
    if (__ldg(ent_src + s) != si) mx = fmaxf(mx, ENm[(size_t)s * ld + c]);
  const float es = expf(e_self - mx);
  float den = es, dot = es * EMx[idx] * d;
  for (int s = q0; s < q1; ++s)
    if (__ldg(ent_src + s) != si) {
      const float e = expf(ENm[(size_t)s * ld + c] - mx);
      den += e;
      dot = fmaf(e, EMm[(size_t)s * ld + c] * d, dot);
    }
  const float inv = 1.f / den;
  dot *= inv;
  const float a = es * inv;
  dEMx[idx] += a * d;
  dENx[idx] += a * (EMx[idx] * d - dot);
  st_mx[idx] = mx; st_inv[idx] = inv; st_dot[idx] = dot;
}
// sender-side pass: bond s = (j, k) feeds every receiver r = (i, j) with i != k, i.e. the bonds whose
// SOURCE slot is j = ent_dst[s] (src-CSR row of j), except the reverse bond.
//   dEMm[s] = sum_r a_rs d_r ;  dENm[s] = sum_r a_rs (EMm[s] d_r - dot_r)     (plain store: one writer per (s,c))
__global__ void __launch_bounds__(256) emn_aggregate_bwd_send_kernel(
    float* __restrict__ dEMm, float* __restrict__ dENm, const float* __restrict__ st_mx,
    const float* __restrict__ st_inv, const float* __restrict__ st_dot, const float* __restrict__ dmsg,
    const float* __restrict__ EMm, const float* __restrict__ ENm, int ld, const int* __restrict__ ent_dst,
    const int* __restrict__ ent_src, const int* __restrict__ src_ptr, const int* __restrict__ src_ent, long long E,
    const int* __restrict__ live) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long m = live_rows(live, E);
  if (idx >= m * ld) return;
  const long long s = idx / ld;
  const int c = (int)(idx % ld);
  const int tail = __ldg(ent_dst + s);   // j: the atom bond s leaves from (its row)
  const int head = __ldg(ent_src + s);   // k
  const int q0 = __ldg(src_ptr + tail), q1 = __ldg(src_ptr + tail + 1);
  const float en = ENm[idx], em = EMm[idx];
  float gm = 0.f, gn = 0.f;
  for (int q = q0; q < q1; ++q) {
    const int r = __ldg(src_ent + q);        // receiver r = (i, j): ent_src[r] == tail
    // a receiver past the live count exists only in an overflowing batch (src_ent may name a bond the capacity cut
    // off): it has no softmax state
    if (r >= m) continue;
    if (__ldg(ent_dst + r) == head) continue;  // i == k: reverse bond excluded (edge_mpnn.py:158-160)
    const size_t o = (size_t)r * ld + c;
    const float a = expf(en - st_mx[o]) * st_inv[o];
    const float d = dmsg[o];
    gm = fmaf(a, d, gm);
    gn = fmaf(a, em * d - st_dot[o], gn);
  }
  dEMm[idx] = gm;
  dENm[idx] = gn;
}
int emn_aggregate_bwd(float* dEMx, float* dENx, float* dEMm, float* dENm, float* st3, const float* dmsg,
                      const float* EMx, const float* ENx, const float* EMm, const float* ENm, int ld,
                      const GraphArrays& ga, long long E, const int* live, cudaStream_t st) {
  if (E <= 0) return 0;
  float* st_mx = st3;
  float* st_inv = st3 + (size_t)E * ld;
  float* st_dot = st3 + (size_t)2 * E * ld;
  emn_aggregate_bwd_recv_kernel<<<GIB_1D(E * ld, 256), 0, st>>>(dEMx, dENx, st_mx, st_inv, st_dot, dmsg, EMx, ENx, EMm,
                                                               ENm, ld, ga.ent_dst, ga.ent_src, ga.dst_ptr, E, live);
  GIB_LAUNCH_CHECK();
  emn_aggregate_bwd_send_kernel<<<GIB_1D(E * ld, 256), 0, st>>>(dEMm, dENm, st_mx, st_inv, st_dot, dmsg, EMm, ENm, ld,
                                                               ga.ent_dst, ga.ent_src, ga.src_ptr, ga.src_ent, E,
                                                               live);
  GIB_LAUNCH_CHECK();
  return 0;
}

// elementwise helpers -------------------------------------------------------------------
// G = d * selu'(y) over rows x ld
__global__ void mul_dselu_kernel(float* __restrict__ G, const float* __restrict__ d, const float* __restrict__ y,
                                 long long rows, int ld, const int* __restrict__ live) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < live_rows(live, rows) * ld) G[i] = d[i] * dselu_from_out(y[i]);
}
int mul_dselu(float* G, const float* d, const float* y, long long rows, int ld, const int* live, cudaStream_t st) {
  if (rows <= 0) return 0;
  mul_dselu_kernel<<<GIB_1D(rows * ld, 256), 0, st>>>(G, d, y, rows, ld, live);
  GIB_LAUNCH_CHECK();
  return 0;
}
// ------------------------------------------------------------------------------------
// parameter packing: reference-shaped weight [nblk*Rb, C] (element (r,c) at src[r*rs + c*cs])
//   -> Wp  [nblk*Rbp, Cp]   zero padded, K-contiguous      (forward  B operand)
//   -> WTp [Ctp, nblk*Rbp]  transposed, first Ct columns   (backward dX B operand)
//   -> bp  [nblk*Rbp]
// ------------------------------------------------------------------------------------
__global__ void pack_weight_kernel(float* __restrict__ Wp, float* __restrict__ WTp, float* __restrict__ bp,
                                   const float* __restrict__ W, const float* __restrict__ bias, long long rs,
                                   long long cs, int nblk, int Rb, int Rbp, int C, int Cp, int Ct, int Ctp) {
  const int Rp = nblk * Rbp;
  const long long n1 = (long long)Rp * Cp, n2 = (long long)Ctp * Rp;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < n1) {
    const int pr = (int)(idx / Cp), c = (int)(idx % Cp);
    const int g = pr / Rbp, rr = pr % Rbp;
    float v = 0.f;
    if (rr < Rb && c < C) v = W[(long long)(g * Rb + rr) * rs + c * cs];
    Wp[idx] = v;
  } else if (idx < n1 + n2) {
    const long long k = idx - n1;
    const int c = (int)(k / Rp), pr = (int)(k % Rp);
    const int g = pr / Rbp, rr = pr % Rbp;
    float v = 0.f;
    if (rr < Rb && c < Ct) v = W[(long long)(g * Rb + rr) * rs + c * cs];
    WTp[k] = v;
  } else if (idx < n1 + n2 + Rp) {
    const int pr = (int)(idx - n1 - n2);
    const int g = pr / Rbp, rr = pr % Rbp;
    bp[pr] = (bias && rr < Rb) ? bias[g * Rb + rr] : 0.f;
  }
}
int pack_weight(float* Wp, float* WTp, float* bp, const float* W, const float* bias, long long rs, long long cs,
                int nblk, int Rb, int Rbp, int C, int Cp, int Ct, int Ctp, cudaStream_t st) {
  const long long tot = (long long)nblk * Rbp * Cp + (long long)Ctp * nblk * Rbp + nblk * Rbp;
  pack_weight_kernel<<<GIB_1D(tot, 256), 0, st>>>(Wp, WTp, bp, W, bias, rs, cs, nblk, Rb, Rbp, C, Cp, Ct, Ctp);
  GIB_LAUNCH_CHECK();
  return 0;
}


__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// element i of a 16-bit plane (h16 1: bf16, 2: fp16) at `plane`: v rounded to nearest-even, as tensor.to(dtype)
__device__ __forceinline__ void store16(float* plane, long long i, float v, int h16) {
  uint16_t u;
  if (h16 == 1) asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(u) : "f"(v));
  else asm("cvt.rn.f16.f32 %0, %1;" : "=h"(u) : "f"(v));
  reinterpret_cast<uint16_t*>(plane)[i] = u;
}

// all Linears of a model in ONE launch: the per-Linear descriptors travel as a kernel parameter (__grid_constant__)
__global__ void __launch_bounds__(256) pack_all_kernel(const __grid_constant__ PackTable T, float* __restrict__ packed) {
  __shared__ int s_idx;
  if (threadIdx.x == 0) {
    int i = 0;
    while (i + 1 < T.n && blockIdx.x >= T.e[i + 1].blk_begin) ++i;
    s_idx = i;
  }
  __syncthreads();
  const PackEntry& E = T.e[s_idx];
  const int Rp = E.nblk * E.Rbp;
  const long long n1 = (long long)Rp * E.Cp, n2 = (long long)E.Ctp * Rp;
  const long long base = (long long)(blockIdx.x - E.blk_begin) * 1024;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const long long idx = base + u * 256 + threadIdx.x;
    if (idx < n1) {
      const int pr = (int)(idx / E.Cp), c = (int)(idx % E.Cp);
      const int g = pr / E.Rbp, rr = pr % E.Rbp;
      float v = 0.f;
      if (rr < E.Rb && c < E.C) v = E.W[(long long)(g * E.Rb + rr) * E.rs + c * E.cs];
      packed[E.ow + idx] = v;
      const float h = tf32_rna(v);
      packed[E.ow_hi + idx] = h;
      if (T.h16) store16(packed + E.ow_lo, idx, v, T.h16);
      else packed[E.ow_lo + idx] = tf32_rna(v - h);
    } else if (idx < n1 + n2) {
      const long long k = idx - n1;
      const int c = (int)(k / Rp), pr = (int)(k % Rp);
      const int g = pr / E.Rbp, rr = pr % E.Rbp;
      float v = 0.f;
      if (rr < E.Rb && c < E.Ct) v = E.W[(long long)(g * E.Rb + rr) * E.rs + c * E.cs];
      packed[E.owt + k] = v;
      const float h = tf32_rna(v);
      packed[E.owt_hi + k] = h;
      if (T.h16) store16(packed + E.owt_lo, k, v, T.h16);
      else packed[E.owt_lo + k] = tf32_rna(v - h);
    } else if (idx < n1 + n2 + Rp) {
      const int pr = (int)(idx - n1 - n2);
      const int g = pr / E.Rbp, rr = pr % E.Rbp;
      packed[E.ob + pr] = (E.bias && rr < E.Rb) ? E.bias[g * E.Rb + rr] : 0.f;
    }
  }
}
int pack_all(const PackTable& T, float* packed, cudaStream_t st) {
  if (T.n <= 0) return 0;
  pack_all_kernel<<<T.total_blocks, 256, 0, st>>>(T, packed);
  GIB_LAUNCH_CHECK();
  return 0;
}

}  // namespace gib
