// K0: dense bond tensor -> bond-entry lists + CSR (by destination atom and by source atom).
//
// Replaces the prologue of the reference forwards:
//   gnn/summation_mpnn.py:102-118   (adjacency, nonzero -> COO, dense [V,E] summation matrix)
//   gnn/aggregation_mpnn.py:105-148 (COO, degrees, padded neighbour tensors, per-node Python loops)
//   gnn/edge_mpnn.py:104-173        (COO, line-graph incidence via per-edge Python loops)
//
// Vocabulary: a "slot" is one atom position (b, i) -> b*N + i.  A directed bond (b, i, j) has
// dst = i (the row that receives the message) and src = j, exactly as `adjacency.nonzero()`
// orders them in the reference (row-major (b, i, j), so the bond list is already dst-sorted).
// A "bond entry" is one non-zero element edges[b, i, j, t]; entries are laid out grouped by
// bond type t (each group starts on a 128-row boundary, pad rows have src = dst = -1, w = 0)
// so the per-type message MLP is a plain GEMM over a contiguous row range.
//
// Two phases so that exact-size buffers can be allocated in between (one 64-byte D2H read):
//   count: per-molecule per-type entry counts, then one single-CTA scan -> header
//   fill : entry arrays + both CSRs, deterministic order, no atomics on the data path
#include "graph.cuh"

namespace gib {

template <int NT>
__device__ __forceinline__ int block_exscan(int v, int* sm, int* total) {
  // exclusive prefix of v over the NT threads of the CTA; *total = sum.  sm: NT/32 + 1 ints.
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();  // protect sm reuse across calls
  if (lane == 31) sm[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int wv = lane < NT / 32 ? sm[lane] : 0;
    int winc = wv;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    if (lane < NT / 32) sm[lane] = winc - wv;
    if (lane == 31) sm[NT / 32] = winc;
  }
  __syncthreads();
  *total = sm[NT / 32];
  return sm[wid] + inc - v;
}

// ---------------------------------------------------------------------------------
// phase 1a: per-molecule counts
// ---------------------------------------------------------------------------------
// bond values arrive as float32 or as the int8 of the reference's HDF5 files (BlockDatasetLoader.py:139-143 widens
// them on the host; here K0 reads the bytes directly: 4x less traffic on its dominant operand)
template <typename T> __device__ __forceinline__ float ld_val(const T* p) { return (float)__ldg(p); }

template <typename T>
__global__ void __launch_bounds__(128) k0_count_kernel(const T* __restrict__ edges, int B, int N, int Ef,
                                                       int G, int* __restrict__ cnt, int* __restrict__ hdr) {
  __shared__ int sm[8];
  const int b = blockIdx.x;
  const T* e = edges + (size_t)b * N * N * Ef;
  int c[4] = {0, 0, 0, 0};
  int flags = 0;
  for (int cell = threadIdx.x; cell < N * N; cell += 128) {
    int nz = 0;
    for (int t = 0; t < Ef; ++t) {
      float v = ld_val(e + (size_t)cell * Ef + t);
      if (v != 0.f) {
        ++nz;
        if (G > 1) ++c[t];
        if (v != 1.f) flags |= GRAPH_FLAG_NONBINARY;
      }
    }
    if (nz > 1) flags |= GRAPH_FLAG_MULTITYPE;
    if (G == 1 && nz > 0) ++c[0];
  }
  for (int g = 0; g < G; ++g) {
    int tot;
    block_exscan<128>(c[g], sm, &tot);
    if (threadIdx.x == 0) cnt[g * B + b] = tot;
  }
  if (flags) atomicOr(&hdr[HDR_FLAGS], flags);
}

// ---------------------------------------------------------------------------------
// phase 1b: scans over molecules (single CTA) + header
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k0_scan_kernel(int B, int G, const int* __restrict__ cnt,
                                                       int* __restrict__ off, int* __restrict__ ent_off,
                                                       int* __restrict__ hdr) {
  __shared__ int sm[34];
  const int L = ceil_div(B, 1024);
  const int lo = threadIdx.x * L, hi = min(B, lo + L);
  int base = 0;
  for (int g = 0; g <= G; ++g) {  // g == G: per-molecule totals over all groups
    int s = 0;
    for (int b = lo; b < hi; ++b) {
      int v = 0;
      if (g < G) v = cnt[g * B + b];
      else for (int q = 0; q < G; ++q) v += cnt[q * B + b];
      s += v;
    }
    int tot;
    int run = block_exscan<1024>(s, sm, &tot);
    for (int b = lo; b < hi; ++b) {
      int v = 0;
      if (g < G) { v = cnt[g * B + b]; off[g * B + b] = run; }
      else { for (int q = 0; q < G; ++q) v += cnt[q * B + b]; ent_off[b] = run; }
      run += v;
    }
    if (threadIdx.x == 0) {
      if (g < G) {
        hdr[HDR_TYPE_COUNT + g] = tot;
        hdr[HDR_TYPE_BASE + g] = base;
      } else {
        hdr[HDR_E] = tot;
        hdr[HDR_P] = base;
        hdr[HDR_TYPE_BASE + G] = base;
      }
    }
    base += ceil_div(tot, kTileRows) * kTileRows;
  }
}

// ---------------------------------------------------------------------------------
// phase 2: entries + CSR by dst + CSR by src, one CTA per molecule
// ---------------------------------------------------------------------------------
// position -> cell maps of the three orders (cell index is memory order (i*N + j)*G + t)
__device__ __forceinline__ int cell_of_type_order(int pos, int NN, int G) { return (pos % NN) * G + pos / NN; }
__device__ __forceinline__ int cell_of_src_order(int pos, int N, int G) {
  const int t = pos % G, ji = pos / G, j = ji / N, i = ji % N;
  return (i * N + j) * G + t;
}

template <typename T>
__global__ void __launch_bounds__(256) k0_fill_kernel(const T* __restrict__ edges, int B, int N, int Ef, int G,
                                                      const int* __restrict__ cnt, const int* __restrict__ off,
                                                      const int* __restrict__ ent_off, const int* __restrict__ hdr,
                                                      GraphArrays ga, int cap_E, int cap_P) {
  extern __shared__ unsigned char smem_raw[];
  const int NN = N * N, cells = NN * G;
  unsigned short* rank_mem = reinterpret_cast<unsigned short*>(smem_raw);
  unsigned short* rank_typ = rank_mem + cells + 2;
  unsigned short* rank_src = rank_typ + cells + 2;
  unsigned char* flag = reinterpret_cast<unsigned char*>(rank_src + cells + 2);
  __shared__ int sm[10];

  const int b = blockIdx.x;
  const T* e = edges + (size_t)b * NN * Ef;
  for (int c = threadIdx.x; c < cells; c += 256) {
    unsigned char f;
    if (G > 1) f = ld_val(e + c) != 0.f;
    else {
      f = 0;
      for (int t = 0; t < Ef; ++t) f |= (ld_val(e + (size_t)c * Ef + t) != 0.f);
    }
    flag[c] = f;
  }
  __syncthreads();

  const int L = ceil_div(cells, 256);
  const int lo = min(cells, (int)threadIdx.x * L), hi = min(cells, lo + L);
  int total_b = 0;
  for (int order = 0; order < 3; ++order) {
    unsigned short* rk = order == 0 ? rank_mem : (order == 1 ? rank_typ : rank_src);
    int s = 0;
    for (int pos = lo; pos < hi; ++pos) {
      int c = order == 0 ? pos : (order == 1 ? cell_of_type_order(pos, NN, G) : cell_of_src_order(pos, N, G));
      s += flag[c];
    }
    int tot;
    int run = block_exscan<256>(s, sm, &tot);
    for (int pos = lo; pos < hi; ++pos) {
      int c = order == 0 ? pos : (order == 1 ? cell_of_type_order(pos, NN, G) : cell_of_src_order(pos, N, G));
      rk[c] = (unsigned short)run;
      run += flag[c];
    }
    total_b = tot;
  }
  __syncthreads();

  const int eoff = ent_off[b];
  int tstart[4], tbase[4];
  {
    int acc = 0;
    for (int g = 0; g < G; ++g) {
      tstart[g] = acc;
      acc += cnt[g * B + b];
      tbase[g] = hdr[HDR_TYPE_BASE + g] + off[g * B + b];
    }
  }
  for (int c = threadIdx.x; c < cells; c += 256) {
    if (!flag[c]) continue;
    const int t = c % G, ij = c / G, i = ij / N, j = ij % N;
    const int p = tbase[t] + (int)rank_typ[c] - tstart[t];
    if (p < cap_P) {                     // capacity mode: an overflowing batch is truncated (and flagged), never
      ga.ent_src[p] = b * N + j;         // written out of bounds
      ga.ent_dst[p] = b * N + i;
      ga.ent_w[p] = (G > 1) ? ld_val(e + c) : 1.f;
    }
    const int qd = eoff + rank_mem[c], qs = eoff + rank_src[c];
    if (qd < cap_E) ga.dst_ent[qd] = p < cap_P ? p : 0;
    if (qs < cap_E) ga.src_ent[qs] = p < cap_P ? p : 0;
  }
  for (int i = threadIdx.x; i < N; i += 256) {
    ga.dst_ptr[b * N + i] = min(cap_E, eoff + rank_mem[(i * N) * G]);      // first cell of row i
    ga.src_ptr[b * N + i] = min(cap_E, eoff + rank_src[(0 * N + i) * G]);  // cell (i'=0, j=i, t=0) opens column i
  }
  if (b == B - 1 && threadIdx.x == 0) {
    ga.dst_ptr[B * N] = min(cap_E, eoff + total_b);
    ga.src_ptr[B * N] = min(cap_E, eoff + total_b);
  }
}

// pad rows of every type group; capacity mode: block G also pads the tail [P, cap_P) and raises the overflow flag
__global__ void k0_pad_kernel(int* __restrict__ hdr, int G, GraphArrays ga, int cap_E, int cap_P) {
  const int g = blockIdx.x;
  int lo, hi;
  if (g < G) {
    lo = hdr[HDR_TYPE_BASE + g] + hdr[HDR_TYPE_COUNT + g];
    hi = hdr[HDR_TYPE_BASE + g + 1];
  } else {
    lo = hdr[HDR_P];
    hi = cap_P;
    if (threadIdx.x == 0 && (hdr[HDR_E] > cap_E || hdr[HDR_P] > cap_P)) atomicOr(&hdr[HDR_FLAGS], GRAPH_FLAG_OVERFLOW);
  }
  hi = min(hi, cap_P);
  for (int p = lo + threadIdx.x; p < hi; p += blockDim.x) {
    ga.ent_src[p] = -1;
    ga.ent_dst[p] = -1;
    ga.ent_w[p] = 0.f;
  }
}

size_t graph_count_ws_ints(int B, int G) { return (size_t)2 * G * B + B + HDR_INTS; }

int graph_count(const void* edges, int in_dtype, int B, int N, int Ef, int by_type, int* ws, cudaStream_t st) {
  const int G = by_type ? Ef : 1;
  if (B <= 0 || N <= 0 || Ef <= 0 || Ef > 4 || (long long)N * N * G > 32768) {
    set_error("graph_count: unsupported dims B=%d N=%d Ef=%d (need 1 <= n_edge_features <= 4, N*N*groups<=32768)", B, N, Ef);
    return -1;
  }
  int* hdr = ws;
  int* cnt = ws + HDR_INTS;
  int* off = cnt + (size_t)G * B;
  int* ent_off = off + (size_t)G * B;
  GIB_CUDA_TRY(cudaMemsetAsync(hdr, 0, HDR_INTS * sizeof(int), st));
  if (in_dtype == 0)
    k0_count_kernel<float><<<B, 128, 0, st>>>(reinterpret_cast<const float*>(edges), B, N, Ef, G, cnt, hdr);
  else
    k0_count_kernel<signed char><<<B, 128, 0, st>>>(reinterpret_cast<const signed char*>(edges), B, N, Ef, G, cnt, hdr);
  GIB_LAUNCH_CHECK();
  k0_scan_kernel<<<1, 1024, 0, st>>>(B, G, cnt, off, ent_off, hdr);
  GIB_LAUNCH_CHECK();
  return 0;
}

int graph_fill(const void* edges, int in_dtype, int B, int N, int Ef, int by_type, int* ws, GraphArrays ga, int cap_E,
               int cap_P, cudaStream_t st) {
  const int G = by_type ? Ef : 1;
  int* hdr = ws;
  const int* cnt = ws + HDR_INTS;
  const int* off = cnt + (size_t)G * B;
  const int* ent_off = off + (size_t)G * B;
  const int cells = N * N * G;
  const size_t smem = (size_t)3 * (cells + 2) * sizeof(unsigned short) + cells + 16;
  if (smem > 48 * 1024) {   // opt in to more dynamic shared memory (per device and per instantiation; cheap, idempotent)
    if (in_dtype == 0)
      GIB_CUDA_TRY(cudaFuncSetAttribute(k0_fill_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    else
      GIB_CUDA_TRY(cudaFuncSetAttribute(k0_fill_kernel<signed char>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  const bool capm = cap_P > 0;
  const int cE = capm ? cap_E : 0x7fffffff, cP = capm ? cap_P : 0x7fffffff;
  if (in_dtype == 0)
    k0_fill_kernel<float><<<B, 256, smem, st>>>(reinterpret_cast<const float*>(edges), B, N, Ef, G, cnt, off, ent_off,
                                                 hdr, ga, cE, cP);
  else
    k0_fill_kernel<signed char><<<B, 256, smem, st>>>(reinterpret_cast<const signed char*>(edges), B, N, Ef, G, cnt,
                                                       off, ent_off, hdr, ga, cE, cP);
  GIB_LAUNCH_CHECK();
  k0_pad_kernel<<<capm ? G + 1 : G, 128, 0, st>>>(hdr, G, ga, cE, cP);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------
// message-row table (graph.cuh: MsgRows): count / scan / fill / finish, like K0 -- one CTA per molecule counts and
// fills, one CTA scans over molecules, no atomics.  Every index written is bounded by the array it goes to, so a
// capacity-mode batch that overflowed (flagged by K0, results invalid) stays inside the buffers.
// ---------------------------------------------------------------------------------
struct TypeBases { int tb[5]; };

__device__ __forceinline__ int type_of_row(int p, const int* tb, int G) {
  int t = G - 1;
  while (t > 0 && p < tb[t]) --t;
  return t;
}

// a source-CSR position that lists a kept entry (capacity mode: K0 writes row 0 for an entry it dropped)
__device__ __forceinline__ bool listed(const GraphArrays& ga, int e, int s) { return __ldg(ga.ent_src + e) == s; }

// entries of source slot s per type: m1 with w == 1 (one shared row), nn with another value (one row each)
__device__ __forceinline__ void slot_counts(int s, const GraphArrays& ga, const int* tb, int G, int* m1, int* nn) {
  for (int t = 0; t < 4; ++t) m1[t] = nn[t] = 0;
  const int q1 = __ldg(ga.src_ptr + s + 1);
  for (int q = __ldg(ga.src_ptr + s); q < q1; ++q) {
    const int e = __ldg(ga.src_ent + q);
    if (!listed(ga, e, s)) continue;
    const int t = type_of_row(e, tb, G);
    if (__ldg(ga.ent_w + e) == 1.f) ++m1[t];
    else ++nn[t];
  }
}

__device__ __forceinline__ void load_bases(int* tb, const int* dev_hdr, const TypeBases& hb, int G) {
  if (threadIdx.x <= (unsigned)G) tb[threadIdx.x] = dev_hdr ? dev_hdr[HDR_TYPE_BASE + threadIdx.x] : hb.tb[threadIdx.x];
  __syncthreads();
}

// tmp layout: molU[(G+1) B] (g == G: all types), molE[G B], offU[(G+1) B], offE[G B]
size_t msg_rows_tmp_ints(int B, int G) { return (size_t)(4 * G + 2) * B; }

__global__ void __launch_bounds__(128) mr_count_kernel(GraphArrays ga, MsgRows mr, const int* __restrict__ dev_hdr,
                                                       TypeBases hb, int N, int B, int G, int P) {
  __shared__ int sm[8];
  __shared__ int tb[5];
  for (long long p = (long long)blockIdx.x * 128 + threadIdx.x; p < P; p += (long long)gridDim.x * 128) mr.ent_u[p] = -1;
  load_bases(tb, dev_hdr, hb, G);
  const int b = blockIdx.x;
  int su[5] = {0, 0, 0, 0, 0}, se[4] = {0, 0, 0, 0};
  for (int i = threadIdx.x; i < N; i += 128) {
    int m1[4], nn[4];
    slot_counts(b * N + i, ga, tb, G, m1, nn);
    for (int t = 0; t < G; ++t) {
      const int u = (m1[t] > 0) + nn[t];
      su[t] += u; su[4] += u; se[t] += m1[t] + nn[t];
    }
  }
  int* molU = mr.tmp;
  int* molE = molU + (size_t)(G + 1) * B;
  for (int g = 0; g <= G; ++g) {
    int tot;
    block_exscan<128>(g < G ? su[g] : su[4], sm, &tot);
    if (threadIdx.x == 0) molU[(size_t)g * B + b] = tot;
    if (g < G) {
      block_exscan<128>(se[g], sm, &tot);
      if (threadIdx.x == 0) molE[(size_t)g * B + b] = tot;
    }
  }
}

__global__ void __launch_bounds__(1024) mr_scan_kernel(MsgRows mr, const int* __restrict__ dev_hdr, TypeBases hb, int B,
                                                       int G) {
  __shared__ int sm[34];
  __shared__ int tb[5];
  if (threadIdx.x < MR_META_INTS) mr.meta[threadIdx.x] = 0;   // the words of absent types (ordered by the barrier)
  load_bases(tb, dev_hdr, hb, G);
  const int* molU = mr.tmp;
  const int* molE = molU + (size_t)(G + 1) * B;
  int* offU = mr.tmp + (size_t)(2 * G + 1) * B;
  int* offE = offU + (size_t)(G + 1) * B;
  const int L = ceil_div(B, 1024);
  const int lo = min(B, (int)threadIdx.x * L), hi = min(B, lo + L);
  int eoff = 0;
  for (int k = 0; k <= 2 * G; ++k) {      // k < G: rows of type k; k == G: rows of all types; k > G: entries of type k-G-1
    const bool rows = k <= G;
    const int g = rows ? k : k - G - 1;
    const int* cnt = (rows ? molU : molE) + (size_t)g * B;
    int* off = (rows ? offU : offE) + (size_t)g * B;
    int s = 0;
    for (int b = lo; b < hi; ++b) s += cnt[b];
    int tot;
    int run = block_exscan<1024>(s, sm, &tot);
    for (int b = lo; b < hi; ++b) { off[b] = run; run += cnt[b]; }
    if (threadIdx.x == 0) {
      if (k < G) mr.meta[MR_COUNT + g] = max(0, min(tot, tb[g + 1] - tb[g]));   // an overflowing batch: no group spills
      else if (k == G) mr.meta[MR_TOTAL] = tot;
      else { mr.meta[MR_EOFF + g] = eoff; eoff += tot; }
    }
  }
  if (threadIdx.x <= (unsigned)G) mr.meta[MR_BASE + threadIdx.x] = tb[threadIdx.x];
  if (threadIdx.x == 0) mr.meta[MR_EOFF + G] = eoff;
}

__global__ void __launch_bounds__(128) mr_fill_kernel(GraphArrays ga, MsgRows mr, int N, int B, int G, int E, int P) {
  __shared__ int sm[8];
  __shared__ int meta[MR_META_INTS];
  if (threadIdx.x < MR_META_INTS) meta[threadIdx.x] = mr.meta[threadIdx.x];
  __syncthreads();
  const int* tb = meta + MR_BASE;
  const int b = blockIdx.x;
  const int* offU = mr.tmp + (size_t)(2 * G + 1) * B;
  const int* offE = offU + (size_t)(G + 1) * B;
  // each thread owns a contiguous run of the molecule's slots (N <= 181: at most two)
  const int L = ceil_div(N, 128);
  const int lo = min(N, (int)threadIdx.x * L), hi = min(N, lo + L);
  int runU[5], runE[4];
  for (int g = 0; g <= G; ++g) {
    int su = 0, se = 0;
    for (int i = lo; i < hi; ++i) {
      int m1[4], nn[4];
      slot_counts(b * N + i, ga, tb, G, m1, nn);
      if (g < G) { su += (m1[g] > 0) + nn[g]; se += m1[g] + nn[g]; }
      else for (int t = 0; t < G; ++t) su += (m1[t] > 0) + nn[t];
    }
    int tot;
    runU[g] = offU[(size_t)g * B + b] + block_exscan<128>(su, sm, &tot);
    if (g < G) runE[g] = meta[MR_EOFF + g] + offE[(size_t)g * B + b] + block_exscan<128>(se, sm, &tot);
  }
  for (int i = lo; i < hi; ++i) {
    const int s = b * N + i;
    int m1[4], nn[4];
    slot_counts(s, ga, tb, G, m1, nn);
    mr.s_ptr[s] = min(E, runU[G]);
    const int q0 = __ldg(ga.src_ptr + s), q1 = __ldg(ga.src_ptr + s + 1);
    for (int t = 0; t < G; ++t) {
      const int has1 = m1[t] > 0, r0 = runU[t], p0 = runE[t];
      auto row_of = [&](int local) { return local < meta[MR_COUNT + t] ? tb[t] + local : -1; };
      // rows of (s, t): the shared row first, then one per other entry; s_u lists them in the same order
      for (int k = 0; k < has1 + nn[t]; ++k) {
        const int row = row_of(r0 + k);
        if (row >= 0 && row < P) mr.u_ptr[row] = min(E, p0 + (k == 0 || !has1 ? k : m1[t] + k - 1));
        if (runU[G] + k < E) mr.s_u[runU[G] + k] = row < P ? row : -1;
      }
      int k1 = 0, kn = 0;
      for (int q = q0; q < q1; ++q) {
        const int e = __ldg(ga.src_ent + q);
        if (!listed(ga, e, s) || type_of_row(e, tb, G) != t) continue;
        const float w = __ldg(ga.ent_w + e);
        const bool shared = w == 1.f;
        const int local = shared ? r0 : r0 + has1 + kn;
        const int pos = shared ? p0 + k1 : p0 + m1[t] + kn;
        k1 += shared; kn += !shared;
        const int row = row_of(local);
        if (row >= 0 && row < P) {
          mr.u_src[row] = s;
          mr.u_w[row] = w;
          mr.ent_u[e] = row;
        }
        if (pos < E) mr.u_dst[pos] = __ldg(ga.ent_dst + e);
      }
      runU[t] += has1 + nn[t];
      runE[t] += m1[t] + nn[t];
      runU[G] += has1 + nn[t];
    }
  }
}

// pad rows, the closing CSR pointers, dst_u, and the unused tails of the E-sized arrays
__global__ void mr_finish_kernel(GraphArrays ga, MsgRows mr, long long S, int G, int E, int P) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int* meta = mr.meta;
  const int* tb = meta + MR_BASE;
  if (i < P) {
    const int p = (int)i, t = type_of_row(p, tb, G);
    if (p >= tb[t] + meta[MR_COUNT + t] || p >= tb[G]) {   // (type_of_row: p >= tb[t])
      mr.u_src[p] = -1;
      mr.u_w[p] = 0.f;
      mr.u_ptr[p] = min(E, meta[MR_EOFF + t + 1]);
    }
  }
  if (i < E) {
    const int q = (int)i;
    mr.dst_u[q] = q < __ldg(ga.dst_ptr + S) ? mr.ent_u[__ldg(ga.dst_ent + q)] : -1;
    if (q >= meta[MR_EOFF + G]) mr.u_dst[q] = -1;
    if (q >= meta[MR_TOTAL]) mr.s_u[q] = -1;
  }
  if (i == 0) {
    mr.u_ptr[P] = min(E, meta[MR_EOFF + G]);
    mr.s_ptr[S] = min(E, meta[MR_TOTAL]);
  }
}

int msg_rows_build(const GraphArrays& ga, const MsgRows& mr, const int* dev_hdr, const int* tb, int B, int N, int G,
                   int E, int P, cudaStream_t st) {
  if (G < 1 || G > 4 || B < 1) { set_error("msg_rows_build: %d bond-type groups, %d molecules", G, B); return -1; }
  TypeBases hb{};
  for (int g = 0; g <= G; ++g) hb.tb[g] = dev_hdr ? 0 : tb[g];
  mr_count_kernel<<<B, 128, 0, st>>>(ga, mr, dev_hdr, hb, N, B, G, P);
  GIB_LAUNCH_CHECK();
  mr_scan_kernel<<<1, 1024, 0, st>>>(mr, dev_hdr, hb, B, G);
  GIB_LAUNCH_CHECK();
  mr_fill_kernel<<<B, 128, 0, st>>>(ga, mr, N, B, G, E, P);
  GIB_LAUNCH_CHECK();
  const long long n = (P > E ? P : E) + 1;
  mr_finish_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(ga, mr, (long long)B * N, G, E, P);
  GIB_LAUNCH_CHECK();
  return 0;
}

}  // namespace gib
