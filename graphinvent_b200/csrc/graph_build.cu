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

}  // namespace gib
