// Generated batches -> the host table that `graph_to_graph` reads (GraphGenerator.py:659-804) and the histograms of
// `Analyzer.get_molecular_properties` (Analyzer.py:311-599), each in one pass over the batch.
//
// The table (int32 words, layout in include/gib200.h) is built as count / scan / fill: per-molecule counts, one
// single-CTA scan over molecules, then every record at its final offset.  No atomics; bonds come out in the order of
// `torch.nonzero(edge_features * triu(ones(N, N), 1))` (row-major (i, j, type) over the padded N x N x Ef).
// The statistics are a per-molecule pass into a workspace and one single-CTA pass that sums it over molecules in
// molecule order, as the reference's Python loops do.  The same per-molecule pass, on the int8 chunk of
// gib_preprocess_chunk, gives the training-set properties of each group it completed (one CTA per group, integer sums).
#include "common.cuh"
#include "../../include/gib200.h"

namespace gib {

namespace {

constexpr int kHdr = GIB_MOL_HDR_WORDS;
constexpr int kMolWords = GIB_MOL_WORDS;
constexpr int kNT = 128;
constexpr int kStatNT = 256;
constexpr int kMaxN = 255, kMaxEf = 16, kMaxF = 32767;

// torch.nonzero's notion of non-zero: NaN counts
__device__ __forceinline__ bool nonzero_f(float v) { return !(v == 0.f); }

// the bond list entry (i, j, t) of edge_features * triu(ones, 1): a NaN or an inf on or below the diagonal times 0 is
// NaN, which is listed
__device__ __forceinline__ bool listed(float v, int i, int j) { return nonzero_f(v * (j > i ? 1.f : 0.f)); }

__device__ __forceinline__ bool py_index_ok(int idx, int len) { return idx >= -len && idx < len; }

struct AtomRec {
  int nnz, i0, i1, i2, last;
};

__device__ __forceinline__ AtomRec atom_record(const float* row, int F) {
  AtomRec r{0, -1, -1, -1, -1};
  for (int f = 0; f < F; ++f) {
    if (nonzero_f(row[f])) {
      if (r.nnz == 0) r.i0 = f;
      else if (r.nnz == 1) r.i1 = f;
      else if (r.nnz == 2) r.i2 = f;
      r.last = f;
      ++r.nnz;
    }
  }
  return r;
}

// does `_features_to_atom` (GraphGenerator.py:672-730) return for this row, rather than raise IndexError?
__device__ __forceinline__ bool atom_decodes(const AtomRec& r, const gib_mol_layout& L) {
  if (r.nnz < 1 || !py_index_ok(r.i0, L.len_atom_types)) return false;
  if (r.nnz < 2 || !py_index_ok(r.i1 - L.n_atom_types, L.len_formal_charge)) return false;
  if (L.use_imp_H && (r.nnz < 3 || !py_index_ok(r.i2 - L.n_atom_types - L.n_formal_charge, L.len_imp_H)))
    return false;
  if (L.use_chirality &&
      !py_index_ok(r.last - L.n_atom_types - L.n_formal_charge - (L.use_imp_H ? L.n_imp_H : 0), L.len_chirality))
    return false;
  return true;
}

// ---- table phase 1: per-molecule counts and flags -------------------------------------------------------------
__global__ void __launch_bounds__(kNT) mol_count_kernel(int N, int F, int Ef, gib_mol_layout L,
                                                        const float* __restrict__ nodes,
                                                        const float* __restrict__ edges,
                                                        const signed char* __restrict__ n_nodes,
                                                        int* __restrict__ table) {
  __shared__ int sm[kNT / 32];
  const int b = blockIdx.x;
  const int n = n_nodes[b];
  const int na = min(max(n, 0), N);
  const float* nd = nodes + (size_t)b * N * F;
  const float* e = edges + (size_t)b * N * N * Ef;
  bool bad = false;
  for (int a = threadIdx.x; a < na; a += kNT) bad |= !atom_decodes(atom_record(nd + (size_t)a * F, F), L);
  // bonds: count, a bond to an atom >= n_nodes (KeyError in node_to_idx), an unordered pair listed twice
  int cnt = 0, flags = 0;
  for (int p = threadIdx.x; p < N * N; p += kNT) {
    const int i = p / N, j = p % N;
    int here = 0;
    for (int t = 0; t < Ef; ++t) here += listed(e[(size_t)p * Ef + t], i, j);
    cnt += here;
    if (here && (i >= n || j >= n)) flags |= GIB_MOL_KEY_ERROR;
    if (i <= j) {
      int pair = here;
      if (i < j)
        for (int t = 0; t < Ef; ++t) pair += listed(e[((size_t)j * N + i) * Ef + t], j, i);
      if (pair > 1 || (i == j && pair)) flags |= GIB_MOL_DUPLICATE_BOND;  // RDKit refuses a self bond too
    }
  }
  int total = 0;
  {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int v = cnt;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sm[wid] = v;
    __syncthreads();
    for (int w = 0; w < kNT / 32; ++w) total += sm[w];
  }
  const int any_bad = __syncthreads_or(bad);
  const int all_flags = __syncthreads_or(flags & GIB_MOL_KEY_ERROR) ? GIB_MOL_KEY_ERROR : 0;
  const int dup = __syncthreads_or(flags & GIB_MOL_DUPLICATE_BOND) ? GIB_MOL_DUPLICATE_BOND : 0;
  if (threadIdx.x == 0) {
    int* m = table + kHdr + (size_t)b * kMolWords;
    const bool decodes = !any_bad && n <= N;  // row N does not exist: node_features[N] raises IndexError
    m[0] = n;
    m[1] = na;
    m[2] = total;
    m[5] = (decodes ? GIB_MOL_DECODES : 0) | all_flags | dup;
  }
}

// ---- table phase 2: offsets (single CTA, molecule order) --------------------------------------------------------
template <int NT>
__device__ __forceinline__ int cta_exscan(int v, int* sm, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();
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

__global__ void __launch_bounds__(1024) mol_scan_kernel(int B, int* __restrict__ table) {
  __shared__ int sm[1024 / 32 + 1];
  const int L = ceil_div(B, 1024);
  const int lo = min(B, (int)threadIdx.x * L), hi = min(B, lo + L);
  int flags_or = 0;
  for (int k = 0; k < 2; ++k) {  // k = 0: atom records, 1: bonds
    int s = 0;
    for (int b = lo; b < hi; ++b) s += table[kHdr + (size_t)b * kMolWords + 1 + k];
    int tot;
    int run = cta_exscan<1024>(s, sm, &tot);
    for (int b = lo; b < hi; ++b) {
      int* m = table + kHdr + (size_t)b * kMolWords;
      m[3 + k] = run;
      run += m[1 + k];
      if (k == 0) flags_or |= m[5];
    }
    if (threadIdx.x == 0) table[k] = tot;
  }
  const int key_error = __syncthreads_or(flags_or & GIB_MOL_KEY_ERROR);
  const int duplicate = __syncthreads_or(flags_or & GIB_MOL_DUPLICATE_BOND);
  flags_or = (key_error ? GIB_MOL_KEY_ERROR : 0) | (duplicate ? GIB_MOL_DUPLICATE_BOND : 0);
  if (threadIdx.x == 0) {
    table[2] = -1;  // statistics error words: written by gib_graph_statistics
    table[3] = 0;
    table[4] = 0;
    table[5] = flags_or;
    table[6] = 0;
    table[7] = 0;
  }
}

// ---- table phase 3: atom and bond records at their offsets ------------------------------------------------------
__global__ void __launch_bounds__(kNT) mol_fill_kernel(int B, int N, int F, int Ef, const float* __restrict__ nodes,
                                                       const float* __restrict__ edges, int* __restrict__ table) {
  __shared__ int sm[kNT / 32 + 1];
  const int b = blockIdx.x;
  const int* m = table + kHdr + (size_t)b * kMolWords;
  const int na = m[1], atom_off = m[3], bond_off = m[4];
  const size_t atom_base = kHdr + (size_t)B * kMolWords;
  const size_t bond_base = atom_base + (size_t)GIB_MOL_ATOM_WORDS * table[0];
  const float* nd = nodes + (size_t)b * N * F;
  short* atoms = reinterpret_cast<short*>(table + atom_base) + (size_t)atom_off * 2 * GIB_MOL_ATOM_WORDS;
  for (int a = threadIdx.x; a < na; a += kNT) {
    const AtomRec r = atom_record(nd + (size_t)a * F, F);
    short* o = atoms + (size_t)a * 2 * GIB_MOL_ATOM_WORDS;
    o[0] = (short)r.nnz;
    o[1] = (short)r.i0;
    o[2] = (short)r.i1;
    o[3] = (short)r.i2;
    o[4] = (short)r.last;
    o[5] = 0;
  }
  // bonds: ordered compaction over the row-major (i, j, t) entries, kNT entries per step
  const float* e = edges + (size_t)b * N * N * Ef;
  unsigned* bonds = reinterpret_cast<unsigned*>(table + bond_base) + bond_off;
  const int total = N * N * Ef;
  int run = 0;
  for (int base = 0; base < total; base += kNT) {
    const int q = base + threadIdx.x;
    int v = 0, i = 0, j = 0, t = 0;
    if (q < total) {
      t = q % Ef;
      const int p = q / Ef;
      i = p / N;
      j = p % N;
      v = listed(e[q], i, j);
    }
    int step;
    const int pos = cta_exscan<kNT>(v, sm, &step);
    if (v) bonds[run + pos] = (unsigned)i | ((unsigned)j << 8) | ((unsigned)t << 16);
    run += step;
  }
}

// ---- statistics: per molecule ---------------------------------------------------------------------------------
// workspace per molecule: F column sums, Ef bond-type sums (f32), 10 n_edges bins, n_nodes, error (i32)
__host__ __device__ inline size_t stat_ws_words(int F, int Ef) { return (size_t)F + Ef + 10 + 2; }

// One molecule's partials, shared by the generated batches (float32 input) and the preprocessed chunks (int8 input):
// n_eff atoms are binned; s_row / s_bin are shared scratch of the calling CTA (kStatNT threads).
template <typename T>
__device__ __forceinline__ void mol_stats_one(int N, int F, int Ef, int n_eff, const T* __restrict__ nd,
                                              const T* __restrict__ e, float* __restrict__ w, float* s_row,
                                              int* s_bin) {
  int* wi = reinterpret_cast<int*>(w + F + Ef);
  for (int f = threadIdx.x; f < F; f += kStatNT) {  // torch.sum(node_features, dim=0) over all N padded rows
    float acc = 0.f;
    for (int r = 0; r < N; ++r) acc += (float)nd[(size_t)r * F + f];
    w[f] = acc;
  }
  for (int i = threadIdx.x; i < N; i += kStatNT) {  // torch.sum(edges[i, :, t])
    for (int t = 0; t < Ef; ++t) {
      float acc = 0.f;
      for (int j = 0; j < N; ++j) acc += (float)e[((size_t)i * N + j) * Ef + t];
      s_row[i * Ef + t] = acc;
    }
  }
  __syncthreads();
  // per atom: n_edges = sum_t int(row sum), clamped at 10, binned at n_edges - 1 (Python's negative indexing)
  for (int i = threadIdx.x; i < n_eff; i += kStatNT) {
    long long ne = 0;
    int code = 0;
    for (int t = 0; t < Ef && !code; ++t) {
      const float s = s_row[i * Ef + t];
      if (isnan(s)) code = GIB_MOL_ERR_VALUE;          // int(nan): ValueError
      else if (isinf(s)) code = GIB_MOL_ERR_OVERFLOW;  // int(inf): OverflowError
      else ne += (long long)fmaxf(fminf(truncf(s), 1e12f), -1e12f);
    }
    int bin = -1;
    if (!code) {
      const long long idx = min(ne, 10LL) - 1;
      if (idx < -10) code = GIB_MOL_ERR_INDEX;
      else bin = (int)(idx < 0 ? idx + 10 : idx);
    }
    s_bin[i] = code ? -code : bin;
  }
  __syncthreads();
  if (threadIdx.x < 10) {
    int c = 0;
    for (int i = 0; i < n_eff; ++i) c += s_bin[i] == (int)threadIdx.x;
    wi[threadIdx.x] = c;
  } else if (threadIdx.x == 10) {
    int err = -1;
    for (int i = 0; i < n_eff && err < 0; ++i)
      if (s_bin[i] < 0) err = i * 4 - s_bin[i];
    wi[11] = err;
  } else if (threadIdx.x == 11) {
    wi[10] = n_eff;
  } else if (threadIdx.x >= 32 && threadIdx.x < 32 + Ef) {  // torch.sum(edges[:, :, t]) over the padded N x N
    const int t = threadIdx.x - 32;
    float acc = 0.f;
    for (int i = 0; i < N; ++i) acc += s_row[i * Ef + t];
    w[F + t] = acc;
  }
}

__global__ void __launch_bounds__(kStatNT) mol_stats_kernel(int N, int F, int Ef, const float* __restrict__ nodes,
                                                            const float* __restrict__ edges,
                                                            const int* __restrict__ table, float* __restrict__ ws) {
  __shared__ float s_row[kMaxN * kMaxEf];
  __shared__ int s_bin[kMaxN];
  const int b = blockIdx.x;
  const int* m = table + kHdr + (size_t)b * kMolWords;
  // GenerationGraph.n_nodes: molecule.GetNumAtoms(), 0 when graph_to_graph gave mol = None
  const int n_eff = (m[5] & GIB_MOL_DECODES) ? max(m[0], 0) : 0;
  mol_stats_one(N, F, Ef, n_eff, nodes + (size_t)b * N * F, edges + (size_t)b * N * N * Ef,
                ws + (size_t)b * stat_ws_words(F, Ef), s_row, s_bin);
}

// ---- statistics: over molecules, in molecule order (single CTA) -------------------------------------------------
__global__ void __launch_bounds__(kStatNT) mol_stats_sum_kernel(int B, int N, int F, int Ef,
                                                                const float* __restrict__ ws, int* __restrict__ table,
                                                                float* __restrict__ out) {
  const size_t W = stat_ws_words(F, Ef);
  const int o_nf = N + 1, o_ne = o_nf + F, o_ef = o_ne + 10, o_sum = o_ef + Ef;
  for (int k = threadIdx.x; k <= N; k += kStatNT) {
    int c = 0;
    for (int b = 0; b < B; ++b) c += reinterpret_cast<const int*>(ws + b * W + F + Ef)[10] == k;
    out[k] = (float)c;
  }
  for (int f = threadIdx.x; f < F; f += kStatNT) {
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc += ws[b * W + f];
    out[o_nf + f] = acc;
  }
  for (int k = threadIdx.x; k < 10; k += kStatNT) {
    int c = 0;
    for (int b = 0; b < B; ++b) c += reinterpret_cast<const int*>(ws + b * W + F + Ef)[k];
    out[o_ne + k] = (float)c;
  }
  for (int t = threadIdx.x; t < Ef; t += kStatNT) {  // edge_feature_hist[t] += torch.sum(edges[:, :, t]) / 2
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc += ws[b * W + F + t] * 0.5f;
    out[o_ef + t] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {  // sum_n_nodes = sum_k k * n_nodes_hist[k]
    float acc = 0.f;
    for (int k = 0; k <= N; ++k) acc += (float)k * out[k];
    out[o_sum] = acc;
  } else if (threadIdx.x == 32) {  // sum_n_edges = sum_k (k + 1) * n_edges_hist[k]
    float acc = 0.f;
    for (int k = 0; k < 10; ++k) acc += (float)(k + 1) * out[o_ne + k];
    out[o_sum + 1] = acc;
  } else if (threadIdx.x == 64) {  // the first molecule whose statistics raise in the reference
    int mol = -1, err = -1;
    for (int b = 0; b < B && mol < 0; ++b) {
      const int v = reinterpret_cast<const int*>(ws + b * W + F + Ef)[11];
      if (v >= 0) {
        mol = b;
        err = v;
      }
    }
    table[2] = mol;
    table[3] = mol < 0 ? 0 : err & 3;
    table[4] = mol < 0 ? 0 : err >> 2;
  }
}

// ---- training-set properties of the groups of one gib_preprocess_chunk call ----------------------------------------
// per molecule of the chunk that ended up in a group: the partials above from the int8 graph, with
// n_nodes = the rows up to the last non-zero one (PreprocessingGraph.n_nodes = GetNumAtoms(): the chunk pass refuses a
// zero row between atoms)
__global__ void __launch_bounds__(kStatNT) pp_mol_stats_kernel(int N, int F, int Ef,
                                                               const signed char* __restrict__ nodes,
                                                               const signed char* __restrict__ edges,
                                                               const int* __restrict__ status, float* __restrict__ ws) {
  __shared__ float s_row[kMaxN * kMaxEf];
  __shared__ int s_bin[kMaxN];
  __shared__ int s_last;
  const int b = blockIdx.x;
  if (b >= status[1]) return;  // not in a completed group (status[1] is 0 when the chunk was refused)
  const signed char* nd = nodes + (size_t)b * N * F;
  if (threadIdx.x == 0) s_last = -1;
  __syncthreads();
  int last = -1;
  for (int r = threadIdx.x; r < N; r += kStatNT) {
    bool any = false;
    for (int f = 0; f < F; ++f) any |= nd[(size_t)r * F + f] != 0;
    if (any) last = r;
  }
  atomicMax(&s_last, last);
  __syncthreads();
  mol_stats_one(N, F, Ef, s_last + 1, nd, edges + (size_t)b * N * N * Ef, ws + (size_t)b * stat_ws_words(F, Ef),
                s_row, s_bin);
}

// one CTA per group, each output word summed over the group's molecules in molecule order, in integers
__host__ __device__ inline int pp_stat_words(int N, int F, int Ef) { return 4 + N + 1 + F + 10 + Ef; }

__global__ void __launch_bounds__(kStatNT) pp_group_stats_kernel(int N, int F, int Ef, const float* __restrict__ ws,
                                                                 const int* __restrict__ groups,
                                                                 const int* __restrict__ status, int* __restrict__ out) {
  const size_t W = stat_ws_words(F, Ef);
  const int S = pp_stat_words(N, F, Ef);
  const int o_nf = 4 + N + 1, o_ne = o_nf + F, o_ef = o_ne + 10;
  const int ng = status[0];
  for (int g = blockIdx.x; g < ng; g += gridDim.x) {
    const int s = groups[4 * g], e = groups[4 * g + 1];
    int* o = out + (size_t)g * S;
    for (int k = threadIdx.x; k < S; k += kStatNT) {
      int acc = 0;
      if (k < 4) {
        acc = groups[4 * g + k];
      } else if (k < o_nf) {                           // n_nodes_hist[k - 4]
        for (int m = s; m < e; ++m) acc += reinterpret_cast<const int*>(ws + m * W + F + Ef)[10] == k - 4;
      } else if (k < o_ne) {                           // node-feature column sums
        for (int m = s; m < e; ++m) acc += (int)ws[m * W + (k - o_nf)];
      } else if (k < o_ef) {                           // n_edges_hist
        for (int m = s; m < e; ++m) acc += reinterpret_cast<const int*>(ws + m * W + F + Ef)[k - o_ne];
      } else {                                         // bonds per type: the symmetric entry sum / 2
        for (int m = s; m < e; ++m) acc += (int)ws[m * W + F + (k - o_ef)] / 2;
      }
      o[k] = acc;
    }
  }
}

int check_mol_dims(const char* who, int B, int N, int F, int Ef) {
  if (B < 1 || N < 1 || N > kMaxN || F < 1 || F > kMaxF || Ef < 1 || Ef > kMaxEf) {
    set_error("%s: unsupported dims B=%d N=%d F=%d Ef=%d (need B >= 1, 1 <= N <= %d, 1 <= F <= %d, 1 <= Ef <= %d)",
              who, B, N, F, Ef, kMaxN, kMaxF, kMaxEf);
    return -1;
  }
  return 0;
}

}  // namespace
}  // namespace gib

using namespace gib;

extern "C" {

size_t gib_molecule_table_bytes(int B, int N, int F, int Ef) {
  if (check_mol_dims("gib_molecule_table_bytes", B, N, F, Ef)) return 0;
  return 4 * ((size_t)kHdr + (size_t)B * kMolWords + (size_t)B * N * GIB_MOL_ATOM_WORDS + (size_t)B * N * N * Ef);
}

int gib_molecule_table(int B, int N, int F, int Ef, const gib_mol_layout* layout, const float* nodes,
                       const float* edges, const signed char* n_nodes, int* table, gib_stream stream) {
  GIB_TRY(check_mol_dims("gib_molecule_table", B, N, F, Ef));
  if (!layout || !nodes || !edges || !n_nodes || !table) {
    set_error("gib_molecule_table: null argument");
    return -1;
  }
  const gib_mol_layout L = *layout;
  if (L.n_atom_types < 0 || L.n_formal_charge < 0 || L.n_imp_H < 0 || L.len_atom_types < 0 ||
      L.len_formal_charge < 0 || L.len_imp_H < 0 || L.len_chirality < 0) {
    set_error("gib_molecule_table: negative layout field");
    return -1;
  }
  cudaStream_t s = (cudaStream_t)stream;
  mol_count_kernel<<<B, kNT, 0, s>>>(N, F, Ef, L, nodes, edges, n_nodes, table);
  GIB_LAUNCH_CHECK();
  mol_scan_kernel<<<1, 1024, 0, s>>>(B, table);
  GIB_LAUNCH_CHECK();
  mol_fill_kernel<<<B, kNT, 0, s>>>(B, N, F, Ef, nodes, edges, table);
  GIB_LAUNCH_CHECK();
  return 0;
}

size_t gib_graph_statistics_bytes(int N, int F, int Ef) {
  if (check_mol_dims("gib_graph_statistics_bytes", 1, N, F, Ef)) return 0;
  return 4 * ((size_t)N + 1 + F + 10 + Ef + 2);
}

size_t gib_graph_statistics_ws_bytes(int B, int N, int F, int Ef) {
  if (check_mol_dims("gib_graph_statistics_ws_bytes", B, N, F, Ef)) return 0;
  return 4 * (size_t)B * stat_ws_words(F, Ef);
}

int gib_graph_statistics(int B, int N, int F, int Ef, const float* nodes, const float* edges, int* table, float* out,
                         void* ws, gib_stream stream) {
  GIB_TRY(check_mol_dims("gib_graph_statistics", B, N, F, Ef));
  if (!nodes || !edges || !table || !out || !ws) {
    set_error("gib_graph_statistics: null argument");
    return -1;
  }
  cudaStream_t s = (cudaStream_t)stream;
  mol_stats_kernel<<<B, kStatNT, 0, s>>>(N, F, Ef, nodes, edges, table, (float*)ws);
  GIB_LAUNCH_CHECK();
  mol_stats_sum_kernel<<<1, kStatNT, 0, s>>>(B, N, F, Ef, (const float*)ws, table, out);
  GIB_LAUNCH_CHECK();
  return 0;
}

size_t gib_preprocess_group_statistics_bytes(const gib_pp_dims* d, int max_groups) {
  if (gib_preprocess_apd_length(d) < 0) return 0;
  if (check_mol_dims("gib_preprocess_group_statistics_bytes", max_groups, d->N, d->F, d->Ef)) return 0;
  return 4 * (size_t)max_groups * pp_stat_words(d->N, d->F, d->Ef);
}

size_t gib_preprocess_group_statistics_ws_bytes(const gib_pp_dims* d, int max_molecules) {
  if (gib_preprocess_apd_length(d) < 0) return 0;
  if (check_mol_dims("gib_preprocess_group_statistics_ws_bytes", max_molecules, d->N, d->F, d->Ef)) return 0;
  return 4 * (size_t)max_molecules * stat_ws_words(d->F, d->Ef);
}

int gib_preprocess_group_statistics(const gib_pp_dims* d, const signed char* nodes, const signed char* edges,
                                    int n_molecules, int max_molecules, const int* groups, const int* status,
                                    void* ws, int* out, gib_stream stream) {
  if (!gib_preprocess_group_statistics_ws_bytes(d, max_molecules)) return -1;
  if (n_molecules < 1 || n_molecules > max_molecules) {
    set_error("gib_preprocess_group_statistics: n_molecules %d outside [1, max_molecules = %d]", n_molecules,
              max_molecules);
    return -1;
  }
  if (!nodes || !edges || !groups || !status || !ws || !out) {
    set_error("gib_preprocess_group_statistics: null argument");
    return -1;
  }
  cudaStream_t s = (cudaStream_t)stream;
  pp_mol_stats_kernel<<<n_molecules, kStatNT, 0, s>>>(d->N, d->F, d->Ef, nodes, edges, status, (float*)ws);
  GIB_LAUNCH_CHECK();
  pp_group_stats_kernel<<<min(n_molecules, 1024), kStatNT, 0, s>>>(d->N, d->F, d->Ef, (const float*)ws, groups,
                                                                    status, out);
  GIB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
