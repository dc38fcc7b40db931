// Training-set construction (DataProcesser.get_subgraphs, DataProcesser.py:167-271, over the decoding routes of
// PreprocessingGraph, MolecularGraph.py:463-555, 635-732) for one chunk of molecules:
//
//   count   one warp per molecule: validates the padded one-hot graph, route length n_edges + 2
//   scan    one CTA: the molecules' first state index (states of the chunk are numbered in route order)
//   route   one warp per molecule, graph in shared memory: truncates step by step and emits per state the flat target
//           APD index, the node count and a 64-bit content hash (a sum of per-byte mixes, updated as bytes are
//           zeroed), plus per molecule the step at which each bond goes (`rs`): state k holds the bonds with rs > k
//           and node rows [0, nn)
//   group   one CTA, groups in order, the group's state in device memory: streams the group's states in tiles of
//           1024, finds each state's first occurrence in the group (hash table + exact byte comparison of the
//           candidates, never the hash alone), applies the reference's append rule, counts rows and cuts at B
//   emit    one CTA per row: the row's int8 bytes from the input graph and `rs`, a zeroed int32 APD row
//   scatter one thread per processed state: +1 at (row of its first occurrence, APD) and, for a row appended by the
//           "match on the last row" rule, at its own row too (integer atomics: order-free, deterministic)
//
// Append rule (DataProcesser.py:204-231): the reference scans its rows for the first equal one, adds the APD there,
// and appends the state when no row matched OR the match was the last row.  Rows are appended in state order and a
// first occurrence is always appended, so with pf(i) = the latest first occurrence at or before state i, a repeated
// state i is appended iff first(i) == pf(i) and no state in (pf(i), i) was appended the same way.
#include <algorithm>
#include <climits>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "action_mask.cuh"
#include "scaffold_mask.cuh"
#include "../../include/gib200.h"

namespace gib {

namespace {

constexpr int kGroupNT = 1024;
constexpr int kEmitNT = 128;
constexpr int kMaxNodeBytes = 8192;
constexpr unsigned long long kEmpty = ~0ull;

// status words (int32 [GIB_PP_STATUS_INTS], documented per entry point in gib200.h)
constexpr int kStGroups = 0;       // gib_preprocess_chunk: groups written
constexpr int kStSetSize = 0;      // gib_molset_identify: the set's entries before the call
constexpr int kStNext = 1;         // gib_preprocess_chunk: the molecule after the last one visited
constexpr int kStRouteFlags = 1;   // the conditional route plan: GIB_ROUTE_* flags
constexpr int kStRows = 2;         // gib_preprocess_chunk: rows written
constexpr int kStRouteFirst = 2;   // the conditional route plan: the first molecule with a GIB_ROUTE_* flag
constexpr int kStFlags = 3;        // GIB_PP_* flags
constexpr int kStFirstBad = 4;     // the first molecule with a GIB_PP_* flag
constexpr int kStTotal = 5;        // the scan's total: the chunk's states, gib_murcko's new entries
constexpr int kCursor = 6;         // the route fill: replays of the chunk done so far (its batch index)

struct PP {
  int N, F, Ef, B;
  int nseg, seg[4];
  int f_add;      // len_f_add_per_node = prod(seg) * Ef
  int apd_len;    // N * (f_add + Ef) + 1
  int s_max;      // most states of one valid molecule: N (N - 1) / 2 + 2
};

struct WsLayout {
  size_t len, n0, off, rs, hash, apd, nn, mol, slot, row_of, dst, own, row_state, keys, vals, total;
  long long states, table;
};

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// a workspace cut into consecutive 256-byte-aligned pieces: take(bytes) is the next piece's offset, end the total
struct Carve {
  size_t end = 0;
  size_t take(size_t bytes) {
    const size_t r = end;
    end = align256(end + bytes);
    return r;
  }
};

WsLayout ws_layout(const PP& p, int max_mols, int max_rows) {
  WsLayout w{};
  w.states = (long long)max_mols * p.s_max;
  const long long window = (long long)(max_mols < p.B ? max_mols : p.B) * p.s_max;
  w.table = 1024;
  while (w.table < 2 * window) w.table <<= 1;
  Carve c;
  w.len = c.take(4ull * max_mols);
  w.n0 = c.take(4ull * max_mols);
  w.off = c.take(4ull * (max_mols + 1));
  w.rs = c.take(2ull * max_mols * p.N * p.N);
  w.hash = c.take(8ull * w.states);
  w.apd = c.take(4ull * w.states);
  w.nn = c.take(4ull * w.states);
  w.mol = c.take(4ull * w.states);
  w.slot = c.take(4ull * w.states);
  w.row_of = c.take(4ull * w.states);
  w.dst = c.take(4ull * w.states);
  w.own = c.take(4ull * w.states);
  w.row_state = c.take(4ull * max_rows);
  w.keys = c.take(8ull * w.table);
  w.vals = c.take(4ull * w.table);
  w.total = c.end;
  return w;
}

int make_pp(const char* who, const gib_pp_dims* d, PP* out) {
  if (!d) {
    set_error("%s: null dims", who);
    return -1;
  }
  PP p{};
  p.N = d->N, p.F = d->F, p.Ef = d->Ef, p.B = d->batch_size;
  if (p.N < 1 || p.F < 1 || p.Ef < 1 || (long long)p.N * p.N * p.Ef > 32768) {
    set_error("%s: unsupported dims N=%d F=%d Ef=%d (need N, F, Ef >= 1 and N*N*Ef <= 32768)", who, p.N, p.F, p.Ef);
    return -1;
  }
  if ((long long)p.N * p.F > kMaxNodeBytes) {
    set_error("%s: N*F = %lld exceeds %d", who, (long long)p.N * p.F, kMaxNodeBytes);
    return -1;
  }
  if (p.B < 1) {
    set_error("%s: batch_size %d < 1", who, p.B);
    return -1;
  }
  if (d->n_atom_types < 1 || d->n_formal_charge < 1 || d->n_imp_H < 0 || d->n_chirality < 0) {
    set_error("%s: layout needs n_atom_types >= 1, n_formal_charge >= 1, n_imp_H >= 0, n_chirality >= 0 "
              "(0 = segment absent), got %d %d %d %d", who, d->n_atom_types, d->n_formal_charge, d->n_imp_H,
              d->n_chirality);
    return -1;
  }
  const int segs[4] = {d->n_atom_types, d->n_formal_charge, d->n_imp_H, d->n_chirality};
  long long width = 0, prod = 1;
  for (int s : segs) {
    if (s == 0) continue;
    p.seg[p.nseg++] = s;
    width += s;
    prod *= s;
  }
  if (width != p.F) {
    set_error("%s: F=%d is not the sum of the layout's segment widths (%lld)", who, p.F, width);
    return -1;
  }
  const long long f_add = prod * p.Ef, apd = (long long)p.N * (f_add + p.Ef) + 1;
  if (apd > INT_MAX / 2) {
    set_error("%s: APD length %lld exceeds %d", who, apd, INT_MAX / 2);
    return -1;
  }
  p.f_add = (int)f_add;
  p.apd_len = (int)apd;
  p.s_max = p.N * (p.N - 1) / 2 + 2;
  *out = p;
  return 0;
}

// ---- hashing: sum over the state's non-zero bytes of a 64-bit mix of (position, byte) ----------------------------
__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ unsigned long long byte_hash(long long pos, signed char v) {
  return v ? mix64(((unsigned long long)pos << 8) | (unsigned char)v) : 0ull;
}
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_max(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- bond cell (i, j) of the dense edges E [N, N, Ef] ---------------------------------------------------------------
// a bond: any non-zero byte
__device__ __forceinline__ bool has_bond(const signed char* E, int N, int Ef, int i, int j) {
  const signed char* c = E + ((size_t)i * N + j) * Ef;
  bool any = false;
  for (int t = 0; t < Ef; ++t) any |= c[t] != 0;
  return any;
}
// its type: the first non-zero byte's index, -1 without a bond
__device__ __forceinline__ int bond_type(const signed char* E, int N, int Ef, int i, int j) {
  const signed char* c = E + ((size_t)i * N + j) * Ef;
  for (int t = 0; t < Ef; ++t)
    if (c[t]) return t;
  return -1;
}

__device__ __forceinline__ void flag_bad(int* status, int flags, int m) {
  atomicOr(&status[kStFlags], flags);
  atomicMin(&status[kStFirstBad], m);
}

// scaffold != 0 (the conditional route plan): the first molecule with a GIB_ROUTE_* flag starts at INT_MAX
__global__ void pp_init_kernel(int* status, unsigned long long* keys, int* vals, long long table, int scaffold) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (int i = 0; i < GIB_PP_STATUS_INTS; ++i) status[i] = 0;
    status[kStFirstBad] = INT_MAX;
    if (scaffold) status[kStRouteFirst] = INT_MAX;
  }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < table; i += (long long)gridDim.x * blockDim.x) {
    keys[i] = kEmpty;
    vals[i] = INT_MAX;
  }
}

__device__ __forceinline__ void flag_scaffold(int* status, int flags, int m) {
  atomicOr(&status[kStRouteFlags], flags);
  atomicMin(&status[kStRouteFirst], m);
}

// The comparison that defines "molecule atoms phi(0..k-1) are scaffold s": node row phi(i) equals scaffold row i in
// all F bytes and, for every i, j < k, edge cell (phi(i), phi(j)) equals scaffold cell (i, j) in all Ef bytes (an
// induced match: an extra bond among the image differs).  phi = null is the identity, the prefix rule of the
// conditional route plan; scaffold_first_kernel confirms every embedding its search finds with it.  One warp, every
// lane gets the answer; *nnz (per lane, summed by the caller) counts the scaffold's non-zero edge bytes.
__device__ bool scaffold_differs(const PP& p, const signed char* X, const signed char* E, const signed char* SX,
                                 const signed char* SE, int k, const short* phi, int* nnz) {
  const int lane = threadIdx.x & 31;
  const int N = p.N, F = p.F, Ef = p.Ef;
  bool diff = false;
  int z = 0;
  // a molecule of fewer atoms has a zero row there, the scaffold does not
  for (int q = lane; q < k * F; q += 32) {
    const int i = q / F, a = phi ? phi[i] : i;
    diff |= X[(size_t)a * F + q % F] != SX[q];
  }
  for (int q = lane; q < k * k; q += 32) {
    const int i = q / k, j = q % k;
    const size_t ij = (size_t)i * N + j, ab = (size_t)(phi ? phi[i] : i) * N + (phi ? phi[j] : j);
    for (int t = 0; t < Ef; ++t) {
      const signed char w = SE[ij * Ef + t];
      diff |= E[ab * Ef + t] != w;
      z += w != 0;
    }
  }
  *nnz = z;
  return __any_sync(0xffffffffu, diff);
}

// the conditional route of molecule m decorating scaffold ids[m] (>= 0): its first k_s node rows and the edges among
// them must equal the scaffold's (one warp, every lane gets the answer).  Returns the states kept, n_edges - m_k + 1
// (m_k: the scaffold's bonds), or 0 with a GIB_ROUTE_* flag raised.  ids[m] = -1: the whole route, n_edges + 2.
__device__ int conditional_length(const PP& p, const gib_scaffolds& sc, int sid, const signed char* X,
                                  const signed char* E, int e, int m, int* status) {
  const int lane = threadIdx.x & 31;
  const int N = p.N, F = p.F, Ef = p.Ef;
  if (sid < -1 || sid >= sc.S) {
    if (lane == 0) flag_scaffold(status, GIB_ROUTE_BAD_ID, m);
    return 0;
  }
  if (sid < 0) return e + 2;
  const int k = sc.n_atoms[sid];
  int nnz;
  if (scaffold_differs(p, X, E, sc.nodes + (size_t)sid * N * F, sc.edges + (size_t)sid * N * N * Ef, k, nullptr,
                       &nnz)) {
    if (lane == 0) flag_scaffold(status, GIB_ROUTE_NOT_PREFIX, m);
    return 0;
  }
  return e - warp_sum(nnz) / 2 + 1;
}

// ---- the input checks of one padded graph (one warp, every lane gets the results) -------------------------------
// Returns its GIB_PP_BAD_NODES / GIB_PP_BAD_EDGES / GIB_PP_EMPTY flags; *n = its atom count (rows up to the last
// non-zero one), *nnz = its non-zero edge bytes.
__device__ int validate_graph(const PP& p, const signed char* X, const signed char* E, int* n_out, int* nnz_out) {
  const int lane = threadIdx.x & 31;
  const int N = p.N, F = p.F, Ef = p.Ef;
  int last = -1, bad = 0;
  for (int r = lane; r < N; r += 32) {
    const signed char* row = X + (size_t)r * F;
    bool any = false, ok = true;
    int base = 0;
    for (int j = 0; j < p.nseg; ++j) {
      int c = 0;
      for (int f = 0; f < p.seg[j]; ++f) {
        const signed char v = row[base + f];
        c += v != 0;
        ok &= v == 0 || v == 1;
      }
      any |= c > 0;
      ok &= c == 1;
      base += p.seg[j];
    }
    if (any) last = r;
    if (any && !ok) bad |= GIB_PP_BAD_NODES;
  }
  const int n = warp_max(last) + 1;
  // every row below n must be a node
  for (int r = lane; r < n; r += 32) {
    bool any = false;
    for (int f = 0; f < F; ++f) any |= X[(size_t)r * F + f] != 0;
    if (!any) bad |= GIB_PP_BAD_NODES;
  }
  int nnz = 0;
  for (int q = lane; q < N * N; q += 32) {
    const int i = q / N, j = q % N;
    int c = 0;
    for (int t = 0; t < Ef; ++t) {
      const signed char v = E[(size_t)q * Ef + t];
      const signed char w = E[((size_t)j * N + i) * Ef + t];
      c += v != 0;
      if (v != w || (v != 0 && (v != 1 || i == j || i >= n || j >= n))) bad |= GIB_PP_BAD_EDGES;
    }
    if (c > 1) bad |= GIB_PP_BAD_EDGES;
    nnz += c;
  }
  nnz = warp_sum(nnz);
  bad = __reduce_or_sync(0xffffffffu, bad);
  if (n == 0) bad |= GIB_PP_EMPTY;
  *n_out = n;
  *nnz_out = nnz;
  return bad;
}

// ---- count: validation and route length (one warp per molecule) ------------------------------------------------
// ids != null (the conditional route plan): the length is that of molecule m's conditional route.  bad_out != null:
// each molecule's GIB_PP_* input flags (0: it passed), for a later kernel that must leave refused molecules alone
__global__ void __launch_bounds__(32) pp_count_kernel(PP p, const signed char* __restrict__ nodes,
                                                      const signed char* __restrict__ edges, int* len, int* n0,
                                                      int* status, const int* __restrict__ ids, gib_scaffolds sc,
                                                      int* bad_out = nullptr) {
  const int m = blockIdx.x;
  const int N = p.N, F = p.F, Ef = p.Ef;
  const signed char* X = nodes + (size_t)m * N * F;
  const signed char* E = edges + (size_t)m * N * N * Ef;
  int n, nnz;
  const int bad = validate_graph(p, X, E, &n, &nnz);
  const int e = min(nnz / 2, p.s_max - 2);
  const int kept = ids && !bad ? conditional_length(p, sc, ids[m], X, E, e, m, status) : e + 2;
  if (threadIdx.x == 0) {
    if (bad) flag_bad(status, bad, m);
    len[m] = bad ? 2 : kept;
    n0[m] = n;
    if (bad_out) bad_out[m] = bad;
  }
}

// ---- scan: off[m] = sum of len[0, m), off[n] = total (one CTA) ---------------------------------------------------
__global__ void __launch_bounds__(1024) pp_scan_kernel(int n, const int* len, int* off, int* status) {
  __shared__ int sm[32];
  __shared__ int carry;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < n ? len[i] : 0;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) sm[wid] = inc;
    __syncthreads();
    if (wid == 0) {
      int w = sm[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += t;
      }
      sm[lane] = w;
    }
    __syncthreads();
    const int c = carry;
    const int excl = c + (wid ? sm[wid - 1] : 0) + inc - v;
    if (i < n) off[i] = excl;
    __syncthreads();
    if (threadIdx.x == 0) carry = c + sm[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    off[n] = carry;
    status[kStTotal] = carry;
  }
}

// ---- route: one warp per molecule ------------------------------------------------------------------------------
// ids != null (the conditional route plan): only the first off[m+1] - off[m] states (truncation order) are emitted --
// the conditional route, from the full graph back to the scaffold's state -- each kept action is checked against the
// attachment-point rule (GIB_ROUTE_MASKED), and the scaffold's bonds, which no kept step removes, get step SHRT_MAX
__global__ void __launch_bounds__(32) pp_route_kernel(PP p, const signed char* __restrict__ nodes,
                                                      const signed char* __restrict__ edges, const int* off,
                                                      const int* n0, unsigned long long* hash, int* apd, int* nn,
                                                      int* mol, short* rs_all, int* status,
                                                      const int* __restrict__ ids, gib_scaffolds sc) {
  extern __shared__ __align__(16) unsigned char smem[];
  if (status[kStFlags]) return;
  const int m = blockIdx.x, lane = threadIdx.x;
  if (ids && off[m + 1] == off[m]) return;      // refused by the count stage (GIB_ROUTE_NOT_PREFIX / _BAD_ID)
  const int sid = ids ? ids[m] : -1;
  const unsigned int* pm = sid >= 0 && sc.protect ? sc.protect + (size_t)sid * 4 : nullptr;
  const int ks = sid >= 0 ? sc.n_atoms[sid] : 0;
  const int N = p.N, F = p.F, Ef = p.Ef;
  const int nb = N * F, eb = N * N * Ef;
  int* sflat = reinterpret_cast<int*>(smem);
  signed char* X = reinterpret_cast<signed char*>(smem + 4 * N);
  signed char* E = X + nb;
  const signed char* Xg = nodes + (size_t)m * nb;
  const signed char* Eg = edges + (size_t)m * eb;
  short* rs = rs_all + (size_t)m * N * N;
  unsigned long long h = 0;
  for (int q = lane; q < nb; q += 32) {
    X[q] = Xg[q];
    h += byte_hash(q, X[q]);
  }
  for (int q = lane; q < eb; q += 32) {
    E[q] = Eg[q];
    h += byte_hash(nb + q, E[q]);
  }
  for (int q = lane; q < N * N; q += 32) rs[q] = 0;
  h = warp_sum_u64(h);
  int n = n0[m];
  for (int r = lane; r < n; r += 32) {        // flat (segment-relative) index of the node's one-hot entries
    int flat = 0, base = 0;
    for (int j = 0; j < p.nseg; ++j) {
      int idx = 0;
      for (int f = 0; f < p.seg[j]; ++f)
        if (X[r * F + base + f]) idx = f;
      flat = flat * p.seg[j] + idx;
      base += p.seg[j];
    }
    sflat[r] = flat;
  }
  __syncwarp();
  const int s0 = off[m], steps = off[m + 1] - s0 - 1;
  auto emit = [&](int k, int a) {
    if (lane == 0) {
      const int i = s0 + k;
      hash[i] = h == kEmpty ? kEmpty - 1 : h;
      apd[i] = a;
      nn[i] = n;
      mol[i] = m;
      if (pm && scaffold_forbidden(a, n, ks, pm, N, Ef, p.f_add)) flag_scaffold(status, GIB_ROUTE_MASKED, m);
    }
  };
  emit(0, p.apd_len - 1);
  for (int k = 1; k <= steps; ++k) {
    const int last = n - 1;
    int deg = 0, key = -1;
    for (int q = lane; q < N * Ef; q += 32) {
      const int v = q / Ef, t = q % Ef;
      if (E[((size_t)v * N + last) * Ef + t]) {
        ++deg;
        key = max(key, t * N + v);
      }
    }
    deg = warp_sum(deg);
    key = warp_max(key);
    const int v = key % N, t = key / N;
    int a;
    if (deg == 0) a = sflat[last] * Ef;
    else if (deg == 1) a = v * p.f_add + sflat[last] * Ef + t;
    else a = N * p.f_add + v * Ef + t;
    if (n > 1 && deg == 0) {                     // the reference's truncate_graph raises IndexError here
      if (lane == 0) flag_bad(status, GIB_PP_DISCONNECTED, m);
      return;
    }
    unsigned long long dh = 0;
    if (n == 1 || deg == 1) {
      for (int f = lane; f < F; f += 32) {
        dh += byte_hash((long long)last * F + f, X[last * F + f]);
        X[last * F + f] = 0;
      }
    }
    if (n > 1) {
      for (int u = lane; u < 2 * Ef; u += 32) {
        const int tt = u % Ef;
        const size_t q = u < Ef ? ((size_t)v * N + last) * Ef + tt : ((size_t)last * N + v) * Ef + tt;
        dh += byte_hash(nb + (long long)q, E[q]);
        E[q] = 0;
      }
      if (lane == 0) rs[v * N + last] = rs[last * N + v] = (short)k;
    }
    h -= warp_sum_u64(dh);
    if (n == 1 || deg == 1) --n;
    __syncwarp();
    emit(k, a);
  }
  if (ids)
    for (int q = lane; q < N * N; q += 32)
      if (has_bond(E, N, Ef, q / N, q % N)) rs[q] = SHRT_MAX;
}

// ---- exact comparison of two states (one warp; every lane gets the answer) --------------------------------------
struct StateRef {
  const int* off;
  const int* nn;
  const int* mol;
  const short* rs;
  const signed char* nodes;
  const signed char* edges;
};

__device__ bool warp_states_equal(const PP& p, const StateRef& S, int i1, int i2) {
  const int n = S.nn[i1];
  if (S.nn[i2] != n) return false;
  const int m1 = S.mol[i1], m2 = S.mol[i2];
  const int k1 = i1 - S.off[m1], k2 = i2 - S.off[m2];
  const int N = p.N, F = p.F, Ef = p.Ef;
  const signed char* X1 = S.nodes + (size_t)m1 * N * F;
  const signed char* X2 = S.nodes + (size_t)m2 * N * F;
  const signed char* E1 = S.edges + (size_t)m1 * N * N * Ef;
  const signed char* E2 = S.edges + (size_t)m2 * N * N * Ef;
  const short* r1 = S.rs + (size_t)m1 * N * N;
  const short* r2 = S.rs + (size_t)m2 * N * N;
  bool diff = false;
  // node rows >= n and bonds touching them are zero in both states (count / route invariants)
  for (int q = threadIdx.x & 31; q < n * F; q += 32) diff |= X1[q] != X2[q];
  for (int q = threadIdx.x & 31; q < n * n; q += 32) {
    const int a = q / n, b = q % n, ab = a * N + b;
    const bool p1 = r1[ab] > k1, p2 = r2[ab] > k2;
    for (int t = 0; t < Ef; ++t) {
      const signed char v1 = p1 ? E1[(size_t)ab * Ef + t] : 0;
      const signed char v2 = p2 ? E2[(size_t)ab * Ef + t] : 0;
      diff |= v1 != v2;
    }
  }
  return !__any_sync(0xffffffffu, diff);
}

// the first state in [t0, i) equal to state i (i itself when none): the path taken when the table's earliest state
// of i's hash differs from it in content
__device__ int warp_first_equal(const PP& p, const StateRef& S, const unsigned long long* hash, int t0, int i,
                                unsigned long long h) {
  const int lane = threadIdx.x & 31;
  for (int jb = t0; jb < i; jb += 32) {
    const int j = jb + lane;
    unsigned cand = __ballot_sync(0xffffffffu, j < i && hash[j] == h);
    while (cand) {
      const int src = __ffs(cand) - 1;
      cand &= cand - 1;
      if (warp_states_equal(p, S, jb + src, i)) return jb + src;
    }
  }
  return i;
}

// CTA-wide inclusive scans / reductions over kGroupNT threads; `total` gets the CTA-wide result
__device__ __forceinline__ int cta_scan(int v, bool is_max, int* sm, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc = is_max ? max(inc, t) : inc + t;
  }
  __syncthreads();
  if (lane == 31) sm[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int w = sm[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w = is_max ? max(w, t) : w + t;
    }
    sm[lane] = w;
  }
  __syncthreads();
  if (wid) inc = is_max ? max(inc, sm[wid - 1]) : inc + sm[wid - 1];
  *total = sm[31];
  return inc;
}

__device__ __forceinline__ int tbl_insert(unsigned long long* keys, unsigned long long h, long long mask) {
  long long s = (long long)(h & (unsigned long long)mask);
  while (true) {
    const unsigned long long k = atomicCAS(&keys[s], kEmpty, h);
    if (k == kEmpty || k == h) return (int)s;
    s = (s + 1) & mask;
  }
}

__global__ void __launch_bounds__(kGroupNT) pp_group_kernel(PP p, StateRef S, int n_mols, int last_chunk,
                                                            int max_rows, const unsigned long long* hash,
                                                            unsigned long long* keys, int* vals, long long mask,
                                                            int* slot, int* row_of, int* dst, int* own,
                                                            int* row_state, int* groups, int* status) {
  __shared__ int sm[32];
  __shared__ int prev[kGroupNT];
  __shared__ int cut_sm;
  const int tid = threadIdx.x, lane = tid & 31;
  if (status[kStFlags]) {
    __syncthreads();
    if (tid == 0) status[kStGroups] = status[kStNext] = status[kStRows] = 0;
    return;
  }
  const int B = p.B;
  const int* off = S.off;
  int s = 0, rows_used = 0, ng = 0;
  while (s < n_mols && rows_used + B <= max_rows) {
    const int w_end = min(s + B, n_mols);
    const bool truncated = s + B > n_mols && !last_chunk;
    const int t0 = off[s], t1 = off[w_end];
    int pf = -1, lastcand = -1, rows = 0, cut = -1, tend = t0;
    for (int base = t0; base < t1 && cut < 0; base += kGroupNT) {
      const int i = base + tid;
      const bool valid = i < t1;
      tend = min(base + kGroupNT, t1);
      unsigned long long h = 0;
      int sl = -1;
      if (valid) {
        h = hash[i];
        sl = tbl_insert(keys, h, mask);
        atomicMin(&vals[sl], i);
        slot[i] = sl;
      }
      __syncthreads();
      int f = valid ? __ldcg(&vals[sl]) : -1;
      unsigned need = __ballot_sync(0xffffffffu, valid && f != i);
      while (need) {
        const int src = __ffs(need) - 1;
        need &= need - 1;
        const int ii = __shfl_sync(0xffffffffu, i, src), ff = __shfl_sync(0xffffffffu, f, src);
        const unsigned long long hh = __shfl_sync(0xffffffffu, h, src);
        int res = ff;
        if (!warp_states_equal(p, S, ii, ff)) res = warp_first_equal(p, S, hash, t0, ii, hh);
        if (lane == src) f = res;
      }
      const bool fo = valid && f == i;
      int tot;
      const int pfi = max(pf, cta_scan(fo ? i : -1, true, sm, &tot));
      const int pf_next = max(pf, tot);
      const bool cand = valid && !fo && f == pfi;
      const int cinc = cta_scan(cand ? i : -1, true, sm, &tot);
      const int lastcand_next = max(lastcand, tot);
      // the largest candidate index strictly below i: the inclusive scan of the previous thread
      prev[tid] = cinc;
      __syncthreads();
      const int below = max(lastcand, tid ? prev[tid - 1] : -1);
      const bool app = fo || (cand && below < pfi);
      const int cnt = rows + cta_scan(app ? 1 : 0, false, sm, &tot);
      const int cnt_total = rows + tot;
      // the cut: the state whose append makes the group B rows (at most one per tile)
      if (tid == 0) cut_sm = INT_MAX;
      __syncthreads();
      if (app && cnt == B) cut_sm = i;
      __syncthreads();
      const int c = cut_sm;
      const bool proc = valid && i <= c;
      if (proc && app) {
        row_of[i] = rows_used + cnt - 1;
        row_state[rows_used + cnt - 1] = i;
      }
      __syncthreads();
      if (valid) {
        dst[i] = proc ? row_of[f] : -1;
        own[i] = proc && app && !fo ? row_of[i] : -1;
      }
      pf = pf_next;
      lastcand = lastcand_next;
      if (c != INT_MAX) {
        cut = c;
        rows = B;
      } else {
        rows = cnt_total;
      }
      __syncthreads();
    }
    if (cut < 0 && truncated) {
      for (int i = t0 + tid; i < tend; i += kGroupNT) {
        keys[slot[i]] = kEmpty;
        vals[slot[i]] = INT_MAX;
      }
      break;
    }
    const int e = cut >= 0 ? S.mol[cut] + 1 : w_end;
    for (int i = tend + tid; i < off[e]; i += kGroupNT) dst[i] = own[i] = -1;   // the cut molecule's dropped states
    for (int i = t0 + tid; i < tend; i += kGroupNT) {
      keys[slot[i]] = kEmpty;
      vals[slot[i]] = INT_MAX;
    }
    if (tid == 0) {
      groups[4 * ng + 0] = s;
      groups[4 * ng + 1] = e;
      groups[4 * ng + 2] = rows_used;
      groups[4 * ng + 3] = rows;
    }
    ++ng;
    rows_used += rows;
    s = e;
    __syncthreads();
  }
  if (tid == 0) {
    status[kStGroups] = ng;
    status[kStNext] = s;
    status[kStRows] = rows_used;
  }
}

// ---- emit: one CTA per row ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(kEmitNT) pp_emit_kernel(PP p, StateRef S, const int* row_state, const int* status,
                                                          signed char* out_nodes, signed char* out_edges,
                                                          int* out_apds) {
  const int rows = status[kStRows];
  const int N = p.N, F = p.F, Ef = p.Ef;
  for (int r = blockIdx.x; r < rows; r += gridDim.x) {
    const int i = row_state[r];
    const int m = S.mol[i], k = i - S.off[m], n = S.nn[i];
    const signed char* X = S.nodes + (size_t)m * N * F;
    const signed char* E = S.edges + (size_t)m * N * N * Ef;
    const short* rs = S.rs + (size_t)m * N * N;
    signed char* on = out_nodes + (size_t)r * N * F;
    signed char* oe = out_edges + (size_t)r * N * N * Ef;
    int* oa = out_apds + (size_t)r * p.apd_len;
    for (int q = threadIdx.x; q < N * F; q += kEmitNT) on[q] = q / F < n ? X[q] : 0;
    for (int q = threadIdx.x; q < N * N * Ef; q += kEmitNT) oe[q] = rs[q / Ef] > k ? E[q] : 0;
    for (int q = threadIdx.x; q < p.apd_len; q += kEmitNT) oa[q] = 0;
  }
}

__global__ void pp_scatter_kernel(PP p, const int* off, const int* apd, const int* dst, const int* own,
                                  const int* status, int* out_apds) {
  const int n = off[status[kStNext]];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int a = apd[i], d = dst[i], o = own[i];
    if (d >= 0) atomicAdd(&out_apds[(size_t)d * p.apd_len + a], 1);
    if (o >= 0) atomicAdd(&out_apds[(size_t)o * p.apd_len + a], 1);
  }
}

// ---- count -> scan -> route: the decoding routes of n molecules, shared by the training-set construction and the
// route scorer ----------------------------------------------------------------------------------------------------
struct RouteBufs {
  int* len;
  int* n0;
  int* off;
  short* rs;
  unsigned long long* hash;
  int* apd;
  int* nn;
  int* mol;
};

// ids / sc (the conditional route plan): each molecule's route from its scaffold's state on, see pp_count_kernel
int launch_route(const PP& p, const signed char* nodes, const signed char* edges, int n, const RouteBufs& r,
                 int* status, cudaStream_t s, const int* ids = nullptr, const gib_scaffolds* sc = nullptr) {
  const gib_scaffolds scv = sc ? *sc : gib_scaffolds{};
  pp_count_kernel<<<n, 32, 0, s>>>(p, nodes, edges, r.len, r.n0, status, ids, scv);
  GIB_LAUNCH_CHECK();
  pp_scan_kernel<<<1, 1024, 0, s>>>(n, r.len, r.off, status);
  GIB_LAUNCH_CHECK();
  const size_t smem = 4 * (size_t)p.N + (size_t)p.N * p.F + (size_t)p.N * p.N * p.Ef;
  pp_route_kernel<<<n, 32, smem, s>>>(p, nodes, edges, r.off, r.n0, r.hash, r.apd, r.nn, r.mol, r.rs, status, ids,
                                      scv);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ---- the route scorer (graphinvent_b200.graphed.RouteScorer): its plan workspace, the fill of one batch of route
// states into the model's static int8 inputs, the per-molecule reduction ----------------------------------------
constexpr int kFillNT = 256;
constexpr int kFillMaxBlocks = 4096;

struct RouteWs {
  size_t len, n0, rs, hash, apd, nn, mol, total;
};

RouteWs route_ws_layout(const PP& p, int max_mols) {
  RouteWs w{};
  const long long states = (long long)max_mols * p.s_max;
  Carve c;
  w.len = c.take(4ull * max_mols);
  w.n0 = c.take(4ull * max_mols);
  w.rs = c.take(2ull * max_mols * p.N * p.N);
  w.hash = c.take(8ull * states);
  w.apd = c.take(4ull * states);
  w.nn = c.take(4ull * states);
  w.mol = c.take(4ull * states);
  w.total = c.end;
  return w;
}

struct FillSrc {
  const signed char* nodes;
  const signed char* edges;
  const int* off;
  const int* nn;
  const int* mol;
  const int* apd;
  const short* rs;
};

// one 16-byte chunk of the flat [B, rb] output (edges_part: the edges array, else the nodes array): each row segment
// it covers comes from its state's molecule through the aligned-word funnel, then the bytes the state does not hold
// (node rows >= nn, bonds with rs <= k) are cleared.  Rows past the chunk's last state are zero.
__device__ __forceinline__ void fill_chunk(const PP& p, const FillSrc& f, bool edges_part, long long c, int s0,
                                           int S, signed char* dst) {
  const int rb = edges_part ? p.N * p.N * p.Ef : p.N * p.F;
  const long long total = (long long)p.B * rb;
  const long long e0 = c * 16;
  const int n = (int)min(16LL, total - e0);
  long long r = e0 / rb;
  int col = (int)(e0 - r * rb);
  u128 v = 0;
  for (int k = 0; k < n;) {
    const int seg = min(n - k, rb - col);
    const int i = s0 + (int)r;
    if (i < S) {
      const int m = f.mol[i];
      const uint8_t* src = reinterpret_cast<const uint8_t*>(edges_part ? f.edges : f.nodes) + (size_t)m * rb + col;
      u128 s = load_span(src, seg);
      if (edges_part) {
        const int step = i - f.off[m];
        const short* rs = f.rs + (size_t)m * p.N * p.N;
        for (int j = 0; j < seg; ++j)
          if (rs[(col + j) / p.Ef] <= step) s &= ~((u128)0xff << (8 * j));
      } else {
        const int nn = f.nn[i];
        for (int j = 0; j < seg; ++j)
          if ((col + j) / p.F >= nn) s &= ~((u128)0xff << (8 * j));
      }
      if (seg < 16) s &= ((u128)1 << (8 * seg)) - 1;
      v |= s << (8 * k);
    }
    k += seg;
    ++r;
    col = 0;
  }
  signed char* out = dst + e0;
  if (n == 16) {
    st16(out, v);
  } else {
    for (int j = 0; j < n; ++j) out[j] = (signed char)(uint8_t)(v >> (8 * j));
  }
}

// states [s0, s0 + B) of the chunk, s0 = status[kCursor] * B, into the model's int8 inputs; per slot b its action and
// its place in the likelihood buffer (build order: the molecule's empty graph first), -1 / -1 past the last state.
// ids != null (the conditional route): also each slot's scaffold id and atom count, the mask's inputs (-1 / -1 for
// a molecule scored whole and past the last state)
__global__ void __launch_bounds__(kFillNT) route_fill_kernel(PP p, FillSrc f, const int* __restrict__ status,
                                                             gib_batch_ctl* ctl, int* __restrict__ slots,
                                                             signed char* __restrict__ out_nodes,
                                                             signed char* __restrict__ out_edges,
                                                             long long node_chunks, long long edge_chunks,
                                                             const int* __restrict__ ids, int* __restrict__ slot_ids,
                                                             int* __restrict__ slot_n) {
  const int B = p.B, S = status[kStTotal], s0 = status[kCursor] * B;
  const long long tid = (long long)blockIdx.x * kFillNT + threadIdx.x, stride = (long long)gridDim.x * kFillNT;
  if (tid == 0) ctl->live = max(0, min(B, S - s0));
  for (long long b = tid; b < B; b += stride) {
    const int i = s0 + (int)b;
    int a = -1, d = -1, sid = -1, n = -1;
    if (i < S) {
      const int m = f.mol[i];
      a = f.apd[i];
      d = f.off[m] + f.off[m + 1] - 1 - i;
      if (ids && ids[m] >= 0) {
        sid = ids[m];
        n = f.nn[i];
      }
    }
    slots[b] = a;
    slots[B + b] = d;
    if (ids) {
      slot_ids[b] = sid;
      slot_n[b] = n;
    }
  }
  for (long long c = tid; c < node_chunks + edge_chunks; c += stride) {
    if (c < node_chunks) fill_chunk(p, f, false, c, s0, S, out_nodes);
    else fill_chunk(p, f, true, c - node_chunks, s0, S, out_edges);
  }
}

// per molecule, in build order: nll = -sum log p and final = log(sum p), both accumulated in fp64 and rounded once
__global__ void route_reduce_kernel(int n, const int* __restrict__ off, const float* __restrict__ lik,
                                    float* __restrict__ nll, float* __restrict__ fin) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n) return;
  double l = 0.0, s = 0.0;
  for (int i = off[m]; i < off[m + 1]; ++i) {
    const double q = (double)lik[i];
    l -= log(q);
    s += q;
  }
  nll[m] = (float)l;
  fin[m] = (float)log(s);
}

// the backward of route_probs + route_reduce in log p, one warp per molecule: coef[s] = dL/d log p_s =
// g_lik[s] p_s - g_nll[m] + g_final[m] p_s / sum p, with sum p summed in fp64 in build order as route_reduce sums it
// (lane 0), each coefficient evaluated in fp64 and rounded once.  A null gradient counts as zero.
constexpr int kCoefWarps = 4;
__global__ void __launch_bounds__(32 * kCoefWarps) route_grad_coef_kernel(int n, const int* __restrict__ off,
                                                                          const float* __restrict__ lik,
                                                                          const float* __restrict__ g_lik,
                                                                          const float* __restrict__ g_nll,
                                                                          const float* __restrict__ g_fin,
                                                                          float* __restrict__ coef) {
  const int m = blockIdx.x * kCoefWarps + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (m >= n) return;
  const int a = off[m], e = off[m + 1];
  const double gn = g_nll ? (double)g_nll[m] : 0.0;
  const double gf = g_fin ? (double)g_fin[m] : 0.0;
  double s = 0.0;
  if (gf != 0.0 && lane == 0)
    for (int i = a; i < e; ++i) s += (double)lik[i];
  s = __shfl_sync(0xffffffffu, s, 0);
  for (int i = a + lane; i < e; i += 32) {
    const double p = (double)lik[i];
    double c = -gn;
    if (g_lik) c += (double)g_lik[i] * p;
    if (gf != 0.0) c += gf * p / s;
    coef[i] = (float)c;
  }
}

// the action mask's rule on the planned routes: one warp per molecule.  Every kept state's action against the structural
// rule with its state's atom count -- a route state never holds the bond its connect adds, so the duplicate-bond test
// has nothing to find -- and, with valence, every atom of the whole molecule (state 0 of the plan: valences only grow
// along a route, so its states are all within the table exactly when the molecule is)
__global__ void __launch_bounds__(32) route_action_check_kernel(ActionLayout L, int F, const int* __restrict__ off,
                                                                const int* __restrict__ apd,
                                                                const int* __restrict__ nn,
                                                                const signed char* __restrict__ nodes,
                                                                const signed char* __restrict__ edges, int valence,
                                                                const int* __restrict__ table, int* result) {
  const int m = blockIdx.x, lane = threadIdx.x, N = L.N;
  const int s0 = off[m], s1 = off[m + 1];
  if (s1 == s0) return;                       // refused by the plan (GIB_ROUTE_NOT_PREFIX / _BAD_ID)
  bool bad = false;
  for (int s = s0 + lane; s < s1; s += 32) bad |= structure_forbidden(decode_action(apd[s], L), L, nn[s], 0.f);
  if (valence) {
    const int* order = table + L.A * L.CH;
    const int n = min(max(nn[s0], 0), N);
    for (int i = lane; i < n; i += 32) {
      const int2 u = atom_usage(nodes + ((size_t)m * N + i) * F, edges + (((size_t)m * N + i) * N) * L.Ef, L, table,
                                order, order + L.Ef);
      bad |= u.x > u.y;
    }
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) {
    atomicOr(&result[0], GIB_ROUTE_ACTION);
    atomicMin(&result[1], m);
  }
}

bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

int route_limits(const char* who, const gib_pp_dims* d, int max_molecules, PP* p) {
  GIB_TRY(make_pp(who, d, p));
  if (max_molecules < 1 || (long long)max_molecules * p->s_max >= INT_MAX / 2) {
    set_error("%s: need max_molecules >= 1 and max_molecules * (N*(N-1)/2 + 2) < %d states, got %d", who,
              INT_MAX / 2, max_molecules);
    return -1;
  }
  return 0;
}

// the scaffold table of the conditional route plan and of gib_scaffold_first
int check_scaffolds(const char* who, const gib_scaffolds* sc, const PP& p) {
  if (!sc || sc->S <= 0 || !sc->nodes || !sc->edges || !sc->n_atoms) {
    set_error("%s: the scaffold table needs S >= 1 and its nodes, edges and n_atoms buffers", who);
    return -1;
  }
  if (sc->protect && p.N > 127) {     // protect holds 4 x 32 bits per scaffold, as the generator's mask reads it
    set_error("%s: attachment points need N <= 127 (4 protect words per scaffold), got N=%d", who, p.N);
    return -1;
  }
  return 0;
}

// gib_route_plan (sc, ids null), and with conditional set gib_route_plan_scaffold
int route_plan(const char* who, const gib_pp_dims* d, const signed char* nodes, const signed char* edges,
               int n_molecules, int max_molecules, bool conditional, const gib_scaffolds* sc, const int* ids,
               void* ws, int* offsets, int* status, gib_stream stream) {
  PP p;
  GIB_TRY(route_limits(who, d, max_molecules, &p));
  if (n_molecules < 1 || n_molecules > max_molecules) {
    set_error("%s: n_molecules %d outside [1, max_molecules = %d]", who, n_molecules, max_molecules);
    return -1;
  }
  if (!nodes || !edges || !ws || !offsets || !status || (conditional && !ids)) {
    set_error("%s: null argument", who);
    return -1;
  }
  if (conditional) GIB_TRY(check_scaffolds(who, sc, p));
  const RouteWs w = route_ws_layout(p, max_molecules);
  char* b = static_cast<char*>(ws);
  cudaStream_t s = (cudaStream_t)stream;
  pp_init_kernel<<<1, 32, 0, s>>>(status, nullptr, nullptr, 0, conditional);
  GIB_LAUNCH_CHECK();
  return launch_route(p, nodes, edges, n_molecules,
                      RouteBufs{(int*)(b + w.len), (int*)(b + w.n0), offsets, (short*)(b + w.rs),
                                (unsigned long long*)(b + w.hash), (int*)(b + w.apd), (int*)(b + w.nn),
                                (int*)(b + w.mol)},
                      status, s, ids, sc);
}

// gib_route_fill (ids, slot_ids, slot_n null), and with conditional set gib_route_fill_scaffold
int route_fill(const char* who, const gib_pp_dims* d, const signed char* nodes, const signed char* edges,
               int max_molecules, const void* ws, const int* offsets, const int* status, bool conditional,
               const int* ids, gib_batch_ctl* ctl, int* slots, int* slot_ids, int* slot_n, signed char* out_nodes,
               signed char* out_edges, gib_stream stream) {
  PP p;
  GIB_TRY(route_limits(who, d, max_molecules, &p));
  if (!nodes || !edges || !ws || !offsets || !status || !ctl || !slots || !out_nodes || !out_edges ||
      (conditional && (!ids || !slot_ids || !slot_n))) {
    set_error("%s: null argument", who);
    return -1;
  }
  if (!aligned16(nodes) || !aligned16(edges) || !aligned16(out_nodes) || !aligned16(out_edges)) {
    set_error("%s: nodes, edges, out_nodes and out_edges must be 16-byte aligned", who);
    return -1;
  }
  const RouteWs w = route_ws_layout(p, max_molecules);
  const char* b = static_cast<const char*>(ws);
  const FillSrc f{nodes, edges, offsets, (const int*)(b + w.nn), (const int*)(b + w.mol), (const int*)(b + w.apd),
                  (const short*)(b + w.rs)};
  const long long nc = ceil_div_ll((long long)p.B * p.N * p.F, 16);
  const long long ec = ceil_div_ll((long long)p.B * p.N * p.N * p.Ef, 16);
  const long long need = std::max<long long>(ceil_div_ll(nc + ec, kFillNT), ceil_div_ll(p.B, kFillNT));
  const int blocks = (int)std::min<long long>(need, kFillMaxBlocks);
  route_fill_kernel<<<blocks, kFillNT, 0, (cudaStream_t)stream>>>(
      p, f, status, ctl, slots, out_nodes, out_edges, nc, ec, ids, slot_ids, slot_n);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ---- node_remap (MolecularGraph.py:435-461, 328-433, 592-614): one warp per molecule -------------------------------
// The BFS / DFS of the reference from atom ranking[0], then reorder_nodes.  Adjacency bitsets and the ranking live in
// shared memory; the search runs on lane 0 and the reordered bytes are written by the whole warp.
constexpr int kReorderMaxN = 181;                           // N*N*Ef <= 32768
constexpr int kReorderWords = (kReorderMaxN + 31) / 32;
constexpr int kSetMaxSlots = 512;                           // the table of a set of <= 306 small ints (CPython 3.12)
constexpr int kSetLinearProbes = 9, kSetPerturbShift = 5;   // Objects/setobject.c

// ---- per-molecule graph helpers of the one-warp-per-molecule kernels below -------------------------------------------
// The bonds among atoms 0..n-1 of E as bitsets, bit j of row i (one warp): `any` [N][kReorderWords] every bond, and
// `typed` [Ef][N][ceil(N / 32)] each bond under its bond_type; either may be null.  The N atoms' rows are cleared
// first.  Returns this lane's count of bonded cells (i, j).
__device__ int load_adjacency(const signed char* E, int N, int Ef, int n, unsigned (*any)[kReorderWords],
                              unsigned* typed) {
  const int lane = threadIdx.x & 31, W = (N + 31) / 32;
  if (any)
    for (int q = lane; q < N * W; q += 32) any[q / W][q % W] = 0;
  if (typed)
    for (int q = lane; q < Ef * N * W; q += 32) typed[q] = 0;
  __syncwarp();
  int cells = 0;
  for (int q = lane; q < n * n; q += 32) {
    const int i = q / n, j = q % n, t = bond_type(E, N, Ef, i, j);
    if (t < 0) continue;
    ++cells;
    if (any) atomicOr(&any[i][j >> 5], 1u << (j & 31));
    if (typed) atomicOr(&typed[((size_t)t * N + i) * W + (j >> 5)], 1u << (j & 31));
  }
  __syncwarp();
  return cells;
}

// deg[i] = atom i's bonds among atoms 0..k-1 (0 for i >= k), i < N (one warp); returns their bonds (every lane)
__device__ int prefix_degrees(const signed char* E, int N, int Ef, int k, short* deg) {
  int total = 0;
  for (int i = threadIdx.x & 31; i < N; i += 32) {
    int d = 0;
    for (int j = 0; j < k && i < k; ++j) d += has_bond(E, N, Ef, i, j);
    deg[i] = (short)d;
    total += d;
  }
  return warp_sum(total) / 2;
}

// lane 0: how many atoms the bitset rows adj reach from `start` (start included), frontier by frontier
__device__ int reach(const unsigned (*adj)[kReorderWords], int W, int start) {
  unsigned vis[kReorderWords], front[kReorderWords];
#pragma unroll
  for (int w = 0; w < kReorderWords; ++w) vis[w] = front[w] = w == start >> 5 ? 1u << (start & 31) : 0u;
  int count = 1;
  for (bool grew = true; grew;) {
    unsigned next[kReorderWords] = {};
#pragma unroll
    for (int w = 0; w < kReorderWords; ++w)
      for (unsigned b = front[w]; b; b &= b - 1) {
        const int a = w * 32 + __ffs(b) - 1;
#pragma unroll
        for (int v = 0; v < kReorderWords; ++v)
          if (v < W) next[v] |= adj[a][v];
      }
    grew = false;
#pragma unroll
    for (int w = 0; w < kReorderWords; ++w) {
      front[w] = next[w] & ~vis[w];
      vis[w] |= front[w];
      count += __popc(front[w]);
      grew |= front[w] != 0;
    }
  }
  return count;
}

// CPython 3.12's set table for small non-negative ints (hash = value, no deletions): set_add_entry's probe sequence
// (LINEAR_PROBES slots after the home slot while they fit, then perturbation), set_table_resize on the fill rule
// (fill * 5 >= mask * 3 -> the smallest power of two above used * 4) re-inserting in old-table order.  Iterating the
// table in slot order is list(set(...)).
struct PySet {
  short* slot;   // [kSetMaxSlots], -1 = empty
  short* tmp;    // [kReorderMaxN]
  int mask, used;

  __device__ void clear() {
    mask = 7;
    used = 0;
    for (int i = 0; i <= mask; ++i) slot[i] = -1;
  }
  // set_insert_clean / the probe of set_add_entry; returns the slot holding `key` or the empty slot for it
  __device__ int find(int key) const {
    size_t perturb = (size_t)key, i = (size_t)key & mask;
    while (true) {
      const int probes = i + kSetLinearProbes <= (size_t)mask ? kSetLinearProbes : 0;
      for (int j = 0; j <= probes; ++j)
        if (slot[i + j] < 0 || slot[i + j] == key) return (int)(i + j);
      perturb >>= kSetPerturbShift;
      i = (i * 5 + 1 + perturb) & mask;
    }
  }
  __device__ void add(int key) {
    const int s = find(key);
    if (slot[s] == key) return;
    slot[s] = (short)key;
    ++used;                                                 // fill == used: nothing is ever deleted
    if ((size_t)used * 5 < (size_t)mask * 3) return;
    int n = 0;
    for (int i = 0; i <= mask; ++i)
      if (slot[i] >= 0) tmp[n++] = slot[i];
    int size = 8;
    while (size <= used * 4) size <<= 1;
    mask = size - 1;
    for (int i = 0; i <= mask; ++i) slot[i] = -1;
    for (int k = 0; k < n; ++k) slot[find(tmp[k])] = tmp[k];
  }
};

// the highest-ranked atom of bitset `cand` (-1: empty)
__device__ __forceinline__ int best_of(const unsigned* cand, const int* rank, int W) {
  int best = -1, br = -1;
  for (int w = 0; w < W; ++w)
    for (unsigned b = cand[w]; b; b &= b - 1) {
      const int a = w * 32 + __ffs(b) - 1;
      if (rank[a] > br) br = rank[a], best = a;
    }
  return best;
}

// a uniformly random permutation of 0..n-1 per molecule, a function of (seed, epoch, molecule) only: atom i's rank is
// its place among the counter-based keys mix64(seed, epoch, molecule, i), ties broken by atom index
__device__ void draw_ranking(unsigned long long seed, long long epoch, long long molecule, int n, int* rank,
                             unsigned long long* key) {
  const int lane = threadIdx.x & 31;
  const unsigned long long h = mix64(mix64(mix64(seed) ^ (unsigned long long)epoch) ^ (unsigned long long)molecule);
  for (int i = lane; i < n; i += 32) key[i] = mix64(h ^ (unsigned long long)i);
  __syncwarp();
  for (int i = lane; i < n; i += 32) {
    const unsigned long long k = key[i];
    int r = 0;
    for (int j = 0; j < n; ++j) r += key[j] < k || (key[j] == k && j < i);
    rank[i] = r;
  }
  __syncwarp();
}

__global__ void __launch_bounds__(32) rank_draw_kernel(int N, const int* __restrict__ n_atoms, unsigned long long seed,
                                                       long long epoch, long long first, int* rankings) {
  __shared__ int rank[kReorderMaxN];
  __shared__ unsigned long long key[kReorderMaxN];
  const int m = blockIdx.x, lane = threadIdx.x;
  const int n = min(max(n_atoms[m], 0), N);
  draw_ranking(seed, epoch, first + m, n, rank, key);
  for (int i = lane; i < N; i += 32) rankings[(size_t)m * N + i] = i < n ? rank[i] : -1;
}

// molecule m's ranking into rank[0, n) (one warp): drawn from (seed, epoch, first + m) and written to R (-1 past n),
// or read from R.  seen [kReorderWords] must be zero on entry.  False, with GIB_PP_BAD_RANKING raised, when it is not
// a permutation of 0..n-1.
__device__ bool load_ranking(int N, int n, int draw, unsigned long long seed, long long epoch, long long first, int m,
                             int* R, int* rank, unsigned long long* key, unsigned* seen, int* status) {
  const int lane = threadIdx.x & 31;
  if (draw) {
    draw_ranking(seed, epoch, first + m, n, rank, key);
    for (int i = lane; i < N; i += 32) R[i] = i < n ? rank[i] : -1;
  } else {
    for (int i = lane; i < n; i += 32) rank[i] = R[i];
  }
  __syncwarp();
  bool bad_rank = false;
  for (int i = lane; i < n; i += 32) {
    const int r = rank[i];
    if (r < 0 || r >= n || (atomicOr(&seen[r >> 5], 1u << (r & 31)) >> (r & 31) & 1u)) bad_rank = true;
  }
  bad_rank = __any_sync(0xffffffffu, bad_rank);
  if (bad_rank && lane == 0) flag_bad(status, GIB_PP_BAD_RANKING, m);
  return !bad_rank;
}

// reorder_nodes (one warp): the atom at new position k is old atom ord[k] for k < nk; order row O = ord, -1 past nk
// (O may be null), node rows / edge rows and columns of the molecule (X, E) into OX / OE, zero past nk
__device__ void write_reordered(const PP& p, const signed char* X, const signed char* E, const int* ord, int nk,
                                int* O, signed char* OX, signed char* OE) {
  const int lane = threadIdx.x & 31;
  const int N = p.N, F = p.F, Ef = p.Ef;
  if (O)
    for (int i = lane; i < N; i += 32) O[i] = i < nk ? ord[i] : -1;
  for (int q = lane; q < N * F; q += 32) {
    const int k = q / F;
    OX[q] = k < nk ? X[(size_t)ord[k] * F + q % F] : 0;
  }
  for (int q = lane; q < N * N * Ef; q += 32) {
    const int k = q / (N * Ef), l = q / Ef % N, t = q % Ef;
    OE[q] = k < nk && l < nk ? E[((size_t)ord[k] * N + ord[l]) * Ef + t] : 0;
  }
}

// route: 0 = BFS, 1 = DFS.  draw != 0: the ranking is drawn (draw_ranking) and written to `rankings`, else read from it
__global__ void __launch_bounds__(32) reorder_kernel(PP p, const signed char* __restrict__ nodes,
                                                     const signed char* __restrict__ edges, const int* __restrict__ n0,
                                                     int route, int draw, unsigned long long seed, long long epoch,
                                                     long long first, int* rankings, int* order,
                                                     signed char* out_nodes, signed char* out_edges, int* status) {
  __shared__ unsigned adj[kReorderMaxN][kReorderWords];
  __shared__ unsigned seen[kReorderWords];
  __shared__ int rank[kReorderMaxN], ord[kReorderMaxN], pos[kReorderMaxN];
  __shared__ unsigned long long key[kReorderMaxN];
  __shared__ short table[kSetMaxSlots], tmp[kReorderMaxN];
  __shared__ int ok;
  const int m = blockIdx.x, lane = threadIdx.x;
  const int N = p.N, F = p.F, Ef = p.Ef, W = (N + 31) / 32;
  const int n = n0[m];
  const signed char* X = nodes + (size_t)m * N * F;
  const signed char* E = edges + (size_t)m * N * N * Ef;
  int* R = rankings + (size_t)m * N;
  if (lane < W) seen[lane] = 0;
  if (lane == 0) ok = n > 0;
  load_adjacency(E, N, Ef, n, adj, nullptr);
  if (!load_ranking(N, n, draw, seed, epoch, first, m, R, rank, key, seen, status) && lane == 0) ok = 0;
  __syncwarp();
  if (lane == 0 && ok) {
    const int start = rank[0];                              // node_init = atom_ranking[0]
    // connectivity first: both reference searches loop forever on a disconnected graph
    if (reach(adj, W, start) != n) {
      flag_bad(status, GIB_PP_DISCONNECTED, m);
      ok = 0;
    } else {
      unsigned* vis = seen;                                 // reused: the visited set
      for (int w = 0; w < W; ++w) vis[w] = 0;
      vis[start >> 5] |= 1u << (start & 31);
      ord[0] = start;
      pos[start] = 0;
      int count = 1;
      unsigned cand[kReorderWords];
      if (route == 0) {
        // breadth_first_search: per layer, each last-layer atom's unvisited neighbours by falling rank into one set;
        // the set's iteration order is the layer's order (nodes_visited.extend(set(...)), last_nodes_visited = set(...))
        PySet set{table, tmp, 0, 0};
        int lo = 0, hi = 1;
        while (count < n) {
          set.clear();
          for (int k = lo; k < hi; ++k) {
            for (int w = 0; w < W; ++w) cand[w] = adj[ord[k]][w] & ~vis[w];
            for (int a = best_of(cand, rank, W); a >= 0; a = best_of(cand, rank, W)) {
              set.add(a);
              cand[a >> 5] &= ~(1u << (a & 31));
            }
          }
          lo = hi;
          for (int i = 0; i <= set.mask; ++i)
            if (table[i] >= 0) {
              const int a = table[i];
              vis[a >> 5] |= 1u << (a & 31);
              ord[count++] = a;
            }
          hi = count;
        }
      } else {
        // depth_first_search: the highest-ranked unvisited neighbour of the last atom; none -> back to the atom
        // before it in visit order (nodes_visited[idx - 1], index -1 = the last one)
        int last = start;
        while (count < n) {
          for (int w = 0; w < W; ++w) cand[w] = adj[last][w] & ~vis[w];
          const int a = best_of(cand, rank, W);
          if (a < 0) {
            const int idx = pos[last];
            last = ord[idx ? idx - 1 : count - 1];
            continue;
          }
          vis[a >> 5] |= 1u << (a & 31);
          pos[a] = count;
          ord[count++] = a;
          last = a;
        }
      }
    }
  }
  __syncwarp();
  // a refused molecule's outputs are zero
  write_reordered(p, X, E, ord, ok ? n : 0, order + (size_t)m * N, out_nodes + (size_t)m * N * F,
                  out_edges + (size_t)m * N * N * Ef);
}

// ---- scaffold-first decoding order (gib_scaffold_first): one warp per molecule -------------------------------------
// The embedding search is a depth-first search over scaffold atoms 0..k-1 with the candidate sets as bitsets in shared
// memory: depth i's candidates are label(i) (molecule atoms whose node row is scaffold row i, of a degree that fits)
// minus the atoms in use, intersected, for every assigned j < i, with the bond-type-t neighbours of phi(j) when
// scaffold atoms i, j share a type-t bond and with the non-neighbours of phi(j) when they share none.  The lanes
// compute that over the words, lane 0 moves the search; candidates are taken lowest index first, so the first leaf is
// the lexicographically smallest embedding.
constexpr int kMatchAdjWords = 2048;     // Ef * N * ceil(N / 32) words of per-bond-type adjacency

// per scaffold s (one warp each): deg[s, i] = scaffold atom i's bonds (0 past k_s), bonds[s] = its bonds in all
__global__ void __launch_bounds__(32) scaffold_degree_kernel(PP p, gib_scaffolds sc, short* deg, int* bonds) {
  const int s = blockIdx.x, N = p.N, Ef = p.Ef;
  const int k = min(max(sc.n_atoms[s], 0), N);
  const int b = prefix_degrees(sc.edges + (size_t)s * N * N * Ef, N, Ef, k, deg + (size_t)s * N);
  if (threadIdx.x == 0) bonds[s] = b;
}

// lane 0: the layered breadth-first search from ord[0, c) (marked in vis): layer L + 1 is the unvisited neighbours of
// layer L, appended highest-ranked first (best_of).  Returns the atoms reached.
__device__ int layered_bfs(const unsigned (*adj)[kReorderWords], int W, const int* rank, unsigned* vis, int* ord,
                           int c) {
  unsigned next[kReorderWords];
  for (int lo = 0, hi = c; lo < hi; lo = hi, hi = c) {
    for (int w = 0; w < W; ++w) next[w] = 0;
    for (int k = lo; k < hi; ++k)
      for (int w = 0; w < W; ++w) next[w] |= adj[ord[k]][w];
    for (int w = 0; w < W; ++w) {
      next[w] &= ~vis[w];
      vis[w] |= next[w];
    }
    for (int a = best_of(next, rank, W); a >= 0; a = best_of(next, rank, W)) {
      ord[c++] = a;
      next[a >> 5] &= ~(1u << (a & 31));
    }
  }
  return c;
}

struct MatchSmem {
  unsigned adj[kMatchAdjWords];                       // [Ef][N][W]: bit b of (t, a) = a bond of type t between a, b
  unsigned any[kReorderMaxN][kReorderWords];          // a bond of any type
  unsigned label[kReorderMaxN][kReorderWords];        // per scaffold atom: the molecule atoms it may map to
  unsigned cand[kReorderMaxN][kReorderWords];         // the search stack: depth i's untried candidates
  unsigned used[kReorderWords];                       // the atoms phi(0..depth-1)
  short phi[kReorderMaxN], mdeg[kReorderMaxN];
};

// depth i's candidate set into S.cand[i] (phi(0..i-1) assigned)
__device__ void match_candidates(const PP& p, MatchSmem& S, const signed char* SE, int i, int W) {
  const int lane = threadIdx.x & 31, N = p.N, Ef = p.Ef;
  unsigned acc[kReorderWords];
#pragma unroll
  for (int w = 0; w < kReorderWords; ++w) acc[w] = ~0u;
  for (int j = lane; j < i; j += 32) {
    const int t = bond_type(SE, N, Ef, i, j);
    const int a = S.phi[j];
    const unsigned* nb = t >= 0 ? S.adj + ((size_t)t * N + a) * W : S.any[a];
#pragma unroll
    for (int w = 0; w < kReorderWords; ++w)
      if (w < W) acc[w] &= t >= 0 ? nb[w] : ~nb[w];
  }
#pragma unroll
  for (int w = 0; w < kReorderWords; ++w) acc[w] = __reduce_and_sync(0xffffffffu, acc[w]);
  if (lane == 0)
    for (int w = 0; w < W; ++w) S.cand[i][w] = S.label[i][w] & ~S.used[w] & acc[w];
  __syncwarp();
}

// the molecule side of match_scaffold for the graph E of n atoms: S.adj, S.any and S.mdeg.  Returns the degree sum
// (every lane).
__device__ int match_load(const PP& p, MatchSmem& S, const signed char* E, int n) {
  const int lane = threadIdx.x & 31, W = (p.N + 31) / 32;
  const int deg_sum = warp_sum(load_adjacency(E, p.N, p.Ef, n, S.any, S.adj));
  for (int i = lane; i < n; i += 32) {
    int d = 0;
    for (int w = 0; w < W; ++w) d += __popc(S.any[i][w]);
    S.mdeg[i] = (short)d;
  }
  __syncwarp();
  return deg_sum;
}

// the smallest embedding of scaffold s (k atoms) in the molecule (X, E, n atoms) into S.phi: 1 found, 0 none, -1 the
// search would take more than `budget` assignments.  Every lane gets the answer.
__device__ int match_scaffold(const PP& p, MatchSmem& S, const signed char* X, const signed char* E, int n,
                              const gib_scaffolds& sc, const short* sdeg, int s, int k, long long budget) {
  const int lane = threadIdx.x & 31, N = p.N, F = p.F, W = (N + 31) / 32;
  const signed char* SX = sc.nodes + (size_t)s * N * F;
  const signed char* SE = sc.edges + (size_t)s * N * N * p.Ef;
  const unsigned* pm = sc.protect ? sc.protect + (size_t)s * 4 : nullptr;
  const short* sd = sdeg + (size_t)s * N;
  for (int q = lane; q < k * W; q += 32) S.label[q / W][q % W] = 0;
  if (lane < W) S.used[lane] = 0;
  __syncwarp();
  // labels: the node row equals scaffold row i (all F bytes, as scaffold_differs compares it), the degree is at least
  // scaffold atom i's, and exactly its for a protected atom (no bond may leave the image there)
  for (int q = lane; q < k * n; q += 32) {
    const int i = q / n, a = q % n;
    bool eq = S.mdeg[a] == sd[i] || (S.mdeg[a] > sd[i] && !(pm && scaffold_protected(pm, i)));
    for (int f = 0; f < F && eq; ++f) eq = X[(size_t)a * F + f] == SX[(size_t)i * F + f];
    if (eq) atomicOr(&S.label[i][a >> 5], 1u << (a & 31));
  }
  __syncwarp();
  match_candidates(p, S, SE, 0, W);
  long long nodes = 0;
  int d = 0;
  while (true) {
    int a = -1;
    for (int w = 0; w < W && a < 0; ++w)
      if (S.cand[d][w]) a = w * 32 + __ffs(S.cand[d][w]) - 1;
    __syncwarp();
    if (a < 0) {                                            // depth d exhausted: back to depth d - 1
      if (d == 0) return 0;
      --d;
      if (lane == 0) S.used[S.phi[d] >> 5] &= ~(1u << (S.phi[d] & 31));
      __syncwarp();
      continue;
    }
    if (++nodes > budget) return -1;
    if (lane == 0) {
      S.cand[d][a >> 5] &= ~(1u << (a & 31));
      S.phi[d] = (short)a;
      S.used[a >> 5] |= 1u << (a & 31);
    }
    __syncwarp();
    if (d + 1 < k) {
      match_candidates(p, S, SE, ++d, W);
      continue;
    }
    int nnz;
    if (!scaffold_differs(p, X, E, SX, SE, k, S.phi, &nnz)) return 1;
    if (lane == 0) S.used[a >> 5] &= ~(1u << (a & 31));  // a leaf the byte comparison rejects: the next candidate
    __syncwarp();
  }
}

// ids != null: molecule m tries scaffold ids[m] only (-1, or an id outside [0, S): none); null: scaffolds 0..S-1 in
// order until one embeds.  draw / rankings as in reorder_kernel.  bad: pp_count_kernel's per-molecule flags.
__global__ void __launch_bounds__(32) scaffold_first_kernel(
    PP p, const signed char* __restrict__ nodes, const signed char* __restrict__ edges, const int* __restrict__ n0,
    const int* __restrict__ bad, gib_scaffolds sc, const short* __restrict__ sdeg, const int* __restrict__ sbonds,
    const int* __restrict__ ids, int draw, unsigned long long seed, long long epoch, long long first, int* rankings,
    long long budget, int* order, int* out_ids, signed char* out_nodes, signed char* out_edges, int* status) {
  __shared__ MatchSmem S;
  __shared__ int rank[kReorderMaxN], ord[kReorderMaxN];
  __shared__ unsigned long long key[kReorderMaxN];
  __shared__ unsigned seen[kReorderWords];
  __shared__ int ok;
  const int m = blockIdx.x, lane = threadIdx.x;
  const int N = p.N, F = p.F, Ef = p.Ef, W = (N + 31) / 32;
  const int n = n0[m];
  const signed char* X = nodes + (size_t)m * N * F;
  const signed char* E = edges + (size_t)m * N * N * Ef;
  if (lane < W) seen[lane] = 0;
  if (lane == 0) ok = n > 0 && !bad[m];                     // refused by the input checks: left alone, outputs zero
  const int deg_sum = match_load(p, S, E, n);
  if (!load_ranking(N, n, draw, seed, epoch, first, m, rankings + (size_t)m * N, rank, key, seen, status) && lane == 0)
    ok = 0;
  __syncwarp();
  // connectivity first, as gib_reorder checks it: atom 0 must reach every atom
  if (lane == 0 && ok && reach(S.any, W, 0) != n) {
    flag_bad(status, GIB_PP_DISCONNECTED, m);
    ok = 0;
  }
  __syncwarp();
  int sid = -1;
  if (ok) {
    int s0 = 0, s1 = sc.S;
    if (ids) {
      s0 = ids[m];
      s1 = s0 >= 0 && s0 < sc.S ? s0 + 1 : s0;
    }
    for (int s = s0; s < s1; ++s) {
      const int k = sc.n_atoms[s];
      if (k < 1 || k > n || 2 * sbonds[s] > deg_sum) continue;     // cheap rejects before any search
      const int r = match_scaffold(p, S, X, E, n, sc, sdeg, s, k, budget);
      if (r < 0) {
        if (lane == 0) {
          flag_bad(status, GIB_PP_MATCH_BUDGET, m);
          ok = 0;
        }
        __syncwarp();
        break;
      }
      if (r > 0) {
        sid = s;
        break;
      }
    }
  }
  // the order: phi's image, then its layers; the identity without an embedding
  if (lane == 0 && ok) {
    if (sid >= 0) {
      const int k = sc.n_atoms[sid];
      for (int w = 0; w < W; ++w) seen[w] = 0;
      for (int i = 0; i < k; ++i) {
        ord[i] = S.phi[i];
        seen[S.phi[i] >> 5] |= 1u << (S.phi[i] & 31);
      }
      layered_bfs(S.any, W, rank, seen, ord, k);
    } else {
      for (int i = 0; i < n; ++i) ord[i] = i;
    }
  }
  __syncwarp();
  if (lane == 0) out_ids[m] = ok ? sid : -1;
  // a refused molecule's outputs are zero
  write_reordered(p, X, E, ord, ok ? n : 0, order + (size_t)m * N, out_nodes + (size_t)m * N * F,
                  out_edges + (size_t)m * N * N * Ef);
}

// ---- graph identity: the 1-WL hash and the one-pass deduplication of gib_murcko and the molecule set ---------------
// The items of one call are graphs in canonical order (every prefix connected, so the embedding search stays on
// connected partial maps).  rep[i]: the item whose class item i belongs to, kItemNone (no graph, skipped or refused)
// or kItemOpen (to be searched); an item that starts with rep[i] = i (a known table entry) is fixed.
constexpr int kItemNone = -1, kItemOpen = -2;

// item i < K is row i of the known table, item K + m row m of the call's canonical graphs
struct GraphItems {
  const signed char* known_nodes;   // [K, N, F]
  const signed char* known_edges;   // [K, N, N, Ef]
  const signed char* nodes;         // [n, N, F]
  const signed char* edges;
  int K;
  __device__ const signed char* X(const PP& p, int i) const {
    return i < K ? known_nodes + (size_t)i * p.N * p.F : nodes + (size_t)(i - K) * p.N * p.F;
  }
  __device__ const signed char* E(const PP& p, int i) const {
    const size_t eb = (size_t)p.N * p.N * p.Ef;
    return i < K ? known_edges + (size_t)i * eb : edges + (size_t)(i - K) * eb;
  }
};

// one warp: the graph's atom count k (rows up to the last non-zero one), bonds, and its colour-refinement (1-WL) hash
//   c_0(a) = mix64(sum_f byte_hash(f, X[a][f])),
//   c_r(a) = mix64(c_{r-1}(a) + sum over bonds (a, b) of type t of mix64(c_{r-1}(b) ^ (t + 1) << 56)), r = 1..k,
//   hash   = mix64(sum_a mix64(c_k(a)) ^ (k << 32 | bonds))   (kEmpty -> kEmpty - 1),
// the type being the bond's first non-zero edge byte.  Isomorphic graphs hash equal; equal hashes prove nothing.
// adj [kMatchAdjWords] and col [2][kReorderMaxN] are the warp's shared scratch.  Every lane gets the results.
__device__ unsigned long long wl_hash(const PP& p, const signed char* X, const signed char* E, unsigned* adj,
                                      unsigned long long (*col)[kReorderMaxN], int* k_out, int* bonds_out) {
  const int lane = threadIdx.x & 31;
  const int N = p.N, F = p.F, Ef = p.Ef, W = (N + 31) / 32;
  int last = -1;
  for (int r = lane; r < N; r += 32) {
    bool any = false;
    for (int f = 0; f < F; ++f) any |= X[(size_t)r * F + f] != 0;
    if (any) last = r;
  }
  const int k = warp_max(last) + 1;
  const int bonds = warp_sum(load_adjacency(E, N, Ef, k, nullptr, adj)) / 2;
  for (int a = lane; a < k; a += 32) {
    unsigned long long h = 0;
    for (int f = 0; f < F; ++f) h += byte_hash(f, X[(size_t)a * F + f]);
    col[0][a] = mix64(h);
  }
  __syncwarp();
  for (int r = 0; r < k; ++r) {
    const unsigned long long* src = col[r & 1];
    unsigned long long* dst = col[(r + 1) & 1];
    for (int a = lane; a < k; a += 32) {
      unsigned long long s = src[a];
      for (int t = 0; t < Ef; ++t)
        for (int w = 0; w < W; ++w)
          for (unsigned bits = adj[((size_t)t * N + a) * W + w]; bits; bits &= bits - 1)
            s += mix64(src[w * 32 + __ffs(bits) - 1] ^ ((unsigned long long)(t + 1) << 56));
      dst[a] = mix64(s);
    }
    __syncwarp();
  }
  unsigned long long sum = 0;
  for (int a = lane; a < k; a += 32) sum += mix64(col[k & 1][a]);
  sum = warp_sum_u64(sum);
  unsigned long long h = mix64(sum ^ ((unsigned long long)k << 32 | (unsigned)bonds));
  if (h == kEmpty) h = kEmpty - 1;
  *k_out = k;
  *bonds_out = bonds;
  return h;
}

// does graph (RX, RE) of k atoms embed in the graph (X, E) of k atoms whose molecule side match_load put in S?  Between
// graphs of equal atom and bond counts an induced embedding is an isomorphism (the smallest one lands in S.phi).  1 yes,
// 0 no, -1 the search would take more than `budget` nodes; two empty graphs are isomorphic.  Every lane gets the answer.
__device__ int match_graph(const PP& p, MatchSmem& S, short* rdeg, const signed char* X, const signed char* E,
                           const signed char* RX, const signed char* RE, int k, long long budget) {
  if (k == 0) return 1;
  prefix_degrees(RE, p.N, p.Ef, k, rdeg);
  __syncwarp();
  gib_scaffolds view{};
  view.nodes = RX;
  view.edges = RE;
  return match_scaffold(p, S, X, E, k, view, rdeg, 0, k, budget);
}

// Grouping: the items' (hash, index) pairs are radix-sorted by hash (stable: each group in ascending index), and
// first[i] / pos[i] are the sorted positions of item i's group start and of item i itself (one CTA).
__global__ void __launch_bounds__(kGroupNT) group_kernel(int n, const unsigned long long* __restrict__ skey,
                                                         const int* __restrict__ sval, int* first, int* pos) {
  __shared__ int sm[32];
  int carry = 0;
  for (int base = 0; base < n; base += kGroupNT) {
    const int q = base + threadIdx.x;
    const bool head = q < n && (q == 0 || skey[q] != skey[q - 1]);
    int total;
    const int start = max(carry, cta_scan(head ? q : 0, true, sm, &total));
    if (q < n) {
      first[sval[q]] = start;
      pos[sval[q]] = q;
    }
    carry = max(carry, total);
  }
}

// workspace of the radix sort: CUB's temporary storage is sized at call time and checked against this bound
size_t sort_tmp_bytes(long long items) { return align256((1u << 20) + 8ull * items); }

// sorts the pairs (k0[i], v0[i]) by key, stably; *skey / *sval: the buffers holding the sorted pairs
int sort_groups(const char* who, unsigned long long* k0, unsigned long long* k1, int* v0, int* v1, int items,
                void* tmp, size_t tmp_bytes, cudaStream_t s, const unsigned long long** skey, const int** sval) {
  cub::DoubleBuffer<unsigned long long> k(k0, k1);
  cub::DoubleBuffer<int> v(v0, v1);
  size_t need = 0;
  GIB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, need, k, v, items, 0, 64, s));
  if (need > tmp_bytes) {
    set_error("%s: the radix sort of %d items needs %zu bytes of workspace, %zu reserved", who, items, need, tmp_bytes);
    return -1;
  }
  GIB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, need, k, v, items, 0, 64, s));
  *skey = k.Current();
  *sval = v.Current();
  return 0;
}

// The one-pass deduplication, one warp per open item i: its representative is the smallest item j <= i of its hash
// group in its class.  Isomorphism is an equivalence, so that j is the first item of the class and i finds it alone:
// it tests the earlier items of its group in ascending order and stops at the first match (no rounds, no dependency
// between items).  Candidates must have i's atom and bond counts; the test is match_graph (j embedded in i), whose
// smallest isomorphism goes to phi (when given; the identity for a representative).  cls (may be null): an item of
// cls >= 0 is already known to be class cls (a set entry) and matches exactly the earlier items of the same cls; the
// others skip those.  A search beyond `budget` refuses the item (GIB_PP_MATCH_BUDGET, molecule i - K).
__global__ void __launch_bounds__(32) dedup_kernel(PP p, GraphItems it, const int* __restrict__ sval,
                                                   const int* __restrict__ first, const int* __restrict__ pos,
                                                   const int* __restrict__ item_k, const int* __restrict__ item_bonds,
                                                   const int* __restrict__ cls, long long budget, int* rep, short* phi,
                                                   int* status) {
  __shared__ MatchSmem S;
  __shared__ short rdeg[kReorderMaxN];
  const int i = blockIdx.x, lane = threadIdx.x;
  if (rep[i] != kItemOpen) return;                          // from here on rep[i] is written by this warp alone
  const int k = item_k[i], bonds = item_bonds[i], c = cls ? cls[i] : -1;
  const signed char* X = it.X(p, i);
  const signed char* E = it.E(p, i);
  bool loaded = false;
  int res = 0, r = i;
  for (int q = first[i], end = pos[i]; q < end; ++q) {
    const int j = sval[q], cj = cls ? cls[j] : -1;
    if (c >= 0 || cj >= 0) {
      if (cj != c) continue;
      res = 1;
      r = j;
      break;
    }
    if (item_k[j] != k || item_bonds[j] != bonds) continue;
    if (!loaded) {
      match_load(p, S, E, k);
      loaded = true;
    }
    res = match_graph(p, S, rdeg, X, E, it.X(p, j), it.E(p, j), k, budget);
    if (res) {
      r = j;
      break;
    }
  }
  if (res < 0) {
    if (lane == 0) {
      rep[i] = kItemNone;
      flag_bad(status, GIB_PP_MATCH_BUDGET, i - it.K);
    }
    return;
  }
  if (phi) {
    short* ph = phi + (size_t)(i - it.K) * p.N;
    for (int a = lane; a < k; a += 32) ph[a] = r == i ? (short)a : S.phi[a];
  }
  if (lane == 0) rep[i] = r;
}

// is_new[m] = 1 when item K + m represents a class that is not a known entry
__global__ void new_class_kernel(int n, int K, const int* __restrict__ rep, const int* __restrict__ cls, int* is_new) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m < n) is_new[m] = rep[K + m] == K + m && !(cls && cls[K + m] >= 0);
}

// ---- Murcko scaffolds (gib_murcko) ---------------------------------------------------------------------------------
// Items: the known table's entries 0..K-1 (fixed), then the scaffolds of the chunk's molecules K..K+n-1.

// one warp per molecule: keep = the 2-core (atoms of degree <= 1 removed, all at once, until none is left) plus the
// atoms outside it with a double bond (edge feature 1) to it; the scaffold is the molecule's induced subgraph on them,
// written in canonical order (breadth-first from the lowest kept index, each layer in increasing index) with its
// order row (molecule atom per scaffold position, -1 past k).  No ring: nothing kept, k = 0, zero bytes.
__global__ void __launch_bounds__(32) murcko_kernel(PP p, const signed char* __restrict__ nodes,
                                                    const signed char* __restrict__ edges,
                                                    const int* __restrict__ n0, const int* __restrict__ bad,
                                                    unsigned char* keep_out, int* sorder, signed char* sc_nodes,
                                                    signed char* sc_edges, int* status) {
  __shared__ unsigned adj[kReorderMaxN][kReorderWords], dbl[kReorderMaxN][kReorderWords];
  __shared__ unsigned alive[kReorderWords], keep[kReorderWords], vis[kReorderWords];
  __shared__ int rank[kReorderMaxN], ord[kReorderMaxN];
  __shared__ int ok, k;
  const int m = blockIdx.x, lane = threadIdx.x;
  const int N = p.N, F = p.F, Ef = p.Ef, W = (N + 31) / 32;
  const int n = n0[m];
  const signed char* X = nodes + (size_t)m * N * F;
  const signed char* E = edges + (size_t)m * N * N * Ef;
  for (int q = lane; q < N * W; q += 32) dbl[q / W][q % W] = 0;
  for (int i = lane; i < N; i += 32) rank[i] = N - i;      // layered_bfs takes the highest rank first
  if (lane < W) alive[lane] = keep[lane] = 0;
  if (lane == 0) {
    ok = n > 0 && !bad[m];
    k = 0;
  }
  load_adjacency(E, N, Ef, n, adj, nullptr);
  if (Ef > 1)
    for (int q = lane; q < n * n; q += 32) {
      const int i = q / n, j = q % n;
      if (E[((size_t)i * N + j) * Ef + 1]) atomicOr(&dbl[i][j >> 5], 1u << (j & 31));
    }
  for (int a = lane; a < n; a += 32) atomicOr(&alive[a >> 5], 1u << (a & 31));
  __syncwarp();
  if (lane == 0 && ok && reach(adj, W, 0) != n) {          // connectivity, as gib_reorder checks it
    flag_bad(status, GIB_PP_DISCONNECTED, m);
    ok = 0;
  }
  __syncwarp();
  if (ok) {
    // atom w * 32 + lane is bit `lane` of word w: one ballot per word gives the atoms that go
    for (bool again = true; again;) {
      unsigned gone[kReorderWords];
      again = false;
#pragma unroll
      for (int w = 0; w < kReorderWords; ++w) {
        bool go = false;
        const int a = w * 32 + lane;
        if (w < W && a < n && (alive[w] >> lane & 1u)) {
          int d = 0;
          for (int v = 0; v < W; ++v) d += __popc(adj[a][v] & alive[v]);
          go = d <= 1;
        }
        gone[w] = __ballot_sync(0xffffffffu, go);
        again |= gone[w] != 0;
      }
      __syncwarp();
      if (lane == 0) {
#pragma unroll
        for (int w = 0; w < kReorderWords; ++w)
          if (w < W) alive[w] &= ~gone[w];
      }
      __syncwarp();
    }
#pragma unroll
    for (int w = 0; w < kReorderWords; ++w) {
      const int a = w * 32 + lane;
      bool kp = false;
      if (w < W && a < n) {
        kp = alive[w] >> lane & 1u;
        for (int v = 0; v < W && !kp; ++v) kp = (dbl[a][v] & alive[v]) != 0;
      }
      const unsigned kw = __ballot_sync(0xffffffffu, kp);
      if (lane == 0 && w < W) keep[w] = kw;
    }
    __syncwarp();
    if (lane == 0) {
      int start = -1;
      for (int w = 0; w < W && start < 0; ++w)
        if (keep[w]) start = w * 32 + __ffs(keep[w]) - 1;
      if (start >= 0) {
        for (int w = 0; w < W; ++w) vis[w] = ~keep[w];     // only kept atoms are reached
        vis[start >> 5] |= 1u << (start & 31);
        ord[0] = start;
        k = layered_bfs(adj, W, rank, vis, ord, 1);
      }
    }
    __syncwarp();
  }
  for (int a = lane; a < N; a += 32) keep_out[(size_t)m * N + a] = ok && (keep[a >> 5] >> (a & 31) & 1u);
  write_reordered(p, X, E, ord, k, sorder + (size_t)m * N, sc_nodes + (size_t)m * N * F,
                  sc_edges + (size_t)m * N * N * Ef);
}

// one warp per item: its atom count, bonds and sort key (wl_hash; kEmpty without a scaffold, sorted past every group)
__global__ void __launch_bounds__(32) murcko_hash_kernel(PP p, GraphItems it, int* item_k, int* item_bonds,
                                                         unsigned long long* key, int* val, int* rep) {
  __shared__ unsigned adj[kMatchAdjWords];
  __shared__ unsigned long long col[2][kReorderMaxN];
  const int i = blockIdx.x;
  int k, bonds;
  const unsigned long long h = wl_hash(p, it.X(p, i), it.E(p, i), adj, col, &k, &bonds);
  if (threadIdx.x == 0) {
    item_k[i] = k;
    item_bonds[i] = bonds;
    key[i] = k > 0 ? h : kEmpty;
    val[i] = i;
    rep[i] = k == 0 ? kItemNone : i < it.K ? i : kItemOpen;
  }
}

// one warp per molecule: its entry id (a new entry's id is K + its rank among the chunk's new representatives, off),
// the count, a new entry's bytes into the table, and the attachment points: entry atom i is one when the molecule atom
// it maps to (through phi and the scaffold's order row) has a bond to an atom outside the scaffold
__global__ void __launch_bounds__(32) murcko_emit_kernel(PP p, GraphItems it, const signed char* __restrict__ edges,
                                                         const int* __restrict__ n0,
                                                         const unsigned char* __restrict__ keep,
                                                         const int* __restrict__ sorder, const int* __restrict__ rep,
                                                         const int* __restrict__ off, const short* __restrict__ phi,
                                                         const int* __restrict__ item_k, int* ids,
                                                         signed char* table_nodes, signed char* table_edges,
                                                         unsigned long long* counts, unsigned char* attach) {
  const int m = blockIdx.x, lane = threadIdx.x, K = it.K;
  const int N = p.N, F = p.F, Ef = p.Ef;
  const int r = rep[K + m];
  const int id = r < 0 ? -1 : r < K ? r : K + off[r - K];
  if (lane == 0) {
    ids[m] = id;
    if (id >= 0) atomicAdd(&counts[id], 1ull);
  }
  if (id < 0) return;
  if (r == K + m) {
    const signed char* X = it.X(p, r);
    const signed char* E = it.E(p, r);
    for (int q = lane; q < N * F; q += 32) table_nodes[(size_t)id * N * F + q] = X[q];
    for (int q = lane; q < N * N * Ef; q += 32) table_edges[(size_t)id * N * N * Ef + q] = E[q];
  }
  const int k = item_k[K + m], n = n0[m];
  const signed char* E = edges + (size_t)m * N * N * Ef;
  const unsigned char* kp = keep + (size_t)m * N;
  const int* o = sorder + (size_t)m * N;
  const short* ph = phi + (size_t)m * N;
  for (int q = lane; q < k * n; q += 32) {
    const int i = q / n, b = q % n, a = o[ph[i]];
    if (!kp[b] && has_bond(E, N, Ef, a, b)) attach[(size_t)id * N + i] = 1;
  }
}

struct MurckoWs {
  size_t len, n0, bad, off, sorder, phi, sc_nodes, sc_edges, item_k, item_bonds, rep, key0, key1, val0, val1, first,
      pos, sort_tmp, total;
};

MurckoWs murcko_ws_layout(const PP& p, int n, int K) {
  MurckoWs w{};
  const long long items = (long long)n + K;
  Carve c;
  w.len = c.take(4ull * n);
  w.n0 = c.take(4ull * n);
  w.bad = c.take(4ull * n);
  w.off = c.take(4ull * (n + 1));
  w.sorder = c.take(4ull * n * p.N);
  w.phi = c.take(2ull * n * p.N);
  w.sc_nodes = c.take((size_t)n * p.N * p.F);
  w.sc_edges = c.take((size_t)n * p.N * p.N * p.Ef);
  w.item_k = c.take(4ull * items);
  w.item_bonds = c.take(4ull * items);
  w.rep = c.take(4ull * items);
  w.key0 = c.take(8ull * items);
  w.key1 = c.take(8ull * items);
  w.val0 = c.take(4ull * items);
  w.val1 = c.take(4ull * items);
  w.first = c.take(4ull * items);
  w.pos = c.take(4ull * items);
  w.sort_tmp = c.take(sort_tmp_bytes(items));
  w.total = c.end;
  return w;
}

// the shared-memory shapes of match_scaffold (MatchSmem), for gib_scaffold_first and gib_murcko
int match_limits(const char* who, const PP& p) {
  if (p.N > kReorderMaxN || (long long)p.Ef * p.N * ((p.N + 31) / 32) > kMatchAdjWords) {
    set_error("%s: need N <= %d and Ef * N * ceil(N / 32) <= %d, got N=%d Ef=%d", who, kReorderMaxN, kMatchAdjWords,
              p.N, p.Ef);
    return -1;
  }
  return 0;
}

int murcko_limits(const char* who, const gib_pp_dims* d, int n_molecules, int n_known, PP* p) {
  GIB_TRY(make_pp(who, d, p));
  GIB_TRY(match_limits(who, *p));
  if (n_molecules < 1 || n_known < 0 || (long long)n_molecules + n_known > INT_MAX / 4) {
    set_error("%s: need n_molecules >= 1, n_known >= 0 and n_molecules + n_known <= %d, got %d and %d", who,
              INT_MAX / 4, n_molecules, n_known);
    return -1;
  }
  return 0;
}

// ---- the molecule set (gib_molset_*): a persistent table of distinct molecules -------------------------------------
// Items of a call: its n molecules, in canonical order in the workspace.  cls[i]: the set entry molecule i is (-1: none).

// one warp per molecule: skipped (valid[m] == 0) or refused -> kItemNone; else the input checks (gib_preprocess_chunk's,
// an empty graph allowed), connectivity, the canonical order (breadth-first from atom 0, each layer in increasing
// index) into (CX, CE), and the item's atom count, bonds and hash (copied to its sort key)
__global__ void __launch_bounds__(32) molset_prepare_kernel(PP p, const signed char* __restrict__ nodes,
                                                            const signed char* __restrict__ edges,
                                                            const unsigned char* __restrict__ valid, signed char* CX,
                                                            signed char* CE, int* item_k, int* item_bonds,
                                                            unsigned long long* hash, unsigned long long* key,
                                                            int* val, int* rep, int* status) {
  __shared__ unsigned any[kReorderMaxN][kReorderWords];
  __shared__ unsigned typed[kMatchAdjWords];
  __shared__ unsigned long long col[2][kReorderMaxN];
  __shared__ int rank[kReorderMaxN], ord[kReorderMaxN];
  __shared__ unsigned vis[kReorderWords];
  __shared__ int bad_s;
  const int m = blockIdx.x, lane = threadIdx.x;
  const int N = p.N, F = p.F, Ef = p.Ef, W = (N + 31) / 32;
  const signed char* X = nodes + (size_t)m * N * F;
  const signed char* E = edges + (size_t)m * N * N * Ef;
  const bool use = !valid || valid[m];
  int n = 0, nnz, bad = 0;
  if (use) {
    bad = validate_graph(p, X, E, &n, &nnz) & ~GIB_PP_EMPTY;
    if (!bad && n > 0) {
      load_adjacency(E, N, Ef, n, any, nullptr);
      for (int i = lane; i < N; i += 32) rank[i] = N - i;   // layered_bfs takes the highest rank first
      if (lane < W) vis[lane] = 0;
      __syncwarp();
      if (lane == 0) {
        bad_s = 0;
        if (reach(any, W, 0) != n) {
          bad_s = GIB_PP_DISCONNECTED;
        } else {
          vis[0] = 1u;
          ord[0] = 0;
          layered_bfs(any, W, rank, vis, ord, 1);
        }
      }
      __syncwarp();
      bad = bad_s;
    }
  }
  const bool ok = use && !bad;
  write_reordered(p, X, E, ord, ok ? n : 0, nullptr, CX + (size_t)m * N * F, CE + (size_t)m * N * N * Ef);
  int k = 0, bonds = 0;
  const unsigned long long h = ok ? wl_hash(p, X, E, typed, col, &k, &bonds) : kEmpty;
  if (lane == 0) {
    if (bad) flag_bad(status, bad, m);
    item_k[m] = k;
    item_bonds[m] = bonds;
    hash[m] = key[m] = h;
    val[m] = m;
    rep[m] = ok ? kItemOpen : kItemNone;
  }
}

// the index slot of hash h (-1: not in the set)
__device__ __forceinline__ long long molset_slot(const gib_molset& set, unsigned long long h) {
  const long long mask = (long long)set.slots - 1;
  for (long long s = (long long)(h & (unsigned long long)mask);; s = (s + 1) & mask) {
    const unsigned long long k = set.index_keys[s];
    if (k == h) return s;
    if (k == kEmpty) return -1;
  }
}

// one warp per open item: the set entry it is (cls[i], -1: none), found along its hash's chain; entries are distinct,
// so at most one matches.  A search beyond `budget` refuses the molecule.
__global__ void __launch_bounds__(32) molset_lookup_kernel(PP p, gib_molset set, GraphItems it,
                                                           const int* __restrict__ item_k,
                                                           const int* __restrict__ item_bonds,
                                                           const unsigned long long* __restrict__ hash, int* rep,
                                                           long long budget, int* cls, int* status) {
  __shared__ MatchSmem S;
  __shared__ short rdeg[kReorderMaxN];
  const int i = blockIdx.x, lane = threadIdx.x, N = p.N, F = p.F, Ef = p.Ef;
  int found = -1, res = 0;
  if (rep[i] == kItemOpen) {
    const long long s = molset_slot(set, hash[i]);
    const int k = item_k[i], bonds = item_bonds[i];
    bool loaded = false;
    for (int e = s < 0 ? -1 : set.index_first[s]; e >= 0; e = set.next[e]) {
      if (set.n_atoms[e] != k || set.n_bonds[e] != bonds) continue;
      if (!loaded) {
        match_load(p, S, it.E(p, i), k);
        loaded = true;
      }
      res = match_graph(p, S, rdeg, it.X(p, i), it.E(p, i), set.nodes + (size_t)e * N * F,
                        set.edges + (size_t)e * N * N * Ef, k, budget);
      if (res) {
        found = res > 0 ? e : -1;
        break;
      }
    }
  }
  if (lane == 0) {
    cls[i] = found;
    if (res < 0) {
      rep[i] = kItemNone;
      flag_bad(status, GIB_PP_MATCH_BUDGET, i);
    }
  }
}

// one thread, after the scan: refuses an insert that does not fit (GIB_PP_CAPACITY), records the entry count before
// the call in status and, when the call inserts, the count after it in the set
__global__ void molset_commit_kernel(gib_molset set, int insert, int* status) {
  const int S = *set.size;
  status[kStSetSize] = S;
  if (!insert || status[kStFlags]) return;
  if ((long long)S + status[kStTotal] > set.capacity) {
    atomicOr(&status[kStFlags], GIB_PP_CAPACITY);           // the molecule is named by molset_emit_kernel
    return;
  }
  *set.size = S + status[kStTotal];
}

// one warp per molecule: ids and flags; when the call inserts, counts and the new entries (canonical bytes, hash, atom
// and bond counts, the end of a chain).  A refused call writes none of the set: ids -1 and no flags, and under
// GIB_PP_CAPACITY the first molecule of the first class that does not fit is named.
__global__ void __launch_bounds__(32) molset_emit_kernel(PP p, gib_molset set, GraphItems it,
                                                         const int* __restrict__ item_k,
                                                         const int* __restrict__ item_bonds,
                                                         const unsigned long long* __restrict__ hash,
                                                         const int* __restrict__ rep, const int* __restrict__ cls,
                                                         const int* __restrict__ off, int insert, int* ids,
                                                         unsigned char* is_new, unsigned char* is_first, int* status) {
  const int i = blockIdx.x, lane = threadIdx.x, N = p.N, F = p.F, Ef = p.Ef;
  const int flags = status[kStFlags], S = status[kStSetSize], r = rep[i];
  const bool found = r >= 0 && cls[i] >= 0;
  const int id = r < 0 ? -1 : found ? cls[i] : S + off[r];
  if (flags) {
    if (lane == 0) {
      ids[i] = -1;
      is_new[i] = is_first[i] = 0;
      if (flags == GIB_PP_CAPACITY && r == i && !found && id == set.capacity) atomicMin(&status[kStFirstBad], i);
    }
    return;
  }
  if (lane == 0) {
    ids[i] = found || insert ? id : -1;
    is_new[i] = r >= 0 && !found;
    is_first[i] = r == i;
    if (insert && id >= 0) atomicAdd((unsigned long long*)&set.counts[id], 1ull);
  }
  if (!insert || found || r != i) return;
  const signed char* X = it.X(p, i);
  const signed char* E = it.E(p, i);
  for (int q = lane; q < N * F; q += 32) set.nodes[(size_t)id * N * F + q] = X[q];
  for (int q = lane; q < N * N * Ef; q += 32) set.edges[(size_t)id * N * N * Ef + q] = E[q];
  if (lane == 0) {
    set.hash[id] = hash[i];
    set.n_atoms[id] = item_k[i];
    set.n_bonds[id] = item_bonds[i];
    set.next[id] = -1;
  }
}

// one CTA, after molset_emit_kernel of an inserting call: links the new entries into the index.  Within a hash group
// (sorted positions, ascending item index) the new entries follow each other in id order; the first one of a hash
// either takes an empty index slot or is appended to the end of the chain already there.
__global__ void __launch_bounds__(kGroupNT) molset_link_kernel(gib_molset set, int n,
                                                               const unsigned long long* __restrict__ skey,
                                                               const int* __restrict__ sval,
                                                               const int* __restrict__ first,
                                                               const int* __restrict__ rep,
                                                               const int* __restrict__ cls,
                                                               const int* __restrict__ off,
                                                               const int* __restrict__ status) {
  __shared__ int sm[32], incl[kGroupNT];
  if (status[kStFlags]) return;
  const int S = status[kStSetSize];
  const long long mask = (long long)set.slots - 1;
  int carry = -1;
  for (int base = 0; base < n; base += kGroupNT) {
    const int q = base + threadIdx.x;
    const int j = q < n ? sval[q] : -1;
    const bool fresh = j >= 0 && rep[j] == j && cls[j] < 0;
    int total;
    const int inc = max(carry, cta_scan(fresh ? q : -1, true, sm, &total));
    incl[threadIdx.x] = inc;
    __syncthreads();
    const int prev = threadIdx.x ? incl[threadIdx.x - 1] : carry;    // the last new entry before position q
    if (fresh) {
      const int id = S + off[j];
      if (prev >= first[j]) {
        set.next[S + off[sval[prev]]] = id;
      } else {
        const unsigned long long h = skey[q];
        for (long long s = (long long)(h & (unsigned long long)mask);; s = (s + 1) & mask) {
          const unsigned long long k = atomicCAS(&set.index_keys[s], kEmpty, h);
          if (k == kEmpty) {
            set.index_first[s] = id;
            break;
          }
          if (k == h) {
            int e = set.index_first[s];
            while (set.next[e] >= 0) e = set.next[e];
            set.next[e] = id;
            break;
          }
        }
      }
    }
    carry = max(carry, total);
    __syncthreads();
  }
}

struct MolsetWs {
  size_t cx, ce, item_k, item_bonds, hash, rep, cls, is_new, off, key0, key1, val0, val1, first, pos, sort_tmp, total;
};

MolsetWs molset_ws_layout(const PP& p, int n) {
  MolsetWs w{};
  Carve c;
  w.cx = c.take((size_t)n * p.N * p.F);
  w.ce = c.take((size_t)n * p.N * p.N * p.Ef);
  w.item_k = c.take(4ull * n);
  w.item_bonds = c.take(4ull * n);
  w.hash = c.take(8ull * n);
  w.rep = c.take(4ull * n);
  w.cls = c.take(4ull * n);
  w.is_new = c.take(4ull * n);
  w.off = c.take(4ull * (n + 1));
  w.key0 = c.take(8ull * n);
  w.key1 = c.take(8ull * n);
  w.val0 = c.take(4ull * n);
  w.val1 = c.take(4ull * n);
  w.first = c.take(4ull * n);
  w.pos = c.take(4ull * n);
  w.sort_tmp = c.take(sort_tmp_bytes(n));
  w.total = c.end;
  return w;
}

// the index slots of a set of `capacity` entries: the smallest power of two >= 2 * capacity (0: capacity out of range)
long long molset_slots(int capacity) {
  if (capacity < 1 || capacity > (1 << 29)) return 0;
  long long s = 1;
  while (s < 2ll * capacity) s <<= 1;
  return s;
}

int molset_limits(const char* who, const gib_pp_dims* d, PP* p) {
  GIB_TRY(make_pp(who, d, p));
  return match_limits(who, *p);
}

int check_molset(const char* who, const gib_molset* set) {
  if (!set || !set->nodes || !set->edges || !set->hash || !set->n_atoms || !set->n_bonds || !set->counts ||
      !set->next || !set->index_keys || !set->index_first || !set->size) {
    set_error("%s: null set or set buffer", who);
    return -1;
  }
  if (set->slots != molset_slots(set->capacity)) {
    set_error("%s: a set of capacity %d needs %lld index slots, got %d", who, set->capacity,
              molset_slots(set->capacity), set->slots);
    return -1;
  }
  return 0;
}

__global__ void molset_from_float_kernel(const float* __restrict__ x, signed char* out, long long count) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < count; q += (long long)gridDim.x * blockDim.x) {
    const float v = x[q];
    out[q] = v == 0.f ? 0 : v == 1.f ? 1 : 2;
  }
}

// gib_reorder's workspace: the count stage's len and n0 [n]
struct ReorderWs {
  size_t len, n0, total;
};

ReorderWs reorder_ws_layout(int n) {
  ReorderWs w{};
  Carve c;
  w.len = c.take(4ull * n);
  w.n0 = c.take(4ull * n);
  w.total = c.end;
  return w;
}

// gib_scaffold_first's workspace: the count stage's len, n0 and bad [n], the scaffold degrees short [S, N] and bonds [S]
struct ScaffoldFirstWs {
  size_t len, n0, bad, sdeg, sbonds, total;
};

ScaffoldFirstWs scaffold_first_ws_layout(const PP& p, int n, int S) {
  ScaffoldFirstWs w{};
  Carve c;
  w.len = c.take(4ull * n);
  w.n0 = c.take(4ull * n);
  w.bad = c.take(4ull * n);
  w.sdeg = c.take(2ull * S * p.N);
  w.sbonds = c.take(4ull * S);
  w.total = c.end;
  return w;
}

// the status words reset, then pp_count_kernel's validation of n molecules: len, n0 and, when bad != null, each
// molecule's GIB_PP_* flags
int launch_count(const PP& p, const signed char* nodes, const signed char* edges, int n, int* len, int* n0, int* bad,
                 int* status, cudaStream_t s) {
  pp_init_kernel<<<1, 32, 0, s>>>(status, nullptr, nullptr, 0, 0);
  GIB_LAUNCH_CHECK();
  pp_count_kernel<<<n, 32, 0, s>>>(p, nodes, edges, len, n0, status, nullptr, gib_scaffolds{}, bad);
  GIB_LAUNCH_CHECK();
  return 0;
}

}  // namespace
}  // namespace gib

using namespace gib;

extern "C" {

int gib_preprocess_apd_length(const gib_pp_dims* d) {
  PP p;
  GIB_TRY(make_pp("gib_preprocess_apd_length", d, &p));
  return p.apd_len;
}

size_t gib_preprocess_ws_bytes(const gib_pp_dims* d, int max_molecules, int max_rows) {
  PP p;
  if (make_pp("gib_preprocess_ws_bytes", d, &p)) return 0;
  if (max_molecules < 1 || max_rows < p.B) {
    set_error("gib_preprocess_ws_bytes: need max_molecules >= 1 and max_rows >= batch_size (%d), got %d and %d",
              p.B, max_molecules, max_rows);
    return 0;
  }
  if ((long long)max_molecules * p.s_max >= INT_MAX / 2) {
    set_error("gib_preprocess_ws_bytes: max_molecules * (N*(N-1)/2 + 2) = %lld states exceeds %d",
              (long long)max_molecules * p.s_max, INT_MAX / 2);
    return 0;
  }
  return ws_layout(p, max_molecules, max_rows).total;
}

int gib_preprocess_chunk(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int n_molecules,
                         int last_chunk, int max_molecules, int max_rows, void* ws, signed char* out_nodes,
                         signed char* out_edges, int* out_apds, int* groups, int* status, gib_stream stream) {
  PP p;
  GIB_TRY(make_pp("gib_preprocess_chunk", d, &p));
  if (!gib_preprocess_ws_bytes(d, max_molecules, max_rows)) return -1;
  if (n_molecules < 1 || n_molecules > max_molecules) {
    set_error("gib_preprocess_chunk: n_molecules %d outside [1, max_molecules = %d]", n_molecules, max_molecules);
    return -1;
  }
  if (!nodes || !edges || !ws || !out_nodes || !out_edges || !out_apds || !groups || !status) {
    set_error("gib_preprocess_chunk: null argument");
    return -1;
  }
  const WsLayout w = ws_layout(p, max_molecules, max_rows);
  char* b = static_cast<char*>(ws);
  int* len = (int*)(b + w.len);
  int* n0 = (int*)(b + w.n0);
  int* off = (int*)(b + w.off);
  short* rs = (short*)(b + w.rs);
  unsigned long long* hash = (unsigned long long*)(b + w.hash);
  int* apd = (int*)(b + w.apd);
  int* nn = (int*)(b + w.nn);
  int* mol = (int*)(b + w.mol);
  unsigned long long* keys = (unsigned long long*)(b + w.keys);
  int* vals = (int*)(b + w.vals);
  cudaStream_t s = (cudaStream_t)stream;
  const int init_blocks = (int)(w.table / 256 < 1024 ? w.table / 256 : 1024);
  pp_init_kernel<<<init_blocks, 256, 0, s>>>(status, keys, vals, w.table, 0);
  GIB_LAUNCH_CHECK();
  GIB_TRY(launch_route(p, nodes, edges, n_molecules, RouteBufs{len, n0, off, rs, hash, apd, nn, mol}, status, s));
  const StateRef S{off, nn, mol, rs, nodes, edges};
  pp_group_kernel<<<1, kGroupNT, 0, s>>>(p, S, n_molecules, last_chunk, max_rows, hash, keys, vals, w.table - 1,
                                         (int*)(b + w.slot), (int*)(b + w.row_of), (int*)(b + w.dst),
                                         (int*)(b + w.own), (int*)(b + w.row_state), groups, status);
  GIB_LAUNCH_CHECK();
  pp_emit_kernel<<<min(max_rows, 4096), kEmitNT, 0, s>>>(p, S, (const int*)(b + w.row_state), status, out_nodes,
                                                         out_edges, out_apds);
  GIB_LAUNCH_CHECK();
  pp_scatter_kernel<<<1024, 256, 0, s>>>(p, off, apd, (const int*)(b + w.dst), (const int*)(b + w.own), status,
                                         out_apds);
  GIB_LAUNCH_CHECK();
  return 0;
}

size_t gib_route_plan_ws_bytes(const gib_pp_dims* d, int max_molecules) {
  PP p;
  if (route_limits("gib_route_plan_ws_bytes", d, max_molecules, &p)) return 0;
  return route_ws_layout(p, max_molecules).total;
}

long long gib_route_max_states(const gib_pp_dims* d, int max_molecules) {
  PP p;
  GIB_TRY(route_limits("gib_route_max_states", d, max_molecules, &p));
  return (long long)max_molecules * p.s_max;
}

int gib_route_plan(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int n_molecules,
                   int max_molecules, void* ws, int* offsets, int* status, gib_stream stream) {
  return route_plan("gib_route_plan", d, nodes, edges, n_molecules, max_molecules, false, nullptr, nullptr, ws, offsets,
                    status, stream);
}

int gib_test_route_plan_offsets(const gib_pp_dims* d, int max_molecules, long long* out) {
  PP p;
  GIB_TRY(route_limits("gib_test_route_plan_offsets", d, max_molecules, &p));
  if (!out) {
    set_error("gib_test_route_plan_offsets: null out");
    return -1;
  }
  const RouteWs w = route_ws_layout(p, max_molecules);
  out[0] = (long long)w.hash;
  out[1] = (long long)w.apd;
  out[2] = (long long)w.nn;
  out[3] = (long long)w.mol;
  return 0;
}

int gib_route_fill(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int max_molecules,
                   const void* ws, const int* offsets, const int* status, gib_batch_ctl* ctl, int* slots,
                   signed char* out_nodes, signed char* out_edges, gib_stream stream) {
  return route_fill("gib_route_fill", d, nodes, edges, max_molecules, ws, offsets, status, false, nullptr, ctl, slots,
                    nullptr, nullptr, out_nodes, out_edges, stream);
}

int gib_route_plan_scaffold(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int n_molecules,
                            int max_molecules, const gib_scaffolds* sc, const int* scaffold_ids, void* ws,
                            int* offsets, int* status, gib_stream stream) {
  return route_plan("gib_route_plan_scaffold", d, nodes, edges, n_molecules, max_molecules, true, sc, scaffold_ids, ws,
                    offsets, status, stream);
}

int gib_route_fill_scaffold(const gib_pp_dims* d, const signed char* nodes, const signed char* edges,
                            int max_molecules, const void* ws, const int* offsets, const int* status,
                            const int* scaffold_ids, gib_batch_ctl* ctl, int* slots, int* slot_ids, int* slot_n,
                            signed char* out_nodes, signed char* out_edges, gib_stream stream) {
  return route_fill("gib_route_fill_scaffold", d, nodes, edges, max_molecules, ws, offsets, status, true, scaffold_ids,
                    ctl, slots, slot_ids, slot_n, out_nodes, out_edges, stream);
}

int gib_route_check_actions(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int n_molecules,
                            int max_molecules, const void* ws, const int* offsets, int mode, const int* table,
                            int* result, gib_stream stream) {
  PP p;
  GIB_TRY(route_limits("gib_route_check_actions", d, max_molecules, &p));
  if (n_molecules < 1 || n_molecules > max_molecules || p.N > 127 || !nodes || !edges || !ws || !offsets ||
      !result || (mode != GIB_ACTION_MASK_STRUCTURE && mode != GIB_ACTION_MASK_VALENCE) ||
      (mode == GIB_ACTION_MASK_VALENCE && !table)) {
    set_error("gib_route_check_actions: bad arguments (n_molecules=%d max_molecules=%d N=%d mode=%d; N <= 127, the "
              "buffers must be given, the valence mode needs the table)", n_molecules, max_molecules, p.N, mode);
    return -1;
  }
  const ActionLayout L{p.N, d->n_atom_types, d->n_formal_charge, d->n_imp_H, d->n_chirality, p.Ef};
  const RouteWs w = route_ws_layout(p, max_molecules);
  const char* b = static_cast<const char*>(ws);
  cudaStream_t s = (cudaStream_t)stream;
  GIB_CUDA_TRY(cudaMemsetAsync(result, 0, sizeof(int), s));
  GIB_CUDA_TRY(cudaMemsetAsync(result + 1, 0x7f, sizeof(int), s));     // 0x7f7f7f7f: no molecule yet
  route_action_check_kernel<<<n_molecules, 32, 0, s>>>(L, p.F, offsets, (const int*)(b + w.apd),
                                                       (const int*)(b + w.nn), nodes, edges,
                                                       mode == GIB_ACTION_MASK_VALENCE, table, result);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gib_route_reduce(int n_molecules, const int* offsets, const float* likelihoods, float* nll, float* final_,
                     gib_stream stream) {
  if (n_molecules < 1 || !offsets || !likelihoods || !nll || !final_) {
    set_error("gib_route_reduce: need n_molecules >= 1 and every pointer, got n_molecules = %d", n_molecules);
    return -1;
  }
  route_reduce_kernel<<<ceil_div(n_molecules, 128), 128, 0, (cudaStream_t)stream>>>(n_molecules, offsets,
                                                                                    likelihoods, nll, final_);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gib_route_grad_coef(int n_molecules, const int* offsets, const float* likelihoods, const float* g_lik,
                        const float* g_nll, const float* g_final, float* coef, gib_stream stream) {
  if (n_molecules < 1 || !offsets || !likelihoods || !coef) {
    set_error("gib_route_grad_coef: need n_molecules >= 1, offsets, likelihoods and coef, got n_molecules = %d",
              n_molecules);
    return -1;
  }
  route_grad_coef_kernel<<<ceil_div(n_molecules, kCoefWarps), 32 * kCoefWarps, 0, (cudaStream_t)stream>>>(
      n_molecules, offsets, likelihoods, g_lik, g_nll, g_final, coef);
  GIB_LAUNCH_CHECK();
  return 0;
}

size_t gib_reorder_ws_bytes(int n_molecules) { return n_molecules < 1 ? 0 : reorder_ws_layout(n_molecules).total; }

int gib_draw_rankings(int n_molecules, int N, const int* n_atoms, unsigned long long seed, long long epoch,
                      long long first_molecule, int* rankings, gib_stream stream) {
  if (n_molecules < 1 || N < 1 || N > kReorderMaxN || first_molecule < 0 || !n_atoms || !rankings) {
    set_error("gib_draw_rankings: need n_molecules >= 1, 1 <= N <= %d, first_molecule >= 0 and non-null buffers "
              "(got %d, %d, %lld)", kReorderMaxN, n_molecules, N, first_molecule);
    return -1;
  }
  rank_draw_kernel<<<n_molecules, 32, 0, (cudaStream_t)stream>>>(N, n_atoms, seed, epoch, first_molecule, rankings);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gib_reorder(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int n_molecules, int route,
                int draw, unsigned long long seed, long long epoch, long long first_molecule, int* rankings,
                int* order, signed char* out_nodes, signed char* out_edges, void* ws, int* status, gib_stream stream) {
  PP p;
  GIB_TRY(make_pp("gib_reorder", d, &p));
  if (n_molecules < 1 || (route != GIB_ROUTE_BFS && route != GIB_ROUTE_DFS) || first_molecule < 0) {
    set_error("gib_reorder: need n_molecules >= 1, route GIB_ROUTE_BFS or GIB_ROUTE_DFS and first_molecule >= 0 "
              "(got %d, %d, %lld)", n_molecules, route, first_molecule);
    return -1;
  }
  if (!nodes || !edges || !rankings || !order || !out_nodes || !out_edges || !ws || !status) {
    set_error("gib_reorder: null argument");
    return -1;
  }
  const ReorderWs w = reorder_ws_layout(n_molecules);
  char* b = static_cast<char*>(ws);
  int* n0 = (int*)(b + w.n0);
  cudaStream_t s = (cudaStream_t)stream;
  GIB_TRY(launch_count(p, nodes, edges, n_molecules, (int*)(b + w.len), n0, nullptr, status, s));
  reorder_kernel<<<n_molecules, 32, 0, s>>>(p, nodes, edges, n0, route, draw, seed, epoch, first_molecule, rankings,
                                            order, out_nodes, out_edges, status);
  GIB_LAUNCH_CHECK();
  return 0;
}

size_t gib_scaffold_first_ws_bytes(const gib_pp_dims* d, int n_molecules, int n_scaffolds) {
  PP p;
  if (make_pp("gib_scaffold_first_ws_bytes", d, &p)) return 0;
  if (n_molecules < 1 || n_scaffolds < 1) {
    set_error("gib_scaffold_first_ws_bytes: need n_molecules >= 1 and n_scaffolds >= 1, got %d and %d", n_molecules,
              n_scaffolds);
    return 0;
  }
  return scaffold_first_ws_layout(p, n_molecules, n_scaffolds).total;
}

int gib_scaffold_first(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int n_molecules,
                       const gib_scaffolds* sc, const int* scaffold_ids, int draw, unsigned long long seed,
                       long long epoch, long long first_molecule, int* rankings, long long budget, int* order,
                       int* ids, signed char* out_nodes, signed char* out_edges, void* ws, int* status,
                       gib_stream stream) {
  PP p;
  GIB_TRY(make_pp("gib_scaffold_first", d, &p));
  GIB_TRY(match_limits("gib_scaffold_first", p));
  if (n_molecules < 1 || first_molecule < 0 || budget < 1) {
    set_error("gib_scaffold_first: need n_molecules >= 1, first_molecule >= 0 and budget >= 1 (got %d, %lld, %lld)",
              n_molecules, first_molecule, budget);
    return -1;
  }
  if (!nodes || !edges || !rankings || !order || !ids || !out_nodes || !out_edges || !ws || !status) {
    set_error("gib_scaffold_first: null argument");
    return -1;
  }
  GIB_TRY(check_scaffolds("gib_scaffold_first", sc, p));
  const ScaffoldFirstWs w = scaffold_first_ws_layout(p, n_molecules, sc->S);
  char* b = static_cast<char*>(ws);
  int* n0 = (int*)(b + w.n0);
  int* bad = (int*)(b + w.bad);
  short* sdeg = (short*)(b + w.sdeg);
  int* sbonds = (int*)(b + w.sbonds);
  cudaStream_t s = (cudaStream_t)stream;
  GIB_TRY(launch_count(p, nodes, edges, n_molecules, (int*)(b + w.len), n0, bad, status, s));
  scaffold_degree_kernel<<<sc->S, 32, 0, s>>>(p, *sc, sdeg, sbonds);
  GIB_LAUNCH_CHECK();
  scaffold_first_kernel<<<n_molecules, 32, 0, s>>>(p, nodes, edges, n0, bad, *sc, sdeg, sbonds, scaffold_ids, draw,
                                                   seed, epoch, first_molecule, rankings, budget, order, ids,
                                                   out_nodes, out_edges, status);
  GIB_LAUNCH_CHECK();
  return 0;
}

size_t gib_murcko_ws_bytes(const gib_pp_dims* d, int n_molecules, int n_known) {
  PP p;
  if (murcko_limits("gib_murcko_ws_bytes", d, n_molecules, n_known, &p)) return 0;
  return murcko_ws_layout(p, n_molecules, n_known).total;
}

int gib_murcko(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int n_molecules, int n_known,
               signed char* table_nodes, signed char* table_edges, long long* counts, unsigned char* attachment,
               long long budget, unsigned char* keep, int* ids, void* ws, int* status, gib_stream stream) {
  PP p;
  GIB_TRY(murcko_limits("gib_murcko", d, n_molecules, n_known, &p));
  if (budget < 1) {
    set_error("gib_murcko: need budget >= 1, got %lld", budget);
    return -1;
  }
  if (!nodes || !edges || !table_nodes || !table_edges || !counts || !attachment || !keep || !ids || !ws || !status) {
    set_error("gib_murcko: null argument");
    return -1;
  }
  const MurckoWs w = murcko_ws_layout(p, n_molecules, n_known);
  char* b = static_cast<char*>(ws);
  int* len = (int*)(b + w.len);
  int* n0 = (int*)(b + w.n0);
  int* bad = (int*)(b + w.bad);
  int* off = (int*)(b + w.off);
  int* sorder = (int*)(b + w.sorder);
  short* phi = (short*)(b + w.phi);
  int* item_k = (int*)(b + w.item_k);
  int* item_bonds = (int*)(b + w.item_bonds);
  int* rep = (int*)(b + w.rep);
  int* first = (int*)(b + w.first);
  int* pos = (int*)(b + w.pos);
  const GraphItems it{table_nodes, table_edges, (const signed char*)(b + w.sc_nodes),
                      (const signed char*)(b + w.sc_edges), n_known};
  const int n = n_molecules, items = n + n_known;
  cudaStream_t s = (cudaStream_t)stream;
  GIB_TRY(launch_count(p, nodes, edges, n, len, n0, bad, status, s));
  murcko_kernel<<<n, 32, 0, s>>>(p, nodes, edges, n0, bad, keep, sorder, (signed char*)(b + w.sc_nodes),
                                 (signed char*)(b + w.sc_edges), status);
  GIB_LAUNCH_CHECK();
  murcko_hash_kernel<<<items, 32, 0, s>>>(p, it, item_k, item_bonds, (unsigned long long*)(b + w.key0),
                                          (int*)(b + w.val0), rep);
  GIB_LAUNCH_CHECK();
  const unsigned long long* skey;
  const int* sval;
  GIB_TRY(sort_groups("gib_murcko", (unsigned long long*)(b + w.key0), (unsigned long long*)(b + w.key1),
                      (int*)(b + w.val0), (int*)(b + w.val1), items, b + w.sort_tmp, sort_tmp_bytes(items), s,
                      &skey, &sval));
  group_kernel<<<1, kGroupNT, 0, s>>>(items, skey, sval, first, pos);
  GIB_LAUNCH_CHECK();
  dedup_kernel<<<items, 32, 0, s>>>(p, it, sval, first, pos, item_k, item_bonds, nullptr, budget, rep, phi, status);
  GIB_LAUNCH_CHECK();
  new_class_kernel<<<ceil_div(n, 256), 256, 0, s>>>(n, n_known, rep, nullptr, len);
  GIB_LAUNCH_CHECK();
  pp_scan_kernel<<<1, 1024, 0, s>>>(n, len, off, status);
  GIB_LAUNCH_CHECK();
  murcko_emit_kernel<<<n, 32, 0, s>>>(p, it, edges, n0, keep, sorder, rep, off, phi, item_k, ids, table_nodes,
                                      table_edges, (unsigned long long*)counts, attachment);
  GIB_LAUNCH_CHECK();
  return 0;
}

size_t gib_molset_bytes(const gib_pp_dims* d, int capacity) {
  PP p;
  if (molset_limits("gib_molset_bytes", d, &p)) return 0;
  const long long slots = molset_slots(capacity);
  if (!slots) {
    set_error("gib_molset_bytes: capacity %d outside [1, 2^29]", capacity);
    return 0;
  }
  // per entry: node and edge bytes, hash, atom and bond counts, count, next; per slot: key and first entry; the size
  const size_t entry = (size_t)p.N * p.F + (size_t)p.N * p.N * p.Ef + 8 + 4 + 4 + 8 + 4;
  return entry * capacity + 12ull * slots + 4;
}

int gib_molset_slots(int capacity) {
  const long long slots = molset_slots(capacity);
  if (!slots) {
    set_error("gib_molset_slots: capacity %d outside [1, 2^29]", capacity);
    return -1;
  }
  return (int)slots;
}

int gib_molset_init(const gib_molset* set, gib_stream stream) {
  GIB_TRY(check_molset("gib_molset_init", set));
  cudaStream_t s = (cudaStream_t)stream;
  GIB_CUDA_TRY(cudaMemsetAsync(set->index_keys, 0xff, 8ull * set->slots, s));      // kEmpty
  GIB_CUDA_TRY(cudaMemsetAsync(set->counts, 0, 8ull * set->capacity, s));
  GIB_CUDA_TRY(cudaMemsetAsync(set->size, 0, sizeof(int), s));
  return 0;
}

size_t gib_molset_ws_bytes(const gib_pp_dims* d, int n_molecules) {
  PP p;
  if (molset_limits("gib_molset_ws_bytes", d, &p)) return 0;
  if (n_molecules < 1 || n_molecules > INT_MAX / 4) {
    set_error("gib_molset_ws_bytes: n_molecules %d outside [1, %d]", n_molecules, INT_MAX / 4);
    return 0;
  }
  return molset_ws_layout(p, n_molecules).total;
}

int gib_molset_identify(const gib_pp_dims* d, const gib_molset* set, const signed char* nodes,
                        const signed char* edges, const unsigned char* valid, int n_molecules, int insert,
                        long long budget, int* ids, unsigned char* is_new, unsigned char* is_first, void* ws,
                        int* status, gib_stream stream) {
  PP p;
  GIB_TRY(molset_limits("gib_molset_identify", d, &p));
  GIB_TRY(check_molset("gib_molset_identify", set));
  if (n_molecules < 1 || n_molecules > INT_MAX / 4 || budget < 1 || (insert != 0 && insert != 1)) {
    set_error("gib_molset_identify: need 1 <= n_molecules <= %d, budget >= 1 and insert 0 or 1 (got %d, %lld, %d)",
              INT_MAX / 4, n_molecules, budget, insert);
    return -1;
  }
  if (!nodes || !edges || !ids || !is_new || !is_first || !ws || !status) {
    set_error("gib_molset_identify: null argument");
    return -1;
  }
  const int n = n_molecules;
  const MolsetWs w = molset_ws_layout(p, n);
  char* b = static_cast<char*>(ws);
  signed char* cx = (signed char*)(b + w.cx);
  signed char* ce = (signed char*)(b + w.ce);
  int* item_k = (int*)(b + w.item_k);
  int* item_bonds = (int*)(b + w.item_bonds);
  int* rep = (int*)(b + w.rep);
  int* cls = (int*)(b + w.cls);
  int* fresh = (int*)(b + w.is_new);
  int* off = (int*)(b + w.off);
  int* first = (int*)(b + w.first);
  int* pos = (int*)(b + w.pos);
  unsigned long long* hash = (unsigned long long*)(b + w.hash);
  unsigned long long* key = (unsigned long long*)(b + w.key0);
  const GraphItems it{nullptr, nullptr, cx, ce, 0};
  cudaStream_t s = (cudaStream_t)stream;
  pp_init_kernel<<<1, 32, 0, s>>>(status, nullptr, nullptr, 0, 0);
  GIB_LAUNCH_CHECK();
  molset_prepare_kernel<<<n, 32, 0, s>>>(p, nodes, edges, valid, cx, ce, item_k, item_bonds, hash, key,
                                         (int*)(b + w.val0), rep, status);
  GIB_LAUNCH_CHECK();
  molset_lookup_kernel<<<n, 32, 0, s>>>(p, *set, it, item_k, item_bonds, hash, rep, budget, cls, status);
  GIB_LAUNCH_CHECK();
  const unsigned long long* skey;
  const int* sval;
  GIB_TRY(sort_groups("gib_molset_identify", key, (unsigned long long*)(b + w.key1), (int*)(b + w.val0),
                      (int*)(b + w.val1), n, b + w.sort_tmp, sort_tmp_bytes(n), s, &skey, &sval));
  group_kernel<<<1, kGroupNT, 0, s>>>(n, skey, sval, first, pos);
  GIB_LAUNCH_CHECK();
  dedup_kernel<<<n, 32, 0, s>>>(p, it, sval, first, pos, item_k, item_bonds, cls, budget, rep, nullptr, status);
  GIB_LAUNCH_CHECK();
  new_class_kernel<<<ceil_div(n, 256), 256, 0, s>>>(n, 0, rep, cls, fresh);
  GIB_LAUNCH_CHECK();
  pp_scan_kernel<<<1, 1024, 0, s>>>(n, fresh, off, status);
  GIB_LAUNCH_CHECK();
  molset_commit_kernel<<<1, 1, 0, s>>>(*set, insert, status);
  GIB_LAUNCH_CHECK();
  molset_emit_kernel<<<n, 32, 0, s>>>(p, *set, it, item_k, item_bonds, hash, rep, cls, off, insert, ids, is_new,
                                      is_first, status);
  GIB_LAUNCH_CHECK();
  if (insert) {
    molset_link_kernel<<<1, kGroupNT, 0, s>>>(*set, n, skey, sval, first, rep, cls, off, status);
    GIB_LAUNCH_CHECK();
  }
  return 0;
}

int gib_molset_from_float(const float* x, signed char* out, long long count, gib_stream stream) {
  if (count < 0 || (count && (!x || !out))) {
    set_error("gib_molset_from_float: need count >= 0 and both buffers, got count = %lld", count);
    return -1;
  }
  if (!count) return 0;
  const int blocks = (int)std::min<long long>(ceil_div_ll(count, 256), 4096);
  molset_from_float_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, out, count);
  GIB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"

