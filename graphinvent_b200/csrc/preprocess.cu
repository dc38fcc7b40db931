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

#include "common.cuh"
#include "../../include/gib200.h"

namespace gib {

namespace {

constexpr int kGroupNT = 1024;
constexpr int kEmitNT = 128;
constexpr int kMaxNodeBytes = 8192;
constexpr unsigned long long kEmpty = ~0ull;

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

WsLayout ws_layout(const PP& p, int max_mols, int max_rows) {
  WsLayout w{};
  w.states = (long long)max_mols * p.s_max;
  const long long window = (long long)(max_mols < p.B ? max_mols : p.B) * p.s_max;
  w.table = 1024;
  while (w.table < 2 * window) w.table <<= 1;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = align256(o + bytes); return r; };
  w.len = take(4ull * max_mols);
  w.n0 = take(4ull * max_mols);
  w.off = take(4ull * (max_mols + 1));
  w.rs = take(2ull * max_mols * p.N * p.N);
  w.hash = take(8ull * w.states);
  w.apd = take(4ull * w.states);
  w.nn = take(4ull * w.states);
  w.mol = take(4ull * w.states);
  w.slot = take(4ull * w.states);
  w.row_of = take(4ull * w.states);
  w.dst = take(4ull * w.states);
  w.own = take(4ull * w.states);
  w.row_state = take(4ull * max_rows);
  w.keys = take(8ull * w.table);
  w.vals = take(4ull * w.table);
  w.total = o;
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

__device__ __forceinline__ void flag_bad(int* status, int flags, int m) {
  atomicOr(&status[3], flags);
  atomicMin(&status[4], m);
}

__global__ void pp_init_kernel(int* status, unsigned long long* keys, int* vals, long long table) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    status[0] = status[1] = status[2] = status[3] = status[5] = status[6] = status[7] = 0;
    status[4] = INT_MAX;
  }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < table; i += (long long)gridDim.x * blockDim.x) {
    keys[i] = kEmpty;
    vals[i] = INT_MAX;
  }
}

// ---- count: validation and route length (one warp per molecule) ------------------------------------------------
__global__ void __launch_bounds__(32) pp_count_kernel(PP p, const signed char* __restrict__ nodes,
                                                      const signed char* __restrict__ edges, int* len, int* n0,
                                                      int* status) {
  const int m = blockIdx.x, lane = threadIdx.x;
  const int N = p.N, F = p.F, Ef = p.Ef;
  const signed char* X = nodes + (size_t)m * N * F;
  const signed char* E = edges + (size_t)m * N * N * Ef;
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
  if (lane == 0) {
    if (bad) flag_bad(status, bad, m);
    const int e = nnz / 2;
    len[m] = bad ? 2 : min(e, p.s_max - 2) + 2;
    n0[m] = n;
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
    status[5] = carry;
  }
}

// ---- route: one warp per molecule ------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) pp_route_kernel(PP p, const signed char* __restrict__ nodes,
                                                      const signed char* __restrict__ edges, const int* off,
                                                      const int* n0, unsigned long long* hash, int* apd, int* nn,
                                                      int* mol, short* rs_all, int* status) {
  extern __shared__ __align__(16) unsigned char smem[];
  if (status[3]) return;
  const int m = blockIdx.x, lane = threadIdx.x;
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
  if (status[3]) {
    __syncthreads();
    if (tid == 0) status[0] = status[1] = status[2] = 0;
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
    status[0] = ng;
    status[1] = s;
    status[2] = rows_used;
  }
}

// ---- emit: one CTA per row ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(kEmitNT) pp_emit_kernel(PP p, StateRef S, const int* row_state, const int* status,
                                                          signed char* out_nodes, signed char* out_edges,
                                                          int* out_apds) {
  const int rows = status[2];
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
  const int n = off[status[1]];
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

int launch_route(const PP& p, const signed char* nodes, const signed char* edges, int n, const RouteBufs& r,
                 int* status, cudaStream_t s) {
  pp_count_kernel<<<n, 32, 0, s>>>(p, nodes, edges, r.len, r.n0, status);
  GIB_LAUNCH_CHECK();
  pp_scan_kernel<<<1, 1024, 0, s>>>(n, r.len, r.off, status);
  GIB_LAUNCH_CHECK();
  const size_t smem = 4 * (size_t)p.N + (size_t)p.N * p.F + (size_t)p.N * p.N * p.Ef;
  pp_route_kernel<<<n, 32, smem, s>>>(p, nodes, edges, r.off, r.n0, r.hash, r.apd, r.nn, r.mol, r.rs, status);
  GIB_LAUNCH_CHECK();
  return 0;
}

// ---- the route scorer (graphinvent_b200.graphed.RouteScorer): its plan workspace, the fill of one batch of route
// states into the model's static int8 inputs, the per-molecule reduction ----------------------------------------
constexpr int kFillNT = 256;
constexpr int kFillMaxBlocks = 4096;
constexpr int kCursor = 6;      // status word: replays of the chunk done so far (the fill's batch index)

struct RouteWs {
  size_t len, n0, rs, hash, apd, nn, mol, total;
};

RouteWs route_ws_layout(const PP& p, int max_mols) {
  RouteWs w{};
  const long long states = (long long)max_mols * p.s_max;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = align256(o + bytes); return r; };
  w.len = take(4ull * max_mols);
  w.n0 = take(4ull * max_mols);
  w.rs = take(2ull * max_mols * p.N * p.N);
  w.hash = take(8ull * states);
  w.apd = take(4ull * states);
  w.nn = take(4ull * states);
  w.mol = take(4ull * states);
  w.total = o;
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
// its place in the likelihood buffer (build order: the molecule's empty graph first), -1 / -1 past the last state
__global__ void __launch_bounds__(kFillNT) route_fill_kernel(PP p, FillSrc f, const int* __restrict__ status,
                                                             gib_batch_ctl* ctl, int* __restrict__ slots,
                                                             signed char* __restrict__ out_nodes,
                                                             signed char* __restrict__ out_edges,
                                                             long long node_chunks, long long edge_chunks) {
  const int B = p.B, S = status[5], s0 = status[kCursor] * B;
  const long long tid = (long long)blockIdx.x * kFillNT + threadIdx.x, stride = (long long)gridDim.x * kFillNT;
  if (tid == 0) ctl->live = max(0, min(B, S - s0));
  for (long long b = tid; b < B; b += stride) {
    const int i = s0 + (int)b;
    int a = -1, d = -1;
    if (i < S) {
      const int m = f.mol[i];
      a = f.apd[i];
      d = f.off[m] + f.off[m + 1] - 1 - i;
    }
    slots[b] = a;
    slots[B + b] = d;
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
  pp_init_kernel<<<init_blocks, 256, 0, s>>>(status, keys, vals, w.table);
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
  PP p;
  GIB_TRY(route_limits("gib_route_plan", d, max_molecules, &p));
  if (n_molecules < 1 || n_molecules > max_molecules) {
    set_error("gib_route_plan: n_molecules %d outside [1, max_molecules = %d]", n_molecules, max_molecules);
    return -1;
  }
  if (!nodes || !edges || !ws || !offsets || !status) {
    set_error("gib_route_plan: null argument");
    return -1;
  }
  const RouteWs w = route_ws_layout(p, max_molecules);
  char* b = static_cast<char*>(ws);
  cudaStream_t s = (cudaStream_t)stream;
  pp_init_kernel<<<1, 32, 0, s>>>(status, nullptr, nullptr, 0);
  GIB_LAUNCH_CHECK();
  return launch_route(p, nodes, edges, n_molecules,
                      RouteBufs{(int*)(b + w.len), (int*)(b + w.n0), offsets, (short*)(b + w.rs),
                                (unsigned long long*)(b + w.hash), (int*)(b + w.apd), (int*)(b + w.nn),
                                (int*)(b + w.mol)},
                      status, s);
}

int gib_route_fill(const gib_pp_dims* d, const signed char* nodes, const signed char* edges, int max_molecules,
                   const void* ws, const int* offsets, const int* status, gib_batch_ctl* ctl, int* slots,
                   signed char* out_nodes, signed char* out_edges, gib_stream stream) {
  PP p;
  GIB_TRY(route_limits("gib_route_fill", d, max_molecules, &p));
  if (!nodes || !edges || !ws || !offsets || !status || !ctl || !slots || !out_nodes || !out_edges) {
    set_error("gib_route_fill: null argument");
    return -1;
  }
  if (!aligned16(nodes) || !aligned16(edges) || !aligned16(out_nodes) || !aligned16(out_edges)) {
    set_error("gib_route_fill: nodes, edges, out_nodes and out_edges must be 16-byte aligned");
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
  route_fill_kernel<<<blocks, kFillNT, 0, (cudaStream_t)stream>>>(p, f, status, ctl, slots, out_nodes, out_edges, nc,
                                                                  ec);
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

}  // extern "C"
