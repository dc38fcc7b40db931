// The generator's action rule (include/gib200.h, gib_action_mask_logits), shared by the round's decode kernel, which
// flags a sampled action invalid, and the action mask, which gives the same actions logit -inf before the sampler
// (both in generate.cu).  One predicate for both, so that "valid actions only" sampling removes exactly the actions
// the state machine would reject.  With n atoms in the state and the flat APD index decoded as in generate.cu:
//   structure (the reference's get_invalid_actions, GraphGenerator.py:573-657, quirks included):
//     - an add is forbidden when n >= N, when n > 0 and bond_to >= n, when n == 0 and bond_to != 0, and when the
//       layout's element 5 (bond_from in L0, bond type in L1 / L2, chirality in L3) is >= N;
//     - a connect is forbidden when n == 0, bond_to >= n, bond_to == n - 1 (a self loop), or when the bond-type
//       entries of the pair (bond_to, n - 1) sum to exactly 1 (the bond exists);
//     - terminate never is;
//   valence (optional), in half-bond units so that aromatic bonds stay exact: order(e) = 2 / 4 / 6 / 3 for single /
//   double / triple / aromatic, used(i) = sum_j sum_e order(e) * edges[i, j, e] + 2 * h_i (h_i: atom i's implicit-H
//   count, implicit-H layouts only), limit(i) = 2 * V[type_i, charge_i]:
//     - an add into a non-empty graph is forbidden when used(bond_to) + order(e) > limit(bond_to) or when the new atom
//       would start over its own limit, order(e) + 2 * h_new > 2 * V[t, c]; the first add into an empty graph has no
//       bond, so only 2 * h_new > 2 * V[t, c] forbids it;
//     - a connect is forbidden when either endpoint, bond_to or n - 1, would exceed its limit.
#pragma once
#include <cuda_runtime.h>

namespace gib {

enum : int { ACT_ADD = 0, ACT_CONN = 1, ACT_TERM = 2 };

// the action layout: H / C = implicit-H / chirality index counts, 0 = segment absent
struct ActionLayout { int N, A, CH, H, C, Ef; };

struct Action { int kind, bond_to, atom, charge, imp_h, chir, btype; };

__host__ __device__ __forceinline__ int layout_len_add(const ActionLayout& L) {
  return L.N * L.A * L.CH * (L.H > 0 ? L.H : 1) * (L.C > 0 ? L.C : 1) * L.Ef;
}

// flat APD index a in [0, apd) -> its fields: f_add[bond_to, atom, charge, (imp_h,) (chirality,) bond_type] |
// f_conn[bond_to, bond_type] | terminate
__device__ __forceinline__ Action decode_action(int a, const ActionLayout& L) {
  Action x{ACT_TERM, 0, 0, 0, 0, 0, 0};
  const int len_add = layout_len_add(L);
  if (a < len_add) {
    x.kind = ACT_ADD;
    int r = a;
    x.btype = r % L.Ef;
    r /= L.Ef;
    if (L.C) { x.chir = r % L.C; r /= L.C; }
    if (L.H) { x.imp_h = r % L.H; r /= L.H; }
    x.charge = r % L.CH;
    r /= L.CH;
    x.atom = r % L.A;
    x.bond_to = r / L.A;
  } else if (a < len_add + L.N * L.Ef) {
    x.kind = ACT_CONN;
    const int c = a - len_add;
    x.btype = c % L.Ef;
    x.bond_to = c / L.Ef;
  }
  return x;
}

// which field is element 5 of the reference's add tuple (f_add_idc[5]): 0 = bond_from (L0), 1 = bond type (L1, L2),
// 2 = chirality (L3)
__host__ __device__ __forceinline__ int layout_e5_sel(const ActionLayout& L) {
  return (L.H == 0 && L.C == 0) ? 0 : (L.H && L.C) ? 2 : 1;
}

__device__ __forceinline__ int add_e5(const Action& x, const ActionLayout& L, int n) {
  const int sel = layout_e5_sel(L);
  return sel == 0 ? n : sel == 2 ? x.chir : x.btype;
}

// sum of the bond-type entries of the pair (bond_to, n - 1) in one slot's edges [N, N, Ef] (n - 1 = -1 wraps to the
// last atom, as Python indexing does)
template <typename T>
__device__ __forceinline__ float pair_sum(const T* __restrict__ e, int N, int Ef, int bond_to, int n) {
  const int bf = n - 1 < 0 ? n - 1 + N : n - 1;
  const T* p = e + ((size_t)bond_to * N + bf) * Ef;
  float s = 0.f;
  for (int t = 0; t < Ef; ++t) s += (float)p[t];
  return s;
}

// the structural rule; `psum` = pair_sum(...) of a connect (not read for other kinds)
__device__ __forceinline__ bool structure_forbidden(const Action& x, const ActionLayout& L, int n, float psum) {
  if (x.kind == ACT_ADD)
    return n >= L.N || (n > 0 && x.bond_to >= n) || (n == 0 && x.bond_to != 0) || add_e5(x, L, n) >= L.N;
  if (x.kind == ACT_CONN) return n == 0 || x.bond_to >= n || x.bond_to == n - 1 || psum == 1.f;
  return false;
}

// the valence inputs of one state: used(i) and limit(i) of its atoms (half-bond units), and the rule table
struct Valence {
  const int* used;        // [n]
  const int* limit;       // [n]
  const int* V;           // [A * CH] max valence per (atom type, charge)
  const int* order;       // [Ef] bond orders in half-bond units
  const int* imp_h;       // [H] implicit-H count of each index (H > 0)
};

// index of the first non-zero entry of one one-hot segment (0 when there is none)
template <typename T>
__device__ __forceinline__ int first_set(const T* __restrict__ p, int len) {
  for (int k = 0; k < len; ++k)
    if (p[k] != T(0)) return k;
  return 0;
}

// (used(i), limit(i)) of atom i, from its node row nr [F] and edge row er [N, Ef]
template <typename T>
__device__ __forceinline__ int2 atom_usage(const T* __restrict__ nr, const T* __restrict__ er, const ActionLayout& L,
                                           const int* V, const int* order, const int* imp_h) {
  const int t = first_set(nr, L.A), c = first_set(nr + L.A, L.CH);
  int u = L.H ? 2 * imp_h[first_set(nr + L.A + L.CH, L.H)] : 0;
  for (int j = 0; j < L.N * L.Ef; ++j) u += order[j % L.Ef] * (int)er[j];
  return make_int2(u, 2 * V[t * L.CH + c]);
}

// the valence rule of an action the structural rule allows
__device__ __forceinline__ bool valence_forbidden(const Action& x, const ActionLayout& L, int n, const Valence& v) {
  if (x.kind == ACT_ADD) {
    const int own = 2 * (L.H ? v.imp_h[x.imp_h] : 0), lim = 2 * v.V[x.atom * L.CH + x.charge];
    if (n == 0) return own > lim;
    const int o = v.order[x.btype];
    return o + own > lim || v.used[x.bond_to] + o > v.limit[x.bond_to];
  }
  if (x.kind == ACT_CONN) {
    const int o = v.order[x.btype], j = n - 1;
    return v.used[x.bond_to] + o > v.limit[x.bond_to] || v.used[j] + o > v.limit[j];
  }
  return false;
}

// the whole rule for flat APD index a in a state of n atoms (0 <= n <= N) with edges e [N, N, Ef]; valence = false:
// the structural part only (v is not read)
template <typename T>
__device__ __forceinline__ bool action_forbidden(int a, const ActionLayout& L, int n, const T* __restrict__ e,
                                                 bool valence, const Valence& v) {
  const Action x = decode_action(a, L);
  const float psum = (x.kind == ACT_CONN && n > 0 && x.bond_to < n) ? pair_sum(e, L.N, L.Ef, x.bond_to, n) : 0.f;
  if (structure_forbidden(x, L, n, psum)) return true;
  return valence && valence_forbidden(x, L, n, v);
}

}  // namespace gib
