// The generator's constraint rule (include/gib200.h, gib_constraints_set): what a molecule may contain, as a mask on
// the actions.  One predicate shared by the constrained action mask (gib_action_mask_logits_constrained) and the
// molecule check (gib_constraints_check), both in generate.cu.  For a state of n atoms the rule reads
//   count_t   atoms of type t, count_c atoms of formal-charge index c (the node rows 0..n-1);
//   bonds_e   entries of bond type e in the upper triangle of the edges (i < j < n);
//   rank      the cycle rank sum_e bonds_e - n + 1 for n >= 1 (0 for the empty graph): every connect raises it by one,
//             an add keeps it, so it counts the rings the route has closed;
//   dist(i)   the shortest-path distance from n - 1 to atom i in the current graph (BFS).
// and forbids (a field at its "off" value forbids nothing; a table with every field off masks nothing):
//   max_atoms      every add when n >= max_atoms;
//   max_type[t]    an add of atom type t when count_t >= max_type[t];
//   max_charge[c]  an add with charge index c when count_c >= max_charge[c];
//   max_bond[e]    an add into a non-empty graph (the first add has no bond) or a connect of bond type e when
//                  bonds_e >= max_bond[e];
//   max_rings      a connect when rank >= max_rings;
//   min_ring_size  a connect from n - 1 to bond_to when dist(bond_to) + 1 < min_ring_size: the smallest ring the new
//                  bond closes is dist + 1 atoms long;
//   minima         terminate while n < min_atoms, count_t < min_type[t] for some t, or rank < min_rings -- but only
//                  when some other action survives every rule of the same launch (structure, valence when on, the
//                  attachment points, these maxima).  Otherwise terminate stays allowed (a dead end) and the molecule
//                  ends under its minimum: every row keeps an action of non-zero probability.
//
// Why the maxima and the ring-size bound are properties of the finished molecule, whatever route built it (so that
// gib_constraints_check, and the route scorer through it, can judge a molecule without its route):
//   - counts, bonds_e and rank only grow along a route, by one per action that the matching maximum forbids at the
//     bound.  A route is allowed by max X exactly when its final value is <= X: if it ends at K <= X every step
//     started below K, and if it ends above X some step started at X.
//   - min_ring_size m is "girth >= m" of the final graph.  Every ring a connect closes is a cycle of the final graph,
//     so a girth >= m graph was never refused.  Conversely take a shortest cycle C of the final graph and the last of
//     its bonds to be placed.  That bond is a connect (an add bonds a new atom of degree 1, which lies on no cycle
//     yet), and when it was placed the rest of C was already there, so it closed a ring of at most |C| atoms: a girth
//     < m graph took a refused connect.  The same argument holds for any order of the bonds, which is how the check
//     finds the girth: for each bond (u, v), the distance from u to v without that bond, plus one.
//   - the minima concern only the final terminate: the molecule is under a minimum or not, and the dead-end rule
//     decides whether its terminate had probability 0.
// A maximum ring size has no such property ("the smallest ring a connect closes <= U" depends on the route: building
// naphthalene's outer ring first closes a 10-ring), so there is none.
#pragma once
#include <cuda_runtime.h>
#include "action_mask.cuh"

namespace gib {

// the table's header words (include/gib200.h GIB_CONS_*); the per-index arrays follow: min_type [A], max_type [A],
// max_charge [CH], max_bond [Ef]
enum : int {
  CONS_MIN_ATOMS = 0, CONS_MAX_ATOMS = 1, CONS_MIN_RINGS = 2, CONS_MAX_RINGS = 3, CONS_MIN_RING_SIZE = 4,
  CONS_HDR = 8
};
constexpr int CONS_FAR = 1 << 20;          // dist of an atom the BFS did not reach

// one state's summary, per CTA in shared memory (N <= 127, counts <= 255: one atom per thread of a 128-thread CTA)
struct ConsState {
  int type_cnt[256], charge_cnt[256], bond_cnt[256];
  unsigned int adj[128][4];                // bit j of adj[i] = atoms i and j are bonded
  int dist[128];
  unsigned int frontier[4];
  int n, rank, below;
};

struct ConsTable {
  const int* t;
  int A, CH;
  __device__ __forceinline__ int min_type(int i) const { return t[CONS_HDR + i]; }
  __device__ __forceinline__ int max_type(int i) const { return t[CONS_HDR + A + i]; }
  __device__ __forceinline__ int max_charge(int c) const { return t[CONS_HDR + 2 * A + c]; }
  __device__ __forceinline__ int max_bond(int e) const { return t[CONS_HDR + 2 * A + CH + e]; }
};

// BFS distances from `src` into s.dist, for `levels` levels (atoms further away keep CONS_FAR); skip >= 0: the bond
// (src, skip) is left out (skip is not reached in the first level).  All 128 threads call it.
__device__ __forceinline__ void cons_bfs(ConsState& s, int src, int skip, int levels) {
  const int i = threadIdx.x, n = s.n;
  __syncthreads();                         // the previous distances may still be read
  if (i < 128) s.dist[i] = i == src ? 0 : CONS_FAR;
  for (int lvl = 0; lvl < levels; ++lvl) {
    const unsigned int ball = __ballot_sync(0xffffffffu, i < n && s.dist[i] == lvl);
    if ((i & 31) == 0) s.frontier[i >> 5] = ball;
    __syncthreads();
    const unsigned int f0 = s.frontier[0], f1 = s.frontier[1], f2 = s.frontier[2], f3 = s.frontier[3];
    if ((f0 | f1 | f2 | f3) == 0) break;   // uniform: every thread read the same words
    if (i < n && s.dist[i] == CONS_FAR && !(lvl == 0 && i == skip) &&
        ((s.adj[i][0] & f0) | (s.adj[i][1] & f1) | (s.adj[i][2] & f2) | (s.adj[i][3] & f3)))
      s.dist[i] = lvl + 1;
    __syncthreads();
  }
  __syncthreads();
}

// the summary of one state of n atoms: node rows nb [N, F], edges e [N, N, Ef]; bfs: dist from n - 1 as far as
// min_ring_size needs.  All 128 threads call it; s is ready when it returns.
template <typename T>
__device__ __forceinline__ void cons_load(ConsState& s, const ConsTable& ct, const ActionLayout& L, int F,
                                          const T* __restrict__ nb, const T* __restrict__ e, int n) {
  const int N = L.N, Ef = L.Ef, i = threadIdx.x;
  for (int k = i; k < 256; k += 128) { s.type_cnt[k] = 0; s.charge_cnt[k] = 0; s.bond_cnt[k] = 0; }
  __syncthreads();
  unsigned int row[4] = {0u, 0u, 0u, 0u};
  if (i < n) {
    const T* nr = nb + (size_t)i * F;
    atomicAdd(&s.type_cnt[first_set(nr, L.A)], 1);
    atomicAdd(&s.charge_cnt[first_set(nr + L.A, L.CH)], 1);
    const T* er = e + (size_t)i * N * Ef;
    for (int j = 0; j < n; ++j) {
      bool any = false;
      for (int t = 0; t < Ef; ++t) {
        if (er[(size_t)j * Ef + t] == T(0)) continue;
        any = true;
        if (j > i) atomicAdd(&s.bond_cnt[t], 1);
      }
      if (any) row[j >> 5] |= 1u << (j & 31);
    }
  }
  if (i < 128)
    for (int w = 0; w < 4; ++w) s.adj[i][w] = row[w];
  __syncthreads();
  if (i == 0) {
    int bonds = 0;
    for (int t = 0; t < Ef; ++t) bonds += s.bond_cnt[t];
    const int rank = n >= 1 ? bonds - n + 1 : 0;
    bool below = n < ct.t[CONS_MIN_ATOMS] || rank < ct.t[CONS_MIN_RINGS];
    for (int t = 0; t < L.A && !below; ++t) below = s.type_cnt[t] < ct.min_type(t);
    s.n = n;
    s.rank = rank;
    s.below = below;
  }
  __syncthreads();
  const int m = ct.t[CONS_MIN_RING_SIZE];
  if (m > 0 && n >= 1) cons_bfs(s, n - 1, -1, min(m - 2, n));
}

// the maxima and the ring-size bound for decoded action x in the state s
__device__ __forceinline__ bool cons_forbidden(const Action& x, const ConsState& s, const ConsTable& ct) {
  const int n = s.n;
  if (x.kind == ACT_ADD) {
    const int ma = ct.t[CONS_MAX_ATOMS], mt = ct.max_type(x.atom), mc = ct.max_charge(x.charge);
    if ((ma >= 0 && n >= ma) || (mt >= 0 && s.type_cnt[x.atom] >= mt) || (mc >= 0 && s.charge_cnt[x.charge] >= mc))
      return true;
    const int mb = ct.max_bond(x.btype);
    return n > 0 && mb >= 0 && s.bond_cnt[x.btype] >= mb;
  }
  if (x.kind == ACT_CONN) {
    const int mb = ct.max_bond(x.btype), mr = ct.t[CONS_MAX_RINGS], m = ct.t[CONS_MIN_RING_SIZE];
    if ((mb >= 0 && s.bond_cnt[x.btype] >= mb) || (mr >= 0 && s.rank >= mr)) return true;
    return m > 0 && x.bond_to < n && s.dist[x.bond_to] + 1 < m;
  }
  return false;
}

// a maximum the finished state s is over (the route-independent form of the maxima above)
__device__ __forceinline__ bool cons_over_max(const ConsState& s, const ConsTable& ct, int A, int CH, int Ef) {
  const int ma = ct.t[CONS_MAX_ATOMS], mr = ct.t[CONS_MAX_RINGS];
  bool over = (ma >= 0 && s.n > ma) || (mr >= 0 && s.rank > mr);
  for (int t = 0; t < A; ++t) over |= ct.max_type(t) >= 0 && s.type_cnt[t] > ct.max_type(t);
  for (int c = 0; c < CH; ++c) over |= ct.max_charge(c) >= 0 && s.charge_cnt[c] > ct.max_charge(c);
  for (int e = 0; e < Ef; ++e) over |= ct.max_bond(e) >= 0 && s.bond_cnt[e] > ct.max_bond(e);
  return over;
}

}  // namespace gib
