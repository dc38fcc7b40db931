// One round of the batched graph-generation state machine on the device (SURVEY.md §8f rank 1).
//
// Replaces, per round, the ~800 ATen dispatches of the reference's
//   GraphGenerator.get_actions / get_invalid_actions  (GraphGenerator.py:467-657)
//   GraphGenerator.copy_terminated_graphs             (:340-385)
//   GraphGenerator.apply_actions                      (:211-338)
//   GraphGenerator.reset_graphs                       (:425-465)
// with three launches.  Semantics are the reference's, quirks included (they are observable in its outputs):
//   * the flat APD index decodes row-major as
//       f_add[bond_to, atom, charge, (imp_h,) (chirality,) bond_type] | f_conn[bond_to, bond_type] | term
//     where the implicit-H and chirality segments are present when their count (H, C) is > 0 (constants.py:23-95:
//     L0 = neither, the layout of the shipped gdb13 data; L1 = implicit H; L2 = chirality; L3 = both).  An add sets one
//     node feature per segment: atom, A + charge, A + CH + imp_h, A + CH + H + chirality;
//   * bond_from = n_nodes for add, n_nodes - 1 for connect (-1 wraps to the last atom, as Python indexing does);
//   * element 5 of the reference's add tuple (`f_add_idc[5]`, GraphGenerator.py:568, 618) is bond_from only in L0; it is
//     bond_type in L1 / L2 and chirality in L3.  Its "max nodes" rule (element 5 >= max_n_nodes -> invalid) and its
//     reset (element 5 = 0 for such adds and for every add into an empty graph) are applied to that element as the
//     reference applies them: in L3 the chirality of every molecule's first atom is stored as index 0;
//   * deliberate deviation: outside L0 the reference has no result for an add into a graph that already holds
//     max_n_nodes atoms (it indexes nodes[b, N] and raises IndexError).  Here such a slot terminates as invalid, with
//     bond_from = 0, in every layout -- which is the reference's own L0 outcome;
//   * a slot terminates when it samples terminate or an invalid action; slot 0 (the dummy graph) never does, is never
//     zeroed, and is re-stamped every round (so bonds it samples accumulate);
//   * terminated graphs are copied out in their PRE-action state, terminate-sampled slots first (ascending), then
//     invalid ones (ascending); `properly_terminated[k : k + #terminate-sampled]` counts slot 0 if it sampled terminate;
//   * likelihoods are stored at the GLOBAL round index.
//
// gib_generation_sample_round runs the same kernels behind the sampler with the round index and the loop condition of
// GraphGenerator.build_graphs in device memory (so a captured round can be replayed without reading anything back):
// the sampler decides once per call whether the round runs and leaves the round index (or -1: inert) in `ctl`, which
// the decode, scan and apply kernels read instead of their `round` argument.  The plain entry points pass ctl = null.
#include <type_traits>
#include "../../include/gib200.h"
#include "common.cuh"
#include "ops.cuh"
#include "action_mask.cuh"
#include "scaffold_mask.cuh"
#include "constraints.cuh"

namespace gib {

// H / C = implicit-H / chirality index counts, 0 = segment absent; Lw = likelihood columns (2 * max_n_nodes)
struct GenDims { int B, N, F, Ef, A, CH, H, C, Lw; };

// per slot: decoded action + validity  (one thread per slot)
__global__ void gen_decode_kernel(GenDims d, const int* __restrict__ action, const float* __restrict__ edges,
                                  const int* __restrict__ n_nodes, int4* __restrict__ rec, int* __restrict__ flags,
                                  const int* __restrict__ ctl) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= d.B || (ctl && ctl[0] < 0)) return;
  const int a = action[b];
  const int n = n_nodes[b];
  const ActionLayout L{d.N, d.A, d.CH, d.H, d.C, d.Ef};
  const int len_add = layout_len_add(L), len_conn = d.N * d.Ef;
  Action x{ACT_TERM, 0, 0, 0, 0, 0, 0};
  int bond_from = 0, invalid = 0;
  if (a < 0 || a > len_add + len_conn) {
    // not an APD index (a corrupted replay trace, or the sampler's NaN fallback): an invalid action that edits
    // nothing -- the slot terminates as "invalid" and is reset, no field of `rec` is out of range
    invalid = 1;
  } else {
    // the rule of action_mask.cuh (GraphGenerator.py:573-657): the mask of gib_action_mask_logits forbids exactly
    // the actions flagged invalid here
    x = decode_action(a, L);
    float psum = 0.f;
    if (x.kind == ACT_CONN) psum = pair_sum(edges + (size_t)b * d.N * d.N * d.Ef, d.N, d.Ef, x.bond_to, n);
    invalid = structure_forbidden(x, L, n, psum) ? 1 : 0;
    if (x.kind == ACT_ADD) {
      bond_from = n;
      // get_actions: f_add_idc[5][max_node_idc] = 0 (:568) for adds past max_n_nodes and every add into an empty graph
      if (add_e5(x, L, n) >= d.N || n == 0) {
        const int e5_sel = layout_e5_sel(L);
        if (e5_sel == 0) bond_from = 0;
        else if (e5_sel == 2) x.chir = 0;
        else x.btype = 0;
      }
      if (n >= d.N) bond_from = 0;                    // full graph: the L0 outcome in every layout (see above)
    } else if (x.kind == ACT_CONN) {
      bond_from = n - 1 < 0 ? n - 1 + d.N : n - 1;    // Python negative index
    }
  }
  const int kind = x.kind;
  rec[b] = make_int4(kind | (invalid << 4), x.bond_to | (bond_from << 8), x.atom | (x.charge << 8),
                     x.btype | (x.imp_h << 8) | (x.chir << 16));
  // one class per slot: an index outside the APD decodes as kind TERM but counts once, as invalid (the scan gives every
  // flagged slot one output row; counting it in both classes left a row unwritten and over-counted n_generated)
  flags[b] = invalid ? 2 : (kind == ACT_TERM ? 1 : 0);
}

// single CTA: output positions of the slots that terminate this round + counters
// counters[0] = n_generated (in/out), counters[1] = written this round
// ctl != null: the round index of this call (< 0: inert), and state = {next round, status} is advanced here
__global__ void __launch_bounds__(1024) gen_scan_kernel(int B, const int* __restrict__ flags, int* __restrict__ pos,
                                                        int* __restrict__ counters,
                                                        signed char* __restrict__ properly_terminated, int cap,
                                                        const int* __restrict__ ctl, int* __restrict__ state,
                                                        int rounds, gib_scaffolds sc) {
  __shared__ int s_cnt[3][1024];
  __shared__ int s_tot[4];
  if (ctl && ctl[0] < 0) return;
  const int L = ceil_div(B, 1024);
  const int lo = min(B, (int)threadIdx.x * L), hi = min(B, lo + L);
  int c_term = 0, c_inv = 0;
  for (int b = lo; b < hi; ++b) {
    if (b == 0) continue;
    c_term += flags[b] & 1;
    c_inv += (flags[b] >> 1) & 1;
  }
  s_cnt[0][threadIdx.x] = c_term;
  s_cnt[1][threadIdx.x] = c_inv;
  // scaffolds: a third prefix, over every restarted slot (either class) in slot order -- its scaffold assignment
  if (sc.slot_ids) s_cnt[2][threadIdx.x] = c_term + c_inv;
  __syncthreads();
  if (threadIdx.x == 0) {   // fixed-order serial prefix over 1024 partials (tiny)
    int run = 0;
    for (int i = 0; i < 1024; ++i) { int v = s_cnt[0][i]; s_cnt[0][i] = run; run += v; }
    s_tot[0] = run;
    int run2 = 0;
    for (int i = 0; i < 1024; ++i) { int v = s_cnt[1][i]; s_cnt[1][i] = run2; run2 += v; }
    s_tot[1] = run2;
    s_tot[2] = counters[0];
    if (sc.slot_ids) {
      int run3 = 0;
      for (int i = 0; i < 1024; ++i) { int v = s_cnt[2][i]; s_cnt[2][i] = run3; run3 += v; }
      s_tot[3] = sc.started[0];
    }
  }
  __syncthreads();
  const int n_term = s_tot[0], n_inv = s_tot[1], k = s_tot[2];
  int rt = s_cnt[0][threadIdx.x], ri = s_cnt[1][threadIdx.x];
  for (int b = lo; b < hi; ++b) {
    int p = -1;
    if (b != 0) {
      if (flags[b] & 1) p = k + rt++;
      else if (flags[b] & 2) p = k + n_term + ri++;
    }
    pos[b] = (p >= 0 && p < cap) ? p : (p >= 0 ? -2 : -1);   // -2: would overflow the output buffers
  }
  if (sc.slot_ids) {
    // each restarted slot: its old scaffold to its output row, then the next scaffold in round-robin order (each
    // thread reads and writes only its own slots; gen_apply_kernel copies the new scaffold in)
    int rs = s_cnt[2][threadIdx.x];
    const int started = s_tot[3];
    for (int b = max(lo, 1); b < hi; ++b) {
      if (flags[b] == 0) continue;
      const int p = pos[b];
      if (p >= 0) sc.gen_scaffolds[p] = sc.slot_ids[b];
      sc.slot_ids[b] = (int)(((long long)started + rs++) % sc.S);
    }
  }
  // properly_terminated[k : k + len(term)] = 1, where len(term) counts the dummy slot too (build_graphs :127)
  const int n_term_all = n_term + ((B > 0 && (flags[0] & 1)) ? 1 : 0);
  for (int i = threadIdx.x; i < n_term_all; i += 1024)
    if (k + i < cap) properly_terminated[k + i] = 1;
  if (threadIdx.x == 0) {
    counters[1] = n_term + n_inv;
    counters[0] = k + n_term + n_inv;
    if (sc.slot_ids) sc.started[0] = s_tot[3] + n_term + n_inv;
    if (ctl) {                        // build_graphs' loop rule: round 2N would be needed -> status 1 (round limit)
      const int next = ctl[0] + 1;
      state[0] = next;
      if (k + n_term + n_inv < B && next >= rounds) state[1] = 1;
    }
  }
}

// scaffold s of the table as float 0/1 into one slot's nodes / edges (all rows: the slot's old content is overwritten)
__device__ __forceinline__ void load_scaffold(const gib_scaffolds& sc, int s, int NF, int NNE, float* nb, float* eb) {
  const signed char* sn = sc.nodes + (size_t)s * NF;
  const signed char* se = sc.edges + (size_t)s * NNE;
  for (int i = threadIdx.x; i < NF; i += blockDim.x) nb[i] = (float)sn[i];
  for (int i = threadIdx.x; i < NNE; i += blockDim.x) eb[i] = (float)se[i];
}

// one CTA per slot: copy-out (pre-action state), apply the action, reset, re-stamp the dummy graph
__global__ void __launch_bounds__(128) gen_apply_kernel(GenDims d, int round, const int4* __restrict__ rec,
                                                        const int* __restrict__ pos, const float* __restrict__ lik,
                                                        float* __restrict__ nodes, float* __restrict__ edges,
                                                        int* __restrict__ n_nodes, float* __restrict__ likelihoods,
                                                        float* __restrict__ g_nodes, float* __restrict__ g_edges,
                                                        signed char* __restrict__ g_n_nodes,
                                                        float* __restrict__ g_lik, const int* __restrict__ ctl,
                                                        gib_scaffolds sc) {
  if (ctl) {
    round = ctl[0];
    if (round < 0) return;
  }
  const int b = blockIdx.x;
  const int NF = d.N * d.F, NNE = d.N * d.N * d.Ef;
  float* nb = nodes + (size_t)b * NF;
  float* eb = edges + (size_t)b * NNE;
  float* lb = likelihoods + (size_t)b * d.Lw;
  const int p = pos[b];
  const int4 r = rec[b];
  const int kind = r.x & 15;
  if (p != -1) {                      // terminates this round (never slot 0)
    if (threadIdx.x == 0) lb[round] = lik[b];                       // copy_terminated_graphs :365
    __syncthreads();
    if (p >= 0) {
      for (int i = threadIdx.x; i < NF; i += 128) g_nodes[(size_t)p * NF + i] = nb[i];
      for (int i = threadIdx.x; i < NNE; i += 128) g_edges[(size_t)p * NNE + i] = eb[i];
      for (int i = threadIdx.x; i < d.Lw; i += 128) g_lik[(size_t)p * d.Lw + i] = lb[i];
      if (threadIdx.x == 0) g_n_nodes[p] = (signed char)n_nodes[b];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < d.Lw; i += 128) lb[i] = 0.f;
    if (sc.slot_ids) {                                                // restart from the scaffold gen_scan assigned
      const int s = sc.slot_ids[b];
      load_scaffold(sc, s, NF, NNE, nb, eb);
      if (threadIdx.x == 0) n_nodes[b] = sc.n_atoms[s];
      return;
    }
    for (int i = threadIdx.x; i < NF; i += 128) nb[i] = 0.f;          // reset_graphs :447-460
    for (int i = threadIdx.x; i < NNE; i += 128) eb[i] = 0.f;
    if (threadIdx.x == 0) n_nodes[b] = 0;
    return;
  }
  if (threadIdx.x == 0) {
    const int bond_to = r.y & 255, bond_from = r.y >> 8, atom = r.z & 255, charge = r.z >> 8, bt = r.w & 255;
    if (kind == ACT_ADD) {                                            // apply_actions._add_nodes :257-306
      nb[bond_from * d.F + atom] = 1.f;
      nb[bond_from * d.F + d.A + charge] = 1.f;
      if (d.H) nb[bond_from * d.F + d.A + d.CH + ((r.w >> 8) & 255)] = 1.f;
      if (d.C) nb[bond_from * d.F + d.A + d.CH + d.H + (r.w >> 16)] = 1.f;
      if (n_nodes[b] != 0) {
        eb[(bond_to * d.N + bond_from) * d.Ef + bt] = 1.f;
        eb[(bond_from * d.N + bond_to) * d.Ef + bt] = 1.f;
      }
      n_nodes[b] += 1;
      lb[round] = lik[b];
    } else if (kind == ACT_CONN) {                                    // _conn_nodes :325-330
      eb[(bond_from * d.N + bond_to) * d.Ef + bt] = 1.f;
      eb[(bond_to * d.N + bond_from) * d.Ef + bt] = 1.f;
      lb[round] = lik[b];
    }
  }
  if (b == 0) {                                                       // dummy graph, reset_graphs :462-465
    __syncthreads();
    for (int i = threadIdx.x; i < NF; i += 128) nb[i] = 1.f;
    if (threadIdx.x == 0) { eb[0] = 1.f; n_nodes[0] = 1; }
  }
}

// the scaffold start state: one CTA per slot b >= 1 (grid B - 1)
__global__ void __launch_bounds__(128) gen_scaffold_init_kernel(int N, int F, int Ef, int Lw, gib_scaffolds sc,
                                                                float* __restrict__ nodes, float* __restrict__ edges,
                                                                int* __restrict__ n_nodes,
                                                                float* __restrict__ likelihoods) {
  const int b = blockIdx.x + 1, B = gridDim.x + 1;
  const int NF = N * F, NNE = N * N * Ef;
  const int s = (b - 1) % sc.S;
  load_scaffold(sc, s, NF, NNE, nodes + (size_t)b * NF, edges + (size_t)b * NNE);
  for (int i = threadIdx.x; i < Lw; i += 128) likelihoods[(size_t)b * Lw + i] = 0.f;
  if (threadIdx.x == 0) {
    n_nodes[b] = sc.n_atoms[s];
    sc.slot_ids[b] = s;
    if (b == 1) { sc.slot_ids[0] = -1; sc.started[0] = B - 1; }
  }
}

// the round gate of a captured round's mask (state != null): the mask runs only when the sampler after it will run
// the round -- fewer than B molecules finished, status 0, a round index in [0, 2N)
__device__ __forceinline__ bool round_gated_off(const int* __restrict__ state, const int* __restrict__ counters, int B,
                                                int N) {
  return state && !(counters[0] < B && state[1] == 0 && state[0] >= 0 && state[0] < 2 * N);
}

// the attachment-point mask (scaffold_mask.cuh): one CTA per slot, -inf into the add blocks and connect entries whose
// bond_to is a protected atom, and into every connect while bond_from = n - 1 is still a scaffold atom (n_nodes only
// grows from k_s, so that is n == k_s).  Terminate is never touched, so a masked row keeps an action of non-zero
// probability.  Slots below first_slot are left alone: 1 skips the generator's dummy slot 0, 0 masks a route batch,
// where slot 0 carries a real state.
__global__ void __launch_bounds__(128) gen_mask_kernel(int N, int Ef, int apd, gib_scaffolds sc,
                                                       const int* __restrict__ slot_ids,
                                                       const int* __restrict__ n_nodes, const int* __restrict__ row,
                                                       const int* __restrict__ state,
                                                       const int* __restrict__ counters, float* __restrict__ logits,
                                                       int first_slot) {
  const int b = blockIdx.x, B = gridDim.x;
  if (round_gated_off(state, counters, B, N)) return;
  const size_t off = row ? (size_t)row[0] * B : 0;
  const int s = slot_ids[off + b];
  if (b < first_slot || s < 0 || s >= sc.S) return;
  const int k = sc.n_atoms[s], n = n_nodes[off + b];
  const unsigned int* pm = sc.protect + (size_t)s * 4;
  const int per_node = (apd - 1) / N - Ef, len_add = N * per_node;
  float* o = logits + (size_t)b * apd;
  const bool conn_all = scaffold_connects_closed(n, k);
  for (int i = 0; i < k; ++i) {
    if (!scaffold_protected(pm, i)) continue;
    for (int t = threadIdx.x; t < per_node; t += 128) o[(size_t)i * per_node + t] = -INFINITY;
    if (!conn_all)
      for (int t = threadIdx.x; t < Ef; t += 128) o[len_add + i * Ef + t] = -INFINITY;
  }
  if (conn_all)
    for (int t = threadIdx.x; t < N * Ef; t += 128) o[len_add + t] = -INFINITY;
}

// what every CTA of the action mask and of the constraint check sets up the same way from one state (node rows nb
// [N, F], edges e [N, N, Ef]): the atom count n (n_nodes[idx] read as the nearest bound of [0, N], or the number of
// non-empty node rows when n_nodes is null; N <= 127 < 128), the valence usage of its atoms into s_used / s_limit
// (valence mode) and the attachment-point mask pm of the scaffold slot_ids[idx] with its k atoms (null without
// attachment points or for an id outside [0, S); slot_ids is given whenever sc.protect is)
struct SlotRules {
  int n, k;
  const unsigned int* pm;
};

template <typename T>
__device__ __forceinline__ SlotRules slot_rules(const ActionLayout& L, int F, int valence, const int* __restrict__ table,
                                                const T* __restrict__ nb, const T* __restrict__ e,
                                                const int* __restrict__ n_nodes, const int* __restrict__ slot_ids,
                                                size_t idx, const gib_scaffolds& sc, int* s_used, int* s_limit) {
  SlotRules r{0, 0, nullptr};
  const int N = L.N;
  if (n_nodes) {
    r.n = min(max(n_nodes[idx], 0), N);
  } else {
    int live = 0;
    if ((int)threadIdx.x < N) {
      const T* nr = nb + (size_t)threadIdx.x * F;
      for (int f = 0; f < F; ++f) live |= nr[f] != T(0);
    }
    r.n = __syncthreads_count(live);
  }
  if (valence) {
    const int* order = table + L.A * L.CH;
    for (int i = threadIdx.x; i < r.n; i += 128) {
      const int2 u = atom_usage(nb + (size_t)i * F, e + (size_t)i * N * L.Ef, L, table, order, order + L.Ef);
      s_used[i] = u.x;
      s_limit[i] = u.y;
    }
    __syncthreads();
  }
  if (sc.protect) {
    const int s = slot_ids[idx];
    if (s >= 0 && s < sc.S) {
      r.pm = sc.protect + (size_t)s * 4;
      r.k = sc.n_atoms[s];
    }
  }
  return r;
}

// the action mask (action_mask.cuh): one CTA per slot, -inf into every entry of the slot's logits row that the rule
// forbids in its state (nodes [B, N, F] / edges [B, N, N, Ef], float in the generator, int8 in route batches), OR-ed
// with the attachment-point rule of the slot's scaffold when sc.protect is given.  The gate, `row` and first_slot mean
// what they mean for gen_mask_kernel; `row` selects the row of n_nodes and slot_ids only, the state is always
// [B, ...].  table = V [A * CH] | bond orders [Ef] | implicit-H counts [H].  Terminate is never touched, except with
// kCons: the constraint rule (constraints.cuh, table `cons`) joins the OR, and terminate gets -inf while the state is
// under a minimum and some other entry survives (a block-wide OR over the row).
template <typename T, bool kCons>
__global__ void __launch_bounds__(128) gen_action_mask_kernel(ActionLayout L, int F, int apd, int valence,
                                                              const int* __restrict__ table,
                                                              const T* __restrict__ nodes, const T* __restrict__ edges,
                                                              const int* __restrict__ n_nodes, gib_scaffolds sc,
                                                              const int* __restrict__ slot_ids,
                                                              const int* __restrict__ row,
                                                              const int* __restrict__ state,
                                                              const int* __restrict__ counters,
                                                              float* __restrict__ logits, int first_slot,
                                                              const int* __restrict__ cons) {
  __shared__ int s_used[128], s_limit[128];
  __shared__ ConsState s;                                  // referenced, and so allocated, with kCons only
  const int b = blockIdx.x, B = gridDim.x, N = L.N, Ef = L.Ef;
  if (b < first_slot || round_gated_off(state, counters, B, N)) return;
  const size_t off = row ? (size_t)row[0] * B : 0;
  const T* nb = nodes + (size_t)b * N * F;
  const T* e = edges + (size_t)b * N * N * Ef;
  const SlotRules r = slot_rules(L, F, valence, table, nb, e, n_nodes, slot_ids, off + b, sc, s_used, s_limit);
  const ConsTable ct{cons, L.A, L.CH};
  if constexpr (kCons) cons_load(s, ct, L, F, nb, e, r.n);
  const int* order = valence ? table + L.A * L.CH : nullptr;
  const Valence v{s_used, s_limit, valence ? table : nullptr, order, valence ? order + Ef : nullptr};
  const int per_node = (apd - 1) / N - Ef;
  float* o = logits + (size_t)b * apd;
  int survives = 0;
  for (int a = threadIdx.x; a < apd - 1; a += 128) {
    if (action_forbidden(a, L, r.n, e, valence != 0, v) ||
        (r.pm && scaffold_forbidden(a, r.n, r.k, r.pm, N, Ef, per_node)) ||
        (kCons && cons_forbidden(decode_action(a, L), s, ct)))
      o[a] = -INFINITY;
    else
      survives = 1;
  }
  if constexpr (kCons)
    if (__syncthreads_or(survives) && s.below && threadIdx.x == 0) o[apd - 1] = -INFINITY;
}

// gib_constraints_check: one CTA per finished molecule, its flag bits (GIB_CONS_*)
template <typename T>
__global__ void __launch_bounds__(128) constraints_check_kernel(ActionLayout L, int F, int apd, int valence,
                                                                const int* __restrict__ table,
                                                                const T* __restrict__ nodes,
                                                                const T* __restrict__ edges,
                                                                const int* __restrict__ n_nodes, gib_scaffolds sc,
                                                                const int* __restrict__ scaffold_ids,
                                                                const int* __restrict__ cons, int* __restrict__ flags) {
  __shared__ int s_used[128], s_limit[128];
  __shared__ ConsState s;
  const int g = blockIdx.x, N = L.N, Ef = L.Ef;
  const T* nb = nodes + (size_t)g * N * F;
  const T* e = edges + (size_t)g * N * N * Ef;
  const SlotRules cs = slot_rules(L, F, valence, table, nb, e, n_nodes, scaffold_ids, g, sc, s_used, s_limit);
  const ConsTable ct{cons, L.A, L.CH};
  cons_load(s, ct, L, F, nb, e, cs.n);
  int f = cons_over_max(s, ct, L.A, L.CH, Ef) ? GIB_CONS_OVER_MAX : 0;
  if (s.below) {                       // did its terminate have probability 0?
    const int* order = valence ? table + L.A * L.CH : nullptr;
    const Valence v{s_used, s_limit, valence ? table : nullptr, order, valence ? order + Ef : nullptr};
    const int per_node = (apd - 1) / N - Ef;
    int survives = 0;
    for (int a = threadIdx.x; a < apd - 1 && !survives; a += 128)
      survives = !(action_forbidden(a, L, cs.n, e, valence != 0, v) ||
                   (cs.pm && scaffold_forbidden(a, cs.n, cs.k, cs.pm, N, Ef, per_node)) ||
                   cons_forbidden(decode_action(a, L), s, ct));
    f |= __syncthreads_or(survives) ? GIB_CONS_UNDER_MIN : GIB_CONS_DEAD_END;
  }
  // girth < m: some bond (u, v) whose ends are within m - 2 bonds of each other without it
  const int m = cons[CONS_MIN_RING_SIZE];
  if (m > 0 && s.rank > 0) {
    bool small = false;
    for (int u = 0; u < s.n && !small; ++u)
      for (int w = u + 1; w < s.n && !small; ++w) {
        if (!((s.adj[u][w >> 5] >> (w & 31)) & 1u)) continue;
        cons_bfs(s, u, w, min(m - 2, s.n));
        small = s.dist[w] <= m - 2;
      }
    if (small) f |= GIB_CONS_SMALL_RING;
  }
  if (threadIdx.x == 0) flags[g] = f;
}

}  // namespace gib

using namespace gib;

// arguments shared by every round entry point; the messages name gib_generation_round
static int check_round_args(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H, int n_chirality,
                            int round) {
  // every index travels in 8 bits of the int4 record; counts <= 255 keep each index <= 254
  const bool counts_ok = n_atom_types > 0 && n_charges > 0 && Ef > 0 && n_imp_H >= 0 && n_chirality >= 0 &&
                         n_atom_types <= 255 && n_charges <= 255 && Ef <= 255 && n_imp_H <= 255 && n_chirality <= 255;
  if (!counts_ok) {
    set_error("gib_generation_round: index counts must lie in 1..255 (0..255 for implicit H / chirality): "
              "A=%d CH=%d H=%d C=%d Ef=%d", n_atom_types, n_charges, n_imp_H, n_chirality, Ef);
    return -1;
  }
  const long long len_add = (long long)N * n_atom_types * n_charges * (n_imp_H ? n_imp_H : 1) *
                            (n_chirality ? n_chirality : 1) * Ef;
  if (B <= 0 || N <= 0 || N > 127 || n_atom_types + n_charges + n_imp_H + n_chirality != F || round < 0 ||
      round >= 2 * N || len_add + (long long)N * Ef >= (1ll << 31)) {
    set_error("gib_generation_round: unsupported arguments (B=%d N=%d F=%d A=%d CH=%d H=%d C=%d round=%d; F must be "
              "A + CH + H + C, and the likelihood buffer holds 2N rounds)",
              B, N, F, n_atom_types, n_charges, n_imp_H, n_chirality, round);
    return -1;
  }
  return 0;
}

// decode -> scan -> apply on the scratch layout of gib_generation_scratch_bytes: rec int4[B], flags int[B], pos int[B],
// then the control word of gib_generation_sample_round in the 64 spare bytes
static int launch_round(const GenDims& d, int round, const int* ctl, int* state, const int* action,
                        const float* likelihood, float* nodes, float* edges, int* n_nodes, float* likelihoods,
                        float* gen_nodes, float* gen_edges, signed char* gen_n_nodes, float* gen_likelihoods,
                        signed char* properly_terminated, int capacity, int* counters, void* scratch,
                        cudaStream_t st, const gib_scaffolds* sc = nullptr) {
  const int B = d.B;
  const gib_scaffolds scv = sc ? *sc : gib_scaffolds{};
  int4* rec = reinterpret_cast<int4*>(scratch);
  int* flags = reinterpret_cast<int*>(rec + B);
  int* pos = flags + B;
  gen_decode_kernel<<<ceil_div(B, 128), 128, 0, st>>>(d, action, edges, n_nodes, rec, flags, ctl);
  GIB_LAUNCH_CHECK();
  gen_scan_kernel<<<1, 1024, 0, st>>>(B, flags, pos, counters, properly_terminated, capacity, ctl, state, d.Lw,
                                       scv);
  GIB_LAUNCH_CHECK();
  gen_apply_kernel<<<B, 128, 0, st>>>(d, round, rec, pos, likelihood, nodes, edges, n_nodes, likelihoods, gen_nodes,
                                      gen_edges, gen_n_nodes, gen_likelihoods, ctl, scv);
  GIB_LAUNCH_CHECK();
  return 0;
}

static int* round_ctl(void* scratch, int B) {
  return reinterpret_cast<int*>(reinterpret_cast<int4*>(scratch) + B) + 2 * B;   // behind rec, flags and pos
}

// a scaffold table the round kernels can use; `who` names the entry point
static int check_scaffolds(const char* who, const gib_scaffolds* sc) {
  if (!sc || sc->S <= 0 || !sc->nodes || !sc->edges || !sc->n_atoms || !sc->slot_ids || !sc->started ||
      !sc->gen_scaffolds) {
    set_error("%s: the scaffold table needs S >= 1 and its nodes, edges, n_atoms, slot_ids, started and gen_scaffolds "
              "buffers", who);
    return -1;
  }
  return 0;
}

static int round_layout(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H, int n_chirality,
                        const gib_scaffolds* sc, int round, const int* action, const float* likelihood, float* nodes,
                        float* edges, int* n_nodes, float* likelihoods, float* gen_nodes, float* gen_edges,
                        signed char* gen_n_nodes, float* gen_likelihoods, signed char* properly_terminated,
                        int capacity, int* counters, void* scratch, gib_stream stream) {
  GIB_TRY(check_round_args(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, round));
  GenDims d{B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, 2 * N};
  return launch_round(d, round, nullptr, nullptr, action, likelihood, nodes, edges, n_nodes, likelihoods, gen_nodes,
                      gen_edges, gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters, scratch,
                      reinterpret_cast<cudaStream_t>(stream), sc);
}

extern "C" int gib_generation_round_layout(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                           int n_chirality, int round, const int* action, const float* likelihood,
                                           float* nodes, float* edges, int* n_nodes, float* likelihoods,
                                           float* gen_nodes, float* gen_edges, signed char* gen_n_nodes,
                                           float* gen_likelihoods, signed char* properly_terminated, int capacity,
                                           int* counters, void* scratch, gib_stream stream) {
  return round_layout(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, nullptr, round, action, likelihood,
                      nodes, edges, n_nodes, likelihoods, gen_nodes, gen_edges, gen_n_nodes, gen_likelihoods,
                      properly_terminated, capacity, counters, scratch, stream);
}

extern "C" int gib_generation_round_scaffold(int B, int N, int F, int Ef, int n_atom_types, int n_charges,
                                             int n_imp_H, int n_chirality, const gib_scaffolds* sc, int round,
                                             const int* action, const float* likelihood, float* nodes, float* edges,
                                             int* n_nodes, float* likelihoods, float* gen_nodes, float* gen_edges,
                                             signed char* gen_n_nodes, float* gen_likelihoods,
                                             signed char* properly_terminated, int capacity, int* counters,
                                             void* scratch, gib_stream stream) {
  GIB_TRY(check_scaffolds("gib_generation_round_scaffold", sc));
  return round_layout(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, sc, round, action, likelihood,
                      nodes, edges, n_nodes, likelihoods, gen_nodes, gen_edges, gen_n_nodes, gen_likelihoods,
                      properly_terminated, capacity, counters, scratch, stream);
}

static long long layout_apd(int N, int Ef, int n_atom_types, int n_charges, int n_imp_H, int n_chirality) {
  return (long long)N * n_atom_types * n_charges * (n_imp_H ? n_imp_H : 1) * (n_chirality ? n_chirality : 1) * Ef +
         (long long)N * Ef + 1;
}

static int sample_round(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H, int n_chirality,
                        const gib_scaffolds* sc, const float* logits, int apd, const float* uniforms, int* state,
                        int* action, float* likelihood, float* nodes, float* edges, int* n_nodes, float* likelihoods,
                        float* gen_nodes, float* gen_edges, signed char* gen_n_nodes, float* gen_likelihoods,
                        signed char* properly_terminated, int capacity, int* counters, void* scratch,
                        gib_stream stream, const gib_sampling_policy* policy) {
  GIB_TRY(check_round_args(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, 0));
  const long long want = layout_apd(N, Ef, n_atom_types, n_charges, n_imp_H, n_chirality);
  if (apd != want) {
    set_error("gib_generation_round: apd=%d, the action layout (N=%d A=%d CH=%d H=%d C=%d Ef=%d) has %lld actions",
              apd, N, n_atom_types, n_charges, n_imp_H, n_chirality, Ef, want);
    return -1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  GenDims d{B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, 2 * N};
  int* ctl = round_ctl(scratch, B);
  const RoundGate gate{state, counters, ctl, 2 * N};
  if (policy)
    GIB_TRY(policy_sample_launch(logits, B, apd, uniforms, policy, action, likelihood, nullptr, &gate, st));
  else
    GIB_TRY(sample_actions_launch(logits, B, apd, uniforms, action, likelihood, &gate, st));
  return launch_round(d, 0, ctl, state, action, likelihood, nodes, edges, n_nodes, likelihoods, gen_nodes, gen_edges,
                      gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters, scratch, st, sc);
}

extern "C" int gib_generation_sample_round(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                           int n_chirality, const float* logits, int apd, const float* uniforms,
                                           int* state, int* action, float* likelihood, float* nodes, float* edges,
                                           int* n_nodes, float* likelihoods, float* gen_nodes, float* gen_edges,
                                           signed char* gen_n_nodes, float* gen_likelihoods,
                                           signed char* properly_terminated, int capacity, int* counters,
                                           void* scratch, gib_stream stream) {
  return sample_round(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, nullptr, logits, apd, uniforms,
                      state, action, likelihood, nodes, edges, n_nodes, likelihoods, gen_nodes, gen_edges,
                      gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters, scratch, stream, nullptr);
}

extern "C" int gib_generation_sample_round_scaffold(int B, int N, int F, int Ef, int n_atom_types, int n_charges,
                                                    int n_imp_H, int n_chirality, const gib_scaffolds* sc,
                                                    const float* logits, int apd, const float* uniforms, int* state,
                                                    int* action, float* likelihood, float* nodes, float* edges,
                                                    int* n_nodes, float* likelihoods, float* gen_nodes,
                                                    float* gen_edges, signed char* gen_n_nodes,
                                                    float* gen_likelihoods, signed char* properly_terminated,
                                                    int capacity, int* counters, void* scratch, gib_stream stream) {
  GIB_TRY(check_scaffolds("gib_generation_sample_round_scaffold", sc));
  return sample_round(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, sc, logits, apd, uniforms, state,
                      action, likelihood, nodes, edges, n_nodes, likelihoods, gen_nodes, gen_edges, gen_n_nodes,
                      gen_likelihoods, properly_terminated, capacity, counters, scratch, stream, nullptr);
}

static int rl_sample_round(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H, int n_chirality,
                           const gib_scaffolds* sc, const float* logits_a, const float* logits_b, int apd,
                           const float* uniforms, const int* actions, int* state, int* act_rec, float* p_a,
                           float* p_b, int* action, float* tags, float* nodes, float* edges, int* n_nodes,
                           float* likelihoods, float* gen_nodes, float* gen_edges, signed char* gen_n_nodes,
                           float* gen_likelihoods, signed char* properly_terminated, int capacity, int* counters,
                           void* scratch, gib_stream stream, const gib_sampling_policy* policy) {
  GIB_TRY(check_round_args(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, 0));
  const long long want = layout_apd(N, Ef, n_atom_types, n_charges, n_imp_H, n_chirality);
  if (apd != want || B + 1 >= (1 << 24) || !logits_a || !logits_b || (!uniforms && !actions) || !act_rec || !p_a ||
      !p_b) {
    set_error("gib_rl_sample_round: apd=%d (the action layout N=%d A=%d CH=%d H=%d C=%d Ef=%d has %lld actions), "
              "B=%d (slot tags travel as fp32: B < 2^24 - 1), and logits, draws and record tables must be given",
              apd, N, n_atom_types, n_charges, n_imp_H, n_chirality, Ef, want, B);
    return -1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  GenDims d{B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, 2 * N};
  int* ctl = round_ctl(scratch, B);
  const RoundGate gate{state, counters, ctl, 2 * N, actions};
  if (policy && !actions)    // recorded actions are taken as they are
    GIB_TRY(policy_sample_launch(logits_a, B, apd, uniforms, policy, action, tags, nullptr, &gate, st));
  else
    GIB_TRY(sample_actions_launch(logits_a, B, apd, uniforms, action, tags, &gate, st));
  GIB_TRY(rl_probs_launch(logits_a, logits_b, B, apd, action, ctl, act_rec, p_a, p_b, tags, st));
  return launch_round(d, 0, ctl, state, action, tags, nodes, edges, n_nodes, likelihoods, gen_nodes, gen_edges,
                      gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters, scratch, st, sc);
}

extern "C" int gib_rl_sample_round(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                   int n_chirality, const float* logits_a, const float* logits_b, int apd,
                                   const float* uniforms, const int* actions, int* state, int* act_rec, float* p_a,
                                   float* p_b, int* action, float* tags, float* nodes, float* edges, int* n_nodes,
                                   float* likelihoods, float* gen_nodes, float* gen_edges, signed char* gen_n_nodes,
                                   float* gen_likelihoods, signed char* properly_terminated, int capacity,
                                   int* counters, void* scratch, gib_stream stream) {
  return rl_sample_round(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, nullptr, logits_a, logits_b, apd,
                         uniforms, actions, state, act_rec, p_a, p_b, action, tags, nodes, edges, n_nodes, likelihoods,
                         gen_nodes, gen_edges, gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters,
                         scratch, stream, nullptr);
}

extern "C" int gib_rl_sample_round_scaffold(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                            int n_chirality, const gib_scaffolds* sc, const float* logits_a,
                                            const float* logits_b, int apd, const float* uniforms, const int* actions,
                                            int* state, int* act_rec, float* p_a, float* p_b, int* action,
                                            float* tags, float* nodes, float* edges, int* n_nodes,
                                            float* likelihoods, float* gen_nodes, float* gen_edges,
                                            signed char* gen_n_nodes, float* gen_likelihoods,
                                            signed char* properly_terminated, int capacity, int* counters,
                                            void* scratch, gib_stream stream) {
  GIB_TRY(check_scaffolds("gib_rl_sample_round_scaffold", sc));
  return rl_sample_round(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, sc, logits_a, logits_b, apd,
                         uniforms, actions, state, act_rec, p_a, p_b, action, tags, nodes, edges, n_nodes, likelihoods,
                         gen_nodes, gen_edges, gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters,
                         scratch, stream, nullptr);
}

extern "C" int gib_generation_scaffold_init(int B, int N, int F, int Ef, const gib_scaffolds* sc, float* nodes,
                                            float* edges, int* n_nodes, float* likelihoods, gib_stream stream) {
  GIB_TRY(check_scaffolds("gib_generation_scaffold_init", sc));
  if (B <= 0 || N <= 0 || N > 127 || F <= 0 || Ef <= 0 || !nodes || !edges || !n_nodes || !likelihoods) {
    set_error("gib_generation_scaffold_init: unsupported arguments (B=%d N=%d F=%d Ef=%d; the state buffers must be "
              "given)", B, N, F, Ef);
    return -1;
  }
  if (B == 1) {                      // only the dummy slot: started = B - 1 = 0, slot_ids[0] = -1 (all bits set)
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    GIB_CUDA_TRY(cudaMemsetAsync(sc->started, 0, sizeof(int), st));
    GIB_CUDA_TRY(cudaMemsetAsync(sc->slot_ids, 0xff, sizeof(int), st));
    return 0;
  }
  gen_scaffold_init_kernel<<<B - 1, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(N, F, Ef, 2 * N, *sc, nodes,
                                                                                      edges, n_nodes, likelihoods);
  GIB_LAUNCH_CHECK();
  return 0;
}

// the attachment-point mask alone (`who` names the entry point; first_slot and the gate as for gen_mask_kernel)
static int attachment_mask_launch(const char* who, int B, int N, int Ef, int apd, const gib_scaffolds* sc,
                                  const int* slot_ids, const int* n_nodes, const int* row, const int* state,
                                  const int* counters, float* logits, int first_slot, gib_stream stream) {
  if (!sc || sc->S <= 0 || !sc->n_atoms || B <= 0 || N <= 0 || N > 127 || Ef <= 0 || apd < 1 ||
      (apd - 1) % N != 0 || (apd - 1) / N <= Ef || !slot_ids || !n_nodes || !logits || (!state != !counters)) {
    set_error("%s: bad arguments (B=%d N=%d Ef=%d apd=%d; apd - 1 must be N times the per-node add and connect "
              "lengths, the table, slot_ids, n_nodes and logits must be given, and state and counters together or "
              "neither)", who, B, N, Ef, apd);
    return -1;
  }
  if (!sc->protect) return 0;       // no attachment points: nothing is masked
  gen_mask_kernel<<<B, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(N, Ef, apd, *sc, slot_ids, n_nodes, row,
                                                                         state, counters, logits, first_slot);
  GIB_LAUNCH_CHECK();
  return 0;
}

extern "C" int gib_generation_mask_logits(int B, int N, int Ef, int apd, const gib_scaffolds* sc, const int* slot_ids,
                                          const int* n_nodes, const int* row, const int* state, const int* counters,
                                          float* logits, gib_stream stream) {
  return attachment_mask_launch("gib_generation_mask_logits", B, N, Ef, apd, sc, slot_ids, n_nodes, row, state,
                                counters, logits, 1, stream);
}

extern "C" int gib_route_mask_logits(int B, int N, int Ef, int apd, const gib_scaffolds* sc, const int* slot_ids,
                                     const int* n_nodes, float* logits, gib_stream stream) {
  return attachment_mask_launch("gib_route_mask_logits", B, N, Ef, apd, sc, slot_ids, n_nodes, nullptr, nullptr,
                                nullptr, logits, 0, stream);
}

// the arguments of the action mask and of the constraint check (`who` names the entry point); *scv receives the
// scaffold table to apply (empty without attachment points)
static int check_mask_args(const char* who, int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                           int n_chirality, int apd, int mode, const int* table, const float* nodes,
                           const float* edges, const signed char* nodes_i8, const signed char* edges_i8,
                           const gib_scaffolds* sc, const int* slot_ids, gib_scaffolds* scv) {
  const bool counts_ok = n_atom_types > 0 && n_charges > 0 && Ef > 0 && n_imp_H >= 0 && n_chirality >= 0 &&
                         n_atom_types <= 255 && n_charges <= 255 && Ef <= 255 && n_imp_H <= 255 && n_chirality <= 255;
  if (!counts_ok || B <= 0 || N <= 0 || N > 127 || n_atom_types + n_charges + n_imp_H + n_chirality != F) {
    set_error("%s: unsupported dims (B=%d N=%d F=%d A=%d CH=%d H=%d C=%d Ef=%d; N <= 127, the "
              "counts lie in 1..255 (0..255 for implicit H / chirality) and F = A + CH + H + C)", who, B, N, F,
              n_atom_types, n_charges, n_imp_H, n_chirality, Ef);
    return -1;
  }
  const long long want = layout_apd(N, Ef, n_atom_types, n_charges, n_imp_H, n_chirality);
  if (apd != want || want >= (1ll << 31)) {
    set_error("%s: apd=%d, the action layout (N=%d A=%d CH=%d H=%d C=%d Ef=%d) has %lld actions",
              who, apd, N, n_atom_types, n_charges, n_imp_H, n_chirality, Ef, want);
    return -1;
  }
  const bool as_float = nodes && edges, as_i8 = nodes_i8 && edges_i8;
  const int n_state = !!nodes + !!edges + !!nodes_i8 + !!edges_i8;
  if ((mode != GIB_ACTION_MASK_STRUCTURE && mode != GIB_ACTION_MASK_VALENCE) || n_state != 2 ||
      !(as_float || as_i8) || (mode == GIB_ACTION_MASK_VALENCE && !table)) {
    set_error("%s: bad arguments (mode=%d; mode is GIB_ACTION_MASK_STRUCTURE or GIB_ACTION_MASK_VALENCE, the "
              "valence mode needs the table, the state is given as float nodes and edges or as int8 nodes and edges)",
              who, mode);
    return -1;
  }
  *scv = gib_scaffolds{};
  if (sc && sc->protect) {
    if (sc->S <= 0 || !sc->n_atoms || !slot_ids) {
      set_error("%s: a scaffold table with attachment points needs S >= 1, n_atoms and slot_ids", who);
      return -1;
    }
    *scv = *sc;
  }
  return 0;
}

static int action_mask_launch(const char* who, int B, int N, int F, int Ef, int n_atom_types, int n_charges,
                              int n_imp_H, int n_chirality, int apd, int mode, const int* table, const float* nodes,
                              const float* edges, const signed char* nodes_i8, const signed char* edges_i8,
                              const int* n_nodes, const gib_scaffolds* sc, const int* slot_ids, const int* row,
                              const int* state, const int* counters, float* logits, int first_slot,
                              gib_stream stream, const int* cons) {
  gib_scaffolds scv;
  GIB_TRY(check_mask_args(who, B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, apd, mode, table, nodes,
                          edges, nodes_i8, edges_i8, sc, slot_ids, &scv));
  if (!logits || (!state != !counters) || (first_slot != 0 && first_slot != 1)) {
    set_error("%s: bad arguments (first_slot=%d; logits must be given, state and counters together or neither, "
              "first_slot is 0 or 1)", who, first_slot);
    return -1;
  }
  const ActionLayout L{N, n_atom_types, n_charges, n_imp_H, n_chirality, Ef};
  const int valence = mode == GIB_ACTION_MASK_VALENCE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto launch = [&](const auto* nodes_t, const auto* edges_t) {
    using T = std::decay_t<decltype(*nodes_t)>;                     // float or signed char
    const auto kernel = cons ? gen_action_mask_kernel<T, true> : gen_action_mask_kernel<T, false>;
    kernel<<<B, 128, 0, st>>>(L, F, apd, valence, table, nodes_t, edges_t, n_nodes, scv, slot_ids, row, state,
                              counters, logits, first_slot, cons);
  };
  if (nodes && edges) launch(nodes, edges);
  else launch(nodes_i8, edges_i8);
  GIB_LAUNCH_CHECK();
  return 0;
}

extern "C" int gib_action_mask_logits(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                      int n_chirality, int apd, int mode, const int* table, const float* nodes,
                                      const float* edges, const signed char* nodes_i8, const signed char* edges_i8,
                                      const int* n_nodes, const gib_scaffolds* sc, const int* slot_ids,
                                      const int* row, const int* state, const int* counters, float* logits,
                                      int first_slot, gib_stream stream) {
  return action_mask_launch("gib_action_mask_logits", B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality,
                            apd, mode, table, nodes, edges, nodes_i8, edges_i8, n_nodes, sc, slot_ids, row, state,
                            counters, logits, first_slot, stream, nullptr);
}

// ---- constraints (constraints.cuh) ----
extern "C" int gib_action_mask_logits_constrained(int B, int N, int F, int Ef, int n_atom_types, int n_charges,
                                                  int n_imp_H, int n_chirality, int apd, int mode, const int* table,
                                                  const float* nodes, const float* edges,
                                                  const signed char* nodes_i8, const signed char* edges_i8,
                                                  const int* n_nodes, const gib_scaffolds* sc, const int* slot_ids,
                                                  const int* row, const int* state, const int* counters,
                                                  float* logits, int first_slot, gib_stream stream,
                                                  const int* constraints) {
  return action_mask_launch("gib_action_mask_logits_constrained", B, N, F, Ef, n_atom_types, n_charges, n_imp_H,
                            n_chirality, apd, mode, table, nodes, edges, nodes_i8, edges_i8, n_nodes, sc, slot_ids,
                            row, state, counters, logits, first_slot, stream, constraints);
}

extern "C" size_t gib_constraints_ints(int n_atom_types, int n_charges, int Ef) {
  if (n_atom_types <= 0 || n_charges <= 0 || Ef <= 0 || n_atom_types > 255 || n_charges > 255 || Ef > 255) return 0;
  return (size_t)GIB_CONS_HDR_INTS + 2 * n_atom_types + n_charges + Ef;
}

extern "C" int gib_constraints_set(int* table, const int* values, int N, int n_atom_types, int n_charges, int Ef,
                                   gib_stream stream) {
  const size_t len = gib_constraints_ints(n_atom_types, n_charges, Ef);
  if (!table || !values || len == 0 || N <= 0 || N > 127) {
    set_error("gib_constraints_set: refused (table %s, values %s, N=%d A=%d CH=%d Ef=%d; N <= 127 and the counts lie "
              "in 1..255)", table ? "given" : "null", values ? "given" : "null", N, n_atom_types, n_charges, Ef);
    return -1;
  }
  const int A = n_atom_types, CH = n_charges;
  const int* v = values;
  const int min_atoms = v[GIB_CONS_MIN_ATOMS], max_atoms = v[GIB_CONS_MAX_ATOMS];
  const int min_rings = v[GIB_CONS_MIN_RINGS], max_rings = v[GIB_CONS_MAX_RINGS], ring = v[GIB_CONS_MIN_RING_SIZE];
  const int* min_type = v + GIB_CONS_HDR_INTS;
  const int* max_type = min_type + A;
  const int* rest = max_type + A;           // max_charge [CH], max_bond [Ef]
  const char* why = nullptr;
  int idx = -1;
  long long sum_min = 0;
  if (min_atoms < 0 || min_rings < 0 || ring < 0) why = "a minimum or min_ring_size is negative";
  else if (max_atoms < -1 || max_rings < -1) why = "a maximum is below -1 (-1 = off)";
  else if (max_atoms > N) why = "max_atoms is over max_n_nodes";
  else if (min_atoms > N) why = "min_atoms is over max_n_nodes";
  else if (max_atoms >= 0 && min_atoms > max_atoms) why = "min_atoms is over max_atoms";
  else if (max_rings >= 0 && min_rings > max_rings) why = "min_rings is over max_rings";
  else if (ring == 1 || ring == 2) why = "min_ring_size is 1 or 2 (0 = off, a ring has at least 3 atoms)";
  for (int t = 0; t < A && !why; ++t) {
    idx = t;
    if (min_type[t] < 0) why = "min_type is negative";
    else if (max_type[t] < -1) why = "max_type is below -1 (-1 = off)";
    else if (max_type[t] >= 0 && min_type[t] > max_type[t]) why = "min_type is over max_type";
    sum_min += min_type[t];
  }
  for (int c = 0; c < CH + Ef && !why; ++c) {
    idx = c < CH ? c : c - CH;
    if (rest[c] < -1) why = c < CH ? "max_charge is below -1 (-1 = off)" : "max_bond is below -1 (-1 = off)";
  }
  if (!why && sum_min > (max_atoms >= 0 ? max_atoms : N)) {
    idx = -1;
    why = "the per-type minima add up to more atoms than max_atoms (or max_n_nodes)";
  }
  if (why) {
    set_error("gib_constraints_set: refused: %s (index %d; min_atoms=%d max_atoms=%d min_rings=%d max_rings=%d "
              "min_ring_size=%d, N=%d)", why, idx, min_atoms, max_atoms, min_rings, max_rings, ring, N);
    return -1;
  }
  // staged copy with the layout words filled in; pageable source: the call returns once the value is staged
  int staged[GIB_CONS_HDR_INTS + 2 * 255 + 255 + 255];
  for (size_t i = 0; i < len; ++i) staged[i] = v[i];
  staged[GIB_CONS_N_ATOM_TYPES] = A;
  staged[GIB_CONS_N_CHARGES] = CH;
  staged[GIB_CONS_N_BOND_TYPES] = Ef;
  GIB_CUDA_TRY(cudaMemcpyAsync(table, staged, len * sizeof(int), cudaMemcpyHostToDevice,
                               reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

extern "C" int gib_constraints_check(int M, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                     int n_chirality, int mode, const int* table, const float* nodes,
                                     const float* edges, const signed char* nodes_i8, const signed char* edges_i8,
                                     const int* n_nodes, const gib_scaffolds* sc, const int* scaffold_ids,
                                     const int* constraints, int* flags, gib_stream stream) {
  if (M == 0) return 0;
  const long long apd = layout_apd(N, Ef, n_atom_types, n_charges, n_imp_H > 0 ? n_imp_H : 0,
                                   n_chirality > 0 ? n_chirality : 0);
  gib_scaffolds scv;
  GIB_TRY(check_mask_args("gib_constraints_check", M, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality,
                          (int)apd, mode, table, nodes, edges, nodes_i8, edges_i8, sc, scaffold_ids, &scv));
  if (!constraints || !flags) {
    set_error("gib_constraints_check: the constraint table and the flags must be given");
    return -1;
  }
  const ActionLayout L{N, n_atom_types, n_charges, n_imp_H, n_chirality, Ef};
  const int valence = mode == GIB_ACTION_MASK_VALENCE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (nodes && edges)
    constraints_check_kernel<float><<<M, 128, 0, st>>>(L, F, (int)apd, valence, table, nodes, edges, n_nodes, scv,
                                                       scaffold_ids, constraints, flags);
  else
    constraints_check_kernel<signed char><<<M, 128, 0, st>>>(L, F, (int)apd, valence, table, nodes_i8, edges_i8,
                                                             n_nodes, scv, scaffold_ids, constraints, flags);
  GIB_LAUNCH_CHECK();
  return 0;
}
extern "C" int gib_generation_round(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int round,
                                    const int* action, const float* likelihood, float* nodes, float* edges,
                                    int* n_nodes, float* likelihoods, float* gen_nodes, float* gen_edges,
                                    signed char* gen_n_nodes, float* gen_likelihoods,
                                    signed char* properly_terminated, int capacity, int* counters, void* scratch,
                                    gib_stream stream) {
  return gib_generation_round_layout(B, N, F, Ef, n_atom_types, n_charges, 0, 0, round, action, likelihood, nodes,
                                     edges, n_nodes, likelihoods, gen_nodes, gen_edges, gen_n_nodes, gen_likelihoods,
                                     properly_terminated, capacity, counters, scratch, stream);
}

extern "C" size_t gib_generation_scratch_bytes(int B) { return (size_t)B * (sizeof(int4) + 2 * sizeof(int)) + 64; }

// ---- the sample rounds under a sampling policy (sampling.cu); policy = null: the entry points above ----
extern "C" int gib_generation_sample_round_policy(int B, int N, int F, int Ef, int n_atom_types, int n_charges,
                                                  int n_imp_H, int n_chirality, const float* logits, int apd,
                                                  const float* uniforms, int* state, int* action, float* likelihood,
                                                  float* nodes, float* edges, int* n_nodes, float* likelihoods,
                                                  float* gen_nodes, float* gen_edges, signed char* gen_n_nodes,
                                                  float* gen_likelihoods, signed char* properly_terminated,
                                                  int capacity, int* counters, void* scratch, gib_stream stream,
                                                  const gib_sampling_policy* policy) {
  return sample_round(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, nullptr, logits, apd, uniforms,
                      state, action, likelihood, nodes, edges, n_nodes, likelihoods, gen_nodes, gen_edges,
                      gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters, scratch, stream, policy);
}

extern "C" int gib_generation_sample_round_scaffold_policy(
    int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H, int n_chirality,
    const gib_scaffolds* sc, const float* logits, int apd, const float* uniforms, int* state, int* action,
    float* likelihood, float* nodes, float* edges, int* n_nodes, float* likelihoods, float* gen_nodes,
    float* gen_edges, signed char* gen_n_nodes, float* gen_likelihoods, signed char* properly_terminated,
    int capacity, int* counters, void* scratch, gib_stream stream, const gib_sampling_policy* policy) {
  GIB_TRY(check_scaffolds("gib_generation_sample_round_scaffold_policy", sc));
  return sample_round(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, sc, logits, apd, uniforms, state,
                      action, likelihood, nodes, edges, n_nodes, likelihoods, gen_nodes, gen_edges, gen_n_nodes,
                      gen_likelihoods, properly_terminated, capacity, counters, scratch, stream, policy);
}

extern "C" int gib_rl_sample_round_policy(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                          int n_chirality, const float* logits_a, const float* logits_b, int apd,
                                          const float* uniforms, const int* actions, int* state, int* act_rec,
                                          float* p_a, float* p_b, int* action, float* tags, float* nodes,
                                          float* edges, int* n_nodes, float* likelihoods, float* gen_nodes,
                                          float* gen_edges, signed char* gen_n_nodes, float* gen_likelihoods,
                                          signed char* properly_terminated, int capacity, int* counters,
                                          void* scratch, gib_stream stream, const gib_sampling_policy* policy) {
  return rl_sample_round(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, nullptr, logits_a, logits_b, apd,
                         uniforms, actions, state, act_rec, p_a, p_b, action, tags, nodes, edges, n_nodes, likelihoods,
                         gen_nodes, gen_edges, gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters,
                         scratch, stream, policy);
}

extern "C" int gib_rl_sample_round_scaffold_policy(
    int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H, int n_chirality,
    const gib_scaffolds* sc, const float* logits_a, const float* logits_b, int apd, const float* uniforms,
    const int* actions, int* state, int* act_rec, float* p_a, float* p_b, int* action, float* tags, float* nodes,
    float* edges, int* n_nodes, float* likelihoods, float* gen_nodes, float* gen_edges, signed char* gen_n_nodes,
    float* gen_likelihoods, signed char* properly_terminated, int capacity, int* counters, void* scratch,
    gib_stream stream, const gib_sampling_policy* policy) {
  GIB_TRY(check_scaffolds("gib_rl_sample_round_scaffold_policy", sc));
  return rl_sample_round(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, sc, logits_a, logits_b, apd,
                         uniforms, actions, state, act_rec, p_a, p_b, action, tags, nodes, edges, n_nodes, likelihoods,
                         gen_nodes, gen_edges, gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters,
                         scratch, stream, policy);
}
