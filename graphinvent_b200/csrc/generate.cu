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
#include "../../include/gib200.h"
#include "common.cuh"
#include "ops.cuh"

namespace gib {

// H / C = implicit-H / chirality index counts, 0 = segment absent; Lw = likelihood columns (2 * max_n_nodes)
struct GenDims { int B, N, F, Ef, A, CH, H, C, Lw; };

enum : int { ACT_ADD = 0, ACT_CONN = 1, ACT_TERM = 2 };

// per slot: decoded action + validity  (one thread per slot)
__global__ void gen_decode_kernel(GenDims d, const int* __restrict__ action, const float* __restrict__ edges,
                                  const int* __restrict__ n_nodes, int4* __restrict__ rec, int* __restrict__ flags,
                                  const int* __restrict__ ctl) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= d.B || (ctl && ctl[0] < 0)) return;
  const int a = action[b];
  const int n = n_nodes[b];
  const int len_add = d.N * d.A * d.CH * max(d.H, 1) * max(d.C, 1) * d.Ef, len_conn = d.N * d.Ef;
  int kind, bond_to = 0, atom = 0, charge = 0, imp_h = 0, chir = 0, btype = 0, bond_from = 0, invalid = 0;
  if (a < 0 || a > len_add + len_conn) {
    // not an APD index (a corrupted replay trace, or the sampler's NaN fallback): an invalid action that edits
    // nothing -- the slot terminates as "invalid" and is reset, no field of `rec` is out of range
    kind = ACT_TERM;
    invalid = 1;
  } else if (a < len_add) {
    kind = ACT_ADD;
    int r = a;
    btype = r % d.Ef;
    r /= d.Ef;
    if (d.C) { chir = r % d.C; r /= d.C; }
    if (d.H) { imp_h = r % d.H; r /= d.H; }
    charge = r % d.CH;
    r /= d.CH;
    atom = r % d.A;
    bond_to = r / d.A;
    bond_from = n;
    const bool empty = n == 0;
    if (!empty && bond_to >= n) invalid = 1;          // bond to a non-existing atom          (:600-604)
    if (empty && bond_to != 0) invalid = 1;           // first atom must use slot 0           (:606-610)
    // f_add_idc[5]: bond_from (L0), bond_type (L1, L2) or chirality (L3)
    const int e5_sel = (d.H == 0 && d.C == 0) ? 0 : (d.H && d.C) ? 2 : 1;
    const int e5 = e5_sel == 0 ? bond_from : e5_sel == 2 ? chir : btype;
    const bool madd = e5 >= d.N;
    if (madd) invalid = 1;                            // "graph already holds max_n_nodes atoms" (:618)
    if (madd || empty) {                              // get_actions: f_add_idc[5][max_node_idc] = 0   (:568)
      if (e5_sel == 0) bond_from = 0;
      else if (e5_sel == 2) chir = 0;
      else btype = 0;
    }
    if (n >= d.N) { invalid = 1; bond_from = 0; }     // full graph: the L0 outcome in every layout (see above)
  } else if (a < len_add + len_conn) {
    kind = ACT_CONN;
    const int c = a - len_add;
    btype = c % d.Ef;
    bond_to = c / d.Ef;
    bond_from = n - 1;
    if (bond_to >= n) invalid = 1;                    // (:616)
    if (n == 0) invalid = 1;                          // (:619)
    if (bond_to == bond_from) invalid = 1;            // self loop (:622)
    const int bf = bond_from < 0 ? bond_from + d.N : bond_from;   // Python negative index
    const float* e = edges + (((size_t)b * d.N + bond_to) * d.N + bf) * d.Ef;
    float s = 0.f;
    for (int t = 0; t < d.Ef; ++t) s += e[t];
    if (s == 1.f) invalid = 1;                        // bond already present (:625-629)
    bond_from = bf;
  } else {
    kind = ACT_TERM;
  }
  rec[b] = make_int4(kind | (invalid << 4), bond_to | (bond_from << 8), atom | (charge << 8),
                     btype | (imp_h << 8) | (chir << 16));
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
                                                        int rounds) {
  __shared__ int s_cnt[2][1024];
  __shared__ int s_tot[3];
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
  __syncthreads();
  if (threadIdx.x == 0) {   // fixed-order serial prefix over 1024 partials (tiny)
    int run = 0;
    for (int i = 0; i < 1024; ++i) { int v = s_cnt[0][i]; s_cnt[0][i] = run; run += v; }
    s_tot[0] = run;
    int run2 = 0;
    for (int i = 0; i < 1024; ++i) { int v = s_cnt[1][i]; s_cnt[1][i] = run2; run2 += v; }
    s_tot[1] = run2;
    s_tot[2] = counters[0];
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
  // properly_terminated[k : k + len(term)] = 1, where len(term) counts the dummy slot too (build_graphs :127)
  const int n_term_all = n_term + ((B > 0 && (flags[0] & 1)) ? 1 : 0);
  for (int i = threadIdx.x; i < n_term_all; i += 1024)
    if (k + i < cap) properly_terminated[k + i] = 1;
  if (threadIdx.x == 0) {
    counters[1] = n_term + n_inv;
    counters[0] = k + n_term + n_inv;
    if (ctl) {                        // build_graphs' loop rule: round 2N would be needed -> status 1 (round limit)
      const int next = ctl[0] + 1;
      state[0] = next;
      if (k + n_term + n_inv < B && next >= rounds) state[1] = 1;
    }
  }
}

// one CTA per slot: copy-out (pre-action state), apply the action, reset, re-stamp the dummy graph
__global__ void __launch_bounds__(128) gen_apply_kernel(GenDims d, int round, const int4* __restrict__ rec,
                                                        const int* __restrict__ pos, const float* __restrict__ lik,
                                                        float* __restrict__ nodes, float* __restrict__ edges,
                                                        int* __restrict__ n_nodes, float* __restrict__ likelihoods,
                                                        float* __restrict__ g_nodes, float* __restrict__ g_edges,
                                                        signed char* __restrict__ g_n_nodes,
                                                        float* __restrict__ g_lik, const int* __restrict__ ctl) {
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
    for (int i = threadIdx.x; i < NF; i += 128) nb[i] = 0.f;          // reset_graphs :447-460
    for (int i = threadIdx.x; i < NNE; i += 128) eb[i] = 0.f;
    for (int i = threadIdx.x; i < d.Lw; i += 128) lb[i] = 0.f;
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
                        cudaStream_t st) {
  const int B = d.B;
  int4* rec = reinterpret_cast<int4*>(scratch);
  int* flags = reinterpret_cast<int*>(rec + B);
  int* pos = flags + B;
  gen_decode_kernel<<<ceil_div(B, 128), 128, 0, st>>>(d, action, edges, n_nodes, rec, flags, ctl);
  GIB_LAUNCH_CHECK();
  gen_scan_kernel<<<1, 1024, 0, st>>>(B, flags, pos, counters, properly_terminated, capacity, ctl, state, d.Lw);
  GIB_LAUNCH_CHECK();
  gen_apply_kernel<<<B, 128, 0, st>>>(d, round, rec, pos, likelihood, nodes, edges, n_nodes, likelihoods, gen_nodes,
                                      gen_edges, gen_n_nodes, gen_likelihoods, ctl);
  GIB_LAUNCH_CHECK();
  return 0;
}

static int* round_ctl(void* scratch, int B) {
  return reinterpret_cast<int*>(reinterpret_cast<int4*>(scratch) + B) + 2 * B;   // behind rec, flags and pos
}

extern "C" int gib_generation_round_layout(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                           int n_chirality, int round, const int* action, const float* likelihood,
                                           float* nodes, float* edges, int* n_nodes, float* likelihoods,
                                           float* gen_nodes, float* gen_edges, signed char* gen_n_nodes,
                                           float* gen_likelihoods, signed char* properly_terminated, int capacity,
                                           int* counters, void* scratch, gib_stream stream) {
  GIB_TRY(check_round_args(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, round));
  GenDims d{B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, 2 * N};
  return launch_round(d, round, nullptr, nullptr, action, likelihood, nodes, edges, n_nodes, likelihoods, gen_nodes,
                      gen_edges, gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters, scratch,
                      reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int gib_generation_sample_round(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                           int n_chirality, const float* logits, int apd, const float* uniforms,
                                           int* state, int* action, float* likelihood, float* nodes, float* edges,
                                           int* n_nodes, float* likelihoods, float* gen_nodes, float* gen_edges,
                                           signed char* gen_n_nodes, float* gen_likelihoods,
                                           signed char* properly_terminated, int capacity, int* counters,
                                           void* scratch, gib_stream stream) {
  GIB_TRY(check_round_args(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, 0));
  const long long want = (long long)N * n_atom_types * n_charges * (n_imp_H ? n_imp_H : 1) *
                         (n_chirality ? n_chirality : 1) * Ef + (long long)N * Ef + 1;
  if (apd != want) {
    set_error("gib_generation_round: apd=%d, the action layout (N=%d A=%d CH=%d H=%d C=%d Ef=%d) has %lld actions",
              apd, N, n_atom_types, n_charges, n_imp_H, n_chirality, Ef, want);
    return -1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  GenDims d{B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, 2 * N};
  int* ctl = round_ctl(scratch, B);
  const RoundGate gate{state, counters, ctl, 2 * N};
  GIB_TRY(sample_actions_launch(logits, B, apd, uniforms, action, likelihood, &gate, st));
  return launch_round(d, 0, ctl, state, action, likelihood, nodes, edges, n_nodes, likelihoods, gen_nodes, gen_edges,
                      gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters, scratch, st);
}

extern "C" int gib_rl_sample_round(int B, int N, int F, int Ef, int n_atom_types, int n_charges, int n_imp_H,
                                   int n_chirality, const float* logits_a, const float* logits_b, int apd,
                                   const float* uniforms, const int* actions, int* state, int* act_rec, float* p_a,
                                   float* p_b, int* action, float* tags, float* nodes, float* edges, int* n_nodes,
                                   float* likelihoods, float* gen_nodes, float* gen_edges, signed char* gen_n_nodes,
                                   float* gen_likelihoods, signed char* properly_terminated, int capacity,
                                   int* counters, void* scratch, gib_stream stream) {
  GIB_TRY(check_round_args(B, N, F, Ef, n_atom_types, n_charges, n_imp_H, n_chirality, 0));
  const long long want = (long long)N * n_atom_types * n_charges * (n_imp_H ? n_imp_H : 1) *
                         (n_chirality ? n_chirality : 1) * Ef + (long long)N * Ef + 1;
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
  GIB_TRY(sample_actions_launch(logits_a, B, apd, uniforms, action, tags, &gate, st));
  GIB_TRY(rl_probs_launch(logits_a, logits_b, B, apd, action, ctl, act_rec, p_a, p_b, tags, st));
  return launch_round(d, 0, ctl, state, action, tags, nodes, edges, n_nodes, likelihoods, gen_nodes, gen_edges,
                      gen_n_nodes, gen_likelihoods, properly_terminated, capacity, counters, scratch, st);
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
