// Whole-model forward / backward orchestration for the four GraphINVENT MPNNs that construct
// in the reference (GGNN, MNN, AttentionGGNN, EMN).  Host code only: it sequences the kernels
// of gemm_*.cu / graph_ops.cu on one stream, with every buffer carved out of caller-provided
// workspaces by a deterministic bump layout (no allocation, no host sync).
//
// Reference call sites replaced:
//   SummationMPNN.forward    gnn/summation_mpnn.py:80-149   (GGNN mpnn.py:229-303, MNN mpnn.py:16-74)
//   AggregationMPNN.forward  gnn/aggregation_mpnn.py:83-168 (AttentionGGNN mpnn.py:306-398)
//   EdgeMPNN.forward         gnn/edge_mpnn.py:82-192        (EMN mpnn.py:401-494)
//   GraphGather / GlobalReadout gnn/modules.py:39-52, 237-281
//   and the autograd backward of all of them (Workflow.py:794).
#include <vector>

#include "../../include/gib200.h"
#include "gemm.cuh"
#include "model.cuh"
#include "ops.cuh"

namespace gib {

// ------------------------------------------------------------------------------------
// plan: parameter table + packed-arena layout
// ------------------------------------------------------------------------------------
static void finish_lin(Plan& pl, Lin& l) {
  l.Rbp = pad16(l.Rb);
  l.Rp = l.nblk * l.Rbp;
  l.Cp = pad16(l.C);
  l.Ctp = pad16(l.Ct);
  l.ow = pl.packed_floats;  pl.packed_floats += (size_t)l.Rp * l.Cp;
  l.owt = pl.packed_floats; pl.packed_floats += (size_t)l.Ctp * l.Rp;
  l.ob = pl.packed_floats;  pl.packed_floats += (size_t)l.Rp;
  pl.packed_floats = (pl.packed_floats + 31) & ~(size_t)31;
  l.ow_hi = pl.packed_floats;  pl.packed_floats += (size_t)l.Rp * l.Cp;
  l.ow_lo = pl.packed_floats;  pl.packed_floats += (size_t)l.Rp * l.Cp;
  l.owt_hi = pl.packed_floats; pl.packed_floats += (size_t)l.Ctp * l.Rp;
  l.owt_lo = pl.packed_floats; pl.packed_floats += (size_t)l.Ctp * l.Rp;
  pl.packed_floats = (pl.packed_floats + 31) & ~(size_t)31;
}

static Mlp add_mlp(Plan& pl, int fin, int hidden, int depth, int fout, int ct_first = -1) {
  Mlp m;
  m.first = (int)pl.lins.size();
  m.n = depth + 1;
  m.act = ACT_SELU;
  int in = fin;
  for (int li = 0; li <= depth; ++li) {
    const int out = (li == depth) ? fout : hidden;
    Lin l{};
    l.pw = (int)pl.param_numel.size();
    pl.param_numel.push_back((long long)out * in);
    l.pb = (int)pl.param_numel.size();
    pl.param_numel.push_back(out);
    l.R = out; l.C = in; l.nblk = 1; l.Rb = out; l.rs = in; l.cs = 1; l.src_off = 0;
    l.Ct = (li == 0 && ct_first >= 0) ? ct_first : in;
    finish_lin(pl, l);
    pl.lins.push_back(l);
    in = out;
  }
  return m;
}

static void add_gru(Plan& pl, int in, int H) {
  const int base = (int)pl.param_numel.size();
  pl.param_numel.push_back((long long)3 * H * in);  // weight_ih
  pl.param_numel.push_back((long long)3 * H * H);   // weight_hh
  pl.param_numel.push_back(3 * H);                  // bias_ih
  pl.param_numel.push_back(3 * H);                  // bias_hh
  Lin a{};
  a.pw = base; a.pb = base + 2; a.R = 3 * H; a.C = in; a.nblk = 3; a.Rb = H; a.rs = in; a.cs = 1; a.Ct = in;
  finish_lin(pl, a);
  pl.gru_ih = (int)pl.lins.size();
  pl.lins.push_back(a);
  Lin b{};
  b.pw = base + 1; b.pb = base + 3; b.R = 3 * H; b.C = H; b.nblk = 3; b.Rb = H; b.rs = H; b.cs = 1; b.Ct = H;
  finish_lin(pl, b);
  pl.gru_hh = (int)pl.lins.size();
  pl.lins.push_back(b);
}

int build_plan(const gib_dims& d, Plan& pl) {
  pl = Plan();
  pl.d = d;
  if (d.model < 0 || d.model > 3 || d.Ef < 1 || d.Ef > 4 || d.T < 1 || d.T > kMaxPasses || d.N < 1 || d.F < 1 ||
      d.H < 1 || d.M < 1 || d.f_add < 1 || d.f_conn < 1) {
    set_error("build_plan: unsupported dims (model=%d Ef=%d T=%d; need 1 <= n_edge_features <= 4, "
              "1 <= message_passes <= %d)", d.model, d.Ef, d.T, kMaxPasses);
    return -1;
  }
  // an MLP of depth k has k + 1 Linears; the chained backward keeps one gradient buffer per layer (BwdBufs::Gl)
  const int depths[7] = {d.mlp1_depth, d.mlp2_depth, d.msg_depth, d.att_depth, d.gatt_depth, d.gemb_depth, d.eemb_depth};
  for (int k : depths)
    if (k < 0 || k > 7) {
      set_error("build_plan: MLP depth %d unsupported (need 0 <= depth <= 7)", k);
      return -1;
    }
  if (d.model != GIB_EMN && d.H < d.F) {
    set_error("build_plan: hidden_node_features (%d) < n_node_features (%d)", d.H, d.F);
    return -1;
  }
  const int H = d.H, M = d.M, F = d.F, Ef = d.Ef, N = d.N;
  pl.Hp = pad16(H); pl.Mp = pad16(M);
  if (d.model == GIB_MNN) {
    const int pw = (int)pl.param_numel.size();
    pl.param_numel.push_back((long long)M * H * Ef);  // message_weights [msg, H, Ef]
    for (int t = 0; t < Ef; ++t) {
      Lin l{};
      l.pw = pw; l.pb = -1; l.R = M; l.C = H; l.nblk = 1; l.Rb = M; l.rs = (long long)H * Ef; l.cs = Ef;
      l.src_off = t; l.Ct = H;
      finish_lin(pl, l);
      pl.msg[t].first = (int)pl.lins.size(); pl.msg[t].n = 1; pl.msg[t].act = ACT_NONE;
      pl.lins.push_back(l);
    }
    add_gru(pl, M, H);
    pl.G = H;
  } else if (d.model == GIB_GGNN || d.model == GIB_ATTGGNN) {
    for (int t = 0; t < Ef; ++t) pl.msg[t] = add_mlp(pl, H, d.msg_hidden, d.msg_depth, M);
    if (d.model == GIB_ATTGGNN)
      for (int t = 0; t < Ef; ++t) pl.att[t] = add_mlp(pl, H, d.att_hidden, d.att_depth, M);
    add_gru(pl, M, H);
    pl.gatt = add_mlp(pl, H + F, d.gatt_hidden, d.gatt_depth, d.gather_width, /*ct_first=*/H);
    pl.gemb = add_mlp(pl, H, d.gemb_hidden, d.gemb_depth, d.gather_width);
    pl.G = d.gather_width;
  } else {  // EMN: H = M = edge_emb_size
    pl.embnn = add_mlp(pl, 2 * F + Ef, d.eemb_hidden, d.eemb_depth, H, /*ct_first=*/0);
    pl.emsg = add_mlp(pl, H, d.msg_hidden, d.msg_depth, H);
    pl.eatt = add_mlp(pl, H, d.att_hidden, d.att_depth, H);
    add_gru(pl, H, H);
    pl.gatt = add_mlp(pl, 2 * H, d.gatt_hidden, d.gatt_depth, d.gather_width);
    pl.gemb = add_mlp(pl, H, d.gemb_hidden, d.gemb_depth, d.gather_width);
    pl.G = d.gather_width;
  }
  pl.Gp = pad16(pl.G);
  pl.fadd1 = add_mlp(pl, H, d.mlp1_hidden, d.mlp1_depth, d.f_add);
  pl.fconn1 = add_mlp(pl, H, d.mlp1_hidden, d.mlp1_depth, d.f_conn);
  pl.fadd2 = add_mlp(pl, N * d.f_add + pl.G, d.mlp2_hidden, d.mlp2_depth, N * d.f_add);
  pl.fconn2 = add_mlp(pl, N * d.f_conn + pl.G, d.mlp2_hidden, d.mlp2_depth, N * d.f_conn);
  pl.fterm2 = add_mlp(pl, pl.G, d.mlp2_hidden, d.mlp2_depth, 1);
  pl.apd = N * d.f_add + N * d.f_conn + 1;
  // checked here rather than at packing time, so that every size query refuses such a model with the same message
  if ((int)pl.lins.size() > kMaxPackEntries) {
    set_error("build_plan: %d Linears exceed the packing descriptor table (at most %d Linears)", (int)pl.lins.size(),
              kMaxPackEntries);
    return -1;
  }
  return 0;
}

int pack_params(const Plan& pl, const float* const* params, float* packed, int prec, cudaStream_t st) {
  GIB_TRY(check_precision(prec, "gib_model_pack"));
  {   // one launch for the whole model (52-67 Linears at the reference's defaults, at most kMaxPackEntries)
    PackTable T;
    T.n = (int)pl.lins.size();
    T.h16 = prec >= 2 ? prec - 1 : 0;
    unsigned blk = 0;
    for (int i = 0; i < T.n; ++i) {
      const Lin& l = pl.lins[i];
      PackEntry& e = T.e[i];
      e.W = params[l.pw] + l.src_off;
      e.bias = l.pb >= 0 ? params[l.pb] : nullptr;
      e.rs = l.rs; e.cs = l.cs; e.ow = (long long)l.ow; e.owt = (long long)l.owt; e.ob = (long long)l.ob;
      e.ow_hi = (long long)l.ow_hi; e.ow_lo = (long long)l.ow_lo; e.owt_hi = (long long)l.owt_hi; e.owt_lo = (long long)l.owt_lo;
      e.nblk = l.nblk; e.Rb = l.Rb; e.Rbp = l.Rbp; e.C = l.C; e.Cp = l.Cp; e.Ct = l.Ct; e.Ctp = l.Ctp;
      e.blk_begin = blk;
      const long long tot = (long long)l.Rp * l.Cp + (long long)l.Ctp * l.Rp + l.Rp;
      blk += (unsigned)ceil_div_ll(tot, 1024);
    }
    T.total_blocks = blk;
    return pack_all(T, packed, st);
  }
  return 0;
}

// ------------------------------------------------------------------------------------
// run context + layouts
// ------------------------------------------------------------------------------------
struct Bump {
  size_t off = 0;
  size_t take(size_t nfloats) {
    size_t o = off;
    off += (nfloats + 31) & ~(size_t)31;  // keep every buffer 128-byte aligned
    return o;
  }
};

// counters of one dependent-chain launch: <= kTc3MaxProblems problems x (row blocks + 1)
static size_t chain_flag_floats(size_t max_rows) { return (size_t)kTc3MaxProblems * (max_rows / 128 + 2); }

static void mlp_act_layout(const Plan& pl, const Mlp& m, size_t rows, Bump& bp, MlpAct& a, bool last_external) {
  for (int l = 1; l <= m.n; ++l) {
    const Lin& L = pl.lins[m.first + l - 1];
    a.ld[l] = L.Rp;
    a.y[l] = (l == m.n && last_external) ? (size_t)-1 : bp.take(rows * L.Rp);
  }
}

size_t graph_buf_ints(long long S, int E, int P) {
  // ent_src[P] ent_dst[P] ent_w[P] dst_ptr[S+1] dst_ent[E] src_ptr[S+1] src_ent[E], each 128B aligned
  auto al = [](long long n) { return (size_t)((n + 31) & ~31LL); };
  return 3 * al(P) + 2 * al(S + 1) + 2 * al(E);
}
GraphArrays graph_arrays(void* buf, long long S, int E, int P) {
  auto al = [](long long n) { return (size_t)((n + 31) & ~31LL); };
  int* p = reinterpret_cast<int*>(buf);
  GraphArrays ga;
  ga.ent_src = p; p += al(P);
  ga.ent_dst = p; p += al(P);
  ga.ent_w = reinterpret_cast<float*>(p); p += al(P);
  ga.dst_ptr = p; p += al(S + 1);
  ga.dst_ent = p; p += al(E);
  ga.src_ptr = p; p += al(S + 1);
  ga.src_ent = p;
  return ga;
}

// Exact mode: would the message MLPs on the entry groups' host row counts run on the tensor-core kernels (a chain of all
// layers, or one grouped launch per layer; mlp_forward_multi / gemm_nt_group)?  Only then do the message rows run on
// their device-side counts -- the same kernels, so the logits stay those of the per-entry path to the bit; otherwise
// (tensor cores off, small batches on the fp32 SIMT kernel) they run on the entry groups' host ranges, pad rows included.
static bool msg_mlp_on_tc3(const Run& r) {
  if (!g_use_tc || (g_tc_debug & 1)) return false;
  const Plan& pl = r.pl;
  const int depth = pl.msg[0].n, n = r.ngroups;
  const bool chain = depth >= 2 && depth * n <= kTc3MaxProblems && (g_tc_debug & 2) == 0;
  long long chain_tiles = 0;
  for (int l = 0; l < depth; ++l) {
    long long tiles = 0;
    int live = 0, big = 0;
    for (int g = 0; g < n; ++g) {
      const Lin& L = pl.lins[pl.msg[g].first + l];
      const int M = r.tc[g];
      if (M <= 0) continue;
      if (L.Rp < 48 || L.Cp < 32) return false;
      tiles += (long long)ceil_div(M, 128) * ceil_div(L.Rp, 128);
      ++live;
      big += M >= 256;
    }
    chain_tiles += tiles;
    if (!chain && !(live > 1 ? tiles >= 4 || big == live : big == live)) return false;
  }
  return !chain || chain_tiles >= 16;
}

int make_run(const gib_dims& d, const int* hdr, Run& r) {
  GIB_TRY(build_plan(d, r.pl));
  r.tf32 = d.tf32;
  r.E = hdr[HDR_E];
  r.P = hdr[HDR_P];
  const int G = d.model == GIB_EMN ? 1 : d.Ef;
  r.cap = hdr[HDR_CAPACITY] != 0;
  r.dev_hdr = nullptr;
  if (r.cap) {
    // capacity header (gib_graph_header_capacity): E / P are static capacities, the live counts stay in device memory;
    // every bond-type group is planned with the whole capacity and located through the device header at run time
    // (EMN: one untyped group, its bond rows [0, TYPE_COUNT[0]) of buffers of E rows)
    unsigned long long a = (unsigned)hdr[HDR_DEV_LO] | ((unsigned long long)(unsigned)hdr[HDR_DEV_HI] << 32);
    r.dev_hdr = reinterpret_cast<const int*>(a);
    if (!r.dev_hdr) { set_error("capacity header without a device header address"); return -1; }
    for (int g = 0; g < 4; ++g) r.tc[g] = g < G ? r.P : 0;
    for (int g = 0; g < 5; ++g) r.tb[g] = 0;
    r.unit_bonds = false;
  } else {
    for (int g = 0; g < 4; ++g) r.tc[g] = g < G ? hdr[HDR_TYPE_COUNT + g] : 0;
    for (int g = 0; g < 5; ++g) r.tb[g] = g <= G ? hdr[HDR_TYPE_BASE + g] : r.P;
    r.unit_bonds = (hdr[HDR_FLAGS] & GRAPH_FLAG_NONBINARY) == 0;   // every bond value is exactly 1: skip the w reads
  }
  r.ngroups = G;
  r.S = (long long)d.B * d.N;
  if (d.B < 1 || r.E < 0 || r.P < r.E) {
    set_error("make_run: inconsistent graph header (B=%d E=%d P=%d)", d.B, r.E, r.P);
    return -1;
  }
  if (!r.cap && (d.model == GIB_ATTGGNN) && (hdr[HDR_FLAGS] & GRAPH_FLAG_MULTITYPE)) {
    // (the reference's AggregationMPNN prologue fails on such input as well: aggregation_mpnn.py:115-141 sizes the
    // neighbour slots by the summed bond VALUES and the index assignment raises a shape mismatch)
    set_error("AttentionGGNN path requires one bond type per bond (a bond with several non-zero types was found)");
    return -3;
  }
  // ---- forward workspace layout ----
  const Plan& pl = r.pl;
  Layout& L = r.L;
  Bump bp;
  const size_t S = (size_t)r.S, P = (size_t)r.P, B = (size_t)d.B;
  const int Hp = pl.Hp, Mp = pl.Mp, Gp = pl.Gp;
  if (d.model != GIB_EMN) {
    for (int t = 0; t <= d.T; ++t) L.h[t] = bp.take(S * Hp);
    for (int t = 0; t < d.T; ++t) {
      L.x0[t] = bp.take(P * Hp);
      L.msg[t].ld[0] = Hp;
      mlp_act_layout(pl, pl.msg[0], P, bp, L.msg[t], false);
      if (d.model == GIB_ATTGGNN) {
        L.att[t].ld[0] = Hp;
        mlp_act_layout(pl, pl.att[0], P, bp, L.att[t], false);
      }
      L.msum[t] = bp.take(S * Mp);
      L.gi[t] = bp.take(S * 3 * Hp);
      L.gh[t] = bp.take(S * 3 * Hp);
    }
    L.hfinal = L.h[d.T];
    if (d.model != GIB_ATTGGNN) {   // reserved whatever gib_tc_debug says: the workspace size does not depend on it
      const size_t E = (size_t)r.E;
      L.mr_src = bp.take(P); L.mr_w = bp.take(P); L.mr_ptr = bp.take(P + 1); L.mr_ent = bp.take(P);
      L.mr_dst = bp.take(E); L.mr_dst_u = bp.take(E); L.mr_su = bp.take(E); L.mr_sptr = bp.take(S + 1);
      L.mr_meta = bp.take(MR_META_INTS); L.mr_tmp = bp.take(msg_rows_tmp_ints(d.B, G));
      r.msg_rows = (g_tc_debug & 8) == 0;
      r.msg_dev_rows = r.msg_rows && (r.cap || msg_mlp_on_tc3(r));
    }
  } else {
    const size_t E = (size_t)r.E;
    L.xin = bp.take(E * pl.lins[pl.embnn.first].Cp);
    L.embnn.ld[0] = pl.lins[pl.embnn.first].Cp;
    mlp_act_layout(pl, pl.embnn, E, bp, L.embnn, false);
    L.xt = bp.take(E * Hp);
    L.emx.ld[0] = Hp; mlp_act_layout(pl, pl.emsg, E, bp, L.emx, false);
    L.enx.ld[0] = Hp; mlp_act_layout(pl, pl.eatt, E, bp, L.enx, false);
    for (int t = 0; t <= d.T; ++t) L.mem[t] = bp.take(E * Hp);
    for (int t = 0; t < d.T; ++t) {
      L.emm[t].ld[0] = Hp; mlp_act_layout(pl, pl.emsg, E, bp, L.emm[t], false);
      L.enm[t].ld[0] = Hp; mlp_act_layout(pl, pl.eatt, E, bp, L.enm[t], false);
      L.emsg[t] = bp.take(E * Hp);
      L.gi[t] = bp.take(E * 3 * Hp);
    }
    L.hfinal = bp.take(S * Hp);
  }
  if (d.model != GIB_MNN) {
    L.cat_att = bp.take(S * pl.lins[pl.gatt.first].Cp);
    L.gatt.ld[0] = pl.lins[pl.gatt.first].Cp;
    mlp_act_layout(pl, pl.gatt, S, bp, L.gatt, false);
    L.gemb.ld[0] = Hp;
    mlp_act_layout(pl, pl.gemb, S, bp, L.gemb, false);
    L.attn = bp.take(S * Gp);
  }
  L.g = bp.take(B * Gp);
  L.fadd1.ld[0] = Hp;  mlp_act_layout(pl, pl.fadd1, S, bp, L.fadd1, false);
  L.fconn1.ld[0] = Hp; mlp_act_layout(pl, pl.fconn1, S, bp, L.fconn1, false);
  L.cat_add = bp.take(B * pl.lins[pl.fadd2.first].Cp);
  L.fadd2.ld[0] = pl.lins[pl.fadd2.first].Cp;
  mlp_act_layout(pl, pl.fadd2, B, bp, L.fadd2, true);
  L.cat_conn = bp.take(B * pl.lins[pl.fconn2.first].Cp);
  L.fconn2.ld[0] = pl.lins[pl.fconn2.first].Cp;
  mlp_act_layout(pl, pl.fconn2, B, bp, L.fconn2, true);
  L.fterm2.ld[0] = Gp;
  mlp_act_layout(pl, pl.fterm2, B, bp, L.fterm2, true);
  L.flags = bp.take(chain_flag_floats(std::max(std::max(S, P), std::max(B, (size_t)r.E))));
  L.total = bp.off;
  return 0;
}

// ------------------------------------------------------------------------------------
// the GEMM problems of one Linear: the only code that reads a Lin's packed-arena offsets
// ------------------------------------------------------------------------------------
// Each problem covers rows [0, rows) of its operands, or with m_dev set (capacity mode, device-side row counts) the
// rows [*base_dev, *base_dev + *m_dev) of buffers of `rows` rows.  work counts the real extents: 2 rows R C (Ct for dX).

// B = the packed copy at `w`, plus the planes the tensor-core kernels read: the TF32 (hi, lo) planes, or in the 16-bit
// modes the 16-bit plane that gib_model_pack writes over the bytes of the lo plane (as B_hi; B_lo unused)
static void set_b(const Run& r, GemmNT& p, size_t w, size_t hi, size_t lo, int ldb) {
  p.B = r.packed + w; p.ldb = ldb;
  p.B_hi = r.packed + (r.tf32 >= 2 ? lo : hi);
  p.B_lo = r.tf32 >= 2 ? nullptr : r.packed + lo;
}

// forward: C = act(X W^T + b), X [rows, Cp] at ld ldx, C [rows, Rp] at ld ldc
static GemmNT lin_fwd(const Run& r, const Lin& L, const float* X, int ldx, int rows, int act, float* C, int ldc,
                      const int* m_dev = nullptr, const int* base_dev = nullptr) {
  GemmNT p;
  p.A = X; p.lda = ldx;
  set_b(r, p, L.ow, L.ow_hi, L.ow_lo, L.Cp);
  p.C = C; p.ldc = ldc;
  p.M = rows; p.N = L.Rp; p.K = L.Cp;
  p.bias = L.pb >= 0 ? r.packed + L.ob : nullptr;
  p.act = act; p.mode = EPI_ACT;
  p.n_store = p.n_valid = L.Rp;
  p.work = 2.0 * rows * (double)L.R * L.C;
  p.m_dev = m_dev; p.base_dev = base_dev; p.tf32 = r.tf32;
  return p;
}

// input gradient: C = G W over the leading Ct input columns, G [rows, Rp], C [rows, Ctp] at ld ldc, stored as is;
// callers switch the epilogue to EPI_MUL_DACT (through the previous layer's activation) or EPI_ADD
static GemmNT lin_dx(const Run& r, const Lin& L, const float* G, int rows, float* C, int ldc,
                     const int* m_dev = nullptr, const int* base_dev = nullptr) {
  GemmNT p;
  p.A = G; p.lda = L.Rp;
  set_b(r, p, L.owt, L.owt_hi, L.owt_lo, L.Rp);
  p.C = C; p.ldc = ldc;
  p.M = rows; p.N = L.Ctp; p.K = L.Rp;
  p.act = ACT_NONE; p.mode = EPI_ACT;
  p.n_store = p.n_valid = L.Ctp;
  p.work = 2.0 * rows * (double)L.R * L.Ct;
  p.m_dev = m_dev; p.base_dev = base_dev; p.tf32 = r.tf32;
  return p;
}

// weight gradient: grads[pw] += G^T X at the Linear's source strides (and grads[pb] += column sums of G), G [rows, Rp],
// X [rows, Cp] at ld ldx, through the dW scratch of bb
static GemmDW lin_dw(const Run& r, const BwdBufs& bb, const Lin& L, const float* G, const float* X, int ldx, int rows,
                     const int* m_dev = nullptr, const int* base_dev = nullptr) {
  GemmDW q;
  q.G = G; q.ldg = L.Rp; q.Nn = L.Rp;
  q.X = X; q.ldx = ldx; q.Kk = L.Cp;
  q.M = rows;
  q.dW = r.grads[L.pw] + L.src_off;
  q.dbias = L.pb >= 0 ? r.grads[L.pb] : nullptr;
  q.R = L.R; q.C = L.C; q.Rb = L.Rb; q.Rbp = L.Rbp; q.rs = L.rs; q.cs = L.cs;
  q.scratch = r.scratch + bb.dw; q.half_floats = bb.dw_half;
  q.work = 2.0 * rows * (double)L.R * L.C;
  q.m_dev = m_dev; q.base_dev = base_dev; q.tf32 = r.tf32;
  return q;
}

// ------------------------------------------------------------------------------------
// MLP forward / backward over a row range
// ------------------------------------------------------------------------------------
// Gtop: gradient w.r.t. the PRE-activation of the last layer, [rows, Rp_last] at Gtop (row 0 = row0).
// dX0 (optional): [rows, ld_dx] ; dx_aux (optional) is added (may alias dX0).
static int mlp_backward(const Run& r, const BwdBufs& bb, const Mlp& m, const float* X0, const MlpAct& a,
                        long long row0, int rows, const float* Gtop, float* dX0, int ld_dx, const float* dx_aux) {
  if (rows <= 0) return 0;
  const float* G = Gtop;
  float* ping = r.scratch + bb.GA;
  float* pong = r.scratch + bb.GB;
  for (int l = m.n; l >= 1; --l) {
    const Lin& L = r.pl.lins[m.first + l - 1];
    const float* Xin = (l == 1) ? X0 + (size_t)row0 * a.ld[0] : r.ws + a.y[l - 1] + (size_t)row0 * a.ld[l - 1];
    const int ldxin = a.ld[l - 1];
    GIB_TRY(gemm_dw(lin_dw(r, bb, L, G, Xin, ldxin, rows), r.st));
    if (l > 1) {
      GemmNT p = lin_dx(r, L, G, rows, (G == ping) ? pong : ping, L.Ctp);
      p.mode = EPI_MUL_DACT; p.act = m.act; p.aux = Xin; p.ldaux = ldxin;
      GIB_TRY(gemm_nt(p, r.st));
      G = p.C;
    } else if (dX0) {
      GemmNT p = lin_dx(r, L, G, rows, dX0, ld_dx);
      if (dx_aux) { p.mode = EPI_ADD; p.aux = dx_aux; p.ldaux = ld_dx; }
      GIB_TRY(gemm_nt(p, r.st));
    }
  }
  // single-layer MLP: the pending side-stream job reads the caller's Gtop buffer -- finish it before returning
  if (m.n == 1) GIB_TRY(dw_join(r.st));
  return 0;
}

// ---- several MLPs of equal depth advanced layer by layer, each layer as ONE grouped GEMM launch --------------
// A job covers rows [row0, row0 + rows) of the activation buffers; X0 points at row 0 of the input buffer.
struct MlpJob {
  const Mlp* m; const float* X0; const MlpAct* a; long long row0; int rows;
  float* ext_out; int ext_ld, ext_valid;
  const int* m_dev = nullptr; const int* base_dev = nullptr;   // capacity mode: live row range on the device
};
struct MlpBwdJob {
  const Mlp* m; const float* X0; const MlpAct* a; long long row0; int rows;
  const float* Gtop; float* dX0; int ld_dx; const float* dx_aux;
  const int* m_dev = nullptr; const int* base_dev = nullptr;
};
static int* fwd_flags(const Run& r) { return reinterpret_cast<int*>(r.ws + r.L.flags); }
static const int* type_count_dev(const Run& r, int g) { return r.cap ? r.dev_hdr + HDR_TYPE_COUNT + g : nullptr; }
static const int* type_base_dev(const Run& r, int g) { return r.cap ? r.dev_hdr + HDR_TYPE_BASE + g : nullptr; }

static MsgRows msg_rows_of(const Run& r) {
  const Layout& L = r.L;
  auto ip = [&](size_t off) { return reinterpret_cast<int*>(r.ws + off); };
  MsgRows mr;
  mr.u_src = ip(L.mr_src); mr.u_w = r.ws + L.mr_w; mr.u_ptr = ip(L.mr_ptr); mr.u_dst = ip(L.mr_dst);
  mr.ent_u = ip(L.mr_ent); mr.dst_u = ip(L.mr_dst_u); mr.s_ptr = ip(L.mr_sptr); mr.s_u = ip(L.mr_su);
  mr.meta = ip(L.mr_meta); mr.tmp = ip(L.mr_tmp);
  return mr;
}
// rows the message MLP of bond type g runs on: [row0, row0 + rows), or on the device-side range inside them
struct MsgRange { long long row0; int rows; const int* m_dev; const int* base_dev; };
static bool msg_dev(const Run& r) { return r.cap || r.msg_dev_rows; }
static MsgRange msg_range(const Run& r, int g) {
  if (r.msg_dev_rows) {
    const int* meta = reinterpret_cast<const int*>(r.ws + r.L.mr_meta);
    return {0, r.P, meta + MR_COUNT + g, meta + MR_BASE + g};
  }
  return {r.tb[g], r.tc[g], type_count_dev(r, g), type_base_dev(r, g)};
}

static size_t mlp_max_ld(const Plan& pl, const Mlp& m) {
  size_t w = 16;
  for (int l = 0; l < m.n; ++l) w = std::max(w, (size_t)std::max(pl.lins[m.first + l].Rp, pl.lins[m.first + l].Cp));
  return w;
}

static int mlp_forward_multi(const Run& r, const MlpJob* jobs, int n, int* flags = nullptr) {
  bool same = n <= 4;
  for (int i = 1; i < n && same; ++i) same = jobs[i].m->n == jobs[0].m->n;
  if (!same) {
    // one call per MLP: on host rows layer by layer, on device-side row counts (grouped call pattern) still as a chain
    for (int i = 0; i < n; ++i) GIB_TRY(mlp_forward_multi(r, jobs + i, 1, jobs[i].m_dev ? flags : nullptr));
    return 0;
  }
  const float* x[4]; int ldx[4];
  for (int i = 0; i < n; ++i) { x[i] = jobs[i].X0 + (size_t)jobs[i].row0 * jobs[i].a->ld[0]; ldx[i] = jobs[i].a->ld[0]; }
  const int depth = jobs[0].m->n;
  GemmNT all[kTc3MaxProblems];
  int dep[kTc3MaxProblems], layer_of[kTc3MaxProblems], last[4] = {-1, -1, -1, -1}, nall = 0;
  const bool try_chain = depth >= 2 && depth * n <= kTc3MaxProblems;
  for (int l = 1; l <= depth; ++l) {
    GemmNT ps[4];
    int np = 0, idx[4];
    for (int i = 0; i < n; ++i) {
      const MlpJob& j = jobs[i];
      if (j.rows <= 0) continue;
      const Lin& L = r.pl.lins[j.m->first + l - 1];
      GemmNT& p = ps[np];
      if (l == j.m->n && j.ext_out) {
        p = lin_fwd(r, L, x[i], ldx[i], j.rows, j.m->act, j.ext_out + (size_t)j.row0 * j.ext_ld, j.ext_ld, j.m_dev,
                    j.base_dev);
        p.n_store = p.n_valid = j.ext_valid;
      } else {
        p = lin_fwd(r, L, x[i], ldx[i], j.rows, j.m->act, r.ws + j.a->y[l] + (size_t)j.row0 * j.a->ld[l], j.a->ld[l],
                    j.m_dev, j.base_dev);
      }
      if (ldx[i] < L.Cp) { set_error("mlp_forward_multi: input ld %d < padded K %d", ldx[i], L.Cp); return -2; }
      idx[np++] = i;
    }
    if (try_chain) {       // collect: the layers of all members become ONE dependent-chain launch below
      for (int k = 0; k < np; ++k) {
        all[nall] = ps[k];
        dep[nall] = last[idx[k]];
        layer_of[nall] = l;
        last[idx[k]] = nall++;
      }
    } else {
      GIB_TRY(gemm_nt_group(ps, np, r.st));
    }
    for (int k = 0; k < np; ++k) { x[idx[k]] = ps[k].C; ldx[idx[k]] = ps[k].ldc; }
  }
  if (try_chain && nall) {
    if (flags && gemm_nt_chain_ok(all, nall)) return gemm_nt_chain(all, dep, nall, flags, r.st);
    // a narrow output layer (the 3 / 39 / 45-wide APD heads) must not cost the hidden layers their chain: the longest
    // prefix of whole layers that qualifies runs as a chain, the rest layer by layer (members of a layer are
    // contiguous in `all`)
    int k0 = 0;
    if (flags) {
      int k = nall;
      while (k > 0 && layer_of[k - 1] >= 3) {              // candidate prefixes: layers 1..l for l = depth-1 .. 2
        const int l = layer_of[k - 1];
        while (k > 0 && layer_of[k - 1] == l) --k;
        if (gemm_nt_chain_ok(all, k)) {
          GIB_TRY(gemm_nt_chain(all, dep, k, flags, r.st));
          k0 = k;
          break;
        }
      }
    }
    while (k0 < nall) {
      int k1 = k0 + 1;
      while (k1 < nall && layer_of[k1] == layer_of[k0]) ++k1;
      GIB_TRY(gemm_nt_group(all + k0, k1 - k0, r.st));
      k0 = k1;
    }
  }
  return 0;
}

// Sibling MLPs whose layers do not all fit one grouped launch (unequal depths, or more than kTc3MaxProblems layers in
// all, e.g. 4 bond types x 5 Linears) run their backward in sub-groups: [i, i + k) is the longest run of members of
// member i's depth that fits.
static int sub_group(const Mlp* const* ms, int n, int i) {
  const int per = std::max(1, kTc3MaxProblems / ms[i]->n);
  int k = 1;
  while (i + k < n && k < per && ms[i + k]->n == ms[i]->n) ++k;
  return k;
}

// Backward of sibling MLPs of equal depth.  Three launches' worth of structure instead of three per layer:
//   (A) the input-gradient GEMMs of layers n..2 (G_{l-1} = (G_l W_l) . selu'(X_{l-1})) as ONE dependent chain,
//       every G_l kept in its own buffer;
//   (B) the weight gradients of ALL layers and members (dW_l = G_l^T X_{l-1}) as ONE grouped launch + ONE reduction;
//   (C) the first layer's input gradient (if wanted).
// plan_rows: expected total rows of the members of ONE layer (capacity mode: the entry capacity the bond-type groups
// share, or n x the capacity for the EMN's siblings, which each span it), 0 = their sum.
// same_rows (capacity mode): the members run on the SAME device row range (the EMN's siblings) and keep one gradient
// slice each; otherwise members with device row ranges are the disjoint bond-type groups of ONE buffer of `rows` rows
// and share one slice.
static int mlp_backward_multi(const Run& r, const BwdBufs& bb, const MlpBwdJob* jobs, int n, long long plan_rows = 0,
                              bool same_rows = false) {
  bool same = n <= 4;
  for (int i = 1; i < n && same; ++i) same = jobs[i].m->n == jobs[0].m->n;
  const int depth = jobs[0].m->n;
  if (!same || depth * n > kTc3MaxProblems) {
    if (jobs[0].m_dev) {
      // device-side row counts need the grouped call pattern: sub-groups that fit one launch, each planned with the
      // whole group's plan rows (make_bwd sizes the same split through group_extent)
      const Mlp* ms[4];
      for (int i = 0; i < n; ++i) ms[i] = jobs[i].m;
      for (int i = 0, k; i < n; i += k) {
        k = sub_group(ms, n, i);
        GIB_TRY(mlp_backward_multi(r, bb, jobs + i, k, plan_rows, same_rows));
      }
      return 0;
    }
    for (int i = 0; i < n; ++i)
      GIB_TRY(mlp_backward(r, bb, *jobs[i].m, jobs[i].X0, *jobs[i].a, jobs[i].row0, jobs[i].rows, jobs[i].Gtop,
                           jobs[i].dX0, jobs[i].ld_dx, jobs[i].dx_aux));
    return 0;
  }
  // G[l][i]: gradient w.r.t. the pre-activation of layer l of member i; G[depth] = the caller's Gtop
  const float* G[9][4];
  size_t off = 0;
  for (int i = 0; i < n; ++i) {
    G[depth][i] = jobs[i].Gtop;
    for (int l = 1; l < depth; ++l) G[l][i] = r.scratch + bb.Gl[l] + off;
    if (!jobs[i].m_dev || same_rows)
      off += ((size_t)std::max(jobs[i].rows, 0) * mlp_max_ld(r.pl, *jobs[i].m) + 31) & ~(size_t)31;
  }
  auto x_in = [&](const MlpBwdJob& j, int l, int* ld) -> const float* {   // input activations of layer l
    *ld = j.a->ld[l - 1];
    return (l == 1) ? j.X0 + (size_t)j.row0 * j.a->ld[0] : r.ws + j.a->y[l - 1] + (size_t)j.row0 * j.a->ld[l - 1];
  };
  // ---- (A) input gradients of layers depth..2 ------------------------------------------------------------------
  GemmNT all[kTc3MaxProblems];
  int dep[kTc3MaxProblems], layer_of[kTc3MaxProblems], last[4] = {-1, -1, -1, -1}, nall = 0;
  for (int l = depth; l >= 2; --l)
    for (int i = 0; i < n; ++i) {
      const MlpBwdJob& j = jobs[i];
      if (j.rows <= 0) continue;
      const Lin& L = r.pl.lins[j.m->first + l - 1];
      int ldxin;
      const float* Xin = x_in(j, l, &ldxin);
      GemmNT& p = all[nall];
      p = lin_dx(r, L, G[l][i], j.rows, const_cast<float*>(G[l - 1][i]), L.Ctp, j.m_dev, j.base_dev);
      p.mode = EPI_MUL_DACT; p.act = j.m->act; p.aux = Xin; p.ldaux = ldxin;
      dep[nall] = last[i];
      layer_of[nall] = l;
      last[i] = nall++;
    }
  if (nall) {
    // the top layer of an APD head reduces over 3 / 39 / 45 columns and does not qualify for the tensor-core chain:
    // leading layers run one by one until the remaining suffix of whole layers qualifies as a chain
    int k0 = 0;
    while (k0 < nall) {
      if (nall - k0 >= 2 && gemm_nt_chain_ok(all + k0, nall - k0)) {
        int dep2[kTc3MaxProblems];
        for (int k = k0; k < nall; ++k) dep2[k - k0] = dep[k] >= k0 ? dep[k] - k0 : -1;   // earlier layers: stream order
        GIB_TRY(gemm_nt_chain(all + k0, dep2, nall - k0, reinterpret_cast<int*>(r.scratch + bb.flags), r.st));
        break;
      }
      int k1 = k0 + 1;
      while (k1 < nall && layer_of[k1] == layer_of[k0]) ++k1;
      GIB_TRY(gemm_nt_group(all + k0, k1 - k0, r.st));
      k0 = k1;
    }
  }
  // ---- (C) input gradient of the first layer (may chain through a shared buffer via aux: keep the members in order)
  for (int i = 0; i < n; ++i) {
    const MlpBwdJob& j = jobs[i];
    if (j.rows <= 0 || !j.dX0) continue;
    GemmNT p1 = lin_dx(r, r.pl.lins[j.m->first], G[1][i], j.rows, j.dX0, j.ld_dx, j.m_dev, j.base_dev);
    if (j.dx_aux) { p1.mode = EPI_ADD; p1.aux = j.dx_aux; p1.ldaux = j.ld_dx; }
    GIB_TRY(gemm_nt(p1, r.st));
  }
  // ---- (B) weight gradients of every layer and member: one grouped launch + one reduction -----------------------
  GemmDW qs[kTc3MaxProblems];
  int nq = 0;
  for (int l = depth; l >= 1; --l)
    for (int i = 0; i < n; ++i) {
      const MlpBwdJob& j = jobs[i];
      if (j.rows <= 0) continue;
      const Lin& L = r.pl.lins[j.m->first + l - 1];
      int ldxin;
      const float* Xin = x_in(j, l, &ldxin);
      qs[nq++] = lin_dw(r, bb, L, G[l][i], Xin, ldxin, j.rows, j.m_dev, j.base_dev);
    }
  GIB_TRY(gemm_dw_group(qs, nq, plan_rows * depth, r.st));
  // the side-stream reduction reads only its scratch half; a first-generation / SIMT fallback job may still read
  // the caller's Gtop buffer: finish it before returning
  if (!(g_use_tc && (g_tc_debug & 1) == 0)) GIB_TRY(dw_join(r.st));
  return 0;
}

// ------------------------------------------------------------------------------------
// readout (GraphGather / sum + GlobalReadout)
// ------------------------------------------------------------------------------------
static int readout_forward(const Run& r, float* out) {
  const gib_dims& d = r.pl.d;
  const Plan& pl = r.pl;
  const Layout& L = r.L;
  const long long S = r.S;
  const int Hp = pl.Hp, Gp = pl.Gp;
  const float* hT = r.ws + L.hfinal;
  if (d.model == GIB_MNN) {
    GIB_TRY(sum_nodes_fwd(r.ws + L.g, hT, Hp, d.N, d.B, r.st));                       // mpnn.py:72
  } else {
    const int ldc = L.gatt.ld[0];
    if (d.model == GIB_EMN) GIB_TRY(concat2(r.ws + L.cat_att, ldc, hT, Hp, d.H, hT, Hp, d.H, S, r.st));
    else GIB_TRY(concat2_in(r.ws + L.cat_att, ldc, hT, Hp, d.H, 0, r.nodes, d.F, d.F, d.in_dtype, S, r.st));  // modules.py:46
    {   // att_nn(cat) and emb_nn(hidden) are independent: one grouped launch per layer
      MlpJob jobs[2] = {{&pl.gatt, r.ws + L.cat_att, &L.gatt, 0, (int)S, nullptr, 0, 0},
                        {&pl.gemb, hT, &L.gemb, 0, (int)S, nullptr, 0, 0}};
      GIB_TRY(mlp_forward_multi(r, jobs, 2, fwd_flags(r)));
    }
    GIB_TRY(graph_gather_fwd(r.ws + L.g, r.ws + L.attn, r.ws + L.gatt.y[pl.gatt.n], r.ws + L.gemb.y[pl.gemb.n], Gp,
                             r.ga.dst_ptr, d.N, d.B, d.big, r.st));                   // modules.py:47-52
  }
  {   // modules.py:250-251: the two tier-1 heads share their input
    MlpJob jobs[2] = {{&pl.fadd1, hT, &L.fadd1, 0, (int)S, nullptr, 0, 0},
                      {&pl.fconn1, hT, &L.fconn1, 0, (int)S, nullptr, 0, 0}};
    GIB_TRY(mlp_forward_multi(r, jobs, 2, fwd_flags(r)));
  }
  GIB_TRY(concat_flat(r.ws + L.cat_add, L.fadd2.ld[0], r.ws + L.fadd1.y[pl.fadd1.n], L.fadd1.ld[pl.fadd1.n], d.N,
                      d.f_add, r.ws + L.g, Gp, pl.G, d.B, r.st));
  GIB_TRY(concat_flat(r.ws + L.cat_conn, L.fconn2.ld[0], r.ws + L.fconn1.y[pl.fconn1.n], L.fconn1.ld[pl.fconn1.n],
                      d.N, d.f_conn, r.ws + L.g, Gp, pl.G, d.B, r.st));
  const int na = d.N * d.f_add, nc = d.N * d.f_conn;
  {   // modules.py:270-276: the three tier-2 heads
    MlpJob jobs[3] = {{&pl.fadd2, r.ws + L.cat_add, &L.fadd2, 0, d.B, out, pl.apd, na},
                      {&pl.fconn2, r.ws + L.cat_conn, &L.fconn2, 0, d.B, out + na, pl.apd, nc},
                      {&pl.fterm2, r.ws + L.g, &L.fterm2, 0, d.B, out + na + nc, pl.apd, 1}};
    GIB_TRY(mlp_forward_multi(r, jobs, 3, fwd_flags(r)));
  }
  return 0;
}

// backward of the readout; leaves d(h_final) in scratch[bb.dh] ([S, Hp])
static int readout_backward(const Run& r, const BwdBufs& bb, const float* out, const float* dout) {
  const gib_dims& d = r.pl.d;
  const Plan& pl = r.pl;
  const Layout& L = r.L;
  const long long S = r.S;
  const int Hp = pl.Hp, Gp = pl.Gp;
  const float* hT = r.ws + L.hfinal;
  float* sc = r.scratch;
  const int na = d.N * d.f_add, nc = d.N * d.f_conn;
  float* T1 = sc + bb.T1;
  float* T2 = sc + bb.T2;
  // tier 2: three heads
  struct Head { const Mlp* m; const MlpAct* a; const float* x0; int off, width; size_t dcat; int ldcat; };
  Head heads[3] = {{&pl.fadd2, &L.fadd2, r.ws + L.cat_add, 0, na, bb.dcat_add, L.fadd2.ld[0]},
                   {&pl.fconn2, &L.fconn2, r.ws + L.cat_conn, na, nc, bb.dcat_conn, L.fconn2.ld[0]},
                   {&pl.fterm2, &L.fterm2, r.ws + L.g, na + nc, 1, bb.dgterm, Gp}};
  {   // three heads of equal depth: top gradients into three slices of T1, then one grouped backward
    MlpBwdJob jobs[3];
    size_t off = 0;
    for (int i = 0; i < 3; ++i) {
      const Head& h = heads[i];
      const Lin& last = pl.lins[h.m->first + h.m->n - 1];
      float* gt = T1 + off;
      GIB_TRY(dact_slice(gt, last.Rp, dout, out, pl.apd, h.off, h.width, ACT_SELU, d.B, r.st));
      jobs[i] = MlpBwdJob{h.m, h.x0, h.a, 0, d.B, gt, sc + h.dcat, h.ldcat, nullptr};
      off += ((size_t)d.B * last.Rp + 31) & ~(size_t)31;
    }
    GIB_TRY(mlp_backward_multi(r, bb, jobs, 3));
  }
  // d(graph embedding) = tail columns of the two cat gradients + the terminate head
  GIB_TRY(sum3_cols(sc + bb.dg, Gp, pl.G, sc + bb.dcat_add, L.fadd2.ld[0], na, sc + bb.dcat_conn, L.fconn2.ld[0], nc,
                    sc + bb.dgterm, Gp, d.B, r.st));
  // tier 1
  float* dh = sc + bb.dh;
  {
    const int ldf = L.fadd1.ld[pl.fadd1.n];
    GIB_TRY(unflatten_dact(T1, ldf, sc + bb.dcat_add, L.fadd2.ld[0], r.ws + L.fadd1.y[pl.fadd1.n], d.N, d.f_add, S,
                           r.st));
    const int ldc = L.fconn1.ld[pl.fconn1.n];
    GIB_TRY(unflatten_dact(T2, ldc, sc + bb.dcat_conn, L.fconn2.ld[0], r.ws + L.fconn1.y[pl.fconn1.n], d.N, d.f_conn,
                           S, r.st));
    MlpBwdJob jobs[2] = {{&pl.fadd1, hT, &L.fadd1, 0, (int)S, T1, dh, Hp, nullptr},
                         {&pl.fconn1, hT, &L.fconn1, 0, (int)S, T2, dh, Hp, dh}};
    GIB_TRY(mlp_backward_multi(r, bb, jobs, 2));
  }
  if (d.model == GIB_MNN) {
    GIB_TRY(bcast_nodes_add(dh, sc + bb.dg, Hp, d.N, S, r.st));
    return 0;
  }
  GIB_TRY(graph_gather_bwd(T1, T2, sc + bb.dg, r.ws + L.attn, r.ws + L.gatt.y[pl.gatt.n], r.ws + L.gemb.y[pl.gemb.n],
                           Gp, d.N, d.B, r.st));
  if (d.model == GIB_EMN) {
    // cat = [h | h]: both halves flow back into h
    const int ldc = L.gatt.ld[0];
    MlpBwdJob jobs[2] = {{&pl.gemb, hT, &L.gemb, 0, (int)S, T2, dh, Hp, dh},
                         {&pl.gatt, r.ws + L.cat_att, &L.gatt, 0, (int)S, T1, sc + bb.dcat_att, ldc, nullptr}};
    GIB_TRY(mlp_backward_multi(r, bb, jobs, 2));
    GIB_TRY(sum3_cols(dh, Hp, d.H, sc + bb.dcat_att, ldc, 0, sc + bb.dcat_att, ldc, d.H, dh, Hp, (int)S, r.st));
  } else {
    // only the hidden half of cat(hidden, nodes) needs a gradient: the transposed copy of
    // layer 0 holds just its first H columns (Ct = H), so the output is [S, Hp] directly.
    MlpBwdJob jobs[2] = {{&pl.gemb, hT, &L.gemb, 0, (int)S, T2, dh, Hp, dh},
                         {&pl.gatt, r.ws + L.cat_att, &L.gatt, 0, (int)S, T1, dh, Hp, dh}};
    GIB_TRY(mlp_backward_multi(r, bb, jobs, 2));
  }
  return 0;
}

// ------------------------------------------------------------------------------------
// node-state models: GGNN, MNN, AttentionGGNN
// ------------------------------------------------------------------------------------
static int node_model_forward(const Run& r, float* out) {
  const gib_dims& d = r.pl.d;
  const Plan& pl = r.pl;
  const Layout& L = r.L;
  const long long S = r.S;
  const int Hp = pl.Hp, Mp = pl.Mp;
  const Lin& ih = pl.lins[pl.gru_ih];
  const Lin& hh = pl.lins[pl.gru_hh];
  // summation_mpnn.py:121-125: zero-padded node features
  GIB_TRY(concat2_in(r.ws + L.h[0], Hp, r.nodes, d.F, d.F, d.in_dtype, nullptr, 0, 0, 0, S, r.st));
  // rows of the message MLPs: message rows (mpnn.py:60-65, 284-294 read only the source atom's state, the bond type
  // and the bond value), or one per bond entry
  const MsgRows mr = r.msg_rows ? msg_rows_of(r) : MsgRows{};
  if (r.msg_rows)
    GIB_TRY(msg_rows_build(r.ga, mr, r.cap ? r.dev_hdr : nullptr, r.tb, d.B, d.N, r.ngroups, r.E, r.P, r.st));
  const int* row_src = r.msg_rows ? mr.u_src : r.ga.ent_src;
  const int* dst_rows = r.msg_rows ? mr.dst_u : r.ga.dst_ent;
  const float* row_w = r.msg_rows ? (r.unit_bonds ? nullptr : mr.u_w) : r.w();
  for (int t = 0; t < d.T; ++t) {
    const float* h = r.ws + L.h[t];
    // mpnn.py:286-288 scales the neighbour state by the bond value for GGNN only
    GIB_TRY(gather_rows(r.ws + L.x0[t], h, Hp, row_src, row_w, d.model == GIB_GGNN, r.P, nullptr, r.st));
    {   // one grouped launch per layer over the bond types (same input rows layout, per-type weights)
      MlpJob jobs[4];
      for (int g = 0; g < r.ngroups; ++g) {
        const MsgRange rr = msg_range(r, g);
        jobs[g] = MlpJob{&pl.msg[g], r.ws + L.x0[t], &L.msg[t], rr.row0, rr.rows, nullptr, 0, 0, rr.m_dev, rr.base_dev};
      }
      GIB_TRY(mlp_forward_multi(r, jobs, r.ngroups, fwd_flags(r)));
      if (d.model == GIB_ATTGGNN) {
        for (int g = 0; g < r.ngroups; ++g)
          jobs[g] = MlpJob{&pl.att[g], r.ws + L.x0[t], &L.att[t], r.tb[g], r.tc[g], nullptr, 0, 0,
                           type_count_dev(r, g), type_base_dev(r, g)};
        GIB_TRY(mlp_forward_multi(r, jobs, r.ngroups, fwd_flags(r)));
      }
    }
    const float* msgs = r.ws + L.msg[t].y[pl.msg[0].n];
    if (d.model == GIB_ATTGGNN)
      GIB_TRY(seg_softmax_fwd(r.ws + L.msum[t], msgs, r.ws + L.att[t].y[pl.att[0].n], Mp, r.ga.dst_ptr, r.ga.dst_ent,
                              r.w(), S, r.st));
    else
      GIB_TRY(scatter_sum(r.ws + L.msum[t], msgs, Mp, r.ga.dst_ptr, dst_rows, row_w, 0, S, r.st,
                          r.cap ? 0.0 : 4.0 * ((double)r.E * d.M + (double)S * d.M + (double)(S + 1))));   // SURVEY.md 8d bytes
    {   // the two GRU input projections are independent: one grouped launch
      const GemmNT ps[2] = {lin_fwd(r, ih, r.ws + L.msum[t], Mp, (int)S, ACT_NONE, r.ws + L.gi[t], ih.Rp),
                            lin_fwd(r, hh, h, Hp, (int)S, ACT_NONE, r.ws + L.gh[t], hh.Rp)};
      GIB_TRY(gemm_nt_group(ps, 2, r.st));
    }
    GIB_TRY(gru_fwd(r.ws + L.h[t + 1], r.ws + L.gi[t], r.ws + L.gh[t], h, Hp, r.ga.dst_ptr, S, nullptr, r.st));
  }
  return readout_forward(r, out);
}

// part 0: everything; part 1: the readout only (leaves d h_final in scratch[bb.dh]; the gradients of the gather /
// APDReadout parameters -- the tail of the gradient bucket, 79 % of it -- are final afterwards); part 2: the message
// passes only (continues from scratch[bb.dh]).  Splitting lets a data-parallel caller start the all-reduce of the
// readout gradients while the message-passing backward still runs (SURVEY.md 8e).
static int node_model_backward(const Run& r, const BwdBufs& bb, const float* out, const float* dout, int part) {
  const gib_dims& d = r.pl.d;
  const Plan& pl = r.pl;
  const Layout& L = r.L;
  const long long S = r.S;
  const int Hp = pl.Hp, Mp = pl.Mp;
  const Lin& ih = pl.lins[pl.gru_ih];
  const Lin& hh = pl.lins[pl.gru_hh];
  float* sc = r.scratch;
  if (part != 2) GIB_TRY(readout_backward(r, bb, out, dout));
  if (part == 1) return 0;
  float* dh = sc + bb.dh;        // d h[t+1]
  float* dh_dir = sc + bb.dh2;   // direct path through the GRU
  const MsgRows mr = r.msg_rows ? msg_rows_of(r) : MsgRows{};   // built by the forward
  const float* row_w = r.unit_bonds ? nullptr : mr.u_w;
  for (int t = d.T - 1; t >= 0; --t) {
    const float* h = r.ws + L.h[t];
    GIB_TRY(gru_bwd(sc + bb.dgi, sc + bb.dgh, dh_dir, dh, r.ws + L.gi[t], r.ws + L.gh[t], h, Hp, r.ga.dst_ptr, S,
                    nullptr, r.st));
    {   // weight gradients of the two GRU projections: one grouped launch
      const GemmDW qs[2] = {lin_dw(r, bb, ih, sc + bb.dgi, r.ws + L.msum[t], Mp, (int)S),
                            lin_dw(r, bb, hh, sc + bb.dgh, h, Hp, (int)S)};
      GIB_TRY(gemm_dw_group(qs, 2, 0, r.st));
    }
    {   // dMsum = dgi W_ih  and  dh[t] = dgh W_hh + direct  (dh[t+1] is dead after gru_bwd): one grouped launch
      GemmNT ps[2] = {lin_dx(r, ih, sc + bb.dgi, (int)S, sc + bb.dmsum, Mp), lin_dx(r, hh, sc + bb.dgh, (int)S, dh, Hp)};
      ps[1].mode = EPI_ADD; ps[1].aux = dh_dir; ps[1].ldaux = Hp;
      // h[0] is the zero-padded input (summation_mpnn.py:121-125): nothing consumes d h[0], so at t == 0 the dh GEMM,
      // the first-layer input gradients of the message MLPs and their scatter are skipped
      GIB_TRY(gemm_nt_group(ps, t == 0 ? 1 : 2, r.st));
    }
    // through the aggregation into the per-bond message MLPs
    float* T1 = sc + bb.T1;
    float* T2 = sc + bb.T2;
    float* dx0 = sc + bb.dx0;
    const int nm = pl.msg[0].n;
    if (d.model == GIB_ATTGGNN) {
      GIB_CUDA_TRY(cudaMemsetAsync(T1, 0, (size_t)r.P * Mp * sizeof(float), r.st));
      GIB_CUDA_TRY(cudaMemsetAsync(T2, 0, (size_t)r.P * Mp * sizeof(float), r.st));
      GIB_TRY(seg_softmax_bwd(T1, T2, sc + bb.dmsum, r.ws + L.msg[t].y[nm], r.ws + L.att[t].y[pl.att[0].n], Mp,
                              r.ga.dst_ptr, r.ga.dst_ent, r.w(), S, r.st));
    } else if (r.msg_rows) {
      // every entry of a message row adds its destination's gradient: duplicates are summed before the GEMMs
      GIB_TRY(seg_reduce_dact(T1, sc + bb.dmsum, r.ws + L.msg[t].y[nm], Mp, mr.u_ptr, mr.u_dst, row_w, pl.msg[0].act,
                              r.P, r.st));
    } else {
      GIB_TRY(scatter_bwd(T1, sc + bb.dmsum, r.ws + L.msg[t].y[nm], Mp, r.ga.ent_dst, r.w(), pl.msg[0].act, r.P,
                          r.st));
    }
    {
      MlpBwdJob jobs[4];
      for (int g = 0; g < r.ngroups; ++g) {
        const MsgRange rr = msg_range(r, g);
        const size_t ro = (size_t)rr.row0;
        jobs[g] = MlpBwdJob{&pl.msg[g], r.ws + L.x0[t], &L.msg[t], rr.row0, rr.rows, T1 + ro * Mp,
                            t == 0 ? nullptr : dx0 + ro * Hp, Hp, nullptr, rr.m_dev, rr.base_dev};
      }
      GIB_TRY(mlp_backward_multi(r, bb, jobs, r.ngroups, msg_dev(r) ? r.P : 0));
      if (d.model == GIB_ATTGGNN) {
        for (int g = 0; g < r.ngroups; ++g) {
          const size_t ro = (size_t)r.tb[g];
          jobs[g] = MlpBwdJob{&pl.att[g], r.ws + L.x0[t], &L.att[t], r.tb[g], r.tc[g], T2 + ro * Mp,
                              t == 0 ? nullptr : dx0 + ro * Hp, Hp, dx0 + ro * Hp, type_count_dev(r, g),
                              type_base_dev(r, g)};
        }
        GIB_TRY(mlp_backward_multi(r, bb, jobs, r.ngroups, r.cap ? r.P : 0));
      }
    }
    // dh[t][src] += (w) dX0   -- deterministic gather-reduce over the by-source CSR (of message rows or of entries; the
    // host knows the row count of the latter only)
    if (t > 0) {
      if (r.msg_rows)
        GIB_TRY(scatter_sum(dh, dx0, Hp, mr.s_ptr, mr.s_u, d.model == GIB_GGNN ? row_w : nullptr, 1, S, r.st));
      else
        GIB_TRY(scatter_sum(dh, dx0, Hp, r.ga.src_ptr, r.ga.src_ent, d.model == GIB_GGNN ? r.w() : nullptr, 1, S,
                            r.st, r.cap ? 0.0 : 4.0 * ((double)r.E * d.H + 2.0 * S * d.H + (double)(S + 1))));
    }
  }
  return 0;
}

// ------------------------------------------------------------------------------------
// EMN
// ------------------------------------------------------------------------------------
// Capacity mode: E is the entry capacity; the live bond rows are [0, live) with live = TYPE_COUNT[0] in the device
// header (the EMN's one untyped group starts at row 0).  Every MLP / GEMM runs on that device row range, every bond-row
// kernel gets the count, and rows past it are neither written nor read by a live row.
static int emn_forward(const Run& r, float* out) {
  const gib_dims& d = r.pl.d;
  const Plan& pl = r.pl;
  const Layout& L = r.L;
  const int Hp = pl.Hp, E = r.E;
  const Lin& ih = pl.lins[pl.gru_ih];
  const Lin& hh = pl.lins[pl.gru_hh];
  const int* live = type_count_dev(r, 0);
  const int* base = type_base_dev(r, 0);
  GIB_TRY(emn_input(r.ws + L.xin, L.embnn.ld[0], r.nodes, r.edges, d.in_dtype, r.ga.ent_dst, r.ga.ent_src, d.N, d.F,
                    d.Ef, E, r.st));
  {   // the layers of an MLP run as one dependent-chain launch (mlp_forward_multi)
    MlpJob j[1] = {{&pl.embnn, r.ws + L.xin, &L.embnn, 0, E, nullptr, 0, 0, live, base}};
    GIB_TRY(mlp_forward_multi(r, j, 1, fwd_flags(r)));
  }
  GIB_TRY(tanh_fwd(r.ws + L.xt, r.ws + L.embnn.y[pl.embnn.n], E, Hp, live, r.st));      // mpnn.py:469
  {   // emb_msg_nn and att_msg_nn read the same rows: sibling chains in one launch
    MlpJob j[2] = {{&pl.emsg, r.ws + L.xt, &L.emx, 0, E, nullptr, 0, 0, live, base},
                   {&pl.eatt, r.ws + L.xt, &L.enx, 0, E, nullptr, 0, 0, live, base}};
    GIB_TRY(mlp_forward_multi(r, j, 2, fwd_flags(r)));
  }
  if (E > 0) GIB_CUDA_TRY(cudaMemsetAsync(r.ws + L.mem[0], 0, (size_t)E * Hp * sizeof(float), r.st));
  for (int t = 0; t < d.T; ++t) {
    {
      MlpJob j[2] = {{&pl.emsg, r.ws + L.mem[t], &L.emm[t], 0, E, nullptr, 0, 0, live, base},
                     {&pl.eatt, r.ws + L.mem[t], &L.enm[t], 0, E, nullptr, 0, 0, live, base}};
      GIB_TRY(mlp_forward_multi(r, j, 2, fwd_flags(r)));
    }
    GIB_TRY(emn_aggregate_fwd(r.ws + L.emsg[t], r.ws + L.emx.y[pl.emsg.n], r.ws + L.enx.y[pl.eatt.n],
                              r.ws + L.emm[t].y[pl.emsg.n], r.ws + L.enm[t].y[pl.eatt.n], Hp, r.ga.ent_dst,
                              r.ga.ent_src, r.ga.dst_ptr, E, live, r.st));
    GIB_TRY(gemm_nt(lin_fwd(r, ih, r.ws + L.emsg[t], Hp, E, ACT_NONE, r.ws + L.gi[t], ih.Rp, live, base), r.st));
    // GRUCell(message) with hx=None (mpnn.py:488): h = 0, so W_hh h + b_hh = b_hh
    GIB_TRY(gru_fwd(r.ws + L.mem[t + 1], r.ws + L.gi[t], r.packed + hh.ob, nullptr, Hp, nullptr, E, live, r.st));
  }
  // edge_mpnn.py:178-189: node vector = sum of the memories of the bonds leaving it
  GIB_TRY(scatter_sum(r.ws + L.hfinal, r.ws + L.mem[d.T], Hp, r.ga.dst_ptr, r.ga.dst_ent, nullptr, 0, r.S, r.st));
  return readout_forward(r, out);
}

// backward of emb_msg_nn and att_msg_nn over the same bond rows: chained input gradients + one grouped weight-gradient
// launch.  Capacity mode: the group is planned for both members' rows, and siblings of unequal depth (msg_depth !=
// att_depth) run one after the other, each still on the device row range.
static int emn_siblings_backward(const Run& r, const BwdBufs& bb, const MlpBwdJob* j) {
  if (!r.cap) return mlp_backward_multi(r, bb, j, 2);
  if (j[0].m->n == j[1].m->n) return mlp_backward_multi(r, bb, j, 2, 2LL * r.E, /*same_rows=*/true);
  GIB_TRY(mlp_backward_multi(r, bb, j, 1, r.E));
  return mlp_backward_multi(r, bb, j + 1, 1, r.E);
}

static int emn_backward(const Run& r, const BwdBufs& bb, const float* out, const float* dout, int part) {
  const gib_dims& d = r.pl.d;
  const Plan& pl = r.pl;
  const Layout& L = r.L;
  const int Hp = pl.Hp, E = r.E;
  const Lin& ih = pl.lins[pl.gru_ih];
  const Lin& hh = pl.lins[pl.gru_hh];
  const int* live = type_count_dev(r, 0);
  const int* base = type_base_dev(r, 0);
  float* sc = r.scratch;
  if (part != 2) GIB_TRY(readout_backward(r, bb, out, dout));
  if (part == 1 || E == 0) return 0;
  const size_t EH = (size_t)E * Hp;
  float* dmem = sc + bb.dmem;      // d mem[t+1]
  float* dmem2 = sc + bb.dmem2;
  float* T1 = sc + bb.T1;
  float* T2 = sc + bb.T2;
  GIB_TRY(gather_rows(dmem, sc + bb.dh, Hp, r.ga.ent_dst, nullptr, 0, E, live, r.st));
  GIB_CUDA_TRY(cudaMemsetAsync(sc + bb.dEMx, 0, EH * sizeof(float), r.st));
  GIB_CUDA_TRY(cudaMemsetAsync(sc + bb.dENx, 0, EH * sizeof(float), r.st));
  for (int t = d.T - 1; t >= 0; --t) {
    GIB_TRY(gru_bwd(sc + bb.dgi, sc + bb.dgh, nullptr, dmem, r.ws + L.gi[t], r.packed + hh.ob, nullptr, Hp, nullptr,
                    E, live, r.st));
    GIB_TRY(gemm_dw(lin_dw(r, bb, ih, sc + bb.dgi, r.ws + L.emsg[t], Hp, E, live, base), r.st));
    GIB_TRY(colsum_add(r.grads[hh.pb], sc + bb.dgh, hh.Rp, E, hh.R, hh.Rb, hh.Rbp, live, r.st));  // d b_hh; d W_hh = 0
    GIB_TRY(gemm_nt(lin_dx(r, ih, sc + bb.dgi, E, sc + bb.dmsum, Hp, live, base), r.st));
    const float* EMm = r.ws + L.emm[t].y[pl.emsg.n];
    const float* ENm = r.ws + L.enm[t].y[pl.eatt.n];
    GIB_TRY(emn_aggregate_bwd(sc + bb.dEMx, sc + bb.dENx, sc + bb.dEMm, sc + bb.dENm, sc + bb.st3, sc + bb.dmsum,
                              r.ws + L.emx.y[pl.emsg.n], r.ws + L.enx.y[pl.eatt.n], EMm, ENm, Hp, r.ga, E, live, r.st));
    GIB_TRY(mul_dselu(T1, sc + bb.dEMm, EMm, E, Hp, live, r.st));
    GIB_TRY(mul_dselu(T2, sc + bb.dENm, ENm, E, Hp, live, r.st));
    {
      MlpBwdJob j[2] = {{&pl.emsg, r.ws + L.mem[t], &L.emm[t], 0, E, T1, dmem2, Hp, nullptr, live, base},
                        {&pl.eatt, r.ws + L.mem[t], &L.enm[t], 0, E, T2, dmem, Hp, dmem2, live, base}};
      GIB_TRY(emn_siblings_backward(r, bb, j));
    }
  }
  // pass-independent branch through x = tanh(embedding_nn(.))
  GIB_TRY(mul_dselu(T1, sc + bb.dEMx, r.ws + L.emx.y[pl.emsg.n], E, Hp, live, r.st));
  GIB_TRY(mul_dselu(T2, sc + bb.dENx, r.ws + L.enx.y[pl.eatt.n], E, Hp, live, r.st));
  {
    MlpBwdJob j[2] = {{&pl.emsg, r.ws + L.xt, &L.emx, 0, E, T1, dmem2, Hp, nullptr, live, base},
                      {&pl.eatt, r.ws + L.xt, &L.enx, 0, E, T2, dmem, Hp, dmem2, live, base}};
    GIB_TRY(emn_siblings_backward(r, bb, j));
  }
  GIB_TRY(tanh_selu_bwd(T1, dmem, r.ws + L.xt, r.ws + L.embnn.y[pl.embnn.n], E, Hp, live, r.st));
  {
    MlpBwdJob j[1] = {{&pl.embnn, r.ws + L.xin, &L.embnn, 0, E, T1, nullptr, 0, nullptr, live, base}};
    GIB_TRY(mlp_backward_multi(r, bb, j, 1, r.cap ? r.E : 0));
  }
  return 0;
}

// ------------------------------------------------------------------------------------
// backward scratch layout
// ------------------------------------------------------------------------------------
static void mlp_extent(const Plan& pl, const Mlp& m, size_t rows, size_t& big, size_t& dw) {
  if (m.n == 0 || rows == 0) return;
  for (int l = 0; l < m.n; ++l) {
    const Lin& L = pl.lins[m.first + l];
    big = std::max(big, rows * (size_t)std::max(L.Rp, L.Cp));
    dw = std::max(dw, gemm_dw_scratch_floats((int)rows, L.Rp, L.Cp));
  }
}
// the same for sibling MLPs of equal depth whose weight gradients run as one grouped launch per layer; split: siblings
// that do not fit one launch run in the sub-groups of mlp_backward_multi (capacity mode), else one by one (mlp_extent)
static void group_extent(const Plan& pl, const Mlp* const* ms, const size_t* rows, int n, long long plan_rows, size_t& dw,
                         bool split = false) {
  bool same = true;
  for (int i = 1; i < n; ++i) same = same && ms[i]->n == ms[0]->n;
  const int depth = ms[0]->n;
  if (!same || depth * n > kTc3MaxProblems) {
    if (split)
      for (int i = 0, k; i < n; i += k) {
        k = sub_group(ms, n, i);
        group_extent(pl, ms + i, rows + i, k, plan_rows, dw);
      }
    return;
  }
  GemmDW qs[kTc3MaxProblems];     // all layers of all members: one grouped launch (mlp_backward_multi)
  int nq = 0;
  for (int l = 0; l < depth; ++l)
    for (int i = 0; i < n; ++i) {
      if (rows[i] == 0) continue;
      const Lin& L = pl.lins[ms[i]->first + l];
      qs[nq].M = (int)rows[i]; qs[nq].Nn = L.Rp; qs[nq].Kk = L.Cp;
      ++nq;
    }
  if (nq) dw = std::max(dw, 2 * gemm_dw_group_half_floats(qs, nq, plan_rows * depth));
}

void make_bwd(const Run& r, BwdBufs& bb) {
  const gib_dims& d = r.pl.d;
  const Plan& pl = r.pl;
  const size_t S = (size_t)r.S, B = (size_t)d.B, P = (size_t)r.P, E = (size_t)r.E;
  const int Hp = pl.Hp, Mp = pl.Mp, Gp = pl.Gp;
  size_t big = 32, dw = 32;
  size_t maxtc = 0;
  for (int g = 0; g < r.ngroups; ++g) maxtc = std::max(maxtc, (size_t)r.tc[g]);
  // planned rows of the message MLPs (msg_range): the whole buffer per type on device-side row counts
  const bool dev = msg_dev(r);
  size_t mrows[4] = {0, 0, 0, 0};
  for (int g = 0; g < r.ngroups; ++g) mrows[g] = dev ? P : (size_t)r.tc[g];
  if (d.model != GIB_EMN) {
    for (int g = 0; g < r.ngroups; ++g) {
      mlp_extent(pl, pl.msg[g], mrows[g], big, dw);
      if (d.model == GIB_ATTGGNN) mlp_extent(pl, pl.att[g], mrows[g], big, dw);
    }
    big = std::max(big, P * (size_t)std::max(Mp, Hp));
    {
      const Mlp* ms[4];
      for (int g = 0; g < r.ngroups; ++g) ms[g] = &pl.msg[g];
      group_extent(pl, ms, mrows, r.ngroups, dev ? r.P : 0, dw, dev);
      if (d.model == GIB_ATTGGNN) {
        for (int g = 0; g < r.ngroups; ++g) ms[g] = &pl.att[g];
        group_extent(pl, ms, mrows, r.ngroups, dev ? r.P : 0, dw, dev);
      }
    }
  } else {
    mlp_extent(pl, pl.embnn, E, big, dw);
    mlp_extent(pl, pl.emsg, E, big, dw);
    mlp_extent(pl, pl.eatt, E, big, dw);
    // the same plan rows as emn_backward / emn_siblings_backward (the split of a grouped weight gradient depends on them)
    const Mlp* one[1] = {&pl.embnn}; const size_t re[2] = {E, E};
    group_extent(pl, one, re, 1, r.cap ? (long long)E : 0, dw);
    const Mlp* two[2] = {&pl.emsg, &pl.eatt};
    group_extent(pl, two, re, 2, r.cap ? 2LL * (long long)E : 0, dw);
    if (r.cap && pl.emsg.n != pl.eatt.n) {
      group_extent(pl, two, re, 1, (long long)E, dw);
      group_extent(pl, two + 1, re, 1, (long long)E, dw);
    }
    big = std::max(big, E * (mlp_max_ld(pl, pl.emsg) + mlp_max_ld(pl, pl.eatt)) + 64);
  }
  const size_t gru_rows = d.model == GIB_EMN ? E : S;
  dw = std::max(dw, gemm_dw_scratch_floats((int)gru_rows, pl.lins[pl.gru_ih].Rp, pl.lins[pl.gru_ih].Cp));
  dw = std::max(dw, gemm_dw_scratch_floats((int)gru_rows, pl.lins[pl.gru_hh].Rp, pl.lins[pl.gru_hh].Cp));
  if (d.model != GIB_MNN) { mlp_extent(pl, pl.gatt, S, big, dw); mlp_extent(pl, pl.gemb, S, big, dw); }
  mlp_extent(pl, pl.fadd1, S, big, dw);
  mlp_extent(pl, pl.fconn1, S, big, dw);
  mlp_extent(pl, pl.fadd2, B, big, dw);
  mlp_extent(pl, pl.fconn2, B, big, dw);
  mlp_extent(pl, pl.fterm2, B, big, dw);
  {
    const Mlp* t2[3] = {&pl.fadd2, &pl.fconn2, &pl.fterm2}; const size_t r2[3] = {B, B, B};
    group_extent(pl, t2, r2, 3, 0, dw);
    const Mlp* t1[2] = {&pl.fadd1, &pl.fconn1}; const size_t r1[2] = {S, S};
    group_extent(pl, t1, r1, 2, 0, dw);
    if (d.model != GIB_MNN) {
      const Mlp* ga[2] = {&pl.gemb, &pl.gatt};
      group_extent(pl, ga, r1, 2, 0, dw);
    }
    GemmDW qs[2];
    qs[0].M = qs[1].M = (int)gru_rows;
    qs[0].Nn = pl.lins[pl.gru_ih].Rp; qs[0].Kk = pl.lins[pl.gru_ih].Cp;
    qs[1].Nn = pl.lins[pl.gru_hh].Rp; qs[1].Kk = pl.lins[pl.gru_hh].Cp;
    dw = std::max(dw, 2 * gemm_dw_group_half_floats(qs, 2, 0));
  }
  // grouped backward passes keep one ping/pong slice per member inside GA / GB
  {
    size_t types = 64;
    for (int g = 0; g < r.ngroups && d.model != GIB_EMN; ++g) {
      size_t w = mlp_max_ld(pl, pl.msg[g]);
      if (d.model == GIB_ATTGGNN) w = std::max(w, mlp_max_ld(pl, pl.att[g]));
      if (dev) types = std::max(types, (size_t)r.P * w + 64);   // device-side row counts: the groups share one slice
      else types += (size_t)r.tc[g] * w + 32;
    }
    big = std::max(big, types);
    big = std::max(big, S * (mlp_max_ld(pl, pl.fadd1) + mlp_max_ld(pl, pl.fconn1)) + 64);
    big = std::max(big, B * (mlp_max_ld(pl, pl.fadd2) + mlp_max_ld(pl, pl.fconn2) + mlp_max_ld(pl, pl.fterm2)) + 128);
    if (d.model != GIB_MNN) big = std::max(big, S * (mlp_max_ld(pl, pl.gatt) + mlp_max_ld(pl, pl.gemb)) + 64);
  }
  Bump bp;
  int max_depth = 2;
  {
    const Mlp* every[] = {&pl.msg[0], &pl.att[0], &pl.gatt, &pl.gemb, &pl.fadd1, &pl.fconn1, &pl.fadd2, &pl.fconn2,
                          &pl.fterm2, &pl.embnn, &pl.emsg, &pl.eatt};
    for (const Mlp* m : every) max_depth = std::max(max_depth, std::min(m->n, 8));
  }
  for (int l = 0; l < 8; ++l) bb.Gl[l] = 0;
  for (int l = 1; l < std::max(max_depth, 3); ++l) bb.Gl[l] = bp.take(big);   // one gradient buffer per layer (chains)
  bb.GA = bb.Gl[1]; bb.GB = bb.Gl[2];                                         // ping / pong of the single-MLP path
  bb.T1 = bp.take(big); bb.T2 = bp.take(big);
  bb.flags = bp.take(chain_flag_floats(std::max(std::max(S, P), std::max(B, E))));
  bb.dw = bp.take(dw);
  bb.dw_half = dw / 2;          // gemm_dw alternates between two halves (helper side stream)
  bb.dh = bp.take(S * Hp); bb.dh2 = bp.take(S * Hp);
  bb.dmsum = bp.take(std::max(S, E) * (size_t)std::max(Mp, Hp));
  bb.dgi = bp.take(std::max(S, E) * 3 * Hp); bb.dgh = bp.take(std::max(S, E) * 3 * Hp);
  bb.dx0 = bp.take(P * Hp);
  bb.dcat_att = d.model != GIB_MNN ? bp.take(S * pl.lins[pl.gatt.first].Cp) : 0;
  bb.dcat_add = bp.take(B * pl.lins[pl.fadd2.first].Cp);
  bb.dcat_conn = bp.take(B * pl.lins[pl.fconn2.first].Cp);
  bb.dgterm = bp.take(B * Gp); bb.dg = bp.take(B * Gp);
  if (d.model == GIB_EMN) {
    bb.dmem = bp.take(E * Hp); bb.dmem2 = bp.take(E * Hp);
    bb.dEMx = bp.take(E * Hp); bb.dENx = bp.take(E * Hp); bb.dEMm = bp.take(E * Hp); bb.dENm = bp.take(E * Hp);
    bb.st3 = bp.take(3 * E * Hp);
  }
  bb.total = bp.off;
}

int model_forward(const Run& r, float* out) {
  return r.pl.d.model == GIB_EMN ? emn_forward(r, out) : node_model_forward(r, out);
}
int model_backward(const Run& r, const BwdBufs& bb, const float* out, const float* dout, int part) {
  if (part < 0 || part > 2) { set_error("model_backward: part %d", part); return -2; }
  GIB_TRY(dw_begin());
  const int rc = r.pl.d.model == GIB_EMN ? emn_backward(r, bb, out, dout, part)
                                         : node_model_backward(r, bb, out, dout, part);
  const int rj = dw_join(r.st);   // the last reduction job runs on the helper side stream: order it before the caller
  return rc ? rc : rj;
}

}  // namespace gib
