// Host-side structures of the whole-model orchestration (model.cu).
#pragma once
#include <algorithm>
#include <vector>

#include "../../include/gib200.h"
#include "common.cuh"
#include "graph.cuh"

namespace gib {

constexpr int kMaxPasses = 16;

// one reference weight (+bias) and where its packed copies live
struct Lin {
  int pw, pb;             // indices into the parameter pointer table (pb = -1: no bias)
  int R, C;               // real out / in features
  int nblk, Rb;           // row blocks (GRU gates): R = nblk * Rb
  long long rs, cs;       // source strides: element (r, c) at W[src_off + r*rs + c*cs]
  long long src_off;
  int Ct;                 // leading input columns kept in the transposed copy
  int Rbp, Rp, Cp, Ctp;   // padded extents
  size_t ow, owt, ob;     // float offsets of Wp [Rp, Cp], WTp [Ctp, Rp], bp [Rp] in the packed arena
  size_t ow_hi, ow_lo, owt_hi, owt_lo;   // TF32 hi / lo planes of Wp and WTp (pre-split B operands of the tensor-core GEMM)
};

struct Mlp {
  int first = 0, n = 0;   // lins[first .. first + n)
  int act = ACT_SELU;     // activation after EVERY layer (modules.py:127-142)
};

struct Plan {
  gib_dims d;
  std::vector<Lin> lins;
  std::vector<long long> param_numel;
  Mlp msg[4], att[4];
  int gru_ih = -1, gru_hh = -1;
  Mlp gatt, gemb, fadd1, fconn1, fadd2, fconn2, fterm2;
  Mlp embnn, emsg, eatt;
  size_t packed_floats = 0;
  int Hp = 0, Mp = 0, G = 0, Gp = 0, apd = 0;
};

struct MlpAct {
  size_t y[9];  // y[l] = float offset of layer l's output in the workspace (y[0] unused)
  int ld[9];    // ld[0] = leading dimension of the input
};

struct Layout {
  size_t h[kMaxPasses + 1];
  size_t x0[kMaxPasses];
  MlpAct msg[kMaxPasses], att[kMaxPasses];
  size_t msum[kMaxPasses], gi[kMaxPasses], gh[kMaxPasses];
  // GGNN / MNN: the message-row table (graph.cuh: MsgRows), int / float arrays
  size_t mr_src, mr_w, mr_ptr, mr_dst, mr_ent, mr_dst_u, mr_sptr, mr_su, mr_meta, mr_tmp;
  // EMN
  size_t xin, xt, mem[kMaxPasses + 1], emsg[kMaxPasses];
  MlpAct embnn, emx, enx, emm[kMaxPasses], enm[kMaxPasses];
  // readout
  size_t hfinal, cat_att, attn, g, cat_add, cat_conn;
  MlpAct gatt, gemb, fadd1, fconn1, fadd2, fconn2, fterm2;
  size_t flags;     // row-block counters of the dependent-chain GEMM launches (ints, zeroed per launch)
  size_t total;
};

struct BwdBufs {
  size_t dw_half;
  size_t GA, GB, T1, T2, dw, dh, dh2, dmsum, dgi, dgh, dx0, dcat_att, dcat_add, dcat_conn, dgterm, dg;
  size_t dmem, dmem2, dEMx, dENx, dEMm, dENm, st3;
  size_t Gl[8];     // per-layer gradient buffers of a chained MLP backward (Gl[0] unused)
  size_t flags;
  size_t total;
};

struct Run {
  Plan pl;
  Layout L;
  int E = 0, P = 0, ngroups = 0;
  bool unit_bonds = false;
  // GGNN / MNN: the message MLPs run on message rows (one per source atom and bond type, graph.cuh: MsgRows) unless
  // gib_tc_debug bit 3 asks for one row per bond entry; msg_dev_rows: on the device-side row counts of the table (the
  // grouped tensor-core call pattern), else on the entry groups' host row ranges, pad rows included
  bool msg_rows = false, msg_dev_rows = false;
  bool cap = false;                // capacity header: E / P / tc are capacities, live counts are read from dev_hdr
  const int* dev_hdr = nullptr;     // device copy of the graph header (written by K0)
  const float* w() const { return unit_bonds ? nullptr : ga.ent_w; }
  int tc[4], tb[5];
  long long S = 0;
  const void* nodes = nullptr;     // float32 or int8 (dims.in_dtype)
  const void* edges = nullptr;
  GraphArrays ga;
  const float* packed = nullptr;
  float* ws = nullptr;          // forward workspace (saved activations)
  float* scratch = nullptr;     // backward scratch
  float* const* grads = nullptr;
  cudaStream_t st = nullptr;
  int tf32 = 0;                 // precision of every tensor-core GEMM of the call (GemmNT::tf32), from gib_dims.tf32
};

int build_plan(const gib_dims& d, Plan& pl);
// prec: the matmul precision code (gib_dims.tf32) whose planes to write (0 / 1: TF32 hi / lo, 2 / 3: bf16 / fp16)
int pack_params(const Plan& pl, const float* const* params, float* packed, int prec, cudaStream_t st);
size_t graph_buf_ints(long long S, int E, int P);
GraphArrays graph_arrays(void* buf, long long S, int E, int P);
int make_run(const gib_dims& d, const int* hdr, Run& r);
void make_bwd(const Run& r, BwdBufs& bb);
int model_forward(const Run& r, float* out);
int model_backward(const Run& r, const BwdBufs& bb, const float* out, const float* dout, int part = 0);

}  // namespace gib
