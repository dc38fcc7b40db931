// Tensor-core GEMM with fp32-accurate 3xTF32 operand splitting, sm_90a (Hopper).
//
//   NT :  C[M, :N]   = epi( A[M,K] * W[N,K]^T )     A = fp32 activations (row-major, K contiguous), W = a packed weight,
//                                                    given as its TF32 hi / lo planes (gib_model_pack) or raw fp32
//   TN :  P[s][n][k] = sum_{m in segment s} G[m,n] * X[m,k]   (weight-gradient partial tiles; G, X fp32 row-major
//         pb[s][n]   = sum_{m in segment s} G[m,n]            activations; bias-gradient partials from the G
//                                                              fragments in registers; segments: see dw_plan)
//
// Why 3xTF32: the parity bar is 1e-4 on the logits; one TF32 pass is 1.8e-2 off (SURVEY.md §7).  Each operand x is
// split into hi = tf32(x) and lo = x - hi; the product is accumulated as hi*hi + (lo*hi + hi*lo) (the dropped lo*lo term
// is ~2^-22 relative).  The cross terms, 2^-11 of the main ones, get their own accumulator so that their roundings stay
// away from the large running sum; the two are added in fp32 in the epilogue.
//
// Single-pass TF32 (template parameter TF1; GemmNT::tf32 / GemmDW::tf32, set when the caller accepts TF32 matmuls):
// the product is the hi*hi term alone -- W from its hi plane only (raw W rounded in the kernel as gib_model_pack
// rounds it), the activations rounded in registers or in the X transpose with the same round-to-nearest, one
// accumulator, no lo loads and no cross-term MMAs.  Schedules, stage rings, epilogues, chains and the split-K
// reduction are those of the 3xTF32 kernels.
//
// 16-bit operands (template parameter H16 = 1 bf16 / 2 fp16 of the two wgmma kernels; GemmNT::tf32 / GemmDW::tf32 =
// 2 / 3, set when the caller runs under torch.autocast): every operand rounded to nearest-even to 16 bits, as
// tensor.to(dtype) rounds, fp32 accumulation.  W is one K-major 16-bit plane (gib_model_pack writes it over the bytes
// of the lo plane; the problem's W_hi points at it), read by TMA as [128 x 32] boxes of 64-byte rows with the 64-byte
// swizzle, so the k-block stays 32 and the stage rings, schedules, epilogues, chains and the split-K reduction are
// shared.  The A / G fragments are rounded in registers from the fp32 tiles (cvt.rn.{bf16,f16}x2.f32), the X
// transpose writes a 16-bit K-major plane; per k-block one group of 2 wgmma.m64n128k16 (A from registers).  No run-time
// branch in the inner loop; the raw-W mma.sync kernel has no 16-bit instantiation.
//
// The kernels are persistent (one CTA per SM, work items = output tiles of up to 16 problems, or in TN mode the
// segments of an even split of all k-blocks of the launch) and fed by one TMA lane through a ring of shared-memory stages (cp.async.bulk.tensor with
// the 128-byte swizzle, mbarrier expect_tx per stage).
//
// tc3_wgmma_kernel: NT with W as pre-split (hi, lo) planes, the model's call pattern.  384 threads, 4-stage ring of
// 48 KB stages, 128 x 128 output tiles:
//   warpgroup 2     TMA producer   raw A tile [128 x 32 fp32] + W_hi and W_lo tiles [128 x 32] per k-block
//                                  (setmaxnreg.dec: one lane issues, the rest idle)
//   warpgroups 0-1  consumers      64 x 128 outputs each (setmaxnreg.inc): per half k-block (2 k-steps) the A
//                                  fragments are read from the swizzled tile and split into (hi, lo) in registers,
//                                  then 6 wgmma.m64n128k8 TF32 (A from registers, W_hi / W_lo straight from shared
//                                  memory through descriptors) into two fp32 register accumulators, one wgmma group.
//                                  The A fragments of the next half are prepared while the group of this one runs; a
//                                  stage is handed back to the producer once the last group that reads it has retired
// tc3_wgmma_dw_kernel: TN (weight gradients).  384 threads, 128 (Nn) x 128 (Kk) output tiles.  Both operands are
// MN-major (row-major activations, reduced over rows) and TF32 wgmma reads shared-memory operands K-major only, so X
// is transposed in shared memory:
//   warpgroup 2     warp 8, one lane: TMA of G and X as [32 rows x 32 floats] boxes (4 + 4 per k-block of 32 rows)
//                   into a 4-stage ring of 32 KB raw stages;
//                   warps 9-11: transpose X into X_hi^T / X_lo^T [128 x 32] K-major tiles with the 128-byte swizzle
//                   (the layout TMA gives the W planes above) in a 3-stage ring of 32 KB plane stages, split with the
//                   same round-to-nearest, reduction rows past the segment / row count written as 0
//   warpgroups 0-1  consumers      64 x 128 outputs each: G^T fragments read in transposed order from the raw boxes and
//                                  split in registers (the bias-gradient partials are summed from them), X planes
//                                  through descriptors; the same half-k-block wgmma pipeline as tc3_wgmma_kernel
// tc3_gemm_kernel: NT with raw fp32 W.  288 threads, 6-stage ring of 24 KB stages, 128 x 64 output tiles:
//   warp 8      TMA producer   raw A tile [128 x 32 fp32] + raw W tile [64 x 32]
//   warps 0-7   consumers      4 (M) x 2 (N) warps, 32 x 32 outputs each: fragments straight from the swizzled tiles
//                              (conflict-free for K-major operands), split into (hi, lo) in registers,
//                              mma.sync.m16n8k8 TF32 into two fp32 register accumulators, one mbarrier arrival per warp
//                              frees the stage
// All three end in the same epilogue from registers (bias / SELU / dSELU / residual and the stores), except
// tc3_wgmma_kernel with a specialised epilogue: a 3-stage ring, and the epilogue through a shared-memory tile buffer
// that warpgroup 2 fills (aux or bias) and drains to C (see the kernel).
//
// Dynamic row counts: a problem may name device ints (m_dev, base_dev) -- the bond-type group sizes written by K0 --
// instead of host values; tile counts are then computed on the device, so the launch needs no device->host read
// and can be captured in a CUDA graph (include/gib200.h, capacity mode).
#include <cuda.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <unordered_map>

#include "gemm.cuh"
#include "tc_ptx.cuh"

namespace gib {

namespace tc3 {

using namespace tcptx;

constexpr int BM = 128, BKF = 32;                 // output tile rows and k-block (one 128-byte swizzle row of fp32)
constexpr int A_BYTES = BM * BKF * 4;             // 16 KB
constexpr int CONS_WARPS = 8;                     // consumer warps of both kernels

// tc3_gemm_kernel (mma.sync).  An SM sub-partition holds 16K registers and receives every fourth warp of the CTA:
// with 9 warps (3 on one sub-partition) a thread may use at most 168, which two register accumulators of 32 x 32
// outputs (64) leave room for.
constexpr int BN = 64;
constexpr int STAGES = 6;
constexpr int B_BYTES = BN * BKF * 4;             // 8 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;   // A raw | W raw
constexpr int NUM_THREADS = 32 * CONS_WARPS + 32;   // 288
constexpr int WM = 32, WN = 32;                   // warp tile
constexpr int MI = WM / 16, NI = WN / 8;          // m16n8k8 MMAs per warp tile and k-step
constexpr int OFF_BARS = STAGES * STAGE_BYTES;
constexpr int OFF_SCHED = OFF_BARS + 256;
constexpr int SMEM_BYTES = OFF_SCHED + 512 + 1024 /*align slack*/;

// tc3_wgmma_kernel.  Register split by setmaxnreg: 256 consumer threads x 232 + 128 producer threads x 40 = 64512 of
// the SM's 65536.  A consumer holds two accumulators of 64 outputs (128 registers) and two buffers of half a
// k-block's A fragments in (hi, lo) (2 x 16).  Buffers of a whole k-block (2 x 32) do not fit beside the
// accumulators: ptxas then serialises every wgmma.
constexpr int WG_BN = 128;
constexpr int WG_STAGES = 4;
constexpr int WG_B_BYTES = WG_BN * BKF * 4;       // 16 KB
constexpr int WG_B16_BYTES = WG_BN * BKF * 2;     // 8 KB: the 16-bit W tile (at the W hi offset of a stage)
constexpr int WG_STAGE_BYTES = A_BYTES + 2 * WG_B_BYTES;   // 48 KB: A raw | W hi | W lo
constexpr int WG_THREADS = 32 * CONS_WARPS + 128;   // 384
constexpr int WG_OFF_BARS = WG_STAGES * WG_STAGE_BYTES;
constexpr int WG_OFF_SCHED = WG_OFF_BARS + 256;
constexpr int WG_SMEM_BYTES = WG_OFF_SCHED + 512 + 1024 /*align slack*/;
static_assert(WG_SMEM_BYTES <= 227 * 1024, "wgmma stages exceed the shared memory of an SM");
// The same kernel with a specialised epilogue (EPI != EPI_SPEC_GENERIC) drains its tiles through shared memory: a
// 3-stage ring, then one 64 KB tile buffer (4 TMA boxes [128 x 32] with the 128-byte swizzle) that receives the aux
// block and is overwritten in place by the results, and the bias slice of the tile.
constexpr int WG_EPI_STAGES = 3;
constexpr int WG_EPI_BUF_BYTES = BM * WG_BN * 4;                    // 64 KB
constexpr int WG_EPI_OFF_BUF = WG_EPI_STAGES * WG_STAGE_BYTES;
constexpr int WG_EPI_OFF_BARS = WG_EPI_OFF_BUF + WG_EPI_BUF_BYTES;
constexpr int WG_EPI_OFF_SCHED = WG_EPI_OFF_BARS + 256;
constexpr int WG_EPI_OFF_BIAS = WG_EPI_OFF_SCHED + 512;
constexpr int WG_EPI_SMEM_BYTES = WG_EPI_OFF_BIAS + WG_BN * 4 + 1024 /*align slack*/;
static_assert(WG_EPI_SMEM_BYTES <= 227 * 1024, "wgmma stages and tile buffer exceed the shared memory of an SM");
constexpr int WG_STORE_WARPS = 2;                                    // warps 10-11

// tc3_wgmma_dw_kernel: 384 threads, registers 256 consumer threads x 224 + 128 producer / transpose threads x 56 =
// 64512 (the transpose holds a 4 x 4 block and its split: ptxas spills it at 48).  Per k-block of 32 reduction rows the raw stage holds
// G [32 x 128 columns] and X [32 x 128 columns] as 4 + 4 boxes of [32 rows x 32 floats]; the plane stage holds
// X_hi^T | X_lo^T [128 x 32], K-major.
constexpr int DW_BN = 128;
constexpr int DW_RAW_STAGES = 4;
constexpr int DW_RAW_BYTES = 2 * A_BYTES;                      // 32 KB: G boxes | X boxes
constexpr int DW_PLANE_STAGES = 3;
constexpr int DW_PLANE_BYTES = 2 * DW_BN * BKF * 4;           // 32 KB: X_hi^T | X_lo^T
constexpr int DW_TR_WARPS = 3;                                 // warps 9-11
constexpr int DW_OFF_PLANES = DW_RAW_STAGES * DW_RAW_BYTES;
constexpr int DW_OFF_BARS = DW_OFF_PLANES + DW_PLANE_STAGES * DW_PLANE_BYTES;
constexpr int DW_OFF_SCHED = DW_OFF_BARS + 256;
constexpr int DW_SCHED_BYTES = 1536;
constexpr int DW_SMEM_BYTES = DW_OFF_SCHED + DW_SCHED_BYTES + 1024 /*align slack*/;
static_assert(DW_SMEM_BYTES <= 227 * 1024, "weight-gradient stages exceed the shared memory of an SM");

constexpr int MAXP = kTc3MaxProblems;   // 16: e.g. the 5 layers x 3 bond types of a message MLP as one dependent chain

struct Maps {   // TMA descriptors in kernel-parameter space
  CUtensorMap a[MAXP];      // NT: activations A (box 128 x 32)    TN: G (box 32 x 32)
  CUtensorMap b[MAXP];      // NT: W hi plane (box 128 x 32) or raw W (box 64 x 32)    TN: X (box 32 x 32)
  CUtensorMap b_lo[MAXP];   // NT: W lo plane (box 128 x 32; pre-split weights only)
  CUtensorMap aux[MAXP];    // NT, EPI_SPEC_DSELU / EPI_SPEC_ADD: aux [M x n_store] (box 128 x 32)
};

struct Params {
  GemmNT g[MAXP];
  int n_tiles[MAXP];        // column tiles of the output: ceil(N / tile width)
  int k_blocks[MAXP];       // ceil(K / 32)
  // dependent chains (NT): problem p reads as its A operand what problem dep[p] writes (the next layer of an MLP);
  // a tile of p at row block i may start once all n_tiles[dep[p]] tiles of row block i of dep[p] are stored.
  // flags[flag_off[p] + i] counts the stored tiles of row block i of problem p (zeroed by the host before the launch).
  int dep[MAXP];
  int flag_off[MAXP];
  int* flags;
  int nprob;
  long long* trace;         // diagnosis: per-tile clock64 stamps of CTA 0 ([tile][16] int64, gib_tc_trace), else nullptr
  int trace_tiles;
};

struct Sched {              // computed once per CTA from host values or the device-side row counts
  int M[MAXP], base[MAXP], begin[MAXP + 1];
};

struct Item { int p, m0, n0, nkb, z, r0, rows, ps; };

// TBN: output tile width of the kernel
template <int TBN>
__device__ __forceinline__ Item decode_item(const Params& P, const Sched& S, int item) {
  Item it;
  int p = 0;
  while (p + 1 < P.nprob && item >= S.begin[p + 1]) ++p;
  const int local = item - S.begin[p];
  it.p = p;
  it.z = 0; it.r0 = 0; it.rows = 0; it.ps = 0;
  it.m0 = (local / P.n_tiles[p]) * BM;
  it.n0 = (local % P.n_tiles[p]) * TBN;
  it.nkb = P.k_blocks[p];
  return it;
}

// ---- schedule of a weight-gradient launch: an even split of its k-blocks (stream-K) -------------------------------
// A work unit is one k-block (32 reduction rows) of one pass of one 128 x 128 output tile of one member; units are
// numbered member-major, then tile, then pass, then k-block, U in all (a member with a pass extent reduces over the same
// rows of each of its passes' slices; a segment may cross a pass boundary and keeps one accumulator across it).  CTA b of G = min(SMs, ceil(U / 8)) takes the units
// [floor(U b / G), floor(U (b + 1) / G)) -- at least one, about U / G -- and cuts them at tile boundaries into
// segments.  The segment of CTA b in tile gt (tile index over the whole group) writes its partial tile to scratch slot
// b + gt: the CTAs that cover one tile are consecutive and a CTA's tiles are consecutive, so no two segments share a
// slot and every slot is below G + T (T: tiles of the group).  The reduction sums, for each tile, the slots of the
// CTAs owner(first unit) .. owner(last unit) in that order.  The split depends on the live row counts, the member
// shapes and the SM count only, never on a buffer's capacity: a launch on device-side row counts computes what the
// same launch on host counts computes, bit for bit.
constexpr int kDwMinUnits = 8;    // k-blocks per CTA at least: amortise the tile drain
constexpr int DW_MAXP = kDwMaxProblems;   // members of one launch (the 15 message-MLP layers and the GRU pair at C2)

struct DwMaps {                   // TMA descriptors of the weight-gradient kernel: G and X, boxes 32 x 32 (x 1)
  CUtensorMap g[DW_MAXP];
  CUtensorMap x[DW_MAXP];
};

struct DwGroup {                  // the schedule inputs of a launch, shared by the GEMM and the reduction
  const int* m_dev[DW_MAXP];         // device-side row count inside a buffer of M rows (nullptr: M is the count)
  const int* base_dev[DW_MAXP];
  int M[DW_MAXP];
  int mt[DW_MAXP], nt[DW_MAXP];         // tiles of the output: ceil(Nn / 128) x ceil(Kk / 128)
  int passes[DW_MAXP];               // slices reduced over (GemmDW::passes)
  int n, sms;
};

struct DwPlan {
  long long U;
  long long ubegin[DW_MAXP + 1];     // first unit of each member
  int tbegin[DW_MAXP + 1];           // first tile of each member
  int M[DW_MAXP], base[DW_MAXP], kb[DW_MAXP], nt[DW_MAXP];   // live rows, first row, k-blocks per pass, column tiles
  int np[DW_MAXP];                   // passes
  int n, G;
};
static_assert(sizeof(DwPlan) <= DW_SCHED_BYTES, "the plan lives in the schedule area of the kernel's shared memory");

// the plan from live row counts (host: the schedule test hook; device: dw_plan_dev)
__host__ __device__ inline void dw_plan(DwPlan& S, const int* live, const int* base, const int* mt, const int* nt,
                                        const int* passes, int n, int sms) {
  long long u = 0;
  int t = 0;
  for (int p = 0; p < n; ++p) {
    S.M[p] = live[p]; S.base[p] = base[p]; S.nt[p] = nt[p]; S.np[p] = passes[p];
    S.kb[p] = ceil_div(live[p], BKF);
    S.ubegin[p] = u; S.tbegin[p] = t;
    u += (long long)mt[p] * nt[p] * S.kb[p] * passes[p];
    t += mt[p] * nt[p];
  }
  S.ubegin[n] = u; S.tbegin[n] = t;
  S.n = n; S.U = u;
  const long long g = ceil_div_ll(u, kDwMinUnits);
  S.G = (int)(g < sms ? g : sms);
}

// the plan of a launch, from its host or device-side row counts (clamped to the buffer as init_sched clamps them)
__device__ inline void dw_plan_dev(const DwGroup& g, DwPlan& S) {
  for (int p = 0; p < g.n; ++p) {   // into S.M / S.base, which dw_plan keeps
    const int base = g.base_dev[p] ? __ldg(g.base_dev[p]) : 0;
    int M = g.M[p];
    if (g.m_dev[p]) {
      M = __ldg(g.m_dev[p]);
      if (M > g.M[p] - base) M = g.M[p] - base;
      if (M < 0) M = 0;
    }
    S.M[p] = M; S.base[p] = base;
  }
  dw_plan(S, S.M, S.base, g.mt, g.nt, g.passes, g.n, g.sms);
}

// units [u0, u1) of CTA b (empty for b >= G)
__host__ __device__ inline void dw_range(const DwPlan& S, int b, long long& u0, long long& u1) {
  if (b >= S.G) { u0 = u1 = 0; return; }
  u0 = S.U * b / S.G;
  u1 = S.U * (b + 1) / S.G;
}

// the CTA whose range holds unit u < U
__host__ __device__ inline int dw_owner(const DwPlan& S, long long u) { return (int)(((u + 1) * S.G - 1) / S.U); }

// k-blocks of one output tile of member p over all its passes
__host__ __device__ inline long long dw_tile_units(const DwPlan& S, int p) { return (long long)S.kb[p] * S.np[p]; }

// the segment of CTA b that starts at unit u < u1 (the end of its range): z = its scratch slot, ps / r0 = the pass and
// the reduction row (relative to the member's first row) of its first k-block, nkb its k-blocks (which continue into
// the next pass at row 0); rows = its reduction rows when it stays inside one pass
__host__ __device__ inline Item dw_segment(const DwPlan& S, int b, long long u, long long u1) {
  int p = 0;
  while (p + 1 < S.n && u >= S.ubegin[p + 1]) ++p;
  const long long local = u - S.ubegin[p];
  const long long tu = dw_tile_units(S, p);
  const int t = (int)(local / tu);
  const int k = (int)(local - (long long)t * tu);   // pass * kb + k-block
  const long long left = u1 - u;
  Item it;
  it.p = p;
  it.m0 = (t / S.nt[p]) * BM;
  it.n0 = (t % S.nt[p]) * DW_BN;
  it.nkb = left < tu - k ? (int)left : (int)(tu - k);
  it.z = b + S.tbegin[p] + t;
  it.ps = k / S.kb[p];
  it.r0 = (k - it.ps * S.kb[p]) * BKF;
  it.rows = S.M[p] - it.r0 < it.nkb * BKF ? S.M[p] - it.r0 : it.nkb * BKF;
  return it;
}

struct DwParams {
  DwGroup grp;
  int Nn[DW_MAXP], Kk[DW_MAXP];
  unsigned bias_mask;             // bit p: member p wants the bias-gradient partials
  float* part;                    // [slots][128][128] partial tiles (row: G column - m0, column: X column - n0)
  float* part_bias;               // [slots][128] partial column sums of G (tiles with n0 == 0)
  long long* trace;               // as Params::trace
  int trace_tiles;
};

// kernel parameters beyond 4 KB: Hopper with CUDA >= 12.1 takes up to 32 764 bytes
static_assert(sizeof(DwMaps) + sizeof(DwParams) <= 32764, "weight-gradient kernel parameters exceed 32 764 bytes");

__device__ __forceinline__ float lds32(uint32_t saddr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr) : "memory");
  return v;
}

// byte offset of element (row r, float c < 32) in a TMA tile of 128-byte rows written with CU_TENSOR_MAP_SWIZZLE_128B:
// 16-byte chunk j of row r sits at chunk j ^ (r & 7) (tile bases are 1024-byte aligned)
__device__ __forceinline__ uint32_t swz(int r, int c) {
  return (uint32_t)r * 128u + ((((uint32_t)c >> 2) ^ (uint32_t)r) & 7u) * 16u + ((uint32_t)c & 3u) * 4u;
}

// byte offset of 16-bit element (row r, value c < 32) in a tile of 64-byte rows written with CU_TENSOR_MAP_SWIZZLE_64B:
// 16-byte chunk j of row r sits at chunk j ^ ((r >> 1) & 3) (tile bases are 512-byte aligned)
__device__ __forceinline__ uint32_t swz64(int r, int c) {
  return (uint32_t)r * 64u + ((((uint32_t)c >> 3) ^ ((uint32_t)r >> 1)) & 3u) * 16u + ((uint32_t)c & 7u) * 2u;
}

__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// Split into TF32 (hi, lo): hi rounded to NEAREST (ties away, what cvt.rna does, as integer arithmetic: + half an ulp
// of the 10-bit mantissa, clear 13 bits; inf stays inf), lo = x - hi exact in fp32 (the tensor core reads its top
// 19 bits).  With hi = trunc(x), lo would always carry the sign of x and its truncation would be a systematic bias
// towards zero that adds up linearly over K; with hi rounded to nearest the sign of lo is random.
__device__ __forceinline__ uint32_t tf32_rn(float x) { return (__float_as_uint(x) + 0x1000u) & 0xffffe000u; }
__device__ __forceinline__ void split_tf32_rn(float x, uint32_t& hi, uint32_t& lo) {
  hi = tf32_rn(x);
  lo = __float_as_uint(x - __uint_as_float(hi));
}
// TF1: hi only (single-pass TF32); lo is left untouched and never read
template <bool TF1>
__device__ __forceinline__ void round_or_split(float x, uint32_t& hi, uint32_t& lo) {
  if constexpr (TF1) hi = tf32_rn(x);
  else split_tf32_rn(x, hi, lo);
}
// the accumulated product: main + cross-term accumulator, or (TF1) the main one alone
template <bool TF1>
__device__ __forceinline__ float acc_total(float acc, float accx) {
  if constexpr (TF1) return acc;
  else return acc + accx;
}

__device__ __forceinline__ void mma_tf32(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// chain hand-off: all THREADS threads that store the tile (named barrier BAR, led by thread LEAD) have stored their
// part -> one release increment of the row block's counter
template <int BAR, int THREADS, int LEAD>
__device__ __forceinline__ void signal_tile(int* flag) {
  fence_proxy_async_all();
  __threadfence();
  asm volatile("bar.sync %0, %1;" ::"n"(BAR), "n"(THREADS) : "memory");
  if (threadIdx.x == LEAD) {
    __threadfence();
    atomicAdd(flag, 1);
  }
}

// EPI: epilogue specialisation shared by every problem of the launch (keeps the per-element code a few instructions)
//   EPI_SPEC_GENERIC   any mode / activation / alignment (run-time branches)
//   EPI_SPEC_SELU      C = selu(acc + bias)          EPI_SPEC_LINEAR  C = acc (+ bias)
//   EPI_SPEC_DSELU     C = acc * selu'(aux)          EPI_SPEC_ADD     C = acc + aux
// The specialised ones need 8-byte aligned column pairs (ldc, ldaux even) and n_store == n_valid, a multiple of 4 --
// the padded-layout contract of every internal buffer.
enum { EPI_SPEC_GENERIC = 0, EPI_SPEC_SELU = 1, EPI_SPEC_LINEAR = 2, EPI_SPEC_DSELU = 3, EPI_SPEC_ADD = 4 };

template <int EPI>
__device__ __forceinline__ float epi_one(float v, float b, float x, int mode, int act) {
  if constexpr (EPI == EPI_SPEC_SELU) return act_fast(v + b, ACT_SELU);
  else if constexpr (EPI == EPI_SPEC_LINEAR) return v + b;
  else if constexpr (EPI == EPI_SPEC_DSELU) return v * dselu_from_out(x);
  else if constexpr (EPI == EPI_SPEC_ADD) return v + x;
  else {
    if (mode == EPI_ACT) return act_fast(v + b, act);
    if (mode == EPI_MUL_DACT) return v * dact_from_out(x, act);
    return v + x;
  }
}

// Schedule of the launch from host values or the device-side row counts (thread 0 only).
__device__ __forceinline__ void init_sched(const Params& P, Sched& S) {
  int total = 0;
  for (int p = 0; p < P.nprob; ++p) {
    const GemmNT& g = P.g[p];
    const int base = g.base_dev ? __ldg(g.base_dev) : 0;
    int M = g.M;
    if (g.m_dev) {                        // device-side row count inside a buffer of g.M rows
      M = __ldg(g.m_dev);
      if (M > g.M - base) M = g.M - base;
      if (M < 0) M = 0;
    }
    S.M[p] = M; S.base[p] = base; S.begin[p] = total;
    total += ceil_div(M, BM) * P.n_tiles[p];
  }
  for (int p = P.nprob; p <= MAXP; ++p) S.begin[p] = total;
}

// dependent chain (NT producer): wait until the row block of the layer below that work item w reads is complete
__device__ __forceinline__ void wait_rows(const Params& P, const Item& w) {
  const int d = P.dep[w.p];
  const int* f = P.flags + P.flag_off[d] + w.m0 / BM;
  const int need = P.n_tiles[d];
  const long long t0 = clock64();
  int have;
  do {
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(have) : "l"(f) : "memory");
    if (have < need) {
      __nanosleep(64);
      if (clock64() - t0 > 20000000000LL) __trap();   // ~10 s: a dead-lock, not contention
    }
  } while (have < need);
  fence_proxy_async_all();               // other SMs' generic-proxy stores -> this SM's async-proxy (TMA) reads
}

// one problem's epilogue operands, resolved once per tile
struct EpiArgs {
  float* C;                // row 0 of the output rows the tile indexes
  const float* X;          // aux, same rows (nullptr: none)
  const float* bias;       // EPI_ACT only
  int ldc, ldaux, n_store, n_valid, Ncols, Mrows, mode, act;
  bool vec_c, vec_x;
};

__device__ __forceinline__ EpiArgs epi_args(const GemmNT& g, float* C, size_t row_base, int Mrows) {
  EpiArgs e;
  e.C = C;
  e.X = g.aux ? g.aux + row_base * g.ldaux : nullptr;
  e.bias = (g.mode == EPI_ACT) ? g.bias : nullptr;
  e.ldc = g.ldc; e.ldaux = g.ldaux; e.n_store = g.n_store; e.n_valid = g.n_valid; e.Ncols = g.N; e.Mrows = Mrows;
  e.mode = g.mode; e.act = g.act;
  e.vec_c = (g.ldc & 1) == 0 && (reinterpret_cast<uintptr_t>(g.C) & 7) == 0;
  e.vec_x = e.X && (g.ldaux & 1) == 0 && (reinterpret_cast<uintptr_t>(g.aux) & 7) == 0;
  return e;
}

// bias of this lane's column pair (n, n + 1), n < n_store
template <int EPI>
__device__ __forceinline__ void epi_bias(const EpiArgs& e, int n, float* b) {
  b[0] = 0.f; b[1] = 0.f;
  if (EPI == EPI_SPEC_SELU || EPI == EPI_SPEC_LINEAR || EPI == EPI_SPEC_GENERIC) {
    if (e.bias) {
      if (n < e.Ncols) b[0] = __ldg(e.bias + n);
      if (n + 1 < e.Ncols) b[1] = __ldg(e.bias + n + 1);
    }
  }
}

// epilogue and store of the accumulated pair v at (row m < Mrows, columns n, n + 1), n < n_store
template <int EPI>
__device__ __forceinline__ void epi_store(const EpiArgs& e, int m, int n, float v0, float v1, const float* b) {
  float v[2] = {v0, v1};
  float x[2] = {0.f, 0.f};
  const bool need_x = (EPI == EPI_SPEC_DSELU || EPI == EPI_SPEC_ADD) || (EPI == EPI_SPEC_GENERIC && e.mode != EPI_ACT);
  if (need_x) {
    const float* ax = e.X + (size_t)m * e.ldaux + n;
    if ((EPI != EPI_SPEC_GENERIC || e.vec_x) && n + 1 < e.n_store) {
      const float2 t2 = __ldg(reinterpret_cast<const float2*>(ax));
      x[0] = t2.x; x[1] = t2.y;
    } else {
      x[0] = ax[0];
      if (n + 1 < e.n_store) x[1] = ax[1];
    }
  }
  v[0] = epi_one<EPI>(v[0], b[0], x[0], e.mode, e.act);
  v[1] = epi_one<EPI>(v[1], b[1], x[1], e.mode, e.act);
  if (EPI == EPI_SPEC_GENERIC) {
    if (n >= e.n_valid) v[0] = 0.f;
    if (n + 1 >= e.n_valid) v[1] = 0.f;
  }
  float* dst = e.C + (size_t)m * e.ldc + n;
  if ((EPI != EPI_SPEC_GENERIC || e.vec_c) && n + 1 < e.n_store) {
    *reinterpret_cast<float2*>(dst) = make_float2(v[0], v[1]);
  } else {
    dst[0] = v[0];
    if (n + 1 < e.n_store) dst[1] = v[1];
  }
}

// ---- mma.sync kernel: NT with raw fp32 W ----
template <int EPI, bool TF1>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tc3_gemm_kernel(const __grid_constant__ Maps maps, const Params P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BARS);
  uint64_t* full = bars;                    // [STAGES] TMA -> consumers
  uint64_t* empty = bars + STAGES;          // [STAGES] consumers -> TMA
  Sched& S = *reinterpret_cast<Sched*>(smem + OFF_SCHED);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CONS_WARPS);     // one arrival per consumer warp (after __syncwarp)
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    init_sched(P, S);
  }
  __syncthreads();
  const int num_items = S.begin[MAXP];

  if (warp == CONS_WARPS) {
    // ================= TMA producer =================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const Item w = decode_item<BN>(P, S, item);
        const int base = S.base[w.p];
        if (P.flags && P.dep[w.p] >= 0) wait_rows(P, w);
        for (int kb = 0; kb < w.nkb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* st = smem + stage * STAGE_BYTES;
          mbar_arrive_expect_tx(&full[stage], A_BYTES + B_BYTES);
          tma_load_2d(&maps.a[w.p], &full[stage], st, kb * BKF, base + w.m0);
          tma_load_2d(&maps.b[w.p], &full[stage], st + A_BYTES, kb * BKF, w.n0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ================= consumers: fragments -> (hi, lo) -> mma.sync -> epilogue =================
    const int wm = warp >> 1, wn = warp & 1;     // 4 x 2 warps
    const int g8 = lane >> 2, t4 = lane & 3;     // mma fragment coordinates
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x, ++it) {
      const Item w = decode_item<BN>(P, S, item);
      const bool tr = P.trace && blockIdx.x == 0 && it < P.trace_tiles && threadIdx.x == 0;
      if (tr) P.trace[it * 16 + 0] = clock64();
      float acc[MI][NI][4], accx[MI][NI][4];
#pragma unroll
      for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NI; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) { acc[i][j][e] = 0.f; accx[i][j][e] = 0.f; }

      for (int kb = 0; kb < w.nkb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
        const uint32_t sb = sa + A_BYTES;
#pragma unroll
        for (int ks = 0; ks < BKF / 8; ++ks) {
          const int k0 = ks * 8 + t4, k1 = k0 + 4;
          // B fragments of the k-step for all NI column blocks, then the A rows one 16-row block at a time
          uint32_t bh[NI][2], bl[NI][2];
#pragma unroll
          for (int j = 0; j < NI; ++j) {
            const int n = wn * WN + j * 8 + g8;
            round_or_split<TF1>(lds32(sb + swz(n, k0)), bh[j][0], bl[j][0]);
            round_or_split<TF1>(lds32(sb + swz(n, k1)), bh[j][1], bl[j][1]);
          }
#pragma unroll
          for (int i = 0; i < MI; ++i) {
            const int r0 = wm * WM + i * 16 + g8, r1 = r0 + 8;
            float a[4];
            a[0] = lds32(sa + swz(r0, k0)); a[1] = lds32(sa + swz(r1, k0));
            a[2] = lds32(sa + swz(r0, k1)); a[3] = lds32(sa + swz(r1, k1));
            uint32_t ahi[4], alo[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) round_or_split<TF1>(a[e], ahi[e], alo[e]);
#pragma unroll
            for (int j = 0; j < NI; ++j) {
              mma_tf32(acc[i][j], ahi, bh[j][0], bh[j][1]);
              if constexpr (!TF1) {
                mma_tf32(accx[i][j], alo, bh[j][0], bh[j][1]);
                mma_tf32(accx[i][j], ahi, bl[j][0], bl[j][1]);
              }
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);   // this warp is done with the stage
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }

      const GemmNT& g = P.g[w.p];
      const int Mrows = S.M[w.p];
      const size_t row_base = (size_t)S.base[w.p];
      const EpiArgs e = epi_args(g, g.C + row_base * g.ldc, row_base, Mrows);
#pragma unroll
      for (int j = 0; j < NI; ++j) {
        const int n = w.n0 + wn * WN + j * 8 + 2 * t4;    // this lane's column pair
        if (n >= e.n_store) continue;
        float b[2];
        epi_bias<EPI>(e, n, b);
#pragma unroll
        for (int i = 0; i < MI; ++i)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int m = w.m0 + wm * WM + i * 16 + h * 8 + g8;
            if (m >= Mrows) continue;
            epi_store<EPI>(e, m, n, acc_total<TF1>(acc[i][j][2 * h], accx[i][j][2 * h]),
                           acc_total<TF1>(acc[i][j][2 * h + 1], accx[i][j][2 * h + 1]), b);
          }
      }
      if (P.flags) signal_tile<1, 32 * CONS_WARPS, 0>(P.flags + P.flag_off[w.p] + w.m0 / BM);
      if (tr) P.trace[it * 16 + 6] = clock64();
    }
  }
}

__device__ __forceinline__ void lds64(uint32_t saddr, float& x, float& y) {
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(x), "=f"(y) : "r"(saddr) : "memory");
}
__device__ __forceinline__ void sts64(uint32_t saddr, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(saddr), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr) : "memory");
  return v;
}

// byte offset of output element (row r, column c < 128) in the tile buffer: box c / 32, swizzled as TMA writes it
__device__ __forceinline__ uint32_t epi_off(int r, int c) { return (uint32_t)(c >> 5) * (BM * BKF * 4) + swz(r, c & 31); }

// 16-bit A fragments of one k-block (two k16 steps) for rows r0, r0 + 8 (r0 & 7 = g) from the fp32 activation tile at
// sa: f[s] = the m16n8k16 fragment of k16 step s.  A lane reads its four column pairs (step s, half h: columns
// 16 s + 8 h + 2t, +1) of a row as 8-byte loads, in a lane-dependent order -- load i takes (s, h) = (i1 ^ g1, i0 ^ g0)
// -- so that the 16 lanes of each half-warp phase (g < 4 or g >= 4, t < 4) hit 16 distinct 8-byte slots: with the
// 128-byte swizzle the chunk index is (4 s + 2 h + t1) ^ g, whose bits are (i1 ^ g1 ^ g2, i0 ^ g0 ^ g1, t1 ^ g0), a
// bijection of (g1, g0, t1); in natural order lanes g and g ^ 1 would share chunks (2-way conflicts).  Two selects per
// register then undo the permutation.
template <int H16>
__device__ __forceinline__ void a_frags16(uint32_t sa, int r0, int g, int t4, uint32_t (&f)[2][4]) {
  const bool g0 = g & 1, g1 = (g >> 1) & 1;
#pragma unroll
  for (int h8 = 0; h8 < 2; ++h8) {
    uint32_t q[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int s = (i >> 1) ^ (int)g1, hh = (i & 1) ^ (int)g0;
      float x, y;
      lds64(sa + swz(r0 + 8 * h8, 16 * s + 8 * hh + 2 * t4), x, y);
      q[i] = pack16<H16>(x, y);
    }
    const uint32_t p0 = g0 ? q[1] : q[0], p1 = g0 ? q[0] : q[1], p2 = g0 ? q[3] : q[2], p3 = g0 ? q[2] : q[3];
    f[0][h8] = g1 ? p2 : p0;          // (s 0, h 0)
    f[0][2 + h8] = g1 ? p3 : p1;      // (s 0, h 1)
    f[1][h8] = g1 ? p0 : p2;          // (s 1, h 0)
    f[1][2 + h8] = g1 ? p1 : p3;      // (s 1, h 1)
  }
}

// ---- wgmma kernel: NT with pre-split W ----
//
// With a specialised epilogue (SE) the consumers only touch registers and shared memory between a tile's last wgmma
// and the next tile's first; warpgroup 2 does the global-memory side of the epilogue:
//   warp 8, lane 0    k-block TMA (as in the generic kernel)
//   warp 9            epilogue operands of tile t into the tile buffer once the stores of tile t - 1 have drained it:
//                     the aux block by TMA (DSELU / ADD; rows past the map and columns >= n_store zero-filled), or the
//                     bias slice by plain loads (SELU / LINEAR) -> epi_full
//   warps 0-7         epi(acc + accx) in place over the tile buffer -> epi_done
//   warps 10-11       tile buffer -> C with 16-byte stores (rows < the live row count, columns < n_store) -> epi_empty,
//                     then the chain hand-off of the tile.  They wait on nothing but epi_done, so a chain cannot
//                     dead-lock on them.
// H16 (bf16 / fp16 operands, instantiated with TF1 = true: one accumulator): W is the 16-bit plane, one 8 KB box per
// k-block at the W hi offset of the stage, and the consumers issue one group of 2 k16 wgmma per k-block.
template <int EPI, bool TF1, int H16 = 0>
__global__ void __launch_bounds__(WG_THREADS, 1)
tc3_wgmma_kernel(const __grid_constant__ Maps maps, const Params P) {
  static_assert(H16 == 0 || TF1, "16-bit operands use the single accumulator");
  constexpr bool SE = EPI != EPI_SPEC_GENERIC;
  constexpr bool AUX = EPI == EPI_SPEC_DSELU || EPI == EPI_SPEC_ADD;
  constexpr int NST = SE ? WG_EPI_STAGES : WG_STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (SE ? WG_EPI_OFF_BARS : WG_OFF_BARS));
  uint64_t* full = bars;                    // [NST] TMA -> consumers
  uint64_t* empty = bars + NST;             // [NST] consumers -> TMA
  uint64_t* epi_full = bars + 2 * NST;      // SE: epilogue operands of the tile are in the buffer
  uint64_t* epi_done = epi_full + 1;        // SE: results of the tile are in the buffer
  uint64_t* epi_empty = epi_full + 2;       // SE: the buffer is drained
  Sched& S = *reinterpret_cast<Sched*>(smem + (SE ? WG_EPI_OFF_SCHED : WG_OFF_SCHED));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NST; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CONS_WARPS);     // one arrival per consumer warp, once its wgmma group has retired
    }
    if (SE) {
      mbar_init(epi_full, 1);
      mbar_init(epi_done, CONS_WARPS);
      mbar_init(epi_empty, WG_STORE_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    init_sched(P, S);
  }
  __syncthreads();
  const int num_items = S.begin[MAXP];

  if (warp >= CONS_WARPS) {
    // ================= warpgroup 2: TMA producer, epilogue operands, stores =================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == CONS_WARPS && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const Item w = decode_item<WG_BN>(P, S, item);
        const int base = S.base[w.p];
        if (P.flags && P.dep[w.p] >= 0) wait_rows(P, w);
        for (int kb = 0; kb < w.nkb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* st = smem + stage * WG_STAGE_BYTES;
          mbar_arrive_expect_tx(&full[stage], H16 ? A_BYTES + WG_B16_BYTES : TF1 ? A_BYTES + WG_B_BYTES : WG_STAGE_BYTES);
          tma_load_2d(&maps.a[w.p], &full[stage], st, kb * BKF, base + w.m0);
          tma_load_2d(&maps.b[w.p], &full[stage], st + A_BYTES, kb * BKF, w.n0);
          if (!TF1) tma_load_2d(&maps.b_lo[w.p], &full[stage], st + A_BYTES + WG_B_BYTES, kb * BKF, w.n0);
          if (++stage == NST) { stage = 0; phase ^= 1; }
        }
      }
    } else if (SE && warp == CONS_WARPS + 1) {
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x, phase ^= 1) {
        const Item w = decode_item<WG_BN>(P, S, item);
        const GemmNT& g = P.g[w.p];
        mbar_wait(epi_empty, phase ^ 1);
        if constexpr (AUX) {
          if (lane == 0) {
            if (P.flags && P.dep[w.p] >= 0) wait_rows(P, w);   // aux is read no earlier than the A operand
            const int boxes = min(WG_BN / BKF, ceil_div(g.n_store - w.n0, BKF));
            mbar_arrive_expect_tx(epi_full, boxes * A_BYTES);
            for (int b = 0; b < boxes; ++b)
              tma_load_2d(&maps.aux[w.p], epi_full, smem + WG_EPI_OFF_BUF + b * A_BYTES, w.n0 + b * BKF,
                          S.base[w.p] + w.m0);
          }
        } else {
          const float* bias = g.bias;
          float* sb = reinterpret_cast<float*>(smem + WG_EPI_OFF_BIAS);
          for (int c = lane; c < WG_BN; c += 32) {
            const int n = w.n0 + c;
            sb[c] = (bias && n < g.N) ? __ldg(bias + n) : 0.f;
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(epi_full);
        }
      }
    } else if (SE && warp >= CONS_WARPS + 2) {
      const int sw = warp - (CONS_WARPS + 2);   // store warp 0 / 1: rows sw, sw + 2, ...
      uint32_t phase = 0;
      int it = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x, phase ^= 1, ++it) {
        const Item w = decode_item<WG_BN>(P, S, item);
        const GemmNT& g = P.g[w.p];
        const int rows = min(BM, S.M[w.p] - w.m0);
        const int chunks = min(WG_BN, g.n_store - w.n0) >> 2;    // 16-byte chunks per row (n_store % 4 == 0)
        float* C = g.C + ((size_t)S.base[w.p] + w.m0) * g.ldc + w.n0 + 4 * lane;
        const uint32_t src = smem_u32(smem + WG_EPI_OFF_BUF) + (uint32_t)(lane >> 3) * (BM * BKF * 4);
        mbar_wait(epi_done, phase);
        if (lane < chunks) {
#pragma unroll 2
          for (int r = sw; r < rows; r += WG_STORE_WARPS) {
            const float4 v = lds128(src + swz(r, 4 * (lane & 7)));
            *reinterpret_cast<float4*>(C + (size_t)r * g.ldc) = v;
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic reads of the buffer -> next TMA write
        __syncwarp();
        if (lane == 0) mbar_arrive(epi_empty);
        if (P.flags) signal_tile<2, 32 * WG_STORE_WARPS, 32 * (CONS_WARPS + 2)>(P.flags + P.flag_off[w.p] + w.m0 / BM);
        if (P.trace && blockIdx.x == 0 && it < P.trace_tiles && threadIdx.x == 32 * (CONS_WARPS + 2))
          P.trace[it * 16 + 3] = clock64();
      }
    }
  } else {
    // ================= consumers (warpgroups 0-1): A fragments -> (hi, lo) -> wgmma -> epilogue =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int g8 = lane >> 2, t4 = lane & 3;     // fragment coordinates
    const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + g8;   // this lane's A / output rows in the tile: r0, r0 + 8
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x, ++it) {
      const Item w = decode_item<WG_BN>(P, S, item);
      const bool tr = P.trace && blockIdx.x == 0 && it < P.trace_tiles && threadIdx.x == 0;
      if (tr) P.trace[it * 16 + 0] = clock64();
      float acc[64], accx[64];
#pragma unroll
      for (int e = 0; e < 64; ++e) { acc[e] = 0.f; accx[e] = 0.f; }

      // A fragments are staged half a k-block (2 k-steps) at a time in two register buffers: half 0 of every k-block
      // in (ah0, al0), half 1 in (ah1, al1), each followed by its 6 wgmma as one group.  wait_group 1 after each
      // commit retires the group before it, so a buffer is rewritten only after the group that read it has retired,
      // and the stage of k-block kb - 1 goes back to the producer once the group of its half 1 has retired (in
      // half 0 of k-block kb) -- while the A fragments of the next half are prepared, a group is in flight.
      uint32_t ah0[2][4], al0[2][4], ah1[2][4], al1[2][4];
      int prev = -1;
      auto half = [&](uint32_t sa, int hk, uint32_t (&ah)[2][4], uint32_t (&al)[2][4]) {
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          const int k0 = (2 * hk + s) * 8 + t4, k1 = k0 + 4;
          round_or_split<TF1>(lds32(sa + swz(r0, k0)), ah[s][0], al[s][0]);
          round_or_split<TF1>(lds32(sa + swz(r0 + 8, k0)), ah[s][1], al[s][1]);
          round_or_split<TF1>(lds32(sa + swz(r0, k1)), ah[s][2], al[s][2]);
          round_or_split<TF1>(lds32(sa + swz(r0 + 8, k1)), ah[s][3], al[s][3]);
        }
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          const uint32_t ko = (2 * hk + s) * 32;
          const uint64_t dh = wgmma_desc_sw128(sa + A_BYTES + ko);
          wgmma_m64n128k8_tf32(acc, ah[s], dh);
          if constexpr (!TF1) {
            const uint64_t dl = wgmma_desc_sw128(sa + A_BYTES + WG_B_BYTES + ko);
            wgmma_m64n128k8_tf32(accx, al[s], dh);
            wgmma_m64n128k8_tf32(accx, ah[s], dl);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
      };
      // H16: a whole k-block's fragments per buffer and group (even k-blocks in f0, odd in f1), the same wait_group 1
      // discipline: the group of k-block kb - 1 has retired once that of kb is committed, and its stage goes back
      uint32_t f0[2][4], f1[2][4];
      auto kblock16 = [&](uint32_t sa, uint32_t (&f)[2][4]) {
        a_frags16<H16 ? H16 : 1>(sa, r0, g8, t4, f);
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < 2; ++s) wgmma_m64n128k16_h16<H16 ? H16 : 1>(acc, f[s], wgmma_desc_sw64(sa + A_BYTES + s * 32));
        wgmma_commit();
        wgmma_wait<1>();
      };
      for (int kb = 0; kb < w.nkb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * WG_STAGE_BYTES);
        if constexpr (H16) {
          if (kb & 1) kblock16(sa, f1);
          else kblock16(sa, f0);
        } else {
          half(sa, 0, ah0, al0);
        }
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[prev]);
        }
        if constexpr (!H16) half(sa, 1, ah1, al1);
        prev = stage;
        if (++stage == NST) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev]);
      if (tr) P.trace[it * 16 + 1] = clock64();

      if constexpr (SE) {
        // epi(acc + accx) in place over the tile buffer: each lane reads (aux) and writes its own column pairs
        mbar_wait(epi_full, it & 1);
        const uint32_t ebuf = smem_u32(smem + WG_EPI_OFF_BUF), ebias = smem_u32(smem + WG_EPI_OFF_BIAS);
#pragma unroll
        for (int j = 0; j < WG_BN / 8; ++j) {
          const int c = j * 8 + 2 * t4;
          float b[2] = {0.f, 0.f};
          if (!AUX) lds64(ebias + c * 4, b[0], b[1]);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t a = ebuf + epi_off(r0 + h * 8, c);
            float x[2] = {0.f, 0.f};
            if (AUX) lds64(a, x[0], x[1]);
            sts64(a, epi_one<EPI>(acc_total<TF1>(acc[4 * j + 2 * h], accx[4 * j + 2 * h]), b[0], x[0], 0, 0),
                  epi_one<EPI>(acc_total<TF1>(acc[4 * j + 2 * h + 1], accx[4 * j + 2 * h + 1]), b[1], x[1], 0, 0));
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(epi_done);
        if (tr) P.trace[it * 16 + 2] = clock64();
        continue;
      }

      const GemmNT& g = P.g[w.p];
      const int Mrows = S.M[w.p];
      const size_t row_base = (size_t)S.base[w.p];
      const EpiArgs e = epi_args(g, g.C + row_base * g.ldc, row_base, Mrows);
#pragma unroll
      for (int j = 0; j < WG_BN / 8; ++j) {
        const int n = w.n0 + j * 8 + 2 * t4;      // this lane's column pair
        if (n >= e.n_store) continue;
        float b[2];
        epi_bias<EPI>(e, n, b);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = w.m0 + r0 + h * 8;
          if (m >= Mrows) continue;
          epi_store<EPI>(e, m, n, acc_total<TF1>(acc[4 * j + 2 * h], accx[4 * j + 2 * h]),
                         acc_total<TF1>(acc[4 * j + 2 * h + 1], accx[4 * j + 2 * h + 1]), b);
        }
      }
      if (P.flags) signal_tile<1, 32 * CONS_WARPS, 0>(P.flags + P.flag_off[w.p] + w.m0 / BM);
      if (tr) P.trace[it * 16 + 6] = clock64();
    }
  }
}

__device__ __forceinline__ void sts128(uint32_t saddr, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}

// One 4 x 4 block of the X transpose: reduction rows k = 4a .. 4a + 3 of the raw X boxes at sx (valid: rows below it
// are live; the others may hold anything, NaN included, and are written as 0) x columns n = 4b .. 4b + 3 of the tile,
// into rows n, chunk a of the K-major (hi, lo) planes at sp.  Block t of the 256 of a k-block:
//   t bits 0-2 = l, bits 3-4 = b >> 3 (the box), bit 5 = a >> 2, bits 6-7 = u;  b = 8 (b >> 3) + l,
//   a = 4 (a >> 2) + 2 (l2 ^ u1) + (l1 ^ u0).
// A 128-bit shared access is served 8 lanes at a time, and the 8 lanes of a group share everything but l: the raw
// row k sits at 16-byte chunk l ^ (k & 7) with k & 7 = 4 (l1 ^ u0) + i, the plane row n = 4b + j at a ^ (n & 7) with
// n & 7 = 4 l0 + j -- both take 8 distinct values over l, so reads and writes are free of bank conflicts.
// TF1: the X_hi^T plane only.
template <bool TF1>
__device__ __forceinline__ void dw_transpose_block(uint32_t sx, uint32_t sp, int t, int valid) {
  const int l = t & 7, u = t >> 6;
  const int b = ((t >> 3) & 3) * 8 + l;
  const int a = ((t >> 5) & 1) * 4 + ((((l >> 2) ^ (u >> 1)) & 1) << 1) + (((l >> 1) ^ u) & 1);
  float4 v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = 4 * a + i;
    v[i] = lds128(sx + (b >> 3) * 4096 + swz(k, 4 * (b & 7)));
    if (k >= valid) v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      round_or_split<TF1>(j == 0 ? v[i].x : j == 1 ? v[i].y : j == 2 ? v[i].z : v[i].w, hi[i], lo[i]);
    const uint32_t o = swz(4 * b + j, 4 * a);
    sts128(sp + o, hi[0], hi[1], hi[2], hi[3]);
    if (!TF1) sts128(sp + DW_BN * BKF * 4 + o, lo[0], lo[1], lo[2], lo[3]);
  }
}

// The same 4 x 4 block into the 16-bit K-major X^T plane (64-byte rows, 64-byte swizzle, swz64): the four reduction
// rows of plane row n = 4b + j are one 8-byte store.  The raw reads are those above; the stores of a group of 8 lanes
// take 8 distinct 8-byte slots of one 64-byte bank range (the chunk (a >> 1) ^ (n >> 1) and the half a & 1 take 8
// values over l), and the two groups of a half-warp phase share it: 2-way, on half the bytes the TF32 planes store.
template <int H16>
__device__ __forceinline__ void dw_transpose_block16(uint32_t sx, uint32_t sp, int t, int valid) {
  const int l = t & 7, u = t >> 6;
  const int b = ((t >> 3) & 3) * 8 + l;
  const int a = ((t >> 5) & 1) * 4 + ((((l >> 2) ^ (u >> 1)) & 1) << 1) + (((l >> 1) ^ u) & 1);
  float4 v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = 4 * a + i;
    v[i] = lds128(sx + (b >> 3) * 4096 + swz(k, 4 * (b & 7)));
    if (k >= valid) v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  auto c = [](const float4& x, int j) { return j == 0 ? x.x : j == 1 ? x.y : j == 2 ? x.z : x.w; };
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t lo = pack16<H16>(c(v[0], j), c(v[1], j)), hi = pack16<H16>(c(v[2], j), c(v[3], j));
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(sp + swz64(4 * b + j, 4 * a)), "r"(lo), "r"(hi) : "memory");
  }
}

// ---- wgmma kernel: TN (weight-gradient partials) ----
// H16 (instantiated with TF1 = true): G fragments rounded in registers, X transposed into one 16-bit plane, one group
// of 2 k16 wgmma per k-block.
template <bool TF1, int H16 = 0>
__global__ void __launch_bounds__(WG_THREADS, 1)
tc3_wgmma_dw_kernel(const __grid_constant__ DwMaps maps, const DwParams P) {
  static_assert(H16 == 0 || TF1, "16-bit operands use the single accumulator");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + DW_OFF_BARS);
  uint64_t* raw_full = bars;                            // [DW_RAW_STAGES] TMA -> consumers (G), transposers (X)
  uint64_t* raw_empty = raw_full + DW_RAW_STAGES;       // [DW_RAW_STAGES] consumers + transposers -> TMA
  uint64_t* pl_full = raw_empty + DW_RAW_STAGES;        // [DW_PLANE_STAGES] transposers -> consumers
  uint64_t* pl_empty = pl_full + DW_PLANE_STAGES;       // [DW_PLANE_STAGES] consumers -> transposers
  DwPlan& S = *reinterpret_cast<DwPlan*>(smem + DW_OFF_SCHED);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < DW_RAW_STAGES; ++s) {
      mbar_init(&raw_full[s], 1);
      mbar_init(&raw_empty[s], CONS_WARPS + DW_TR_WARPS);
    }
    for (int s = 0; s < DW_PLANE_STAGES; ++s) {
      mbar_init(&pl_full[s], DW_TR_WARPS);
      mbar_init(&pl_empty[s], CONS_WARPS);   // once the last wgmma group reading the planes has retired
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    dw_plan_dev(P.grp, S);
  }
  __syncthreads();
  // every role walks the same segments: this CTA's units [u0, u1), cut at tile boundaries
  long long u0, u1;
  dw_range(S, blockIdx.x, u0, u1);

  if (warp >= CONS_WARPS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
    if (warp == CONS_WARPS) {
      // ================= TMA producer =================
      if (lane == 0) {
        int stage = 0;
        uint32_t phase = 0;
        for (long long u = u0; u < u1;) {
          const Item w = dw_segment(S, blockIdx.x, u, u1);
          u += w.nkb;
          int row = S.base[w.p] + w.r0, pass = w.ps;
          const int row_end = S.base[w.p] + S.kb[w.p] * BKF;
          for (int kb = 0; kb < w.nkb; ++kb) {
            mbar_wait(&raw_empty[stage], phase ^ 1);
            uint8_t* st = smem + stage * DW_RAW_BYTES;
            mbar_arrive_expect_tx(&raw_full[stage], DW_RAW_BYTES);
#pragma unroll
            for (int j = 0; j < BM / 32; ++j)          // 32-float column groups of G
              tma_load_3d(&maps.g[w.p], &raw_full[stage], st + j * 4096, w.m0 + 32 * j, row, pass);
#pragma unroll
            for (int j = 0; j < DW_BN / 32; ++j)       // and of X
              tma_load_3d(&maps.x[w.p], &raw_full[stage], st + A_BYTES + j * 4096, w.n0 + 32 * j, row, pass);
            if (++stage == DW_RAW_STAGES) { stage = 0; phase ^= 1; }
            row += BKF;
            if (row == row_end) { row = S.base[w.p]; ++pass; }   // the next pass's slice, same rows
          }
        }
      }
    } else {
      // ================= transposers: raw X -> (X_hi^T, X_lo^T) planes =================
      const int tt = threadIdx.x - 32 * (CONS_WARPS + 1);
      int rs = 0, ps = 0;
      uint32_t rph = 0, pph = 0;
      for (long long u = u0; u < u1;) {
        const Item w = dw_segment(S, blockIdx.x, u, u1);
        u += w.nkb;
        int valid = S.M[w.p] - w.r0;                // live rows from the k-block's first row on
        for (int kb = 0; kb < w.nkb; ++kb) {
          mbar_wait(&pl_empty[ps], pph ^ 1);
          mbar_wait(&raw_full[rs], rph);
          const uint32_t sx = smem_u32(smem + rs * DW_RAW_BYTES + A_BYTES);
          const uint32_t sp = smem_u32(smem + DW_OFF_PLANES + ps * DW_PLANE_BYTES);
          for (int t = tt; t < 256; t += 32 * DW_TR_WARPS) {
            if constexpr (H16) dw_transpose_block16<H16>(sx, sp, t, valid);
            else dw_transpose_block<TF1>(sx, sp, t, valid);
          }
          valid -= BKF;
          if (valid <= 0) valid = S.M[w.p];        // next pass (a segment's k-blocks all hold live rows)
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> wgmma reads
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(&raw_empty[rs]);
            mbar_arrive(&pl_full[ps]);
          }
          if (++rs == DW_RAW_STAGES) { rs = 0; rph ^= 1; }
          if (++ps == DW_PLANE_STAGES) { ps = 0; pph ^= 1; }
        }
      }
    }
  } else {
    // ================= consumers (warpgroups 0-1): G^T fragments -> (hi, lo) -> wgmma -> partials =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
    const int g8 = lane >> 2, t4 = lane & 3;     // fragment coordinates
    const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + g8;   // this lane's G columns / output rows: r0, r0 + 8
    // element (reduction row k, G column r) of the raw stage: box r / 32, swizzled row k
    const uint32_t go0 = (r0 >> 5) * 4096, go1 = ((r0 + 8) >> 5) * 4096;
    const int c0 = r0 & 31, c1 = (r0 + 8) & 31;
    int rs = 0, ps = 0;
    uint32_t rph = 0, pph = 0;
    int it = 0;
    for (long long u = u0; u < u1; ++it) {
      const Item w = dw_segment(S, blockIdx.x, u, u1);
      u += w.nkb;
      const bool tr = P.trace && blockIdx.x == 0 && it < P.trace_tiles && threadIdx.x == 0;
      if (tr) P.trace[it * 16 + 0] = clock64();
      float acc[64], accx[64];
#pragma unroll
      for (int e = 0; e < 64; ++e) { acc[e] = 0.f; accx[e] = 0.f; }
      float cs0 = 0.f, cs1 = 0.f;                // bias-gradient partials of this lane's G columns
      const bool want_cs = ((P.bias_mask >> w.p) & 1u) && w.n0 == 0;

      // the pipeline of tc3_wgmma_kernel: half a k-block of fragments per buffer and wgmma group, wait_group 1; the
      // raw stage (G only) is released as soon as the fragments of its half 1 are in registers, the plane stage once
      // the group of its half 1 has retired
      uint32_t ah0[2][4], al0[2][4], ah1[2][4], al1[2][4];
      int prev = -1;
      auto half = [&](uint32_t sg, uint32_t sp, int valid, int hk, uint32_t (&ah)[2][4], uint32_t (&al)[2][4]) {
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          const int k0 = (2 * hk + s) * 8 + t4, k1 = k0 + 4;
          float a[4];
          a[0] = lds32(sg + go0 + swz(k0, c0)); a[1] = lds32(sg + go1 + swz(k0, c1));
          a[2] = lds32(sg + go0 + swz(k1, c0)); a[3] = lds32(sg + go1 + swz(k1, c1));
          if (k0 >= valid) { a[0] = 0.f; a[1] = 0.f; }   // rows past the segment / row count may hold anything
          if (k1 >= valid) { a[2] = 0.f; a[3] = 0.f; }
          if (want_cs) { cs0 += a[0] + a[2]; cs1 += a[1] + a[3]; }
#pragma unroll
          for (int e = 0; e < 4; ++e) round_or_split<TF1>(a[e], ah[s][e], al[s][e]);
        }
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          const uint32_t ko = (2 * hk + s) * 32;
          const uint64_t dh = wgmma_desc_sw128(sp + ko);
          wgmma_m64n128k8_tf32(acc, ah[s], dh);
          if constexpr (!TF1) {
            const uint64_t dl = wgmma_desc_sw128(sp + DW_BN * BKF * 4 + ko);
            wgmma_m64n128k8_tf32(accx, al[s], dh);
            wgmma_m64n128k8_tf32(accx, ah[s], dl);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
      };
      // H16: a whole k-block per buffer and group (even k-blocks in f0, odd in f1).  Fragment register 2h + e of k16
      // step s holds G column r0 + 8e at reduction rows k = 16 s + 8 h + 2t, +1; these 4-byte reads are free of bank
      // conflicts (chunk (c >> 2) ^ (k & 7) with k & 7 = 2t + const: 8 distinct chunks over (g >> 2, t)).
      uint32_t f0[2][4], f1[2][4];
      auto kblock16 = [&](uint32_t sg, uint32_t sp, int valid, uint32_t (&f)[2][4]) {
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int k = 16 * s + 8 * h + 2 * t4;
            float a[4];
            a[0] = lds32(sg + go0 + swz(k, c0)); a[1] = lds32(sg + go0 + swz(k + 1, c0));
            a[2] = lds32(sg + go1 + swz(k, c1)); a[3] = lds32(sg + go1 + swz(k + 1, c1));
            if (k >= valid) { a[0] = 0.f; a[2] = 0.f; }     // rows past the segment / row count may hold anything
            if (k + 1 >= valid) { a[1] = 0.f; a[3] = 0.f; }
            if (want_cs) { cs0 += a[0] + a[1]; cs1 += a[2] + a[3]; }
            f[s][2 * h] = pack16<H16 ? H16 : 1>(a[0], a[1]);
            f[s][2 * h + 1] = pack16<H16 ? H16 : 1>(a[2], a[3]);
          }
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < 2; ++s) wgmma_m64n128k16_h16<H16 ? H16 : 1>(acc, f[s], wgmma_desc_sw64(sp + s * 32));
        wgmma_commit();
        wgmma_wait<1>();
      };
      int valid = S.M[w.p] - w.r0;                // live rows from the k-block's first row on (as the transposers)
      for (int kb = 0; kb < w.nkb; ++kb) {
        mbar_wait(&raw_full[rs], rph);
        mbar_wait(&pl_full[ps], pph);
        const uint32_t sg = smem_u32(smem + rs * DW_RAW_BYTES);
        const uint32_t sp = smem_u32(smem + DW_OFF_PLANES + ps * DW_PLANE_BYTES);
        if constexpr (H16) {
          if (kb & 1) kblock16(sg, sp, valid, f1);
          else kblock16(sg, sp, valid, f0);
        } else {
          half(sg, sp, valid, 0, ah0, al0);
        }
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&pl_empty[prev]);
        }
        if constexpr (!H16) half(sg, sp, valid, 1, ah1, al1);
        __syncwarp();
        if (lane == 0) mbar_arrive(&raw_empty[rs]);
        prev = ps;
        if (++rs == DW_RAW_STAGES) { rs = 0; rph ^= 1; }
        if (++ps == DW_PLANE_STAGES) { ps = 0; pph ^= 1; }
        valid -= BKF;
        if (valid <= 0) valid = S.M[w.p];
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&pl_empty[prev]);

      // the partial tile into the segment's slot, at tile-local coordinates
      const int Nn = P.Nn[w.p], Kk = P.Kk[w.p];
      if (want_cs) {
        float* bp = P.part_bias + (size_t)w.z * BM;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float s = h ? cs1 : cs0;
          s += __shfl_xor_sync(0xffffffffu, s, 1);
          s += __shfl_xor_sync(0xffffffffu, s, 2);
          const int m = r0 + h * 8;
          if (t4 == 0 && w.m0 + m < Nn) bp[m] = s;
        }
      }
      float* const out = P.part + (size_t)w.z * (BM * DW_BN);
#pragma unroll
      for (int j = 0; j < DW_BN / 8; ++j) {
        const int n = j * 8 + 2 * t4;             // this lane's column pair (Kk % 4 == 0: both valid or neither)
        if (w.n0 + n >= Kk) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = r0 + h * 8;
          if (w.m0 + m >= Nn) continue;
          *reinterpret_cast<float2*>(out + m * DW_BN + n) =
              make_float2(acc_total<TF1>(acc[4 * j + 2 * h], accx[4 * j + 2 * h]),
                          acc_total<TF1>(acc[4 * j + 2 * h + 1], accx[4 * j + 2 * h + 1]));
        }
      }
      if (tr) P.trace[it * 16 + 6] = clock64();
    }
  }
}

// ---- fixed-order reduction of the partial tiles into the gradient tensors, all problems of a group in one launch.
//      blocks [blk_w[p], blk_b[p]):    dW_p[r*rs + c*cs] += sum_b part[b + gt][prow(r) % 128][c % 128]   (one thread per
//                                      element; gt: the tile of (prow(r), c), b: the CTAs that cover it, ascending)
//      blocks [blk_b[p], blk_w[p+1]):  db_p[r]           += sum_b part_bias[b + gt][prow(r) % 128]  (gt: column tile 0)
//      The segments are recomputed from the same host / device row counts the GEMM used (dw_plan_dev).
struct ReduceProb {
  float* dW; float* db;
  int R, C, Rb, Rbp;
  long long rs, cs;
  int blk_w, blk_b;
};
struct ReduceTable { DwGroup grp; ReduceProb q[DW_MAXP]; const float* part; const float* part_bias; };

__global__ void __launch_bounds__(256) reduce_grads3_kernel(const ReduceTable T) {
  __shared__ DwPlan S;
  if (threadIdx.x == 0) dw_plan_dev(T.grp, S);
  __syncthreads();
  int p = 0;
  while (p + 1 < T.grp.n && (int)blockIdx.x >= T.q[p + 1].blk_w) ++p;
  const ReduceProb& q = T.q[p];
  const long long tu = dw_tile_units(S, p);
  // the slots of tile t of problem p, in the order of the CTAs that cover it
  auto sum_tile = [&](const float* src, int t, size_t slot_floats) {
    float s = 0.f;
    if (tu > 0) {
      const long long u = S.ubegin[p] + (long long)t * tu;
      const int b1 = dw_owner(S, u + tu - 1);
      src += (size_t)(S.tbegin[p] + t) * slot_floats;
      for (int b = dw_owner(S, u); b <= b1; ++b) s += src[(size_t)b * slot_floats];
    }
    return s;
  };
  if ((int)blockIdx.x < q.blk_b) {
    const long long idx = (long long)((int)blockIdx.x - q.blk_w) * 256 + threadIdx.x;
    if (idx >= (long long)q.R * q.C) return;
    const int r = (int)(idx / q.C), c = (int)(idx % q.C);
    const int prow = (r / q.Rb) * q.Rbp + (r % q.Rb);
    const int t = (prow / BM) * S.nt[p] + c / DW_BN;
    q.dW[r * q.rs + c * q.cs] += sum_tile(T.part + (prow % BM) * DW_BN + c % DW_BN, t, (size_t)BM * DW_BN);
  } else {
    const int r = ((int)blockIdx.x - q.blk_b) * 256 + threadIdx.x;
    if (r >= q.R) return;
    const int prow = (r / q.Rb) * q.Rbp + (r % q.Rb);
    q.db[r] += sum_tile(T.part_bias + prow % BM, (prow / BM) * S.nt[p], BM);
  }
}

// ---- host side ---------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// Encoded descriptors are pure functions of (base, rows, cols, ld, box): the training step presents the same few
// hundred operands every iteration, so they are memoised (an encode costs ~1 us of host time, 3-12 per launch).
// Every tile is a [box_rows x 32 fp32] box with the 128-byte swizzle the consumers decode (swz()), or (kind 1 / 2: a
// bf16 / fp16 plane, ld in 16-bit elements) a [box_rows x 32] box of 16-bit values with the 64-byte swizzle (swz64()).
// passes > 0: a 3-D map of `passes` such [rows x cols] slices pstride elements apart, boxes [box_rows x 32 x 1].
struct MapKey {
  const void* base; int rows, cols, ld, box_rows, kind, passes; long long pstride;
  bool operator==(const MapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows &&
           kind == o.kind && passes == o.passes && pstride == o.pstride;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.base);
    h = h * 1000003u ^ (size_t)k.rows;
    h = h * 1000003u ^ (size_t)k.cols;
    h = h * 1000003u ^ (size_t)k.ld;
    h = h * 1000003u ^ (size_t)k.box_rows;
    h = h * 1000003u ^ (size_t)k.kind;
    h = h * 1000003u ^ (size_t)k.passes;
    h = h * 1000003u ^ (size_t)k.pstride;
    return h;
  }
};
static std::mutex g_map_mu;
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_map_cache;

static int make_map(CUtensorMap* map, const float* base, int rows, int cols, int ld, int box_rows, int kind = 0,
                    int passes = 0, long long pstride = 0) {
  const MapKey key{base, rows, cols, ld, box_rows, kind, passes, pstride};
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_map_cache.find(key);
    if (it != g_map_cache.end()) { memcpy(map, &it->second, sizeof(CUtensorMap)); return 0; }
  }
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return -4; }
  const size_t esz = kind ? 2 : 4;
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)passes};
  cuuint64_t strides[2] = {(cuuint64_t)ld * esz, (cuuint64_t)pstride * esz};
  cuuint32_t box[3] = {(cuuint32_t)BKF, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  const CUtensorMapDataType dt = kind == 1   ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                 : kind == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                             : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = fn(map, dt, passes > 0 ? 3 : 2, const_cast<float*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  kind ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) rows=%d cols=%d ld=%d box_rows=%d kind=%d passes=%d pstride=%lld",
              (int)r, rows, cols, ld, box_rows, kind, passes, pstride);
    return -4;
  }
  std::lock_guard<std::mutex> lk(g_map_mu);
  if (g_map_cache.size() > 16384) g_map_cache.clear();   // bounded: a long generation run sees many batch sizes
  g_map_cache.emplace(key, *map);
  return 0;
}

long long* g_trace = nullptr;   // gib_tc_trace
int g_trace_tiles = 0;

struct DevInfo { int num_sms = 0; bool attr_done = false; };
static std::mutex g_dev_mu;
static DevInfo g_dev[64];

// shared-memory attributes of one precision's kernels
template <bool TF1>
static int set_attributes() {
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_gemm_kernel<EPI_SPEC_GENERIC, TF1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_gemm_kernel<EPI_SPEC_SELU, TF1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_gemm_kernel<EPI_SPEC_LINEAR, TF1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_gemm_kernel<EPI_SPEC_DSELU, TF1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_gemm_kernel<EPI_SPEC_ADD, TF1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_kernel<EPI_SPEC_GENERIC, TF1>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_kernel<EPI_SPEC_SELU, TF1>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_EPI_SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_kernel<EPI_SPEC_LINEAR, TF1>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_EPI_SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_kernel<EPI_SPEC_DSELU, TF1>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_EPI_SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_kernel<EPI_SPEC_ADD, TF1>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_EPI_SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_dw_kernel<TF1>, cudaFuncAttributeMaxDynamicSharedMemorySize, DW_SMEM_BYTES));
  return 0;
}
// and of one 16-bit type's (wgmma kernels only)
template <int H16>
static int set_attributes16() {
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_kernel<EPI_SPEC_GENERIC, true, H16>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_kernel<EPI_SPEC_SELU, true, H16>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_EPI_SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_kernel<EPI_SPEC_LINEAR, true, H16>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_EPI_SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_kernel<EPI_SPEC_DSELU, true, H16>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_EPI_SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_kernel<EPI_SPEC_ADD, true, H16>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_EPI_SMEM_BYTES));
  GIB_CUDA_TRY(cudaFuncSetAttribute(tc3_wgmma_dw_kernel<true, H16>, cudaFuncAttributeMaxDynamicSharedMemorySize, DW_SMEM_BYTES));
  return 0;
}

static int prepare(int* num_sms_out) {
  int dev = 0;
  GIB_CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) { set_error("device index %d out of range", dev); return -4; }
  std::lock_guard<std::mutex> lk(g_dev_mu);
  DevInfo& d = g_dev[dev];
  if (!d.attr_done) {   // function attributes are per device
    GIB_CUDA_TRY(cudaDeviceGetAttribute(&d.num_sms, cudaDevAttrMultiProcessorCount, dev));
    GIB_TRY(set_attributes<false>());
    GIB_TRY(set_attributes<true>());
    GIB_TRY(set_attributes16<1>());
    GIB_TRY(set_attributes16<2>());
    d.attr_done = true;
  }
  *num_sms_out = d.num_sms;
  return 0;
}

// which compact epilogue a problem can use (EPI_SPEC_GENERIC: none)
static int epi_spec(const GemmNT& p) {
  auto al = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if ((p.ldc & 3) || !al(p.C) || (p.n_store & 3) || p.n_valid != p.n_store) return EPI_SPEC_GENERIC;
  if (p.mode == EPI_ACT) {
    if (p.bias && p.N < p.n_store) return EPI_SPEC_GENERIC;
    if (p.act == ACT_SELU) return EPI_SPEC_SELU;
    if (p.act == ACT_NONE) return EPI_SPEC_LINEAR;
    return EPI_SPEC_GENERIC;
  }
  if (!p.aux || (p.ldaux & 3) || !al(p.aux)) return EPI_SPEC_GENERIC;
  if (p.mode == EPI_MUL_DACT) return p.act == ACT_SELU ? EPI_SPEC_DSELU : EPI_SPEC_GENERIC;
  return EPI_SPEC_ADD;
}

// W given as the planes of the problem's precision: aligned (hi, lo) TF32 planes, or (16-bit modes) one aligned
// 16-bit plane at B_hi whose rows are whole 16-byte units (the TMA stride rule)
static bool presplit(const GemmNT& p) {
  if (p.tf32 >= 2) return p.B_hi && (reinterpret_cast<uintptr_t>(p.B_hi) & 15) == 0 && (p.ldb % 8) == 0;
  return p.B_hi && p.B_lo && (reinterpret_cast<uintptr_t>(p.B_hi) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.B_lo) & 15) == 0;
}

}  // namespace tc3

bool g_use_tc = true;
int g_tc_debug = 0;

void tc3_set_trace(long long* buf, int tiles) { tc3::g_trace = buf; tc3::g_trace_tiles = tiles; }

int device_sm_count() {
  int n = 0;
  if (tc3::prepare(&n) != 0 || n <= 0) n = 132;
  return n;
}

// any NT problem the kernel can load through TMA (W raw or as planes)
bool tc_eligible(const GemmNT& p) {
  return p.M >= 1 && p.N >= 1 && p.K >= 16 && (p.K % 16) == 0 && (p.lda % 4) == 0 && (p.ldb % 4) == 0 &&
         (reinterpret_cast<uintptr_t>(p.A) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.B) & 15) == 0;
}

// the model's call pattern: W as pre-split planes
bool tc3_eligible(const GemmNT& p) {
  auto al = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  return p.M >= 1 && p.N >= 1 && p.K >= 16 && (p.K % 16) == 0 && (p.lda % 4) == 0 && (p.ldb % 4) == 0 && al(p.A) &&
         tc3::presplit(p);
}

template <bool TF1>
static void launch_nt_kernel(const tc3::Maps& maps, const tc3::Params& P, bool raw, int spec, int grid,
                             cudaStream_t st) {
  using namespace tc3;
  if (raw) {
    switch (spec) {
      case EPI_SPEC_SELU: tc3_gemm_kernel<EPI_SPEC_SELU, TF1><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(maps, P); break;
      case EPI_SPEC_LINEAR: tc3_gemm_kernel<EPI_SPEC_LINEAR, TF1><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(maps, P); break;
      case EPI_SPEC_DSELU: tc3_gemm_kernel<EPI_SPEC_DSELU, TF1><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(maps, P); break;
      case EPI_SPEC_ADD: tc3_gemm_kernel<EPI_SPEC_ADD, TF1><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(maps, P); break;
      default: tc3_gemm_kernel<EPI_SPEC_GENERIC, TF1><<<grid, NUM_THREADS, SMEM_BYTES, st>>>(maps, P); break;
    }
  } else {
    switch (spec) {
      case EPI_SPEC_SELU: tc3_wgmma_kernel<EPI_SPEC_SELU, TF1><<<grid, WG_THREADS, WG_EPI_SMEM_BYTES, st>>>(maps, P); break;
      case EPI_SPEC_LINEAR: tc3_wgmma_kernel<EPI_SPEC_LINEAR, TF1><<<grid, WG_THREADS, WG_EPI_SMEM_BYTES, st>>>(maps, P); break;
      case EPI_SPEC_DSELU: tc3_wgmma_kernel<EPI_SPEC_DSELU, TF1><<<grid, WG_THREADS, WG_EPI_SMEM_BYTES, st>>>(maps, P); break;
      case EPI_SPEC_ADD: tc3_wgmma_kernel<EPI_SPEC_ADD, TF1><<<grid, WG_THREADS, WG_EPI_SMEM_BYTES, st>>>(maps, P); break;
      default: tc3_wgmma_kernel<EPI_SPEC_GENERIC, TF1><<<grid, WG_THREADS, WG_SMEM_BYTES, st>>>(maps, P); break;
    }
  }
}
template <int H16>
static void launch_nt_kernel16(const tc3::Maps& maps, const tc3::Params& P, int spec, int grid, cudaStream_t st) {
  using namespace tc3;
  switch (spec) {
    case EPI_SPEC_SELU: tc3_wgmma_kernel<EPI_SPEC_SELU, true, H16><<<grid, WG_THREADS, WG_EPI_SMEM_BYTES, st>>>(maps, P); break;
    case EPI_SPEC_LINEAR: tc3_wgmma_kernel<EPI_SPEC_LINEAR, true, H16><<<grid, WG_THREADS, WG_EPI_SMEM_BYTES, st>>>(maps, P); break;
    case EPI_SPEC_DSELU: tc3_wgmma_kernel<EPI_SPEC_DSELU, true, H16><<<grid, WG_THREADS, WG_EPI_SMEM_BYTES, st>>>(maps, P); break;
    case EPI_SPEC_ADD: tc3_wgmma_kernel<EPI_SPEC_ADD, true, H16><<<grid, WG_THREADS, WG_EPI_SMEM_BYTES, st>>>(maps, P); break;
    default: tc3_wgmma_kernel<EPI_SPEC_GENERIC, true, H16><<<grid, WG_THREADS, WG_SMEM_BYTES, st>>>(maps, P); break;
  }
}

// up to MAXP NT problems in one persistent launch; dep == nullptr: independent.  raw: every W is raw fp32 (split in
// the kernel; mma.sync kernel), else every W comes as aligned (hi, lo) planes (wgmma kernel).  Every problem of a
// launch has the same precision (GemmNT::tf32).
static int launch_nt(const GemmNT* ps, const int* dep, int n, int* flags, bool raw, cudaStream_t st) {
  using namespace tc3;
  if (n < 1 || n > MAXP) { set_error("gemm_nt_tc3: %d problems (max %d)", n, MAXP); return -2; }
  int num_sms = 0;
  GIB_TRY(prepare(&num_sms));
  const int tbn = raw ? BN : WG_BN;
  Maps maps;
  Params P;
  memset(&P, 0, sizeof(P));
  double work = 0;
  ProfRows dyn[MAXP];
  int ndyn = 0;
  long long tiles = 0;
  int np = 0;
  int spec = -1;
  int slot[MAXP];                 // input index -> launch slot (-1: skipped, no rows)
  int flag_ints = 0;
  const int prec = ps[0].tf32;
  const bool tf32 = prec != 0;
  const int h16 = prec >= 2 ? prec - 1 : 0;      // 16-bit operand kind: 1 bf16, 2 fp16
  if (prec < 0 || prec > 3) { set_error("gemm_nt_tc3: unknown precision %d", prec); return -2; }
  if (h16 && raw) {
    set_error("gemm_nt_tc3: 16-bit operands need W as a 16-bit plane (W_hi); raw fp32 W runs in the TF32 modes only");
    return -2;
  }
  for (int i = 0; i < n; ++i) {
    const GemmNT& p = ps[i];
    slot[i] = -1;
    if (p.tf32 != prec) { set_error("gemm_nt_tc3: problems of one launch with different precisions"); return -2; }
    if (p.M <= 0 || p.N <= 0) continue;
    if (!(raw ? tc_eligible(p) : presplit(p) && tc3_eligible(p))) {
      set_error("gemm_nt_tc3: operands violate the TMA alignment / pre-split contract");
      return -2;
    }
    const int sp = epi_spec(p);
    spec = (spec < 0 || spec == sp) ? sp : EPI_SPEC_GENERIC;     // one epilogue specialisation per launch
    GIB_TRY(make_map(&maps.a[np], p.A, p.M, p.K, p.lda, BM));
    GIB_TRY(make_map(&maps.b[np], raw ? p.B : p.B_hi, p.N, p.K, p.ldb, tbn, h16));
    if (!raw && !tf32) GIB_TRY(make_map(&maps.b_lo[np], p.B_lo, p.N, p.K, p.ldb, tbn));
    if (!raw && (sp == EPI_SPEC_DSELU || sp == EPI_SPEC_ADD)) GIB_TRY(make_map(&maps.aux[np], p.aux, p.M, p.n_store, p.ldaux, BM));
    P.g[np] = p;
    P.n_tiles[np] = ceil_div(std::max(p.N, p.n_store), tbn);   // columns [N, n_store) are stored too (zeros / epi(0))
    P.k_blocks[np] = ceil_div(p.K, BKF);
    P.dep[np] = -1;
    P.flag_off[np] = flag_ints;
    flag_ints += ceil_div(p.M, BM) + 1;                         // row blocks of the (capacity) row count
    if (dep && dep[i] >= 0) {
      if (dep[i] >= i || slot[dep[i]] < 0) { set_error("gemm_nt_tc3_chain: problem %d depends on %d", i, dep[i]); return -2; }
      const GemmNT& d = ps[dep[i]];
      if (d.M != p.M || d.m_dev != p.m_dev || d.base_dev != p.base_dev || d.C != p.A) {
        set_error("gemm_nt_tc3_chain: problem %d does not consume the rows problem %d produces", i, dep[i]);
        return -2;
      }
      P.dep[np] = slot[dep[i]];
    }
    slot[i] = np;
    tiles += (long long)ceil_div(p.M, BM) * P.n_tiles[np];      // upper bound when the row count lives on the device
    const double pw = p.work > 0 ? p.work : 2.0 * p.M * (double)p.N * p.K;
    if (p.m_dev) dyn[ndyn++] = ProfRows{p.m_dev, p.base_dev, p.M, pw / p.M};   // the rows launched, not the capacity
    else work += pw;
    ++np;
  }
  if (np == 0) return 0;
  P.nprob = np;
  P.trace = g_trace; P.trace_tiles = g_trace_tiles;
  if (dep) {
    P.flags = flags;
    GIB_CUDA_TRY(cudaMemsetAsync(flags, 0, (size_t)flag_ints * sizeof(int), st));
  }
  const int grid = (int)(tiles < num_sms ? tiles : num_sms);
  ProfScope prof(PROF_GEMM_NT, work, st, dyn, ndyn);
  if (h16 == 1) launch_nt_kernel16<1>(maps, P, spec, grid, st);
  else if (h16 == 2) launch_nt_kernel16<2>(maps, P, spec, grid, st);
  else if (tf32) launch_nt_kernel<true>(maps, P, raw, spec, grid, st);
  else launch_nt_kernel<false>(maps, P, raw, spec, grid, st);
  GIB_LAUNCH_CHECK();
  return 0;
}

int gemm_nt_tc3_group(const GemmNT* ps, int n, cudaStream_t st) { return launch_nt(ps, nullptr, n, nullptr, false, st); }

// up to 4 independent problems whose weights may be raw fp32 (split in the kernel): members with aligned planes run
// on the wgmma kernel, the others on the mma.sync kernel, one launch for each kind present
int gemm_nt_tc_group(const GemmNT* ps, int n, cudaStream_t st) {
  if (n < 1 || n > 4) { set_error("gemm_nt_tc_group: %d problems (max 4)", n); return -2; }
  GemmNT planes[4], raw[4];
  int np = 0, nr = 0;
  for (int i = 0; i < n; ++i) {
    if (tc3::presplit(ps[i])) planes[np++] = ps[i];
    else raw[nr++] = ps[i];
  }
  if (np) GIB_TRY(launch_nt(planes, nullptr, np, nullptr, false, st));
  if (nr) GIB_TRY(launch_nt(raw, nullptr, nr, nullptr, true, st));
  return 0;
}

int gemm_nt_tc(const GemmNT& p, cudaStream_t st) { return gemm_nt_tc_group(&p, 1, st); }

size_t tc3_chain_flag_ints(const GemmNT* ps, int n) {
  size_t f = 0;
  for (int i = 0; i < n; ++i) f += (size_t)ceil_div(ps[i].M > 0 ? ps[i].M : 0, tc3::BM) + 1;
  return f;
}

int gemm_nt_tc3_chain(const GemmNT* ps, const int* dep, int n, int* flags, cudaStream_t st) {
  if (!flags) { set_error("gemm_nt_tc3_chain: no flag buffer"); return -2; }
  return launch_nt(ps, dep, n, flags, false, st);
}

// ---- weight gradients --------------------------------------------------------------------------------------------
bool tc3_dw_eligible(const GemmDW& q) {
  auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  return q.dW && q.M >= 1 && q.Nn >= 16 && q.Kk >= 16 && (q.Nn % 4) == 0 && (q.Kk % 4) == 0 && (q.ldg % 4) == 0 &&
         (q.ldx % 4) == 0 && al(q.G) && al(q.X) &&
         (q.passes == 1 || (q.passes > 1 && (q.pass_g % 4) == 0 && (q.pass_x % 4) == 0 && q.pass_g > 0 && q.pass_x > 0));
}

// the schedule inputs of a launch (the members' host row counts, or their buffers' rows with m_dev)
static void dw_group(const GemmDW* qs, int n, int sms, tc3::DwGroup& g) {
  using namespace tc3;
  memset(&g, 0, sizeof(g));
  g.n = n; g.sms = sms;
  for (int i = 0; i < n; ++i) {
    g.m_dev[i] = qs[i].m_dev; g.base_dev[i] = qs[i].base_dev; g.M[i] = qs[i].M;
    g.mt[i] = ceil_div(qs[i].Nn, BM); g.nt[i] = ceil_div(qs[i].Kk, DW_BN);
    g.passes[i] = std::max(qs[i].passes, 1);
  }
}

// Scratch of a group: one partial tile [128][128] and one bias partial [128] per slot.  dw_plan needs at most G + T
// slots; G = min(SMs, ceil(U / 8)) is bounded here with U from q.M (the capacity when the count is on the device).
void tc3_dw_layout(const GemmDW* qs, int n, Dw3Layout* L) {
  using namespace tc3;
  int tiles = 0;
  long long units = 0;
  for (int i = 0; i < n; ++i) {
    const int t = ceil_div(qs[i].Nn, BM) * ceil_div(qs[i].Kk, DW_BN);
    tiles += t;
    units += (long long)t * ceil_div(std::max(qs[i].M, 0), BKF) * std::max(qs[i].passes, 1);
  }
  L->slots = (int)std::min<long long>(device_sm_count(), ceil_div_ll(units, kDwMinUnits)) + tiles;
  L->floats = (size_t)L->slots * (BM * DW_BN + BM);
}

int gemm_dw_tc3_partials(const GemmDW* qs, int n, const Dw3Layout& L, float* scratch, cudaStream_t st) {
  using namespace tc3;
  if (n < 1 || n > DW_MAXP) { set_error("gemm_dw_tc3_partials: %d problems (max %d)", n, DW_MAXP); return -2; }
  int num_sms = 0;
  GIB_TRY(prepare(&num_sms));
  DwMaps maps;
  DwParams P;
  memset(&P, 0, sizeof(P));
  dw_group(qs, n, num_sms, P.grp);
  long long units = 0;        // upper bound when a row count lives on the device
  const int prec = qs[0].tf32;
  const bool tf32 = prec != 0;
  if (prec < 0 || prec > 3) { set_error("gemm_dw_tc3: unknown precision %d", prec); return -2; }
  for (int i = 0; i < n; ++i) {
    const GemmDW& q = qs[i];
    if (!tc3_dw_eligible(q)) { set_error("gemm_dw_tc3: operands violate the TMA alignment contract"); return -2; }
    if (q.tf32 != prec) { set_error("gemm_dw_tc3: problems of one launch with different precisions"); return -2; }
    // 3-D maps, the pass outermost (one pass: a stride past the slice, never stepped over): 32 x 32 x 1 boxes
    const int np = P.grp.passes[i];
    GIB_TRY(make_map(&maps.g[i], q.G, q.M, q.Nn, q.ldg, BKF, 0, np, np > 1 ? q.pass_g : (long long)q.M * q.ldg));
    GIB_TRY(make_map(&maps.x[i], q.X, q.M, q.Kk, q.ldx, BKF, 0, np, np > 1 ? q.pass_x : (long long)q.M * q.ldx));
    P.Nn[i] = q.Nn; P.Kk[i] = q.Kk;
    if (q.dbias) P.bias_mask |= 1u << i;
    units += (long long)P.grp.mt[i] * P.grp.nt[i] * ceil_div(q.M, BKF) * np;
  }
  P.part = scratch;
  P.part_bias = scratch + (size_t)L.slots * BM * DW_BN;
  P.trace = g_trace; P.trace_tiles = g_trace_tiles;
  // the device plan's G = min(SMs, ceil(U / 8)) never exceeds this grid; CTAs past it find no units
  const long long want = std::max(1LL, ceil_div_ll(units, kDwMinUnits));
  const int grid = (int)std::min<long long>(want, num_sms);
  if (prec == 2) tc3_wgmma_dw_kernel<true, 1><<<grid, WG_THREADS, DW_SMEM_BYTES, st>>>(maps, P);
  else if (prec == 3) tc3_wgmma_dw_kernel<true, 2><<<grid, WG_THREADS, DW_SMEM_BYTES, st>>>(maps, P);
  else if (tf32) tc3_wgmma_dw_kernel<true><<<grid, WG_THREADS, DW_SMEM_BYTES, st>>>(maps, P);
  else tc3_wgmma_dw_kernel<false><<<grid, WG_THREADS, DW_SMEM_BYTES, st>>>(maps, P);
  GIB_LAUNCH_CHECK();
  return 0;
}

// fixed-order reduction of the group's partials into the gradient tensors (any stream ordered after the partials)
int gemm_dw_tc3_reduce(const GemmDW* qs, int n, const Dw3Layout& L, const float* scratch, cudaStream_t st) {
  using namespace tc3;
  int num_sms = 0;
  GIB_TRY(prepare(&num_sms));
  ReduceTable T;
  memset(&T, 0, sizeof(T));
  dw_group(qs, n, num_sms, T.grp);
  T.part = scratch;
  T.part_bias = scratch + (size_t)L.slots * BM * DW_BN;
  int blk = 0;
  for (int i = 0; i < n; ++i) {
    const GemmDW& q = qs[i];
    ReduceProb& r = T.q[i];
    r.dW = q.dW; r.db = q.dbias;
    r.R = q.R; r.C = q.C; r.Rb = q.Rb; r.Rbp = q.Rbp; r.rs = q.rs; r.cs = q.cs;
    r.blk_w = blk; blk += q.dW ? (int)ceil_div_ll((long long)q.R * q.C, 256) : 0;
    r.blk_b = blk; blk += q.dbias ? ceil_div(q.R, 256) : 0;
  }
  if (blk == 0) return 0;
  reduce_grads3_kernel<<<blk, 256, 0, st>>>(T);
  GIB_LAUNCH_CHECK();
  return 0;
}

// the segments dw_plan gives a group with host row counts (test hook): per segment (CTA, member, tile, first row,
// rows, slot), or with seg_ints == 7 (CTA, member, tile, first pass, first row in it, k-blocks, slot); per tile the
// first and last CTA the reduction reads (-1, -1: no rows)
int tc3_dw_schedule(const int* rows, const int* passes, const int* Nn, const int* Kk, int n, int sms, int* segs,
                    int seg_ints, int max_segs, int* tile_ctas, int* G_out) {
  using namespace tc3;
  if (n < 1 || n > DW_MAXP || sms < 1 || (seg_ints != 6 && seg_ints != 7)) {
    set_error("tc3_dw_schedule: n=%d sms=%d seg_ints=%d", n, sms, seg_ints);
    return -2;
  }
  int mt[DW_MAXP], nt[DW_MAXP], np[DW_MAXP], base[DW_MAXP] = {0};
  for (int i = 0; i < n; ++i) {
    np[i] = passes ? passes[i] : 1;
    if (rows[i] < 0 || np[i] < 1) { set_error("tc3_dw_schedule: negative row count or pass count < 1"); return -2; }
    mt[i] = ceil_div(Nn[i], BM); nt[i] = ceil_div(Kk[i], DW_BN);
  }
  DwPlan S;
  dw_plan(S, rows, base, mt, nt, np, n, sms);
  *G_out = S.G;
  int ns = 0;
  for (int b = 0; b < S.G; ++b) {
    long long u0, u1;
    dw_range(S, b, u0, u1);
    for (long long u = u0; u < u1;) {
      const Item w = dw_segment(S, b, u, u1);
      u += w.nkb;
      if (ns == max_segs) { set_error("tc3_dw_schedule: more than %d segments", max_segs); return -3; }
      int* o = segs + seg_ints * ns++;
      o[0] = b; o[1] = w.p; o[2] = (w.m0 / BM) * nt[w.p] + w.n0 / DW_BN;
      if (seg_ints == 6) { o[3] = w.r0; o[4] = w.rows; o[5] = w.z; }
      else { o[3] = w.ps; o[4] = w.r0; o[5] = w.nkb; o[6] = w.z; }
    }
  }
  for (int p = 0; p < n; ++p)
    for (int t = 0; t < mt[p] * nt[p]; ++t) {
      int* o = tile_ctas + 2 * (S.tbegin[p] + t);
      o[0] = o[1] = -1;
      const long long tu = dw_tile_units(S, p);
      if (tu > 0) {
        const long long u = S.ubegin[p] + (long long)t * tu;
        o[0] = dw_owner(S, u); o[1] = dw_owner(S, u + tu - 1);
      }
    }
  return ns;
}

}  // namespace gib
