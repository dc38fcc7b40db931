// The batch gather of the device-resident data loader (graphinvent_b200/loader.py): one launch turns a list of row
// indices into a block of int8 rows into the static model inputs of a step.
//
// The three outputs are contiguous [B, row bytes] arrays, handled as one flat sequence of 16-element chunks.  A thread
// owns one output chunk: it walks the chunk's row segments (a chunk crosses at most a few row boundaries), loads each
// segment's source bytes with at most two aligned 16-byte loads, funnels them into a 128-bit register and stores the
// chunk as one 16-byte store (int8) or four 16-byte stores (float32).  Rows [b, B) are zero and read nothing.  Block
// rows are not 16-byte aligned in general (gdb13: 104, 507 and 625 bytes), hence the aligned-word funnel.  Every
// aligned word it loads holds at least one byte of the segment, so no load leaves a 16-byte aligned allocation.
#include <algorithm>

#include "common.cuh"
#include "../../include/gib200.h"

namespace gib {

namespace {

constexpr int kGatherNT = 256;
constexpr int kGatherMaxBlocks = 4096;

struct GatherArray {
  const uint8_t* src;     // block rows, row-major
  void* dst;              // [B, rb], int8 or float32
  int rb;                 // elements per row
  int widen;              // 1: float32 output
  long long chunks;       // ceil(B * rb / 16)
};

__device__ __forceinline__ void gather_chunk(const GatherArray& g, long long c, const int* __restrict__ rows, int b,
                                             int B) {
  const long long total = (long long)B * g.rb;
  const long long e0 = c * 16;
  const int n = (int)min(16LL, total - e0);
  long long r = e0 / g.rb;
  int col = (int)(e0 - r * g.rb);
  u128 v = 0;
  for (int k = 0; k < n;) {
    const int seg = min(n - k, g.rb - col);
    if (r < b) {
      u128 s = load_span(g.src + (size_t)rows[r] * g.rb + col, seg);
      if (seg < 16) s &= ((u128)1 << (8 * seg)) - 1;
      v |= s << (8 * k);
    }
    k += seg;
    ++r;
    col = 0;
  }
  if (!g.widen) {
    int8_t* out = static_cast<int8_t*>(g.dst) + e0;
    if (n == 16) {
      st16(out, v);
    } else {
      for (int j = 0; j < n; ++j) out[j] = (int8_t)(uint8_t)(v >> (8 * j));
    }
    return;
  }
  float* out = static_cast<float*>(g.dst) + e0;
  if (n == 16) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const unsigned w = (unsigned)(v >> (32 * q));
      reinterpret_cast<float4*>(out)[q] = make_float4((float)(int8_t)(w & 0xff), (float)(int8_t)((w >> 8) & 0xff),
                                                      (float)(int8_t)((w >> 16) & 0xff), (float)(int8_t)(w >> 24));
    }
  } else {
    for (int j = 0; j < n; ++j) out[j] = (float)(int8_t)(uint8_t)(v >> (8 * j));
  }
}

__global__ void __launch_bounds__(kGatherNT) gather_rows_kernel(GatherArray g0, GatherArray g1, GatherArray g2,
                                                                const int* __restrict__ rows, int b, int B,
                                                                gib_batch_ctl* ctl) {
  if (ctl && blockIdx.x == 0 && threadIdx.x == 0) {
    ctl->live = b;
    ctl->scale = b > 0 ? (float)(1.0 / (double)b) : 0.f;   // the host's float32(1.0 / b), bit for bit
  }
  const long long total = g0.chunks + g1.chunks + g2.chunks;
  for (long long c = (long long)blockIdx.x * kGatherNT + threadIdx.x; c < total;
       c += (long long)gridDim.x * kGatherNT) {
    if (c < g0.chunks) {
      gather_chunk(g0, c, rows, b, B);
    } else if (c < g0.chunks + g1.chunks) {
      gather_chunk(g1, c - g0.chunks, rows, b, B);
    } else {
      gather_chunk(g2, c - g0.chunks - g1.chunks, rows, b, B);
    }
  }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace
}  // namespace gib

using namespace gib;

extern "C" {

int gib_gather_rows(const signed char* nodes, const signed char* edges, const signed char* apds, const int* rows,
                    int b, int B, int row_nodes, int row_edges, int apd, void* out_nodes, void* out_edges, int out_dtype,
                    float* out_target, gib_batch_ctl* ctl, gib_stream stream) {
  if (B <= 0 || row_nodes <= 0 || row_edges <= 0 || apd <= 0 || b < 0 || b > B) {
    set_error("gib_gather_rows: need 0 <= b <= B and B, row_nodes, row_edges, apd > 0, got b = %d, B = %d, "
              "row_nodes = %d, row_edges = %d, apd = %d", b, B, row_nodes, row_edges, apd);
    return -1;
  }
  if (out_dtype != 0 && out_dtype != 1) {
    set_error("gib_gather_rows: out_dtype %d (0 = float32, 1 = int8)", out_dtype);
    return -1;
  }
  if (!nodes || !edges || !apds || !out_nodes || !out_edges || !out_target || (b > 0 && !rows)) {
    set_error("gib_gather_rows: null pointer (every block and output pointer, and rows when b > 0)");
    return -1;
  }
  if (!aligned16(nodes) || !aligned16(edges) || !aligned16(apds) || !aligned16(out_nodes) || !aligned16(out_edges) ||
      !aligned16(out_target)) {
    set_error("gib_gather_rows: the block and output pointers must be 16-byte aligned");
    return -1;
  }
  const int widen = out_dtype == 0;
  GatherArray g0{reinterpret_cast<const uint8_t*>(nodes), out_nodes, row_nodes, widen,
                 ceil_div_ll((long long)B * row_nodes, 16)};
  GatherArray g1{reinterpret_cast<const uint8_t*>(edges), out_edges, row_edges, widen,
                 ceil_div_ll((long long)B * row_edges, 16)};
  GatherArray g2{reinterpret_cast<const uint8_t*>(apds), out_target, apd, 1, ceil_div_ll((long long)B * apd, 16)};
  const long long total = g0.chunks + g1.chunks + g2.chunks;
  const int blocks = (int)std::min<long long>(ceil_div_ll(total, kGatherNT), kGatherMaxBlocks);
  gather_rows_kernel<<<blocks, kGatherNT, 0, (cudaStream_t)stream>>>(g0, g1, g2, rows, b, B, ctl);
  GIB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
