// Device-side molecular-graph structure produced by K0 (graph_build.cu).
#pragma once
#include "common.cuh"

namespace gib {

// header ints written by the scan kernel and read back by the host (16 ints = 64 B)
enum : int {
  HDR_E = 0,            // number of bond entries (non-zero elements of `edges`)
  HDR_P = 1,            // rows of the type-grouped entry arrays (each group padded to 128)
  HDR_TYPE_COUNT = 2,   // [4] entries per bond type
  HDR_TYPE_BASE = 6,    // [5] first row of each type group (multiples of 128); [G] == P
  HDR_FLAGS = 11,
  HDR_CAPACITY = 12,    // host header only: != 0 -> E / P are capacities, the live header stays on the device ...
  HDR_DEV_LO = 13,      // ... at this address (low / high 32 bits)
  HDR_DEV_HI = 14,
  HDR_INTS = 16
};
enum : int {
  GRAPH_FLAG_MULTITYPE = 1,  // some (b,i,j) carries more than one non-zero bond type
  GRAPH_FLAG_NONBINARY = 2,  // some non-zero bond value differs from 1
  GRAPH_FLAG_OVERFLOW = 4    // capacity mode: the batch holds more bond entries than the capacity (results invalid)
};

struct GraphArrays {
  int* ent_src;    // [P] source slot (b*N + j) of the entry, -1 on pad rows
  int* ent_dst;    // [P] destination slot (b*N + i), -1 on pad rows
  float* ent_w;    // [P] bond value edges[b,i,j,t] (1 for one-hot), 0 on pad rows
  int* dst_ptr;    // [S+1] CSR over destination slots
  int* dst_ent;    // [E]   entry rows, ordered (b, i, j, t)  == reference nonzero() order
  int* src_ptr;    // [S+1] CSR over source slots
  int* src_ent;    // [E]   entry rows, ordered (b, j, i, t)
};

// Message rows of the GGNN / MNN (built from K0's arrays into the forward workspace, model.cu).  A message depends only on
// the source atom's state, the bond type and, for the GGNN, the bond value that scales its input.  The entries with
// w == 1 that share (molecule, source slot, type) share ONE message row; an entry with any other w has a row of its own.
// Rows are grouped by type, group t starting at the entry group's first row TYPE_BASE[t] (so a group never holds more
// rows than the entry group it replaces); inside a group rows ascend by source slot, and within (slot, type) the shared
// row comes first, then one row per other entry in source-CSR order.  Pad rows: src = -1, w = 0, no entries.
enum : int {
  MR_COUNT = 0,   // [4] message rows per bond type
  MR_BASE = 4,    // [5] first row of each type group (== the entry groups' TYPE_BASE); [G] = end of the last group
  MR_EOFF = 9,    // [5] first position of each type's entries in u_dst; [G] = entries listed in all
  MR_TOTAL = 14,  // message rows of all types
  MR_META_INTS = 16
};
struct MsgRows {
  int* u_src;     // [P]   source slot of the message row, -1 on pad rows
  float* u_w;     // [P]   bond value of the row's entries (1 on a shared row), 0 on pad rows
  int* u_ptr;     // [P+1] CSR message row -> its entries' positions in u_dst (pad rows: empty)
  int* u_dst;     // [E]   destination slot of each entry, grouped by message row (-1 past the last entry)
  int* ent_u;     // [P]   entry row -> its message row (-1: an entry the source CSR does not list)
  int* dst_u;     // [E]   dst_ent with every entry replaced by its message row (-1 past the live entries)
  int* s_ptr;     // [S+1] CSR source slot -> its message rows
  int* s_u;       // [E]   message rows of each source slot, by type (-1 past the last row)
  int* meta;      // [MR_META_INTS] see MR_*
  int* tmp;       // build scratch: per-molecule counts and offsets, msg_rows_tmp_ints(B, G)
};
size_t msg_rows_tmp_ints(int B, int G);
// type bases: dev_hdr (capacity mode: the device header K0 wrote) or, when dev_hdr is null, tb[0..G] (host header)
int msg_rows_build(const GraphArrays& ga, const MsgRows& mr, const int* dev_hdr, const int* tb, int B, int N, int G,
                   int E, int P, cudaStream_t st);

size_t graph_count_ws_ints(int B, int G);
// `edges` is float32 (in_dtype 0) or int8 / uint8 (in_dtype 1: the reference's on-disk format, DataProcesser.py:157-161)
int graph_count(const void* edges, int in_dtype, int B, int N, int Ef, int by_type, int* ws, cudaStream_t st);
// cap_E / cap_P > 0: capacity mode -- arrays hold cap_E entries / cap_P rows; writes beyond are dropped, the tail rows
// [P, cap_P) are padded, and GRAPH_FLAG_OVERFLOW is raised in the device header when the batch does not fit
int graph_fill(const void* edges, int in_dtype, int B, int N, int Ef, int by_type, int* ws, GraphArrays ga, int cap_E,
               int cap_P, cudaStream_t st);

}  // namespace gib
