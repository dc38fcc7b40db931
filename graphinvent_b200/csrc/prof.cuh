// Optional per-kernel-class timing with CUDA events on the launching stream (bench.py uses it to
// report roofline.achieved from live launches inside the timed region).  Off by default: the
// hooks then cost one predictable branch.
#pragma once
#include <cuda_runtime.h>

namespace gib {

// 0 / 1: launches of the tensor-core kernels (forward + dX, weight gradients); 3 / 4: the same contracts on the fp32 SIMT
// kernels (narrow / tiny problems, and everything when tensor cores are off)
enum ProfClass : int { PROF_GEMM_NT = 0, PROF_GEMM_DW = 1, PROF_SCATTER = 2, PROF_GEMM_NT_SIMT = 3, PROF_GEMM_DW_SIMT = 4,
                       PROF_NCLASS = 5 };

extern bool g_prof_on;
// Work of a problem whose row count lives on the device (GemmNT::m_dev): per_row x min(*m_dev, cap - *base_dev) rows.
// The two ints are copied to pinned host memory ahead of the launch's first event and resolved when the records are read
// (after the caller's stream sync), so that the record holds the rows actually launched without a host synchronisation.
struct ProfRows { const int* m_dev; const int* base_dev; int cap; double per_row; };
void prof_begin(int cls, double work, cudaStream_t st, const ProfRows* rows = nullptr, int nrows = 0);
void prof_end(cudaStream_t st);

struct ProfScope {
  cudaStream_t st;
  bool on;
  ProfScope(int cls, double work, cudaStream_t s, const ProfRows* rows = nullptr, int nrows = 0)
      : st(s), on(g_prof_on) {
    if (on) prof_begin(cls, work, st, rows, nrows);
  }
  ~ProfScope() {
    if (on) prof_end(st);
  }
};

}  // namespace gib
