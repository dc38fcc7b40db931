#include <vector>

#include "../../include/gib200.h"
#include "prof.cuh"
#include "common.cuh"

namespace gib {

bool g_prof_on = false;
long long g_launch_count = 0;

struct Rec { cudaEvent_t a, b; int cls; double work; size_t rows0; int nrows; };
static std::vector<Rec> g_pool;   // event pairs, reused across collections

// device-side row counts of the records since gib_profile_enable(1): snapshots in pinned chunks that never move
struct RowTerm { int* snap; int cap; double per_row; };   // snap[0] = *m_dev, snap[1] = *base_dev
static std::vector<RowTerm> g_rows;
static std::vector<int*> g_snap_chunks;
constexpr size_t kSnapChunkInts = 4096;
static size_t g_used = 0, g_rows_used = 0;

static int* snap_slot(size_t i) {
  const size_t chunk = 2 * i / kSnapChunkInts;
  while (g_snap_chunks.size() <= chunk) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, kSnapChunkInts * sizeof(int), cudaHostAllocDefault) != cudaSuccess) return nullptr;
    g_snap_chunks.push_back(static_cast<int*>(p));
  }
  return g_snap_chunks[chunk] + 2 * i % kSnapChunkInts;
}

void prof_begin(int cls, double work, cudaStream_t st, const ProfRows* rows, int nrows) {
  if (g_used == g_pool.size()) {
    Rec r{};
    cudaEventCreate(&r.a);
    cudaEventCreate(&r.b);
    g_pool.push_back(r);
  }
  Rec& r = g_pool[g_used];
  r.cls = cls;
  r.work = work;
  r.rows0 = g_rows_used;
  r.nrows = 0;
  for (int k = 0; k < nrows; ++k) {
    int* s = snap_slot(g_rows_used);
    if (!s) continue;   // no pinned memory: the launch's work stays counted without these rows
    s[1] = 0;
    cudaMemcpyAsync(s, rows[k].m_dev, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (rows[k].base_dev) cudaMemcpyAsync(s + 1, rows[k].base_dev, sizeof(int), cudaMemcpyDeviceToHost, st);
    const RowTerm t{s, rows[k].cap, rows[k].per_row};
    if (g_rows_used == g_rows.size()) g_rows.push_back(t);
    else g_rows[g_rows_used] = t;
    ++g_rows_used;
    ++r.nrows;
  }
  cudaEventRecord(r.a, st);
}
void prof_end(cudaStream_t st) {
  cudaEventRecord(g_pool[g_used].b, st);
  ++g_used;
}

// the record's work with its device-side row counts resolved (the snapshots are complete after the caller's sync)
static double rec_work(const Rec& r) {
  double w = r.work;
  for (int k = 0; k < r.nrows; ++k) {
    const RowTerm& t = g_rows[r.rows0 + k];
    long long m = t.snap[0];
    const long long room = (long long)t.cap - t.snap[1];
    if (m > room) m = room;
    if (m < 0) m = 0;
    w += t.per_row * (double)m;
  }
  return w;
}

}  // namespace gib

using namespace gib;

extern "C" {

long long gib_launch_count(void) { return g_launch_count; }

void gib_profile_enable(int on) {
  g_prof_on = on != 0;
  if (on) g_used = g_rows_used = 0;
}

// Per-launch records since gib_profile_enable(1), in launch order (call before gib_profile_collect, which clears them):
// fills at most cap entries and returns the number of records (or a negative CUDA error).
int gib_profile_records(double* ms, double* work, int* cls, int cap) {
  for (size_t i = 0; i < g_used && (int)i < cap; ++i) {
    float t = 0.f;
    cudaError_t e = cudaEventElapsedTime(&t, g_pool[i].a, g_pool[i].b);
    if (e != cudaSuccess) return -(int)e;
    ms[i] = t; work[i] = rec_work(g_pool[i]); cls[i] = g_pool[i].cls;
  }
  return (int)g_used;
}

// Call after synchronising the stream.  For each class c: ms[c] = summed event time,
// work[c] = summed algorithmic FLOPs (GEMM classes) or bytes (scatter), count[c] = launches.
int gib_profile_collect(double* ms, double* work, long long* count) {
  for (int c = 0; c < PROF_NCLASS; ++c) { ms[c] = 0; work[c] = 0; count[c] = 0; }
  for (size_t i = 0; i < g_used; ++i) {
    float t = 0.f;
    cudaError_t e = cudaEventElapsedTime(&t, g_pool[i].a, g_pool[i].b);
    if (e != cudaSuccess) return (int)e;
    ms[g_pool[i].cls] += t;
    work[g_pool[i].cls] += rec_work(g_pool[i]);
    count[g_pool[i].cls] += 1;
  }
  g_used = g_rows_used = 0;
  return 0;
}

}  // extern "C"
