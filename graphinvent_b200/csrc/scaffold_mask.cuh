// The attachment-point rule of scaffold decoration (gib_scaffolds, include/gib200.h), shared by the generator's logit
// mask (generate.cu) and the conditional route plan's check of each kept action (preprocess.cu).  Scaffold s has
// k_s atoms; bit i of protect[s] marks a scaffold atom that is not an attachment point.  With n atoms in the state:
//   - an add whose bond_to is a protected atom is forbidden;
//   - a connect whose bond_to is a protected atom is forbidden;
//   - every connect is forbidden while bond_from = n - 1 is still a scaffold atom (n - 1 < k_s);
//   - terminate never is.
#pragma once
#include <cuda_runtime.h>

namespace gib {

__device__ __forceinline__ bool scaffold_protected(const unsigned int* pm, int i) {
  return (pm[i >> 5] >> (i & 31)) & 1u;
}

// every connect is closed while the newest atom is a scaffold atom
__device__ __forceinline__ bool scaffold_connects_closed(int n, int k) { return n - 1 < k; }

// the rule for one flat APD index a (adds [0, N * per_node), connects [N * per_node, N * (per_node + Ef)), terminate
// last) in a state of n atoms decorating a scaffold of k atoms with protect words pm
__device__ __forceinline__ bool scaffold_forbidden(int a, int n, int k, const unsigned int* pm, int N, int Ef,
                                                   int per_node) {
  const int len_add = N * per_node;
  if (a < len_add) {
    const int i = a / per_node;
    return i < k && scaffold_protected(pm, i);
  }
  if (a < len_add + N * Ef) {
    const int i = (a - len_add) / Ef;
    return scaffold_connects_closed(n, k) || (i < k && scaffold_protected(pm, i));
  }
  return false;
}

}  // namespace gib
