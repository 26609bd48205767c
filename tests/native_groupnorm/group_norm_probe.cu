// Test-only entry points into TrajNet's GroupNorm + Mish kernel (rohm_b200/csrc/groupnorm.cu) with an explicit cluster
// size, driven from Python through ctypes by tests/group_norm_probe.py.  Returns 0 or a cudaError_t.
#include "../../rohm_b200/csrc/groupnorm.cuh"

using namespace rohm;

extern "C" {

// `reps` back-to-back GroupNorm + Mish launches with clusters of n CTAs per (clip, group) on the default stream, the
// kernel's shared-memory limit raised to the slice first (so n = 1 also runs groups above the default 48 KB).
int probe_group_norm(const GnArgs* a, int B, int n, int reps) {
  if (reps < 1 || B < 1) return static_cast<int>(cudaErrorInvalidValue);
  cudaError_t rc = gn_reserve_smem(gn_slice_bytes(a->T, a->C, a->groups, n));
  for (int i = 0; i < reps && rc == cudaSuccess; ++i) rc = launch_gn_mish(*a, B, n, nullptr, false);
  return static_cast<int>(rc);
}

// The cluster size rohm_trajnet_create chooses for a (clip, group) of T rows of C / groups channels; 0 on error.
int probe_group_norm_cluster(int T, int C, int groups) {
  size_t budget = 0, max_budget = 0;
  if (gn_smem_budgets(&budget, &max_budget) != cudaSuccess) return 0;
  return gn_pick_cluster(T, C, groups, budget);
}

}  // extern "C"
