// SPDX-License-Identifier: MIT
// TEST INFRASTRUCTURE -- not part of the product, never loaded by small_gicp_b200.
// The GNC weight formulas (gnc_weight) and mu schedule (gnc_stage_begin) of sgb_math.cuh, which the gnc_* kernels of sgb_batch.cu inline,
// compiled for the HOST without FMA contraction behind a small C entry point: tests/test_np_gnc.py holds them against tests/np_gnc.py bit
// for bit, on a machine without a GPU.
#include <cstddef>

#include "sgb_math.cuh"

extern "C" {

// out[i] = gnc_weight<kind>(r2[i], mu[i], c2[i])
void sgbg_weight(int kind, size_t n, const double* r2, const double* mu, const double* c2, double* out) {
  for (size_t i = 0; i < n; i++)
    out[i] = kind == sgb::kGncTls ? sgb::gnc_weight<sgb::kGncTls>(r2[i], mu[i], c2[i]) : sgb::gnc_weight<sgb::kGncGemanMcClure>(r2[i], mu[i], c2[i]);
}

// gnc_stage_begin from a member's r2max until its schedule marks a stage the last: each stage's mu into mus (at most max_stages);
// returns the stage count
int sgbg_schedule(int kind, double r2max, double c2, int max_stages, double* mus) {
  sgb::GncState g = {};
  g.r2max = r2max;
  do {
    sgb::gnc_stage_begin(kind, c2, max_stages, g);
    mus[g.stages - 1] = g.mu;
  } while (!g.last);
  return g.stages;
}
}
