// SPDX-License-Identifier: MIT
// TEST INFRASTRUCTURE: the joint window step of sgb_math.cuh on the host (tests/test_joint_step_on_host.py), run as joint_step_kernel
// runs it with one thread for the CTA.
#include <vector>

#include "sgb_math.cuh"

using namespace sgb;

namespace {
AlignOptions options(const double* o) {  // lm, max_iterations, max_inner_iterations, gn_lambda, init_lambda, lambda_factor, rot_eps, trans_eps, mask[6]
  AlignOptions a;
  a.lm = static_cast<int>(o[0]);
  a.max_iterations = static_cast<int>(o[1]);
  a.max_inner_iterations = static_cast<int>(o[2]);
  a.gn_lambda = o[3];
  a.init_lambda = o[4];
  a.lambda_factor = o[5];
  a.rotation_eps = o[6];
  a.translation_eps = o[7];
  for (int i = 0; i < 6; i++) a.dof_mask[i] = o[8 + i];
  return a;
}
}  // namespace

extern "C" {

void sgbj_solve_ldlt6(const double* A36, const double* rhs, double* x) {
  double A[36];
  for (int i = 0; i < 36; i++) A[i] = A36[i];
  solve_ldlt6(A, rhs, x);
}

/// A: symmetric n x n (row- or column-major alike); only its lower triangle is passed on
void sgbj_solve_ldlt_n(int n, const double* A, const double* rhs, double* x) {
  std::vector<double> L(n * (n + 1) / 2), y(n);
  std::vector<int> perm(n);
  for (int r = 0; r < n; r++)
    for (int c = 0; c <= r; c++) L[packed_index(r, c)] = A[r * n + c];
  solve_ldlt_n(n, L.data(), rhs, x, perm.data(), y.data(), 0, 1);
}

void sgbj_edge_adjoint(const double* T16, double* A36) { edge_adjoint(T16, A36); }

int sgbj_state_size() { return static_cast<int>(sizeof(WindowState)); }

void sgbj_init(const double* o, int n_free, int n_edges, WindowState* s) { joint_init(options(o), n_free, n_edges, *s); }

/// One joint_step_kernel CTA for one window: out = the edges' 44 sums (linearize) or e (error()), in the window's edge order.  X, cand:
/// [n_frames][16] column-major; delta [6 n_free]; sums [n_edges][44] kept across calls.  poses_out [n_edges][16]: the edges' next poses.
void sgbj_step(const double* o, int n_frames, const int* free, int n_edges, const int* ei, const int* ej, double* sums, double* X, double* cand,
               double* delta, WindowState* s, int linearize, const double* out, double* poses_out) {
  const AlignOptions a = options(o);
  int n_free = 0;
  for (int k = 0; k < n_frames; k++) n_free += free[k] >= 0;
  std::vector<double> work(joint_work_doubles(n_free));
  JointWindow w;
  w.n_frames = n_frames;
  w.n_free = n_free;
  w.n_edges = n_edges;
  w.free = free;
  w.ei = ei;
  w.ej = ej;
  w.sums = sums;
  w.X = X;
  w.cand = cand;
  w.delta = delta;
  w.s = s;
  w.work = work.data();
  if (linearize) {
    for (int k = 0; k < 44 * n_edges; k++) sums[k] = out[k];
    joint_after_linearize(a, w, 0, 1);
  } else {
    double ce = 0.0;
    for (int q = 0; q < n_edges; q++) ce += out[q];
    joint_after_error(a, w, ce, 0, 1);
  }
  const double* P = s->phase == kPhaseTrial ? cand : X;
  for (int q = 0; q < n_edges; q++) edge_pose(P + 16 * ei[q], P + 16 * ej[q], poses_out + 16 * q);
}

}  // extern "C"
