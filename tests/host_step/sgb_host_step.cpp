// SPDX-License-Identifier: MIT
// TEST INFRASTRUCTURE -- not part of the product, never loaded by small_gicp_b200.
// The optimiser step of batched align() (small_gicp_b200/csrc/sgb_math.cuh: solve_ldlt6, se3_exp6, pose_mul and the per-member state
// machine that batch_step_kernel runs) compiled for the HOST next to the C++ host mirror's core.hpp / registration.hpp, both without FMA
// contraction, behind a small C entry point: tests/test_batch_step_on_host.py holds the two against each other bit for bit, on a
// machine without a GPU.
#include <cstddef>
#include <cstring>
#include <tuple>
#include <vector>

#include "sgb_math.cuh"
#include "small_gicp_b200/registration.hpp"  // the host mirror's optimizers: the reference the batched align step is held to

namespace {

namespace M = small_gicp_b200;

// A deterministic stand-in for Reduction: H, b, e and error() are functions of the pose only (plus a count of linearize calls), so the
// device step (sgb::align_*) and the mirror's optimizers can be driven through the same sequence and compared bit for bit.
//   d = x(T) - x*, x(T) = (skew part of R, t);  H = s (diag(w) + coupling (1 - I)), s = 1 + |d|^2;  b = gain H d;
//   e = error(T) = 1/2 sum w_i d_i^2 + bump |d|^4 (+ 1e6 after the reject_from-th linearize: every later trial is rejected)
// gain > 1 overshoots (rejected trials until lambda has grown), gain < 1 converges slowly (runs out of iterations), x* = x(T0) gives b = 0.
struct FakeModel {
  double target[6], w[6], coupling, gain, bump;
  int reject_from, n_points;
};

struct FakeReduction {
  const FakeModel* f;
  int n_lin = 0;

  void delta(const double* T, double* d) const {
    const double x[6] = {0.5 * (T[6] - T[9]), 0.5 * (T[8] - T[2]), 0.5 * (T[1] - T[4]), T[12], T[13], T[14]};
    for (int i = 0; i < 6; i++) d[i] = x[i] - f->target[i];
  }
  double model_error(const double* T) const {
    double d[6], q = 0.0, e = 0.0;
    delta(T, d);
    for (int i = 0; i < 6; i++) q += d[i] * d[i];
    for (int i = 0; i < 6; i++) e += 0.5 * f->w[i] * d[i] * d[i];
    return e + f->bump * q * q + (n_lin >= f->reject_from ? 1e6 : 0.0);
  }
  /// out44 = H | b | e | inliers at T (H symmetric); counts the call
  void linearize44(const double* T, double* out44) {
    double d[6], q = 0.0;
    delta(T, d);
    for (int i = 0; i < 6; i++) q += d[i] * d[i];
    const double s = 1.0 + q;
    for (int r = 0; r < 6; r++)
      for (int c = 0; c < 6; c++) out44[r * 6 + c] = s * (r == c ? f->w[r] : f->coupling);
    for (int r = 0; r < 6; r++) {
      double v = 0.0;
      for (int c = 0; c < 6; c++) v += out44[r * 6 + c] * d[c];
      out44[36 + r] = f->gain * v;
    }
    out44[42] = model_error(T);  // before the count: the penalty applies to the trials after the reject_from-th linearize
    n_lin++;
    out44[43] = f->n_points - n_lin;
  }

  // ---- the Reduction interface of registration.hpp ----
  template <typename Target, typename Source, typename Tree, typename Rejector, typename Factor>
  std::tuple<M::Matrix6d, M::Vector6d, double> linearize(const Target&, const Source&, const Tree&, const Rejector&, const M::Isometry3d& T,
                                                         std::vector<Factor>&) {
    double o[44];
    linearize44(T.data(), o);
    M::Matrix6d H;
    M::Vector6d b;
    std::memcpy(H.data(), o, 36 * sizeof(double));
    std::memcpy(b.data(), o + 36, 6 * sizeof(double));
    return {H, b, o[42]};
  }
  template <typename Target, typename Source, typename Factor>
  double error(const Target&, const Source&, const M::Isometry3d& T, std::vector<Factor>&) const {
    return model_error(T.data());
  }
  template <typename Factor>
  void sync_factors(std::vector<Factor>& factors) const {  // the inliers of the last linearize: the first n_points - n_lin (none before one)
    const int n = n_lin ? f->n_points - n_lin : 0;
    for (size_t i = 0; i < factors.size(); i++) factors[i].target_index = static_cast<int>(i) < n ? i : static_cast<size_t>(-1);
  }
};

/// out = T(16) | converged, iterations, num_inliers, error | H(36) | b(6)
void write_out(const M::RegistrationResult& r, double* out) {
  std::memcpy(out, r.T_target_source.data(), 16 * sizeof(double));
  out[16] = r.converged;
  out[17] = static_cast<double>(r.iterations);
  out[18] = static_cast<double>(r.num_inliers);
  out[19] = r.error;
  std::memcpy(out + 20, r.H.data(), 36 * sizeof(double));
  std::memcpy(out + 56, r.b.data(), 6 * sizeof(double));
}

template <typename Optimizer, typename General>
void run_mirror(const Optimizer& opt, General general, const sgb::AlignOptions& o, const FakeModel& f, const double* T0, double* out) {
  M::TerminationCriteria crit;
  crit.rotation_eps = o.rotation_eps;
  crit.translation_eps = o.translation_eps;
  FakeReduction red{&f};
  std::vector<M::ICPFactor> factors(f.n_points);
  M::Isometry3d init;
  std::memcpy(init.matrix().data(), T0, 16 * sizeof(double));
  const int dummy = 0;
  write_out(opt.optimize(dummy, dummy, dummy, M::DistanceRejector(), crit, red, init, factors, general), out);
}

}  // namespace

extern "C" {

/// The batched align step's solve against the mirror's: (H + DoF term + lambda I) x = -b.  H: 36 doubles (column-major, symmetric),
/// mask: 6 doubles or NULL (NullFactor).  x_step / x_mirror: 6 doubles each.
void sgbm_damped_step(const double* H36, const double* b6, double lambda, const double* mask6, double* x_step, double* x_mirror) {
  sgb::MemberState s;
  sgb::AlignOptions o = {};
  for (int i = 0; i < 6; i++) o.dof_mask[i] = mask6 ? mask6[i] : 1.0;
  double out44[44] = {0.0};
  std::memcpy(out44, H36, 36 * sizeof(double));
  std::memcpy(out44 + 36, b6, 6 * sizeof(double));
  o.lm = 1;
  o.max_iterations = o.max_inner_iterations = 1;
  o.init_lambda = lambda;
  const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  sgb::align_init(o, I, s);
  sgb::align_after_linearize(o, s, out44);  // LM: the pending trial's increment is the damped step
  std::memcpy(x_step, s.delta, 6 * sizeof(double));
  M::Matrix6d H;
  M::Vector6d b;
  std::memcpy(H.data(), H36, 36 * sizeof(double));
  std::memcpy(b.data(), b6, 6 * sizeof(double));
  if (mask6) {
    M::RestrictDoFFactor g;
    g.set_rotation_mask(mask6[0], mask6[1], mask6[2]);
    g.set_translation_mask(mask6[3], mask6[4], mask6[5]);
    const int dummy = 0;
    g.update_linearized_system(dummy, dummy, dummy, M::Isometry3d(), &H, &b, nullptr);
  }
  const M::Vector6d x = M::detail::damped_step(H, b, lambda);
  std::memcpy(x_mirror, x.data(), 6 * sizeof(double));
}

/// T * se3_exp(a) by the step (se3_exp6 + pose_mul) and by the mirror (se3_exp + Isometry3d::operator*); exp_* = se3_exp(a) alone.
void sgbm_pose_update(const double* T16, const double* a6, double* exp_step16, double* exp_mirror16, double* T_step16, double* T_mirror16) {
  sgb::se3_exp6(a6, exp_step16);
  sgb::pose_mul(T16, exp_step16, T_step16);
  M::Vector6d a;
  std::memcpy(a.data(), a6, 6 * sizeof(double));
  M::Isometry3d T;
  std::memcpy(T.matrix().data(), T16, 16 * sizeof(double));
  const M::Isometry3d E = M::se3_exp(a);
  std::memcpy(exp_mirror16, E.data(), 16 * sizeof(double));
  std::memcpy(T_mirror16, (T * E).data(), 16 * sizeof(double));
}

/// One align() against the fake reduction, by the device step's state machine and by the mirror's optimizer.
/// opt12 = lm, max_iterations, max_inner_iterations, gn_lambda, init_lambda, lambda_factor, rotation_eps, translation_eps, use_mask, -, -, -;
/// mask6; model20 = target(6), w(6), coupling, gain, bump, reject_from, n_points, -, -, -.  out_step / out_mirror: 62 doubles
/// (T | converged, iterations, inliers, error | H | b); rounds2 = linearize rounds, error rounds of the step.
void sgbm_align_fake(const double* opt12, const double* mask6, const double* model20, const double* T0, double* out_step, double* out_mirror, double* rounds2) {
  sgb::AlignOptions o;
  o.lm = static_cast<int>(opt12[0]);
  o.max_iterations = static_cast<int>(opt12[1]);
  o.max_inner_iterations = static_cast<int>(opt12[2]);
  o.gn_lambda = opt12[3];
  o.init_lambda = opt12[4];
  o.lambda_factor = opt12[5];
  o.rotation_eps = opt12[6];
  o.translation_eps = opt12[7];
  const bool use_mask = opt12[8] != 0.0;
  for (int i = 0; i < 6; i++) o.dof_mask[i] = use_mask ? mask6[i] : 1.0;
  FakeModel f;
  for (int i = 0; i < 6; i++) f.target[i] = model20[i], f.w[i] = model20[6 + i];
  f.coupling = model20[12];
  f.gain = model20[13];
  f.bump = model20[14];
  f.reject_from = static_cast<int>(model20[15]);
  f.n_points = static_cast<int>(model20[16]);

  // the step: what sgb_align_batch and batch_step_kernel do for one member
  FakeReduction red{&f};
  sgb::MemberState s;
  sgb::align_init(o, T0, s);
  rounds2[0] = rounds2[1] = 0;
  while (s.phase != sgb::kPhaseDone) {
    if (s.phase == sgb::kPhaseLinearize) {
      double out44[44];
      red.linearize44(s.T, out44);
      sgb::align_after_linearize(o, s, out44);
      rounds2[0]++;
    } else {
      sgb::align_after_error(o, s, red.model_error(s.cand));
      rounds2[1]++;
    }
  }
  std::memcpy(out_step, s.T, 16 * sizeof(double));
  out_step[16] = s.converged;
  out_step[17] = s.iterations;
  out_step[18] = s.inliers;
  out_step[19] = s.e;
  std::memcpy(out_step + 20, s.H, 36 * sizeof(double));
  std::memcpy(out_step + 56, s.b, 6 * sizeof(double));

  // the mirror
  M::RestrictDoFFactor dof;
  if (use_mask) {
    dof.set_rotation_mask(mask6[0], mask6[1], mask6[2]);
    dof.set_translation_mask(mask6[3], mask6[4], mask6[5]);
  }
  const M::NullFactor none;
  if (o.lm) {
    M::LevenbergMarquardtOptimizer opt;
    opt.max_iterations = o.max_iterations;
    opt.max_inner_iterations = o.max_inner_iterations;
    opt.init_lambda = o.init_lambda;
    opt.lambda_factor = o.lambda_factor;
    use_mask ? run_mirror(opt, dof, o, f, T0, out_mirror) : run_mirror(opt, none, o, f, T0, out_mirror);
  } else {
    M::GaussNewtonOptimizer opt;
    opt.max_iterations = o.max_iterations;
    opt.lambda = o.gn_lambda;
    use_mask ? run_mirror(opt, dof, o, f, T0, out_mirror) : run_mirror(opt, none, o, f, T0, out_mirror);
  }
}

}  // extern "C"
