// SPDX-License-Identifier: MIT
// BatchRegistration: Registration<>::align (registration.hpp) of many source clouds against one target, each from its own initial pose,
// in one sgb_align_batch call.  The optimiser runs on the device, one step per member and round, with the arithmetic and the decisions of
// GaussNewtonOptimizer / LevenbergMarquardtOptimizer (include/sgicp_b200.h, DESIGN.md §11).  The types below are only mapped to
// sgb_align_options, as ParallelReductionCUDA maps them to kernel selectors; unsupported types are compile errors.
#pragma once
#include <cstring>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "../../../../include/sgicp_b200.h"
#include "core.hpp"
#include "factors.hpp"
#include "reduction_cuda.hpp"
#include "registration.hpp"

namespace small_gicp_b200 {

namespace detail {
template <typename Optimizer>
void set_optimizer(sgb_align_options& o, const Optimizer& opt) {
  if constexpr (std::is_same_v<Optimizer, GaussNewtonOptimizer>) {
    o.optimizer_kind = SGB_OPT_GAUSS_NEWTON;
    o.gn_lambda = opt.lambda;
  } else if constexpr (std::is_same_v<Optimizer, LevenbergMarquardtOptimizer>) {
    o.optimizer_kind = SGB_OPT_LEVENBERG_MARQUARDT;
    o.max_inner_iterations = opt.max_inner_iterations;
    o.init_lambda = opt.init_lambda;
    o.lambda_factor = opt.lambda_factor;
  } else {
    static_assert(dependent_false<Optimizer>::value, "BatchRegistration: GaussNewtonOptimizer or LevenbergMarquardtOptimizer");
  }
  o.max_iterations = opt.max_iterations;
}

template <typename GeneralFactor>
void set_general_factor(sgb_align_options& o, const GeneralFactor& g) {
  if constexpr (std::is_same_v<GeneralFactor, NullFactor>) {
    for (int i = 0; i < 6; i++) o.dof_mask[i] = 1.0;
  } else if constexpr (std::is_same_v<GeneralFactor, RestrictDoFFactor>) {
    if (g.lambda != 1e9) throw std::runtime_error("BatchRegistration: RestrictDoFFactor::lambda must be 1e9 (the device step adds 1e9 |mask_i - 1|)");
    for (int i = 0; i < 6; i++) o.dof_mask[i] = g.mask[i];
  } else {
    static_assert(dependent_false<GeneralFactor>::value, "BatchRegistration: NullFactor or RestrictDoFFactor");
  }
}
}  // namespace detail

template <typename PointFactor, typename GeneralFactor = NullFactor, typename CorrespondenceRejector = DistanceRejector,
          typename Optimizer = LevenbergMarquardtOptimizer>
struct BatchRegistration {
  using PointFactorSetting = typename PointFactor::Setting;

  /// One RegistrationResult per source, in order.  init_Ts: one initial pose per source.  The target is mirrored to the device through
  /// reduction (a ParallelReductionCUDA, whose context and target mirror are kept across calls like Registration<>'s).
  template <typename Target, typename Tree, typename Source>
  std::vector<RegistrationResult> align(const Target& target, const Tree& target_tree, const std::vector<Source>& sources,
                                        const std::vector<Isometry3d>& init_Ts) const {
    if (sources.size() != init_Ts.size()) throw std::runtime_error("BatchRegistration: one initial pose per source");
    sgb_ctx* ctx = reduction.batch_context(target, target_tree);
    // the members concatenated in the C-ABI's layout; covariances only if every non-empty member has them
    const size_t B = sources.size();
    std::vector<size_t> offsets(B + 1, 0);
    std::vector<detail::CloudArrays<Source>> arrays;
    arrays.reserve(B);
    bool covs = true;
    for (size_t m = 0; m < B; m++) {
      arrays.emplace_back(sources[m], false);
      offsets[m + 1] = offsets[m] + arrays[m].n;
      covs = covs && (arrays[m].n == 0 || arrays[m].covs);
    }
    std::vector<double> points(4 * offsets[B]), cov(covs ? 16 * offsets[B] : 0);
    for (size_t m = 0; m < B; m++) {
      if (arrays[m].n == 0) continue;
      std::memcpy(points.data() + 4 * offsets[m], arrays[m].points, arrays[m].n * 4 * sizeof(double));
      if (covs) std::memcpy(cov.data() + 16 * offsets[m], arrays[m].covs, arrays[m].n * 16 * sizeof(double));
    }
    check(ctx, sgb_source_set_batch(ctx, B, offsets.data(), points.data(), covs ? cov.data() : nullptr));

    const FactorDescriptor fd = factor_traits<PointFactor>::describe(PointFactor(point_factor));
    sgb_align_options o = {};
    o.factor_kind = fd.factor_kind;
    o.robust_kind = fd.robust_kind;
    o.robust_c = fd.robust_c;
    o.rejector_kind = CorrespondenceRejector::kind;
    o.max_dist_sq = rejector.threshold();
    o.rotation_eps = criteria.rotation_eps;
    o.translation_eps = criteria.translation_eps;
    detail::set_optimizer(o, optimizer);
    detail::set_general_factor(o, general_factor);

    std::vector<double> init(16 * B), T(16 * B), info(4 * B), Hb(42 * B);
    for (size_t m = 0; m < B; m++) std::memcpy(init.data() + 16 * m, init_Ts[m].data(), 16 * sizeof(double));
    check(ctx, sgb_align_batch(ctx, &o, init.data(), T.data(), info.data(), Hb.data()));
    std::vector<RegistrationResult> out(B);
    for (size_t m = 0; m < B; m++) {
      RegistrationResult& r = out[m];
      std::memcpy(r.T_target_source.matrix().data(), T.data() + 16 * m, 16 * sizeof(double));
      r.converged = info[4 * m] != 0.0;
      r.iterations = static_cast<size_t>(info[4 * m + 1]);
      r.num_inliers = static_cast<size_t>(info[4 * m + 2]);
      r.error = info[4 * m + 3];
      std::memcpy(r.H.data(), Hb.data() + 42 * m, 36 * sizeof(double));
      std::memcpy(r.b.data(), Hb.data() + 42 * m + 36, 6 * sizeof(double));
    }
    return out;
  }

  TerminationCriteria criteria;
  CorrespondenceRejector rejector;
  PointFactorSetting point_factor;
  GeneralFactor general_factor;
  ParallelReductionCUDA reduction;
  Optimizer optimizer;

private:
  static void check(sgb_ctx* ctx, int rc) {
    if (rc != 0) throw std::runtime_error(std::string("BatchRegistration: ") + sgb_last_error(ctx));
  }
};

}  // namespace small_gicp_b200
