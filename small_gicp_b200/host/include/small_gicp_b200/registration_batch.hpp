// SPDX-License-Identifier: MIT
// BatchRegistration: Registration<>::align (registration.hpp) of many source clouds against one target, each from its own initial pose,
// in one sgb_align_batch call.  The optimiser runs on the device, one step per member and round, with the arithmetic and the decisions of
// GaussNewtonOptimizer / LevenbergMarquardtOptimizer (include/sgicp_b200.h, DESIGN.md §11).  The types below are only mapped to
// sgb_align_options, as ParallelReductionCUDA maps them to kernel selectors; unsupported types are compile errors.
#pragma once
#include <cstring>
#include <stdexcept>
#include <tuple>
#include <string>
#include <type_traits>
#include <utility>
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
/// point-to-plane, with or without a robust kernel: its residual n o r is not rotation invariant, so it has no meaning against maps
/// that each sit at a pose of their own (sgb_source_set_submaps)
template <typename Factor>
struct is_point_to_plane : std::false_type {};
template <>
struct is_point_to_plane<PointToPlaneICPFactor> : std::true_type {};
template <typename Kernel>
struct is_point_to_plane<RobustFactor<Kernel, PointToPlaneICPFactor>> : std::true_type {};
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
    const Concatenated src(sources);
    check(ctx, sgb_source_set_batch(ctx, sources.size(), src.offsets.data(), src.points.data(), src.covs_or_null()));
    return run(ctx, init_Ts);
  }

  /// One RegistrationResult per (target, source) pair, in order: source m from init_Ts[m] against a Gaussian voxel map of targets[m]
  /// (GaussianVoxelMap(voxel_resolution) with search_offsets 1 / 7 / 27, inserted once), all pairs in one sgb_align_batch call.  The maps are
  /// built on the device in one sgb_target_build_voxelmaps call; the targets need covariances for GICP.  To pair a cloud with
  /// several others, use the overload with a pair list.  The context's target is replaced, so the reduction's target mirror is dropped.
  template <typename Target, typename Source>
  std::vector<RegistrationResult> align(const std::vector<Target>& targets, const std::vector<Source>& sources, const std::vector<Isometry3d>& init_Ts,
                                        double voxel_resolution, int search_offsets) const {
    if (sources.size() != init_Ts.size()) throw std::runtime_error("BatchRegistration: one initial pose per source");
    if (targets.size() != sources.size()) throw std::runtime_error("BatchRegistration: one target per source");
    sgb_ctx* ctx = reduction.context();
    reduction.invalidate();
    const Concatenated tgt(targets), src(sources);
    check(ctx, sgb_target_build_voxelmaps(ctx, targets.size(), tgt.offsets.data(), tgt.points.data(), tgt.covs_or_null(), voxel_resolution, search_offsets));
    check(ctx, sgb_source_set_batch(ctx, sources.size(), src.offsets.data(), src.points.data(), src.covs_or_null()));
    return run(ctx, init_Ts);
  }

  /// One RegistrationResult per (target, source) pair, in order: source m from init_Ts[m] against targets[m] through its own kd-tree
  /// (Registration<>::align with a KdTree of the target), all pairs in one sgb_align_batch call.  The trees are built on the device in one
  /// sgb_target_build_kdtrees call; the targets need normals for point-to-plane and covariances for GICP.  The context's target is
  /// replaced, so the reduction's target mirror is dropped.
  template <typename Target, typename Source>
  std::vector<RegistrationResult> align(const std::vector<Target>& targets, const std::vector<Source>& sources, const std::vector<Isometry3d>& init_Ts) const {
    if (sources.size() != init_Ts.size()) throw std::runtime_error("BatchRegistration: one initial pose per source");
    if (targets.size() != sources.size()) throw std::runtime_error("BatchRegistration: one target per source");
    sgb_ctx* ctx = reduction.context();
    reduction.invalidate();
    const Concatenated tgt(targets, true), src(sources);
    check(ctx, sgb_target_build_kdtrees(ctx, targets.size(), tgt.offsets.data(), tgt.points.data(), tgt.normals_or_null(), tgt.covs_or_null()));
    check(ctx, sgb_source_set_batch(ctx, sources.size(), src.offsets.data(), src.points.data(), src.covs_or_null()));
    return run(ctx, init_Ts);
  }

  /// One RegistrationResult per (source index, target index) pair, in order: sources[pairs[p].first] from init_Ts[p] against the kd-tree
  /// of targets[pairs[p].second].  Each target's tree is built once and each source uploaded once, however many pairs use it
  /// (sgb_source_set_pairs); all pairs in one sgb_align_batch call.  Normals / covariances as for the one-to-one overload.
  template <typename Target, typename Source>
  std::vector<RegistrationResult> align(const std::vector<Target>& targets, const std::vector<Source>& sources, const std::vector<std::pair<size_t, size_t>>& pairs,
                                        const std::vector<Isometry3d>& init_Ts) const {
    sgb_ctx* ctx = reduction.context();
    reduction.invalidate();
    const Concatenated tgt(targets, true);
    check(ctx, sgb_target_build_kdtrees(ctx, targets.size(), tgt.offsets.data(), tgt.points.data(), tgt.normals_or_null(), tgt.covs_or_null()));
    return run_pairs(ctx, sources, targets.size(), pairs, init_Ts);
  }

  /// The same against a Gaussian voxel map of each target (the voxel-map overload's settings), each map built once.
  template <typename Target, typename Source>
  std::vector<RegistrationResult> align(const std::vector<Target>& targets, const std::vector<Source>& sources, const std::vector<std::pair<size_t, size_t>>& pairs,
                                        const std::vector<Isometry3d>& init_Ts, double voxel_resolution, int search_offsets) const {
    sgb_ctx* ctx = reduction.context();
    reduction.invalidate();
    const Concatenated tgt(targets);
    check(ctx, sgb_target_build_voxelmaps(ctx, targets.size(), tgt.offsets.data(), tgt.points.data(), tgt.covs_or_null(), voxel_resolution, search_offsets));
    return run_pairs(ctx, sources, targets.size(), pairs, init_Ts);
  }

  /// Multi-start: one RegistrationResult per member, in order: sources[cloud_of_member[p]] from init_Ts[p] against the one target, each
  /// source uploaded once however many starts it has.
  template <typename Target, typename Tree, typename Source>
  std::vector<RegistrationResult> align(const Target& target, const Tree& target_tree, const std::vector<Source>& sources, const std::vector<size_t>& cloud_of_member,
                                        const std::vector<Isometry3d>& init_Ts) const {
    if (cloud_of_member.size() != init_Ts.size()) throw std::runtime_error("BatchRegistration: one initial pose per member");
    sgb_ctx* ctx = reduction.batch_context(target, target_tree);
    const Concatenated src(sources);
    check(ctx, sgb_source_set_batch(ctx, sources.size(), src.offsets.data(), src.points.data(), src.covs_or_null()));
    const std::vector<uint32_t> clouds = indices(cloud_of_member, sources.size(), "source");
    check(ctx, sgb_source_set_pairs(ctx, clouds.size(), clouds.data(), nullptr));
    return run(ctx, init_Ts);
  }

  /// Submaps: one RegistrationResult per member, in order: sources[cloud_of_member[p]] from init_Ts[p] (source -> common frame) against
  /// the UNION of submaps[p], a list of (index into maps, pose of that map in the common frame).  Each map's kd-tree is built once and
  /// no map is transformed, however many lists name it and whatever its poses (sgb_source_set_submaps); all members in one
  /// sgb_align_batch call.  ICP and GICP (the maps need covariances); point-to-plane does not compile.
  template <typename Target, typename Source>
  std::vector<RegistrationResult> align(const std::vector<Target>& maps, const std::vector<Source>& sources, const std::vector<size_t>& cloud_of_member,
                                        const std::vector<std::vector<std::pair<size_t, Isometry3d>>>& submaps, const std::vector<Isometry3d>& init_Ts) const {
    static_assert(!detail::is_point_to_plane<PointFactor>::value,
                  "BatchRegistration: point-to-plane is not available against submaps (its element-wise residual n o r is not invariant under the map poses); use ICPFactor or GICPFactor");
    if (cloud_of_member.size() != init_Ts.size() || submaps.size() != init_Ts.size()) throw std::runtime_error("BatchRegistration: one cloud, one submap list and one initial pose per member");
    sgb_ctx* ctx = reduction.context();
    reduction.invalidate();
    const Concatenated tgt(maps), src(sources);
    check(ctx, sgb_target_build_kdtrees(ctx, maps.size(), tgt.offsets.data(), tgt.points.data(), nullptr, tgt.covs_or_null()));
    check(ctx, sgb_source_set_batch(ctx, sources.size(), src.offsets.data(), src.points.data(), src.covs_or_null()));
    const std::vector<uint32_t> clouds = indices(cloud_of_member, sources.size(), "source");
    std::vector<size_t> list_off(submaps.size() + 1, 0), entry_map;
    std::vector<double> poses;
    for (size_t p = 0; p < submaps.size(); p++) {
      list_off[p + 1] = list_off[p] + submaps[p].size();
      for (const auto& entry : submaps[p]) {
        entry_map.push_back(entry.first);
        poses.insert(poses.end(), entry.second.data(), entry.second.data() + 16);
      }
    }
    const std::vector<uint32_t> entry_maps = indices(entry_map, maps.size(), "map");
    check(ctx, sgb_source_set_submaps(ctx, clouds.size(), clouds.data(), list_off.data(), entry_maps.data(), poses.data()));
    return run(ctx, init_Ts);
  }

  TerminationCriteria criteria;
  CorrespondenceRejector rejector;
  PointFactorSetting point_factor;
  GeneralFactor general_factor;
  ParallelReductionCUDA reduction;
  Optimizer optimizer;

private:
  /// clouds concatenated in the C-ABI's batch layout; covariances (and with want_normals normals) only if every non-empty cloud has them
  struct Concatenated {
    std::vector<size_t> offsets;
    std::vector<double> points, normals, covs;
    bool has_normals = true, has_covs = true;
    template <typename Cloud>
    explicit Concatenated(const std::vector<Cloud>& clouds, bool want_normals = false) : offsets(clouds.size() + 1, 0), has_normals(want_normals) {
      const size_t B = clouds.size();
      std::vector<detail::CloudArrays<Cloud>> arrays;
      arrays.reserve(B);
      for (size_t m = 0; m < B; m++) {
        arrays.emplace_back(clouds[m], want_normals);
        offsets[m + 1] = offsets[m] + arrays[m].n;
        has_normals = has_normals && (arrays[m].n == 0 || arrays[m].normals);
        has_covs = has_covs && (arrays[m].n == 0 || arrays[m].covs);
      }
      points.resize(4 * offsets[B]);
      normals.resize(has_normals ? 4 * offsets[B] : 0);
      covs.resize(has_covs ? 16 * offsets[B] : 0);
      for (size_t m = 0; m < B; m++) {
        if (arrays[m].n == 0) continue;
        std::memcpy(points.data() + 4 * offsets[m], arrays[m].points, arrays[m].n * 4 * sizeof(double));
        if (has_normals) std::memcpy(normals.data() + 4 * offsets[m], arrays[m].normals, arrays[m].n * 4 * sizeof(double));
        if (has_covs) std::memcpy(covs.data() + 16 * offsets[m], arrays[m].covs, arrays[m].n * 16 * sizeof(double));
      }
    }
    const double* normals_or_null() const { return has_normals ? normals.data() : nullptr; }
    const double* covs_or_null() const { return has_covs ? covs.data() : nullptr; }
  };

  static std::vector<uint32_t> indices(const std::vector<size_t>& idx, size_t count, const char* what) {
    std::vector<uint32_t> out(idx.size());
    for (size_t p = 0; p < idx.size(); p++) {
      if (idx[p] >= count) throw std::runtime_error(std::string("BatchRegistration: member ") + std::to_string(p) + " names " + what + " " + std::to_string(idx[p]) + " of " + std::to_string(count));
      out[p] = static_cast<uint32_t>(idx[p]);
    }
    return out;
  }

  /// the sources uploaded once, paired as the list says with the maps of the context's many-maps target, then aligned
  template <typename Source>
  std::vector<RegistrationResult> run_pairs(sgb_ctx* ctx, const std::vector<Source>& sources, size_t n_maps, const std::vector<std::pair<size_t, size_t>>& pairs,
                                            const std::vector<Isometry3d>& init_Ts) const {
    if (pairs.size() != init_Ts.size()) throw std::runtime_error("BatchRegistration: one initial pose per pair");
    std::vector<size_t> c(pairs.size()), t(pairs.size());
    for (size_t p = 0; p < pairs.size(); p++) std::tie(c[p], t[p]) = pairs[p];
    const Concatenated src(sources);
    check(ctx, sgb_source_set_batch(ctx, sources.size(), src.offsets.data(), src.points.data(), src.covs_or_null()));
    const std::vector<uint32_t> clouds = indices(c, sources.size(), "source"), maps = indices(t, n_maps, "target");
    check(ctx, sgb_source_set_pairs(ctx, clouds.size(), clouds.data(), maps.data()));
    return run(ctx, init_Ts);
  }

  /// sgb_align_batch of the context's batch from init_Ts with this registration's settings
  std::vector<RegistrationResult> run(sgb_ctx* ctx, const std::vector<Isometry3d>& init_Ts) const {
    const size_t B = init_Ts.size();
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

  static void check(sgb_ctx* ctx, int rc) {
    if (rc != 0) throw std::runtime_error(std::string("BatchRegistration: ") + sgb_last_error(ctx));
  }
};

}  // namespace small_gicp_b200
