// SPDX-License-Identifier: MIT
// How a user of koide3/small_gicp calls the H100 backend: the three entry levels of the reference's public API -- the one-call
// helper, pre-processing + align, and the Registration<> template -- exercised on a pair of PLY files.  Inside the reference
// tree the includes would be <small_gicp/...> plus <small_gicp/registration/reduction_cuda.hpp> (INTEGRATION.md); here they
// come from this repository's Eigen-free mirror of the same surface.  All per-point work (voxel grid, normals / covariances,
// nearest neighbours, factors, the H | b | e reduction) happens on the GPU inside libsgicp_b200.so; the host only solves 6 x 6.
//
//   make -C examples && examples/registration_on_b200 target.ply source.ply
#include <cstdio>
#include <cstdlib>
#include <iostream>

#include <small_gicp_b200/read_points.hpp>
#include <small_gicp_b200/registration_helper.hpp>

namespace sg = small_gicp_b200;

static void report(const char* title, const sg::RegistrationResult& r) {
  std::printf("== %s\n   converged %d after iteration %zu, %zu inliers, error %.6g\n", title, r.converged ? 1 : 0, r.iterations, r.num_inliers, r.error);
  for (int row = 0; row < 3; row++)
    std::printf("   [% .6f % .6f % .6f | % .4f]\n", r.T_target_source.matrix()(row, 0), r.T_target_source.matrix()(row, 1), r.T_target_source.matrix()(row, 2),
                r.T_target_source.matrix()(row, 3));
  double trace = 0.0;
  for (int k = 0; k < 6; k++) trace += r.H(k, k);
  std::printf("   trace(H) %.6g, |b| %.3g\n", trace, r.b.norm());
}

int main(int argc, char** argv) {
  if (argc < 3) {
    std::fprintf(stderr, "usage: %s target.ply source.ply [cuda device]\n", argv[0]);
    return 1;
  }
  const std::vector<sg::Vector4f> target_raw = sg::read_ply(argv[1]), source_raw = sg::read_ply(argv[2]);
  if (target_raw.empty() || source_raw.empty()) {
    std::fprintf(stderr, "error: could not read %s / %s (binary PLY with float x y z ... expected)\n", argv[1], argv[2]);
    return 1;
  }
  const int device = argc > 3 ? std::atoi(argv[3]) : 0;
  try {
    // Level 1 -- small_gicp::align(points, points, init, setting): raw points in, pose out.
    sg::RegistrationSetting setting;              // GICP, 0.25 m voxel grid, 1 m correspondence distance, 20 LM iterations: the reference's defaults
    setting.type = sg::RegistrationSetting::GICP;
    setting.device = device;                      // the one field the reference does not have (its num_threads is accepted and ignored)
    report("helper align(), GICP", sg::align(target_raw, source_raw, sg::Isometry3d::Identity(), setting));

    // Level 2 -- pre-process once, register many times (both directions here).
    auto [target, target_tree] = sg::preprocess_points(target_raw, setting.downsampling_resolution, /*num_neighbors=*/10, /*num_threads=*/1, device);
    auto [source, source_tree] = sg::preprocess_points(source_raw, setting.downsampling_resolution, 10, 1, device);
    std::printf("   down-sampled to %zu / %zu points\n", target->size(), source->size());
    setting.type = sg::RegistrationSetting::PLANE_ICP;
    report("pre-processed clouds, point-to-plane ICP", sg::align(*target, *source, *target_tree, sg::Isometry3d::Identity(), setting));
    setting.type = sg::RegistrationSetting::GICP;
    report("the same clouds the other way round", sg::align(*source, *target, *source_tree, sg::Isometry3d::Identity(), setting));
    setting.type = sg::RegistrationSetting::VGICP;
    report("VGICP against a Gaussian voxel map", sg::align(*sg::create_gaussian_voxelmap(*target, setting.voxel_resolution), *source, sg::Isometry3d::Identity(), setting));

    // Level 3 -- the template surface: factor, reduction, (general factor, rejector, optimizer) chosen as types.  This is the line
    // that changes in user code: ParallelReductionCUDA where it said ParallelReductionOMP or ParallelReductionTBB.
    sg::Registration<sg::GICPFactor, sg::ParallelReductionCUDA> registration;
    registration.reduction.device = device;
    registration.rejector.max_dist_sq = 1.0;
    registration.optimizer.max_iterations = 30;
    report("Registration<GICPFactor, ParallelReductionCUDA>", registration.align(*target, *source, *target_tree, sg::Isometry3d::Identity()));
  } catch (const std::exception& e) {  // no CUDA device, for one: the backend has no CPU fallback and says so
    std::fprintf(stderr, "error: %s\n", e.what());
    return 2;
  }
  return 0;
}
