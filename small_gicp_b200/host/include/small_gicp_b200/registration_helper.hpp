// SPDX-License-Identifier: MIT
// Convenience API with the reference's names and defaults:
//   RegistrationSetting, preprocess_points(), create_gaussian_voxelmap(), align() x3; preprocess_points_batch() for many clouds (extension)
//   (/root/reference/include/small_gicp/registration/registration_helper.hpp:18-90,
//    /root/reference/src/small_gicp/registration/registration_helper.cpp:22-137)
// Differences by construction: down-sampling and normal/covariance estimation run on the device through the C-ABI
// (sgb_voxelgrid_sampling / sgb_estimate_features) and the reduction is ParallelReductionCUDA instead of
// ParallelReductionOMP; `num_threads` is accepted and ignored.
#pragma once
#include <iostream>
#include <stdexcept>
#include <utility>

#include "read_points.hpp"
#include "core.hpp"
#include "factors.hpp"
#include "kdtree.hpp"
#include "reduction_cuda.hpp"
#include "registration.hpp"
#include "voxelmap.hpp"

namespace small_gicp_b200 {

struct RegistrationSetting {
  enum RegistrationType { ICP, PLANE_ICP, GICP, VGICP };

  RegistrationType type = GICP;
  double voxel_resolution = 1.0;             ///< voxel size of the VGICP target
  double downsampling_resolution = 0.25;     ///< used by the raw-points align() only
  double max_correspondence_distance = 1.0;  ///< [m]
  double rotation_eps = 0.1 * M_PI / 180.0;  ///< [rad]
  double translation_eps = 1e-3;             ///< [m]
  int num_threads = 4;                       ///< kept for source compatibility (host threads are not used on this path)
  int max_iterations = 20;
  bool verbose = false;
  int device = 0;  ///< CUDA device ordinal (extension)
};

namespace detail {
/// one scratch context per thread for the per-cloud preparation calls
inline sgb_ctx* helper_context(int device) {
  struct Holder {
    sgb_ctx* ctx = nullptr;
    int device = -1;
    ~Holder() {
      if (ctx) sgb_destroy(ctx);
    }
  };
  thread_local Holder h;
  if (!h.ctx || h.device != device) {
    if (h.ctx) sgb_destroy(h.ctx);
    h.ctx = nullptr;
    if (sgb_create(device, &h.ctx) != 0) throw std::runtime_error(std::string("small_gicp_b200: ") + sgb_last_error(nullptr));
    h.device = device;
  }
  return h.ctx;
}
inline void helper_check(sgb_ctx* ctx, int rc) {
  if (rc != 0) throw std::runtime_error(std::string("small_gicp_b200: ") + sgb_last_error(ctx));
}
}  // namespace detail

/// Voxel-grid down-sampling on the device (util/downsampling.hpp:22-78 semantics).
inline PointCloud::Ptr voxelgrid_sampling(const PointCloud& points, double leaf_size, int device = 0) {
  auto out = std::make_shared<PointCloud>();
  if (points.empty()) return out;
  sgb_ctx* ctx = detail::helper_context(device);
  std::vector<Vector4d> buf(points.size());
  size_t m = 0;
  detail::helper_check(ctx, sgb_voxelgrid_sampling(ctx, points.size(), points.points[0].data(), leaf_size, buf[0].data(), &m));
  out->resize(m);
  std::copy(buf.begin(), buf.begin() + m, out->points.begin());
  return out;
}

/// Normals and covariances from k nearest neighbours on the device (util/normal_estimation.hpp:128-140 semantics).
inline void estimate_normals_covariances(PointCloud& cloud, int num_neighbors = 20, int device = 0) {
  cloud.resize(cloud.size());
  if (cloud.empty()) return;
  sgb_ctx* ctx = detail::helper_context(device);
  detail::helper_check(ctx, sgb_estimate_features(ctx, cloud.size(), cloud.points[0].data(), num_neighbors, cloud.normals[0].data(), cloud.covs[0].data()));
}
inline void estimate_covariances(PointCloud& cloud, int num_neighbors = 20, int device = 0) {
  cloud.resize(cloud.size());
  if (cloud.empty()) return;
  sgb_ctx* ctx = detail::helper_context(device);
  detail::helper_check(ctx, sgb_estimate_features(ctx, cloud.size(), cloud.points[0].data(), num_neighbors, nullptr, cloud.covs[0].data()));
}
inline void estimate_normals(PointCloud& cloud, int num_neighbors = 20, int device = 0) {
  cloud.resize(cloud.size());
  if (cloud.empty()) return;
  sgb_ctx* ctx = detail::helper_context(device);
  detail::helper_check(ctx, sgb_estimate_features(ctx, cloud.size(), cloud.points[0].data(), num_neighbors, cloud.normals[0].data(), nullptr));
}

/// Down-sample, build the search tree, estimate normals + covariances (registration_helper.cpp:22-33).
inline std::pair<PointCloud::Ptr, std::shared_ptr<KdTree<PointCloud>>> preprocess_points(const PointCloud& points, double downsampling_resolution,
                                                                                         int num_neighbors = 10, int /*num_threads*/ = 4, int device = 0) {
  auto downsampled = voxelgrid_sampling(points, downsampling_resolution, device);
  auto kdtree = std::make_shared<KdTree<PointCloud>>(downsampled);
  estimate_normals_covariances(*downsampled, num_neighbors, device);
  return {downsampled, kdtree};
}

/// Many clouds prepared at once (a sequence of frames): device voxel grid of every cloud in one call (sgb_voxelgrid_sampling_batch), then
/// k-NN normals + covariances of every down-sampled cloud in one call (sgb_estimate_features_batch).  Returns one down-sampled cloud per
/// input; each equals preprocess_points(cloud, downsampling_resolution, num_neighbors).first, up to the exact-FP32-tie clause of
/// sgb_estimate_features_batch.  No host trees are built: sgb_target_build_kdtrees / BatchRegistration build theirs on the device.
inline std::vector<PointCloud::Ptr> preprocess_points_batch(const std::vector<PointCloud>& clouds, double downsampling_resolution, int num_neighbors = 10,
                                                            int device = 0) {
  const size_t B = clouds.size();
  std::vector<PointCloud::Ptr> out(B);
  std::vector<size_t> offsets(B + 1, 0), down_offsets(B + 1, 0);
  for (size_t c = 0; c < B; c++) {
    out[c] = std::make_shared<PointCloud>();
    offsets[c + 1] = offsets[c] + clouds[c].size();
  }
  const size_t n = offsets[B];
  if (n == 0) return out;
  std::vector<Vector4d> pts(n), down(n);
  for (size_t c = 0; c < B; c++) std::copy(clouds[c].points.begin(), clouds[c].points.end(), pts.begin() + offsets[c]);
  sgb_ctx* ctx = detail::helper_context(device);
  detail::helper_check(ctx, sgb_voxelgrid_sampling_batch(ctx, B, offsets.data(), pts[0].data(), downsampling_resolution, down[0].data(), down_offsets.data()));
  const size_t m = down_offsets[B];
  if (m == 0) return out;
  std::vector<Vector4d> normals(m);
  std::vector<Matrix4d> covs(m);
  detail::helper_check(ctx, sgb_estimate_features_batch(ctx, B, down_offsets.data(), down[0].data(), num_neighbors, normals[0].data(), covs[0].data()));
  for (size_t c = 0; c < B; c++) {
    const size_t first = down_offsets[c], count = down_offsets[c + 1] - first;
    PointCloud& o = *out[c];
    o.resize(count);
    std::copy(down.begin() + first, down.begin() + first + count, o.points.begin());
    std::copy(normals.begin() + first, normals.begin() + first + count, o.normals.begin());
    std::copy(covs.begin() + first, covs.begin() + first + count, o.covs.begin());
  }
  return out;
}

inline GaussianVoxelMap::Ptr create_gaussian_voxelmap(const PointCloud& points, double voxel_resolution) {
  auto voxelmap = std::make_shared<GaussianVoxelMap>(voxel_resolution);
  voxelmap->insert(points);
  return voxelmap;
}

/// Pre-processed clouds + tree (registration_helper.cpp:81-122).
inline RegistrationResult align(const PointCloud& target, const PointCloud& source, const KdTree<PointCloud>& target_tree,
                                const Isometry3d& init_T = Isometry3d::Identity(), const RegistrationSetting& setting = RegistrationSetting()) {
  auto run = [&](auto registration) {
    registration.reduction.device = setting.device;
    registration.reduction.use_context(detail::helper_context(setting.device));  // one long-lived context per thread, not one per call
    registration.rejector.max_dist_sq = setting.max_correspondence_distance * setting.max_correspondence_distance;
    registration.criteria.rotation_eps = setting.rotation_eps;
    registration.criteria.translation_eps = setting.translation_eps;
    registration.optimizer.max_iterations = setting.max_iterations;
    registration.optimizer.verbose = setting.verbose;
    return registration.align(target, source, target_tree, init_T);
  };
  switch (setting.type) {
    case RegistrationSetting::ICP:
      return run(Registration<ICPFactor, ParallelReductionCUDA>());
    case RegistrationSetting::PLANE_ICP:
      return run(Registration<PointToPlaneICPFactor, ParallelReductionCUDA>());
    case RegistrationSetting::GICP:
      return run(Registration<GICPFactor, ParallelReductionCUDA>());
    case RegistrationSetting::VGICP:
      std::cerr << "error: use align(const GaussianVoxelMap&, const PointCloud&, ...) for VGICP" << std::endl;
      return RegistrationResult(Isometry3d::Identity());
  }
  throw std::invalid_argument("invalid registration type");
}

/// VGICP against a Gaussian voxel map (registration_helper.cpp:125-137; the rejector keeps its default 1 m^2 there too).
inline RegistrationResult align(const GaussianVoxelMap& target, const PointCloud& source, const Isometry3d& init_T = Isometry3d::Identity(),
                                const RegistrationSetting& setting = RegistrationSetting()) {
  if (setting.type != RegistrationSetting::VGICP) std::cerr << "invalid registration type for GaussianVoxelMap" << std::endl;
  Registration<GICPFactor, ParallelReductionCUDA> registration;
  registration.reduction.device = setting.device;
  registration.reduction.use_context(detail::helper_context(setting.device));
  registration.criteria.rotation_eps = setting.rotation_eps;
  registration.criteria.translation_eps = setting.translation_eps;
  registration.optimizer.max_iterations = setting.max_iterations;
  registration.optimizer.verbose = setting.verbose;
  return registration.align(target, source, target, init_T);
}

/// Raw points in, registration out (registration_helper.cpp:58-69): both clouds are down-sampled and given k = 10 features, then aligned.
/// The reference builds two host kd-trees here (preprocess_points) and throws them away with the call; nothing outside can see them, so this
/// overload keeps everything device-side instead: device voxel grid, device feature estimation -- only what the chosen factor reads
/// (ICP: nothing, point-to-plane: target normals, GICP / VGICP: both covariances) -- and a DeviceKdTree handle, i.e. the search structure is
/// built by sgb_target_build_kdtree inside the reduction's context rather than built on the host and adopted (6k-point pair: 36 -> ~8 ms).
/// Exact nearest neighbours do not depend on which tree is walked; preprocess_points() + align(target, source, tree) remains the
/// reference-shaped path for callers that want the host tree.
inline RegistrationResult align(const PointCloud& target_raw, const PointCloud& source_raw, const Isometry3d& init_T = Isometry3d::Identity(),
                                const RegistrationSetting& setting = RegistrationSetting()) {
  auto target = voxelgrid_sampling(target_raw, setting.downsampling_resolution, setting.device);
  auto source = voxelgrid_sampling(source_raw, setting.downsampling_resolution, setting.device);
  const bool gicp = setting.type == RegistrationSetting::GICP || setting.type == RegistrationSetting::VGICP;
  if (setting.type == RegistrationSetting::PLANE_ICP) estimate_normals(*target, 10, setting.device);
  if (gicp) {
    estimate_covariances(*target, 10, setting.device);
    estimate_covariances(*source, 10, setting.device);
  }
  if (setting.type == RegistrationSetting::VGICP) {
    auto voxelmap = create_gaussian_voxelmap(*target, setting.voxel_resolution);
    return align(*voxelmap, *source, init_T, setting);
  }
  const DeviceKdTree<PointCloud> tree(target);
  auto run = [&](auto registration) {
    registration.reduction.device = setting.device;
    registration.reduction.use_context(detail::helper_context(setting.device));
    registration.rejector.max_dist_sq = setting.max_correspondence_distance * setting.max_correspondence_distance;
    registration.criteria.rotation_eps = setting.rotation_eps;
    registration.criteria.translation_eps = setting.translation_eps;
    registration.optimizer.max_iterations = setting.max_iterations;
    registration.optimizer.verbose = setting.verbose;
    return registration.align(*target, *source, tree, init_T);
  };
  switch (setting.type) {
    case RegistrationSetting::ICP:
      return run(Registration<ICPFactor, ParallelReductionCUDA>());
    case RegistrationSetting::PLANE_ICP:
      return run(Registration<PointToPlaneICPFactor, ParallelReductionCUDA>());
    default:
      return run(Registration<GICPFactor, ParallelReductionCUDA>());
  }
}

/// Raw single-precision points (registration_helper.hpp:26-29: the std::vector<Eigen::Vector4f> overload).
inline std::pair<PointCloud::Ptr, std::shared_ptr<KdTree<PointCloud>>> preprocess_points(const std::vector<Vector4f>& points, double downsampling_resolution,
                                                                                         int num_neighbors = 10, int num_threads = 4, int device = 0) {
  return preprocess_points(*make_point_cloud(points), downsampling_resolution, num_neighbors, num_threads, device);
}

/// Raw single-precision points in, registration out (registration_helper.hpp:57-63, registration_helper.cpp:37-56).
inline RegistrationResult align(const std::vector<Vector4f>& target, const std::vector<Vector4f>& source, const Isometry3d& init_T = Isometry3d::Identity(),
                                const RegistrationSetting& setting = RegistrationSetting()) {
  return align(*make_point_cloud(target), *make_point_cloud(source), init_T, setting);
}

}  // namespace small_gicp_b200
