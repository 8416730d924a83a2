// SPDX-License-Identifier: MIT
// libsgicp_b200_host.so -- a thin C entry point over the C++ host mirror so that the Python tests can
// drive  Registration<Factor, ParallelReductionCUDA, GeneralFactor, Rejector, Optimizer>::align()
// exactly as a C++ user of the reference would (the template instantiations below are the ones the
// reference's registration_test.cpp:284-292 and registration_helper.cpp:81-137 exercise).
#include <cstring>
#include <memory>
#include <string>

#include <small_gicp_b200/core.hpp>
#include <small_gicp_b200/factors.hpp>
#include <small_gicp_b200/kdtree.hpp>
#include <small_gicp_b200/reduction_cuda.hpp>
#include <small_gicp_b200/registration.hpp>
#include <small_gicp_b200/registration_batch.hpp>
#include <small_gicp_b200/registration_helper.hpp>
#include <small_gicp_b200/voxelmap.hpp>

using namespace small_gicp_b200;

namespace {
thread_local std::string g_error;

struct Options {
  int factor;          // sgb_factor_kind
  int robust;          // sgb_robust_kind
  double robust_c;
  int rejector;        // sgb_rejector_kind
  double max_dist_sq;
  int optimizer;       // 0 = GaussNewton, 1 = LevenbergMarquardt
  int max_iterations;
  double rotation_eps, translation_eps;
  int tree;            // 0 = host KdTree (reference-layout nodes), 1 = DeviceKdTree, 2 = GaussianVoxelMap target
  double voxel_resolution;
  int voxel_search_offsets;
  int restrict_dof;    // 0 = NullFactor, 1 = RestrictDoFFactor with the mask below
  double dof_mask[6];
  int device;
};

template <typename Reg>
void configure(Reg& reg, const Options& o) {
  reg.criteria.rotation_eps = o.rotation_eps;
  reg.criteria.translation_eps = o.translation_eps;
  reg.optimizer.max_iterations = o.max_iterations;
  reg.reduction.device = o.device;
}
template <typename Reg>
void set_rejector(Reg& reg, const Options& o, std::true_type) {
  reg.rejector.max_dist_sq = o.max_dist_sq;
}
template <typename Reg>
void set_rejector(Reg&, const Options&, std::false_type) {}
template <typename Reg>
void set_general(Reg& reg, const Options& o, std::true_type) {
  reg.general_factor.set_rotation_mask(o.dof_mask[0], o.dof_mask[1], o.dof_mask[2]);
  reg.general_factor.set_translation_mask(o.dof_mask[3], o.dof_mask[4], o.dof_mask[5]);
}
template <typename Reg>
void set_general(Reg&, const Options&, std::false_type) {}
template <typename Setting>
void set_robust(Setting& s, const Options& o, std::true_type) {
  s.robust_kernel.c = o.robust_c;
}
template <typename Setting>
void set_robust(Setting&, const Options&, std::false_type) {}

template <typename Factor, typename General, typename Rejector, typename Optimizer, bool kRobust>
RegistrationResult run(const Options& o, const std::shared_ptr<PointCloud>& target, const std::shared_ptr<PointCloud>& source, const Isometry3d& init) {
  Registration<Factor, ParallelReductionCUDA, General, Rejector, Optimizer> reg;
  configure(reg, o);
  set_rejector(reg, o, std::is_same<Rejector, DistanceRejector>());
  set_general(reg, o, std::is_same<General, RestrictDoFFactor>());
  set_robust(reg.point_factor, o, std::integral_constant<bool, kRobust>());
  if (o.tree == 2) {
    GaussianVoxelMap map(o.voxel_resolution);
    map.set_search_offsets(o.voxel_search_offsets);
    map.insert(*target);
    return reg.align(map, *source, map, init);
  }
  if (o.tree == 1) {
    DeviceKdTree<PointCloud> tree(target);
    return reg.align(*target, *source, tree, init);
  }
  KdTree<PointCloud> tree(target);
  return reg.align(*target, *source, tree, init);
}

/// BatchRegistration<...>::align of every source from its initial pose, configured like run()
template <typename Factor, typename General, typename Rejector, typename Optimizer, bool kRobust>
std::vector<RegistrationResult> run_batch(const Options& o, const std::shared_ptr<PointCloud>& target, const std::vector<PointCloud>& sources,
                                          const std::vector<Isometry3d>& init, const std::vector<size_t>* cloud_of_member) {
  BatchRegistration<Factor, General, Rejector, Optimizer> reg;
  configure(reg, o);
  set_rejector(reg, o, std::is_same<Rejector, DistanceRejector>());
  set_general(reg, o, std::is_same<General, RestrictDoFFactor>());
  set_robust(reg.point_factor, o, std::integral_constant<bool, kRobust>());
  if (o.tree == 2) {
    GaussianVoxelMap map(o.voxel_resolution);
    map.set_search_offsets(o.voxel_search_offsets);
    map.insert(*target);
    return cloud_of_member ? reg.align(map, map, sources, *cloud_of_member, init) : reg.align(map, map, sources, init);
  }
  if (o.tree == 1) {
    DeviceKdTree<PointCloud> tree(target);
    return cloud_of_member ? reg.align(*target, tree, sources, *cloud_of_member, init) : reg.align(*target, tree, sources, init);
  }
  KdTree<PointCloud> tree(target);
  return cloud_of_member ? reg.align(*target, tree, sources, *cloud_of_member, init) : reg.align(*target, tree, sources, init);
}

/// BatchRegistration<...>::align of every (target, source) pair: source m against a Gaussian voxel map of targets[m], configured like run()
template <typename Factor, typename General, typename Rejector, typename Optimizer, bool kRobust>
std::vector<RegistrationResult> run_pairs(const Options& o, const std::vector<PointCloud>& targets, const std::vector<PointCloud>& sources,
                                          const std::vector<Isometry3d>& init, const std::vector<std::pair<size_t, size_t>>* pairs) {
  BatchRegistration<Factor, General, Rejector, Optimizer> reg;
  configure(reg, o);
  set_rejector(reg, o, std::is_same<Rejector, DistanceRejector>());
  set_general(reg, o, std::is_same<General, RestrictDoFFactor>());
  set_robust(reg.point_factor, o, std::integral_constant<bool, kRobust>());
  if (o.tree == 1) return pairs ? reg.align(targets, sources, *pairs, init) : reg.align(targets, sources, init);  // TREE_DEVICE_KDTREE: a kd-tree per target
  return pairs ? reg.align(targets, sources, *pairs, init, o.voxel_resolution, o.voxel_search_offsets)
               : reg.align(targets, sources, init, o.voxel_resolution, o.voxel_search_offsets);
}

/// The registration types chosen by the options: job.call<Factor, GeneralFactor, Rejector, Optimizer, kRobust>().
struct SingleJob {
  const Options& o;
  const std::shared_ptr<PointCloud>& target;
  const std::shared_ptr<PointCloud>& source;
  const Isometry3d& init;
  RegistrationResult result;
  template <typename Factor, typename General, typename Rejector, typename Optimizer, bool kRobust>
  void call() {
    result = run<Factor, General, Rejector, Optimizer, kRobust>(o, target, source, init);
  }
};
struct BatchJob {
  const Options& o;
  const std::shared_ptr<PointCloud>& target;
  const std::vector<PointCloud>& sources;
  const std::vector<Isometry3d>& init;
  const std::vector<size_t>* cloud_of_member;  // or null: one member per source
  std::vector<RegistrationResult> results;
  template <typename Factor, typename General, typename Rejector, typename Optimizer, bool kRobust>
  void call() {
    results = run_batch<Factor, General, Rejector, Optimizer, kRobust>(o, target, sources, init, cloud_of_member);
  }
};

struct PairsJob {
  const Options& o;
  const std::vector<PointCloud>& targets;
  const std::vector<PointCloud>& sources;
  const std::vector<Isometry3d>& init;
  const std::vector<std::pair<size_t, size_t>>* pairs;  // or null: source m against target m
  std::vector<RegistrationResult> results;
  template <typename Factor, typename General, typename Rejector, typename Optimizer, bool kRobust>
  void call() {
    constexpr bool plane = std::is_same_v<Factor, PointToPlaneICPFactor> || std::is_same_v<Factor, RobustFactor<Huber, PointToPlaneICPFactor>> ||
                           std::is_same_v<Factor, RobustFactor<Cauchy, PointToPlaneICPFactor>>;
    if (plane && o.tree != 1) throw std::runtime_error("sgbh_align_batch_pairs: a voxel map has no normals (point-to-plane)");
    results = run_pairs<Factor, General, Rejector, Optimizer, kRobust>(o, targets, sources, init, pairs);
  }
};

struct SubmapsJob {
  const Options& o;
  const std::vector<PointCloud>& maps;
  const std::vector<PointCloud>& sources;
  const std::vector<size_t>& cloud_of_member;
  const std::vector<std::vector<std::pair<size_t, Isometry3d>>>& submaps;
  const std::vector<Isometry3d>& init;
  std::vector<RegistrationResult> results;
  template <typename Factor, typename General, typename Rejector, typename Optimizer, bool kRobust>
  void call() {
    if constexpr (detail::is_point_to_plane<Factor>::value) {  // the overload itself does not compile for it
      throw std::runtime_error("sgbh_align_batch_submaps: point-to-plane is not available against submaps");
    } else {
      BatchRegistration<Factor, General, Rejector, Optimizer> reg;
      configure(reg, o);
      set_rejector(reg, o, std::is_same<Rejector, DistanceRejector>());
      set_general(reg, o, std::is_same<General, RestrictDoFFactor>());
      set_robust(reg.point_factor, o, std::integral_constant<bool, kRobust>());
      results = reg.align(maps, sources, cloud_of_member, submaps, init);
    }
  }
};

template <typename Factor, bool kRobust, typename Job>
void dispatch_rest(const Options& o, Job& job) {
  const int key = (o.restrict_dof ? 4 : 0) | (o.rejector == SGB_REJECT_DISTANCE ? 2 : 0) | (o.optimizer ? 1 : 0);
  switch (key) {
    case 0: return job.template call<Factor, NullFactor, NullRejector, GaussNewtonOptimizer, kRobust>();
    case 1: return job.template call<Factor, NullFactor, NullRejector, LevenbergMarquardtOptimizer, kRobust>();
    case 2: return job.template call<Factor, NullFactor, DistanceRejector, GaussNewtonOptimizer, kRobust>();
    case 3: return job.template call<Factor, NullFactor, DistanceRejector, LevenbergMarquardtOptimizer, kRobust>();
    case 4: return job.template call<Factor, RestrictDoFFactor, NullRejector, GaussNewtonOptimizer, kRobust>();
    case 5: return job.template call<Factor, RestrictDoFFactor, NullRejector, LevenbergMarquardtOptimizer, kRobust>();
    case 6: return job.template call<Factor, RestrictDoFFactor, DistanceRejector, GaussNewtonOptimizer, kRobust>();
    default: return job.template call<Factor, RestrictDoFFactor, DistanceRejector, LevenbergMarquardtOptimizer, kRobust>();
  }
}

template <typename Base, typename Job>
void dispatch_robust(const Options& o, Job& job) {
  if (o.robust == SGB_ROBUST_HUBER) return dispatch_rest<RobustFactor<Huber, Base>, true>(o, job);
  if (o.robust == SGB_ROBUST_CAUCHY) return dispatch_rest<RobustFactor<Cauchy, Base>, true>(o, job);
  return dispatch_rest<Base, false>(o, job);
}

/// false: invalid factor kind
template <typename Job>
bool dispatch(const Options& o, Job& job) {
  switch (o.factor) {
    case SGB_FACTOR_ICP: dispatch_robust<ICPFactor>(o, job); return true;
    case SGB_FACTOR_PLANE_ICP: dispatch_robust<PointToPlaneICPFactor>(o, job); return true;
    case SGB_FACTOR_GICP: dispatch_robust<GICPFactor>(o, job); return true;
    default: return false;
  }
}

Options parse_options(const double* q) {
  Options o;
  o.factor = static_cast<int>(q[0]);
  o.robust = static_cast<int>(q[1]);
  o.robust_c = q[2];
  o.rejector = static_cast<int>(q[3]);
  o.max_dist_sq = q[4];
  o.optimizer = static_cast<int>(q[5]);
  o.max_iterations = static_cast<int>(q[6]);
  o.rotation_eps = q[7];
  o.translation_eps = q[8];
  o.tree = static_cast<int>(q[9]);
  o.voxel_resolution = q[10];
  o.voxel_search_offsets = static_cast<int>(q[11]);
  o.restrict_dof = static_cast<int>(q[12]);
  for (int i = 0; i < 6; i++) o.dof_mask[i] = q[13 + i];
  o.device = static_cast<int>(q[19]);
  return o;
}

void write_result(const RegistrationResult& r, double* T_out16, double* scalars_out4, double* H_out36, double* b_out6) {
  std::memcpy(T_out16, r.T_target_source.matrix().data(), sizeof(double) * 16);
  scalars_out4[0] = r.converged ? 1.0 : 0.0;
  scalars_out4[1] = static_cast<double>(r.iterations);
  scalars_out4[2] = static_cast<double>(r.num_inliers);
  scalars_out4[3] = r.error;
  if (H_out36) std::memcpy(H_out36, r.H.data(), sizeof(double) * 36);
  if (b_out6) std::memcpy(b_out6, r.b.data(), sizeof(double) * 6);
}

std::shared_ptr<PointCloud> make_cloud(size_t n, const double* pts4, const double* normals4, const double* covs16) {
  auto c = std::make_shared<PointCloud>();
  c->resize(n);
  if (n) {
    std::memcpy(c->points[0].data(), pts4, n * sizeof(Vector4d));
    if (normals4) std::memcpy(c->normals[0].data(), normals4, n * sizeof(Vector4d));
    if (covs16) std::memcpy(c->covs[0].data(), covs16, n * sizeof(Matrix4d));
  }
  if (!normals4) c->normals.clear();
  if (!covs16) c->covs.clear();
  return c;
}
}  // namespace

extern "C" {

const char* sgbh_last_error() { return g_error.c_str(); }

/// options: 21 doubles in the order of `Options` (ints passed as doubles).  init_T / T_out: column-major 4x4.
/// scalars_out: [converged, iterations, num_inliers, error].
int sgbh_align(size_t n_target, const double* target_pts4, const double* target_normals4, const double* target_covs16, size_t n_source,
               const double* source_pts4, const double* source_covs16, const double* options21, const double* init_T16, double* T_out16, double* scalars_out4,
               double* H_out36, double* b_out6) {
  try {
    const Options o = parse_options(options21);
    auto target = make_cloud(n_target, target_pts4, target_normals4, target_covs16);
    auto source = make_cloud(n_source, source_pts4, nullptr, source_covs16);
    Isometry3d init;
    std::memcpy(init.matrix().data(), init_T16, sizeof(double) * 16);
    SingleJob job{o, target, source, init, RegistrationResult()};
    if (!dispatch(o, job)) {
      g_error = "sgbh_align: invalid factor kind";
      return 1;
    }
    write_result(job.result, T_out16, scalars_out4, H_out36, b_out6);
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 2;
  }
}

/// BatchRegistration<...>::align: the options of sgbh_align; n_sources sources concatenated (source m = rows offsets[m] .. offsets[m+1]).
/// cloud_of_member NULL: one member per source (n_members = n_sources); else member p is source cloud_of_member[p] (the multi-start
/// overload).  One initial pose per member.  Outputs as sgbh_align's, member after member (16 / 4 / 36 / 6 doubles each).
int sgbh_align_batch(size_t n_target, const double* target_pts4, const double* target_normals4, const double* target_covs16, size_t n_sources,
                     const size_t* offsets, const double* source_pts4, const double* source_covs16, const double* options21, const double* init_T16xB,
                     double* T_out16xB, double* scalars_out4xB, double* H_out36xB, double* b_out6xB, size_t n_members, const size_t* cloud_of_member) {
  try {
    const Options o = parse_options(options21);
    auto target = make_cloud(n_target, target_pts4, target_normals4, target_covs16);
    std::vector<PointCloud> sources(n_sources);
    for (size_t m = 0; m < n_sources; m++) {
      const size_t off = offsets[m], n = offsets[m + 1] - off;
      sources[m] = *make_cloud(n, source_pts4 + 4 * off, nullptr, source_covs16 ? source_covs16 + 16 * off : nullptr);
    }
    if (!cloud_of_member) n_members = n_sources;
    const std::vector<size_t> members(cloud_of_member, cloud_of_member + (cloud_of_member ? n_members : 0));
    std::vector<Isometry3d> init(n_members);
    for (size_t m = 0; m < n_members; m++) std::memcpy(init[m].matrix().data(), init_T16xB + 16 * m, sizeof(double) * 16);
    BatchJob job{o, target, sources, init, cloud_of_member ? &members : nullptr, {}};
    if (!dispatch(o, job)) {
      g_error = "sgbh_align_batch: invalid factor kind";
      return 1;
    }
    for (size_t m = 0; m < n_members; m++)
      write_result(job.results[m], T_out16xB + 16 * m, scalars_out4xB + 4 * m, H_out36xB ? H_out36xB + 36 * m : nullptr, b_out6xB ? b_out6xB + 6 * m : nullptr);
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 2;
  }
}

/// BatchRegistration<...>::align over (target, source) pairs: the options of sgbh_align (tree 1 = TREE_DEVICE_KDTREE: a kd-tree per
/// target; otherwise a Gaussian voxel map per target with voxel_resolution and search offsets); target t = rows target_offsets[t] ..
/// target_offsets[t+1] (with normals / covariances or none), source s likewise.  pairs2 NULL: n_targets = n_sources = n_pairs, source m
/// against target m; else pair p = (source pairs2[2p], target pairs2[2p+1]) (the pair-list overloads).  One initial pose per pair;
/// outputs as sgbh_align_batch's.
int sgbh_align_batch_pairs(size_t n_pairs, const size_t* target_offsets, const double* target_pts4, const double* target_normals4, const double* target_covs16,
                           const size_t* source_offsets,
                           const double* source_pts4, const double* source_covs16, const double* options21, const double* init_T16xB, double* T_out16xB,
                           double* scalars_out4xB, double* H_out36xB, double* b_out6xB, size_t n_targets, size_t n_sources, const size_t* pairs2) {
  try {
    const Options o = parse_options(options21);
    if (!pairs2) n_targets = n_sources = n_pairs;
    std::vector<PointCloud> targets(n_targets), sources(n_sources);
    for (size_t t = 0; t < n_targets; t++) {
      const size_t to = target_offsets[t], tn = target_offsets[t + 1] - to;
      targets[t] = *make_cloud(tn, target_pts4 + 4 * to, target_normals4 ? target_normals4 + 4 * to : nullptr, target_covs16 ? target_covs16 + 16 * to : nullptr);
    }
    for (size_t m = 0; m < n_sources; m++) {
      const size_t so = source_offsets[m], sn = source_offsets[m + 1] - so;
      sources[m] = *make_cloud(sn, source_pts4 + 4 * so, nullptr, source_covs16 ? source_covs16 + 16 * so : nullptr);
    }
    std::vector<Isometry3d> init(n_pairs);
    std::vector<std::pair<size_t, size_t>> pairs(pairs2 ? n_pairs : 0);
    for (size_t p = 0; p < n_pairs; p++) {
      std::memcpy(init[p].matrix().data(), init_T16xB + 16 * p, sizeof(double) * 16);
      if (pairs2) pairs[p] = {pairs2[2 * p], pairs2[2 * p + 1]};
    }
    PairsJob job{o, targets, sources, init, pairs2 ? &pairs : nullptr, {}};
    if (!dispatch(o, job)) {
      g_error = "sgbh_align_batch_pairs: invalid factor kind";
      return 1;
    }
    for (size_t m = 0; m < n_pairs; m++)
      write_result(job.results[m], T_out16xB + 16 * m, scalars_out4xB + 4 * m, H_out36xB ? H_out36xB + 36 * m : nullptr, b_out6xB ? b_out6xB + 6 * m : nullptr);
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 2;
  }
}

/// BatchRegistration<...>::align over submaps: the options of sgbh_align; map t = rows map_offsets[t] .. map_offsets[t+1] (covariances
/// or none), source s likewise; member p = source cloud_of_member[p] against the entries list_off[p] .. list_off[p+1] - 1, entry j = map
/// entry_maps[j] at the column-major pose entry_poses16[16 j ..].  One initial pose per member; outputs as sgbh_align_batch's.
int sgbh_align_batch_submaps(size_t n_members, size_t n_maps, const size_t* map_offsets, const double* map_pts4, const double* map_covs16, size_t n_sources,
                             const size_t* source_offsets, const double* source_pts4, const double* source_covs16, const size_t* cloud_of_member,
                             const size_t* list_off, const size_t* entry_maps, const double* entry_poses16, const double* options21, const double* init_T16xB,
                             double* T_out16xB, double* scalars_out4xB, double* H_out36xB, double* b_out6xB) {
  try {
    const Options o = parse_options(options21);
    std::vector<PointCloud> maps(n_maps), sources(n_sources);
    for (size_t t = 0; t < n_maps; t++) {
      const size_t to = map_offsets[t], tn = map_offsets[t + 1] - to;
      maps[t] = *make_cloud(tn, map_pts4 + 4 * to, nullptr, map_covs16 ? map_covs16 + 16 * to : nullptr);
    }
    for (size_t m = 0; m < n_sources; m++) {
      const size_t so = source_offsets[m], sn = source_offsets[m + 1] - so;
      sources[m] = *make_cloud(sn, source_pts4 + 4 * so, nullptr, source_covs16 ? source_covs16 + 16 * so : nullptr);
    }
    std::vector<Isometry3d> init(n_members);
    std::vector<size_t> clouds(cloud_of_member, cloud_of_member + n_members);
    std::vector<std::vector<std::pair<size_t, Isometry3d>>> submaps(n_members);
    for (size_t p = 0; p < n_members; p++) {
      std::memcpy(init[p].matrix().data(), init_T16xB + 16 * p, sizeof(double) * 16);
      for (size_t j = list_off[p]; j < list_off[p + 1]; j++) {
        Isometry3d P;
        std::memcpy(P.matrix().data(), entry_poses16 + 16 * j, sizeof(double) * 16);
        submaps[p].emplace_back(entry_maps[j], P);
      }
    }
    SubmapsJob job{o, maps, sources, clouds, submaps, init, {}};
    if (!dispatch(o, job)) {
      g_error = "sgbh_align_batch_submaps: invalid factor kind";
      return 1;
    }
    for (size_t m = 0; m < n_members; m++)
      write_result(job.results[m], T_out16xB + 16 * m, scalars_out4xB + 4 * m, H_out36xB ? H_out36xB + 36 * m : nullptr, b_out6xB ? b_out6xB + 6 * m : nullptr);
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 2;
  }
}

/// small_gicp::align(target_points, source_points, init_T, setting) of the helper API (registration_helper.cpp:58-69):
/// raw points in; settings8 = [type, voxel_resolution, downsampling_resolution, max_correspondence_distance, rotation_eps,
/// translation_eps, max_iterations, device].  sizes_out2 = down-sampled target / source sizes (informational).
int sgbh_helper_align(size_t n_target, const double* target_pts4, size_t n_source, const double* source_pts4, const double* settings8, const double* init_T16,
                      double* T_out16, double* scalars_out4, double* sizes_out2) {
  try {
    RegistrationSetting s;
    s.type = static_cast<RegistrationSetting::RegistrationType>(static_cast<int>(settings8[0]));
    s.voxel_resolution = settings8[1];
    s.downsampling_resolution = settings8[2];
    s.max_correspondence_distance = settings8[3];
    s.rotation_eps = settings8[4];
    s.translation_eps = settings8[5];
    s.max_iterations = static_cast<int>(settings8[6]);
    s.device = static_cast<int>(settings8[7]);
    auto target = make_cloud(n_target, target_pts4, nullptr, nullptr);
    auto source = make_cloud(n_source, source_pts4, nullptr, nullptr);
    Isometry3d init;
    std::memcpy(init.matrix().data(), init_T16, sizeof(double) * 16);
    auto [tp, tt] = preprocess_points(*target, s.downsampling_resolution, 10, s.num_threads, s.device);
    auto [sp, st] = preprocess_points(*source, s.downsampling_resolution, 10, s.num_threads, s.device);
    RegistrationResult r;
    if (s.type == RegistrationSetting::VGICP) {
      auto vm = create_gaussian_voxelmap(*tp, s.voxel_resolution);
      r = align(*vm, *sp, init, s);
    } else {
      r = align(*tp, *sp, *tt, init, s);
    }
    std::memcpy(T_out16, r.T_target_source.matrix().data(), sizeof(double) * 16);
    scalars_out4[0] = r.converged ? 1.0 : 0.0;
    scalars_out4[1] = static_cast<double>(r.iterations);
    scalars_out4[2] = static_cast<double>(r.num_inliers);
    scalars_out4[3] = r.error;
    if (sizes_out2) {
      sizes_out2[0] = static_cast<double>(tp->size());
      sizes_out2[1] = static_cast<double>(sp->size());
    }
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 2;
  }
}

/// preprocess_points(cloud, resolution, num_neighbors).first of every cloud (batch = 0), or preprocess_points_batch(clouds, ...)
/// (batch = 1): cloud c = rows offsets[c] .. offsets[c+1].  Outputs concatenated (each buffer holds offsets[n_clouds] rows); out_offsets:
/// n_clouds + 1 entries.
int sgbh_preprocess_points(size_t n_clouds, const size_t* offsets, const double* pts4, double downsampling_resolution, int num_neighbors, int device, int batch,
                           double* out_pts4, double* out_normals4, double* out_covs16, size_t* out_offsets) {
  try {
    std::vector<PointCloud> clouds(n_clouds);
    for (size_t c = 0; c < n_clouds; c++) clouds[c] = *make_cloud(offsets[c + 1] - offsets[c], pts4 + 4 * offsets[c], nullptr, nullptr);
    std::vector<PointCloud::Ptr> out;
    if (batch) {
      out = preprocess_points_batch(clouds, downsampling_resolution, num_neighbors, device);
    } else {
      for (const auto& c : clouds) out.push_back(preprocess_points(c, downsampling_resolution, num_neighbors, 4, device).first);
    }
    out_offsets[0] = 0;
    for (size_t c = 0; c < n_clouds; c++) {
      const PointCloud& o = *out[c];
      const size_t first = out_offsets[c], m = o.size();
      if (m) {
        std::memcpy(out_pts4 + 4 * first, o.points[0].data(), m * sizeof(Vector4d));
        std::memcpy(out_normals4 + 4 * first, o.normals[0].data(), m * sizeof(Vector4d));
        std::memcpy(out_covs16 + 16 * first, o.covs[0].data(), m * sizeof(Matrix4d));
      }
      out_offsets[c + 1] = first + m;
    }
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 2;
  }
}

/// Host KdTree<PointCloud>::knn_search over a batch of queries (API-surface check of the mirror, CPU-only).
int sgbh_kdtree_knn(size_t n, const double* pts4, size_t nq, const double* queries4, int k, uint64_t* idx_out, double* d2_out) {
  try {
    auto cloud = make_cloud(n, pts4, nullptr, nullptr);
    KdTree<PointCloud> tree(cloud);
    std::vector<size_t> ki(k);
    for (size_t i = 0; i < nq; i++) {
      Vector4d q;
      std::memcpy(q.data(), queries4 + i * 4, sizeof(double) * 4);
      tree.knn_search(q, k, ki.data(), d2_out + i * k);
      for (int j = 0; j < k; j++) idx_out[i * k + j] = ki[j];
    }
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 2;
  }
}

/// read_ply / read_points of the host mirror (read_points.hpp): fills at most `capacity` points (x, y, z, 1 as floats), returns the
/// number of points in the file through n_out (API-surface check of the mirror, CPU-only).  kind: 0 = PLY, 1 = KITTI .bin.
int sgbh_read_points(const char* filename, int kind, size_t capacity, float* out_xyz1, size_t* n_out) {
  try {
    const std::vector<Vector4f> pts = kind == 0 ? read_ply(filename) : read_points(filename);
    *n_out = pts.size();
    const size_t m = pts.size() < capacity ? pts.size() : capacity;
    if (m) std::memcpy(out_xyz1, pts.data(), m * sizeof(Vector4f));
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 2;
  }
}

/// write_points of the host mirror.
int sgbh_write_points(const char* filename, size_t n, const float* xyz1) {
  try {
    std::vector<Vector4f> pts(n);
    if (n) std::memcpy(pts.data(), xyz1, n * sizeof(Vector4f));
    write_points(filename, pts);
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 2;
  }
}

}  // extern "C"
