// SPDX-License-Identifier: MIT
// tests/host_ref: the REFERENCE's own Registration<> template (headers included in place from /root/reference/include, nothing
// copied) instantiated with include/small_gicp/registration/reduction_cuda.hpp -- the binding INTEGRATION.md shows -- next to
// the same template on the reference's ParallelReductionOMP, behind C entry points for the Python tests: href_align (the result of
// one align()) and href_align_log (every call the optimizer makes to the reduction, on any of the reference's search structures and
// on a cloud type of the harness' own; tests/np_dropin.py checks the log).
// TEST INFRASTRUCTURE: built only where the reference's sources are at hand (tests/host_ref/Makefile), into oracle/_ref/.
// Eigen is absent from the image: both arms compile against the API shim of oracle/ref_build/eigen_shim (DESIGN.md §2).
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include <small_gicp/ann/gaussian_voxelmap.hpp>
#include <small_gicp/ann/kdtree.hpp>
#include <small_gicp/ann/kdtree_omp.hpp>
#include <small_gicp/factors/gicp_factor.hpp>
#include <small_gicp/factors/icp_factor.hpp>
#include <small_gicp/factors/plane_icp_factor.hpp>
#include <small_gicp/factors/robust_kernel.hpp>
#include <small_gicp/points/point_cloud.hpp>
#include <small_gicp/registration/reduction_cuda.hpp>
#include <small_gicp/registration/reduction_omp.hpp>
#include <small_gicp/registration/registration.hpp>

using namespace small_gicp;

namespace {
thread_local std::string g_error;

struct Args {
  int backend;    // 0 = ParallelReductionOMP (the reference), 1 = ParallelReductionCUDA
  int factor;     // sgb_factor_kind
  int robust;     // sgb_robust_kind
  double robust_c;
  int rejector;   // sgb_rejector_kind
  double max_dist_sq;
  int optimizer;  // 0 = GaussNewton, 1 = LevenbergMarquardt
  int max_iterations;
  int num_threads;
  int vgicp;      // target = GaussianVoxelMap(voxel_resolution) built from the target cloud
  double voxel_resolution;
  int realign;    // > 0: after the first align() shift the SOURCE in place by (0.05, -0.03, 0.02) * realign and align again
                  // (same address, same size, new content: the mirror of a CUDA reduction must not be stale)
  int sync_every_linearize;
  unsigned long long generation;  // ParallelReductionCUDA::{target,source}_generation
};

template <typename R>
void set_common(R& reg, const Args& a) {
  reg.optimizer.max_iterations = a.max_iterations;
  reg.reduction.num_threads = a.num_threads;
}
template <typename Reg>
void set_rejector(Reg& reg, const Args& a, std::true_type) {
  reg.rejector.max_dist_sq = a.max_dist_sq;
}
template <typename Reg>
void set_rejector(Reg&, const Args&, std::false_type) {}
template <typename S>
void set_robust(S& s, const Args& a, std::true_type) {
  s.robust_kernel.c = a.robust_c;
}
template <typename S>
void set_robust(S&, const Args&, std::false_type) {}
inline void set_cuda(ParallelReductionCUDA& r, const Args& a) {
  r.sync_every_linearize = a.sync_every_linearize != 0;
  r.target_generation = r.source_generation = a.generation;
}
inline void set_cuda(ParallelReductionOMP&, const Args&) {}

template <typename Factor, typename Reduction, typename Rejector, typename Optimizer, bool kRobust>
RegistrationResult run(const Args& a, const std::shared_ptr<PointCloud>& target, const std::shared_ptr<PointCloud>& source, const Eigen::Isometry3d& init) {
  Registration<Factor, Reduction, NullFactor, Rejector, Optimizer> reg;
  set_common(reg, a);
  set_rejector(reg, a, std::is_same<Rejector, DistanceRejector>());
  set_robust(reg.point_factor, a, std::integral_constant<bool, kRobust>());
  set_cuda(reg.reduction, a);
  auto shift = [&](int k) {
    for (auto& p : source->points) {
      p[0] += 0.05 * k;
      p[1] -= 0.03 * k;
      p[2] += 0.02 * k;
    }
  };
  if (a.vgicp) {
    // the reference's voxel map has means and covariances only (gaussian_voxelmap.hpp:64-87): VGICP = the GICP factor on it
    if constexpr (!std::is_same_v<typename cuda_detail::unwrap<Factor>::base, GICPFactor>) {
      throw std::runtime_error("host_ref: a GaussianVoxelMap target takes the GICP factor");
    } else {
    GaussianVoxelMap map(a.voxel_resolution);
    map.insert(*target);
    RegistrationResult r = reg.align(map, *source, map, init);
    if (a.realign > 0) {
      shift(a.realign);
      r = reg.align(map, *source, map, init);
      shift(-a.realign);
    }
    return r;
    }
  }
  KdTree<PointCloud> tree(target);
  RegistrationResult r = reg.align(*target, *source, tree, init);
  if (a.realign > 0) {
    shift(a.realign);
    r = reg.align(*target, *source, tree, init);
    shift(-a.realign);
  }
  return r;
}

template <typename Factor, typename Reduction, typename Rejector, bool kRobust>
RegistrationResult by_optimizer(const Args& a, const std::shared_ptr<PointCloud>& t, const std::shared_ptr<PointCloud>& s, const Eigen::Isometry3d& init) {
  if (a.optimizer == 0) return run<Factor, Reduction, Rejector, GaussNewtonOptimizer, kRobust>(a, t, s, init);
  return run<Factor, Reduction, Rejector, LevenbergMarquardtOptimizer, kRobust>(a, t, s, init);
}
template <typename Factor, typename Reduction, bool kRobust>
RegistrationResult by_rejector(const Args& a, const std::shared_ptr<PointCloud>& t, const std::shared_ptr<PointCloud>& s, const Eigen::Isometry3d& init) {
  if (a.rejector == 0) return by_optimizer<Factor, Reduction, NullRejector, kRobust>(a, t, s, init);
  return by_optimizer<Factor, Reduction, DistanceRejector, kRobust>(a, t, s, init);
}
template <typename Base, typename Reduction>
RegistrationResult by_robust(const Args& a, const std::shared_ptr<PointCloud>& t, const std::shared_ptr<PointCloud>& s, const Eigen::Isometry3d& init) {
  if (a.robust == 1) return by_rejector<RobustFactor<Huber, Base>, Reduction, true>(a, t, s, init);
  if (a.robust == 2) return by_rejector<RobustFactor<Cauchy, Base>, Reduction, true>(a, t, s, init);
  return by_rejector<Base, Reduction, false>(a, t, s, init);
}
template <typename Reduction>
RegistrationResult by_factor(const Args& a, const std::shared_ptr<PointCloud>& t, const std::shared_ptr<PointCloud>& s, const Eigen::Isometry3d& init) {
  if (a.factor == 0) return by_robust<ICPFactor, Reduction>(a, t, s, init);
  if (a.factor == 1) return by_robust<PointToPlaneICPFactor, Reduction>(a, t, s, init);
  return by_robust<GICPFactor, Reduction>(a, t, s, init);
}

std::shared_ptr<PointCloud> make_cloud(size_t n, const double* pts4, const double* normals4, const double* covs16) {
  auto c = std::make_shared<PointCloud>();
  c->resize(n);
  if (n) std::memcpy(c->points[0].data(), pts4, n * 4 * sizeof(double));
  if (normals4 && n) std::memcpy(c->normals[0].data(), normals4, n * 4 * sizeof(double));
  if (covs16 && n) std::memcpy(c->covs[0].data(), covs16, n * 16 * sizeof(double));
  return c;
}

// ================================================================ call log (href_align_log)
// Every linearize() / error() the optimizer makes, as the Reduction returned it, and after every linearize() each factor's
// (source_index, target_index) -- what Factor::inlier() and user code read -- next to the correspondences the CUDA context holds
// (read into a copy of the factor vector, so that sync_every_linearize = false stays observable).
struct CallLog {
  std::vector<double> calls;          // per call: kind (0 linearize, 1 error) | align index | T (16, row-major) | H (36) | b (6) | e  = 61
  std::vector<std::uint64_t> idx;     // per linearize: source_index (n) | target_index (n) | device correspondences (n)
  std::vector<double> aligns;         // per align(): structure | T (16, row-major) | iterations | converged | num_inliers | error  = 21
  std::vector<std::int32_t> vox_coords;  // flat_voxels of the voxel map (if one was built): coordinates (3) | mean (4) | cov (16)
  std::vector<double> vox_means, vox_covs;
  int align_index = 0;
};
thread_local CallLog g_log;

void log_call(int kind, const Eigen::Isometry3d& T, const Eigen::Matrix<double, 6, 6>* H, const Eigen::Matrix<double, 6, 1>* b, double e) {
  auto& c = g_log.calls;
  c.push_back(kind);
  c.push_back(g_log.align_index);
  for (int r = 0; r < 4; r++)
    for (int k = 0; k < 4; k++) c.push_back(T.matrix()(r, k));
  for (int r = 0; r < 6; r++)
    for (int k = 0; k < 6; k++) c.push_back(H ? (*H)(r, k) : 0.0);
  for (int r = 0; r < 6; r++) c.push_back(b ? (*b)(r) : 0.0);
  c.push_back(e);
}

/// A Reduction that forwards to `inner` (ParallelReductionCUDA or ParallelReductionOMP) and logs every call.
template <typename Inner>
struct Recording {
  Inner inner;

  template <typename TargetPointCloud, typename SourcePointCloud, typename TargetTree, typename CorrespondenceRejector, typename Factor>
  std::tuple<Eigen::Matrix<double, 6, 6>, Eigen::Matrix<double, 6, 1>, double> linearize(const TargetPointCloud& target, const SourcePointCloud& source,
                                                                                         const TargetTree& tree, const CorrespondenceRejector& rejector,
                                                                                         const Eigen::Isometry3d& T, std::vector<Factor>& factors) const {
    auto r = inner.linearize(target, source, tree, rejector, T, factors);
    log_call(0, T, &std::get<0>(r), &std::get<1>(r), std::get<2>(r));
    using U = cuda_detail::unwrap<Factor>;
    for (auto& f : factors) g_log.idx.push_back(U::state(f).source_index);
    for (auto& f : factors) g_log.idx.push_back(U::state(f).target_index);
    if constexpr (std::is_same_v<Inner, ParallelReductionCUDA>) {
      std::vector<Factor> copy(factors);
      inner.sync_factors(copy);
      for (auto& f : copy) g_log.idx.push_back(U::state(f).target_index);
    } else {
      for (auto& f : factors) g_log.idx.push_back(U::state(f).target_index);
    }
    return r;
  }

  template <typename TargetPointCloud, typename SourcePointCloud, typename Factor>
  double error(const TargetPointCloud& target, const SourcePointCloud& source, const Eigen::Isometry3d& T, std::vector<Factor>& factors) const {
    const double e = inner.error(target, source, T, factors);
    log_call(1, T, nullptr, nullptr, e);
    return e;
  }
};

/// A cloud type of the harness' own, reached only through small_gicp::traits: an array of structs with FP32 fields (as in a PCL
/// point type), so that the drop-in must gather it (CloudArrays) and what it gathers differs from the FP64 input.
struct F32Point {
  float xyz[3];
  float normal[3];
  float cov[6];  // upper triangle (0,0) (0,1) (0,2) (1,1) (1,2) (2,2)
};
struct F32Cloud {
  std::vector<F32Point> pts;
  bool normals = false, covs = false;
};
}  // namespace

namespace small_gicp::traits {
template <>
struct Traits<F32Cloud> {
  static size_t size(const F32Cloud& c) { return c.pts.size(); }
  static bool has_points(const F32Cloud& c) { return !c.pts.empty(); }
  static bool has_normals(const F32Cloud& c) { return c.normals; }
  static bool has_covs(const F32Cloud& c) { return c.covs; }
  static Eigen::Vector4d point(const F32Cloud& c, size_t i) {
    const float* p = c.pts[i].xyz;
    return Eigen::Vector4d(p[0], p[1], p[2], 1.0);
  }
  static Eigen::Vector4d normal(const F32Cloud& c, size_t i) {
    const float* n = c.pts[i].normal;
    return Eigen::Vector4d(n[0], n[1], n[2], 0.0);
  }
  static Eigen::Matrix4d cov(const F32Cloud& c, size_t i) {
    const float* u = c.pts[i].cov;
    Eigen::Matrix4d m = Eigen::Matrix4d::Zero();
    m(0, 0) = u[0];
    m(0, 1) = m(1, 0) = u[1];
    m(0, 2) = m(2, 0) = u[2];
    m(1, 1) = u[3];
    m(1, 2) = m(2, 1) = u[4];
    m(2, 2) = u[5];
    return m;
  }
};
}  // namespace small_gicp::traits

namespace {
template <typename Cloud>
std::shared_ptr<Cloud> make_typed(size_t n, const double* p4, const double* n4, const double* c16) {
  if constexpr (std::is_same_v<Cloud, PointCloud>) {
    return make_cloud(n, p4, n4, c16);
  } else {
    auto c = std::make_shared<F32Cloud>();
    c->pts.resize(n);
    c->normals = n4 != nullptr;
    c->covs = c16 != nullptr;
    static const int tri[6][2] = {{0, 0}, {0, 1}, {0, 2}, {1, 1}, {1, 2}, {2, 2}};
    for (size_t i = 0; i < n; i++) {
      for (int a = 0; a < 3; a++) {
        c->pts[i].xyz[a] = static_cast<float>(p4[i * 4 + a]);
        c->pts[i].normal[a] = n4 ? static_cast<float>(n4[i * 4 + a]) : 0.f;
      }
      for (int k = 0; k < 6; k++) c->pts[i].cov[k] = c16 ? static_cast<float>(c16[i * 16 + tri[k][0] * 4 + tri[k][1]]) : 0.f;  // row-major 4x4
    }
    return c;
  }
}

/// KdTreeBuilder and KdTreeBuilderOMP size the node array to the point count (ann/kdtree.hpp:85, kdtree_omp.hpp:29); with
/// max_leaf_size 1 or 2 a tree has more nodes than points and they write past it.  For those leaf sizes the harness builds with the
/// same create_node into an array of 2n nodes (the most any leaf size makes).
struct RoomyKdTreeBuilder : KdTreeBuilder {
  template <typename Tree, typename Cloud>
  void build_tree(Tree& tree, const Cloud& points) const {
    const size_t n = traits::size(points);
    tree.indices.resize(n);
    for (size_t i = 0; i < n; i++) tree.indices[i] = i;
    tree.nodes.resize(2 * n);
    size_t used = 0;
    tree.root = create_node(tree, used, points, tree.indices.begin(), tree.indices.begin(), tree.indices.end());
    tree.nodes.resize(used);
  }
};

// structure ids of href_align_log
enum { S_KDTREE = 0, S_UNSAFE = 1, S_KDTREE_OMP = 2, S_VOXELMAP = 3 };

struct LogArgs {
  Args a;
  int structure;      // S_*
  int max_leaf_size;  // kd-tree builders
  int offsets;        // voxel map search_offsets
  int lru_horizon, lru_clear_cycle;
  int cloud_type;     // 0 = PointCloud, 1 = F32Cloud
  int scenario;       // 0 = one align(); 1 = one Registration: kd-tree, voxel map, kd-tree; 2 = two Registrations on one context, kd / map / kd / map
};

template <typename Cloud>
struct Targets {
  std::shared_ptr<Cloud> cloud;
  std::unique_ptr<KdTree<Cloud>> kd;
  std::unique_ptr<UnsafeKdTree<Cloud>> unsafe;
  std::unique_ptr<GaussianVoxelMap> map;
  int tree_kind = S_KDTREE;
};

template <typename Cloud>
void build_targets(Targets<Cloud>& t, const LogArgs& la, bool want_tree, bool want_map, size_t n_inserts, const double* insert_poses16) {
  const int leaf = la.max_leaf_size;
  if (want_tree) {
    t.tree_kind = la.structure == S_VOXELMAP ? S_KDTREE : la.structure;
    if (t.tree_kind == S_KDTREE_OMP) {
      KdTreeBuilderOMP b(4);
      b.max_leaf_size = leaf;
      if (leaf < 3) throw std::runtime_error("host_ref: KdTreeBuilderOMP needs max_leaf_size >= 3");
      t.kd = std::make_unique<KdTree<Cloud>>(t.cloud, b);
    } else if (t.tree_kind == S_UNSAFE) {
      if (leaf < 3) {
        RoomyKdTreeBuilder b;
        b.max_leaf_size = leaf;
        t.unsafe = std::make_unique<UnsafeKdTree<Cloud>>(*t.cloud, b);
      } else {
        KdTreeBuilder b;
        b.max_leaf_size = leaf;
        t.unsafe = std::make_unique<UnsafeKdTree<Cloud>>(*t.cloud, b);
      }
    } else if (leaf < 3) {
      RoomyKdTreeBuilder b;
      b.max_leaf_size = leaf;
      t.kd = std::make_unique<KdTree<Cloud>>(t.cloud, b);
    } else {
      KdTreeBuilder b;
      b.max_leaf_size = leaf;
      t.kd = std::make_unique<KdTree<Cloud>>(t.cloud, b);
    }
  }
  if (want_map) {
    // the target cloud in n_inserts consecutive chunks, chunk k inserted at pose k: with a small lru_horizon / lru_clear_cycle the
    // voxels only early chunks touched are evicted (incremental_voxelmap.hpp:74-86)
    t.map = std::make_unique<GaussianVoxelMap>(la.a.voxel_resolution);
    t.map->set_search_offsets(la.offsets);
    t.map->lru_horizon = static_cast<size_t>(la.lru_horizon);
    t.map->lru_clear_cycle = static_cast<size_t>(la.lru_clear_cycle);
    const size_t n = traits::size(*t.cloud), k = std::max<size_t>(1, n_inserts);
    for (size_t c = 0; c < k; c++) {
      Cloud chunk;
      const size_t lo = n * c / k, hi = n * (c + 1) / k;
      if constexpr (std::is_same_v<Cloud, PointCloud>) {
        chunk.resize(hi - lo);
        for (size_t i = lo; i < hi; i++) {
          chunk.points[i - lo] = t.cloud->points[i];
          chunk.covs[i - lo] = t.cloud->covs[i];
        }
      } else {
        chunk.pts.assign(t.cloud->pts.begin() + lo, t.cloud->pts.begin() + hi);
        chunk.covs = true;
      }
      Eigen::Isometry3d pose = Eigen::Isometry3d::Identity();
      if (insert_poses16)
        for (int r = 0; r < 4; r++)
          for (int q = 0; q < 4; q++) pose.matrix()(r, q) = insert_poses16[c * 16 + r * 4 + q];
      t.map->insert(chunk, pose);
    }
    const size_t m = t.map->size();
    g_log.vox_coords.resize(m * 3);
    g_log.vox_means.resize(m * 4);
    g_log.vox_covs.resize(m * 16);
    for (size_t i = 0; i < m; i++) {
      const auto& v = *t.map->flat_voxels[i];
      for (int a = 0; a < 3; a++) g_log.vox_coords[i * 3 + a] = v.first.coord[a];
      for (int a = 0; a < 4; a++) g_log.vox_means[i * 4 + a] = v.second.mean[a];
      for (int r = 0; r < 4; r++)
        for (int q = 0; q < 4; q++) g_log.vox_covs[i * 16 + r * 4 + q] = v.second.cov(r, q);
    }
  }
}

template <bool kGicp, typename Reg, typename Cloud>
void log_align(const Reg& reg, Targets<Cloud>& t, bool on_map, const Cloud& source, const Eigen::Isometry3d& init) {
  RegistrationResult r;
  int structure;
  if (on_map) {
    // the reference's voxel map has means and covariances only (gaussian_voxelmap.hpp:64-87): VGICP = the GICP factor on it
    if constexpr (kGicp) {
      r = reg.align(*t.map, source, *t.map, init);
    } else {
      throw std::runtime_error("host_ref: a GaussianVoxelMap target takes the GICP factor");
    }
    structure = S_VOXELMAP;
  } else if (t.tree_kind == S_UNSAFE) {
    r = reg.align(*t.cloud, source, *t.unsafe, init);
    structure = S_UNSAFE;
  } else {
    r = reg.align(*t.cloud, source, *t.kd, init);
    structure = t.tree_kind;
  }
  auto& o = g_log.aligns;
  o.push_back(structure);
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) o.push_back(r.T_target_source.matrix()(i, j));
  o.push_back(r.iterations);
  o.push_back(r.converged ? 1.0 : 0.0);
  o.push_back(static_cast<double>(r.num_inliers));
  o.push_back(r.error);
  g_log.align_index++;
}

/// Borrowed context of scenario 2 (ParallelReductionCUDA::use_context); nothing for the OMP arm.
struct SharedContext {
  sgb_ctx* ctx = nullptr;
  void attach(ParallelReductionCUDA& r) {
    if (!ctx && sgb_create(r.device, &ctx) != 0) throw std::runtime_error(std::string("host_ref: ") + sgb_last_error(nullptr));
    r.use_context(ctx);
  }
  void attach(ParallelReductionOMP&) {}
  ~SharedContext() {
    if (ctx) sgb_destroy(ctx);
  }
};

template <typename Factor, typename Inner, typename Rejector, typename Optimizer, bool kRobust, typename Cloud>
void run_log(const LogArgs& la, const double* const* arrays, size_t n_tgt, size_t n_src, const Eigen::Isometry3d& init, size_t n_inserts,
             const double* insert_poses16) {
  constexpr bool kGicp = std::is_same_v<typename cuda_detail::unwrap<Factor>::base, GICPFactor>;
  const Args& a = la.a;
  using Reg = Registration<Factor, Recording<Inner>, NullFactor, Rejector, Optimizer>;
  auto setup = [&](Reg& reg) {
    reg.optimizer.max_iterations = a.max_iterations;
    reg.reduction.inner.num_threads = a.num_threads;
    set_rejector(reg, a, std::is_same<Rejector, DistanceRejector>());
    set_robust(reg.point_factor, a, std::integral_constant<bool, kRobust>());
    set_cuda(reg.reduction.inner, a);
  };
  Targets<Cloud> t;
  t.cloud = make_typed<Cloud>(n_tgt, arrays[0], arrays[1], arrays[2]);
  const auto source = make_typed<Cloud>(n_src, arrays[3], nullptr, arrays[4]);
  const bool single_map = la.scenario == 0 && la.structure == S_VOXELMAP;
  build_targets(t, la, !single_map, la.scenario != 0 || single_map, n_inserts, insert_poses16);
  Reg reg;
  setup(reg);
  if (la.scenario == 0) {
    log_align<kGicp>(reg, t, single_map, *source, init);
  } else if (la.scenario == 1) {  // one reduction, one mirror: kd-tree, voxel map, kd-tree
    log_align<kGicp>(reg, t, false, *source, init);
    log_align<kGicp>(reg, t, true, *source, init);
    log_align<kGicp>(reg, t, false, *source, init);
  } else {  // two Registrations sharing one context: each its own mirror of the same device state
    Reg other;
    setup(other);
    SharedContext shared;
    shared.attach(reg.reduction.inner);
    shared.attach(other.reduction.inner);
    log_align<kGicp>(reg, t, false, *source, init);
    log_align<kGicp>(other, t, true, *source, init);
    log_align<kGicp>(reg, t, false, *source, init);
    log_align<kGicp>(other, t, true, *source, init);
  }
}

template <typename Factor, typename Inner, typename Rejector, typename Optimizer, bool kRobust>
void log_by_cloud(const LogArgs& la, const double* const* arrays, size_t nt, size_t ns, const Eigen::Isometry3d& init, size_t ni, const double* ip) {
  if (la.cloud_type == 1) return run_log<Factor, Inner, Rejector, Optimizer, kRobust, F32Cloud>(la, arrays, nt, ns, init, ni, ip);
  run_log<Factor, Inner, Rejector, Optimizer, kRobust, PointCloud>(la, arrays, nt, ns, init, ni, ip);
}
template <typename Factor, typename Inner, typename Rejector, bool kRobust>
void log_by_optimizer(const LogArgs& la, const double* const* arrays, size_t nt, size_t ns, const Eigen::Isometry3d& init, size_t ni, const double* ip) {
  if (la.a.optimizer == 0) return log_by_cloud<Factor, Inner, Rejector, GaussNewtonOptimizer, kRobust>(la, arrays, nt, ns, init, ni, ip);
  log_by_cloud<Factor, Inner, Rejector, LevenbergMarquardtOptimizer, kRobust>(la, arrays, nt, ns, init, ni, ip);
}
template <typename Factor, typename Inner, bool kRobust>
void log_by_rejector(const LogArgs& la, const double* const* arrays, size_t nt, size_t ns, const Eigen::Isometry3d& init, size_t ni, const double* ip) {
  if (la.a.rejector == 0) return log_by_optimizer<Factor, Inner, NullRejector, kRobust>(la, arrays, nt, ns, init, ni, ip);
  log_by_optimizer<Factor, Inner, DistanceRejector, kRobust>(la, arrays, nt, ns, init, ni, ip);
}
template <typename Base, typename Inner>
void log_by_robust(const LogArgs& la, const double* const* arrays, size_t nt, size_t ns, const Eigen::Isometry3d& init, size_t ni, const double* ip) {
  if (la.a.robust == 1) return log_by_rejector<RobustFactor<Huber, Base>, Inner, true>(la, arrays, nt, ns, init, ni, ip);
  if (la.a.robust == 2) return log_by_rejector<RobustFactor<Cauchy, Base>, Inner, true>(la, arrays, nt, ns, init, ni, ip);
  log_by_rejector<Base, Inner, false>(la, arrays, nt, ns, init, ni, ip);
}
template <typename Inner>
void log_by_factor(const LogArgs& la, const double* const* arrays, size_t nt, size_t ns, const Eigen::Isometry3d& init, size_t ni, const double* ip) {
  if (la.a.factor == 0) return log_by_robust<ICPFactor, Inner>(la, arrays, nt, ns, init, ni, ip);
  if (la.a.factor == 1) return log_by_robust<PointToPlaneICPFactor, Inner>(la, arrays, nt, ns, init, ni, ip);
  log_by_robust<GICPFactor, Inner>(la, arrays, nt, ns, init, ni, ip);
}
}  // namespace


extern "C" {

const char* href_last_error() { return g_error.c_str(); }

// args: 14 numbers in the order of struct Args (doubles; integers are rounded).  out: T (16, row-major) | iterations | converged |
// num_inliers | error | H (36) | b (6)  = 62 doubles.
int href_align(const double* args14, size_t n_tgt, const double* tgt_pts4, const double* tgt_normals4, const double* tgt_covs16, size_t n_src,
               const double* src_pts4, const double* src_covs16, const double* init_T_rowmajor16, double* out62) {
  try {
    Args a;
    a.backend = static_cast<int>(args14[0]);
    a.factor = static_cast<int>(args14[1]);
    a.robust = static_cast<int>(args14[2]);
    a.robust_c = args14[3];
    a.rejector = static_cast<int>(args14[4]);
    a.max_dist_sq = args14[5];
    a.optimizer = static_cast<int>(args14[6]);
    a.max_iterations = static_cast<int>(args14[7]);
    a.num_threads = static_cast<int>(args14[8]);
    a.vgicp = static_cast<int>(args14[9]);
    a.voxel_resolution = args14[10];
    a.realign = static_cast<int>(args14[11]);
    a.sync_every_linearize = static_cast<int>(args14[12]);
    a.generation = static_cast<unsigned long long>(args14[13]);
    auto target = make_cloud(n_tgt, tgt_pts4, tgt_normals4, tgt_covs16);
    auto source = make_cloud(n_src, src_pts4, nullptr, src_covs16);
    Eigen::Isometry3d init;
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) init.matrix()(r, c) = init_T_rowmajor16[r * 4 + c];
    const RegistrationResult res = a.backend == 0 ? by_factor<ParallelReductionOMP>(a, target, source, init) : by_factor<ParallelReductionCUDA>(a, target, source, init);
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) out62[r * 4 + c] = res.T_target_source.matrix()(r, c);
    out62[16] = static_cast<double>(res.iterations);
    out62[17] = res.converged ? 1.0 : 0.0;
    out62[18] = static_cast<double>(res.num_inliers);
    out62[19] = res.error;
    for (int r = 0; r < 6; r++) {
      for (int c = 0; c < 6; c++) out62[20 + r * 6 + c] = res.H(r, c);
      out62[56 + r] = res.b(r);
    }
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 1;
  }
}

// The call log of one run (see CallLog).  args: 21 numbers -- backend, factor, robust, robust_c, rejector, max_dist_sq, optimizer,
// max_iterations, num_threads, structure (0 KdTree, 1 UnsafeKdTree, 2 KdTree built by KdTreeBuilderOMP, 3 GaussianVoxelMap),
// max_leaf_size, voxel_resolution, search_offsets, lru_horizon, lru_clear_cycle, cloud type (0 PointCloud, 1 the harness' FP32
// struct), sync_every_linearize, generation, scenario (0 one align(); 1 one Registration: kd-tree, voxel map, kd-tree; 2 two
// Registrations sharing one context through use_context(): kd-tree, voxel map, kd-tree, voxel map), n_inserts (voxel map built from
// the target in that many chunks, chunk k inserted at insert_poses16[k], row-major), unused.  Read the log with href_log_sizes /
// href_log_copy.
int href_align_log(const double* args21, size_t n_tgt, const double* tgt_pts4, const double* tgt_normals4, const double* tgt_covs16, size_t n_src,
                   const double* src_pts4, const double* src_covs16, const double* init_T_rowmajor16, const double* insert_poses16) {
  try {
    g_log = CallLog();
    LogArgs la;
    Args& a = la.a;
    a.backend = static_cast<int>(args21[0]);
    a.factor = static_cast<int>(args21[1]);
    a.robust = static_cast<int>(args21[2]);
    a.robust_c = args21[3];
    a.rejector = static_cast<int>(args21[4]);
    a.max_dist_sq = args21[5];
    a.optimizer = static_cast<int>(args21[6]);
    a.max_iterations = static_cast<int>(args21[7]);
    a.num_threads = static_cast<int>(args21[8]);
    la.structure = static_cast<int>(args21[9]);
    la.max_leaf_size = static_cast<int>(args21[10]);
    a.voxel_resolution = args21[11];
    la.offsets = static_cast<int>(args21[12]);
    la.lru_horizon = static_cast<int>(args21[13]);
    la.lru_clear_cycle = static_cast<int>(args21[14]);
    la.cloud_type = static_cast<int>(args21[15]);
    a.sync_every_linearize = static_cast<int>(args21[16]);
    a.generation = static_cast<unsigned long long>(args21[17]);
    la.scenario = static_cast<int>(args21[18]);
    const size_t n_inserts = static_cast<size_t>(args21[19]);
    a.vgicp = 0;
    a.realign = 0;
    Eigen::Isometry3d init;
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) init.matrix()(r, c) = init_T_rowmajor16[r * 4 + c];
    const double* arrays[5] = {tgt_pts4, tgt_normals4, tgt_covs16, src_pts4, src_covs16};
    if (a.backend == 0)
      log_by_factor<ParallelReductionOMP>(la, arrays, n_tgt, n_src, init, n_inserts, insert_poses16);
    else
      log_by_factor<ParallelReductionCUDA>(la, arrays, n_tgt, n_src, init, n_inserts, insert_poses16);
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return 1;
  }
}

/// sizes[4]: doubles of the call records, uint64 of the factor indices, doubles of the align records, voxels of the map
void href_log_sizes(size_t* sizes4) {
  sizes4[0] = g_log.calls.size();
  sizes4[1] = g_log.idx.size();
  sizes4[2] = g_log.aligns.size();
  sizes4[3] = g_log.vox_coords.size() / 3;
}

void href_log_copy(double* calls, std::uint64_t* idx, double* aligns, std::int32_t* vox_coords3, double* vox_means4, double* vox_covs16) {
  std::copy(g_log.calls.begin(), g_log.calls.end(), calls);
  std::copy(g_log.idx.begin(), g_log.idx.end(), idx);
  std::copy(g_log.aligns.begin(), g_log.aligns.end(), aligns);
  std::copy(g_log.vox_coords.begin(), g_log.vox_coords.end(), vox_coords3);
  std::copy(g_log.vox_means.begin(), g_log.vox_means.end(), vox_means4);
  std::copy(g_log.vox_covs.begin(), g_log.vox_covs.end(), vox_covs16);
}

}  // extern "C"
