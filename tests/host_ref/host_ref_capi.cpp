// SPDX-License-Identifier: MIT
// tests/host_ref: the REFERENCE's own Registration<> template (headers included in place from /root/reference/include, nothing
// copied) instantiated with include/small_gicp/registration/reduction_cuda.hpp -- the binding INTEGRATION.md shows -- next to
// the same template on the reference's ParallelReductionOMP, behind one C entry point for the Python tests.
// TEST INFRASTRUCTURE: built only where the reference's sources are at hand (tests/host_ref/Makefile), into oracle/_ref/.
// Eigen is absent from the image: both arms compile against the API shim of oracle/ref_build/eigen_shim (DESIGN.md §2).
#include <cstring>
#include <memory>
#include <string>

#include <small_gicp/ann/gaussian_voxelmap.hpp>
#include <small_gicp/ann/kdtree.hpp>
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

}  // extern "C"
