// SPDX-License-Identifier: MIT
// The reference's concurrent pattern on the C++ mirror: several Registration<GICPFactor, ParallelReductionCUDA>::align() calls at once
// on std::threads (as its TBB flow-graph odometry runs them), each on its own source and initial pose against one shared target cloud,
// one device context per Registration.  The four results must be bit-identical to the same four aligns run one after another:
// T_target_source, converged, iterations, num_inliers and error.
//
// Exit code 0: all equal; 1: a result differs (printed); 2: a call failed (its message printed).
#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include <small_gicp_b200/core.hpp>
#include <small_gicp_b200/factors.hpp>
#include <small_gicp_b200/kdtree.hpp>
#include <small_gicp_b200/reduction_cuda.hpp>
#include <small_gicp_b200/registration.hpp>
#include <small_gicp_b200/registration_helper.hpp>

using namespace small_gicp_b200;

namespace {

constexpr int kJobs = 4;

/// a fixed 64-bit LCG: the same clouds on every platform and standard library
struct Lcg {
  uint64_t s;
  double uniform() {
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    return static_cast<double>(s >> 11) * (1.0 / 9007199254740992.0);
  }
};

/// a room corner: a floor and two walls, 12 x 10 x 3 m, sampled with 2 cm of noise across each surface
PointCloud::Ptr make_room(size_t n, uint64_t seed) {
  Lcg g{seed};
  auto cloud = std::make_shared<PointCloud>();
  cloud->resize(n);
  for (size_t i = 0; i < n; i++) {
    const double u = g.uniform(), v = g.uniform(), w = (g.uniform() - 0.5) * 0.04;
    Vector4d p;
    switch (i % 3) {
      case 0: p = vec4(12.0 * u, 10.0 * v, w, 1.0); break;  // floor
      case 1: p = vec4(12.0 * u, w, 3.0 * v, 1.0); break;   // wall y = 0
      default: p = vec4(w, 10.0 * u, 3.0 * v, 1.0); break;  // wall x = 0
    }
    cloud->points[i] = p;
  }
  return cloud;
}

Isometry3d pose(double rx, double ry, double rz, double tx, double ty, double tz) {
  Vector6d a;
  a[0] = rx, a[1] = ry, a[2] = rz, a[3] = tx, a[4] = ty, a[5] = tz;
  return se3_exp(a);
}

/// job j's source: every (j + 2)-th target point moved into a sensor frame by the inverse of a ground-truth pose
PointCloud::Ptr make_source(const PointCloud& target, const Isometry3d& truth, int j) {
  const Isometry3d inv = truth.inverse();
  auto src = std::make_shared<PointCloud>();
  for (size_t i = static_cast<size_t>(j); i < target.size(); i += static_cast<size_t>(j + 2)) src->points.push_back(inv * target.points[i]);
  src->resize(src->points.size());
  return src;
}

struct Job {
  PointCloud::Ptr source;
  Isometry3d init;
};

struct Outcome {
  RegistrationResult result;
  std::string error;
};

Outcome run(const PointCloud::Ptr& target, const KdTree<PointCloud>& tree, const Job& job) {
  Outcome o;
  try {
    Registration<GICPFactor, ParallelReductionCUDA> reg;
    reg.rejector.max_dist_sq = 1.0;
    o.result = reg.align(*target, *job.source, tree, job.init);
  } catch (const std::exception& e) {
    o.error = e.what();
  }
  return o;
}

bool same_bits(const void* a, const void* b, size_t n) { return std::memcmp(a, b, n) == 0; }

}  // namespace

int main() {
  const PointCloud::Ptr target = make_room(60000, 1);
  std::vector<Job> jobs(kJobs);
  try {
    estimate_covariances(*target, 20);
    for (int j = 0; j < kJobs; j++) {
      const Isometry3d truth = pose(0.01 * j, -0.02, 0.015 * (j - 1), 0.2 + 0.1 * j, -0.15, 0.05 * j);
      jobs[j].source = make_source(*target, truth, j);
      estimate_covariances(*jobs[j].source, 20);
      jobs[j].init = truth * pose(0.02, -0.01 * j, 0.01, -0.1, 0.05 * j, 0.08);  // each job misaligned its own way
    }
  } catch (const std::exception& e) {
    std::printf("preparation failed: %s\n", e.what());
    return 2;
  }
  const KdTree<PointCloud> tree(target);

  std::vector<Outcome> serial(kJobs), concurrent(kJobs);
  for (int j = 0; j < kJobs; j++) serial[j] = run(target, tree, jobs[j]);

  std::atomic<int> waiting{kJobs};
  std::vector<std::thread> threads;
  for (int j = 0; j < kJobs; j++) {
    threads.emplace_back([&, j] {
      waiting.fetch_sub(1);
      while (waiting.load() > 0) std::this_thread::yield();  // released together
      concurrent[j] = run(target, tree, jobs[j]);
    });
  }
  for (auto& t : threads) t.join();

  int rc = 0;
  for (int j = 0; j < kJobs; j++) {
    for (const Outcome* o : {&serial[j], &concurrent[j]}) {
      if (!o->error.empty()) {
        std::printf("job %d (%s) failed: %s\n", j, o == &serial[j] ? "serial" : "concurrent", o->error.c_str());
        rc = 2;
      }
    }
    if (rc == 2) continue;
    const RegistrationResult &s = serial[j].result, &c = concurrent[j].result;
    const bool equal = same_bits(s.T_target_source.matrix().data(), c.T_target_source.matrix().data(), 16 * sizeof(double)) &&
                       s.converged == c.converged && s.iterations == c.iterations && s.num_inliers == c.num_inliers &&
                       same_bits(&s.error, &c.error, sizeof(double));
    std::printf("job %d: converged %d iterations %zu inliers %zu error %.17g %s\n", j, int(s.converged), s.iterations, s.num_inliers, s.error,
                equal ? "identical" : "DIFFERS");
    if (!equal) {
      std::printf("  concurrent: converged %d iterations %zu inliers %zu error %.17g\n", int(c.converged), c.iterations, c.num_inliers, c.error);
      if (rc == 0) rc = 1;
    }
  }
  return rc;
}
