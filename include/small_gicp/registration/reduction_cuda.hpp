// SPDX-License-Identifier: MIT
// include/small_gicp/registration/reduction_cuda.hpp -- the ONE header a maintainer adds to koide3/small_gicp to get the H100
// backend (plus `target_link_libraries(... sgicp_b200)`).  It is written against the reference's own types and compiled,
// unmodified, by tests/host_ref/ against the reference's include/ directory (its headers in place) -- INTEGRATION.md shows
// this file, not a sketch of it.
//
// ParallelReductionCUDA is a peer of SerialReduction / ParallelReductionOMP / ParallelReductionTBB
// (small_gicp/registration/reduction.hpp:12-63, reduction_omp.hpp:20-73, reduction_tbb.hpp:114-139): the same two const member
// templates, plain public fields for tunables, default-constructible, copyable (copies share one device context).  Everything
// per point -- transform, nearest neighbour, rejection, factor, sum -- runs in libsgicp_b200.so through the C-ABI of
// <sgicp_b200.h>; this glue only mirrors clouds / search structures to the device and maps factor / rejector TYPES to kernel
// selectors.  An unsupported type is a compile error, never a CPU fallback.
#pragma once
#include <cstdint>
#include <cstring>
#include <iterator>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <tuple>
#include <type_traits>
#include <vector>

#include <Eigen/Core>
#include <Eigen/Geometry>
#include <sgicp_b200.h>
#include <small_gicp/ann/gaussian_voxelmap.hpp>
#include <small_gicp/ann/kdtree.hpp>
#include <small_gicp/factors/gicp_factor.hpp>
#include <small_gicp/factors/icp_factor.hpp>
#include <small_gicp/factors/plane_icp_factor.hpp>
#include <small_gicp/factors/robust_kernel.hpp>
#include <small_gicp/points/point_cloud.hpp>
#include <small_gicp/points/traits.hpp>
#include <small_gicp/registration/rejector.hpp>

namespace small_gicp {

namespace cuda_detail {

// ---- factor / rejector TYPE -> kernel selector (compile time) ----
template <typename F>
struct factor_kind;  // no definition: a factor type the kernels do not implement does not compile
template <>
struct factor_kind<ICPFactor> {
  static constexpr int value = SGB_FACTOR_ICP;
};
template <>
struct factor_kind<PointToPlaneICPFactor> {
  static constexpr int value = SGB_FACTOR_PLANE_ICP;
};
template <>
struct factor_kind<GICPFactor> {
  static constexpr int value = SGB_FACTOR_GICP;
};

template <typename F>
struct unwrap {  // plain factor
  using base = F;
  static constexpr int robust = SGB_ROBUST_NONE;
  static double c(const F&) { return 1.0; }
  static F& state(F& f) { return f; }
};
template <typename F>
struct unwrap<RobustFactor<Huber, F>> {
  using base = F;
  static constexpr int robust = SGB_ROBUST_HUBER;
  static double c(const RobustFactor<Huber, F>& f) { return f.robust_kernel.c; }
  static F& state(RobustFactor<Huber, F>& f) { return f.factor; }
};
template <typename F>
struct unwrap<RobustFactor<Cauchy, F>> {
  using base = F;
  static constexpr int robust = SGB_ROBUST_CAUCHY;
  static double c(const RobustFactor<Cauchy, F>& f) { return f.robust_kernel.c; }
  static F& state(RobustFactor<Cauchy, F>& f) { return f.factor; }
};

inline int rejector_kind(const NullRejector&) { return SGB_REJECT_NONE; }
inline int rejector_kind(const DistanceRejector&) { return SGB_REJECT_DISTANCE; }
inline double rejector_threshold(const NullRejector&) { return 0.0; }
inline double rejector_threshold(const DistanceRejector& r) { return r.max_dist_sq; }

/// Identity of a host object as far as its device mirror is concerned.
struct MirrorKey {
  const void* addr = nullptr;
  size_t count = 0;
  std::uint64_t generation = 0;
  bool operator==(const MirrorKey& o) const { return addr == o.addr && count == o.count && generation == o.generation; }
};

struct DeviceMirror {
  sgb_ctx* ctx = nullptr;
  bool owned = true;  // false: borrowed through use_context(), not destroyed here
  MirrorKey target, tree, source;
  bool target_valid = false, source_valid = false;
  ~DeviceMirror() {
    if (ctx && owned) sgb_destroy(ctx);
  }
};

/// The one mirror record of a borrowed context.  Reductions that share a context through use_context() share what they believe it
/// holds: with a record each, one would keep searching a target another has since replaced on the device.  Attaching forgets the
/// record's clouds (a context created at the address of a destroyed one must not inherit its record).
inline std::shared_ptr<DeviceMirror> borrowed_mirror(sgb_ctx* ctx) {
  static std::mutex lock;
  static std::map<sgb_ctx*, std::weak_ptr<DeviceMirror>> by_ctx;
  std::lock_guard<std::mutex> guard(lock);
  for (auto it = by_ctx.begin(); it != by_ctx.end();) it = it->second.expired() ? by_ctx.erase(it) : std::next(it);
  std::shared_ptr<DeviceMirror> m = by_ctx[ctx].lock();
  if (!m) {
    m = std::make_shared<DeviceMirror>();
    m->ctx = ctx;
    m->owned = false;
    by_ctx[ctx] = m;
  }
  m->target_valid = m->source_valid = false;
  return m;
}

/// Contiguous views of a cloud in the C-ABI's layout (N x 4 / N x 16 doubles).  small_gicp::PointCloud's three std::vectors ARE
/// that layout and are passed through without a copy; any other cloud type is gathered through its traits first.
template <typename Cloud>
struct CloudArrays {
  std::vector<Eigen::Vector4d> pts_store, normals_store;
  std::vector<Eigen::Matrix4d> covs_store;
  const double* points = nullptr;
  const double* normals = nullptr;
  const double* covs = nullptr;
  size_t n = 0;

  CloudArrays(const Cloud& cloud, bool want_normals) {
    n = traits::size(cloud);
    if (n == 0) return;
    if constexpr (std::is_same_v<Cloud, PointCloud>) {
      points = cloud.points[0].data();
      if (want_normals && cloud.normals.size() == n) normals = cloud.normals[0].data();
      if (cloud.covs.size() == n) covs = cloud.covs[0].data();
    } else {
      pts_store.resize(n);
      for (size_t i = 0; i < n; i++) pts_store[i] = traits::point(cloud, i);
      points = pts_store[0].data();
      if (want_normals && traits::has_normals(cloud)) {
        normals_store.resize(n);
        for (size_t i = 0; i < n; i++) normals_store[i] = traits::normal(cloud, i);
        normals = normals_store[0].data();
      }
      if (traits::has_covs(cloud)) {
        covs_store.resize(n);
        for (size_t i = 0; i < n; i++) covs_store[i] = traits::cov(cloud, i);
        covs = covs_store[0].data();
      }
    }
  }
};

}  // namespace cuda_detail

/// Reduction on an H100 (one CUDA context per object; copies share it).
///
/// When are the clouds (re)uploaded?  The reference's reductions re-read host memory on every call.  This one mirrors target,
/// search structure and source to the device at the FIRST linearize() of every align() -- recognised by the freshly constructed
/// factor vector Registration::align hands in (registration.hpp:41) -- and re-uses the mirror for the remaining iterations of
/// that align() (the clouds are const there).  A caller whose target (or source) really stays the same over many align() calls
/// (scan-to-model) says so with a non-zero `target_generation` (`source_generation`): the mirror is then kept as long as address,
/// size and generation are unchanged, and the caller bumps the number when it edits the cloud.  invalidate() forgets everything.
struct ParallelReductionCUDA {
  ParallelReductionCUDA() : device(0), num_threads(0), target_generation(0), source_generation(0), sync_every_linearize(true) {}

  template <typename TargetPointCloud, typename SourcePointCloud, typename TargetTree, typename CorrespondenceRejector, typename Factor>
  std::tuple<Eigen::Matrix<double, 6, 6>, Eigen::Matrix<double, 6, 1>, double> linearize(
    const TargetPointCloud& target,
    const SourcePointCloud& source,
    const TargetTree& target_tree,
    const CorrespondenceRejector& rejector,
    const Eigen::Isometry3d& T,
    std::vector<Factor>& factors) const {
    using U = cuda_detail::unwrap<Factor>;
    sgb_ctx* ctx = context();
    if (factors.size() != traits::size(source)) throw std::runtime_error("ParallelReductionCUDA: factors.size() != size(source)");
    // a factor vector nobody has linearized yet = first iteration of an align(): the mirrors are re-validated
    const bool fresh = factors.empty() || U::state(factors[0]).source_index == std::numeric_limits<size_t>::max();
    mirror_target(ctx, target, target_tree, fresh);
    mirror_source(ctx, source, fresh);

    const Factor proto = factors.empty() ? Factor() : factors[0];
    double Tcol[16];  // column-major 4x4 (Eigen's own storage order, written out so that no storage order is assumed)
    for (int c = 0; c < 4; c++)
      for (int r = 0; r < 4; r++) Tcol[c * 4 + r] = T.matrix()(r, c);
    double out[43];
    check(ctx, sgb_linearize(ctx, cuda_detail::factor_kind<typename U::base>::value, U::robust, U::c(proto), cuda_detail::rejector_kind(rejector),
                             cuda_detail::rejector_threshold(rejector), Tcol, out));
    Eigen::Matrix<double, 6, 6> H;
    Eigen::Matrix<double, 6, 1> b;
    for (int r = 0; r < 6; r++) {
      for (int c = 0; c < 6; c++) H(r, c) = out[r * 6 + c];  // symmetric
      b(r) = out[36 + r];
    }
    if (!factors.empty()) U::state(factors[0]).source_index = 0;  // "this vector has been linearized" (see `fresh` above)
    if (sync_every_linearize) sync_factors(factors);
    return {H, b, out[42]};
  }

  /// Sum of the factor errors at a trial pose with the correspondences (and, for GICP, the fused precision matrices) of the last
  /// linearize(): both stay on the device, gicp_factor.hpp:81-89 semantics without shipping `mahalanobis` back.
  template <typename TargetPointCloud, typename SourcePointCloud, typename Factor>
  double error(const TargetPointCloud&, const SourcePointCloud&, const Eigen::Isometry3d& T, std::vector<Factor>&) const {
    sgb_ctx* ctx = context();
    double Tcol[16];
    for (int c = 0; c < 4; c++)
      for (int r = 0; r < 4; r++) Tcol[c * 4 + r] = T.matrix()(r, c);
    double e = 0.0;
    check(ctx, sgb_error(ctx, Tcol, &e));
    return e;
  }

  /// target_index / source_index of the last linearize() into the host factor vector, so that Factor::inlier()
  /// (optimizer.hpp:60,146) and user code reading correspondences keep working.  Called after every linearize() unless
  /// sync_every_linearize is false -- then the optimizers call it once, before their count_if (a 4-line change in optimizer.hpp).
  template <typename Factor>
  void sync_factors(std::vector<Factor>& factors) const {
    if (factors.empty()) return;
    using U = cuda_detail::unwrap<Factor>;
    sgb_ctx* ctx = context();
    corr_.resize(factors.size());
    check(ctx, sgb_correspondences(ctx, corr_.data()));
    for (size_t i = 0; i < factors.size(); i++) {
      auto& st = U::state(factors[i]);
      st.source_index = i;
      st.target_index = static_cast<size_t>(corr_[i]);  // SGB_NO_CORRESPONDENCE == std::numeric_limits<size_t>::max() == "outlier"
    }
  }

  size_t num_inliers() const {
    size_t n = 0;
    check(context(), sgb_num_inliers(context(), &n));
    return n;
  }

  /// Forget the device copies (after editing a cloud in place while keeping its generation, or when calling linearize() directly
  /// with a long-lived factor vector).
  void invalidate() const {
    if (mirror_) mirror_->target_valid = mirror_->source_valid = false;
  }

  /// Run on a context the caller owns (and keeps alive) instead of creating one: creating a context costs milliseconds (stream, page-locked
  /// result slot, first allocations) -- code that constructs a Registration<> per align() call shares one long-lived context this way.
  /// Every reduction given the same context shares one record of what the context holds (cuda_detail::borrowed_mirror).
  void use_context(sgb_ctx* ctx) const { mirror_ = cuda_detail::borrowed_mirror(ctx); }

  sgb_ctx* context() const {
    if (!mirror_) mirror_ = std::make_shared<cuda_detail::DeviceMirror>();
    if (!mirror_->ctx) {
      if (sgb_create(device, &mirror_->ctx) != 0) throw std::runtime_error(std::string("ParallelReductionCUDA: ") + sgb_last_error(nullptr));
    }
    return mirror_->ctx;
  }

public:
  int device;                       ///< CUDA device ordinal
  int num_threads;                  ///< accepted for source compatibility with the OMP / TBB reductions; unused
  std::uint64_t target_generation;  ///< non-zero: keep the target mirror across align() calls while (address, size, generation) match
  std::uint64_t source_generation;  ///< same for the source
  bool sync_every_linearize;        ///< true: stock optimizers work unchanged; false: one sync_factors() call at the end (see above)

private:
  static void check(sgb_ctx* ctx, int rc) {
    if (rc != 0) throw std::runtime_error(std::string("ParallelReductionCUDA: ") + sgb_last_error(ctx));
  }

  bool reusable(const cuda_detail::MirrorKey& have, const cuda_detail::MirrorKey& want, bool valid, bool fresh) const {
    if (!valid || !(have == want)) return false;
    return !fresh || want.generation != 0;  // a new align() re-uploads unless the caller vouches for the cloud with a generation
  }

  template <typename Source>
  void mirror_source(sgb_ctx* ctx, const Source& source, bool fresh) const {
    cuda_detail::MirrorKey key;
    key.addr = &source;
    key.count = traits::size(source);
    key.generation = source_generation;
    if (reusable(mirror_->source, key, mirror_->source_valid, fresh)) return;
    cuda_detail::CloudArrays<Source> a(source, false);
    check(ctx, sgb_source_set_points(ctx, a.n, a.points, a.covs));
    mirror_->source = key;
    mirror_->source_valid = true;
  }

  // ---- target + search structure ----
  template <typename Target, typename Cloud, typename Projection>
  void mirror_target(sgb_ctx* ctx, const Target& target, const KdTree<Cloud, Projection>& tree, bool fresh) const {
    mirror_target(ctx, target, tree.kdtree, fresh);
  }
  template <typename Target, typename Cloud, typename Projection>
  void mirror_target(sgb_ctx* ctx, const Target& target, const UnsafeKdTree<Cloud, Projection>& tree, bool fresh) const {
    static_assert(std::is_same_v<Projection, AxisAlignedProjection>, "the device search adopts axis-aligned kd-trees (ann/projection.hpp:18-55)");
    static_assert(sizeof(KdTreeNode<AxisAlignedProjection>) == 24 && sizeof(size_t) == sizeof(std::uint64_t), "node / index layout of ann/kdtree.hpp:56-71,237");
    cuda_detail::MirrorKey key, tkey;
    key.addr = &target;
    key.count = traits::size(target);
    key.generation = target_generation;
    tkey.addr = &tree;
    tkey.count = tree.nodes.size();
    tkey.generation = target_generation;
    if (reusable(mirror_->target, key, mirror_->target_valid, fresh) && mirror_->tree == tkey) return;
    cuda_detail::CloudArrays<Target> a(target, true);
    check(ctx, sgb_target_set_points(ctx, a.n, a.points, a.normals, a.covs));
    check(ctx, sgb_target_set_kdtree(ctx, tree.nodes.data(), tree.nodes.size(), tree.root, reinterpret_cast<const std::uint64_t*>(tree.indices.data())));
    mirror_->target = key;
    mirror_->tree = tkey;
    mirror_->target_valid = true;
  }
  /// VGICP (registration_helper.cpp:125-137): the Gaussian voxel map is both the target "cloud" and the search structure.
  void mirror_target(sgb_ctx* ctx, const GaussianVoxelMap& target, const GaussianVoxelMap& tree, bool fresh) const {
    if (&target != &tree) throw std::runtime_error("ParallelReductionCUDA: a voxel-map target must also be passed as the target tree");
    cuda_detail::MirrorKey key;
    key.addr = &target;
    key.count = target.size();
    key.generation = target_generation;
    if (reusable(mirror_->target, key, mirror_->target_valid, fresh) && mirror_->tree == key) return;
    const size_t n = target.size();
    std::vector<std::int32_t> coords(n * 3);
    std::vector<Eigen::Vector4d> means(n);
    std::vector<Eigen::Matrix4d> covs(n);
    for (size_t i = 0; i < n; i++) {
      const auto& v = *target.flat_voxels[i];
      for (int a = 0; a < 3; a++) coords[i * 3 + a] = v.first.coord[a];
      means[i] = v.second.mean;
      covs[i] = v.second.cov;
    }
    check(ctx, sgb_target_set_voxelmap(ctx, 1.0 / target.inv_leaf_size, n, coords.data(), n ? means[0].data() : nullptr, n ? covs[0].data() : nullptr,
                                       offset_pattern(target.search_offsets)));
    mirror_->target = mirror_->tree = key;
    mirror_->target_valid = true;
  }

  /// The probe pattern of a map's search_offsets: 1, 7 or 27.  Counted by distinct offsets, not by size(): set_search_offsets(27)
  /// appends the cube to the centre the constructor put there (incremental_voxelmap.hpp:46,176-183), which leaves 28 entries.
  template <typename Offsets>
  static int offset_pattern(const Offsets& offsets) {
    bool seen[27] = {};
    int distinct = 0, axis = 0;
    for (const auto& o : offsets) {
      if (o[0] < -1 || o[0] > 1 || o[1] < -1 || o[1] > 1 || o[2] < -1 || o[2] > 1) throw std::runtime_error("ParallelReductionCUDA: voxel search offset outside the 3x3x3 cube");
      const int k = (o[0] + 1) * 9 + (o[1] + 1) * 3 + (o[2] + 1);
      if (seen[k]) continue;
      seen[k] = true;
      distinct++;
      axis += (o[0] != 0) + (o[1] != 0) + (o[2] != 0) == 1;
    }
    if (distinct == 1 && seen[13]) return 1;
    if (distinct == 7 && seen[13] && axis == 6) return 7;
    if (distinct == 27) return 27;
    throw std::runtime_error("ParallelReductionCUDA: voxel search_offsets must be one of the patterns of set_search_offsets (1, 7 or 27)");
  }

  mutable std::shared_ptr<cuda_detail::DeviceMirror> mirror_;
  mutable std::vector<std::uint64_t> corr_;
};

}  // namespace small_gicp
