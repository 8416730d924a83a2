// SPDX-License-Identifier: MIT
// ParallelReductionCUDA -- the H100 backend as a peer of SerialReduction / ParallelReductionOMP /
// ParallelReductionTBB (/root/reference/include/small_gicp/registration/reduction.hpp:12-63,
// reduction_omp.hpp:20-73, reduction_tbb.hpp:114-139): same two const member templates, plain public fields
// for tunables, default-constructible and copyable (copies share one device context).
//
// All per-point work (transform, NN search, rejection, factor, sum) runs in libsgicp_b200.so through the
// C-ABI in include/sgicp_b200.h.  The glue below only (1) mirrors the clouds / search structure to the
// device when they change and (2) maps factor / rejector TYPES to kernel selectors.  Unsupported
// argument types are compile errors, never a CPU fallback.
#pragma once
#include <cstring>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "../../../../include/sgicp_b200.h"
#include "core.hpp"
#include "factors.hpp"
#include "kdtree.hpp"
#include "voxelmap.hpp"

namespace small_gicp_b200 {

namespace detail {

/// Identity of a host object as far as its device mirror is concerned.  No content sampling: a cloud edited in place between two
/// align() calls is re-uploaded because every align() re-validates its mirrors (see ParallelReductionCUDA), not because a hash of a
/// few points happened to change.
struct MirrorKey {
  const void* addr = nullptr;
  size_t count = 0;
  uint64_t generation = 0;
  bool operator==(const MirrorKey& o) const { return addr == o.addr && count == o.count && generation == o.generation; }
  bool operator!=(const MirrorKey& o) const { return !(*this == o); }
};

/// Contiguous views of a cloud in the C-ABI's layout (N x 4 / N x 16 doubles).  PointCloud is passed
/// through without a copy; any other cloud type is gathered through its traits.
template <typename Cloud>
struct CloudArrays {
  std::vector<Vector4d> pts_store, normals_store;
  std::vector<Matrix4d> covs_store;
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

struct DeviceMirror {
  sgb_ctx* ctx = nullptr;
  bool owned = true;  // false: borrowed through use_context(), not destroyed here
  MirrorKey target_key, tree_key, source_key;
  bool target_valid = false, source_valid = false;
  ~DeviceMirror() {
    if (ctx && owned) sgb_destroy(ctx);
  }
};

template <typename T>
struct dependent_false : std::false_type {};

}  // namespace detail

/// When are the clouds (re)uploaded?  At the FIRST linearize() of every align() -- recognised by the freshly constructed factor vector
/// Registration::align hands in -- and the mirror is re-used for the remaining iterations of that align().  A cloud that stays the same
/// over many align() calls is kept across them when the caller sets a non-zero target_generation / source_generation (and bumps it on
/// every edit).  Same policy, same field names as include/small_gicp/registration/reduction_cuda.hpp (the Eigen-typed twin).
struct ParallelReductionCUDA {
  ParallelReductionCUDA() : device(0), num_threads(0), target_generation(0), source_generation(0) {}

  /// Sum of the linearised per-point factors: (H 6x6, b 6x1, e).
  template <typename TargetPointCloud, typename SourcePointCloud, typename TargetTree, typename CorrespondenceRejector, typename Factor>
  std::tuple<Matrix6d, Vector6d, double> linearize(const TargetPointCloud& target, const SourcePointCloud& source, const TargetTree& target_tree,
                                                   const CorrespondenceRejector& rejector, const Isometry3d& T, std::vector<Factor>& factors) const {
    sgb_ctx* ctx = context();
    if (factors.size() != traits::size(source)) throw std::runtime_error("ParallelReductionCUDA: factors.size() != size(source)");
    // a factor vector nobody has linearized yet = first iteration of an align(): the mirrors are re-validated
    const bool fresh = factors.empty() || factor_traits<Factor>::state(factors[0]).source_index == std::numeric_limits<size_t>::max();
    mirror_target(ctx, target, target_tree, fresh);
    mirror_source(ctx, source, fresh);
    const FactorDescriptor fd = factor_traits<Factor>::describe(factors.empty() ? Factor() : factors[0]);
    double out[43];
    check(ctx, sgb_linearize(ctx, fd.factor_kind, fd.robust_kind, fd.robust_c, CorrespondenceRejector::kind, rejector.threshold(), T.data(), out));
    Matrix6d H;
    Vector6d b;
    std::memcpy(H.data(), out, sizeof(double) * 36);  // symmetric: row/col-major agree
    std::memcpy(b.data(), out + 36, sizeof(double) * 6);
    if (!factors.empty()) factor_traits<Factor>::state(factors[0]).source_index = 0;  // "this vector has been linearized" (see `fresh`)
    return {H, b, out[42]};
  }

  /// Sum of the factor errors at a trial pose, with the correspondences of the last linearize().
  template <typename TargetPointCloud, typename SourcePointCloud, typename Factor>
  double error(const TargetPointCloud&, const SourcePointCloud&, const Isometry3d& T, std::vector<Factor>&) const {
    sgb_ctx* ctx = context();
    double e = 0.0;
    check(ctx, sgb_error(ctx, T.data(), &e));
    return e;
  }

  /// Copy target_index / source_index of the last linearize() into the host factor vector
  /// (so that factor.inlier() and user code reading correspondences keep working).
  template <typename Factor>
  void sync_factors(std::vector<Factor>& factors) const {
    if (factors.empty()) return;
    sgb_ctx* ctx = context();
    std::vector<uint64_t> corr(factors.size());
    check(ctx, sgb_correspondences(ctx, corr.data()));
    for (size_t i = 0; i < factors.size(); i++) {
      auto& st = factor_traits<Factor>::state(factors[i]);
      st.source_index = i;
      st.target_index = static_cast<size_t>(corr[i]);
    }
  }

  size_t num_inliers() const {
    size_t n = 0;
    sgb_ctx* ctx = context();
    check(ctx, sgb_num_inliers(ctx, &n));
    return n;
  }

  /// Forget the device copies (call after mutating a cloud in place between align() calls).
  void invalidate() const {
    if (mirror) mirror->target_valid = mirror->source_valid = false;
  }

  /// Run on a context the caller owns (and keeps alive) instead of creating one: creating a context costs milliseconds (stream, page-locked
  /// result slot, first allocations) -- callers that build a Registration<> per align(), like the helper align() overloads, share one
  /// long-lived context this way.  Its mirrors are invalidated.
  void use_context(sgb_ctx* ctx) const {
    mirror = std::make_shared<detail::DeviceMirror>();
    mirror->ctx = ctx;
    mirror->owned = false;
  }

  /// BatchRegistration: mirror the target and its search structure as the first linearize() of an align() does, and return the context.
  /// The caller replaces the source with a batch, so the source mirror is dropped.
  template <typename Target, typename Tree>
  sgb_ctx* batch_context(const Target& target, const Tree& target_tree) const {
    sgb_ctx* ctx = context();
    mirror_target(ctx, target, target_tree, true);
    mirror->source_valid = false;
    return ctx;
  }

  sgb_ctx* context() const {
    if (!mirror) mirror = std::make_shared<detail::DeviceMirror>();
    if (!mirror->ctx) {
      if (sgb_create(device, &mirror->ctx) != 0) throw std::runtime_error(std::string("ParallelReductionCUDA: ") + sgb_last_error(nullptr));
    }
    return mirror->ctx;
  }

  int device;                  ///< CUDA device ordinal
  int num_threads;             ///< accepted for source compatibility with the OMP / TBB reductions; unused
  uint64_t target_generation;  ///< non-zero: keep the target mirror across align() calls while (address, size, generation) match
  uint64_t source_generation;  ///< same for the source

private:
  static void check(sgb_ctx* ctx, int rc) {
    if (rc != 0) throw std::runtime_error(std::string("ParallelReductionCUDA: ") + sgb_last_error(ctx));
  }

  bool reusable(const detail::MirrorKey& have, const detail::MirrorKey& want, bool valid, bool fresh) const {
    if (!valid || have != want) return false;
    return !fresh || want.generation != 0;  // a new align() re-uploads unless the caller vouches for the cloud with a generation
  }
  template <typename Cloud>
  detail::MirrorKey cloud_key(const Cloud& cloud, uint64_t generation) const {
    detail::MirrorKey k;
    k.addr = &cloud;
    k.count = traits::size(cloud);
    k.generation = generation;
    return k;
  }

  template <typename Source>
  void mirror_source(sgb_ctx* ctx, const Source& source, bool fresh) const {
    const detail::MirrorKey key = cloud_key(source, source_generation);
    if (reusable(mirror->source_key, key, mirror->source_valid, fresh)) return;
    detail::CloudArrays<Source> a(source, false);
    check(ctx, sgb_source_set_points(ctx, a.n, a.points, a.covs));
    mirror->source_key = key;
    mirror->source_valid = true;
  }

  // ---- target + search structure ----
  template <typename Target, typename Cloud, typename Projection>
  void mirror_target(sgb_ctx* ctx, const Target& target, const KdTree<Cloud, Projection>& tree, bool fresh) const {
    mirror_target(ctx, target, tree.kdtree, fresh);
  }
  template <typename Target, typename Cloud, typename Projection>
  void mirror_target(sgb_ctx* ctx, const Target& target, const UnsafeKdTree<Cloud, Projection>& tree, bool fresh) const {
    static_assert(std::is_same_v<Projection, AxisAlignedProjection>, "the device search supports axis-aligned kd-trees");
    const detail::MirrorKey key = cloud_key(target, target_generation);
    detail::MirrorKey tkey;
    tkey.addr = &tree;
    tkey.count = tree.nodes.size();
    tkey.generation = target_generation;
    if (reusable(mirror->target_key, key, mirror->target_valid, fresh) && tkey == mirror->tree_key) return;
    detail::CloudArrays<Target> a(target, true);
    check(ctx, sgb_target_set_points(ctx, a.n, a.points, a.normals, a.covs));
    static_assert(sizeof(size_t) == sizeof(uint64_t), "64-bit size_t expected");
    check(ctx, sgb_target_set_kdtree(ctx, tree.nodes.data(), tree.nodes.size(), tree.root, reinterpret_cast<const uint64_t*>(tree.indices.data())));
    mirror->target_key = key;
    mirror->tree_key = tkey;
    mirror->target_valid = true;
  }
  template <typename Target, typename Cloud>
  void mirror_target(sgb_ctx* ctx, const Target& target, const DeviceKdTree<Cloud>& tree, bool fresh) const {
    const detail::MirrorKey key = cloud_key(target, target_generation);
    detail::MirrorKey tkey;
    tkey.addr = &tree;
    tkey.count = static_cast<size_t>(tree.max_leaf_size);
    tkey.generation = target_generation;
    if (reusable(mirror->target_key, key, mirror->target_valid, fresh) && tkey == mirror->tree_key) return;
    detail::CloudArrays<Target> a(target, true);
    check(ctx, sgb_target_set_points(ctx, a.n, a.points, a.normals, a.covs));
    check(ctx, sgb_target_build_kdtree(ctx, tree.max_leaf_size));
    mirror->target_key = key;
    mirror->tree_key = tkey;
    mirror->target_valid = true;
  }
  /// VGICP: the voxel map is both the target "cloud" and the search structure.
  void mirror_target(sgb_ctx* ctx, const GaussianVoxelMap& target, const GaussianVoxelMap& tree, bool fresh) const {
    if (&target != &tree) throw std::runtime_error("ParallelReductionCUDA: a voxel-map target must also be passed as the target tree");
    detail::MirrorKey key;
    key.addr = &target;
    key.count = target.size();
    key.generation = target_generation ? target_generation * 1315423911ull + target.generation : 0;  // the map counts its own inserts
    if (reusable(mirror->target_key, key, mirror->target_valid, fresh) && key == mirror->tree_key) return;
    const size_t n = target.size();
    std::vector<int32_t> coords(n * 3);
    std::vector<Vector4d> means(n);
    std::vector<Matrix4d> covs(n);
    for (size_t i = 0; i < n; i++) {
      const GaussianVoxel& v = target.flat_voxels[i];
      coords[i * 3 + 0] = v.coord.x;
      coords[i * 3 + 1] = v.coord.y;
      coords[i * 3 + 2] = v.coord.z;
      means[i] = v.mean;
      covs[i] = v.cov;
    }
    check(ctx, sgb_target_set_voxelmap(ctx, target.leaf_size, n, coords.data(), n ? means[0].data() : nullptr, n ? covs[0].data() : nullptr,
                                       static_cast<int>(target.search_offsets.size())));
    mirror->target_key = mirror->tree_key = key;
    mirror->target_valid = true;
  }

  mutable std::shared_ptr<detail::DeviceMirror> mirror;
};

}  // namespace small_gicp_b200
