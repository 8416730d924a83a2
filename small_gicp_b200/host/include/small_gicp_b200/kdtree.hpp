// SPDX-License-Identifier: MIT
// Host-side kd-tree with the reference's public surface (KdTree<PointCloud>, UnsafeKdTree, KdTreeBuilder,
// knn_search / nearest_neighbor_search, traits) -- /root/reference/include/small_gicp/ann/kdtree.hpp:56-304,
// knn_result.hpp:13-108, projection.hpp:18-55 (axis-aligned projection only).
//
// The node array keeps the reference's 24-byte layout because it IS the data contract of
// sgb_target_set_kdtree(); the construction below is iterative (explicit work list, nodes emitted in
// pre-order) instead of the reference's recursion, and the search uses an explicit stack.
// `DeviceKdTree` is the H100-native alternative: no host nodes at all, the context builds the tree.
#pragma once
#include <algorithm>
#include <limits>
#include <numeric>

#include "core.hpp"

namespace small_gicp_b200 {

using NodeIndexType = std::uint32_t;
static constexpr NodeIndexType INVALID_NODE = std::numeric_limits<NodeIndexType>::max();

struct KnnSetting {
  double epsilon = 0.0;  ///< early-out once the k-th distance is below this (0 = exact search)
};

struct ProjectionSetting {
  int max_scan_count = 128;  ///< points sampled when choosing the split axis
};

/// Split along one coordinate axis.
struct AxisAlignedProjection {
  int axis;
  double operator()(const Vector4d& pt) const { return pt[axis]; }
};

/// 24 bytes: {first,last} for leaves or {axis, threshold} for inner nodes, then the two child indices.
struct KdTreeNode {
  union {
    struct {
      NodeIndexType first, last;
    } lr;
    struct {
      AxisAlignedProjection proj;
      double thresh;
    } sub;
  } node_type;
  NodeIndexType left = INVALID_NODE;
  NodeIndexType right = INVALID_NODE;
};
static_assert(sizeof(KdTreeNode) == 24, "KdTreeNode must match the layout sgb_target_set_kdtree() consumes");

/// Sorted list of the k best (index, squared distance) pairs; only strictly closer candidates displace.
class KnnHeap {
public:
  KnnHeap(size_t* indices, double* distances, int k) : k_(k), found_(0), idx_(indices), dist_(distances) {
    std::fill(idx_, idx_ + k_, std::numeric_limits<size_t>::max());
    std::fill(dist_, dist_ + k_, std::numeric_limits<double>::max());
  }
  double worst() const { return dist_[k_ - 1]; }
  size_t num_found() const { return found_; }
  void offer(size_t index, double d) {
    if (d >= worst()) return;
    int pos = std::min(found_, k_ - 1);
    while (pos > 0 && d < dist_[pos - 1]) {
      idx_[pos] = idx_[pos - 1];
      dist_[pos] = dist_[pos - 1];
      pos--;
    }
    idx_[pos] = index;
    dist_[pos] = d;
    found_ = std::min(found_ + 1, k_);
  }

private:
  int k_, found_;
  size_t* idx_;
  double* dist_;
};

/// Single-thread builder (leaf <= max_leaf_size, split axis = largest sample variance, median split).
struct KdTreeBuilder {
  int max_leaf_size = 20;
  ProjectionSetting projection_setting;

  template <typename Tree, typename PointCloud>
  void build_tree(Tree& tree, const PointCloud& points) const {
    const size_t n = traits::size(points);
    tree.indices.resize(n);
    std::iota(tree.indices.begin(), tree.indices.end(), size_t(0));
    tree.nodes.clear();
    tree.nodes.reserve(n / std::max(1, max_leaf_size / 2) + 1);
    tree.root = 0;

    struct Job {
      size_t first, last;
      NodeIndexType parent;  // node whose `right` awaits this job's node index (INVALID_NODE for left children / root)
    };
    std::vector<Job> jobs;
    jobs.push_back({0, n, INVALID_NODE});
    while (!jobs.empty()) {
      const Job job = jobs.back();
      jobs.pop_back();
      const NodeIndexType me = static_cast<NodeIndexType>(tree.nodes.size());
      tree.nodes.emplace_back();
      if (job.parent != INVALID_NODE) tree.nodes[job.parent].right = me;
      const size_t count = job.last - job.first;
      if (count <= static_cast<size_t>(max_leaf_size)) {
        tree.nodes[me].node_type.lr.first = static_cast<NodeIndexType>(job.first);
        tree.nodes[me].node_type.lr.last = static_cast<NodeIndexType>(job.last);
        continue;
      }
      const int axis = pick_axis(points, tree.indices.data() + job.first, count);
      size_t* lo = tree.indices.data() + job.first;
      size_t* mid = lo + count / 2;
      std::nth_element(lo, mid, lo + count, [&](size_t a, size_t b) { return traits::point(points, a)[axis] < traits::point(points, b)[axis]; });
      tree.nodes[me].node_type.sub.proj = AxisAlignedProjection{axis};
      tree.nodes[me].node_type.sub.thresh = traits::point(points, *mid)[axis];
      tree.nodes[me].left = me + 1;  // pre-order: the left subtree follows immediately
      jobs.push_back({job.first + count / 2, job.last, me});
      jobs.push_back({job.first, job.first + count / 2, INVALID_NODE});
    }
  }

private:
  template <typename PointCloud>
  int pick_axis(const PointCloud& points, const size_t* idx, size_t count) const {
    const size_t cap = static_cast<size_t>(projection_setting.max_scan_count);
    const size_t step = count < cap ? 1 : count / cap;
    const size_t samples = count / step;
    double s[3] = {0, 0, 0}, ss[3] = {0, 0, 0};
    for (size_t i = 0; i < samples; i++) {
      const auto p = traits::point(points, idx[i * step]);
      for (int d = 0; d < 3; d++) {
        s[d] += p[d];
        ss[d] += p[d] * p[d];
      }
    }
    double var[3];
    for (int d = 0; d < 3; d++) var[d] = ss[d] - s[d] / static_cast<double>(samples) * s[d];
    return var[0] > var[1] ? (var[0] > var[2] ? 0 : 2) : (var[1] > var[2] ? 1 : 2);
  }
};

/// Non-owning tree over `points` (the caller keeps the cloud alive).
template <typename PointCloud, typename Projection_ = AxisAlignedProjection>
struct UnsafeKdTree {
  using Projection = Projection_;
  using Node = KdTreeNode;

  template <typename Builder = KdTreeBuilder>
  explicit UnsafeKdTree(const PointCloud& points, const Builder& builder = Builder()) : points(points), root(0) {
    if (traits::size(points) == 0) return;
    builder.build_tree(*this, points);
  }

  size_t nearest_neighbor_search(const Vector4d& query, size_t* k_index, double* k_sq_dist, const KnnSetting& setting = KnnSetting()) const {
    return knn_search(query, 1, k_index, k_sq_dist, setting);
  }

  /// k nearest neighbours, ascending squared distance; returns how many were found (min(k, |points|)).
  size_t knn_search(const Vector4d& query, int k, size_t* k_indices, double* k_sq_dists, const KnnSetting& setting = KnnSetting()) const {
    KnnHeap heap(k_indices, k_sq_dists, k);
    if (nodes.empty()) return 0;
    struct Pending {
      NodeIndexType node;
      double cut_sq;
    };
    Pending stack[64];
    int sp = 0;
    NodeIndexType cur = root;
    for (;;) {
      const Node* nd = &nodes[cur];
      while (nd->left != INVALID_NODE) {  // walk down to a leaf, near side first
        const double diff = query[nd->node_type.sub.proj.axis] - nd->node_type.sub.thresh;
        const bool go_left = diff < 0.0;
        stack[sp++] = {go_left ? nd->right : nd->left, diff * diff};
        cur = go_left ? nd->left : nd->right;
        nd = &nodes[cur];
      }
      for (size_t i = nd->node_type.lr.first; i < nd->node_type.lr.last; i++) {
        const size_t pi = indices[i];
        heap.offer(pi, (traits::point(points, pi) - query).squaredNorm());
      }
      if (heap.worst() < setting.epsilon) break;
      bool resumed = false;
      while (sp > 0) {
        const Pending p = stack[--sp];
        if (heap.worst() > p.cut_sq) {
          cur = p.node;
          resumed = true;
          break;
        }
      }
      if (!resumed) break;
    }
    return heap.num_found();
  }

  const PointCloud& points;
  std::vector<size_t> indices;  ///< permutation of point indices; leaves own contiguous ranges of it
  NodeIndexType root;
  std::vector<Node> nodes;
};

/// Owning tree (keeps the cloud alive through a shared_ptr).
template <typename PointCloud, typename Projection = AxisAlignedProjection>
struct KdTree {
  using Ptr = std::shared_ptr<KdTree<PointCloud, Projection>>;
  using ConstPtr = std::shared_ptr<const KdTree<PointCloud, Projection>>;

  template <typename Builder = KdTreeBuilder>
  explicit KdTree(std::shared_ptr<const PointCloud> points, const Builder& builder = Builder()) : points(points), kdtree(*points, builder) {}

  size_t nearest_neighbor_search(const Vector4d& query, size_t* k_index, double* k_sq_dist, const KnnSetting& setting = KnnSetting()) const {
    return kdtree.nearest_neighbor_search(query, k_index, k_sq_dist, setting);
  }
  size_t knn_search(const Vector4d& query, size_t k, size_t* k_indices, double* k_sq_dists, const KnnSetting& setting = KnnSetting()) const {
    return kdtree.knn_search(query, static_cast<int>(k), k_indices, k_sq_dists, setting);
  }

  const std::shared_ptr<const PointCloud> points;
  const UnsafeKdTree<PointCloud, Projection> kdtree;
};

/// H100-native tree handle: nothing is built on the host; ParallelReductionCUDA asks the context to build
/// its own flattened tree over the target (sgb_target_build_kdtree).
template <typename PointCloud>
struct DeviceKdTree {
  explicit DeviceKdTree(std::shared_ptr<const PointCloud> points, int max_leaf_size = 0) : points(points), max_leaf_size(max_leaf_size) {}
  const std::shared_ptr<const PointCloud> points;
  int max_leaf_size;
};

namespace traits {
template <typename PointCloud, typename Projection>
struct Traits<UnsafeKdTree<PointCloud, Projection>> {
  static size_t nearest_neighbor_search(const UnsafeKdTree<PointCloud, Projection>& t, const Vector4d& p, size_t* k, double* d) { return t.nearest_neighbor_search(p, k, d); }
  static size_t knn_search(const UnsafeKdTree<PointCloud, Projection>& t, const Vector4d& p, size_t k, size_t* ki, double* kd) { return t.knn_search(p, static_cast<int>(k), ki, kd); }
};
template <typename PointCloud, typename Projection>
struct Traits<KdTree<PointCloud, Projection>> {
  static size_t nearest_neighbor_search(const KdTree<PointCloud, Projection>& t, const Vector4d& p, size_t* k, double* d) { return t.nearest_neighbor_search(p, k, d); }
  static size_t knn_search(const KdTree<PointCloud, Projection>& t, const Vector4d& p, size_t k, size_t* ki, double* kd) { return t.knn_search(p, k, ki, kd); }
};

template <typename T>
size_t knn_search(const T& tree, const Vector4d& point, size_t k, size_t* k_indices, double* k_sq_dists) {
  return Traits<T>::knn_search(tree, point, k, k_indices, k_sq_dists);
}
template <typename T>
size_t nearest_neighbor_search(const T& tree, const Vector4d& point, size_t* k_index, double* k_sq_dist) {
  return Traits<T>::nearest_neighbor_search(tree, point, k_index, k_sq_dist);
}
}  // namespace traits

}  // namespace small_gicp_b200
