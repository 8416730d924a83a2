// SPDX-License-Identifier: MIT
// Host-side construction of the flattened (pre-order, 8-byte node) kd-tree consumed by the search kernel:
//  (1) adoption of a tree built by the reference (any builder's node order), and
//  (2) this library's own median-split builder (replaces KdTreeBuilder::build_tree,
//      /root/reference/include/small_gicp/ann/kdtree.hpp:74-131; exact-NN results do not depend on the
//      split choices, only exact ties do).
#include "sgb_kdtree_host.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <numeric>

namespace sgb {

namespace {
// Reference node layout (ann/kdtree.hpp:56-71): union{ {u32 first,last} | {int axis; double thresh} } , u32 left, u32 right
struct RefNode {
  union {
    struct {
      uint32_t first, last;
    } lr;
    struct {
      int32_t axis;
      double thresh;
    } sub;
  } u;
  uint32_t left, right;
};
static_assert(sizeof(RefNode) == 24, "reference KdTreeNode<AxisAlignedProjection> is 24 bytes");
constexpr uint32_t kInvalid = 0xFFFFFFFFu;
}  // namespace

bool flatten_reference_tree(const void* nodes24, size_t n_nodes, uint32_t root, const uint64_t* indices, size_t n_points, const double centre[3],
                            FlatTree& out, std::string& err) {
  out.nodes.clear();
  out.perm.clear();
  out.depth = 0;
  if (n_points == 0 || n_nodes == 0) return true;
  if (n_points >= (1ull << 31) || n_nodes >= (1ull << 30)) {
    err = "kd-tree too large for 32-bit device indices";
    return false;
  }
  if (root >= n_nodes) {
    err = "kd-tree root index out of range";
    return false;
  }
  const RefNode* in = static_cast<const RefNode*>(nodes24);
  out.nodes.resize(n_nodes);
  out.perm.resize(n_points);
  for (size_t i = 0; i < n_points; i++) {
    if (indices[i] >= n_points) {
      err = "kd-tree point index out of range";
      return false;
    }
    out.perm[i] = static_cast<uint32_t>(indices[i]);
  }
  // iterative pre-order walk; `fix` = flat index of the parent whose right-child slot must be patched
  struct Item {
    uint32_t ref;
    uint32_t fix;
    int depth;
  };
  std::vector<Item> stack;
  stack.push_back({root, kInvalid, 0});
  uint32_t next = 0;
  size_t visited = 0;
  while (!stack.empty()) {
    const Item it = stack.back();
    stack.pop_back();
    if (++visited > n_nodes) {
      err = "kd-tree has a cycle";
      return false;
    }
    const RefNode& rn = in[it.ref];
    const uint32_t me = next++;
    if (it.fix != kInvalid) out.nodes[it.fix].y |= (me << 2);
    if (rn.left == kInvalid) {  // leaf (ann/kdtree.hpp:197)
      const uint32_t first = rn.u.lr.first, last = rn.u.lr.last;
      if (last < first || last > n_points || (last - first) >= (1u << 30)) {
        err = "kd-tree leaf range out of range";
        return false;
      }
      out.nodes[me] = FlatNode{first, ((last - first) << 2) | 3u};
      out.depth = std::max(out.depth, it.depth);
    } else {
      if (rn.left >= n_nodes || rn.right >= n_nodes || rn.u.sub.axis < 0 || rn.u.sub.axis > 2) {
        err = "kd-tree inner node out of range";
        return false;
      }
      const float th = static_cast<float>(rn.u.sub.thresh - centre[rn.u.sub.axis]);
      uint32_t bits;
      std::memcpy(&bits, &th, 4);
      out.nodes[me] = FlatNode{bits, static_cast<uint32_t>(rn.u.sub.axis)};
      // right is visited after the whole left subtree: push right first
      stack.push_back({rn.right, me, it.depth + 1});
      stack.push_back({rn.left, kInvalid, it.depth + 1});
    }
  }
  out.nodes.resize(next);
  return true;
}

// ---------------------------------------------------------------------------------------------
namespace {
struct Builder {
  const float* pts;  // float4 stride
  uint32_t* perm;
  FlatNode* nodes;
  int max_leaf;
  int depth = 0;
  std::map<size_t, uint32_t> memo;

  uint32_t count_nodes(size_t n) {
    if (n <= static_cast<size_t>(max_leaf)) return 1;
    auto it = memo.find(n);
    if (it != memo.end()) return it->second;
    const uint32_t c = 1 + count_nodes(n / 2) + count_nodes(n - n / 2);
    memo[n] = c;
    return c;
  }
  void prime(size_t n) { count_nodes(n); }
  uint32_t count_nodes_ro(size_t n) const {
    if (n <= static_cast<size_t>(max_leaf)) return 1;
    return memo.find(n)->second;
  }

  void build(uint32_t me, size_t first, size_t last, int d, int* max_depth) const {
    const size_t n = last - first;
    if (n <= static_cast<size_t>(max_leaf)) {
      nodes[me] = FlatNode{static_cast<uint32_t>(first), (static_cast<uint32_t>(n) << 2) | 3u};
      if (d > *max_depth) {
#pragma omp critical(sgb_depth)
        if (d > *max_depth) *max_depth = d;
      }
      return;
    }
    // split the widest extent of the node's bounding box at the median
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (size_t i = first; i < last; i++) {
      const float* p = pts + 4 * static_cast<size_t>(perm[i]);
      for (int a = 0; a < 3; a++) {
        lo[a] = std::min(lo[a], p[a]);
        hi[a] = std::max(hi[a], p[a]);
      }
    }
    int axis = 0;
    float ext = hi[0] - lo[0];
    for (int a = 1; a < 3; a++)
      if (hi[a] - lo[a] > ext) {
        ext = hi[a] - lo[a];
        axis = a;
      }
    const size_t mid = first + n / 2;
    const float* P = pts;
    std::nth_element(perm + first, perm + mid, perm + last,
                     [P, axis](uint32_t a, uint32_t b) { return P[4 * static_cast<size_t>(a) + axis] < P[4 * static_cast<size_t>(b) + axis]; });
    const float th = P[4 * static_cast<size_t>(perm[mid]) + axis];
    uint32_t bits;
    std::memcpy(&bits, &th, 4);
    const uint32_t left = me + 1, right = me + 1 + count_nodes_ro(n / 2);
    nodes[me] = FlatNode{bits, (right << 2) | static_cast<uint32_t>(axis)};
#pragma omp task default(shared) if (n > 4096)
    build(left, first, mid, d + 1, max_depth);
#pragma omp task default(shared) if (n > 4096)
    build(right, mid, last, d + 1, max_depth);
#pragma omp taskwait
  }
};
}  // namespace

bool build_flat_tree(const float* pts_xyzw, size_t n_points, int max_leaf_size, FlatTree& out, std::string& err) {
  out.nodes.clear();
  out.perm.clear();
  out.depth = 0;
  if (n_points == 0) return true;
  if (n_points >= (1ull << 30)) {
    err = "too many points for 32-bit device indices";
    return false;
  }
  if (max_leaf_size <= 0) max_leaf_size = 32;  // one point per lane in the packet search's leaf scan (leaf sizes 8..64 were compared)
  if (max_leaf_size > 64) max_leaf_size = 64;
  out.perm.resize(n_points);
  std::iota(out.perm.begin(), out.perm.end(), 0u);
  Builder b;
  b.pts = pts_xyzw;
  b.perm = out.perm.data();
  b.max_leaf = max_leaf_size;
  b.prime(n_points);
  out.nodes.resize(b.count_nodes_ro(n_points));
  b.nodes = out.nodes.data();
  int max_depth = 0;
#pragma omp parallel
  {
#pragma omp single nowait
    b.build(0, 0, n_points, 0, &max_depth);
  }
  out.depth = max_depth;
  return true;
}

// ---------------------------------------------------------------------------------------------
// Packet (BVH2) form of a flattened kd-tree: one 64-byte record per INNER node holding the tight bounding boxes and the
// descriptors of its two children (see sgb_kernels_packet.cu).  Same leaves, same point permutation.
// ---------------------------------------------------------------------------------------------
bool build_packet_nodes(const FlatTree& tree, const float* pts_xyzw, std::vector<PacketNode>& out, int* max_pending) {
  out.clear();
  *max_pending = 1;
  const size_t nn = tree.nodes.size();
  if (nn == 0) return true;
  struct Box {
    float lo[3], hi[3];
  };
  std::vector<Box> box(nn);
  std::vector<uint32_t> compact(nn, 0);
  // children have larger pre-order indices than their parent: one reverse sweep computes every box
  for (size_t r = nn; r-- > 0;) {
    const FlatNode nd = tree.nodes[r];
    Box b;
    if ((nd.y & 3u) == 3u) {
      for (int a = 0; a < 3; a++) {
        b.lo[a] = INFINITY;
        b.hi[a] = -INFINITY;
      }
      const uint32_t first = nd.x, cnt = nd.y >> 2;
      for (uint32_t j = 0; j < cnt; j++) {
        const float* p = pts_xyzw + 4 * static_cast<size_t>(tree.perm[first + j]);
        for (int a = 0; a < 3; a++) {
          b.lo[a] = std::min(b.lo[a], p[a]);
          b.hi[a] = std::max(b.hi[a], p[a]);
        }
      }
    } else {
      const Box &l = box[r + 1], &rr = box[nd.y >> 2];
      for (int a = 0; a < 3; a++) {
        b.lo[a] = std::min(l.lo[a], rr.lo[a]);
        b.hi[a] = std::max(l.hi[a], rr.hi[a]);
      }
    }
    box[r] = b;
  }
  uint32_t n_inner = 0;
  for (size_t i = 0; i < nn; i++)
    if ((tree.nodes[i].y & 3u) != 3u) compact[i] = n_inner++;
  auto put_child = [&](PacketNode& pn, int side, size_t child) {
    const FlatNode c = tree.nodes[child];
    uint32_t a, b;
    if ((c.y & 3u) == 3u) {
      a = c.x;
      b = c.y >> 2;
    } else {
      a = compact[child];
      b = 0u;
    }
    float* v = pn.v + side * 8;
    for (int k = 0; k < 3; k++) {
      v[k] = box[child].lo[k];
      v[4 + k] = box[child].hi[k];
    }
    std::memcpy(&v[3], &a, 4);
    std::memcpy(&v[7], &b, 4);
    if ((c.y & 3u) == 3u && b == 0u) {  // empty leaf: never wanted
      for (int k = 0; k < 3; k++) {
        v[k] = INFINITY;
        v[4 + k] = -INFINITY;
      }
    }
  };
  auto put_empty = [](PacketNode& pn, int side) {
    float* v = pn.v + side * 8;
    for (int k = 0; k < 3; k++) {
      v[k] = INFINITY;
      v[4 + k] = -INFINITY;
    }
    const uint32_t z = 0u;
    std::memcpy(&v[3], &z, 4);
    std::memcpy(&v[7], &z, 4);
  };
  if (n_inner == 0) {  // the whole tree is one leaf: a root whose only child is that leaf
    out.resize(1);
    put_child(out[0], 0, 0);
    put_empty(out[0], 1);
    if ((tree.nodes[0].y >> 2) == 0u) put_empty(out[0], 0);
    return true;
  }
  out.resize(n_inner);
  for (size_t i = 0; i < nn; i++) {
    const FlatNode nd = tree.nodes[i];
    if ((nd.y & 3u) == 3u) continue;
    PacketNode& pn = out[compact[i]];
    put_child(pn, 0, i + 1);
    put_child(pn, 1, nd.y >> 2);
  }
  *max_pending = tree.depth > 0 ? tree.depth : 1;
  return true;
}

}  // namespace sgb
