// SPDX-License-Identifier: MIT
// Device-side data layout and per-point math of the H100 hot path.  See DESIGN.md §3-4.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cfloat>

#include "sgb_math.cuh"

namespace sgb {

constexpr uint32_t kNone = 0xFFFFFFFFu;  // no correspondence
constexpr int kLinBlock = 128;           // threads per CTA of the linearize / error kernels
constexpr int kPartialStride = 32;       // doubles per CTA partial (28 sums + inlier count, padded)

/// Flattened kd-tree node, 8 bytes, nodes in PRE-ORDER so that the left child of node i is i+1.
///   inner: x = split threshold (float bits), y = (right_child << 2) | axis        (axis in 0..2)
///   leaf : x = first point (offset into the leaf-ordered point arrays), y = (count << 2) | 3
using KdNode = uint2;

struct DevTarget {
  const float4* pts;      // leaf order; xyz relative to `centre`; w = original index (int bits) / unused for voxels
  const float4* normals;  // leaf order (plane ICP) or null
  const float4* covA;     // (xx, xy, xz, yy)
  const float4* covB;     // (yz, zz, 0, 0)
  const KdNode* nodes;    // kd-tree (null for voxel maps)
  const double* centre;   // 3 doubles, device
  // voxel map (VGICP)
  const int4* vox_table;  // open addressing: (x, y, z, voxel_id), voxel_id < 0 = empty
  uint32_t vox_mask;      // capacity - 1 (power of two)
  int vox_num_offsets;    // 1, 7 or 27
  double vox_inv_leaf;
};

struct DevSource {
  const float4* pts;   // Morton order; xyz relative to `centre`
  const float4* covA;  // Morton order
  const float4* covB;
  const double* centre;  // 3 doubles, device
  uint32_t n;
  uint32_t run;  // K: source positions chunk*32K + k*32 + lane hold Morton ranks chunk*32K + lane*K + k (full chunks),
                 // i.e. one lane walks K spatially consecutive points while every load of the warp stays coalesced
};

/// Multi-GPU exchange fused into the finishing CTA of the reduction (one process per GPU, source sharded, SURVEY §8e).
/// Every rank owns a MAILBOX in its device memory that its peers map through CUDA IPC:
///   doubles [2 parities][kMaxPeers senders][kMailStride]   then   unsigned long long flags [2 parities][kMaxPeers senders]
/// Rank r stores its sums into slot (parity, r) of every peer's mailbox over NVLink, fences, stores the call's sequence
/// number into the matching flag, waits until its OWN mailbox shows the sequence number of every sender and adds the
/// slots in rank order (deterministic, identical on all ranks).  Two parities: a rank can be at most one call ahead.
constexpr int kMaxPeers = 8;
constexpr int kMailStride = 64;
constexpr size_t kMailFlagOffset = 2 * kMaxPeers * kMailStride * sizeof(double);
constexpr size_t kMailBytes = kMailFlagOffset + 2 * kMaxPeers * sizeof(unsigned long long);
constexpr unsigned long long kCommPoison = 1ull << 63;  // flag bit: the sender could not run its reduction (its call failed on the host)
constexpr int kCommStampRing = 64;                      // wait times of the last 64 exchanges (sgb_comm_wait_ns)
struct CommParams {
  unsigned char* mail[kMaxPeers];  // mailbox of every rank (mail[rank] is local memory)
  int world, rank;                 // world <= 1: no exchange
  unsigned long long seq;          // sequence number of this call (same on all ranks, > 0)
  unsigned long long timeout_ns;   // give up waiting for a peer after this long (the result is then NaN and *status becomes non-zero)
  unsigned int* status;            // sticky device word: 1 = gave up on a peer, 2 = a peer reported a failed call (never cleared by the kernels)
  unsigned long long* stamps;      // [kCommStampRing]: ns this rank waited for its peers in exchange seq % kCommStampRing (or null)
  int poison;                      // this rank has nothing valid to contribute: tell the peers (host-side failure after the sequence number was taken)
};

struct LinParams {
  DevTarget tgt;
  DevSource src;
  CommParams comm;
  double T[12];      // row-major R (9) then t (3): T_target_source of this call
  double Tlin[12];   // pose of the last linearize (error kernel, GICP precision matrix)
  float max_dist_sq;     // search bound in FP32, a hair above the rejector's threshold (FLT_MAX for NullRejector)
  double max_dist_sq_d;  // the rejector's threshold itself, applied to the FP64 residual (DBL_MAX for NullRejector)
  int use_prev;          // corr[] holds the previous linearize's correspondences for the same clouds: use them as search seeds
  double robust_c;
  uint32_t* corr;     // per source point (Morton order): leaf-order position / voxel id, or kNone
  double* partials;   // gridDim.x * kPartialStride
  unsigned int* ticket;
  double* out;        // 44 doubles: H(36) | b(6) | e | num_inliers     (error kernel: out[0] = e)
};

/// Programmatic dependent launch (sm_90+).  A kernel launched with launch_dependent() (sgb_kernels.h) may be set up and
/// scheduled while its predecessor on the stream is still draining; it must call this before it touches anything the
/// predecessor wrote.  Without the launch attribute the instruction returns immediately.
__device__ __forceinline__ void grid_dependency_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

/// The pose in the centred frames:  p' - c_t = R p_f + t'  with  t' = R c_s + t - c_t.
/// T: row-major R (9) then t (3); (csx, csy, csz) = c_s, the source centre; ct = c_t, the target centre.
__device__ __forceinline__ double3 centred_translation(const double* T, double csx, double csy, double csz, const double* ct) {
  return make_double3(T[0] * csx + T[1] * csy + T[2] * csz + T[9] - ct[0], T[3] * csx + T[4] * csy + T[5] * csz + T[10] - ct[1],
                      T[6] * csx + T[7] * csy + T[8] * csz + T[11] - ct[2]);
}
/// FP64 query of a stored (source-centred FP32) point, in the target-centred frame: R p_f + t'.
__device__ __forceinline__ double3 centred_query(const double* R, const double3& tp, const float4& p) {
  const double sx = p.x, sy = p.y, sz = p.z;
  return make_double3(R[0] * sx + R[1] * sy + R[2] * sz + tp.x, R[3] * sx + R[4] * sy + R[5] * sz + tp.y, R[6] * sx + R[7] * sy + R[8] * sz + tp.z);
}
/// The FP32 search query: the FP64 query rounded once.  Every search kernel and the batch transform derive it here, so a point's
/// query, and therefore its correspondence, is the same whichever path searched it.
__device__ __forceinline__ float3 centred_query_f32(const double* R, const double3& tp, const float4& p) {
  const double3 q = centred_query(R, tp, p);
  return make_float3(static_cast<float>(q.x), static_cast<float>(q.y), static_cast<float>(q.z));
}

/// The pose of a source relative to a placed map: out = Pinv * T, all row-major R (9) then t (3); Pinv = the inverse of the map's
/// placement (R_P^T | -R_P^T t_P).  Submap members (sgb_source_set_submaps): the search and the factor kernels both derive a member's
/// pose in the stored frame of an entry's map here, so a point is searched and linearised at the same pose.
__device__ __forceinline__ void relative_pose(const double* __restrict__ Pinv, const double* __restrict__ T, double* out) {
#pragma unroll
  for (int r = 0; r < 3; r++) {
    const double a = Pinv[3 * r + 0], b = Pinv[3 * r + 1], c = Pinv[3 * r + 2];
#pragma unroll
    for (int k = 0; k < 3; k++) out[3 * r + k] = a * T[k] + b * T[3 + k] + c * T[6 + k];
    out[9 + r] = a * T[9] + b * T[10] + c * T[11] + Pinv[9 + r];
  }
}

/// Squared distance of q to the box [lo, hi] (xyz; 0 inside): the pruning bound of the tree walks.
__device__ __forceinline__ float box_dist2(float qx, float qy, float qz, const float4& lo, const float4& hi) {
  const float dx = fmaxf(fmaxf(lo.x - qx, qx - hi.x), 0.0f);
  const float dy = fmaxf(fmaxf(lo.y - qy, qy - hi.y), 0.0f);
  const float dz = fmaxf(fmaxf(lo.z - qz, qz - hi.z), 0.0f);
  return dx * dx + dy * dy + dz * dz;
}

// ---------------------------------------------------------------------------------------------
/// Slot hash of the voxel-map table.  Also run on the host, which fills the table of sgb_target_set_voxelmap.
__host__ __device__ __forceinline__ uint32_t vox_hash(int x, int y, int z) {
  // any hash works (lookups are exact-match); this is a 32-bit mix of the three coordinates
  uint32_t h = static_cast<uint32_t>(x) * 73856093u ^ static_cast<uint32_t>(y) * 19349669u ^ static_cast<uint32_t>(z) * 83492791u;
  h ^= h >> 15;
  h *= 0x2c1b3c6du;
  h ^= h >> 12;
  return h;
}

// Gaussian-voxel-map target (VGICP): hash probe of 1 / 7 / 27 voxels in the reference's offset order
// (incremental_voxelmap.hpp:157-186), nearest voxel mean wins, first-found wins ties (knn_result.hpp:81-83).
__device__ __forceinline__ void vox_offset(int num, int o, int& dx, int& dy, int& dz) {
  if (num == 27) {  // for i, j, k in -1..1 (lexicographic)
    dx = o / 9 - 1;
    dy = (o / 3) % 3 - 1;
    dz = o % 3 - 1;
  } else {  // 1 or 7: centre, +x, +y, +z, -x, -y, -z
    const int s = o == 0 ? 0 : (o <= 3 ? 1 : -1);
    const int a = o == 0 ? -1 : (o - 1) % 3;
    dx = a == 0 ? s : 0;
    dy = a == 1 ? s : 0;
    dz = a == 2 ? s : 0;
  }
}

/// The voxel id stored for voxel (vx, vy, vz) in a table (region) of mask + 1 slots, or -1: the linear probe from its hash slot
/// (vox_nearest, and the voxel k-NN of sgb_target_batch_knn_maps in sgb_preprocess.cu).
__device__ __forceinline__ int vox_find(const int4* __restrict__ table, uint32_t mask, int vx, int vy, int vz) {
  uint32_t slot = vox_hash(vx, vy, vz) & mask;
  for (;;) {
    const int4 e = __ldg(&table[slot]);
    if (e.w < 0) return -1;
    if (e.x == vx && e.y == vy && e.z == vz) return e.w;
    slot = (slot + 1u) & mask;
  }
}

/// Nearest voxel mean of the (target-centred, FP64) query q, or kNone; DistanceRejector applied (d2 > max_d rejects).
/// (brx, bry, brz) = mean - q of the winner.
__device__ __forceinline__ uint32_t vox_nearest(const DevTarget& tgt, double qx, double qy, double qz, double ctx, double cty, double ctz, double max_d,
                                                double& brx, double& bry, double& brz) {
  // voxel coordinate of the un-centred point, fast_floor semantics == floor (util/fast_floor.hpp:12-15)
  const int cx = static_cast<int>(floor((qx + ctx) * tgt.vox_inv_leaf));
  const int cy = static_cast<int>(floor((qy + cty) * tgt.vox_inv_leaf));
  const int cz = static_cast<int>(floor((qz + ctz) * tgt.vox_inv_leaf));
  double best_d = DBL_MAX;
  uint32_t best = kNone;
  for (int o = 0; o < tgt.vox_num_offsets; o++) {
    int ox, oy, oz;
    vox_offset(tgt.vox_num_offsets, o, ox, oy, oz);
    const int id = vox_find(tgt.vox_table, tgt.vox_mask, cx + ox, cy + oy, cz + oz);
    if (id >= 0) {
      const float4 m = __ldg(&tgt.pts[id]);
      const double dx = static_cast<double>(m.x) - qx, dy = static_cast<double>(m.y) - qy, dz = static_cast<double>(m.z) - qz;
      const double d = dx * dx + dy * dy + dz * dz;
      if (d < best_d) {
        best_d = d;
        best = static_cast<uint32_t>(id);
        brx = dx;
        bry = dy;
        brz = dz;
      }
    }
  }
  if (best != kNone && best_d > max_d) best = kNone;  // DistanceRejector, rejector.hpp:23-25
  return best;
}

/// FP32 packing of a 4x4 double covariance: (xx, xy, xz, yy) and (yz, zz, 0, 0)
__device__ __forceinline__ float4 pack_covA(const double* c) { return make_float4((float)c[0], (float)c[1], (float)c[2], (float)c[5]); }
__device__ __forceinline__ float4 pack_covB(const double* c) { return make_float4((float)c[6], (float)c[10], 0.f, 0.f); }

/// The owner of position x in a prefix table of n owners: the largest o < n with prefix[o * STRIDE] <= x (prefix ascending,
/// prefix[0] <= x).  Owners of nothing (equal prefix entries) are skipped: x belongs to the next one that owns something.
template <uint32_t STRIDE = 1>
__device__ __forceinline__ uint32_t owner_of(const uint32_t* __restrict__ prefix, uint32_t n, uint32_t x) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1u) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(&prefix[mid * STRIDE]) <= x) lo = mid;
    else hi = mid;
  }
  return lo;
}

/// Non-finite input points (a NaN or +-Inf in x, y or z) are inert (sgicp_b200.h): they take no part in a cloud's box, and the store
/// writes them as NaN in all three lanes, so that no infinity survives centring.  A NaN point's squared distance to anything is NaN,
/// which no `d < best` accepts and whose bits order above every finite bound, so the searches never return one; leaf boxes leave it
/// out.  Its own query (NaN) is never searched: box_dist2 would be 0 for every box and nothing would prune the walk, so the grid probe
/// settles it without a correspondence, the tree walks run it as an idle lane and the k-NN returns before walking.
__device__ __forceinline__ bool point_is_finite(double x, double y, double z) { return isfinite(x) && isfinite(y) && isfinite(z); }
/// the stored (centred FP32) point: x - c in each lane, or NaN in all three for a non-finite input point
__device__ __forceinline__ float4 centred_store_point(const double4& p, double x, double y, double z, uint32_t w) {
  const bool ok = point_is_finite(p.x, p.y, p.z);
  return make_float4(ok ? (float)x : __int_as_float(0x7fffffff), ok ? (float)y : __int_as_float(0x7fffffff), ok ? (float)z : __int_as_float(0x7fffffff),
                     __int_as_float(static_cast<int>(w)));
}

/// One CTA of kBoxBlock threads over pts[first, last): the exact box into bounds[6] (unless null) and the centre [4] that centre_kernel
/// derives from it.  Min / max are exact, so both equal what the atomics of launch_bounds_centre give for these points alone.  Only
/// finite points count (point_is_finite).
constexpr int kBoxBlock = 256;
__device__ __forceinline__ void cta_box_centre(const double4* __restrict__ pts, uint32_t first, uint32_t last, double* bounds, double* centre) {
  __shared__ double s_red[kBoxBlock / 32][6];
  double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, hi[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
  for (uint32_t i = first + threadIdx.x; i < last; i += kBoxBlock) {
    const double4 p = pts[i];
    if (!point_is_finite(p.x, p.y, p.z)) continue;
    lo[0] = fmin(lo[0], p.x); lo[1] = fmin(lo[1], p.y); lo[2] = fmin(lo[2], p.z);
    hi[0] = fmax(hi[0], p.x); hi[1] = fmax(hi[1], p.y); hi[2] = fmax(hi[2], p.z);
  }
#pragma unroll
  for (int d = 0; d < 3; d++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[d] = fmin(lo[d], __shfl_down_sync(0xffffffffu, lo[d], o));
      hi[d] = fmax(hi[d], __shfl_down_sync(0xffffffffu, hi[d], o));
    }
  }
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (lane == 0) {
#pragma unroll
    for (int d = 0; d < 3; d++) {
      s_red[warp][d] = lo[d];
      s_red[warp][3 + d] = hi[d];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kBoxBlock / 32; w++) {
#pragma unroll
      for (int d = 0; d < 3; d++) {
        lo[d] = fmin(lo[d], s_red[w][d]);
        hi[d] = fmax(hi[d], s_red[w][3 + d]);
      }
    }
    double ext = 0.0;
    for (int d = 0; d < 3; d++) {
      if (bounds) {
        bounds[d] = lo[d];
        bounds[3 + d] = hi[d];
      }
      centre[d] = (lo[d] <= hi[d]) ? 0.5 * (lo[d] + hi[d]) : 0.0;
      ext = fmax(ext, hi[d] - lo[d]);
    }
    centre[3] = ext > 0.0 ? ext : 1.0;
  }
}

// ---------------------------------------------------------------------------------------------
// kd-tree construction, shared by the single tree (sgb_kernels.cu) and many trees at once (sgb_forest.cu): a tree over n points is the
// implicit balanced tree whose nodes at a level with `count` nodes own contiguous position ranges; its records are 64-byte packets.
// ---------------------------------------------------------------------------------------------
/// first point of node j at a level with `count` nodes (balanced implicit tree over n points)
__device__ __forceinline__ uint32_t tree_bound(uint32_t j, uint32_t count, uint32_t n) {
  return static_cast<uint32_t>((static_cast<uint64_t>(j) * n) / count);
}
/// node (at a level with `count` nodes) that owns position i
__device__ __forceinline__ uint32_t tree_node_of(uint32_t i, uint32_t count, uint32_t n) {
  return static_cast<uint32_t>(((static_cast<uint64_t>(i) + 1u) * count + n - 1u) / n) - 1u;
}

// boxes: count x 6 floats stored as order-preserving uints (lo xyz, hi xyz)
__device__ __forceinline__ uint32_t float_flip(float f) {
  const uint32_t u = __float_as_uint(f);
  return u ^ ((u >> 31) ? 0xFFFFFFFFu : 0x80000000u);
}
__device__ __forceinline__ float float_unflip(uint32_t u) { return __uint_as_float(u ^ ((u >> 31) ? 0x80000000u : 0xFFFFFFFFu)); }
/// a coordinate's contribution to the min / max words of a box: the empty box's word for NaN (a stored non-finite point), which
/// float_flip would order above +Inf (or below -Inf with its sign bit set)
__device__ __forceinline__ uint32_t box_lo_word(float f) { return isnan(f) ? 0xFFFFFFFFu : float_flip(f); }
__device__ __forceinline__ uint32_t box_hi_word(float f) { return isnan(f) ? 0u : float_flip(f); }

/// the child record of heap node child_heap (> 0) in its parent's packet: box [lo, hi], a | b in the w lanes
__device__ __forceinline__ void lbvh_store_child(float4* pnodes, uint32_t child_heap, const float lo[3], const float hi[3], uint32_t a, uint32_t b) {
  const uint32_t parent = (child_heap - 1u) >> 1, side = (child_heap & 1u) ? 0u : 1u;  // odd heap index = left child
  pnodes[parent * 4 + side * 2 + 0] = make_float4(lo[0], lo[1], lo[2], __uint_as_float(a));
  pnodes[parent * 4 + side * 2 + 1] = make_float4(hi[0], hi[1], hi[2], __uint_as_float(b));
}

/// The bounding box of a leaf slot's (at most 32) consecutive points pts[base + first, base + last), one per lane of the warp: lo / hi in
/// every lane (inverted for an empty slot, which no query enters).
__device__ __forceinline__ void lbvh_leaf_box(const float4* __restrict__ pts, uint32_t base, uint32_t first, uint32_t last, uint32_t lane, float lo[3], float hi[3]) {
  const uint32_t idx = first + lane;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    lo[a] = INFINITY;
    hi[a] = -INFINITY;
  }
  const float4 p = idx < last ? pts[base + idx] : make_float4(0.f, 0.f, 0.f, 0.f);
  if (idx < last && !isnan(p.x)) {  // a stored non-finite point (NaN in every lane) leaves the box as it is
    lo[0] = hi[0] = p.x;
    lo[1] = hi[1] = p.y;
    lo[2] = hi[2] = p.z;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int a = 0; a < 3; a++) {
      lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
      hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
    }
  }
}

/// inner node `node` whose children's records are complete: their union box -> the parent's child record (a = node index, b = 0)
__device__ __forceinline__ void lbvh_inner_record(float4* pnodes, uint32_t node) {
  const float4 l0 = pnodes[node * 4 + 0], l1 = pnodes[node * 4 + 1], r0 = pnodes[node * 4 + 2], r1 = pnodes[node * 4 + 3];
  const float lo[3] = {fminf(l0.x, r0.x), fminf(l0.y, r0.y), fminf(l0.z, r0.z)};
  const float hi[3] = {fmaxf(l1.x, r1.x), fmaxf(l1.y, r1.y), fmaxf(l1.z, r1.z)};
  lbvh_store_child(pnodes, node, lo, hi, node, 0u);
}

/// Shared-memory refinement: a node of at most kKdSegMax points, and at most kKdSegNodes nodes of it at one level, refined by one CTA.
constexpr uint32_t kKdSegMax = 2048;
constexpr uint32_t kKdSegNodes = 128;
/// its dynamic shared memory: two point buffers, the keys and slots of the sort, the boxes of one level
constexpr size_t kKdRefineSmem = 2 * kKdSegMax * sizeof(float4) + kKdSegMax * (sizeof(unsigned long long) + sizeof(uint32_t)) + kKdSegNodes * 6 * sizeof(uint32_t);

/// The median-split refinement of a whole SUBTREE of at most kKdSegMax points by one CTA: node b of level `level0` of a tree of `levels`
/// inner levels over the n points pts[0 .. n) (a contiguous position range) is loaded into shared memory and every remaining level runs
/// there -- per level: node boxes (shared-memory atomics on order-preserving integer images of the floats), key = (node, coordinate along
/// the node's widest axis), bitonic sort of (key, slot), permutation of the points.  The same keys and balanced position boundaries as one
/// radix sort per level (ties may land differently -- any order is a valid tree).  The points go back to pts; perm[base + k] receives
/// base + the w (original index within the tree) of the point at position k.
__device__ __forceinline__ void kd_refine_segment(float4* __restrict__ pts, uint32_t* __restrict__ perm, uint32_t base, uint32_t b, uint32_t n, uint32_t level0,
                                                  uint32_t levels) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  float4* s_pts = reinterpret_cast<float4*>(s_raw);                                            // [2][kKdSegMax]
  unsigned long long* s_key = reinterpret_cast<unsigned long long*>(s_raw + 2 * kKdSegMax * sizeof(float4));  // [kKdSegMax]
  uint32_t* s_idx = reinterpret_cast<uint32_t*>(s_key + kKdSegMax);                            // [kKdSegMax]
  uint32_t* s_box = s_idx + kKdSegMax;                                                         // [kKdSegNodes][6]
  const uint32_t tid = threadIdx.x;
  const uint32_t first = tree_bound(b, 1u << level0, n), last = tree_bound(b + 1u, 1u << level0, n), m = last - first;
  for (uint32_t t = tid; t < m; t += blockDim.x) s_pts[t] = pts[first + t];
  uint32_t cur = 0;
  __syncthreads();
  for (uint32_t level = level0; level < levels; level++) {
    const uint32_t count = 1u << level, node_first = b << (level - level0), n_nodes = 1u << (level - level0);
    for (uint32_t t = tid; t < n_nodes * 6u; t += blockDim.x) s_box[t] = (t % 6u) < 3u ? 0xFFFFFFFFu : 0u;
    __syncthreads();
    const float4* P0 = s_pts + cur * kKdSegMax;
    for (uint32_t t = tid; t < m; t += blockDim.x) {
      const float4 p = P0[t];
      uint32_t* bx = s_box + (tree_node_of(first + t, count, n) - node_first) * 6u;
      atomicMin(&bx[0], box_lo_word(p.x));
      atomicMin(&bx[1], box_lo_word(p.y));
      atomicMin(&bx[2], box_lo_word(p.z));
      atomicMax(&bx[3], box_hi_word(p.x));
      atomicMax(&bx[4], box_hi_word(p.y));
      atomicMax(&bx[5], box_hi_word(p.z));
    }
    __syncthreads();
    for (uint32_t t = tid; t < kKdSegMax; t += blockDim.x) {
      unsigned long long key = ~0ull;  // padding sorts to the end
      if (t < m) {
        const uint32_t node = tree_node_of(first + t, count, n) - node_first;
        const uint32_t* bx = s_box + node * 6u;
        const float ex = float_unflip(bx[3]) - float_unflip(bx[0]), ey = float_unflip(bx[4]) - float_unflip(bx[1]), ez = float_unflip(bx[5]) - float_unflip(bx[2]);
        const float4 p = P0[t];
        const float c = ex >= ey ? (ex >= ez ? p.x : p.z) : (ey >= ez ? p.y : p.z);
        key = (static_cast<unsigned long long>(node) << 32) | float_flip(c);
      }
      s_key[t] = key;
      s_idx[t] = t;
    }
    __syncthreads();
    // bitonic sort of (key, slot) over kKdSegMax entries: one compare-exchange per thread and step
    for (uint32_t k = 2; k <= kKdSegMax; k <<= 1) {
      for (uint32_t j = k >> 1; j > 0; j >>= 1) {
        for (uint32_t t = tid; t < kKdSegMax / 2u; t += blockDim.x) {
          const uint32_t lo = ((t & ~(j - 1u)) << 1) | (t & (j - 1u)), hi = lo | j;
          const bool up = (lo & k) == 0u;
          const unsigned long long a = s_key[lo], c = s_key[hi];
          if ((a > c) == up) {
            s_key[lo] = c;
            s_key[hi] = a;
            const uint32_t ia = s_idx[lo];
            s_idx[lo] = s_idx[hi];
            s_idx[hi] = ia;
          }
        }
        __syncthreads();
      }
    }
    float4* P1 = s_pts + (cur ^ 1u) * kKdSegMax;
    for (uint32_t t = tid; t < m; t += blockDim.x) P1[t] = P0[s_idx[t]];
    cur ^= 1u;
    __syncthreads();
  }
  const float4* Pf = s_pts + cur * kKdSegMax;
  for (uint32_t t = tid; t < m; t += blockDim.x) {
    const float4 p = Pf[t];
    pts[first + t] = p;
    perm[base + first + t] = base + static_cast<uint32_t>(__float_as_int(p.w));  // w carries the original index through every permutation
  }
}

// Sym3, the factor algebra and the per-point helpers live in sgb_math.cuh (also compiled for the host by tests/host_math).

/// Exact nearest neighbour of q in the flattened kd-tree (restates the visiting order of
/// UnsafeKdTree::knn_search, ann/kdtree.hpp:193-233, with an explicit stack of far children).
/// `best_d` enters as the search bound (only strictly closer points are accepted, knn_result.hpp:81-83).
/// stack: shared memory, entry (s, lane) at stack[s * kLinBlock + threadIdx.x].
__device__ __forceinline__ uint32_t kd_nearest(const KdNode* __restrict__ nodes, const float4* __restrict__ pts, float qx, float qy, float qz,
                                               float& best_d, uint32_t best, uint2* stack) {
  // `best` / `best_d` may enter seeded with a candidate (an upper bound only prunes: the result is still the
  // exact nearest neighbour, the seed wins only if nothing is strictly closer).
  uint32_t node = 0;
  int sp = 0;
  uint2* my_stack = stack + threadIdx.x;
  for (;;) {
    KdNode nd = __ldg(&nodes[node]);
    uint32_t kind = nd.y & 3u;
    while (kind != 3u) {  // descend; remember the far child only if the current bound does not already prune it
      const float qv = kind == 0u ? qx : (kind == 1u ? qy : qz);
      const float diff = qv - __uint_as_float(nd.x);
      const uint32_t right = nd.y >> 2, left = node + 1u;
      const bool go_left = diff < 0.0f;
      const float cut = diff * diff;
      if (cut < best_d) {
        my_stack[sp * kLinBlock] = make_uint2(go_left ? right : left, __float_as_uint(cut));
        sp++;
      }
      node = go_left ? left : right;
      nd = __ldg(&nodes[node]);
      kind = nd.y & 3u;
    }
    {  // leaf: scan its contiguous block of points
      const uint32_t first = nd.x, cnt = nd.y >> 2;
      const float4* lp = pts + first;
#pragma unroll 4
      for (uint32_t j = 0; j < cnt; j++) {
        const float4 t = __ldg(&lp[j]);
        const float dx = t.x - qx, dy = t.y - qy, dz = t.z - qz;
        const float d = dx * dx + dy * dy + dz * dz;
        if (d < best_d) {
          best_d = d;
          best = first + j;
        }
      }
    }
    // backtrack: nearest pending far child whose splitting plane is closer than the best distance
    bool found = false;
    while (sp > 0) {
      sp--;
      const uint2 e = my_stack[sp * kLinBlock];
      if (__uint_as_float(e.y) < best_d) {
        node = e.x;
        found = true;
        break;
      }
    }
    if (!found) break;
  }
  return best;
}

/// All-reduce(sum) of one value per thread (threads < NVALS of ONE CTA per rank) over the peer mailboxes -- see CommParams.
/// Called by ALL threads of the finishing CTA.  A rank whose peers never show up gives up after c.timeout_ns, returns NaN and
/// raises the context's sticky status word, which the host-facing calls turn into a non-zero return code (a hung collective
/// must not take the GPU down with it, and must not pass for a result either).
template <int NVALS>
__device__ __forceinline__ double comm_all_reduce(const CommParams& c, double v) {
  static_assert(NVALS <= kMailStride, "mailbox slot too small");
  const int tid = threadIdx.x;
  const size_t par = static_cast<size_t>(c.seq & 1ull);
  if (tid < NVALS) {
    for (int p = 0; p < c.world; p++)  // my sums -> slot (par, rank) of every rank's mailbox (remote stores over NVLink)
      reinterpret_cast<double*>(c.mail[p])[(par * kMaxPeers + c.rank) * kMailStride + tid] = v;
  }
  __threadfence_system();
  __syncthreads();
  __shared__ int s_fail;
  if (tid == 0) {
    s_fail = 0;
    if (c.stamps) c.stamps[c.seq % kCommStampRing] = 0ull;
  }
  __syncthreads();
  if (tid < c.world) {
    __threadfence_system();
    volatile unsigned long long* theirs = reinterpret_cast<volatile unsigned long long*>(c.mail[tid] + kMailFlagOffset) + par * kMaxPeers + c.rank;
    *theirs = c.poison ? (c.seq | kCommPoison) : c.seq;  // publish: rank `tid` may now read my slot
    volatile unsigned long long* mine = reinterpret_cast<volatile unsigned long long*>(c.mail[c.rank] + kMailFlagOffset) + par * kMaxPeers + tid;
    unsigned long long t0, t1 = 0, f;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    while (((f = *mine) & ~kCommPoison) != c.seq) {
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      if (t1 - t0 > c.timeout_ns) {
        atomicOr(&s_fail, 1);
        break;
      }
    }
    if (f == (c.seq | kCommPoison)) atomicOr(&s_fail, 2);
    // how long this rank waited for peer `tid` (its own flag is there at once): the slowest peer is the skew + transport,
    // the rank that arrives last sees the bare transport latency (bench.py: comm_wait_ns, min / max over the ranks)
    if (c.stamps) {
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      atomicMax(&c.stamps[c.seq % kCommStampRing], t1 - t0);
    }
  }
  __syncthreads();
  __threadfence_system();
  double s = 0.0;
  if (tid < NVALS) {
    const volatile double* slots = reinterpret_cast<const volatile double*>(c.mail[c.rank]) + par * kMaxPeers * kMailStride;
    for (int p = 0; p < c.world; p++) s += slots[p * kMailStride + tid];  // rank order: the same sum on every rank
    if (s_fail) s = __longlong_as_double(0x7ff8000000000000ll);
  }
  if (tid == 0 && s_fail && c.status) atomicOr(c.status, static_cast<unsigned int>(s_fail));
  return s;
}

/// Sum over the 32 lanes of a warp of N <= 32 values per lane (x[k]: this lane's term of sum k); lane k returns sum k (lanes >= N: 0).
/// The transposing butterfly of block_reduce_and_finish with the lane bits taken from the lowest: every aligned group of eight sums is
/// reduced over lane bits 0..2 (4 + 2 + 1 exchanges), which leaves one value per group and lane, and the (up to) four group values are
/// then reduced over lane bits 3 and 4 (2 + 1 exchanges).  For 29 sums that is 30 exchanges, as few as one butterfly over all of them,
/// but a group's terms are dead once the group is reduced: the compiler can produce and reduce the terms eight at a time.
/// The order of the additions is fixed by the lane numbers: deterministic.
template <int N>
__device__ __forceinline__ double warp_sum_transposed(const double* x) {
  static_assert(N <= 32, "one lane per sum");
  const int lane = threadIdx.x & 31;
  double g[4];
#pragma unroll
  for (int G = 0; G < 4; G++) {
    double v[8];
#pragma unroll
    for (int k = 0; k < 8; k++) v[k] = 8 * G + k < N ? x[8 * G + k] : 0.0;
#pragma unroll
    for (int w = 1; w <= 4; w <<= 1) {  // lane bit w: slots k and k + w (k a multiple of 2w) -> slot k, this lane's half kept
      const bool upper = (lane & w) != 0;
#pragma unroll
      for (int k = 0; k < 8; k += 2 * w) {
        if (8 * G + k >= N) continue;  // both halves are padding
        const double keep = upper ? v[k + w] : v[k];
        const double send = upper ? v[k] : v[k + w];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, w);
      }
    }
    g[G] = v[0];  // lane l: sum of slot 8 G + (l & 7) over the eight lanes l ^ 0..7
  }
#pragma unroll
  for (int w = 1; w <= 2; w <<= 1) {  // lane bits 3 and 4 over the group values (group k and k + w -> group k)
    const bool upper = (lane & (8 * w)) != 0;
#pragma unroll
    for (int k = 0; k < 4; k += 2 * w) {
      if (8 * k >= N) continue;
      const double keep = upper ? g[k + w] : g[k];
      const double send = upper ? g[k] : g[k + w];
      g[k] = keep + __shfl_xor_sync(0xffffffffu, send, 8 * w);
    }
  }
  return g[0];
}

/// CTAs per group of the two-level final reduction (see block_reduce_and_finish)
constexpr unsigned int kFinishGroup = 16;
/// doubles / tickets the reduction needs for a grid of `grid` CTAs
__host__ __device__ inline size_t reduction_partials_doubles(size_t grid) { return (grid + (grid + kFinishGroup - 1) / kFinishGroup) * kPartialStride; }
__host__ __device__ inline size_t reduction_tickets(size_t grid) { return 1 + (grid + kFinishGroup - 1) / kFinishGroup; }

/// Block-wide sum of per-thread accumulators -> partials[blockIdx.x].  The sums of all CTAs are then combined by a
/// two-level tree of tickets: the last CTA of every group of kFinishGroup consecutive CTAs adds that group's partials,
/// the last group to finish adds the group sums and writes the (expanded 44-double) result.  Each level is one batch of
/// independent L2 loads per lane -- a single CTA adding all gridDim.x partials keeps an otherwise idle GPU waiting.  The order of the additions depends on gridDim.x only: deterministic.
/// partials: reduction_partials_doubles(gridDim.x) doubles; ticket: reduction_tickets(gridDim.x) zeroed counters (left zeroed).
/// comm.world > 1: the finishing CTA then exchanges the sums with the other ranks (comm_all_reduce) before writing `out`.
/// tile_sum (sgb_batch.cu) is a copy of the CTA butterfly below: keep the two equal (sharing it changes this function's register allocation).
/// TRANSPOSED: the warps already hold their sums one per lane (acc[0] of lane k is the warp's sum k, e.g. from warp_sum_transposed): no butterfly.
template <int NACC, bool EXPAND, bool TRANSPOSED = false>
__device__ __forceinline__ void block_reduce_and_finish(double* acc, double* partials, unsigned int* ticket, double* out, const CommParams& comm) {
  static_assert(NACC <= 32, "one lane per accumulator");
  __shared__ double s_red[kLinBlock / 32][NACC];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (TRANSPOSED) {
    if (lane < NACC) s_red[warp][lane] = acc[0];
  } else if (NACC > 4) {
    // Transposing butterfly: at every step a lane keeps one half of the values it still owns and hands the other half to its partner,
    // so the 32 lanes end up with ONE fully reduced accumulator each (lane l holds sum l): 16 + 8 + 4 + 2 + 1 = 31 exchanges instead of
    // 5 per accumulator (145 for the 29 sums of linearize).  The order of
    // the additions is fixed by the lane numbers: deterministic.
    double v[32];
#pragma unroll
    for (int k = 0; k < 32; k++) v[k] = k < NACC ? acc[k] : 0.0;
#pragma unroll
    for (int w = 16; w >= 1; w >>= 1) {
      const bool upper = (lane & w) != 0;
#pragma unroll
      for (int k = 0; k < w; k++) {
        if (k >= NACC) continue;  // both halves are padding
        const double keep = upper ? v[k + w] : v[k];
        const double send = upper ? v[k] : v[k + w];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, w);
      }
    }
    if (lane < NACC) s_red[warp][lane] = v[0];
  } else {
#pragma unroll
    for (int k = 0; k < NACC; k++) {
      double v = acc[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
      if (lane == 0) s_red[warp][k] = v;
    }
  }
  __syncthreads();
  if (threadIdx.x < NACC) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < kLinBlock / 32; w++) v += s_red[w][threadIdx.x];
    partials[static_cast<size_t>(blockIdx.x) * kPartialStride + threadIdx.x] = v;
  }
  __threadfence();
  __syncthreads();
  const unsigned int group = blockIdx.x / kFinishGroup, n_groups = (gridDim.x + kFinishGroup - 1) / kFinishGroup;
  const unsigned int group_first = group * kFinishGroup;
  const unsigned int group_size = min(kFinishGroup, gridDim.x - group_first);
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(&ticket[1 + group], 1u);
    s_last = (t == group_size - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double* group_sums = partials + static_cast<size_t>(gridDim.x) * kPartialStride;
  if (threadIdx.x < NACC) {  // level 1: this group's CTAs, in CTA order
    double v = 0.0;
#pragma unroll
    for (unsigned int j = 0; j < kFinishGroup; j++)
      if (j < group_size) v += __ldcg(&partials[static_cast<size_t>(group_first + j) * kPartialStride + threadIdx.x]);
    group_sums[static_cast<size_t>(group) * kPartialStride + threadIdx.x] = v;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    ticket[1 + group] = 0u;  // ready for the next launch on this stream
    const unsigned int t = atomicAdd(&ticket[0], 1u);
    s_last = (t == n_groups - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (threadIdx.x == 0) ticket[0] = 0u;
  double v = 0.0;
  if (threadIdx.x < NACC) {  // level 2: the group sums, in group order
#pragma unroll 8
    for (unsigned int gI = 0; gI < n_groups; gI++) v += __ldcg(&group_sums[static_cast<size_t>(gI) * kPartialStride + threadIdx.x]);
  }
  if (comm.world > 1) v = comm_all_reduce<NACC>(comm, v);  // level 3: the other GPUs (fused exchange over peer memory)
  if (threadIdx.x < NACC) {
    if (!EXPAND) {
      out[threadIdx.x] = v;
    } else {
      // compact sum -> position(s) in H(6x6 row-major) | b | e | inliers (sgb_math.cuh)
      int p0, p1;
      if (expand_positions(threadIdx.x, p0, p1) == 2) out[p1] = v;
      out[p0] = v;
    }
  }
}

}  // namespace sgb
