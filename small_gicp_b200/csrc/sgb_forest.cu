// SPDX-License-Identifier: MIT
// Many kd-trees as ONE target of the batched calls (sgb_target_build_kdtrees; DESIGN.md §11 "Many trees"): member m is searched in map
// m's tree only.  Map m is stored as sgb_target_set_points + sgb_target_build_kdtree store it alone -- centred FP32 on its own box centre,
// w = index within the map, leaves of at most kLbvhLeafPoints points cut by median splits along the widest axis, 64-byte packet records
// -- and the maps are concatenated in map order: points and features in tgt_*, the record blocks in tgt_pnodes at per-map bases.
// Leaf records hold GLOBAL positions, so a correspondence is one position in tgt_pts as for a single tree.
//
// Build (launches depend on the size of the largest map only, never on the map count; no host synchronisation):
//   forest_centres_kernel       one CTA per map: box of its points -> centre, as launch_bounds_centre computes it for one cloud
//   forest_convert_kernel       centred FP32 points and packed features in original order (+ the first working copy of the points, and
//                               for feature estimation the FP32 rounding residuals)
//   forest_boxes_kernel / forest_keys_kernel   one radix level of every map whose nodes at that level still exceed kKdSegMax points;
//                               the caller sorts by (global node, coordinate along the node's widest axis) and re-gathers
//   forest_refine_smem_kernel   every (map, subtree of <= kKdSegMax points) segment refined in shared memory, one CTA each
//   forest_leaf_kernel / forest_level_kernel   the packet records of every map, one launch per tree level
// The refinement and the record kernels run the single tree's helpers and bodies (sgb_device.cuh) on each map's part of the arrays.
// Search:
//   forest_search_kernel        one CTA per BatchTile (128 consecutive stored points of ONE member): warp-cooperative exact nearest-
//                               neighbour walk over that member's map, as packet_search_kernel walks one tree; with SUBMAP, the same
//                               walk for submap members (sgb_source_set_submaps, DESIGN.md §11 "Submaps") over every map of the
//                               member's list, each in its own stored frame, the bound carried from map to map
// The same build over the preprocessing scratch serves sgb_estimate_features_batch (forest_features_kernel, sgb_preprocess.cu).
#include <algorithm>
#include <cfloat>

#include "sgb_batch.h"
#include "sgb_device.cuh"
#include "sgb_forest.h"
#include "sgb_kernels.h"

namespace sgb {

namespace {

/// the node of map-local position `local` at radix level `level` as a global box / key id: the first shared-memory segment it covers
/// (segments are map m's nodes at its level level0, numbered from seg_off[m]); ~0: the map is past its radix levels
__device__ __forceinline__ uint32_t forest_level_node(const ForestTables& F, uint32_t m, uint32_t local, uint32_t n, uint32_t level) {
  const uint32_t l0 = __ldg(&F.level0[m]);
  if (level >= l0) return ~0u;
  return __ldg(&F.seg_off[m]) + (tree_node_of(local, 1u << level, n) << (l0 - level));
}

// one CTA per map: the centre of its box
__global__ void __launch_bounds__(kBoxBlock) forest_centres_kernel(const double4* __restrict__ pts, const ForestTables F, double* centres) {
  const uint32_t m = blockIdx.x;
  cta_box_centre(pts, F.pt_off[m], F.pt_off[m + 1], nullptr, centres + 4 * static_cast<size_t>(m));
}

// raw (double AoS) -> centred float4 in original order (w = index within the map) and its working copy, features packed, perm = identity;
// out_lo (or null): what the rounding to FP32 dropped, convert_kernel's formula (sgb_kernels.cu)
__global__ void forest_convert_kernel(const double4* __restrict__ pts, const double4* __restrict__ normals, const double* __restrict__ covs, uint32_t n,
                                      const ForestTables F, const double* __restrict__ centres, float4* out_pts, float4* work_pts, float4* out_normals,
                                      float4* out_covA, float4* out_covB, uint32_t* perm, float4* out_lo) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t m = owner_of(F.pt_off, F.n_maps, i);
    const double* c = centres + 4 * static_cast<size_t>(m);
    const double4 p = pts[i];
    const double x = p.x - c[0], y = p.y - c[1], z = p.z - c[2];
    const float4 f = centred_store_point(p, x, y, z, i - F.pt_off[m]);
    out_pts[i] = f;
    work_pts[i] = f;
    perm[i] = i;
    if (out_lo) out_lo[i] = make_float4((float)(x - (double)(float)x), (float)(y - (double)(float)y), (float)(z - (double)(float)z), 0.f);
    if (normals) {
      const double4 nn = normals[i];
      out_normals[i] = make_float4((float)nn.x, (float)nn.y, (float)nn.z, 0.f);
    }
    if (covs) {
      const double* cv = covs + static_cast<size_t>(i) * 16;
      out_covA[i] = pack_covA(cv);
      out_covB[i] = pack_covB(cv);
    }
  }
}

__global__ void forest_boxes_init_kernel(uint32_t* boxes, uint32_t count) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < count * 6u) boxes[t] = (t % 6u) < 3u ? 0xFFFFFFFFu : 0u;
}

// node boxes of one radix level (the warp pre-reduction of kd_boxes_kernel in sgb_kernels.cu; a CTA here may span maps)
__global__ void forest_boxes_kernel(const float4* __restrict__ pts, uint32_t n, const ForestTables F, uint32_t level, uint32_t* boxes) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = i < n;
  const uint32_t idx = valid ? i : n - 1u;
  const uint32_t m = owner_of(F.pt_off, F.n_maps, idx), first = F.pt_off[m];
  const uint32_t node = forest_level_node(F, m, idx - first, F.pt_off[m + 1] - first, level);
  const float4 p = pts[idx];
  uint32_t v[6] = {box_lo_word(p.x), box_lo_word(p.y), box_lo_word(p.z), box_hi_word(p.x), box_hi_word(p.y), box_hi_word(p.z)};
  const uint32_t node0 = __shfl_sync(0xffffffffu, node, 0);
  if (__all_sync(0xffffffffu, node == node0)) {
    if (node0 == ~0u) return;
#pragma unroll
    for (int a = 0; a < 3; a++) {
      v[a] = __reduce_min_sync(0xffffffffu, v[a]);
      v[3 + a] = __reduce_max_sync(0xffffffffu, v[3 + a]);
    }
    if ((threadIdx.x & 31u) == 0) {
#pragma unroll
      for (int a = 0; a < 3; a++) {
        atomicMin(&boxes[node0 * 6 + a], v[a]);
        atomicMax(&boxes[node0 * 6 + 3 + a], v[3 + a]);
      }
    }
  } else if (valid && node != ~0u) {
#pragma unroll
    for (int a = 0; a < 3; a++) {
      atomicMin(&boxes[node * 6 + a], v[a]);
      atomicMax(&boxes[node * 6 + 3 + a], v[3 + a]);
    }
  }
}

// key = (global node << 32) | coordinate along the node's widest axis (as kd_keys_kernel in sgb_kernels.cu); a map past its radix levels
// keys all its points (its first segment << 32): the stable sort keeps their order and the maps stay in map order
__global__ void forest_keys_kernel(const float4* __restrict__ pts, uint32_t n, const ForestTables F, uint32_t level, const uint32_t* __restrict__ boxes,
                                   uint64_t* keys) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t m = owner_of(F.pt_off, F.n_maps, i), first = F.pt_off[m];
  const uint32_t node = forest_level_node(F, m, i - first, F.pt_off[m + 1] - first, level);
  if (node == ~0u) {
    keys[i] = static_cast<uint64_t>(F.seg_off[m]) << 32;
    return;
  }
  const float ex = float_unflip(boxes[node * 6 + 3]) - float_unflip(boxes[node * 6 + 0]);
  const float ey = float_unflip(boxes[node * 6 + 4]) - float_unflip(boxes[node * 6 + 1]);
  const float ez = float_unflip(boxes[node * 6 + 5]) - float_unflip(boxes[node * 6 + 2]);
  const float4 p = pts[i];
  const float c = ex >= ey ? (ex >= ez ? p.x : p.z) : (ey >= ez ? p.y : p.z);
  keys[i] = (static_cast<uint64_t>(node) << 32) | float_flip(c);
}

// kd_refine_smem_kernel over every map's segments: CTA b refines segment b - seg_off[m] of map m (a node of its level level0 with at
// most kKdSegMax points).  perm receives global original positions (the map's first position + w).
__global__ void __launch_bounds__(1024) forest_refine_smem_kernel(float4* __restrict__ leaf_pts, uint32_t* __restrict__ perm, const ForestTables F) {
  const uint32_t map = owner_of(F.seg_off, F.n_maps, blockIdx.x);
  const uint32_t b = blockIdx.x - F.seg_off[map], base = F.pt_off[map], n = F.pt_off[map + 1] - base;
  kd_refine_segment(leaf_pts + base, perm, base, b, n, F.level0[map], F.depth[map]);
}

// one warp per leaf slot of any map (lbvh_leaf_kernel in sgb_kernels.cu): the record in the map's record block, a = the leaf's first
// GLOBAL position
__global__ void forest_leaf_kernel(const float4* __restrict__ leaf_pts, const ForestTables F, uint32_t n_slots, float4* pnodes) {
  const uint32_t slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (slot >= n_slots) return;
  const uint32_t m = owner_of(F.slot_off, F.n_maps, slot);
  const uint32_t j = slot - F.slot_off[m], P = F.slot_off[m + 1] - F.slot_off[m];
  const uint32_t base = F.pt_off[m], n = F.pt_off[m + 1] - base;
  const uint32_t first = tree_bound(j, P, n), last = tree_bound(j + 1u, P, n);
  float lo[3], hi[3];
  lbvh_leaf_box(leaf_pts, base, first, last, lane, lo, hi);
  if (lane == 0) {
    const uint32_t cnt = last - first;
    lbvh_store_child(pnodes + 4 * static_cast<size_t>(F.node_base[m]), (P - 1u) + j, lo, hi, cnt ? base + first : 0u, cnt);
  }
}

// the inner nodes at `level` of every map that has that level (lbvh_level_kernel in sgb_kernels.cu)
__global__ void forest_level_kernel(const ForestTables F, uint32_t level, float4* pnodes) {
  const uint64_t total = static_cast<uint64_t>(F.n_maps) << level;
  for (uint64_t t = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; t < total; t += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint32_t m = static_cast<uint32_t>(t >> level);
    if (F.depth[m] <= level) continue;  // the map's inner levels are 0 .. depth - 1
    const uint32_t node = ((1u << level) - 1u) + static_cast<uint32_t>(t & ((1ull << level) - 1ull));
    lbvh_inner_record(pnodes + 4 * static_cast<size_t>(F.node_base[m]), node);
  }
}

// ---- search ----------------------------------------------------------------------------------------------------------------------
constexpr int kForestWarps = kLinBlock / 32;
constexpr int kForestDenseLanes = 18;  // as kPacketDenseLanes (sgb_kernels_packet.cu)
constexpr int kForestStack = 40;

// The FP32 query of stored point sp of member m in the stored frame of submap entry e: the member's pose carried through the inverse of
// the entry's placement, then centred on the entry's map as forest_search_kernel centres on map m.
__device__ __forceinline__ float3 submap_query(const SubmapView& S, uint32_t e, const BatchParams& B, uint32_t m, const float4& sp) {
  const double* cs = B.centres + 4 * static_cast<size_t>(m);
  double Tk[12];
  relative_pose(S.inv_poses + 12 * static_cast<size_t>(e), B.poses + 12 * static_cast<size_t>(m), Tk);
  const double3 tp = centred_translation(Tk, cs[0], cs[1], cs[2], S.centres + 4 * static_cast<size_t>(e));
  return centred_query_f32(Tk, tp, sp);
}

// One CTA per BatchTile: warp w takes the tile's points 32 w .. 32 w + 31, all of ONE member m, and walks map m's tree once for all of
// them -- the walk of packet_search_kernel (sgb_kernels_packet.cu): one shared stack, warp votes, warp-uniform node and leaf loads, the
// dense scan (every lane tests every point) or the sparse one (the whole warp serves one interested lane at a time).  Nothing of any
// other member enters a warp, so a member's correspondences depend on its own points, pose and seeds only.
// SUBMAP (submap members, sgb_source_set_submaps; F.pnodes = every map's records, F's tables unused): the same walk over the tree of
// every entry of the member's list in list order, each in its map's own stored frame.  Rigid placements preserve distances, so the
// nearest point of the placed union is the nearest over the entries, and best_d carried from entry to entry prunes the later trees: one
// that no lane's ball reaches costs its root record's two box tests.  Only a strictly nearer point replaces the best, so at an exact FP32
// tie between two entries the earlier one wins.  The seed is evaluated in the frame of the entry that owned it.  Without SUBMAP, S is
// not read.
// ROUND (a round of sgb_align_batch_async): the grid is sized for every tile, the round's tile count is read from the device and the CTAs
// beyond it (all of them in an error() round) exit at once.
template <bool ROUND, bool SUBMAP>
__global__ void __launch_bounds__(kLinBlock, SUBMAP ? 7 : 8) forest_search_kernel(const __grid_constant__ BatchParams B, const __grid_constant__ ForestView F,
                                                                                  float bound, uint32_t* __restrict__ vcorr, const BatchRound* __restrict__ round,
                                                                                  const __grid_constant__ SubmapView S) {
  if constexpr (ROUND) {
    const BatchRound r = *round;
    if (!r.lin || blockIdx.x >= r.n_tiles) return;
  }
  extern __shared__ float s_dist[];  // [max_depth][kLinBlock] per-lane box distance of each pending subtree
  __shared__ uint2 s_child[kForestWarps][kForestStack];
  const BatchTile t = B.tiles[blockIdx.x];
  const uint32_t lane = threadIdx.x & 31u, wib = threadIdx.x >> 5;
  if (wib * 32u >= t.count) return;  // warp-uniform; no CTA barrier below
  const uint32_t m = t.member;
  const bool valid = threadIdx.x < t.count;
  const uint32_t i = t.first + threadIdx.x, v = t.vfirst + threadIdx.x;
  const uint32_t e0 = SUBMAP ? __ldg(&S.entry_off[m]) : 0u, e1 = SUBMAP ? __ldg(&S.entry_off[m + 1]) : 1u;  // the member's entries
  if constexpr (!SUBMAP) {
    const uint32_t n_map = F.pt_off[m + 1] - F.pt_off[m];
    if (n_map == 0) {
      if (valid) vcorr[v] = kNone;
      return;
    }
  }
  const float4* __restrict__ pnodes = SUBMAP ? F.pnodes : F.pnodes + 4 * static_cast<size_t>(F.node_base[m]);
  const float4* __restrict__ pts = B.tgt.pts;
  float* my_dist = s_dist + threadIdx.x;
  uint2* my_child = s_child[wib];

  float fx = 0.f, fy = 0.f, fz = 0.f;
  float best_d = -1.0f;  // an idle lane is never interested in anything
  uint32_t best = kNone, best_e = 0;
  const float4 p = (SUBMAP && valid) ? __ldg(&B.pts[i]) : make_float4(0.f, 0.f, 0.f, 0.f);  // SUBMAP: the stored point
  if (valid) {
    if constexpr (!SUBMAP) {
      const double* R = B.poses + 12 * static_cast<size_t>(m);
      const double* cs = B.centres + 4 * static_cast<size_t>(m);
      const double3 tp = centred_translation(R, cs[0], cs[1], cs[2], F.centres + 4 * static_cast<size_t>(m));
      const float3 f = centred_query_f32(R, tp, __ldg(&B.pts[i]));
      fx = f.x;
      fy = f.y;
      fz = f.z;
    }
    best_d = isnan(SUBMAP ? p.x : fx) ? -1.0f : bound;  // a stored non-finite point (NaN query): no search, as an idle lane
    // the member's previous correspondence: an upper bound only prunes
    const uint32_t prev = (B.members[m].z & kMemberSeeded) ? B.corr[i] : kNone;
    if (prev != kNone) {
      uint32_t pe = 0;  // SUBMAP: the entry it lies in
      if constexpr (SUBMAP) {
        pe = S.centry[i];
        const float3 f = submap_query(S, e0 + pe, B, m, p);
        fx = f.x;
        fy = f.y;
        fz = f.z;
      }
      const float4 q = __ldg(&pts[prev]);
      const float dx = q.x - fx, dy = q.y - fy, dz = q.z - fz;
      const float d = dx * dx + dy * dy + dz * dz;
      if (d < best_d) {
        best_d = d;
        best = prev;
        best_e = pe;
      }
    }
  }

  // One walk per entry.  Without SUBMAP the loop condition is constant false, so no loop is emitted around the walk: a loop there, even
  // one that runs once, changes the code of the one-map-per-member search.
  uint32_t e = e0;
  if (e < e1) do {
    const float4* __restrict__ tree = pnodes;  // the records walked
    if constexpr (SUBMAP) {
      const uint4 ent = __ldg(&S.entries[e]);
      if (ent.y == 0u) continue;  // an empty map
      const float3 f = submap_query(S, e, B, m, p);
      fx = f.x;
      fy = f.y;
      fz = f.z;
      tree = pnodes + 4 * static_cast<size_t>(ent.z);
    }
    const float before = best_d;
    int sp = 0;
    uint32_t cur = 0;    // inner node being expanded (index within the map's record block)
    bool expand = true;  // false: nothing to expand, take the next pending subtree
    uint32_t leaf_first = 0, leaf_cnt = 0;
    float leaf_d = 0.f;
    for (;;) {
      if (expand) {
        const float4 n0 = __ldg(&tree[cur * 4 + 0]), n1 = __ldg(&tree[cur * 4 + 1]);
        const float4 n2 = __ldg(&tree[cur * 4 + 2]), n3 = __ldg(&tree[cur * 4 + 3]);
        const float dl = box_dist2(fx, fy, fz, n0, n1), dr = box_dist2(fx, fy, fz, n2, n3);
        const bool wl = dl < best_d, wr = dr < best_d;
        const unsigned ml = __ballot_sync(0xffffffffu, wl), mr = __ballot_sync(0xffffffffu, wr);
        uint32_t ca, cb;
        if (ml && mr) {
          const unsigned closer_l = __ballot_sync(0xffffffffu, (wl || wr) && dl <= dr);
          const bool left_first = 2 * __popc(closer_l) >= __popc(ml | mr);
          my_dist[sp * kLinBlock] = left_first ? dr : dl;
          if (lane == 0) my_child[sp] = left_first ? make_uint2(__float_as_uint(n2.w), __float_as_uint(n3.w)) : make_uint2(__float_as_uint(n0.w), __float_as_uint(n1.w));
          sp++;
          ca = left_first ? __float_as_uint(n0.w) : __float_as_uint(n2.w);
          cb = left_first ? __float_as_uint(n1.w) : __float_as_uint(n3.w);
          leaf_d = left_first ? dl : dr;
        } else if (ml) {
          ca = __float_as_uint(n0.w);
          cb = __float_as_uint(n1.w);
          leaf_d = dl;
        } else if (mr) {
          ca = __float_as_uint(n2.w);
          cb = __float_as_uint(n3.w);
          leaf_d = dr;
        } else {
          expand = false;
          continue;
        }
        if (cb == 0u) {  // inner child
          cur = ca;
          continue;
        }
        leaf_first = ca;
        leaf_cnt = cb;
      } else {
        bool got = false;
        uint2 c = make_uint2(0u, 0u);
        while (sp > 0) {
          sp--;
          const float d = my_dist[sp * kLinBlock];
          if (__any_sync(0xffffffffu, d < best_d)) {
            __syncwarp();  // lane 0's push of this entry is visible
            c = my_child[sp];
            __syncwarp();  // ... and every lane has read it before lane 0 may push over it
            leaf_d = d;
            got = true;
            break;
          }
        }
        if (!got) break;
        if (c.y == 0u) {
          cur = c.x;
          expand = true;
          continue;
        }
        leaf_first = c.x;
        leaf_cnt = c.y;
      }
      // ---- leaf (global positions) ----
      const unsigned want = __ballot_sync(0xffffffffu, leaf_d < best_d);
      if (__popc(want) > kForestDenseLanes) {
        const float4* lp = pts + leaf_first;
#pragma unroll 4
        for (uint32_t j = 0; j < leaf_cnt; j++) {
          const float4 q = __ldg(&lp[j]);
          const float dx = q.x - fx, dy = q.y - fy, dz = q.z - fz;
          const float d = dx * dx + dy * dy + dz * dz;
          if (d < best_d) {
            best_d = d;
            best = leaf_first + j;
          }
        }
      } else {
        for (uint32_t base = 0; base < leaf_cnt; base += 32u) {
          const uint32_t j = base + lane;
          float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
          if (j < leaf_cnt) q = __ldg(&pts[leaf_first + j]);
          unsigned todo = want;
          while (todo) {
            const int src = __ffs(todo) - 1;
            todo &= todo - 1;
            const float qx = __shfl_sync(0xffffffffu, fx, src), qy = __shfl_sync(0xffffffffu, fy, src), qz = __shfl_sync(0xffffffffu, fz, src);
            const float dx = q.x - qx, dy = q.y - qy, dz = q.z - qz;
            const uint32_t dbits = j < leaf_cnt ? __float_as_uint(dx * dx + dy * dy + dz * dz) : 0x7f800000u;
            const uint32_t dmin = __reduce_min_sync(0xffffffffu, dbits);
            const unsigned who = __ballot_sync(0xffffffffu, dbits == dmin);  // lowest lane = first point in scan order
            if (static_cast<int>(lane) == src) {
              const float d = __uint_as_float(dmin);
              if (d < best_d) {
                best_d = d;
                best = leaf_first + base + (__ffs(who) - 1);
              }
            }
          }
        }
      }
      expand = false;
    }
    if (best_d < before) best_e = e - e0;
    __syncwarp();
  } while (SUBMAP && ++e < e1);
  if (valid) {
    vcorr[v] = best;
    if constexpr (SUBMAP) S.centry[i] = best_e;
  }
}

}  // namespace

cudaError_t launch_forest_build(const ForestBuild& b, cudaStream_t st, int* launches) {
  const ForestTables& F = b.tables;
  int count = 0;
  const uint32_t n = b.n;
  forest_centres_kernel<<<F.n_maps, kBoxBlock, 0, st>>>(reinterpret_cast<const double4*>(b.points), F, b.centres);
  const uint32_t cgrid = std::min<uint32_t>((n + 255u) / 256u, static_cast<uint32_t>(b.sm_count) * 8u);
  forest_convert_kernel<<<cgrid, 256, 0, st>>>(reinterpret_cast<const double4*>(b.points), reinterpret_cast<const double4*>(b.normals), b.covs, n, F, b.centres,
                                               b.orig_pts, b.leaf_pts, b.orig_normals, b.orig_covA, b.orig_covB, b.perm, b.orig_lo);
  count += 2;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  // radix levels: every map whose nodes at this level still hold more than kKdSegMax points
  for (uint32_t level = 0; level < b.radix_levels; level++) {
    forest_boxes_init_kernel<<<(b.n_segments * 6u + 255u) / 256u, 256, 0, st>>>(b.boxes, b.n_segments);
    forest_boxes_kernel<<<(n + 255u) / 256u, 256, 0, st>>>(b.leaf_pts, n, F, level, b.boxes);
    forest_keys_kernel<<<(n + 255u) / 256u, 256, 0, st>>>(b.leaf_pts, n, F, level, b.boxes, b.keys_in);
    if ((e = cudaMemcpyAsync(b.vals_in, b.perm, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return e;
    size_t tb = b.sort_temp_bytes;
    if ((e = sort_pairs_u64_u32_bits(b.sort_temp, tb, b.keys_in, b.keys_out, b.vals_in, b.perm, n, b.key_bits, st)) != cudaSuccess) return e;
    if ((e = launch_gather(b.perm, n, b.orig_pts, b.leaf_pts, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, b.sm_count, st)) != cudaSuccess) return e;
    count += 6;
  }
  // every (map, segment) below: one CTA each
  if ((e = allow_dynamic_smem(forest_refine_smem_kernel, kKdRefineSmem)) != cudaSuccess) return e;
  forest_refine_smem_kernel<<<b.n_segments, 1024, kKdRefineSmem, st>>>(b.leaf_pts, b.perm, F);
  count += 1;
  if (b.orig_normals || b.orig_covA) {
    if ((e = launch_gather(b.perm, n, nullptr, nullptr, b.orig_normals, b.leaf_normals, b.orig_covA, b.leaf_covA, b.orig_covB, b.leaf_covB, b.sm_count, st)) !=
        cudaSuccess)
      return e;
    count += 1;
  }
  // records: the leaves, then one launch per inner level, deepest first (a map joins once the level is within its depth)
  forest_leaf_kernel<<<(b.n_slots + 7u) / 8u, 256, 0, st>>>(b.leaf_pts, F, b.n_slots, b.pnodes);
  count += 1;
  for (uint32_t level = b.max_depth - 1u; level >= 1u && level < b.max_depth; level--) {
    const uint64_t threads = static_cast<uint64_t>(F.n_maps) << level;
    const uint64_t g = std::min<uint64_t>((threads + 255u) / 256u, static_cast<uint64_t>(b.sm_count) * 16u);
    forest_level_kernel<<<static_cast<unsigned>(g), 256, 0, st>>>(F, level, b.pnodes);
    count += 1;
  }
  if (launches) *launches = count;
  return cudaGetLastError();
}

cudaError_t launch_forest_search(const BatchParams& B, const ForestView& F, const BatchRound* round, uint32_t n_tiles, int max_depth, float bound, uint32_t* vcorr,
                                 cudaStream_t st) {
  if (max_depth < 1 || max_depth > kForestStack) return cudaErrorInvalidValue;
  const size_t smem = static_cast<size_t>(max_depth) * kLinBlock * sizeof(float);
  if (round)
    forest_search_kernel<true, false><<<n_tiles, kLinBlock, smem, st>>>(B, F, bound, vcorr, round, SubmapView{});
  else
    forest_search_kernel<false, false><<<n_tiles, kLinBlock, smem, st>>>(B, F, bound, vcorr, nullptr, SubmapView{});
  return cudaGetLastError();
}

cudaError_t launch_submap_search(const BatchParams& B, const float4* pnodes, const SubmapView& S, const BatchRound* round, uint32_t n_tiles, int max_depth,
                                 float bound, uint32_t* vcorr, cudaStream_t st) {
  if (max_depth < 1 || max_depth > kForestStack) return cudaErrorInvalidValue;
  const size_t smem = static_cast<size_t>(max_depth) * kLinBlock * sizeof(float);
  const ForestView F{pnodes, nullptr, nullptr, nullptr};
  if (round)
    forest_search_kernel<true, true><<<n_tiles, kLinBlock, smem, st>>>(B, F, bound, vcorr, round, S);
  else
    forest_search_kernel<false, true><<<n_tiles, kLinBlock, smem, st>>>(B, F, bound, vcorr, nullptr, S);
  return cudaGetLastError();
}

}  // namespace sgb
