// SPDX-License-Identifier: MIT
// Batched registration (DESIGN.md §11): B source clouds ("members") against the one target of the context, each at its own pose.
//   batch_transform_kernel  member pose applied once per point: the FP32 query of every point of the active members (centred_query_f32,
//                           as in the single-source search kernels), written as a "virtual source" (target-centred, identity pose) that
//                           the single-source search kernels walk unchanged
//   batch_factor_kernel     one CTA per 128-point tile of ONE member: FP64 rejector + factor (or error()) at that member's pose, CTA sum
//                           -> one partial per tile.  Per target kind: the correspondence the search found (one point target, many
//                           kd-trees with member m centred on map m), the voxel-map probe for VGICP (vox_nearest, as in
//                           linearize_vox_kernel; many voxel maps: member m in map m's centre and table region), or submap members, each
//                           point at the member's pose relative to the placement of the entry its correspondence lies in; for the
//                           _points calls also each point's row of terms (BatchRows), and with weights in force each point's terms
//                           times its weight
//   weight_gather_kernel    sgb_source_set_weights: the caller's per-point weights into stored order, each checked finite and >= 0
//   batch_segment_kernel    one CTA per member: its tiles' partials in tile order -> H|b|e|inliers (or e) of that member
//   batch_step_kernel       batched align(): one thread per member, its Gauss-Newton / Levenberg-Marquardt step (sgb_math.cuh) after a
//                           round, its next pose and phase
//   pair_gather_kernel      sgb_source_set_pairs: every member's replica of its stored cloud, in one launch over all member points
//   pair_view_kernel        the many-maps tables above seen through the pairing (member p -> map maps[p]), one CTA
//   submap_view_kernel      the per-entry tables of the submap lists from the target's per-map tables, one thread per entry
//   joint_step_kernel       joint windows: one CTA per window, its system assembled from its edges' sums and solved, its state machine,
//                           its edges' next poses (sgb_align_joint; joint_align_init_kernel / joint_align_finish_kernel: the asynchronous
//                           call's set-up and outputs)
//   gnc_*_kernel            sgb_align_batch_gnc(_async): the largest residual of stage 0, each member's mu and last-stage decision, each
//                           point's GNC weight from its row of the reweighting linearize, each stage's align_init, the step with each
//                           member's stage iterations, each stage's phases, the loops' conditions and the outputs
//   joint_gnc_*_kernel      sgb_align_joint_gnc(_async): the same GNC with the window as its unit (each point's window through its edge),
//                           each window's stage start (joint_init), the joint step with each window's stage iterations, each stage's edge
//                           phases, the loops' conditions and the outputs
// The transform, factor, segment and step kernels serve the rounds the host plans (sgb_{linearize,error,align}_batch, sgb_align_joint) and,
// with ROUND / kModeRound, the rounds batch_plan_kernel plans on the device (sgb_align_batch_async, sgb_align_joint_async and both GNC
// aligns of each, whose rounds are all planned on the device).
// A member's sums depend on its own points, pose and correspondences only, added in an order fixed by its size: bit-identical whatever
// else is in the batch.
#include <algorithm>
#include <cfloat>

#include "sgb_batch.h"
#include "sgb_device.cuh"
#include "sgb_kernels.h"

namespace sgb {

// CTA sum of per-thread accumulators, thread k < NACC returns sum k: the transposing butterfly of block_reduce_and_finish
// (sgb_device.cuh), kept apart from it because inlining a shared helper there changed the register allocation of the
// single-source kernels.
template <int NACC>
__device__ __forceinline__ double tile_sum(const double* acc) {
  __shared__ double s_red[kLinBlock / 32][NACC];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (NACC > 4) {
    double v[32];
#pragma unroll
    for (int k = 0; k < 32; k++) v[k] = k < NACC ? acc[k] : 0.0;
#pragma unroll
    for (int w = 16; w >= 1; w >>= 1) {
      const bool upper = (lane & w) != 0;
#pragma unroll
      for (int k = 0; k < w; k++) {
        if (k >= NACC) continue;
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
  double v = 0.0;
  if (threadIdx.x < NACC) {
#pragma unroll
    for (int w = 0; w < kLinBlock / 32; w++) v += s_red[w][threadIdx.x];
  }
  return v;
}

// What the factor and segment kernels compute: a linearize or an error() round planned on the host, or a round planned on the device
// (either, as round->lin says).
constexpr int kModeLinearize = 0, kModeError = 1, kModeRound = 2;

// ROUND (every kernel below that has it): a round of sgb_align_batch_async, planned on the device -- the grid is sized for the worst
// case, the round's size is read from `round`, and the CTAs beyond it exit at once.
template <bool ROUND>
__global__ void __launch_bounds__(kLinBlock) batch_transform_kernel(const __grid_constant__ BatchParams B, float4* vq, uint32_t* vcorr,
                                                                    const BatchRound* __restrict__ round) {
  if constexpr (ROUND) {
    const BatchRound r = *round;
    if (!r.lin || blockIdx.x >= r.n_tiles) return;
  }
  const BatchTile t = B.tiles[blockIdx.x];
  const uint32_t tid = threadIdx.x;
  if (tid >= t.count) return;
  const uint32_t i = t.first + tid, v = t.vfirst + tid;
  const double* R = B.poses + 12 * static_cast<size_t>(t.member);
  const double* cs = B.centres + 4 * static_cast<size_t>(t.member);
  const double3 tp = centred_translation(R, cs[0], cs[1], cs[2], B.tgt.centre);
  const float3 f = centred_query_f32(R, tp, __ldg(&B.pts[i]));
  vq[v] = make_float4(f.x, f.y, f.z, 0.f);
  // the member's previous correspondence seeds the search (seeds only prune: the result does not depend on them)
  vcorr[v] = (B.members[t.member].z & kMemberSeeded) ? B.corr[i] : kNone;
}

// One tile of batch_factor_kernel.  ERR = false: linearize (VOX: voxel-map probe here; else vcorr = what the search found); ERR = true:
// error() with the cached corr[].  MAPS: a multi-map voxel target -- member m is centred on map m's centre (map_centres[4 m ..]) and
// probes map m's region of the table (map_regions[m]: first slot, mask); otherwise the target's one centre and table.
// SUB: submap members (S, sgb_source_set_submaps) -- the correspondence lies in entry S->centry[i] of the member's list, and the point is
// linearised at the member's pose relative to that entry's placement against the entry's map as stored.  r^T M r and its derivatives by
// the right perturbation of the pose are invariant under the placement, so this IS the point's share of the sums against the union.
// POINTS: the point's row too (rows).  A thread takes one point of the tile, so its acc is 0 + that point's terms: the very summands of
// the tile sum, written before it, whatever the kind (factor_terms_source or accumulate_factor); zeros where the point has no term.
// WEIGHTED: the point's terms (H | b | e, or its error()) times its weight rows->w[i] (sgb_source_set_weights), after the robust kernel and
// before its row and the tile sum; the inlier count stays as it is.
template <int FACTOR, int ROBUST, bool VOX, bool ERR, bool MAPS, bool SUB = false, bool POINTS = false, bool WEIGHTED = false>
__device__ __forceinline__ void batch_factor_tile(const BatchParams& B, const uint32_t* __restrict__ vcorr, const double* __restrict__ map_centres,
                                                  const uint4* __restrict__ map_regions, const SubmapView* S = nullptr, const BatchRows* rows = nullptr) {
  constexpr int NACC = ERR ? 1 : kAcc + 1;
  double acc[NACC];
#pragma unroll
  for (int k = 0; k < NACC; k++) acc[k] = 0.0;
  const BatchTile t = B.tiles[blockIdx.x];
  const uint32_t tid = threadIdx.x;
  if (tid < t.count) {
    const uint32_t i = t.first + tid;
    const double* R = B.poses + 12 * static_cast<size_t>(t.member);
    const double* cs = B.centres + 4 * static_cast<size_t>(t.member);
    const double csx = cs[0], csy = cs[1], csz = cs[2];
    const double* ct = MAPS ? map_centres + 4 * static_cast<size_t>(t.member) : B.tgt.centre;
    const double ctx = ct[0], cty = ct[1], ctz = ct[2];
    const double3 tp = centred_translation(R, csx, csy, csz, ct);
    const float4 sp = __ldg(&B.pts[i]);
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 sA = FACTOR == 2 ? __ldg(&B.covA[i]) : z, sB = FACTOR == 2 ? __ldg(&B.covB[i]) : z;
    if (SUB) {
      uint32_t k = ERR ? B.corr[i] : vcorr[t.vfirst + tid];
      if (k != kNone) {
        const size_t e = __ldg(&S->entry_off[t.member]) + S->centry[i];
        const double* Pinv = S->inv_poses + 12 * e;
        double Rk[12];
        relative_pose(Pinv, R, Rk);
        const double3 tk = centred_translation(Rk, csx, csy, csz, S->centres + 4 * e);
        const float4 tq = __ldg(&B.tgt.pts[k]);
        const float4 t1 = FACTOR == 2 ? __ldg(&B.tgt.covA[k]) : z, t2 = FACTOR == 2 ? __ldg(&B.tgt.covB[k]) : z;
        if (ERR) {
          double Rlin[12];  // the member's linearisation pose through the same placement
          relative_pose(Pinv, B.lin_poses + 12 * static_cast<size_t>(t.member), Rlin);
          acc[0] += point_error<FACTOR, ROBUST>(Rk, tk.x, tk.y, tk.z, Rlin, B.robust_c, sp, sA, sB, tq, t1, t2);
        } else if (!point_linearize_source<FACTOR, ROBUST>(Rk, tk.x, tk.y, tk.z, csx, csy, csz, B.max_dist_sq_d, B.robust_c, sp, &sA, &sB, tq, &t1, &t2, acc)) {
          k = kNone;  // rejected: error() and the correspondences must not see it
        }
      }
      if (!ERR) B.corr[i] = k;
    } else if (ERR) {
      const uint32_t k = B.corr[i];
      if (k != kNone) {
        const float4 tq = __ldg(&B.tgt.pts[k]);
        const float4 t1 = FACTOR == 1 ? __ldg(&B.tgt.normals[k]) : (FACTOR == 2 ? __ldg(&B.tgt.covA[k]) : z);
        const float4 t2 = FACTOR == 2 ? __ldg(&B.tgt.covB[k]) : z;
        // GICP: precision matrix re-derived from THIS member's linearisation pose (gicp_factor.hpp:81-89)
        acc[0] += point_error<FACTOR, ROBUST>(R, tp.x, tp.y, tp.z, B.lin_poses + 12 * static_cast<size_t>(t.member), B.robust_c, sp, sA, sB, tq, t1, t2);
      }
    } else if (VOX) {
      // linearize_vox_kernel's per-point work at this member's pose
      const double sx = sp.x, sy = sp.y, sz = sp.z;
      const double3 q = centred_query(R, tp, sp);
      double brx = 0, bry = 0, brz = 0;
      uint32_t best;
      if (MAPS) {
        // the single map's probe in map m's region of the table
        const uint4 r = map_regions[t.member];
        DevTarget map = B.tgt;
        map.vox_table += r.x;
        map.vox_mask = r.y;
        best = vox_nearest(map, q.x, q.y, q.z, ctx, cty, ctz, B.max_dist_sq_d, brx, bry, brz);
      } else {
        best = vox_nearest(B.tgt, q.x, q.y, q.z, ctx, cty, ctz, B.max_dist_sq_d, brx, bry, brz);
      }
      B.corr[i] = best;
      if (best != kNone) {
        Sym3 M;
        if (FACTOR == 2) {
          M = gicp_precision(R, sA, sB, __ldg(&B.tgt.covA[best]), __ldg(&B.tgt.covB[best]));
        } else {
          M = Sym3{1.0, 0.0, 0.0, 1.0, 0.0, 1.0};
        }
        accumulate_factor<ROBUST>(R, M, brx, bry, brz, csx + sx, csy + sy, csz + sz, B.robust_c, acc);
        acc[kAcc] += 1.0;
      }
    } else {
      // factor_reduce_kernel's per-point work at this member's pose
      uint32_t best = vcorr[t.vfirst + tid];
      if (best != kNone) {
        const float4 tq = __ldg(&B.tgt.pts[best]);
        const float4 t1 = FACTOR == 1 ? __ldg(&B.tgt.normals[best]) : (FACTOR == 2 ? __ldg(&B.tgt.covA[best]) : z);
        const float4 t2 = FACTOR == 2 ? __ldg(&B.tgt.covB[best]) : z;
        if (!point_linearize_source<FACTOR, ROBUST>(R, tp.x, tp.y, tp.z, csx, csy, csz, B.max_dist_sq_d, B.robust_c, sp, &sA, &sB, tq, &t1, &t2, acc))
          best = kNone;  // rejected: error() and the correspondences must not see it
      }
      B.corr[i] = best;
    }
    if constexpr (WEIGHTED) {
      const double w = __ldg(&rows->w[i]);
#pragma unroll
      for (int k = 0; k < (ERR ? 1 : kAcc); k++) acc[k] *= w;
    }
    if constexpr (POINTS) {
      const size_t row = batch_row(rows->member_off, rows->perm, t.member, i);
      if constexpr (ERR) {
        rows->e[row] = acc[0];
      } else {
        if (rows->e) rows->e[row] = acc[kAcc - 1];
        if (rows->Hb) {
          double* o = rows->Hb + 42 * row;
#pragma unroll
          for (int k = 0; k < kAcc - 1; k++) {
            int p0, p1;
            if (expand_positions(k, p0, p1) == 2) o[p1] = acc[k];
            o[p0] = acc[k];
          }
        }
      }
    }
  }
  const double v = tile_sum<NACC>(acc);
  if (tid < NACC) B.tile_partials[static_cast<size_t>(blockIdx.x) * kPartialStride + tid] = v;
}

// One CTA per tile of one member, for the target's KIND: 0 one point target, 1 one voxel map, 2 many voxel maps (member m against map m:
// map_centres and map_regions), 3 many kd-trees (map_centres; vcorr = what forest_search_kernel found in map m), 4 submaps (S; vcorr and
// S.centry = what forest_search_kernel<SUBMAP> found over the member's entries).  MODE: linearize, error() with the cached correspondences, or
// either as the round's planner decided.  POINTS: every processed point's row to `rows` too (in a round: the reweighting round of
// sgb_align_batch_gnc_async only).  WEIGHTED (any mode): each point's terms times its weight rows.w[i].
template <int FACTOR, int ROBUST, int KIND, int MODE, bool POINTS = false, bool WEIGHTED = false>
__global__ void __launch_bounds__(kLinBlock, 4) batch_factor_kernel(const __grid_constant__ BatchParams B, const uint32_t* __restrict__ vcorr,
                                                                   const double* __restrict__ map_centres, const uint4* __restrict__ map_regions,
                                                                   const __grid_constant__ SubmapView S, const BatchRound* __restrict__ round,
                                                                   const __grid_constant__ BatchRows rows) {
  constexpr bool VOX = KIND == 1 || KIND == 2, MAPS = KIND == 2 || KIND == 3, SUB = KIND == 4;
  bool lin = MODE == kModeLinearize;
  if constexpr (MODE == kModeRound) {
    const BatchRound r = *round;
    if (blockIdx.x >= r.n_tiles) return;
    lin = r.lin;
  }
  if (lin)
    batch_factor_tile<FACTOR, ROBUST, VOX, false, MAPS, SUB, POINTS, WEIGHTED>(B, vcorr, map_centres, map_regions, &S, &rows);
  else
    batch_factor_tile<FACTOR, ROBUST, VOX, true, MAPS, SUB, POINTS, WEIGHTED>(B, nullptr, map_centres, map_regions, &S, &rows);
}

// One CTA per member: warp w adds tiles w, w + 8, ... of the member in order, then the 8 warp sums are added in warp order.  The order
// depends on the member's tile count only.  Members without tiles (inactive or empty) get zeros.  LIN: the member's pose becomes its
// linearisation pose (read by later error() calls).
constexpr int kSegWarps = 8;
template <int NACC, bool LIN>
__device__ __forceinline__ void batch_segment(const BatchParams& B, double* out) {
  __shared__ double s_sum[kSegWarps][NACC];
  const uint32_t m = blockIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint4 mem = B.members[m];
  if (lane < static_cast<uint32_t>(NACC)) {
    double v = 0.0;
    for (uint32_t t = warp; t < mem.y; t += kSegWarps) v += __ldcg(&B.tile_partials[static_cast<size_t>(mem.x + t) * kPartialStride + lane]);
    s_sum[warp][lane] = v;
  }
  __syncthreads();
  if (threadIdx.x < static_cast<uint32_t>(NACC)) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < kSegWarps; w++) v += s_sum[w][threadIdx.x];
    if (LIN) {
      double* o = out + 44 * static_cast<size_t>(m);
      int p0, p1;
      if (expand_positions(threadIdx.x, p0, p1) == 2) o[p1] = v;
      o[p0] = v;
    } else {
      out[m] = v;
    }
  }
  if (LIN && (mem.z & kMemberActive) && threadIdx.x < 12) B.lin_poses[12 * static_cast<size_t>(m) + threadIdx.x] = B.poses[12 * static_cast<size_t>(m) + threadIdx.x];
}
template <int MODE>
__global__ void __launch_bounds__(kSegWarps * 32) batch_segment_kernel(const __grid_constant__ BatchParams B, double* out, const BatchRound* __restrict__ round) {
  if (MODE == kModeLinearize || (MODE == kModeRound && round->lin))
    batch_segment<kAcc + 1, true>(B, out);
  else
    batch_segment<1, false>(B, out);
}

// One thread per member: the step is a sequential 6x6 solve and a few 4x4 products (about 2k FP64 operations), and at the 65536-member
// limit that is 512 CTAs of 128 threads.  The state stays in global memory; only the solve's matrix is copied (to local memory: the
// pivot indexes it at run time).
constexpr int kStepBlock = 128;
__device__ __forceinline__ void batch_step_member(const AlignOptions& o, uint32_t m, bool linearize, const double* __restrict__ out,
                                                  MemberState* __restrict__ state, double* __restrict__ poses, uint8_t* __restrict__ phase) {
  MemberState& s = state[m];
  if (linearize && s.phase == kPhaseLinearize)
    align_after_linearize(o, s, out + 44 * static_cast<size_t>(m));
  else if (!linearize && s.phase == kPhaseTrial)
    align_after_error(o, s, out[m]);
  const double* T = s.phase == kPhaseTrial ? s.cand : s.T;
  double* p = poses + 12 * static_cast<size_t>(m);
  for (int i = 0; i < 3; i++) {  // pose_from_colmajor
    for (int j = 0; j < 3; j++) p[i * 3 + j] = T[j * 4 + i];
    p[9 + i] = T[12 + i];
  }
  phase[m] = static_cast<uint8_t>(s.phase);
}
// ROUND: the loop's condition becomes 1 if any member still has a round to go
template <bool ROUND>
__global__ void __launch_bounds__(kStepBlock) batch_step_kernel(const __grid_constant__ AlignOptions o, uint32_t n_members, bool linearize,
                                                                const double* __restrict__ out, MemberState* __restrict__ state,
                                                                double* __restrict__ poses, uint8_t* __restrict__ phase, const BatchRound* __restrict__ round,
                                                                cudaGraphConditionalHandle loop) {
  const uint32_t m = blockIdx.x * kStepBlock + threadIdx.x;
  if constexpr (ROUND) {
    int more = 0;
    if (m < n_members) {
      batch_step_member(o, m, round->lin != 0u, out, state, poses, phase);
      more = phase[m] == kPhaseLinearize || phase[m] == kPhaseTrial;
    }
    if (__syncthreads_or(more) && threadIdx.x == 0) cudaGraphSetConditional(loop, 1u);
  } else {
    if (m >= n_members) return;
    batch_step_member(o, m, linearize, out, state, poses, phase);
  }
}

cudaError_t launch_batch_step(const AlignOptions& o, uint32_t n_members, bool linearize, const BatchRound* round, cudaGraphConditionalHandle loop,
                              const double* out, MemberState* state, double* poses, uint8_t* phase, cudaStream_t st) {
  const uint32_t grid = (n_members + kStepBlock - 1) / kStepBlock;
  if (round)
    batch_step_kernel<true><<<grid, kStepBlock, 0, st>>>(o, n_members, linearize, out, state, poses, phase, round, loop);
  else
    batch_step_kernel<false><<<grid, kStepBlock, 0, st>>>(o, n_members, linearize, out, state, poses, phase, nullptr, loop);
  return cudaGetLastError();
}

// Pair members: member p is a replica of stored cloud clouds[p].  Positions 0 .. n - 1 copy the member points (FP32 point, packed
// covariance, search order -> original index), the next 10 P the member's centre [4] and bounds [6].
__global__ void pair_gather_kernel(const PairGather g) {
  const uint32_t total = g.n + 10u * g.n_members;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    if (i < g.n) {
      const uint32_t p = owner_of(g.member_off, g.n_members, i);
      const uint32_t s = g.cloud_off[g.clouds[p]] + (i - g.member_off[p]);
      g.out_pts[i] = g.pts[s];
      g.out_perm[i] = g.perm[s];
      if (g.covA) {
        g.out_covA[i] = g.covA[s];
        g.out_covB[i] = g.covB[s];
      }
    } else {
      const uint32_t k = i - g.n, p = k / 10u, j = k % 10u, c = g.clouds[p];
      if (j < 4u) g.out_centres[4 * static_cast<size_t>(p) + j] = g.centres[4 * static_cast<size_t>(c) + j];
      else g.out_bounds[6 * static_cast<size_t>(p) + j - 4u] = g.bounds[6 * static_cast<size_t>(c) + j - 4u];
    }
  }
}

// The per-member view of a many-maps target, one CTA: member p reads map maps[p].  Many kd-trees: pt_off = the prefix sum of the members'
// map sizes (the search reads only pt_off[p + 1] - pt_off[p], so the sum may wrap around 2^32: every map is below 2^30 points),
// node_base[p], centres[p].  Voxel maps: centres[p], regions[p].
constexpr int kViewBlock = 1024;
__global__ void __launch_bounds__(kViewBlock) pair_view_kernel(const PairView v) {
  __shared__ uint32_t s_warp[kViewBlock / 32];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t carry = 0;
  for (uint32_t base = 0; base < v.n_members; base += kViewBlock) {
    const uint32_t p = base + threadIdx.x;
    uint32_t size = 0;
    if (p < v.n_members) {
      const uint32_t q = v.maps[p];
      for (int d = 0; d < 4; d++) v.centres[4 * static_cast<size_t>(p) + d] = v.map_centres[4 * static_cast<size_t>(q) + d];
      if (v.map_pt_off) {
        size = v.map_pt_off[q + 1] - v.map_pt_off[q];
        v.node_base[p] = v.map_node_base[q];
      }
      if (v.map_regions) v.regions[p] = v.map_regions[q];
    }
    if (!v.map_pt_off) continue;
    // CTA exclusive scan of the sizes: within each warp, then over the warp totals
    uint32_t incl = size;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= static_cast<uint32_t>(o)) incl += y;
    }
    if (lane == 31u) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = s_warp[lane], wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= static_cast<uint32_t>(o)) wi += y;
      }
      s_warp[lane] = wi - w;  // exclusive prefix of the warp totals
    }
    __syncthreads();
    if (p < v.n_members) v.pt_off[p] = carry + s_warp[warp] + incl - size;
    const uint32_t chunk = __shfl_sync(0xffffffffu, incl, 31) + s_warp[warp];  // the last warp's view of the chunk total
    __syncthreads();  // s_warp is reused by the next chunk
    if (warp == kViewBlock / 32 - 1) s_warp[0] = chunk;
    __syncthreads();
    carry += s_warp[0];
    __syncthreads();
  }
  if (v.map_pt_off && threadIdx.x == 0) v.pt_off[v.n_members] = carry;
}

// Submap entries seen through the target's per-map tables: entry j -> map entry_maps[j], one thread per entry.
__global__ void submap_view_kernel(const SubmapViewBuild v) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < v.n_entries; j += gridDim.x * blockDim.x) {
    const uint32_t q = v.entry_maps[j], first = v.map_pt_off[q];
    v.entries[j] = make_uint4(first, v.map_pt_off[q + 1] - first, v.map_node_base[q], q);
    for (int d = 0; d < 4; d++) v.centres[4 * static_cast<size_t>(j) + d] = v.map_centres[4 * static_cast<size_t>(q) + d];
  }
}

// correspondences of a submap member in the caller's order: out[perm[i]] = (entry << 32) | original index within the entry's map
__global__ void submap_correspondences_kernel(const uint32_t* __restrict__ corr, const uint32_t* __restrict__ centry, const uint32_t* __restrict__ perm, size_t n,
                                              const float4* __restrict__ tgt_pts, uint64_t* out) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const uint32_t k = corr[i];
    out[perm[i]] = k == kNone ? ~0ull : (static_cast<uint64_t>(centry[i]) << 32) | static_cast<uint32_t>(__float_as_int(tgt_pts[k].w));
  }
}

cudaError_t launch_pair_gather(const PairGather& g, int sm_count, cudaStream_t st) {
  const uint64_t total = g.n + 10ull * g.n_members;
  if (total == 0) return cudaSuccess;
  const uint64_t grid = std::min<uint64_t>((total + 255u) / 256u, static_cast<uint64_t>(sm_count) * 8u);
  pair_gather_kernel<<<static_cast<unsigned>(grid), 256, 0, st>>>(g);
  return cudaGetLastError();
}

cudaError_t launch_pair_view(const PairView& v, cudaStream_t st) {
  pair_view_kernel<<<1, kViewBlock, 0, st>>>(v);
  return cudaGetLastError();
}

cudaError_t launch_batch_transform(const BatchParams& B, const BatchRound* round, uint32_t n_tiles, float4* vq, uint32_t* vcorr, cudaStream_t st) {
  if (round)
    batch_transform_kernel<true><<<n_tiles, kLinBlock, 0, st>>>(B, vq, vcorr, round);
  else
    batch_transform_kernel<false><<<n_tiles, kLinBlock, 0, st>>>(B, vq, vcorr, nullptr);
  return cudaGetLastError();
}

// The factor kernel of one kind in one mode.  The kinds without point-to-plane (1, 2, 4: refused by the caller) compile FACTOR 1 as 0, one
// instantiation fewer each.  error() reads the cached correspondences only, so the voxel kinds compute what the kinds with the same
// centres compute there (1 -> 0, 2 -> 3).
template <int F, int R, int MODE, bool POINTS = false, bool WEIGHTED = false>
auto factor_kernel(int kind) -> decltype(&batch_factor_kernel<0, 0, 0, kModeLinearize>) {
  constexpr int G = F == 1 ? 0 : F;
  switch (kind) {
    case 0: return batch_factor_kernel<F, R, 0, MODE, POINTS, WEIGHTED>;
    case 1: if constexpr (MODE == kModeError) return batch_factor_kernel<G, R, 0, MODE, POINTS, WEIGHTED>; else return batch_factor_kernel<G, R, 1, MODE, POINTS, WEIGHTED>;
    case 2: if constexpr (MODE == kModeError) return batch_factor_kernel<G, R, 3, MODE, POINTS, WEIGHTED>; else return batch_factor_kernel<G, R, 2, MODE, POINTS, WEIGHTED>;
    case 3: return batch_factor_kernel<F, R, 3, MODE, POINTS, WEIGHTED>;
    case 4: return batch_factor_kernel<G, R, 4, MODE, POINTS, WEIGHTED>;
    default: return nullptr;
  }
}

// the factor kernel of one kind for a round (device-planned), or for a host-planned mode with or without rows.  A device-planned round
// with rows is the reweighting round of sgb_align_batch_gnc_async: unweighted, no robust kernel (GNC refuses one), its e rows wanted.
template <int F, int R, bool WEIGHTED>
auto factor_kernel(int kind, bool err, bool round, bool rows) -> decltype(&batch_factor_kernel<0, 0, 0, kModeLinearize>) {
  if (round && rows) {
    if constexpr (R == 0 && !WEIGHTED) return factor_kernel<F, R, kModeRound, true, false>(kind);
    else return nullptr;
  }
  if (rows) return err ? factor_kernel<F, R, kModeError, true, WEIGHTED>(kind) : factor_kernel<F, R, kModeLinearize, true, WEIGHTED>(kind);
  return round ? factor_kernel<F, R, kModeRound, false, WEIGHTED>(kind) : err ? factor_kernel<F, R, kModeError, false, WEIGHTED>(kind)
                                                                               : factor_kernel<F, R, kModeLinearize, false, WEIGHTED>(kind);
}

cudaError_t launch_batch_factor(const BatchParams& B, int kind, int factor, int robust, bool err, const BatchRound* round, uint32_t n_tiles, const uint32_t* vcorr,
                                const double* map_centres, const uint4* map_regions, const SubmapView& S, const BatchRows* rows, const double* weights,
                                cudaStream_t st) {
  if (factor == 1 && (kind == 1 || kind == 2 || kind == 4)) return cudaErrorInvalidValue;  // no normals in a voxel map; no point-to-plane against a union
  const auto kernel = dispatch_factor_robust(factor, robust, decltype(&batch_factor_kernel<0, 0, 0, kModeLinearize>){}, [&](auto f, auto r) {
    return weights ? factor_kernel<f, r, true>(kind, err, round, rows) : factor_kernel<f, r, false>(kind, err, round, rows);
  });
  if (!kernel) return cudaErrorInvalidValue;
  BatchRows R = rows ? *rows : BatchRows{};
  R.w = weights;
  kernel<<<n_tiles, kLinBlock, 0, st>>>(B, vcorr, map_centres, map_regions, S, round, R);
  return cudaGetLastError();
}

// One thread per stored point: its weight fetched from the caller's row (batch_row, as the POINTS row write) and checked
__global__ void weight_gather_kernel(const WeightGather g) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += gridDim.x * blockDim.x) {
    const uint32_t m = owner_of(g.member_off, g.n_members, i);
    const size_t row = batch_row(g.member_off, g.perm, m, i);
    const double w = g.src[row];
    g.dst[i] = w;
    if (!(w >= 0.0 && w <= DBL_MAX)) atomicMin(g.bad, static_cast<uint32_t>(row));  // NaN, negative or infinite (-0.0 passes)
  }
}

cudaError_t launch_weight_gather(const WeightGather& g, int sm_count, cudaStream_t st) {
  if (g.n == 0) return cudaSuccess;
  const uint32_t grid = std::min<uint32_t>((g.n + 255u) / 256u, static_cast<uint32_t>(sm_count) * 8u);
  weight_gather_kernel<<<grid, 256, 0, st>>>(g);
  return cudaGetLastError();
}

cudaError_t launch_submap_view(const SubmapViewBuild& v, int sm_count, cudaStream_t st) {
  if (v.n_entries == 0) return cudaSuccess;
  const uint32_t grid = std::min<uint32_t>((v.n_entries + 255u) / 256u, static_cast<uint32_t>(sm_count) * 8u);
  submap_view_kernel<<<grid, 256, 0, st>>>(v);
  return cudaGetLastError();
}

cudaError_t launch_submap_correspondences(const uint32_t* corr, const uint32_t* centry, const uint32_t* perm, size_t n, const float4* tgt_pts, uint64_t* out,
                                          int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  const size_t grid = std::min<size_t>((n + 255u) / 256u, static_cast<size_t>(sm_count) * 8u);
  submap_correspondences_kernel<<<static_cast<unsigned>(grid), 256, 0, st>>>(corr, centry, perm, n, tgt_pts, out);
  return cudaGetLastError();
}

cudaError_t launch_batch_segment(const BatchParams& B, uint32_t n_members, bool linearize, const BatchRound* round, double* out, cudaStream_t st) {
  if (round)
    batch_segment_kernel<kModeRound><<<n_members, kSegWarps * 32, 0, st>>>(B, out, round);
  else if (linearize)
    batch_segment_kernel<kModeLinearize><<<n_members, kSegWarps * 32, 0, st>>>(B, out, nullptr);
  else
    batch_segment_kernel<kModeError><<<n_members, kSegWarps * 32, 0, st>>>(B, out, nullptr);
  return cudaGetLastError();
}

// ---- sgb_align_batch_async: the rounds planned and sized on the device (DESIGN.md §11 "Asynchronous align") ----

// The head of a round, one CTA: the host loop's rule (an error() round while any member has a pending trial, else a linearize round of
// the members still iterating) and batch_tables' tables in the same order -- members in member order, each active non-empty member's
// points in tiles of kLinBlock, the virtual source concatenating the active members -- then the round's sizes.  Members are taken
// 1024 at a time: a CTA scan of the (tile, point) counts, then the chunk's tiles written by all threads (binary search for the owner).
constexpr int kPlanBlock = 1024;
__global__ void __launch_bounds__(kPlanBlock) batch_plan_kernel(const BatchPlan p) {
  __shared__ uint32_t s_wt[32], s_wv[32], s_tot[2];
  __shared__ uint32_t s_end[kPlanBlock], s_first[kPlanBlock], s_n[kPlanBlock], s_v0[kPlanBlock];
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  if (tid == 0) cudaGraphSetConditional(p.loop, 0u);
  for (int k = 0; k < 3; k++)
    if (p.zero[k])
      for (uint32_t j = tid; j < p.zero_n[k]; j += kPlanBlock) p.zero[k][j] = 0u;
  int trial = 0;
  for (uint32_t m = tid; m < p.n_members; m += kPlanBlock) trial |= p.phase[m] == kPhaseTrial;
  const bool lin = !__syncthreads_or(trial);
  const uint8_t want = lin ? kPhaseLinearize : kPhaseTrial;
  uint32_t carry_t = 0, carry_v = 0;
  for (uint32_t base = 0; base < p.n_members; base += kPlanBlock) {
    const uint32_t m = base + tid;
    bool act = false;
    uint32_t first = 0, n = 0;
    if (m < p.n_members) {
      act = p.phase[m] == want;
      first = p.member_off[m];
      n = p.member_off[m + 1] - first;
    }
    const uint32_t nt = act ? (n + kLinBlock - 1u) / kLinBlock : 0u, nv = act ? n : 0u;
    uint32_t it = nt, iv = nv;  // inclusive scan within the warp, then over the warp totals
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t yt = __shfl_up_sync(0xffffffffu, it, o), yv = __shfl_up_sync(0xffffffffu, iv, o);
      if (lane >= static_cast<uint32_t>(o)) {
        it += yt;
        iv += yv;
      }
    }
    if (lane == 31u) {
      s_wt[warp] = it;
      s_wv[warp] = iv;
    }
    __syncthreads();
    if (warp == 0) {
      const uint32_t wt = s_wt[lane], wv = s_wv[lane];
      uint32_t at = wt, av = wv;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t yt = __shfl_up_sync(0xffffffffu, at, o), yv = __shfl_up_sync(0xffffffffu, av, o);
        if (lane >= static_cast<uint32_t>(o)) {
          at += yt;
          av += yv;
        }
      }
      s_wt[lane] = at - wt;
      s_wv[lane] = av - wv;
      if (lane == 31u) {
        s_tot[0] = at;
        s_tot[1] = av;
      }
    }
    __syncthreads();
    const uint32_t et = s_wt[warp] + it - nt, ev = s_wv[warp] + iv - nv;  // exclusive within the chunk
    if (m < p.n_members) {
      const bool seeded = lin && p.seeds && p.seeded[m];
      p.members[m] = p.no_target ? make_uint4(0u, 0u, lin && act ? kMemberActive : 0u, 0u)
                                 : make_uint4(carry_t + et, nt, (act ? kMemberActive : 0u) | (seeded ? kMemberSeeded : 0u), 0u);
      if (lin && act) p.seeded[m] = 1;  // its correspondences are cached by this round
    }
    s_end[tid] = et + nt;
    s_first[tid] = first;
    s_n[tid] = n;
    s_v0[tid] = carry_v + ev;
    __syncthreads();
    const uint32_t tot_t = s_tot[0], tot_v = s_tot[1];
    for (uint32_t k = tid; k < tot_t; k += kPlanBlock) {
      uint32_t lo = 0, hi = kPlanBlock - 1;  // the owner: the first j with s_end[j] > k
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (s_end[mid] > k) hi = mid;
        else lo = mid + 1;
      }
      const uint32_t j = (k - (lo ? s_end[lo - 1] : 0u)) * kLinBlock;
      p.tiles[carry_t + k] = BatchTile{base + lo, s_first[lo] + j, min(static_cast<uint32_t>(kLinBlock), s_n[lo] - j), s_v0[lo] + j};
    }
    carry_t += tot_t;
    carry_v += tot_v;
    __syncthreads();  // the shared tables are reused by the next chunk
  }
  if (tid == 0) *p.round = BatchRound{lin ? 1u : 0u, p.no_target ? 0u : carry_t, lin && !p.no_target ? carry_v : 0u, lin && p.no_target ? carry_t : 0u};
}

// a linearize round against an empty target: every point of the active members is left without a correspondence
__global__ void __launch_bounds__(kLinBlock) batch_unmatch_kernel(const __grid_constant__ BatchParams B, const BatchRound* __restrict__ round) {
  if (blockIdx.x >= round->n_clear) return;
  const BatchTile t = B.tiles[blockIdx.x];
  if (threadIdx.x < t.count) B.corr[t.first + threadIdx.x] = kNone;
}

__global__ void __launch_bounds__(kStepBlock) batch_align_init_kernel(const __grid_constant__ AlignOptions o, uint32_t n_members, const double* __restrict__ init_T16,
                                                                      MemberState* __restrict__ state, double* __restrict__ poses, uint8_t* __restrict__ phase,
                                                                      uint8_t* __restrict__ seeded, int keep_seeds) {
  const uint32_t m = blockIdx.x * kStepBlock + threadIdx.x;
  if (m >= n_members) return;
  const double* T = init_T16 + 16 * static_cast<size_t>(m);
  align_init(o, T, state[m]);
  double* p = poses + 12 * static_cast<size_t>(m);
  for (int i = 0; i < 3; i++) {  // pose_from_colmajor
    for (int j = 0; j < 3; j++) p[i * 3 + j] = T[j * 4 + i];
    p[9 + i] = T[12 + i];
  }
  phase[m] = static_cast<uint8_t>(state[m].phase);
  if (!keep_seeds) seeded[m] = 0;
}

__global__ void __launch_bounds__(kStepBlock) batch_align_finish_kernel(uint32_t n_members, const MemberState* __restrict__ state, double* __restrict__ out_T16,
                                                                        double* __restrict__ out_info4, double* __restrict__ out_Hb42) {
  const uint32_t m = blockIdx.x * kStepBlock + threadIdx.x;
  if (m >= n_members) return;
  const MemberState& s = state[m];
  for (int i = 0; i < 16; i++) out_T16[16 * static_cast<size_t>(m) + i] = s.T[i];
  double* info = out_info4 + 4 * static_cast<size_t>(m);
  info[0] = s.converged ? 1.0 : 0.0;
  info[1] = s.iterations;
  info[2] = s.inliers;
  info[3] = s.e;
  if (out_Hb42) {
    double* hb = out_Hb42 + 42 * static_cast<size_t>(m);
    for (int i = 0; i < 36; i++) hb[i] = s.H[i];
    for (int i = 0; i < 6; i++) hb[36 + i] = s.b[i];
  }
}

cudaError_t launch_batch_plan(const BatchPlan& p, cudaStream_t st) {
  batch_plan_kernel<<<1, kPlanBlock, 0, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_batch_unmatch(const BatchParams& B, const BatchRound* round, uint32_t max_tiles, cudaStream_t st) {
  batch_unmatch_kernel<<<max_tiles, kLinBlock, 0, st>>>(B, round);
  return cudaGetLastError();
}

cudaError_t launch_batch_align_init(const AlignOptions& o, uint32_t n_members, const double* init_T16, MemberState* state, double* poses, uint8_t* phase,
                                    uint8_t* seeded, bool keep_seeds, cudaStream_t st) {
  batch_align_init_kernel<<<(n_members + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(o, n_members, init_T16, state, poses, phase, seeded, keep_seeds ? 1 : 0);
  return cudaGetLastError();
}

cudaError_t launch_batch_align_finish(uint32_t n_members, const MemberState* state, double* out_T16, double* out_info4, double* out_Hb42, cudaStream_t st) {
  batch_align_finish_kernel<<<(n_members + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(n_members, state, out_T16, out_info4, out_Hb42);
  return cudaGetLastError();
}

// ---- sgb_align_batch_gnc (DESIGN.md §11 "Graduated non-convexity") ----

// the grid of a one-thread-per-stored-point GNC kernel (at least one CTA: the launch count does not depend on the point count)
uint32_t gnc_point_grid(uint32_t n, int sm_count) { return std::max<uint32_t>(1u, std::min<uint32_t>((n + 255u) / 256u, static_cast<uint32_t>(sm_count) * 8u)); }

// The GNC unit of member m, whose GncState and live flag its points use: the member itself (sgb_align_batch_gnc), or the window of the
// edge it is (sgb_align_joint_gnc: win[m])
struct GncMemberUnit {
  __device__ __forceinline__ uint32_t operator()(uint32_t m) const { return m; }
};
struct GncWindowUnit {
  const uint32_t* __restrict__ win;
  __device__ __forceinline__ uint32_t operator()(uint32_t m) const { return __ldg(&win[m]); }
};

// every unit's largest r^2 over its points before its stage 0 (no stage begun; the loop of gnc_rmax_kernel and joint_gnc_rmax_kernel,
// launched at every stage of the stage loop)
template <typename Unit>
__device__ __forceinline__ void gnc_rmax_points(const GncParams& p, Unit unit) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
    const uint32_t m = owner_of(p.member_off, p.n_members, i);
    const uint32_t u = unit(m);
    if (!p.live[u] || p.corr[i] == kNone) continue;
    if (p.gnc[u].stages != 0) continue;
    const double r2 = rn_mul(2.0, p.e[batch_row(p.member_off, p.perm, m, i)]);
    // a non-negative double orders as its bit pattern; -0.0, rounding's tiny negatives and NaN never enter
    if (r2 > 0.0) atomicMax(reinterpret_cast<unsigned long long*>(&p.gnc[u].r2max), static_cast<unsigned long long>(__double_as_longlong(r2)));
  }
}

__global__ void gnc_rmax_kernel(const GncParams p) {
  gnc_rmax_points(p, GncMemberUnit{});
}

__global__ void __launch_bounds__(kStepBlock) gnc_stage_kernel(const GncParams p) {
  const uint32_t m = blockIdx.x * kStepBlock + threadIdx.x;
  if (m >= p.n_members || !p.live[m]) return;
  gnc_stage_begin(p.kind, p.c2, p.max_stages, p.gnc[m]);
}

// every point's g of its unit's stage (the loop of gnc_weight_kernel and joint_gnc_weight_kernel)
template <int KIND, typename Unit>
__device__ __forceinline__ void gnc_weight_points(const GncParams& p, Unit unit) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
    const uint32_t m = owner_of(p.member_off, p.n_members, i);
    const uint32_t u = unit(m);
    if (!p.live[u]) continue;
    const size_t row = batch_row(p.member_off, p.perm, m, i);
    double g = 0.0;
    if (p.corr[i] != kNone) {
      const GncState& s = p.gnc[u];
      g = s.ones ? 1.0 : gnc_weight<KIND>(rn_mul(2.0, p.e[row]), s.mu, p.c2);
      if (KIND == kGncTls && g != 0.0 && g != 1.0) atomicOr(&p.gnc[u].not_binary, 1u);
    }
    p.e[row] = g;
    p.wstage[i] = p.w ? rn_mul(__ldg(&p.w[i]), g) : g;
  }
}

template <int KIND>
__global__ void gnc_weight_kernel(const GncParams p) {
  gnc_weight_points<KIND>(p, GncMemberUnit{});
}

// the options of member m's align in the current stage
__device__ __forceinline__ AlignOptions gnc_stage_options(const AlignOptions& o, const GncParams& p, uint32_t m) {
  AlignOptions om = o;
  if (!p.gnc[m].last) om.max_iterations = p.stage_iterations;
  return om;
}

__global__ void __launch_bounds__(kStepBlock) gnc_init_kernel(const GncParams p, const __grid_constant__ AlignOptions o, MemberState* __restrict__ state,
                                                              double* __restrict__ poses, uint8_t* __restrict__ phase) {
  const uint32_t m = blockIdx.x * kStepBlock + threadIdx.x;
  if (m >= p.n_members) return;
  MemberState& s = state[m];
  if (!p.live[m]) {  // finished earlier: its state holds its last stage's result
    s.phase = kPhaseDone;
    phase[m] = kPhaseDone;
    return;
  }
  GncState& g = p.gnc[m];
  if (p.kind == kGncTls && !g.not_binary) g.last = 1;
  p.live[m] = g.last ? 0 : 1;
  g.iterations += s.iterations;
  double T[16];
  for (int i = 0; i < 16; i++) T[i] = s.T[i];
  align_init(gnc_stage_options(o, p, m), T, s);
  double* q = poses + 12 * static_cast<size_t>(m);
  for (int i = 0; i < 3; i++) {  // pose_from_colmajor
    for (int j = 0; j < 3; j++) q[i * 3 + j] = T[j * 4 + i];
    q[9 + i] = T[12 + i];
  }
  phase[m] = static_cast<uint8_t>(s.phase);
}
// A round of a stage, its kind read from `round`; `loop` becomes 1 while a member has a round to go
__global__ void __launch_bounds__(kStepBlock) gnc_step_kernel(const GncParams p, const __grid_constant__ AlignOptions o, const double* __restrict__ out,
                                                              MemberState* __restrict__ state, double* __restrict__ poses, uint8_t* __restrict__ phase,
                                                              const BatchRound* __restrict__ round, cudaGraphConditionalHandle loop) {
  const uint32_t m = blockIdx.x * kStepBlock + threadIdx.x;
  int more = 0;
  if (m < p.n_members) {
    batch_step_member(gnc_stage_options(o, p, m), m, round->lin != 0u, out, state, poses, phase);
    more = phase[m] == kPhaseLinearize || phase[m] == kPhaseTrial;
  }
  if (__syncthreads_or(more) && threadIdx.x == 0) cudaGraphSetConditional(loop, 1u);
}

// ---- sgb_align_batch_gnc_async (DESIGN.md §11 "Asynchronous graduated non-convexity") ----

// The head of a stage: the members still in GNC in kPhaseLinearize, the others done, so that the planner plans the reweighting linearize
// of exactly the members in the stage; `rounds` cleared (gnc_loops_kernel sets it)
__global__ void __launch_bounds__(kStepBlock) gnc_reweigh_kernel(uint32_t n_members, const uint8_t* __restrict__ live, uint8_t* __restrict__ phase,
                                                                 cudaGraphConditionalHandle rounds) {
  const uint32_t m = blockIdx.x * kStepBlock + threadIdx.x;
  if (m == 0) cudaGraphSetConditional(rounds, 0u);
  if (m < n_members) phase[m] = live[m] ? kPhaseLinearize : kPhaseDone;
}

// After gnc_init_kernel: `stages` becomes 1 if a member has a stage to go after this one, `rounds` (cleared by gnc_reweigh_kernel) 1 if
// a member's align has a round to go
__global__ void __launch_bounds__(kStepBlock) gnc_loops_kernel(uint32_t n_members, const uint8_t* __restrict__ live, const uint8_t* __restrict__ phase,
                                                               cudaGraphConditionalHandle stages, cudaGraphConditionalHandle rounds) {
  const uint32_t m = blockIdx.x * kStepBlock + threadIdx.x;
  int more_stages = 0, more_rounds = 0;
  if (m < n_members) {
    more_stages = live[m];
    more_rounds = phase[m] == kPhaseLinearize || phase[m] == kPhaseTrial;
  }
  if (__syncthreads_or(more_stages) && threadIdx.x == 0) cudaGraphSetConditional(stages, 1u);
  if (__syncthreads_or(more_rounds) && threadIdx.x == 0) cudaGraphSetConditional(rounds, 1u);
}

// what sgb_align_batch_gnc adds to batch_align_finish_kernel's outputs: the iterations of the earlier stages, the stages and last mu
__global__ void __launch_bounds__(kStepBlock) gnc_finish_kernel(uint32_t n_members, const MemberState* __restrict__ state, const GncState* __restrict__ gnc,
                                                                double* __restrict__ out_info4, double* __restrict__ out_gnc2) {
  const uint32_t m = blockIdx.x * kStepBlock + threadIdx.x;
  if (m >= n_members) return;
  const GncState& g = gnc[m];
  out_info4[4 * static_cast<size_t>(m) + 1] = state[m].iterations + g.iterations;
  if (out_gnc2) {
    out_gnc2[2 * static_cast<size_t>(m)] = g.stages;
    out_gnc2[2 * static_cast<size_t>(m) + 1] = g.mu;
  }
}

cudaError_t launch_gnc_rmax(const GncParams& p, int sm_count, cudaStream_t st) {
  gnc_rmax_kernel<<<gnc_point_grid(p.n, sm_count), 256, 0, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_gnc_stage(const GncParams& p, cudaStream_t st) {
  gnc_stage_kernel<<<(p.n_members + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_gnc_weight(const GncParams& p, int sm_count, cudaStream_t st) {
  if (p.kind == kGncTls)
    gnc_weight_kernel<kGncTls><<<gnc_point_grid(p.n, sm_count), 256, 0, st>>>(p);
  else
    gnc_weight_kernel<kGncGemanMcClure><<<gnc_point_grid(p.n, sm_count), 256, 0, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_gnc_init(const GncParams& p, const AlignOptions& o, MemberState* state, double* poses, uint8_t* phase, cudaStream_t st) {
  gnc_init_kernel<<<(p.n_members + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(p, o, state, poses, phase);
  return cudaGetLastError();
}

cudaError_t launch_gnc_step(const GncParams& p, const AlignOptions& o, const BatchRound* round, cudaGraphConditionalHandle loop, const double* out,
                            MemberState* state, double* poses, uint8_t* phase, cudaStream_t st) {
  gnc_step_kernel<<<(p.n_members + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(p, o, out, state, poses, phase, round, loop);
  return cudaGetLastError();
}

cudaError_t launch_gnc_reweigh(uint32_t n_members, const uint8_t* live, uint8_t* phase, cudaGraphConditionalHandle rounds, cudaStream_t st) {
  gnc_reweigh_kernel<<<(n_members + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(n_members, live, phase, rounds);
  return cudaGetLastError();
}

cudaError_t launch_gnc_loops(uint32_t n_members, const uint8_t* live, const uint8_t* phase, cudaGraphConditionalHandle stages, cudaGraphConditionalHandle rounds,
                             cudaStream_t st) {
  gnc_loops_kernel<<<(n_members + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(n_members, live, phase, stages, rounds);
  return cudaGetLastError();
}

cudaError_t launch_gnc_finish(uint32_t n_members, const MemberState* state, const GncState* gnc, double* out_info4, double* out_gnc2, cudaStream_t st) {
  gnc_finish_kernel<<<(n_members + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(n_members, state, gnc, out_info4, out_gnc2);
  return cudaGetLastError();
}

// ---- sgb_align_joint (DESIGN.md §11 "Joint windows") ----

__device__ __forceinline__ void joint_write_edge_pose(const JointParams& J, uint32_t q, const double* X) {
  double T[16];
  edge_pose(X + 16 * J.edge_i[q], X + 16 * J.edge_j[q], T);
  double* p = J.poses + 12 * static_cast<size_t>(J.edge_member[q]);
  for (int i = 0; i < 3; i++) {  // pose_from_colmajor
    for (int j = 0; j < 3; j++) p[i * 3 + j] = T[j * 4 + i];
    p[9 + i] = T[12 + i];
  }
}

__global__ void joint_edge_poses_kernel(const __grid_constant__ JointParams J) {
  for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < J.n_edges; q += gridDim.x * blockDim.x)
    joint_write_edge_pose(J, q, J.X + 16 * static_cast<size_t>(J.frame_off[J.edge_win[q]]));
}

// One CTA per window; the window's system (packed lower triangle, up to 192 x 192) and the solve's scratch in dynamic shared memory.
// Threads take the rows of each column of the factorisation (n <= 192 < kJointBlock), the entries of each edge's blocks, the frames.
// ROUND (a round of sgb_align_joint_async): the round's kind is read from `round`; a window outside it sets `loop` to 1 if it still has a
// round to go, a stepped window writes its new phase to its edges' member_phase (what the next round's planner reads) and sets `loop` too.
constexpr int kJointBlock = 256;
template <bool ROUND>
__device__ __forceinline__ void joint_step_window(const AlignOptions& o, const JointParams& J, bool linearize, const double* __restrict__ out,
                                                  const BatchRound* __restrict__ round, cudaGraphConditionalHandle loop, uint8_t* __restrict__ member_phase) {
  extern __shared__ double s_work[];
  const uint32_t w = blockIdx.x;
  const int tid = threadIdx.x, nt = blockDim.x;
  WindowState* s = J.state + w;
  if constexpr (ROUND) {
    linearize = round->lin != 0u;
    const int ph = s->phase;
    if (ph != (linearize ? kPhaseLinearize : kPhaseTrial)) {
      if (tid == 0 && (ph == kPhaseLinearize || ph == kPhaseTrial)) cudaGraphSetConditional(loop, 1u);
      return;
    }
  }
  if (s->phase != (linearize ? kPhaseLinearize : kPhaseTrial)) return;
  const uint32_t f0 = J.frame_off[w], e0 = J.edge_off[w];
  JointWindow win;
  win.n_frames = static_cast<int>(J.frame_off[w + 1] - f0);
  win.n_free = static_cast<int>(J.n_free[w]);
  win.n_edges = static_cast<int>(J.edge_off[w + 1] - e0);
  win.free = J.free + f0;
  win.ei = J.edge_i + e0;
  win.ej = J.edge_j + e0;
  win.sums = J.sums + 44 * static_cast<size_t>(e0);
  win.X = J.X + 16 * static_cast<size_t>(f0);
  win.cand = J.cand + 16 * static_cast<size_t>(f0);
  win.delta = J.delta + 6 * static_cast<size_t>(f0);
  win.s = s;
  win.work = s_work;
  if (linearize) {
    // the edges' sums are kept: error() rounds overwrite `out`, and every further trial re-assembles the system from them
    for (uint32_t k = tid; k < 44u * win.n_edges; k += nt) J.sums[44 * static_cast<size_t>(e0) + k] = out[44 * static_cast<size_t>(J.edge_member[e0 + k / 44u]) + k % 44u];
    __syncthreads();
    joint_after_linearize(o, win, tid, nt);
  } else {
    double ce = 0.0;
    for (int q = 0; q < win.n_edges; q++) ce += out[J.edge_member[e0 + q]];
    joint_after_error(o, win, ce, tid, nt);
  }
  const double* X = s->phase == kPhaseTrial ? win.cand : win.X;
  for (int q = tid; q < win.n_edges; q += nt) joint_write_edge_pose(J, e0 + q, X);
  if (tid == 0) J.phase[w] = static_cast<uint8_t>(s->phase);
  if constexpr (ROUND) {
    const int ph = s->phase;
    for (int q = tid; q < win.n_edges; q += nt) member_phase[J.edge_member[e0 + q]] = static_cast<uint8_t>(ph);
    if (tid == 0 && (ph == kPhaseLinearize || ph == kPhaseTrial)) cudaGraphSetConditional(loop, 1u);
  }
}
template <bool ROUND>
__global__ void __launch_bounds__(kJointBlock) joint_step_kernel(const __grid_constant__ AlignOptions o, const __grid_constant__ JointParams J, bool linearize,
                                                                 const double* __restrict__ out, const BatchRound* __restrict__ round,
                                                                 cudaGraphConditionalHandle loop, uint8_t* __restrict__ member_phase) {
  joint_step_window<ROUND>(o, J, linearize, out, round, loop, member_phase);
}

cudaError_t launch_joint_edge_poses(const JointParams& J, cudaStream_t st) {
  if (!J.n_edges) return cudaSuccess;
  joint_edge_poses_kernel<<<(J.n_edges + 127u) / 128u, 128, 0, st>>>(J);
  return cudaGetLastError();
}

cudaError_t launch_joint_step(const AlignOptions& o, const JointParams& J, int max_free, bool linearize, const BatchRound* round, cudaGraphConditionalHandle loop,
                              uint8_t* member_phase, const double* out, cudaStream_t st) {
  const auto kernel = round ? joint_step_kernel<true> : joint_step_kernel<false>;
  const size_t smem = joint_step_smem(max_free);
  const cudaError_t e = allow_dynamic_smem(kernel, smem);
  if (e != cudaSuccess) return e;
  kernel<<<J.n_windows, kJointBlock, smem, st>>>(o, J, linearize, out, round, loop, member_phase);
  return cudaGetLastError();
}

// ---- sgb_align_joint_async (DESIGN.md §11 "Asynchronous joint windows") ----

// One CTA per window: sgb_align_joint's set-up on the device.  Thread 0 runs joint_init; the frames' X are copied from init_X16; then
// every edge gets its initial pose (joint_write_edge_pose, as joint_edge_poses_kernel), its window's phase as its member phase (what the
// planner reads) and, unless keep_seeds, a cleared seed flag (as batch_align_init_kernel clears a member's).
__global__ void __launch_bounds__(kStepBlock) joint_align_init_kernel(const __grid_constant__ AlignOptions o, const __grid_constant__ JointParams J,
                                                                      const double* __restrict__ init_X16, uint8_t* __restrict__ member_phase,
                                                                      uint8_t* __restrict__ seeded, int keep_seeds) {
  __shared__ uint8_t s_phase;
  const uint32_t w = blockIdx.x, f0 = J.frame_off[w], f1 = J.frame_off[w + 1], e0 = J.edge_off[w], e1 = J.edge_off[w + 1];
  if (threadIdx.x == 0) {
    joint_init(o, static_cast<int>(J.n_free[w]), static_cast<int>(e1 - e0), J.state[w]);
    s_phase = static_cast<uint8_t>(J.state[w].phase);
    J.phase[w] = s_phase;
  }
  for (size_t k = 16 * static_cast<size_t>(f0) + threadIdx.x; k < 16 * static_cast<size_t>(f1); k += kStepBlock) J.X[k] = init_X16[k];
  __syncthreads();
  for (uint32_t q = e0 + threadIdx.x; q < e1; q += kStepBlock) {
    joint_write_edge_pose(J, q, J.X + 16 * static_cast<size_t>(f0));
    const uint32_t m = J.edge_member[q];
    member_phase[m] = s_phase;
    if (!keep_seeds) seeded[m] = 0;
  }
}

// sgb_align_joint's outputs: thread i writes frame i's X (a fixed frame's from init_X16, bit for bit) and window i's info
__global__ void __launch_bounds__(kStepBlock) joint_align_finish_kernel(const __grid_constant__ JointParams J, uint32_t n_frames, const double* __restrict__ init_X16,
                                                                        double* __restrict__ out_X16, double* __restrict__ out_info4) {
  const uint32_t i = blockIdx.x * kStepBlock + threadIdx.x;
  if (i < n_frames) {
    const double* X = (J.free[i] < 0 ? init_X16 : J.X) + 16 * static_cast<size_t>(i);
    for (int k = 0; k < 16; k++) out_X16[16 * static_cast<size_t>(i) + k] = X[k];
  }
  if (i < J.n_windows) {
    const WindowState& s = J.state[i];
    double* info = out_info4 + 4 * static_cast<size_t>(i);
    info[0] = s.converged ? 1.0 : 0.0;
    info[1] = s.iterations;
    info[2] = s.inliers;
    info[3] = s.e;
  }
}

cudaError_t launch_joint_align_init(const AlignOptions& o, const JointParams& J, const double* init_X16, uint8_t* member_phase, uint8_t* seeded, bool keep_seeds,
                                    cudaStream_t st) {
  joint_align_init_kernel<<<J.n_windows, kStepBlock, 0, st>>>(o, J, init_X16, member_phase, seeded, keep_seeds ? 1 : 0);
  return cudaGetLastError();
}

cudaError_t launch_joint_align_finish(const JointParams& J, uint32_t n_frames, const double* init_X16, double* out_X16, double* out_info4, cudaStream_t st) {
  const uint32_t n = std::max(n_frames, J.n_windows);
  joint_align_finish_kernel<<<(n + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(J, n_frames, init_X16, out_X16, out_info4);
  return cudaGetLastError();
}

// ---- sgb_align_joint_gnc (DESIGN.md §11 "Graduated non-convexity for joint windows"): the GNC unit is the window.  p.gnc and p.live are
// per window; the point kernels reach a point's window through its member (edge), member_win[m] ----

__global__ void joint_gnc_rmax_kernel(const GncParams p, const uint32_t* __restrict__ member_win) {
  gnc_rmax_points(p, GncWindowUnit{member_win});
}

template <int KIND>
__global__ void joint_gnc_weight_kernel(const GncParams p, const uint32_t* __restrict__ member_win) {
  gnc_weight_points<KIND>(p, GncWindowUnit{member_win});
}

// One thread per window (p.n_members = the windows), as gnc_init_kernel per member: a window in the stage ends GNC after it if the stage
// is its last (TLS: or its weights are all binary), adds the previous stage's iterations and starts its joint align from its current X
// (joint_init with max_iterations = stage_iterations unless last); every other window is left done.  Its edges' poses are those of its X
// already: the stage's reweighting linearize ran at them.
__global__ void __launch_bounds__(kStepBlock) joint_gnc_init_kernel(const GncParams p, const __grid_constant__ AlignOptions o, const __grid_constant__ JointParams J) {
  const uint32_t w = blockIdx.x * kStepBlock + threadIdx.x;
  if (w >= J.n_windows) return;
  WindowState& s = J.state[w];
  if (!p.live[w]) {  // finished earlier: its state holds its last stage's result
    s.phase = kPhaseDone;
    J.phase[w] = kPhaseDone;
    return;
  }
  GncState& g = p.gnc[w];
  if (p.kind == kGncTls && !g.not_binary) g.last = 1;
  p.live[w] = g.last ? 0 : 1;
  g.iterations += s.iterations;
  joint_init(gnc_stage_options(o, p, w), static_cast<int>(J.n_free[w]), static_cast<int>(J.edge_off[w + 1] - J.edge_off[w]), s);
  J.phase[w] = static_cast<uint8_t>(s.phase);
}

// joint_step_kernel<true> for a round of a GNC stage (its kind read from `round`, each stepped window's phase to its edges' member_phase,
// `loop` set to 1 while a window has a round to go): each window steps with its stage's max_iterations (as joint_gnc_init_kernel chose)
__global__ void __launch_bounds__(kJointBlock) joint_gnc_step_kernel(const __grid_constant__ AlignOptions o, const __grid_constant__ JointParams J,
                                                                     const double* __restrict__ out, const GncParams p, const BatchRound* __restrict__ round,
                                                                     cudaGraphConditionalHandle loop, uint8_t* __restrict__ member_phase) {
  joint_step_window<true>(gnc_stage_options(o, p, blockIdx.x), J, false, out, round, loop, member_phase);  // (the kind is the round's)
}

cudaError_t launch_joint_gnc_rmax(const GncParams& p, const uint32_t* member_win, int sm_count, cudaStream_t st) {
  joint_gnc_rmax_kernel<<<gnc_point_grid(p.n, sm_count), 256, 0, st>>>(p, member_win);
  return cudaGetLastError();
}

cudaError_t launch_joint_gnc_weight(const GncParams& p, const uint32_t* member_win, int sm_count, cudaStream_t st) {
  if (p.kind == kGncTls)
    joint_gnc_weight_kernel<kGncTls><<<gnc_point_grid(p.n, sm_count), 256, 0, st>>>(p, member_win);
  else
    joint_gnc_weight_kernel<kGncGemanMcClure><<<gnc_point_grid(p.n, sm_count), 256, 0, st>>>(p, member_win);
  return cudaGetLastError();
}

cudaError_t launch_joint_gnc_init(const GncParams& pw, const AlignOptions& o, const JointParams& J, cudaStream_t st) {
  joint_gnc_init_kernel<<<(J.n_windows + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(pw, o, J);
  return cudaGetLastError();
}

cudaError_t launch_joint_gnc_step(const AlignOptions& o, const JointParams& J, int max_free, const double* out, const GncParams& pw, const BatchRound* round,
                                  cudaGraphConditionalHandle loop, uint8_t* member_phase, cudaStream_t st) {
  const size_t smem = joint_step_smem(max_free);
  const cudaError_t e = allow_dynamic_smem(joint_gnc_step_kernel, smem);
  if (e != cudaSuccess) return e;
  joint_gnc_step_kernel<<<J.n_windows, kJointBlock, smem, st>>>(o, J, out, pw, round, loop, member_phase);
  return cudaGetLastError();
}

// ---- sgb_align_joint_gnc_async (DESIGN.md §11 "Asynchronous graduated non-convexity for joint windows"): the stages and their joint rounds
// on the device.  The edges are the members of the rounds, each edge's member phase its window's. ----

// The head of a stage, one thread per edge: the edges of the windows still in GNC in kPhaseLinearize, every other edge done, so that the
// planner plans the reweighting linearize of exactly the edges of the windows in the stage; `rounds` cleared (joint_gnc_loops_kernel sets it)
__global__ void __launch_bounds__(kStepBlock) joint_gnc_reweigh_kernel(const __grid_constant__ JointParams J, const uint8_t* __restrict__ live,
                                                                       uint8_t* __restrict__ member_phase, cudaGraphConditionalHandle rounds) {
  const uint32_t q = blockIdx.x * kStepBlock + threadIdx.x;
  if (q == 0) cudaGraphSetConditional(rounds, 0u);
  if (q < J.n_edges) member_phase[J.edge_member[q]] = live[J.edge_win[q]] ? kPhaseLinearize : kPhaseDone;
}

// After joint_gnc_init_kernel, one thread per edge and per window: each edge's member phase becomes its window's new phase (what the
// rounds' planner reads; joint_gnc_init_kernel writes J.phase only); `stages` becomes 1 if a window has a stage to go after this one,
// `rounds` (cleared by joint_gnc_reweigh_kernel) 1 if a window's joint align has a round to go
__global__ void __launch_bounds__(kStepBlock) joint_gnc_loops_kernel(const __grid_constant__ JointParams J, const uint8_t* __restrict__ live,
                                                                     uint8_t* __restrict__ member_phase, cudaGraphConditionalHandle stages,
                                                                     cudaGraphConditionalHandle rounds) {
  const uint32_t i = blockIdx.x * kStepBlock + threadIdx.x;
  if (i < J.n_edges) member_phase[J.edge_member[i]] = J.phase[J.edge_win[i]];
  int more_stages = 0, more_rounds = 0;
  if (i < J.n_windows) {
    more_stages = live[i];
    more_rounds = J.phase[i] == kPhaseLinearize || J.phase[i] == kPhaseTrial;
  }
  if (__syncthreads_or(more_stages) && threadIdx.x == 0) cudaGraphSetConditional(stages, 1u);
  if (__syncthreads_or(more_rounds) && threadIdx.x == 0) cudaGraphSetConditional(rounds, 1u);
}

// what sgb_align_joint_gnc adds to joint_align_finish_kernel's outputs, per window: the iterations of its earlier stages, its stages and last mu
__global__ void __launch_bounds__(kStepBlock) joint_gnc_finish_kernel(uint32_t n_windows, const WindowState* __restrict__ state, const GncState* __restrict__ gnc,
                                                                      double* __restrict__ out_info4, double* __restrict__ out_gnc2) {
  const uint32_t w = blockIdx.x * kStepBlock + threadIdx.x;
  if (w >= n_windows) return;
  const GncState& g = gnc[w];
  out_info4[4 * static_cast<size_t>(w) + 1] = state[w].iterations + g.iterations;
  if (out_gnc2) {
    out_gnc2[2 * static_cast<size_t>(w)] = g.stages;
    out_gnc2[2 * static_cast<size_t>(w) + 1] = g.mu;
  }
}

cudaError_t launch_joint_gnc_reweigh(const JointParams& J, const uint8_t* live, uint8_t* member_phase, cudaGraphConditionalHandle rounds, cudaStream_t st) {
  joint_gnc_reweigh_kernel<<<(J.n_edges + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(J, live, member_phase, rounds);
  return cudaGetLastError();
}

cudaError_t launch_joint_gnc_loops(const JointParams& J, const uint8_t* live, uint8_t* member_phase, cudaGraphConditionalHandle stages,
                                   cudaGraphConditionalHandle rounds, cudaStream_t st) {
  const uint32_t n = std::max(J.n_edges, J.n_windows);
  joint_gnc_loops_kernel<<<(n + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(J, live, member_phase, stages, rounds);
  return cudaGetLastError();
}

cudaError_t launch_joint_gnc_finish(const JointParams& J, const GncState* gnc, double* out_info4, double* out_gnc2, cudaStream_t st) {
  joint_gnc_finish_kernel<<<(J.n_windows + kStepBlock - 1) / kStepBlock, kStepBlock, 0, st>>>(J.n_windows, J.state, gnc, out_info4, out_gnc2);
  return cudaGetLastError();
}

}  // namespace sgb
