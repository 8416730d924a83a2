// SPDX-License-Identifier: MIT
// C-ABI of batched registration (include/sgicp_b200.h: sgb_source_set_batch, sgb_source_set_pairs, sgb_source_set_submaps,
// sgb_source_set_weights, sgb_{linearize,error,align,correspondences}_batch, sgb_{linearize,error}_batch_points, sgb_align_batch_async, sgb_align_joint,
// sgb_align_joint_async, sgb_align_batch_gnc, sgb_align_batch_gnc_async, sgb_joint_edge_poses, sgb_align_joint_gnc, sgb_align_joint_gnc_async).
// Kernels in sgb_batch.cu (many kd-trees and submaps: the searches in sgb_forest.cu); DESIGN.md §11.
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <string>
#include <vector>

#include "../../include/sgicp_b200.h"
#include "sgb_batch.h"
#include "sgb_context.hpp"
#include "sgb_forest.h"
#include "sgb_kernels.h"

using namespace sgb;

namespace {

constexpr double kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};

size_t batch_points(const sgb_ctx* ctx) { return ctx->b_offsets.empty() ? 0 : ctx->b_offsets.back(); }
size_t batch_members(const sgb_ctx* ctx) { return ctx->b_offsets.empty() ? 0 : ctx->b_offsets.size() - 1; }
size_t max_tiles(const sgb_ctx* ctx) { return batch_points(ctx) / kLinBlock + batch_members(ctx) + 1; }

bool many_maps(const sgb_ctx* ctx) { return ctx->tgt_state == TargetState::VoxelMaps || ctx->tgt_state == TargetState::KdTrees; }
// the members read the per-map tables through the pairing's view (PairView)
bool paired_maps(const sgb_ctx* ctx) { return ctx->b_pair_has_maps && many_maps(ctx); }

int batch_check(sgb_ctx* ctx, const char* who, const double* T) {
  if (ctx->src_state != SourceState::Batch) return fail(ctx, 1, std::string(who) + ": the context holds no batch of sources (call sgb_source_set_batch)");
  if (ctx->comm_world > 1) return fail(ctx, 1, std::string(who) + ": batched calls are single-GPU only (call sgb_comm_disconnect first)");
  if (!T) return fail(ctx, 1, std::string(who) + ": null poses");
  if (ctx->b_submaps) {
    // as for a pairing's maps: the target may have been replaced since, so the lists are checked at every call
    if (ctx->tgt_state != TargetState::KdTrees)
      return fail(ctx, 1, std::string(who) + ": the members are aligned against submaps (sgb_source_set_submaps), which are lists of maps of a many-kd-trees target "
                              "(sgb_target_build_kdtrees); the current target is not one (submaps over voxel maps are not supported)");
    if (ctx->b_pair_max_map >= ctx->kt_maps) {
      for (size_t p = 0; p + 1 < ctx->b_sub_off.size(); p++)
        for (uint32_t j = ctx->b_sub_off[p]; j < ctx->b_sub_off[p + 1]; j++)
          if (ctx->b_sub_maps[j] >= ctx->kt_maps)
            return fail(ctx, 1, std::string(who) + ": entry " + std::to_string(j - ctx->b_sub_off[p]) + " of member " + std::to_string(p) + " names map " +
                                    std::to_string(ctx->b_sub_maps[j]) + " but the target holds " + std::to_string(ctx->kt_maps) + " maps");
    }
    return 0;
  }
  if (ctx->b_pair_has_maps) {
    // the target may have been replaced since the pairing: its maps are checked at every call
    if (!many_maps(ctx))
      return fail(ctx, 1, std::string(who) + ": the pairing names a map per member (sgb_source_set_pairs) but the target is not a many-maps or many-kd-trees target");
    const size_t maps = target_maps(ctx);
    if (ctx->b_pair_max_map >= maps) {
      for (size_t p = 0; p < ctx->b_pair_maps.size(); p++)
        if (ctx->b_pair_maps[p] >= maps)
          return fail(ctx, 1, std::string(who) + ": member " + std::to_string(p) + " is paired with map " + std::to_string(ctx->b_pair_maps[p]) +
                                  " but the target holds " + std::to_string(maps) + " maps");
    }
    return 0;
  }
  if (ctx->tgt_state == TargetState::VoxelMaps && batch_members(ctx) != ctx->vm_maps)
    return fail(ctx, 1, std::string(who) + ": the batch has " + std::to_string(batch_members(ctx)) + " members but the target holds " +
                            std::to_string(ctx->vm_maps) + " voxel maps (member m is aligned against map m)");
  if (ctx->tgt_state == TargetState::KdTrees && batch_members(ctx) != ctx->kt_maps)
    return fail(ctx, 1, std::string(who) + ": the batch has " + std::to_string(batch_members(ctx)) + " members but the target holds " +
                            std::to_string(ctx->kt_maps) + " kd-trees (member m is aligned against map m)");
  return 0;
}

// n o r, the reference's point-to-plane residual, changes with the frame it is evaluated in, so it has no meaning against maps that
// each sit in a frame of their own
int submap_factor_check(sgb_ctx* ctx, const char* who, int factor) {
  if (!ctx->b_submaps || factor != SGB_FACTOR_PLANE_ICP) return 0;
  return fail(ctx, 1, std::string(who) + ": SGB_FACTOR_PLANE_ICP is not available against submaps (sgb_source_set_submaps): its residual is the element-wise "
                          "product of the normal and the point difference, which is not invariant under the poses that place the maps; use ICP or GICP");
}

// the layout of s_tables, the one upload of sgb_source_set_submaps: inverse entry poses [entries][12] | entry_off [members + 1] | entry_maps [entries]
struct SubmapTables {
  const double* inv_poses;
  const uint32_t *entry_off, *entry_maps;
};
SubmapTables submap_tables(const sgb_ctx* ctx) {
  const size_t E = ctx->b_sub_maps.size();
  const double* poses = ctx->s_tables.as<double>();
  const uint32_t* off = reinterpret_cast<const uint32_t*>(poses + 12 * E);
  return SubmapTables{poses, off, off + ctx->b_sub_off.size()};
}
SubmapView submap_view(const sgb_ctx* ctx) {
  const SubmapTables t = submap_tables(ctx);
  return SubmapView{t.entry_off, ctx->s_entries.as<uint4>(), ctx->s_centres.as<double>(), t.inv_poses, ctx->b_centry.as<uint32_t>()};
}

bool voxel_target(const sgb_ctx* ctx) { return ctx->tgt_state == TargetState::VoxelMap || ctx->tgt_state == TargetState::VoxelMaps; }

// Builds the pairing's view of the current target (one launch) unless it is up to date: forget_linearisation, which every target
// transition and every pairing goes through, marks it stale.
int pair_view(sgb_ctx* ctx) {
  if (ctx->b_submaps && !ctx->b_view_ok) {  // batch_check has passed: the target is many kd-trees and holds every listed map
    CU(cudaSetDevice(ctx->device));
    const uint32_t* tab = ctx->kt_tables.as<uint32_t>();
    SubmapViewBuild v = {};
    v.n_entries = static_cast<uint32_t>(ctx->b_sub_maps.size());
    v.entry_maps = submap_tables(ctx).entry_maps;
    v.map_pt_off = tab;
    v.map_node_base = tab + 3 * (ctx->kt_maps + 1);
    v.map_centres = ctx->kt_centres.as<double>();
    v.entries = ctx->s_entries.as<uint4>();
    v.centres = ctx->s_centres.as<double>();
    CU(launch_submap_view(v, ctx->sm_count, ctx->stream));
    ctx->launches += v.n_entries ? 1 : 0;
    ctx->b_view_ok = true;
    return 0;
  }
  if (!paired_maps(ctx) || ctx->b_view_ok) return 0;
  CU(cudaSetDevice(ctx->device));
  const size_t P = batch_members(ctx);
  PairView v = {};
  v.n_members = static_cast<uint32_t>(P);
  v.maps = ctx->p_tables.as<uint32_t>() + 2 * P + 1;
  v.centres = ctx->v_centres.as<double>();
  if (ctx->tgt_state == TargetState::KdTrees) {
    const uint32_t* tab = ctx->kt_tables.as<uint32_t>();
    v.map_centres = ctx->kt_centres.as<double>();
    v.map_pt_off = tab;
    v.map_node_base = tab + 3 * (ctx->kt_maps + 1);
    v.pt_off = ctx->v_tables.as<uint32_t>();
    v.node_base = v.pt_off + P + 1;
  } else {
    v.map_centres = ctx->vm_centres.as<double>();
    v.map_regions = ctx->vm_regions.as<uint4>();
    v.regions = ctx->v_regions.as<uint4>();
  }
  CU(launch_pair_view(v, ctx->stream));
  ctx->launches += 1;
  ctx->b_view_ok = true;
  return 0;
}

// The tables of one call: every active non-empty member's points cut into tiles of kLinBlock (the virtual source concatenates the
// active members in member order), each member's pose (row-major R | t; T = nullptr: b_poses already holds them).  Uploaded on the
// context's stream.
int batch_tables(sgb_ctx* ctx, const double* T, const uint8_t* active, bool seeds, uint32_t* n_tiles, uint32_t* n_virtual) {
  const size_t B = batch_members(ctx);
  std::vector<double> poses(T ? 12 * B : 0);
  std::vector<BatchTile> tiles;
  std::vector<uint4> members(B);
  uint32_t v = 0;
  for (size_t m = 0; m < B; m++) {
    if (T) pose_from_colmajor(T + 16 * m, poses.data() + 12 * m);
    const bool act = !active || active[m];
    const uint32_t first = static_cast<uint32_t>(ctx->b_offsets[m]), n = static_cast<uint32_t>(ctx->b_offsets[m + 1] - ctx->b_offsets[m]);
    const uint32_t t0 = static_cast<uint32_t>(tiles.size());
    if (act) {
      for (uint32_t j = 0; j < n; j += kLinBlock) tiles.push_back(BatchTile{static_cast<uint32_t>(m), first + j, std::min<uint32_t>(kLinBlock, n - j), v + j});
      v += n;
    }
    members[m] = make_uint4(t0, static_cast<uint32_t>(tiles.size()) - t0, (act ? kMemberActive : 0u) | (seeds && ctx->b_seeded[m] ? kMemberSeeded : 0u), 0u);
  }
  // pageable host memory: the copies are staged before cudaMemcpyAsync returns
  if (T) CU(cudaMemcpyAsync(ctx->b_poses.p, poses.data(), poses.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(ctx->b_members.p, members.data(), members.size() * sizeof(uint4), cudaMemcpyHostToDevice, ctx->stream));
  if (!tiles.empty()) CU(cudaMemcpyAsync(ctx->b_tiles.p, tiles.data(), tiles.size() * sizeof(BatchTile), cudaMemcpyHostToDevice, ctx->stream));
  *n_tiles = static_cast<uint32_t>(tiles.size());
  *n_virtual = v;
  return 0;
}

BatchParams batch_params(sgb_ctx* ctx, const LinParams& P) {
  BatchParams B = {};
  B.tgt = P.tgt;
  const bool pairs = ctx->b_paired;  // the members' replicas, else the stored clouds themselves
  B.pts = (pairs ? ctx->p_pts : ctx->src_pts).as<float4>();
  B.covA = (pairs ? ctx->p_covA : ctx->src_covA).as<float4>();
  B.covB = (pairs ? ctx->p_covB : ctx->src_covB).as<float4>();
  B.centres = (pairs ? ctx->p_centres : ctx->b_centres).as<double>();
  B.poses = ctx->b_poses.as<double>();
  B.lin_poses = ctx->b_lin_poses.as<double>();
  B.tiles = ctx->b_tiles.as<BatchTile>();
  B.members = ctx->b_members.as<uint4>();
  B.corr = ctx->b_corr.as<uint32_t>();
  B.tile_partials = ctx->b_partials.as<double>();
  return B;
}

int copy_out(sgb_ctx* ctx, double* out, size_t doubles) {
  CU(cudaMemcpyAsync(out, ctx->b_out.p, doubles * sizeof(double), cudaMemcpyDefault, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

// The search of a point target over the virtual source in a round planned on the device: launch_point_search with the query count read on
// the device.  The counters do not alternate (a replayed graph cannot flip host state): the planner clears both pending counters, the
// class counters and both queue counters at the head of every round.
int point_search_round(sgb_ctx* ctx, const LinParams& P, const uint32_t* n_queries, int depth) {
  const size_t n = P.src.n;
  const int sgrid = one_wave_grid((n + 31) / 32 * 32, ctx->sm_count, packet_occupancy(depth));
  const uint8_t* settled = nullptr;
  const uint32_t* pending_count = nullptr;
  ChunkClasses cc = {};
  PendingParams pp = {};
  if (ctx->grid_ready) {
    point_search_params(ctx, n, 0, cc, pp);
    uint32_t* pbase = ctx->grid_pending.as<uint32_t>();
    settled = ctx->grid_state.as<uint8_t>();
    pending_count = pbase;
    CU(launch_grid_probe(P, n_queries, ctx->grid_pts.as<float4>(), ctx->grid_table.as<GridSlot>(), ctx->grid_capacity, pp.g, ctx->grid_state.as<uint8_t>(), pbase,
                         pbase + 2, ctx->grid_pending_q.as<float4>(), pbase + 1, cc, ctx->stream));
  }
  uint32_t* queue = ctx->use_packet_queue ? ctx->packet_queue.as<uint32_t>() : nullptr;
  CU(launch_packet_search(P, n_queries, ctx->tgt_pnodes.as<float4>(), sgrid, depth, settled, pending_count, static_cast<uint32_t>(ctx->pending_div), queue,
                          queue ? queue + 1 : nullptr, cc, pp, false, ctx->stream));
  return 0;
}

// The search and the factor kernel of one round against the current (non-empty) target, for its kind.  round = null: a round planned on
// the host -- exact grids of n_tiles tiles and n_virtual queries, a linearize or (err) an error() round -- counted per launch; else a round
// planned on the device (err = false), its grids sized for every tile (n_tiles = max_tiles) and point (n_virtual = batch_points), counted
// with the graph that holds it.  P: the target's parameters (fill_params at the identity); bound: the FP32 search bound.
int round_kernels(sgb_ctx* ctx, const LinParams& P, const BatchParams& Bp, const BatchRound* round, uint32_t n_tiles, uint32_t n_virtual, bool err, int factor,
                  int robust, float bound, const BatchRows* rows = nullptr) {
  const int counted = round ? 0 : 1;
  // the per-map tables: with a pairing's map table the member-indexed view of the maps, else the map-indexed tables
  const bool view = paired_maps(ctx);
  const double* centres = nullptr;
  const uint4* regions = nullptr;
  int kind = voxel_target(ctx) ? 1 : 0;
  if (ctx->b_submaps) {
    kind = 4;
  } else if (ctx->tgt_state == TargetState::VoxelMaps) {
    kind = 2;
    centres = (view ? ctx->v_centres : ctx->vm_centres).as<double>();
    regions = (view ? ctx->v_regions : ctx->vm_regions).as<uint4>();
  } else if (ctx->tgt_state == TargetState::KdTrees) {
    kind = 3;
    centres = (view ? ctx->v_centres : ctx->kt_centres).as<double>();
  }
  const SubmapView S = ctx->b_submaps ? submap_view(ctx) : SubmapView{};
  uint32_t* vcorr = ctx->b_vcorr.as<uint32_t>();
  if (!err && kind == 4) {
    // submaps: every tile searched in the trees of its member's entries, each in its own stored frame (sgb_forest.cu)
    CU(launch_submap_search(Bp, ctx->tgt_pnodes.as<float4>(), S, round, n_tiles, ctx->kt_depth, bound, vcorr, ctx->stream));
    ctx->launches += counted;
  } else if (!err && kind == 3) {
    // many trees: every tile searched in its member's own tree, straight from the stored points at the member's pose (sgb_forest.cu)
    const uint32_t* tab = (view ? ctx->v_tables : ctx->kt_tables).as<uint32_t>();
    const size_t M = view ? batch_members(ctx) : ctx->kt_maps;
    const ForestView F{ctx->tgt_pnodes.as<float4>(), centres, tab, tab + (view ? M + 1 : 3 * (M + 1))};
    CU(launch_forest_search(Bp, F, round, n_tiles, ctx->kt_depth, bound, vcorr, ctx->stream));
    ctx->launches += counted;
  } else if (!err && kind == 0) {
    // the search runs over the virtual source: the active members' queries, already transformed into the target's frame
    CU(launch_batch_transform(Bp, round, n_tiles, ctx->b_vq.as<float4>(), vcorr, ctx->stream));
    ctx->launches += counted;
    LinParams Q = P;
    Q.src.pts = ctx->b_vq.as<float4>();
    Q.src.covA = Q.src.covB = nullptr;
    Q.src.centre = ctx->tgt_centre.as<double>();  // identity pose, source centre = target centre: the search takes the stored query as is
    Q.src.n = n_virtual;
    Q.src.run = 1;
    Q.corr = vcorr;
    Q.use_prev = 1;  // per member: its previous correspondences, or kNone
    Q.max_dist_sq = bound;
    const int depth = ctx->tree_depth > 0 ? ctx->tree_depth : 1;
    if (int rc = round ? point_search_round(ctx, Q, &round->n_search, depth) : launch_point_search(ctx, Q, depth)) return rc;
    ctx->launches += counted;
  }
  // the weights in force (sgb_source_set_weights), or those of a GNC align's round (RoundWeights)
  const double* weights = ctx->b_wround ? ctx->b_wuse : ctx->b_weighted ? ctx->b_weights.as<double>() : nullptr;
  CU(launch_batch_factor(Bp, kind, factor, robust, err, round, n_tiles, err ? nullptr : vcorr, centres, regions, S, rows, weights, ctx->stream));
  ctx->launches += counted;
  return 0;
}

// What a linearize leaves in the context: the members of the mask (null: every member) linearised against the current target, their
// correspondences usable as seeds, and its factor and robust kernel for error()
void mark_linearised(sgb_ctx* ctx, int factor, int robust, double robust_c, const uint8_t* members) {
  // a new target (or none linearised yet) invalidates every member's cached state; sgb_drop_seeds only the seeds
  if (!ctx->have_lin) std::fill(ctx->b_lin.begin(), ctx->b_lin.end(), 0);
  if (!ctx->corr_seeds) std::fill(ctx->b_seeded.begin(), ctx->b_seeded.end(), 0);
  for (size_t m = 0; m < ctx->b_lin.size(); m++) {
    if (members && !members[m]) continue;
    ctx->b_lin[m] = 1;
    ctx->b_seeded[m] = 1;
  }
  ctx->have_lin = true;
  ctx->corr_seeds = true;
  ctx->lin_factor = factor;
  ctx->lin_robust = robust;
  ctx->lin_c = robust_c;
}

// One linearize of the active members (arguments checked by the caller) into b_out, asynchronous.  T = nullptr: poses already in b_poses.
// rows: the factor kernel's per-point rows too (the rows it does not reach are the caller's to clear: point_rows).
int linearize_round(sgb_ctx* ctx, int factor, int robust, double robust_c, int rejector, double max_dist_sq, const double* T, const uint8_t* active,
                    const BatchRows* rows = nullptr) {
  const size_t B = batch_members(ctx);
  CU(cudaSetDevice(ctx->device));
  const bool voxel = voxel_target(ctx);
  // the same reset as mark_linearised's, here because batch_tables reads the seed flags
  if (!ctx->have_lin) std::fill(ctx->b_lin.begin(), ctx->b_lin.end(), 0);
  if (!ctx->corr_seeds) std::fill(ctx->b_seeded.begin(), ctx->b_seeded.end(), 0);
  uint32_t n_tiles = 0, n_virtual = 0;
  if (int rc = batch_tables(ctx, T, active, !voxel, &n_tiles, &n_virtual)) return rc;
  LinParams P;
  fill_params(ctx, P, kIdentity);
  BatchParams Bp = batch_params(ctx, P);
  Bp.max_dist_sq_d = rejector == SGB_REJECT_DISTANCE ? max_dist_sq : DBL_MAX;
  Bp.robust_c = robust_c;
  if (ctx->n_tgt == 0) {  // nothing to match: every active member's points are unmatched, its sums zero
    n_tiles = 0;
    for (size_t m = 0; m < B; m++) {
      const size_t nm = ctx->b_offsets[m + 1] - ctx->b_offsets[m];
      if ((!active || active[m]) && nm) CU(cudaMemsetAsync(ctx->b_corr.as<uint32_t>() + ctx->b_offsets[m], 0xFF, nm * sizeof(uint32_t), ctx->stream));
    }
    std::vector<uint4> none(B, make_uint4(0, 0, 0, 0));
    for (size_t m = 0; m < B; m++) none[m].z = (!active || active[m]) ? kMemberActive : 0u;
    CU(cudaMemcpyAsync(ctx->b_members.p, none.data(), B * sizeof(uint4), cudaMemcpyHostToDevice, ctx->stream));
  }
  if (n_tiles) {
    if (int rc = round_kernels(ctx, P, Bp, nullptr, n_tiles, n_virtual, false, factor, robust, search_bound(rejector, max_dist_sq), rows)) return rc;
  }
  CU(launch_batch_segment(Bp, static_cast<uint32_t>(B), true, nullptr, ctx->b_out.as<double>(), ctx->stream));
  ctx->launches += 1;
  mark_linearised(ctx, factor, robust, robust_c, active);
  return 0;
}

// One error() of the active members (every one linearised against the current target) into b_out[0, B), asynchronous.  T, rows as above.
int error_round(sgb_ctx* ctx, const double* T, const uint8_t* active, const BatchRows* rows = nullptr) {
  const size_t B = batch_members(ctx);
  CU(cudaSetDevice(ctx->device));
  uint32_t n_tiles = 0, n_virtual = 0;
  if (int rc = batch_tables(ctx, T, active, false, &n_tiles, &n_virtual)) return rc;
  LinParams P;
  fill_params(ctx, P, kIdentity);
  BatchParams Bp = batch_params(ctx, P);
  Bp.robust_c = ctx->lin_c;
  if (n_tiles && ctx->n_tgt) {
    if (int rc = round_kernels(ctx, P, Bp, nullptr, n_tiles, 0, true, ctx->lin_factor, ctx->lin_robust, 0.f, rows)) return rc;
  } else {
    n_tiles = 0;
    std::vector<uint4> none(B, make_uint4(0, 0, 0, 0));
    CU(cudaMemcpyAsync(ctx->b_members.p, none.data(), B * sizeof(uint4), cudaMemcpyHostToDevice, ctx->stream));
  }
  CU(launch_batch_segment(Bp, static_cast<uint32_t>(B), false, nullptr, ctx->b_out.as<double>(), ctx->stream));
  ctx->launches += 1;
  return 0;
}

// Sizes everything a call on the members of b_offsets touches (so that no round allocates), clears their per-member state and
// correspondences: a new batch and a new pairing start alike.
int reserve_members(sgb_ctx* ctx) {
  const size_t n_members = batch_members(ctx), B = std::max<size_t>(n_members, 1), nn = std::max<size_t>(batch_points(ctx), 1);
  ctx->b_lin.assign(n_members, 0);
  ctx->b_seeded.assign(n_members, 0);
  CU(ctx->b_poses.reserve(B * 12 * sizeof(double)));
  CU(ctx->b_lin_poses.reserve(B * 12 * sizeof(double)));
  CU(ctx->b_members.reserve(B * sizeof(uint4)));
  CU(ctx->b_tiles.reserve(max_tiles(ctx) * sizeof(BatchTile)));
  CU(ctx->b_partials.reserve(max_tiles(ctx) * kPartialStride * sizeof(double)));
  CU(ctx->b_out.reserve(B * 44 * sizeof(double)));
  CU(ctx->b_corr.reserve(nn * sizeof(uint32_t)));
  CU(ctx->b_vq.reserve(nn * sizeof(float4)));
  CU(ctx->b_vcorr.reserve(nn * sizeof(uint32_t)));
  CU(cudaMemsetAsync(ctx->b_corr.p, 0xFF, nn * sizeof(uint32_t), ctx->stream));  // no correspondences before the first linearize
  // sgb_align_batch_async: its per-member state, round descriptor and seed flags (cleared by its first call: b_dseed_ok)
  CU(ctx->b_state.reserve(B * sizeof(MemberState)));
  CU(ctx->b_phase.reserve(B));
  CU(ctx->b_dseed.reserve(B));
  CU(ctx->b_round.reserve(sizeof(BatchRound)));
  ctx->b_dseed_ok = false;
  return reserve_query_scratch(ctx, nn);
}

// The batch's members become n_members replicas of its stored clouds (member p = cloud clouds[p], or cloud p), against map maps[p]
// each if maps is given: what sgb_source_set_pairs does, and the member side of sgb_source_set_submaps.  who names the caller.
int pair_members(sgb_ctx* ctx, const char* who, size_t n_members, const uint32_t* clouds, const uint32_t* maps) {
  if (ctx->src_state != SourceState::Batch) return fail(ctx, 1, std::string(who) + ": the context holds no batch of sources (call sgb_source_set_batch)");
  if (n_members > SGB_BATCH_MAX_MEMBERS)
    return fail(ctx, 1, std::string(who) + ": " + std::to_string(n_members) + " members, at most " + std::to_string(SGB_BATCH_MAX_MEMBERS));
  const std::vector<size_t>& coff = ctx->b_cloud_offsets;
  const size_t N = coff.size() - 1, P = n_members;
  if (!clouds && P != N)
    return fail(ctx, 1, std::string(who) + ": without a cloud table member p is cloud p, so the member count (" + std::to_string(P) +
                            ") must equal the cloud count (" + std::to_string(N) + ")");
  // the device table: member offsets [P + 1] | cloud of each member [P] | map of each member [P] (only with maps)
  std::vector<uint32_t> tab(2 * P + 1 + (maps ? P : 0));
  std::vector<size_t> member_off(P + 1, 0);
  uint32_t max_map = 0;
  for (size_t p = 0; p < P; p++) {
    const size_t c = clouds ? clouds[p] : p;
    if (c >= N)
      return fail(ctx, 1, std::string(who) + ": member " + std::to_string(p) + " names cloud " + std::to_string(c) + " but the batch holds " +
                              std::to_string(N) + " clouds");
    member_off[p + 1] = member_off[p] + (coff[c + 1] - coff[c]);
    if (member_off[p + 1] >= (1ull << 31)) return fail(ctx, 1, std::string(who) + ": too many member points (at most 2^31 - 1 in all)");
    tab[P + 1 + p] = static_cast<uint32_t>(c);
    if (maps) {
      tab[2 * P + 1 + p] = maps[p];
      max_map = std::max(max_map, maps[p]);
    }
  }
  for (size_t p = 0; p <= P; p++) tab[p] = static_cast<uint32_t>(member_off[p]);
  const size_t n = member_off[P];
  CU(cudaSetDevice(ctx->device));
  begin_pairs(ctx);
  ctx->b_offsets = member_off;
  ctx->b_pair_has_maps = maps != nullptr;
  if (maps) ctx->b_pair_maps.assign(maps, maps + P);
  ctx->b_pair_clouds.resize(P);
  for (size_t p = 0; p < P; p++) ctx->b_pair_clouds[p] = clouds ? clouds[p] : static_cast<uint32_t>(p);
  ctx->b_pair_max_map = max_map;
  const size_t B = std::max<size_t>(P, 1), nn = std::max<size_t>(n, 1);
  if (int rc = reserve_members(ctx)) return rc;
  CU(ctx->p_tables.reserve(tab.size() * sizeof(uint32_t)));
  CU(ctx->p_pts.reserve(nn * sizeof(float4)));
  CU(ctx->p_perm.reserve(nn * sizeof(uint32_t)));
  CU(ctx->p_centres.reserve(B * 4 * sizeof(double)));
  CU(ctx->p_bounds.reserve(B * 6 * sizeof(double)));
  if (ctx->src_has_covs) {
    CU(ctx->p_covA.reserve(nn * sizeof(float4)));
    CU(ctx->p_covB.reserve(nn * sizeof(float4)));
  }
  if (maps) {  // the view of whatever many-maps target the calls meet (pair_view)
    CU(ctx->v_centres.reserve(B * 4 * sizeof(double)));
    CU(ctx->v_tables.reserve((2 * B + 1) * sizeof(uint32_t)));
    CU(ctx->v_regions.reserve(B * sizeof(uint4)));
  }
  if (P == 0) return 0;
  // pageable host memory: the copy is staged before cudaMemcpyAsync returns
  CU(cudaMemcpyAsync(ctx->p_tables.p, tab.data(), tab.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  PairGather g = {};
  g.n = static_cast<uint32_t>(n);
  g.n_members = static_cast<uint32_t>(P);
  g.member_off = ctx->p_tables.as<uint32_t>();
  g.clouds = g.member_off + P + 1;
  g.cloud_off = ctx->b_cloud_off.as<uint32_t>();
  g.pts = ctx->src_pts.as<float4>();
  g.covA = ctx->src_has_covs ? ctx->src_covA.as<float4>() : nullptr;
  g.covB = ctx->src_covB.as<float4>();
  g.perm = ctx->src_perm.as<uint32_t>();
  g.centres = ctx->b_centres.as<double>();
  g.bounds = ctx->b_bounds.as<double>();
  g.out_pts = ctx->p_pts.as<float4>();
  g.out_covA = ctx->p_covA.as<float4>();
  g.out_covB = ctx->p_covB.as<float4>();
  g.out_perm = ctx->p_perm.as<uint32_t>();
  g.out_centres = ctx->p_centres.as<double>();
  g.out_bounds = ctx->p_bounds.as<double>();
  CU(launch_pair_gather(g, ctx->sm_count, ctx->stream));
  ctx->launches += 1;
  return 0;
}

// ---- the device loops of sgb_align_batch_async, sgb_align_joint_async, sgb_align_batch_gnc_async and sgb_align_joint_gnc_async (DESIGN.md
// §11 "Asynchronous align", "Asynchronous joint windows", "Asynchronous graduated non-convexity", "... for joint windows") ----

// the kernel parameters every round of the device loop shares (those of linearize_round; error() reads the same ones)
void round_params(sgb_ctx* ctx, const sgb_align_options* o, LinParams& P, BatchParams& Bp) {
  fill_params(ctx, P, kIdentity);
  Bp = batch_params(ctx, P);
  Bp.max_dist_sq_d = o->rejector_kind == SGB_REJECT_DISTANCE ? o->max_dist_sq : DBL_MAX;
  Bp.robust_c = o->robust_c;
}

// The head of one round of a device loop on ctx->stream: planner, search, factor, per-member sums into b_out.  Every grid is sized for
// the worst case (every tile, every point, every member); what the round does is read from b_round.  The caller's step follows.  rows
// (null: none): the factor kernel's per-point rows too (sgb_align_batch_gnc_async's reweighting round).
int round_head(sgb_ctx* ctx, const sgb_align_options* o, cudaGraphConditionalHandle loop, const BatchRows* rows = nullptr) {
  const size_t B = batch_members(ctx);
  const uint32_t T = static_cast<uint32_t>(max_tiles(ctx));
  const bool voxel = voxel_target(ctx), no_target = ctx->n_tgt == 0, point = !no_target && !voxel && !ctx->b_submaps && ctx->tgt_state != TargetState::KdTrees;
  BatchRound* round = ctx->b_round.as<BatchRound>();
  LinParams P;
  BatchParams Bp;
  round_params(ctx, o, P, Bp);
  BatchPlan pl = {};
  pl.n_members = static_cast<uint32_t>(B);
  pl.member_off = (ctx->b_paired ? ctx->p_tables : ctx->b_cloud_off).as<uint32_t>();
  pl.phase = ctx->b_phase.as<uint8_t>();
  pl.seeded = ctx->b_dseed.as<uint8_t>();
  pl.seeds = !voxel;
  pl.no_target = no_target;
  pl.tiles = ctx->b_tiles.as<BatchTile>();
  pl.members = ctx->b_members.as<uint4>();
  pl.round = round;
  pl.loop = loop;
  if (point) {
    int k = 0;
    if (ctx->grid_ready) {
      pl.zero[k] = ctx->grid_pending.as<uint32_t>(), pl.zero_n[k++] = 2;
      if (ctx->use_chunk_classes) pl.zero[k] = ctx->chunk_lists.as<uint32_t>(), pl.zero_n[k++] = 8;
    }
    if (ctx->use_packet_queue) pl.zero[k] = ctx->packet_queue.as<uint32_t>(), pl.zero_n[k++] = 2;
  }
  CU(launch_batch_plan(pl, ctx->stream));
  if (no_target) {
    CU(launch_batch_unmatch(Bp, round, T, ctx->stream));
  } else if (int rc = round_kernels(ctx, P, Bp, round, T, static_cast<uint32_t>(batch_points(ctx)), false, o->factor_kind, o->robust_kind,
                                    search_bound(o->rejector_kind, o->max_dist_sq), rows)) {
    return rc;
  }
  CU(launch_batch_segment(Bp, static_cast<uint32_t>(B), true, round, ctx->b_out.as<double>(), ctx->stream));
  return 0;
}

// A conditional handle for a WHILE node of g (null: the graph ctx->stream is being captured into); its condition starts at 1 at every
// launch of g.  Made before the node when kernels captured ahead of the node set it (a loop nested in a loop's body).
int loop_handle(sgb_ctx* ctx, const char* who, cudaGraph_t g, cudaGraphConditionalHandle* h) {
  if (!g) {
    cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
    CU(cudaStreamGetCaptureInfo(ctx->stream, &capture, nullptr, &g, nullptr, nullptr));
  }
  const cudaError_t e = cudaGraphConditionalHandleCreate(h, g, 1, cudaGraphCondAssignDefault);
  if (e != cudaSuccess)
    return fail(ctx, 2, std::string(who) + ": cudaGraphConditionalHandleCreate: " + cudaGetErrorString(e) +
                            " (the device loop needs conditional graph nodes: CUDA 12.4 or later, driver included)");
  return 0;
}

// A WHILE node of h in g (after deps) whose body is whatever body(h) enqueues on ctx->stream, captured on a capture stream of the context:
// cap_stream, or cap_stream_nested for the body of a loop nested in a body being captured on cap_stream.
template <typename Body>
int add_loop(sgb_ctx* ctx, cudaGraph_t g, const std::vector<cudaGraphNode_t>& deps, cudaGraphConditionalHandle h, cudaGraphNode_t* node, Body body) {
  cudaGraphNodeParams np = {};
  np.type = cudaGraphNodeTypeConditional;
  np.conditional.handle = h;
  np.conditional.type = cudaGraphCondTypeWhile;
  np.conditional.size = 1;
  CU(cudaGraphAddNode(node, g, deps.empty() ? nullptr : deps.data(), deps.size(), &np));
  cudaStream_t& cap = ctx->cap_stream && ctx->stream == ctx->cap_stream ? ctx->cap_stream_nested : ctx->cap_stream;
  if (!cap) CU(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking));
  CU(cudaStreamBeginCaptureToGraph(cap, np.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed));
  const cudaStream_t user = ctx->stream;
  ctx->stream = cap;
  const int rc = body(h);
  ctx->stream = user;
  cudaGraph_t captured = nullptr;
  const cudaError_t e = cudaStreamEndCapture(cap, &captured);
  if (rc) return rc;
  CU(e);
  return 0;
}

// While ctx->stream is being captured: a WHILE node of h (add_loop) joins the capture after what it already holds
template <typename Body>
int capture_loop(sgb_ctx* ctx, cudaGraphConditionalHandle h, Body body) {
  cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
  cudaGraph_t g = nullptr;
  const cudaGraphNode_t* d = nullptr;
  size_t nd = 0;
  CU(cudaStreamGetCaptureInfo(ctx->stream, &capture, nullptr, &g, &d, &nd));
  const std::vector<cudaGraphNode_t> deps(d, d + nd);
  cudaGraphNode_t w = nullptr;
  if (int rc = add_loop(ctx, g, deps, h, &w, body)) return rc;
  CU(cudaStreamUpdateCaptureDependencies(ctx->stream, &w, 1, cudaStreamSetCaptureDependencies));
  return 0;
}

// The body of a loop of rounds: round_head, then step(loop), which sets the condition again while a member (or window) has a round to
// go (the planner clears it)
template <typename Step>
auto round_loop(sgb_ctx* ctx, const sgb_align_options* o, Step step) {
  return [=](cudaGraphConditionalHandle h) {
    if (int rc = round_head(ctx, o, h)) return rc;
    return step(h);
  };
}

// One launch of a device loop on ctx->stream.  While the stream is captured the WHILE node joins the capture (capture_loop); otherwise
// the instantiated graph cached in graph is launched, rebuilt first when key (everything the loop captured) differs from graph's.
template <typename Body>
int launch_loop(sgb_ctx* ctx, const char* who, bool capturing, std::vector<unsigned char> key, LoopGraph& graph, Body body) {
  if (capturing) {
    cudaGraphConditionalHandle h;
    if (int rc = loop_handle(ctx, who, nullptr, &h)) return rc;
    return capture_loop(ctx, h, body);
  }
  if (!graph.exec || key != graph.key) {
    graph.drop();
    cudaGraph_t g = nullptr;
    CU(cudaGraphCreate(&g, 0));
    cudaGraphConditionalHandle h;
    cudaGraphNode_t w = nullptr;
    int rc = loop_handle(ctx, who, g, &h);
    if (!rc) rc = add_loop(ctx, g, {}, h, &w, body);
    const cudaError_t e = rc ? cudaSuccess : cudaGraphInstantiate(&graph.exec, g, 0);
    cudaGraphDestroy(g);
    if (rc) return rc;
    CU(e);
    graph.key.swap(key);
  }
  CU(cudaGraphLaunch(graph.exec, ctx->stream));
  return 0;
}

// the search counters are left cleared after a device loop, as the synchronous calls expect them
int clear_search_counters(sgb_ctx* ctx) {
  if (ctx->grid_ready) {
    CU(cudaMemsetAsync(ctx->grid_pending.p, 0, 2 * sizeof(uint32_t), ctx->stream));
    if (ctx->use_chunk_classes) CU(cudaMemsetAsync(ctx->chunk_lists.p, 0, 8 * sizeof(uint32_t), ctx->stream));
  }
  if (ctx->use_packet_queue && ctx->packet_queue.p) CU(cudaMemsetAsync(ctx->packet_queue.p, 0, 2 * sizeof(uint32_t), ctx->stream));
  return 0;
}

// Everything the cached loop graph captured: option values, sizes, the search configuration and every buffer address.
template <typename T>
void key_add(std::vector<unsigned char>& k, const T& v) {
  const unsigned char* b = reinterpret_cast<const unsigned char*>(&v);
  k.insert(k.end(), b, b + sizeof(T));
}
std::vector<unsigned char> loop_key(sgb_ctx* ctx, const sgb_align_options* o) {
  std::vector<unsigned char> k;
  for (int v : {o->factor_kind, o->robust_kind, o->rejector_kind, o->optimizer_kind, o->max_iterations, o->max_inner_iterations}) key_add(k, v);
  for (double v : {o->robust_c, o->max_dist_sq, o->gn_lambda, o->init_lambda, o->lambda_factor, o->rotation_eps, o->translation_eps}) key_add(k, v);
  for (int i = 0; i < 6; i++) key_add(k, o->dof_mask[i]);
  LinParams P;
  BatchParams Bp = {};
  round_params(ctx, o, P, Bp);
  key_add(k, P);
  key_add(k, Bp);
  for (size_t v : {batch_members(ctx), batch_points(ctx), ctx->n_tgt, ctx->kt_maps, ctx->vm_maps})
    key_add(k, v);
  for (int v : {static_cast<int>(ctx->tgt_state), static_cast<int>(ctx->b_submaps), static_cast<int>(ctx->b_paired), static_cast<int>(paired_maps(ctx)),
                static_cast<int>(ctx->grid_ready), static_cast<int>(ctx->use_chunk_classes), static_cast<int>(ctx->use_packet_queue),
                static_cast<int>(ctx->use_ring), ctx->pending_div, ctx->tree_depth, ctx->kt_depth, ctx->sm_count, static_cast<int>(ctx->grid_capacity),
                static_cast<int>(ctx->class_fallback_pct)})
    key_add(k, v);
  for (float v : {ctx->grid_origin[0], ctx->grid_origin[1], ctx->grid_origin[2], ctx->grid_inv_cell, ctx->grid_settle_d2, ctx->grid_cell, ctx->class_wide_cells})
    key_add(k, v);
  for (const DevBuf* b : {&ctx->b_round, &ctx->b_dseed, &ctx->b_state, &ctx->b_phase, &ctx->b_vq, &ctx->b_vcorr, &ctx->b_out, &ctx->p_tables, &ctx->b_cloud_off,
                          &ctx->grid_pts, &ctx->grid_table, &ctx->grid_state, &ctx->grid_pending, &ctx->grid_pending_q, &ctx->chunk_lists, &ctx->packet_queue,
                          &ctx->tgt_pnodes, &ctx->kt_tables, &ctx->kt_centres, &ctx->vm_centres, &ctx->vm_regions, &ctx->v_tables, &ctx->v_centres,
                          &ctx->v_regions, &ctx->s_tables, &ctx->s_entries, &ctx->s_centres, &ctx->b_centry})
    key_add(k, b->p);
  // the weighted factor kernel and the address it reads: a replay reads whatever weights are in force there
  key_add(k, static_cast<int>(ctx->b_weighted));
  key_add(k, ctx->b_weights.p);
  return k;
}

// p is device memory of the context's GPU (cudaPointerGetAttributes)
bool on_device(const sgb_ctx* ctx, const void* p) {
  cudaPointerAttributes a = {};
  const cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) cudaGetLastError();  // (not an error of the context: clear it)
  return e == cudaSuccess && a.type == cudaMemoryTypeDevice && a.device == ctx->device;
}

// The check of who's device-memory arguments: each given one (a required one always) must be device memory of the context's GPU
struct DeviceArg {
  const void* p;
  const char* name;
  bool required;
};
int device_pointers(sgb_ctx* ctx, const std::string& who, std::initializer_list<DeviceArg> args) {
  for (const DeviceArg& a : args)
    if ((a.required || a.p) && !on_device(ctx, a.p))
      return fail(ctx, 1, who + ": " + a.name + " must be device memory of the context's GPU (cuda:" + std::to_string(ctx->device) +
                              "); host, page-locked and managed memory are refused");
  return 0;
}

// Whether ctx->stream is being captured (an invalidated capture fails who's call)
int capture_state(sgb_ctx* ctx, const std::string& who, bool* capturing) {
  cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
  CU(cudaStreamIsCapturing(ctx->stream, &capture));
  if (capture == cudaStreamCaptureStatusInvalidated) return fail(ctx, 1, who + ": the context's stream is in an invalidated capture");
  *capturing = capture == cudaStreamCaptureStatusActive;
  return 0;
}

// The checks both align calls make before anything is launched (who names the caller), and the options of the optimiser's step
int align_checks(sgb_ctx* ctx, const char* who, const sgb_align_options* o, const double* init_T, const double* out_T, const double* out_info,
                 AlignOptions& ao) {
  if (int rc = batch_check(ctx, who, init_T)) return rc;
  if (!o) return fail(ctx, 1, std::string(who) + ": null options");
  if (!out_T || !out_info) return fail(ctx, 1, std::string(who) + ": null output");
  if (o->factor_kind < 0 || o->factor_kind > 2 || o->robust_kind < 0 || o->robust_kind > 2 || o->rejector_kind < 0 || o->rejector_kind > 1 ||
      o->optimizer_kind < 0 || o->optimizer_kind > 1)
    return fail(ctx, 1, std::string(who) + ": invalid factor/robust/rejector/optimizer kind");
  if (int rc = submap_factor_check(ctx, who, o->factor_kind)) return rc;
  if (batch_points(ctx) && ctx->n_tgt) {  // (an empty batch has no points)
    if (int rc = check_target(ctx, who, o->factor_kind)) return rc;
  }
  ao.lm = o->optimizer_kind == SGB_OPT_LEVENBERG_MARQUARDT;
  ao.max_iterations = o->max_iterations;
  ao.max_inner_iterations = o->max_inner_iterations;
  ao.gn_lambda = o->gn_lambda;
  ao.init_lambda = o->init_lambda;
  ao.lambda_factor = o->lambda_factor;
  ao.rotation_eps = o->rotation_eps;
  ao.translation_eps = o->translation_eps;
  for (int i = 0; i < 6; i++) ao.dof_mask[i] = o->dof_mask[i];
  return 0;
}

// ---- sgb_linearize_batch_points / sgb_error_batch_points (DESIGN.md §11 "Per-point terms") ----

// the tables that map a stored point to the caller's row (batch_row): the pairing's member offsets and replicas' order, else the clouds'
void row_layout(const sgb_ctx* ctx, const uint32_t*& member_off, const uint32_t*& perm) {
  member_off = (ctx->b_paired ? ctx->p_tables : ctx->b_cloud_off).as<uint32_t>();
  perm = (ctx->b_paired ? ctx->p_perm : ctx->src_perm).as<uint32_t>();
}

// Where the factor kernel writes the rows of one call: the caller's buffers when they are device memory of the context's GPU, else the
// context's staging buffers (copy_rows copies them out).  The rows the kernel does not reach -- every point of an inactive member, and of
// every member against an empty target -- are cleared here; rejected and unmatched points get zero rows from the kernel itself.
int point_rows(sgb_ctx* ctx, const uint8_t* active, double* out_e, double* out_Hb, BatchRows& rows) {
  const size_t B = batch_members(ctx), nn = std::max<size_t>(batch_points(ctx), 1);
  rows = BatchRows{};
  row_layout(ctx, rows.member_off, rows.perm);
  if (out_e && on_device(ctx, out_e)) {
    rows.e = out_e;
  } else if (out_e) {
    CU(ctx->b_rows_e.reserve(nn * sizeof(double)));
    rows.e = ctx->b_rows_e.as<double>();
  }
  if (out_Hb && on_device(ctx, out_Hb)) {
    rows.Hb = out_Hb;
  } else if (out_Hb) {
    CU(ctx->b_rows_hb.reserve(nn * 42 * sizeof(double)));
    rows.Hb = ctx->b_rows_hb.as<double>();
  }
  const auto reached = [&](size_t m) { return ctx->n_tgt && (!active || active[m]); };
  for (size_t m = 0; m < B;) {  // runs of consecutive members the kernel does not reach: their rows are contiguous
    size_t end = m;
    while (end < B && !reached(end)) end++;
    if (end == m) {
      m++;
      continue;
    }
    const size_t first = ctx->b_offsets[m], n = ctx->b_offsets[end] - first;
    if (n && rows.e) CU(cudaMemsetAsync(rows.e + first, 0, n * sizeof(double), ctx->stream));
    if (n && rows.Hb) CU(cudaMemsetAsync(rows.Hb + 42 * first, 0, 42 * n * sizeof(double), ctx->stream));
    m = end;
  }
  return 0;
}

int copy_rows(sgb_ctx* ctx, const BatchRows& rows, double* out_e, double* out_Hb) {
  const size_t n = batch_points(ctx);
  if (n && out_e && rows.e != out_e) CU(cudaMemcpyAsync(out_e, rows.e, n * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (n && out_Hb && rows.Hb != out_Hb) CU(cudaMemcpyAsync(out_Hb, rows.Hb, 42 * n * sizeof(double), cudaMemcpyDefault, ctx->stream));
  return 0;
}

// sgb_linearize_batch (who, no rows) and sgb_linearize_batch_points (points: rows to out_e and / or out_Hb)
int linearize_batch(sgb_ctx* ctx, const char* who, bool points, int factor, int robust, double robust_c, int rejector, double max_dist_sq, const double* T,
                    const uint8_t* active, double* out44, double* out_e, double* out_Hb) {
  if (!ctx) return 1;
  const std::string w = who;
  if (int rc = batch_check(ctx, who, T)) return rc;
  if (factor < 0 || factor > 2 || robust < 0 || robust > 2 || rejector < 0 || rejector > 1) return fail(ctx, 1, w + ": invalid factor/robust/rejector kind");
  if (!out44) return fail(ctx, 1, w + ": null output");
  if (points && !out_e && !out_Hb) return fail(ctx, 1, w + ": null per-point outputs (out_point_e and out_point_Hb42 both NULL; sgb_linearize_batch gives the sums alone)");
  if (int rc = submap_factor_check(ctx, who, factor)) return rc;
  const size_t B = batch_members(ctx);
  if (B == 0) return 0;
  if (batch_points(ctx) && ctx->n_tgt) {
    if (int rc = check_target(ctx, who, factor)) return rc;
  }
  if (int rc = pair_view(ctx)) return rc;
  BatchRows rows;
  if (points) {
    if (int rc = point_rows(ctx, active, out_e, out_Hb, rows)) return rc;
  }
  if (int rc = linearize_round(ctx, factor, robust, robust_c, rejector, max_dist_sq, T, active, points ? &rows : nullptr)) return rc;
  if (points) {
    if (int rc = copy_rows(ctx, rows, out_e, out_Hb)) return rc;
  }
  return copy_out(ctx, out44, 44 * B);
}

// sgb_error_batch (who, no rows) and sgb_error_batch_points (points: rows to out_e)
int error_batch(sgb_ctx* ctx, const char* who, bool points, const double* T, const uint8_t* active, double* out, double* out_e) {
  if (!ctx) return 1;
  const std::string w = who;
  if (int rc = batch_check(ctx, who, T)) return rc;
  if (!out) return fail(ctx, 1, w + ": null output");
  if (points && !out_e) return fail(ctx, 1, w + ": null per-point output (out_point_e; sgb_error_batch gives the sums alone)");
  const size_t B = batch_members(ctx);
  if (B == 0) return 0;
  if (!ctx->have_lin) return fail(ctx, 1, w + ": no preceding sgb_linearize_batch (the correspondences are cached there)");
  for (size_t m = 0; m < B; m++)
    if ((!active || active[m]) && !ctx->b_lin[m])
      return fail(ctx, 1, w + ": member " + std::to_string(m) + " is active but has not been linearised against the current target");
  if (int rc = pair_view(ctx)) return rc;
  BatchRows rows;
  if (points) {
    if (int rc = point_rows(ctx, active, out_e, nullptr, rows)) return rc;
  }
  if (int rc = error_round(ctx, T, active, points ? &rows : nullptr)) return rc;
  if (points) {
    if (int rc = copy_rows(ctx, rows, out_e, nullptr)) return rc;
  }
  return copy_out(ctx, out, B);
}

// The initial state and poses of sgb_align_batch: the only upload of poses in the whole align
int align_start(sgb_ctx* ctx, const AlignOptions& ao, const double* init_T, std::vector<MemberState>& state, std::vector<uint8_t>& phase) {
  const size_t B = batch_members(ctx);
  state.resize(B);
  phase.resize(B);
  std::vector<double> poses(12 * B);
  for (size_t m = 0; m < B; m++) {
    align_init(ao, init_T + 16 * m, state[m]);
    pose_from_colmajor(init_T + 16 * m, poses.data() + 12 * m);
    phase[m] = static_cast<uint8_t>(state[m].phase);
  }
  CU(ctx->b_state.reserve(B * sizeof(MemberState)));
  CU(ctx->b_phase.reserve(B));
  CU(cudaMemcpyAsync(ctx->b_state.p, state.data(), B * sizeof(MemberState), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(ctx->b_poses.p, poses.data(), poses.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  return 0;
}

// The outputs of an align from the members' final state
void align_results(const std::vector<MemberState>& state, double* out_T, double* out_info, double* out_Hb) {
  for (size_t m = 0; m < state.size(); m++) {
    const MemberState& s = state[m];
    std::memcpy(out_T + 16 * m, s.T, 16 * sizeof(double));
    double* info = out_info + 4 * m;
    info[0] = s.converged ? 1.0 : 0.0;
    info[1] = s.iterations;
    info[2] = s.inliers;
    info[3] = s.e;
    if (out_Hb) {
      std::memcpy(out_Hb + 42 * m, s.H, 36 * sizeof(double));
      std::memcpy(out_Hb + 42 * m + 36, s.b, 6 * sizeof(double));
    }
  }
}

// The rounds of sgb_align_batch from the members' phases (read back after each round), in lockstep: error() for every member with a
// pending trial until none has one, else a linearize of every member still iterating; each round ends with one step launch, step(lin).
// The host only reads the phases to build the next round's tile tables.
template <typename Step>
int align_rounds(sgb_ctx* ctx, const sgb_align_options* o, std::vector<uint8_t>& phase, Step step) {
  const size_t B = batch_members(ctx);
  std::vector<uint8_t> active(B);
  for (;;) {
    bool any_trial = false, any_lin = false;
    for (size_t m = 0; m < B; m++) {
      any_trial |= phase[m] == kPhaseTrial;
      any_lin |= phase[m] == kPhaseLinearize;
    }
    if (!any_trial && !any_lin) return 0;
    const bool lin = !any_trial;
    for (size_t m = 0; m < B; m++) active[m] = phase[m] == (lin ? kPhaseLinearize : kPhaseTrial);
    if (lin) {
      if (int rc = linearize_round(ctx, o->factor_kind, o->robust_kind, o->robust_c, o->rejector_kind, o->max_dist_sq, nullptr, active.data())) return rc;
    } else {
      if (int rc = error_round(ctx, nullptr, active.data())) return rc;
    }
    CU(step(lin));
    ctx->launches += 1;
    CU(cudaMemcpyAsync(phase.data(), ctx->b_phase.p, B, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
}

// A GNC align: the weights its rounds use in place of those in force, until the call returns however it returns
struct RoundWeights {
  sgb_ctx* ctx;
  explicit RoundWeights(sgb_ctx* c) : ctx(c) { ctx->b_wround = true; }
  ~RoundWeights() {
    ctx->b_wround = false;
    ctx->b_wuse = nullptr;
  }
  void use(const double* w) { ctx->b_wuse = w; }
};

// The checks of the GNC options every GNC align makes (who names the caller), after those of its align
int gnc_option_checks(sgb_ctx* ctx, const std::string& who, const sgb_align_options* o, const sgb_gnc_options* gnc) {
  if (!gnc) return fail(ctx, 1, who + ": null GNC options");
  if (o->robust_kind != SGB_ROBUST_NONE)
    return fail(ctx, 1, who + ": robust_kind must be SGB_ROBUST_NONE: the GNC weights are the robust kernel (a fixed-width kernel on top would change the cost "
                              "they anneal)");
  if (gnc->kind != SGB_GNC_GEMAN_MCCLURE && gnc->kind != SGB_GNC_TLS) return fail(ctx, 1, who + ": invalid GNC kind (SGB_GNC_GEMAN_MCCLURE or SGB_GNC_TLS)");
  if (!(std::isfinite(gnc->noise_bound_sq) && gnc->noise_bound_sq > 0.0)) return fail(ctx, 1, who + ": noise_bound_sq must be finite and > 0");
  if (gnc->max_stages < 1) return fail(ctx, 1, who + ": max_stages must be >= 1");
  if (gnc->stage_iterations < 1) return fail(ctx, 1, who + ": stage_iterations must be >= 1");
  return 0;
}

// The checks both batch GNC aligns make before anything is enqueued (who names the caller): align_checks', then the GNC options'
int gnc_checks(sgb_ctx* ctx, const std::string& who, const sgb_align_options* o, const sgb_gnc_options* gnc, const double* init_T, const double* out_T,
               const double* out_info, AlignOptions& ao) {
  if (int rc = align_checks(ctx, who.c_str(), o, init_T, out_T, out_info, ao)) return rc;
  return gnc_option_checks(ctx, who, o, gnc);
}

// A synchronous GNC call refuses a captured stream: it copies its poses in and its outputs out of host memory and waits for them
int gnc_capture_check(sgb_ctx* ctx, const std::string& who) {
  bool capturing = false;
  if (int rc = capture_state(ctx, who, &capturing)) return rc;
  if (capturing)
    return fail(ctx, 1, who + ": the context's stream is being captured, and the call copies host memory and waits for its results; call it outside the "
                              "capture (or use the _async call)");
  return 0;
}

// the bytes of g_w and g_e (a double per member point) and of g_state (GncState | live flag per unit) a GNC align of n_units units
// (members or windows) uses
size_t gnc_w_bytes(const sgb_ctx* ctx) { return std::max<size_t>(batch_points(ctx), 1) * sizeof(double); }
size_t gnc_state_bytes(size_t n_units) { return n_units * (sizeof(GncState) + 1); }
bool gnc_allocates(const sgb_ctx* ctx, size_t n_units) {
  return ctx->g_w.cap < gnc_w_bytes(ctx) || ctx->g_e.cap < gnc_w_bytes(ctx) || ctx->g_state.cap < gnc_state_bytes(n_units);
}
int reserve_gnc(sgb_ctx* ctx, size_t n_units) {
  CU(ctx->g_w.reserve(gnc_w_bytes(ctx)));
  CU(ctx->g_e.reserve(gnc_w_bytes(ctx)));
  CU(ctx->g_state.reserve(gnc_state_bytes(n_units)));
  return 0;
}

// A stream-ordered align's first-use allocations, which a capture cannot hold: the packet search's queue (queue), the capture stream of
// its loop (loops = 1) and of a loop nested in it (loops = 2), and the GNC buffers of gnc_units units (0: none).  extra: the call's own
// (an upload of its tables).  Inside a capture a call that needs any fails with who + refusal; outside, the queue and the GNC buffers
// are reserved here (add_loop makes the streams).
int loop_allocations(sgb_ctx* ctx, const std::string& who, bool capturing, bool extra, bool queue, int loops, size_t gnc_units, const char* refusal) {
  const bool no_queue = queue && ctx->use_packet_queue && !ctx->packet_queue.p;
  const bool allocates = extra || no_queue || (loops > 0 && !ctx->cap_stream) || (loops > 1 && !ctx->cap_stream_nested) ||
                         (gnc_units && gnc_allocates(ctx, gnc_units));
  if (capturing && allocates) return fail(ctx, 1, who + refusal);
  if (no_queue) {
    CU(ctx->packet_queue.reserve(2 * sizeof(uint32_t)));
    CU(cudaMemsetAsync(ctx->packet_queue.p, 0, 2 * sizeof(uint32_t), ctx->stream));
  }
  return gnc_units ? reserve_gnc(ctx, gnc_units) : 0;
}

// The GNC kernels' parameters of a call over g_w, g_e and g_state (reserved for the batch)
GncParams gnc_params(sgb_ctx* ctx, const sgb_gnc_options* gnc) {
  GncParams gp = {};
  gp.n = static_cast<uint32_t>(batch_points(ctx));
  gp.n_members = static_cast<uint32_t>(batch_members(ctx));
  gp.kind = gnc->kind;
  gp.c2 = gnc->noise_bound_sq;
  gp.max_stages = gnc->max_stages;
  gp.stage_iterations = gnc->stage_iterations;
  row_layout(ctx, gp.member_off, gp.perm);
  gp.corr = ctx->b_corr.as<uint32_t>();
  gp.e = ctx->g_e.as<double>();
  gp.w = ctx->b_weighted ? ctx->b_weights.as<double>() : nullptr;
  gp.wstage = ctx->g_w.as<double>();
  gp.gnc = ctx->g_state.as<GncState>();
  gp.live = reinterpret_cast<uint8_t*>(gp.gnc + gp.n_members);
  return gp;
}

// Every one of n_units units starts its stage 0: zero GNC state (r2max = 0, no stage begun, no iterations), live
int gnc_begin(sgb_ctx* ctx, const GncParams& p, size_t n_units) {
  CU(cudaMemsetAsync(p.gnc, 0, n_units * sizeof(GncState), ctx->stream));
  CU(cudaMemsetAsync(p.live, 1, n_units, ctx->stream));
  return 0;
}

// the rows of a reweighting round: each point's e into g_e
BatchRows gnc_rows(const GncParams& p) {
  BatchRows rows = {};
  rows.member_off = p.member_off;
  rows.perm = p.perm;
  rows.e = p.e;
  return rows;
}

// The GNC part of a stage loop's key: the GNC options and every buffer the GNC kernels use (more: the call's own)
void gnc_key(std::vector<unsigned char>& k, const GncParams& p, std::initializer_list<const void*> more) {
  for (int v : {p.kind, p.max_stages, p.stage_iterations}) key_add(k, v);
  key_add(k, p.c2);
  for (const void* v : {static_cast<const void*>(p.member_off), static_cast<const void*>(p.perm), static_cast<const void*>(p.corr),
                        static_cast<const void*>(p.e), static_cast<const void*>(p.w), static_cast<const void*>(p.wstage), static_cast<const void*>(p.gnc),
                        static_cast<const void*>(p.live)})
    key_add(k, v);
  for (const void* v : more) key_add(k, v);
}

// The stream-ordered GNC of both batch GNC aligns, after their checks (who names the caller; capturing: ctx->stream is being captured):
// the stages and their rounds as one device loop from the poses at d_init_T, the outputs to d_out_T, d_out_info and, unless null, d_out_Hb,
// d_out_gnc2 (device memory) and out_point_w (host or device memory).
int batch_gnc_enqueue(sgb_ctx* ctx, const char* who, bool capturing, const sgb_align_options* o, const sgb_gnc_options* gnc, const AlignOptions& ao,
                      const double* d_init_T, double* d_out_T, double* d_out_info, double* d_out_Hb, double* d_out_gnc2, double* out_point_w) {
  const size_t B = batch_members(ctx), n = batch_points(ctx);
  // the GNC buffers, the packet queue and both capture streams (the stages' loop and the rounds' loop nested in it)
  if (int rc = loop_allocations(ctx, who, capturing, false, true, 2, B,
                                ": this call needs an allocation, which a capture cannot hold; call it once outside the capture first"))
    return rc;
  if (int rc = pair_view(ctx)) return rc;
  const GncParams gp = gnc_params(ctx, gnc);
  const BatchRows rows = gnc_rows(gp);
  const uint32_t nb = static_cast<uint32_t>(B);
  MemberState* state = ctx->b_state.as<MemberState>();
  double* poses = ctx->b_poses.as<double>();
  uint8_t* phase = ctx->b_phase.as<uint8_t>();
  // the initial state: every member's align_init at its initial pose, zero GNC state, every member live (the seed flags kept as
  // sgb_align_batch_async keeps them)
  CU(launch_batch_align_init(ao, nb, d_init_T, state, poses, phase, ctx->b_dseed.as<uint8_t>(), ctx->corr_seeds && ctx->b_dseed_ok, ctx->stream));
  if (int rc = gnc_begin(ctx, gp, B)) return rc;
  ctx->launches += 3;  // the initial state here, the outputs below
  // One stage per iteration of the outer loop: the reweighting linearize of the members in the stage (planned by batch_plan_kernel from
  // their phases), the stage kernels, then the stage's align as an inner loop of rounds.  After gnc_init, gnc_loops sets both conditions:
  // the stages' while a member has a stage to go, the rounds' while a member's align has a round to go.
  RoundWeights weights(ctx);
  const auto stage = [&](cudaGraphConditionalHandle stages) {
    cudaGraphConditionalHandle rounds;
    if (int rc = loop_handle(ctx, who, nullptr, &rounds)) return rc;
    CU(launch_gnc_reweigh(nb, gp.live, phase, rounds, ctx->stream));
    weights.use(nullptr);
    if (int rc = round_head(ctx, o, stages, &rows)) return rc;
    CU(launch_gnc_rmax(gp, ctx->sm_count, ctx->stream));
    CU(launch_gnc_stage(gp, ctx->stream));
    CU(launch_gnc_weight(gp, ctx->sm_count, ctx->stream));
    CU(launch_gnc_init(gp, ao, state, poses, phase, ctx->stream));
    CU(launch_gnc_loops(nb, gp.live, phase, stages, rounds, ctx->stream));
    weights.use(gp.wstage);
    return capture_loop(ctx, rounds, round_loop(ctx, o, [&](cudaGraphConditionalHandle h) {
                          CU(launch_gnc_step(gp, ao, ctx->b_round.as<BatchRound>(), h, ctx->b_out.as<double>(), state, poses, phase, ctx->stream));
                          return 0;
                        }));
  };
  std::vector<unsigned char> key;
  if (!capturing) {  // loop_key, plus the GNC options and every buffer the GNC kernels use
    key = loop_key(ctx, o);
    gnc_key(key, gp, {});
  }
  if (int rc = launch_loop(ctx, who, capturing, std::move(key), ctx->gnc_loop, stage)) return rc;
  ctx->launches += 1;
  if (int rc = clear_search_counters(ctx)) return rc;
  CU(launch_batch_align_finish(nb, state, d_out_T, d_out_info, d_out_Hb, ctx->stream));
  CU(launch_gnc_finish(nb, state, gp.gnc, d_out_info, d_out_gnc2, ctx->stream));
  if (out_point_w && n) CU(cudaMemcpyAsync(out_point_w, gp.e, n * sizeof(double), cudaMemcpyDefault, ctx->stream));
  ctx->b_dseed_ok = true;
  // stage 0's reweighting round linearised every member; every round since used robust_kind (NONE)
  mark_linearised(ctx, o->factor_kind, o->robust_kind, o->robust_c, nullptr);
  return 0;
}

// The outputs of a synchronous GNC align from where it staged them to the caller's (host or device memory; a null one is skipped), then
// the call's one synchronisation
struct Staged {
  double* out;
  const double* staged;
  size_t doubles;
};
int copy_staged(sgb_ctx* ctx, std::initializer_list<Staged> outputs) {
  for (const Staged& s : outputs)
    if (s.out) CU(cudaMemcpyAsync(s.out, s.staged, s.doubles * sizeof(double), cudaMemcpyDefault, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

}  // namespace

extern "C" {

int sgb_source_set_batch(sgb_ctx* ctx, size_t n_members, const size_t* offsets, const double* points, const double* covs) {
  if (!ctx) return 1;
  if (n_members > SGB_BATCH_MAX_MEMBERS)
    return fail(ctx, 1, "sgb_source_set_batch: " + std::to_string(n_members) + " members, at most " + std::to_string(SGB_BATCH_MAX_MEMBERS));
  if (!offsets) return fail(ctx, 1, "sgb_source_set_batch: null offsets");
  if (offsets[0] != 0) return fail(ctx, 1, "sgb_source_set_batch: offsets[0] must be 0");
  for (size_t m = 0; m < n_members; m++)
    if (offsets[m + 1] < offsets[m]) return fail(ctx, 1, "sgb_source_set_batch: offsets must be ascending (member " + std::to_string(m) + ")");
  const size_t n = offsets[n_members];
  if (n >= (1ull << 31)) return fail(ctx, 1, "sgb_source_set_batch: too many points");
  if (n && !points) return fail(ctx, 1, "sgb_source_set_batch: null points");
  CU(cudaSetDevice(ctx->device));
  begin_source(ctx, SourceState::Batch, 0, covs != nullptr);
  ctx->b_cloud_offsets.assign(offsets, offsets + n_members + 1);
  ctx->b_offsets = ctx->b_cloud_offsets;  // no pairing: the members are the clouds
  const size_t B = std::max<size_t>(n_members, 1), nn = std::max<size_t>(n, 1);
  CU(ctx->b_centres.reserve(B * 4 * sizeof(double)));
  CU(ctx->b_bounds.reserve(B * 6 * sizeof(double)));
  if (int rc = reserve_members(ctx)) return rc;
  const std::vector<uint32_t> off32(offsets, offsets + n_members + 1);
  CU(ctx->b_cloud_off.reserve(off32.size() * sizeof(uint32_t)));
  CU(cudaMemcpyAsync(ctx->b_cloud_off.p, off32.data(), off32.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  if (n == 0) return 0;
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  CU(ctx->tmp_pts.reserve(n * sizeof(float4)));
  CU(ctx->src_pts.reserve(n * sizeof(float4)));
  CU(ctx->keys_in.reserve(n * sizeof(uint64_t)));
  CU(ctx->keys_out.reserve(n * sizeof(uint64_t)));
  CU(ctx->vals_in.reserve(n * sizeof(uint32_t)));
  CU(ctx->src_perm.reserve(n * sizeof(uint32_t)));
  CU(ctx->src_rank.reserve(n * sizeof(uint32_t)));
  CU(cudaMemcpyAsync(ctx->stage_pts.p, points, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (covs) {
    CU(ctx->stage_covs.reserve(n * 16 * sizeof(double)));
    CU(ctx->src_covA.reserve(n * sizeof(float4)));
    CU(ctx->src_covB.reserve(n * sizeof(float4)));
    CU(cudaMemcpyAsync(ctx->stage_covs.p, covs, n * 16 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  }
  // Every cloud is stored exactly as sgb_source_set_points stores one cloud: centred on its own box, rounded to FP32, sorted along the
  // curve within itself, covariances packed into its search order.  Its slice of the storage is contiguous.
  StoreClouds sc = {};
  sc.n = static_cast<uint32_t>(n);
  sc.n_clouds = static_cast<uint32_t>(n_members);
  sc.cloud_bits = 1;
  while ((1ull << sc.cloud_bits) < n_members) sc.cloud_bits++;
  sc.sm_count = ctx->sm_count;
  sc.points = ctx->stage_pts.as<double>();
  sc.covs = covs ? ctx->stage_covs.as<double>() : nullptr;
  sc.offsets = ctx->b_cloud_off.as<uint32_t>();
  sc.bounds = ctx->b_bounds.as<double>();
  sc.centres = ctx->b_centres.as<double>();
  sc.orig_pts = ctx->tmp_pts.as<float4>();
  sc.keys_a = ctx->keys_in.as<uint64_t>();
  sc.keys_b = ctx->keys_out.as<uint64_t>();
  sc.vals_a = ctx->vals_in.as<uint32_t>();
  sc.vals_b = ctx->src_rank.as<uint32_t>();
  sc.pts = ctx->src_pts.as<float4>();
  sc.covA = ctx->src_covA.as<float4>();
  sc.covB = ctx->src_covB.as<float4>();
  sc.perm = ctx->src_perm.as<uint32_t>();
  size_t key_bytes = 0, cloud_bytes = 0;
  CU(sort_pairs_u64_u32_bits(nullptr, key_bytes, sc.keys_a, sc.keys_b, sc.vals_a, sc.vals_b, n, 63, ctx->stream));
  CU(sort_pairs_u64_u32_bits(nullptr, cloud_bytes, sc.keys_a, sc.keys_b, sc.vals_b, sc.vals_a, n, sc.cloud_bits, ctx->stream));
  sc.sort_temp_bytes = std::max(key_bytes, cloud_bytes);
  CU(ctx->sort_temp.reserve(sc.sort_temp_bytes));
  sc.sort_temp = ctx->sort_temp.p;
  CU(launch_store_clouds(sc, ctx->stream));
  ctx->launches += 6;
  return 0;
}

int sgb_source_set_pairs(sgb_ctx* ctx, size_t n_members, const uint32_t* clouds, const uint32_t* maps) {
  if (!ctx) return 1;
  return pair_members(ctx, "sgb_source_set_pairs", n_members, clouds, maps);
}

}  // extern "C"

// The submap lists of n_lists owners (what: "member" or "set"), checked for who: list_off ascending from 0, fewer than 2^31 entries,
// every pose rigid.  tables = inverse entry poses [entries][12] | list_off [n_lists + 1] | entry_maps [entries] (the layout of s_tables)
int sgb::submap_lists(sgb_ctx* ctx, const std::string& who, const char* what, size_t n_lists, const size_t* list_off, const uint32_t* entry_maps,
                      const double* entry_poses16, std::vector<double>& tables, uint32_t* max_map) {
  if (!list_off) return fail(ctx, 1, who + ": null list offsets");
  if (list_off[0] != 0) return fail(ctx, 1, who + ": list_off[0] must be 0");
  for (size_t p = 0; p < n_lists; p++)
    if (list_off[p + 1] < list_off[p]) return fail(ctx, 1, who + ": list_off must be ascending (" + what + " " + std::to_string(p) + ")");
  const size_t P = n_lists, E = list_off[P];
  if (E >= (1ull << 31)) return fail(ctx, 1, who + ": too many entries (at most 2^31 - 1 in all)");
  if (E && !entry_maps) return fail(ctx, 1, who + ": null entry maps");
  // the inverse of every placement, row-major R^T | -R^T t: the kernels carry the member's pose (or the query) into the map's frame with it
  tables.assign(12 * E + (P + 1 + E + 1) / 2, 0.0);
  for (size_t j = 0; j < E; j++) {
    double R[12];
    pose_from_colmajor(entry_poses16 ? entry_poses16 + 16 * j : kIdentity, R);
    double dev = 0.0;
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) dev = std::max(dev, std::fabs(R[a] * R[b] + R[3 + a] * R[3 + b] + R[6 + a] * R[6 + b] - (a == b ? 1.0 : 0.0)));
    const double* M = entry_poses16 ? entry_poses16 + 16 * j : kIdentity;
    const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) + R[2] * (R[3] * R[7] - R[4] * R[6]);
    if (!(dev <= 1e-6) || !(det > 0.0) || M[3] != 0.0 || M[7] != 0.0 || M[11] != 0.0 || M[15] != 1.0 || !std::isfinite(R[9] + R[10] + R[11]))
      return fail(ctx, 1, who + ": the pose of entry " + std::to_string(j) + " is not a rigid transformation (rotation block orthonormal to 1e-6, last row 0 0 0 1)");
    double* inv = tables.data() + 12 * j;
    for (int a = 0; a < 3; a++) {
      for (int b = 0; b < 3; b++) inv[3 * a + b] = R[3 * b + a];
      inv[9 + a] = -(R[a] * R[9] + R[3 + a] * R[10] + R[6 + a] * R[11]);
    }
  }
  uint32_t* off = reinterpret_cast<uint32_t*>(tables.data() + 12 * E);
  *max_map = 0;
  for (size_t p = 0; p <= P; p++) off[p] = static_cast<uint32_t>(list_off[p]);
  for (size_t j = 0; j < E; j++) {
    off[P + 1 + j] = entry_maps[j];
    *max_map = std::max(*max_map, entry_maps[j]);
  }
  return 0;
}

extern "C" {

int sgb_source_set_submaps(sgb_ctx* ctx, size_t n_members, const uint32_t* clouds, const size_t* list_off, const uint32_t* entry_maps, const double* entry_poses16) {
  if (!ctx) return 1;
  const std::string who = "sgb_source_set_submaps";
  if (ctx->src_state != SourceState::Batch) return fail(ctx, 1, who + ": the context holds no batch of sources (call sgb_source_set_batch)");
  if (n_members > SGB_BATCH_MAX_MEMBERS) return fail(ctx, 1, who + ": " + std::to_string(n_members) + " members, at most " + std::to_string(SGB_BATCH_MAX_MEMBERS));
  std::vector<double> tables;
  uint32_t max_map = 0;
  if (int rc = submap_lists(ctx, who, "member", n_members, list_off, entry_maps, entry_poses16, tables, &max_map)) return rc;
  const size_t P = n_members, E = list_off[P];
  const uint32_t* off = reinterpret_cast<const uint32_t*>(tables.data() + 12 * E);
  if (int rc = pair_members(ctx, who.c_str(), P, clouds, nullptr)) return rc;
  ctx->b_submaps = true;
  ctx->b_sub_off.assign(off, off + P + 1);
  ctx->b_sub_maps.assign(entry_maps, entry_maps + E);
  ctx->b_pair_max_map = max_map;
  CU(ctx->s_tables.reserve(tables.size() * sizeof(double)));
  CU(ctx->s_entries.reserve(std::max<size_t>(E, 1) * sizeof(uint4)));
  CU(ctx->s_centres.reserve(std::max<size_t>(E, 1) * 4 * sizeof(double)));
  CU(ctx->b_centry.reserve(std::max<size_t>(batch_points(ctx), 1) * sizeof(uint32_t)));
  // pageable host memory: the copy is staged before cudaMemcpyAsync returns
  CU(cudaMemcpyAsync(ctx->s_tables.p, tables.data(), tables.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  return 0;
}

int sgb_source_set_weights(sgb_ctx* ctx, const double* weights) {
  if (!ctx) return 1;
  const std::string who = "sgb_source_set_weights";
  if (ctx->src_state != SourceState::Batch) return fail(ctx, 1, who + ": the context holds no batch of sources (call sgb_source_set_batch)");
  if (!weights) {
    ctx->b_weighted = false;
    return 0;
  }
  CU(cudaSetDevice(ctx->device));
  cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
  CU(cudaStreamIsCapturing(ctx->stream, &capture));
  if (capture != cudaStreamCaptureStatusNone)
    return fail(ctx, 1, who + ": the context's stream is being captured, and the call synchronises to check the weights; set them outside the capture "
                              "(a replay reads the weights in force)");
  const size_t n = batch_points(ctx);
  if (n == 0) {
    ctx->b_weighted = true;
    return 0;
  }
  // Gathered into stored order and checked in one launch, into b_wnext: the weights in force stay until every new one has passed.  The
  // weights in force always have the batch's count, so b_weights never reallocates here while they are.
  const double* src = weights;
  if (!on_device(ctx, weights)) {  // host or page-locked memory: one copy to the device first (b_rows_e: scratch of the _points calls)
    CU(ctx->b_rows_e.reserve(n * sizeof(double)));
    CU(cudaMemcpyAsync(ctx->b_rows_e.p, weights, n * sizeof(double), cudaMemcpyDefault, ctx->stream));
    src = ctx->b_rows_e.as<double>();
  }
  CU(ctx->b_wnext.reserve(n * sizeof(double)));
  CU(ctx->b_wbad.reserve(sizeof(uint32_t)));
  CU(cudaMemsetAsync(ctx->b_wbad.p, 0xFF, sizeof(uint32_t), ctx->stream));
  WeightGather g = {};
  g.n = static_cast<uint32_t>(n);
  g.n_members = static_cast<uint32_t>(batch_members(ctx));
  row_layout(ctx, g.member_off, g.perm);
  g.src = src;
  g.dst = ctx->b_wnext.as<double>();
  g.bad = ctx->b_wbad.as<uint32_t>();
  CU(launch_weight_gather(g, ctx->sm_count, ctx->stream));
  ctx->launches += 1;
  uint32_t bad = ~0u;
  CU(cudaMemcpyAsync(&bad, ctx->b_wbad.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (bad != ~0u) {
    double v = 0.0;
    CU(cudaMemcpy(&v, weights + bad, sizeof(double), cudaMemcpyDefault));
    char val[32];
    std::snprintf(val, sizeof(val), "%g", v);
    return fail(ctx, 1, who + ": the weight of row " + std::to_string(bad) + " is " + val + "; every weight must be finite and >= 0 (the weights in force "
                                  "are unchanged)");
  }
  CU(ctx->b_weights.reserve(n * sizeof(double)));
  CU(cudaMemcpyAsync(ctx->b_weights.p, ctx->b_wnext.p, n * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
  ctx->b_weighted = true;
  return 0;
}
int sgb_linearize_batch(sgb_ctx* ctx, int factor, int robust, double robust_c, int rejector, double max_dist_sq, const double* T, const uint8_t* active,
                        double* out44) {
  return linearize_batch(ctx, "sgb_linearize_batch", false, factor, robust, robust_c, rejector, max_dist_sq, T, active, out44, nullptr, nullptr);
}

int sgb_linearize_batch_points(sgb_ctx* ctx, int factor, int robust, double robust_c, int rejector, double max_dist_sq, const double* T, const uint8_t* active,
                               double* out44, double* out_point_e, double* out_point_Hb42) {
  return linearize_batch(ctx, "sgb_linearize_batch_points", true, factor, robust, robust_c, rejector, max_dist_sq, T, active, out44, out_point_e, out_point_Hb42);
}

int sgb_error_batch(sgb_ctx* ctx, const double* T, const uint8_t* active, double* out_e) {
  return error_batch(ctx, "sgb_error_batch", false, T, active, out_e, nullptr);
}

int sgb_error_batch_points(sgb_ctx* ctx, const double* T, const uint8_t* active, double* out_e, double* out_point_e) {
  return error_batch(ctx, "sgb_error_batch_points", true, T, active, out_e, out_point_e);
}

int sgb_align_batch(sgb_ctx* ctx, const sgb_align_options* o, const double* init_T, double* out_T, double* out_info, double* out_Hb) {
  if (!ctx) return 1;
  AlignOptions ao;
  if (int rc = align_checks(ctx, "sgb_align_batch", o, init_T, out_T, out_info, ao)) return rc;
  const size_t B = batch_members(ctx);
  if (B == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  if (int rc = pair_view(ctx)) return rc;
  std::vector<MemberState> state;
  std::vector<uint8_t> phase;
  if (int rc = align_start(ctx, ao, init_T, state, phase)) return rc;
  if (int rc = align_rounds(ctx, o, phase, [&](bool lin) {
        return launch_batch_step(ao, static_cast<uint32_t>(B), lin, nullptr, 0, ctx->b_out.as<double>(), ctx->b_state.as<MemberState>(),
                                 ctx->b_poses.as<double>(), ctx->b_phase.as<uint8_t>(), ctx->stream);
      }))
    return rc;
  CU(cudaMemcpyAsync(state.data(), ctx->b_state.p, B * sizeof(MemberState), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  align_results(state, out_T, out_info, out_Hb);
  return 0;
}

int sgb_align_batch_gnc(sgb_ctx* ctx, const sgb_align_options* o, const sgb_gnc_options* gnc, const double* init_T, double* out_T, double* out_info,
                        double* out_Hb, double* out_gnc2, double* out_point_w) {
  if (!ctx) return 1;
  const std::string who = "sgb_align_batch_gnc";
  AlignOptions ao;
  if (int rc = gnc_checks(ctx, who, o, gnc, init_T, out_T, out_info, ao)) return rc;
  CU(cudaSetDevice(ctx->device));
  if (int rc = gnc_capture_check(ctx, who)) return rc;
  const size_t B = batch_members(ctx);
  if (B == 0) return 0;
  // sgb_align_batch_gnc_async on the poses and outputs staged in device memory: init_T | T | info | H|b | gnc2, 80 doubles per member
  CU(ctx->stage_pts.reserve(80 * B * sizeof(double)));
  double* d_init_T = ctx->stage_pts.as<double>();
  double *d_T = d_init_T + 16 * B, *d_info = d_T + 16 * B, *d_Hb = d_info + 4 * B, *d_gnc2 = d_Hb + 42 * B;
  CU(cudaMemcpyAsync(d_init_T, init_T, 16 * B * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (int rc = batch_gnc_enqueue(ctx, who.c_str(), false, o, gnc, ao, d_init_T, d_T, d_info, out_Hb ? d_Hb : nullptr, out_gnc2 ? d_gnc2 : nullptr, out_point_w))
    return rc;
  return copy_staged(ctx, {{out_T, d_T, 16 * B}, {out_info, d_info, 4 * B}, {out_Hb, d_Hb, 42 * B}, {out_gnc2, d_gnc2, 2 * B}});
}

int sgb_align_batch_gnc_async(sgb_ctx* ctx, const sgb_align_options* o, const sgb_gnc_options* gnc, const double* d_init_T, double* d_out_T, double* d_out_info,
                              double* d_out_Hb, double* d_out_gnc2, double* d_out_point_w) {
  if (!ctx) return 1;
  const char* who = "sgb_align_batch_gnc_async";
  AlignOptions ao;
  if (int rc = gnc_checks(ctx, who, o, gnc, d_init_T, d_out_T, d_out_info, ao)) return rc;
  if (batch_members(ctx) == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  if (int rc = device_pointers(ctx, who, {{d_init_T, "init_T16xB", true}, {d_out_T, "out_T16xB", true}, {d_out_info, "out_info4xB", true},
                                          {d_out_Hb, "out_Hb42xB", false}, {d_out_gnc2, "out_gnc2xB", false}, {d_out_point_w, "out_point_w", false}}))
    return rc;
  bool capturing = false;
  if (int rc = capture_state(ctx, who, &capturing)) return rc;
  return batch_gnc_enqueue(ctx, who, capturing, o, gnc, ao, d_init_T, d_out_T, d_out_info, d_out_Hb, d_out_gnc2, d_out_point_w);
}

}  // extern "C"

namespace {

// ---- joint windows (DESIGN.md §11 "Joint windows", "Asynchronous joint windows") ----

// What both joint aligns build from their arguments: the window tables, each window's free frame and edge counts, and the most free
// frames of a window with an edge (which sizes the step's shared memory).  tab = frame_off [W + 1] | edge_off [W + 1] | n_free [W] |
// edge_member [E] | edge_win [E] | edge_i [E] | edge_j [E] | free [K], the layout JointParams reads, then member_win [E] (the window of
// member p, which sgb_align_joint_gnc's point kernels read).
struct JointLayout {
  size_t W = 0, K = 0, E = 0;
  std::vector<uint32_t> tab, n_free, edge_count;
  int max_free = 0;
  const uint32_t* edge_member() const { return tab.data() + 3 * W + 2; }
  const uint32_t* edge_win() const { return edge_member() + E; }
  const int32_t* free() const { return reinterpret_cast<const int32_t*>(edge_win() + 3 * E); }
  size_t member_win_at() const { return tab.size() - E; }  // (in uint32_t of tab)
};

// The checks every joint call makes before anything is enqueued (who names the caller), and their layout.  align = false: no align
// (sgb_joint_edge_poses; o, out_info and ao unused), the checks of the windows and the pairing alone.
int joint_layout(sgb_ctx* ctx, const std::string& who, const sgb_align_options* o, size_t n_windows, const size_t* window_off, const uint8_t* fixed,
                 const double* init_X, const double* out_X, const double* out_info, AlignOptions& ao, JointLayout& L, bool align = true) {
  if (ctx->src_state != SourceState::Batch) return fail(ctx, 1, who + ": the context holds no batch of sources (call sgb_source_set_batch)");
  if (ctx->b_submaps) return fail(ctx, 1, who + ": the members are submap members (sgb_source_set_submaps); joint windows need (cloud, map) edges");
  if (!ctx->b_paired || !ctx->b_pair_has_maps)
    return fail(ctx, 1, who + ": the edges are the members of a pairing with a maps table (sgb_source_set_pairs with maps); there is none");
  if (!many_maps(ctx))
    return fail(ctx, 1, who + ": the frames are the maps of a many-kd-trees or many-voxel-maps target (sgb_target_build_kdtrees / sgb_target_build_voxelmaps); "
                              "the current target is not one");
  const size_t K = ctx->b_cloud_offsets.size() - 1, E = batch_members(ctx);
  if (K != target_maps(ctx))
    return fail(ctx, 1, who + ": frame k is cloud k with map k, but the batch holds " + std::to_string(K) + " clouds and the target " +
                            std::to_string(target_maps(ctx)) + " maps");
  if (align) {
    if (int rc = align_checks(ctx, who.c_str(), o, init_X, out_X, out_info, ao)) return rc;
  } else if (!init_X || !out_X) {
    return fail(ctx, 1, who + ": null poses or output");
  }
  if (!window_off) return fail(ctx, 1, who + ": null window offsets");
  if (n_windows > SGB_BATCH_MAX_MEMBERS)
    return fail(ctx, 1, who + ": " + std::to_string(n_windows) + " windows, at most " + std::to_string(SGB_BATCH_MAX_MEMBERS));
  if (window_off[0] != 0 || window_off[n_windows] != K)
    return fail(ctx, 1, who + ": window_off must run from 0 to the frame count " + std::to_string(K));
  for (size_t w = 0; w < n_windows; w++) {
    if (window_off[w + 1] < window_off[w]) return fail(ctx, 1, who + ": window_off must be ascending (window " + std::to_string(w) + ")");
    if (window_off[w + 1] - window_off[w] > static_cast<size_t>(kJointMaxFrames))
      return fail(ctx, 1, who + ": window " + std::to_string(w) + " has " + std::to_string(window_off[w + 1] - window_off[w]) + " frames, at most " +
                              std::to_string(kJointMaxFrames));
  }
  // window of every frame; the edges of every window in member order
  std::vector<uint32_t> win_of(K);
  for (size_t w = 0; w < n_windows; w++)
    for (size_t k = window_off[w]; k < window_off[w + 1]; k++) win_of[k] = static_cast<uint32_t>(w);
  std::vector<uint32_t> edge_count(n_windows, 0);
  for (size_t p = 0; p < E; p++) {
    const uint32_t i = ctx->b_pair_clouds[p], j = ctx->b_pair_maps[p];
    if (i == j) return fail(ctx, 1, who + ": member " + std::to_string(p) + " pairs cloud " + std::to_string(i) + " with map " + std::to_string(j) + " of its own frame");
    if (win_of[i] != win_of[j])
      return fail(ctx, 1, who + ": member " + std::to_string(p) + " joins frame " + std::to_string(i) + " (window " + std::to_string(win_of[i]) + ") and frame " +
                              std::to_string(j) + " (window " + std::to_string(win_of[j]) + "); both frames of an edge must lie in one window");
    edge_count[win_of[i]]++;
  }
  std::vector<uint8_t> fix(K);
  for (size_t k = 0; k < K; k++) fix[k] = fixed ? (fixed[k] != 0) : (k == window_off[win_of[k]]);
  std::vector<uint32_t> n_free(n_windows, 0);
  std::vector<int32_t> free_of(K);
  for (size_t w = 0; w < n_windows; w++) {
    for (size_t k = window_off[w]; k < window_off[w + 1]; k++) free_of[k] = fix[k] ? -1 : static_cast<int32_t>(n_free[w]++);
    if (edge_count[w] && n_free[w] == window_off[w + 1] - window_off[w])
      return fail(ctx, 1, who + ": window " + std::to_string(w) + " has edges but no fixed frame (its gauge would be free)");
  }
  const size_t W = n_windows;
  std::vector<uint32_t> tab(2 * (W + 1) + W + 5 * E + K);
  uint32_t* frame_off = tab.data();
  uint32_t* edge_off = frame_off + W + 1;
  uint32_t* nf = edge_off + W + 1;
  uint32_t* edge_member = nf + W;
  uint32_t* edge_win = edge_member + E;
  int32_t* edge_i = reinterpret_cast<int32_t*>(edge_win + E);
  int32_t* edge_j = edge_i + E;
  int32_t* freeidx = edge_j + E;
  uint32_t* member_win = reinterpret_cast<uint32_t*>(freeidx + K);
  for (size_t w = 0; w <= W; w++) frame_off[w] = static_cast<uint32_t>(window_off[w]);
  edge_off[0] = 0;
  for (size_t w = 0; w < W; w++) edge_off[w + 1] = edge_off[w] + edge_count[w];
  std::vector<uint32_t> fill(edge_off, edge_off + W);
  for (size_t p = 0; p < E; p++) {  // member order within each window
    const uint32_t i = ctx->b_pair_clouds[p], j = ctx->b_pair_maps[p], w = win_of[i], q = fill[w]++;
    edge_member[q] = static_cast<uint32_t>(p);
    edge_win[q] = w;
    member_win[p] = w;
    edge_i[q] = static_cast<int32_t>(i - window_off[w]);
    edge_j[q] = static_cast<int32_t>(j - window_off[w]);
  }
  L.max_free = 0;
  for (size_t w = 0; w < W; w++) {
    nf[w] = n_free[w];
    if (edge_count[w]) L.max_free = std::max(L.max_free, static_cast<int>(n_free[w]));
  }
  std::copy(free_of.begin(), free_of.end(), freeidx);
  L.W = W;
  L.K = K;
  L.E = E;
  L.tab.swap(tab);
  L.n_free.swap(n_free);
  L.edge_count.swap(edge_count);
  return 0;
}

// the bytes of each of b's buffers a call of layout L uses, in JointBufs order
std::vector<size_t> joint_bytes(const JointLayout& L) {
  const size_t K1 = std::max<size_t>(L.K, 1), W1 = std::max<size_t>(L.W, 1);
  return {L.tab.size() * sizeof(uint32_t), K1 * 16 * sizeof(double), K1 * 16 * sizeof(double), K1 * 6 * sizeof(double),
          std::max<size_t>(L.E, 1) * 44 * sizeof(double), W1 * sizeof(WindowState), W1};
}
std::vector<DevBuf*> joint_buffers(JointBufs& b) { return {&b.tables, &b.X, &b.cand, &b.delta, &b.sums, &b.state, &b.phase}; }

// JointParams over b (its tables laid out as JointLayout::tab)
JointParams joint_params(sgb_ctx* ctx, const JointBufs& b, size_t W, size_t E) {
  JointParams J = {};
  J.n_windows = static_cast<uint32_t>(W);
  J.n_edges = static_cast<uint32_t>(E);
  const uint32_t* dt = b.tables.as<uint32_t>();
  J.frame_off = dt;
  J.edge_off = dt + W + 1;
  J.n_free = J.edge_off + W + 1;
  J.edge_member = J.n_free + W;
  J.edge_win = J.edge_member + E;
  J.edge_i = reinterpret_cast<const int*>(J.edge_win + E);
  J.edge_j = J.edge_i + E;
  J.free = J.edge_j + E;
  J.X = b.X.as<double>();
  J.cand = b.cand.as<double>();
  J.delta = b.delta.as<double>();
  J.sums = b.sums.as<double>();
  J.state = b.state.as<WindowState>();
  J.phase = b.phase.as<uint8_t>();
  J.poses = ctx->b_poses.as<double>();
  return J;
}

// The rounds of sgb_align_joint from the windows' phases (read back after each round), in lockstep as in sgb_align_batch, per window:
// error() for the edges of every window with a pending trial until none has one, else a linearize of the edges of every window still
// iterating; each round ends with one joint step launch, step(lin).
template <typename Step>
int joint_rounds(sgb_ctx* ctx, const sgb_align_options* o, const JointLayout& L, std::vector<uint8_t>& phase, Step step) {
  const size_t W = L.W, E = L.E;
  const uint32_t* edge_member = L.edge_member();
  const uint32_t* edge_win = L.edge_win();
  std::vector<uint8_t> active(E);
  for (;;) {
    bool any_trial = false, any_lin = false;
    for (size_t w = 0; w < W; w++) {
      any_trial |= phase[w] == kPhaseTrial;
      any_lin |= phase[w] == kPhaseLinearize;
    }
    if (!any_trial && !any_lin) return 0;
    const bool lin = !any_trial;
    for (size_t q = 0; q < E; q++) active[edge_member[q]] = phase[edge_win[q]] == (lin ? kPhaseLinearize : kPhaseTrial);
    if (lin) {
      if (int rc = linearize_round(ctx, o->factor_kind, o->robust_kind, o->robust_c, o->rejector_kind, o->max_dist_sq, nullptr, active.data())) return rc;
    } else {
      if (int rc = error_round(ctx, nullptr, active.data())) return rc;
    }
    CU(step(lin));
    ctx->launches += 1;
    CU(cudaMemcpyAsync(phase.data(), ctx->joint.phase.p, W, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
}

// The window tables of layout L and the frames' X (host memory, column-major; null: left to the caller) uploaded to ctx->joint, its
// buffers reserved for L
int joint_upload(sgb_ctx* ctx, const JointLayout& L, const double* X) {
  const std::vector<size_t> bytes = joint_bytes(L);
  const std::vector<DevBuf*> bufs = joint_buffers(ctx->joint);
  for (size_t i = 0; i < bufs.size(); i++) CU(bufs[i]->reserve(bytes[i]));
  // pageable host memory: the copies are staged before cudaMemcpyAsync returns
  CU(cudaMemcpyAsync(ctx->joint.tables.p, L.tab.data(), L.tab.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  if (L.K && X) CU(cudaMemcpyAsync(ctx->joint.X.p, X, L.K * 16 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  return 0;
}

// The window tables and buffers of sgb_align_joint_async (ctx->joint_async), which sgb_align_joint_gnc_async shares: a call of layout L
// must reserve or upload (neither of which a capture can hold) when a buffer must grow or the tables differ from ja_tab, the host copy of
// what joint_async.tables holds
bool joint_async_stale(sgb_ctx* ctx, const JointLayout& L) {
  const std::vector<size_t> bytes = joint_bytes(L);
  const std::vector<DevBuf*> bufs = joint_buffers(ctx->joint_async);
  for (size_t i = 0; i < bufs.size(); i++)
    if (bytes[i] > bufs[i]->cap) return true;
  return L.tab != ctx->ja_tab;
}

// joint_async reserved for layout L and its tables uploaded (when joint_async_stale: otherwise both are as L needs them already).  ja_tab
// claims what joint_async.tables holds.  The claim is dropped before anything that can replace or lose that content: a reservation frees
// the old buffer before it allocates the new one, and any step below may fail.  So a failed call leaves no claim behind, and the next call
// uploads its tables again.
int joint_async_tables(sgb_ctx* ctx, const JointLayout& L) {
  const std::vector<size_t> bytes = joint_bytes(L);
  const std::vector<DevBuf*> bufs = joint_buffers(ctx->joint_async);
  ctx->ja_tab.clear();
  for (size_t i = 0; i < bufs.size(); i++) CU(bufs[i]->reserve(bytes[i]));
  // pageable host memory: the copy is staged before cudaMemcpyAsync returns
  CU(cudaMemcpyAsync(ctx->joint_async.tables.p, L.tab.data(), L.tab.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  ctx->ja_tab = L.tab;
  return 0;
}

// The outputs of a joint align from the frames' final X and the windows' final state, a fixed frame's X as init_X gives it
void joint_results(const JointLayout& L, const double* init_X, const std::vector<double>& X, const std::vector<WindowState>& state, double* out_X,
                   double* out_info) {
  const int32_t* freeidx = L.free();
  for (size_t k = 0; k < L.K; k++) std::memcpy(out_X + 16 * k, freeidx[k] < 0 ? init_X + 16 * k : X.data() + 16 * k, 16 * sizeof(double));
  for (size_t w = 0; w < L.W; w++) {
    double* info = out_info + 4 * w;
    info[0] = state[w].converged ? 1.0 : 0.0;
    info[1] = state[w].iterations;
    info[2] = state[w].inliers;
    info[3] = state[w].e;
  }
}

// The stream-ordered GNC of both joint GNC aligns, after their checks (who names the caller; capturing: ctx->stream is being captured):
// the stages and their joint rounds as one device loop on the window buffers b, its graph cached in `graph`, from the frames at
// d_init_X, the outputs to d_out_X, d_out_info and, unless null, d_out_gnc2 (device memory) and out_point_w (host or device memory).  b's
// tables hold L's already, or (upload: b is joint_async and joint_async_stale) are uploaded here.  The loop key holds every address of b,
// so each set of buffers keeps a graph of its own.
int joint_gnc_enqueue(sgb_ctx* ctx, const char* who, bool capturing, bool upload, const sgb_align_options* o, const sgb_gnc_options* gnc, const AlignOptions& ao,
                      const JointLayout& L, JointBufs& b, LoopGraph& graph, const double* d_init_X, double* d_out_X, double* d_out_info, double* d_out_gnc2,
                      double* out_point_w) {
  const size_t W = L.W, K = L.K, E = L.E, n = batch_points(ctx);
  // A capture can hold neither an allocation nor an upload from pageable memory: the GNC buffers for W windows, joint_async's tables and
  // buffers (uploaded only when they changed, as sgb_align_joint_async's), and with an edge the first batched call's search queue and both
  // capture streams (the stages' loop and the rounds' loop nested in it) must come from an earlier call
  if (int rc = loop_allocations(ctx, who, capturing, upload, E > 0, E ? 2 : 0, W,
                                ": this call needs an allocation or an upload of its window tables, which a capture cannot hold; call it once outside "
                                "the capture first"))
    return rc;
  if (upload) {
    if (int rc = joint_async_tables(ctx, L)) return rc;
  }
  if (E) {
    if (int rc = pair_view(ctx)) return rc;
  }
  const JointParams J = joint_params(ctx, b, W, E);
  const uint32_t* member_win = b.tables.as<uint32_t>() + L.member_win_at();
  // the GNC state per window: p for the point kernels (over the edges' points), pw for the window kernels
  GncParams p = gnc_params(ctx, gnc);
  p.live = reinterpret_cast<uint8_t*>(p.gnc + W);
  GncParams pw = p;
  pw.n_members = static_cast<uint32_t>(W);
  uint8_t* member_phase = ctx->b_phase.as<uint8_t>();
  // the initial state: the frames' X from d_init_X, zero window and GNC state (r2max = 0, no stage begun, no iterations), every window
  // live; the device's seed flags kept as sgb_align_joint_async keeps them
  if (K) CU(cudaMemcpyAsync(J.X, d_init_X, K * 16 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
  CU(cudaMemsetAsync(J.state, 0, W * sizeof(WindowState), ctx->stream));
  if (int rc = gnc_begin(ctx, p, W)) return rc;
  if (E && !(ctx->corr_seeds && ctx->b_dseed_ok)) CU(cudaMemsetAsync(ctx->b_dseed.p, 0, E, ctx->stream));
  if (!E) {
    // No edge, so no point: one stage of the stage kernels (r_max^2 = 0 makes it every window's last; the largest residual and the
    // weights have nothing to visit) and no round
    CU(launch_gnc_stage(pw, ctx->stream));
    CU(launch_joint_gnc_init(pw, ao, J, ctx->stream));
    ctx->launches += 2;
  } else {
    // One stage per iteration of the outer loop: the edge poses of every window's X, the reweighting linearize of the edges of the
    // windows in the stage (planned by batch_plan_kernel from their member phases), the stage kernels, then the stage's joint align as an
    // inner loop of rounds.  After joint_gnc_init, joint_gnc_loops gives every edge its window's phase and sets both conditions: the
    // stages' while a window has a stage to go, the rounds' while a window's align has a round to go.
    const BatchRows rows = gnc_rows(p);
    RoundWeights weights(ctx);
    const auto stage = [&](cudaGraphConditionalHandle stages) {
      cudaGraphConditionalHandle rounds;
      if (int rc = loop_handle(ctx, who, nullptr, &rounds)) return rc;
      CU(launch_joint_edge_poses(J, ctx->stream));
      CU(launch_joint_gnc_reweigh(J, p.live, member_phase, rounds, ctx->stream));
      weights.use(nullptr);
      if (int rc = round_head(ctx, o, stages, &rows)) return rc;
      CU(launch_joint_gnc_rmax(p, member_win, ctx->sm_count, ctx->stream));
      CU(launch_gnc_stage(pw, ctx->stream));
      CU(launch_joint_gnc_weight(p, member_win, ctx->sm_count, ctx->stream));
      CU(launch_joint_gnc_init(pw, ao, J, ctx->stream));
      CU(launch_joint_gnc_loops(J, p.live, member_phase, stages, rounds, ctx->stream));
      weights.use(p.wstage);
      return capture_loop(ctx, rounds, round_loop(ctx, o, [&](cudaGraphConditionalHandle h) {
                            CU(launch_joint_gnc_step(ao, J, L.max_free, ctx->b_out.as<double>(), pw, ctx->b_round.as<BatchRound>(), h, member_phase, ctx->stream));
                            return 0;
                          }));
    };
    std::vector<unsigned char> key;
    if (!capturing) {  // loop_key, plus the GNC options, every buffer the GNC kernels use, JointParams, the frame count and max_free
      key = loop_key(ctx, o);
      gnc_key(key, p, {member_win});
      key_add(key, J);
      for (size_t v : {K, static_cast<size_t>(L.max_free)}) key_add(key, v);
    }
    if (int rc = launch_loop(ctx, who, capturing, std::move(key), graph, stage)) return rc;
    ctx->launches += 1;
    if (int rc = clear_search_counters(ctx)) return rc;
  }
  CU(launch_joint_align_finish(J, static_cast<uint32_t>(K), d_init_X, d_out_X, d_out_info, ctx->stream));
  CU(launch_joint_gnc_finish(J, p.gnc, d_out_info, d_out_gnc2, ctx->stream));
  ctx->launches += 2;
  if (out_point_w && n) CU(cudaMemcpyAsync(out_point_w, p.e, n * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (E) {
    ctx->b_dseed_ok = true;
    // stage 0's reweighting round linearised every edge (every window is in stage 0); every round since used robust_kind (NONE)
    mark_linearised(ctx, o->factor_kind, o->robust_kind, o->robust_c, nullptr);
  }
  return 0;
}

}  // namespace

extern "C" {

int sgb_align_joint(sgb_ctx* ctx, const sgb_align_options* o, size_t n_windows, const size_t* window_off, const uint8_t* fixed, const double* init_X,
                    double* out_X, double* out_info) {
  if (!ctx) return 1;
  AlignOptions ao;
  JointLayout L;
  if (int rc = joint_layout(ctx, "sgb_align_joint", o, n_windows, window_off, fixed, init_X, out_X, out_info, ao, L)) return rc;
  const size_t W = L.W, K = L.K, E = L.E;
  CU(cudaSetDevice(ctx->device));
  if (E) {
    if (int rc = pair_view(ctx)) return rc;
  }
  std::vector<WindowState> state(W);
  std::vector<uint8_t> phase(W);
  for (size_t w = 0; w < W; w++) {
    joint_init(ao, static_cast<int>(L.n_free[w]), static_cast<int>(L.edge_count[w]), state[w]);
    phase[w] = static_cast<uint8_t>(state[w].phase);
  }
  if (int rc = joint_upload(ctx, L, init_X)) return rc;
  const JointParams J = joint_params(ctx, ctx->joint, W, E);
  if (W) {  // the phases too: a window done from the start is never stepped, and the host reads every window's phase after each round
    CU(cudaMemcpyAsync(ctx->joint.state.p, state.data(), W * sizeof(WindowState), cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->joint.phase.p, phase.data(), W, cudaMemcpyHostToDevice, ctx->stream));
  }
  if (E) {
    CU(launch_joint_edge_poses(J, ctx->stream));
    ctx->launches += 1;
  }
  if (int rc = joint_rounds(ctx, o, L, phase, [&](bool lin) {
        return launch_joint_step(ao, J, L.max_free, lin, nullptr, 0, nullptr, ctx->b_out.as<double>(), ctx->stream);
      }))
    return rc;
  std::vector<double> X(16 * K);
  if (K) CU(cudaMemcpyAsync(X.data(), ctx->joint.X.p, K * 16 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  if (W) CU(cudaMemcpyAsync(state.data(), ctx->joint.state.p, W * sizeof(WindowState), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  joint_results(L, init_X, X, state, out_X, out_info);
  return 0;
}

int sgb_joint_edge_poses(sgb_ctx* ctx, size_t n_windows, const size_t* window_off, const double* X, double* out_T) {
  if (!ctx) return 1;
  AlignOptions ao;
  JointLayout L;
  if (int rc = joint_layout(ctx, "sgb_joint_edge_poses", nullptr, n_windows, window_off, nullptr, X, out_T, nullptr, ao, L, false)) return rc;
  const size_t E = L.E;
  if (E == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  if (int rc = joint_upload(ctx, L, X)) return rc;
  // joint_edge_poses_kernel writes the poses where the joint align's rounds read them (b_poses, row-major R | t per member)
  CU(launch_joint_edge_poses(joint_params(ctx, ctx->joint, L.W, E), ctx->stream));
  ctx->launches += 1;
  std::vector<double> poses(12 * E);
  CU(cudaMemcpyAsync(poses.data(), ctx->b_poses.p, poses.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  for (size_t p = 0; p < E; p++) {
    const double* q = poses.data() + 12 * p;
    double* T = out_T + 16 * p;
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) T[j * 4 + i] = q[i * 3 + j];
      T[12 + i] = q[9 + i];
      T[i * 4 + 3] = 0.0;
    }
    T[15] = 1.0;
  }
  return 0;
}

int sgb_align_joint_gnc(sgb_ctx* ctx, const sgb_align_options* o, const sgb_gnc_options* gnc, size_t n_windows, const size_t* window_off, const uint8_t* fixed,
                        const double* init_X, double* out_X, double* out_info, double* out_gnc2, double* out_point_w) {
  if (!ctx) return 1;
  const std::string who = "sgb_align_joint_gnc";
  AlignOptions ao;
  JointLayout L;
  if (int rc = joint_layout(ctx, who, o, n_windows, window_off, fixed, init_X, out_X, out_info, ao, L)) return rc;
  if (int rc = gnc_option_checks(ctx, who, o, gnc)) return rc;
  CU(cudaSetDevice(ctx->device));
  if (int rc = gnc_capture_check(ctx, who)) return rc;
  const size_t W = L.W, K = L.K;
  if (W == 0) return 0;
  // sgb_align_joint_gnc_async on the window tables of ctx->joint (never joint_async, which a captured asynchronous call may read) and the
  // frames and outputs staged in device memory: init_X | X [frames][16] | info [windows][4] | gnc2 [windows][2]
  CU(ctx->stage_pts.reserve((32 * K + 6 * W) * sizeof(double)));
  double* d_init_X = ctx->stage_pts.as<double>();
  double *d_X = d_init_X + 16 * K, *d_info = d_X + 16 * K, *d_gnc2 = d_info + 4 * W;
  if (K) CU(cudaMemcpyAsync(d_init_X, init_X, 16 * K * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (int rc = joint_upload(ctx, L, nullptr)) return rc;
  if (int rc = joint_gnc_enqueue(ctx, who.c_str(), false, false, o, gnc, ao, L, ctx->joint, ctx->joint_gnc_sync_loop, d_init_X, d_X, d_info,
                                 out_gnc2 ? d_gnc2 : nullptr, out_point_w))
    return rc;
  return copy_staged(ctx, {{out_X, d_X, 16 * K}, {out_info, d_info, 4 * W}, {out_gnc2, d_gnc2, 2 * W}});
}

int sgb_align_batch_async(sgb_ctx* ctx, const sgb_align_options* o, const double* d_init_T, double* d_out_T, double* d_out_info, double* d_out_Hb) {
  if (!ctx) return 1;
  const char* who = "sgb_align_batch_async";
  AlignOptions ao;
  if (int rc = align_checks(ctx, who, o, d_init_T, d_out_T, d_out_info, ao)) return rc;
  const size_t B = batch_members(ctx);
  if (B == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  if (int rc = device_pointers(ctx, who, {{d_init_T, "init_T16xB", true}, {d_out_T, "out_T16xB", true}, {d_out_info, "out_info4xB", true},
                                          {d_out_Hb, "out_Hb42xB", false}}))
    return rc;
  bool capturing = false;
  if (int rc = capture_state(ctx, who, &capturing)) return rc;
  // nothing else allocates: a cudaMalloc may not run while the stream is captured (reserve_members sized everything for the batch)
  if (int rc = loop_allocations(ctx, who, capturing, false, true, 0, 0,
                                ": the first batched call of a context cannot be captured (it allocates); call it once before capturing"))
    return rc;
  if (int rc = pair_view(ctx)) return rc;
  const uint32_t nb = static_cast<uint32_t>(B);
  // the device's seed flags are kept while the host's are valid (the same target, the cached correspondences not dropped)
  CU(launch_batch_align_init(ao, nb, d_init_T, ctx->b_state.as<MemberState>(), ctx->b_poses.as<double>(), ctx->b_phase.as<uint8_t>(), ctx->b_dseed.as<uint8_t>(),
                             ctx->corr_seeds && ctx->b_dseed_ok, ctx->stream));
  ctx->launches += 2;  // the initial state here, the outputs below
  if (o->max_iterations > 0) {
    const auto step = [&](cudaGraphConditionalHandle h) {
      CU(launch_batch_step(ao, nb, true, ctx->b_round.as<BatchRound>(), h, ctx->b_out.as<double>(), ctx->b_state.as<MemberState>(), ctx->b_poses.as<double>(),
                           ctx->b_phase.as<uint8_t>(), ctx->stream));
      return 0;
    };
    if (int rc = launch_loop(ctx, who, capturing, capturing ? std::vector<unsigned char>() : loop_key(ctx, o), ctx->align_loop, round_loop(ctx, o, step)))
      return rc;
    ctx->launches += 1;
    if (int rc = clear_search_counters(ctx)) return rc;
  }
  CU(launch_batch_align_finish(nb, ctx->b_state.as<MemberState>(), d_out_T, d_out_info, d_out_Hb, ctx->stream));
  ctx->b_dseed_ok = true;
  // round 1 linearised every member, as sgb_align_batch's does
  if (o->max_iterations > 0) mark_linearised(ctx, o->factor_kind, o->robust_kind, o->robust_c, nullptr);
  return 0;
}

int sgb_align_joint_async(sgb_ctx* ctx, const sgb_align_options* o, size_t n_windows, const size_t* window_off, const uint8_t* fixed, const double* d_init_X,
                          double* d_out_X, double* d_out_info) {
  if (!ctx) return 1;
  const char* who = "sgb_align_joint_async";
  AlignOptions ao;
  JointLayout L;
  if (int rc = joint_layout(ctx, who, o, n_windows, window_off, fixed, d_init_X, d_out_X, d_out_info, ao, L)) return rc;
  const size_t W = L.W, K = L.K, E = L.E;
  if (W == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  if (int rc = device_pointers(ctx, who, {{d_init_X, "init_X16xK", true}, {d_out_X, "out_X16xK", true}, {d_out_info, "out_info4xW", true}})) return rc;
  bool capturing = false;
  if (int rc = capture_state(ctx, who, &capturing)) return rc;
  const bool loop = o->max_iterations > 0 && E > 0;
  // A capture can hold neither an allocation nor an upload from pageable memory: the buffers, the capture stream and the window tables
  // must come from an earlier call.  Outside a capture the tables are uploaded only when they changed (windows, fixed flags or pairing).
  const bool upload = joint_async_stale(ctx, L);
  if (int rc = loop_allocations(ctx, who, capturing, upload, false, loop ? 1 : 0, 0,
                                ": these windows need an allocation or an upload of their tables, which a capture cannot hold; call it once outside the "
                                "capture first"))
    return rc;
  if (upload) {
    if (int rc = joint_async_tables(ctx, L)) return rc;
  }
  if (E) {
    if (int rc = pair_view(ctx)) return rc;
  }
  const JointParams J = joint_params(ctx, ctx->joint_async, W, E);
  // the edges are the members: each edge's member phase is its window's, which the planner reads as sgb_align_joint's host loop reads
  // the windows' phases; the device's seed flags are kept as sgb_align_batch_async keeps them
  uint8_t* member_phase = ctx->b_phase.as<uint8_t>();
  CU(launch_joint_align_init(ao, J, d_init_X, member_phase, ctx->b_dseed.as<uint8_t>(), ctx->corr_seeds && ctx->b_dseed_ok, ctx->stream));
  ctx->launches += 2;  // the initial state here, the outputs below
  if (loop) {
    const auto step = [&](cudaGraphConditionalHandle h) {
      CU(launch_joint_step(ao, J, L.max_free, true, ctx->b_round.as<BatchRound>(), h, member_phase, ctx->b_out.as<double>(), ctx->stream));
      return 0;
    };
    std::vector<unsigned char> key;
    if (!capturing) {  // loop_key, plus JointParams (window and edge counts, every buffer), the frame count and max_free (the step's shared memory)
      key = loop_key(ctx, o);
      key_add(key, J);
      for (size_t v : {K, static_cast<size_t>(L.max_free)}) key_add(key, v);
    }
    if (int rc = launch_loop(ctx, who, capturing, std::move(key), ctx->joint_loop, round_loop(ctx, o, step))) return rc;
    ctx->launches += 1;
    if (int rc = clear_search_counters(ctx)) return rc;
  }
  CU(launch_joint_align_finish(J, static_cast<uint32_t>(K), d_init_X, d_out_X, d_out_info, ctx->stream));
  ctx->b_dseed_ok = true;
  // Round 1 linearised the edges of every window that started in kPhaseLinearize (one with a free frame and an edge), as sgb_align_joint's
  // first round does; no other edge was ever linearised.  Their flags are set as linearize_round sets them, the others left as they were.
  if (loop) {
    const uint32_t* edge_member = L.edge_member();
    const uint32_t* edge_win = L.edge_win();
    std::vector<uint8_t> linearised(E, 0);
    bool any = false;
    for (size_t q = 0; q < E; q++) any |= (linearised[edge_member[q]] = L.n_free[edge_win[q]] > 0) != 0;
    if (any) mark_linearised(ctx, o->factor_kind, o->robust_kind, o->robust_c, linearised.data());
  }
  return 0;
}

int sgb_align_joint_gnc_async(sgb_ctx* ctx, const sgb_align_options* o, const sgb_gnc_options* gnc, size_t n_windows, const size_t* window_off,
                              const uint8_t* fixed, const double* d_init_X, double* d_out_X, double* d_out_info, double* d_out_gnc2, double* d_out_point_w) {
  if (!ctx) return 1;
  const std::string who = "sgb_align_joint_gnc_async";
  AlignOptions ao;
  JointLayout L;
  if (int rc = joint_layout(ctx, who, o, n_windows, window_off, fixed, d_init_X, d_out_X, d_out_info, ao, L)) return rc;
  if (int rc = gnc_option_checks(ctx, who, o, gnc)) return rc;
  if (L.W == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  if (int rc = device_pointers(ctx, who, {{d_init_X, "init_X16xK", true}, {d_out_X, "out_X16xK", true}, {d_out_info, "out_info4xW", true},
                                          {d_out_gnc2, "out_gnc2xW", false}, {d_out_point_w, "out_point_w", false}}))
    return rc;
  bool capturing = false;
  if (int rc = capture_state(ctx, who, &capturing)) return rc;
  return joint_gnc_enqueue(ctx, who.c_str(), capturing, joint_async_stale(ctx, L), o, gnc, ao, L, ctx->joint_async, ctx->joint_gnc_loop, d_init_X, d_out_X,
                           d_out_info, d_out_gnc2, d_out_point_w);
}

int sgb_correspondences_batch(sgb_ctx* ctx, uint64_t* out) {
  if (!ctx) return 1;
  if (int rc = batch_check(ctx, "sgb_correspondences_batch", kIdentity)) return rc;
  const size_t n = batch_points(ctx);
  if (n == 0) return 0;
  if (!out) return fail(ctx, 1, "sgb_correspondences_batch: null output");
  CU(cudaSetDevice(ctx->device));
  CU(ctx->corr64.reserve(n * sizeof(uint64_t)));
  const uint32_t* perm = (ctx->b_paired ? ctx->p_perm : ctx->src_perm).as<uint32_t>();
  for (size_t m = 0; m + 1 < ctx->b_offsets.size(); m++) {
    const size_t off = ctx->b_offsets[m], nm = ctx->b_offsets[m + 1] - off;
    if (nm == 0) continue;
    // not linearised against the current target (never, or before the target changed: have_lin is cleared with it): no correspondences
    if (!ctx->have_lin || !ctx->b_lin[m]) {
      CU(cudaMemsetAsync(ctx->corr64.as<uint64_t>() + off, 0xFF, nm * sizeof(uint64_t), ctx->stream));
      continue;
    }
    // a multi-map target: the id within the member's own map (tgt_pts[k].w), as a context holding that map alone reports it
    if (ctx->b_submaps)
      CU(launch_submap_correspondences(ctx->b_corr.as<uint32_t>() + off, ctx->b_centry.as<uint32_t>() + off, perm + off, nm, ctx->tgt_pts.as<float4>(),
                                       ctx->corr64.as<uint64_t>() + off, ctx->sm_count, ctx->stream));
    else if (ctx->tgt_state == TargetState::VoxelMaps)
      CU(launch_voxelmaps_correspondences(ctx->b_corr.as<uint32_t>() + off, perm + off, nm, ctx->tgt_pts.as<float4>(), ctx->corr64.as<uint64_t>() + off, ctx->sm_count, ctx->stream));
    else
      CU(launch_correspondences(ctx->b_corr.as<uint32_t>() + off, perm + off, nm, ctx->tgt_pts.as<float4>(), voxel_target(ctx) ? 1 : 0, ctx->corr64.as<uint64_t>() + off, ctx->sm_count, ctx->stream));
    ctx->launches += 1;
  }
  CU(cudaMemcpyAsync(out, ctx->corr64.p, n * sizeof(uint64_t), cudaMemcpyDefault, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

}  // extern "C"
