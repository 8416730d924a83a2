// SPDX-License-Identifier: MIT
// Context + C-ABI (include/sgicp_b200.h) of the H100-native small_gicp hot path.
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/sgicp_b200.h"
#include "sgb_context.hpp"
#include "sgb_kdtree_host.hpp"
#include "sgb_kernels.h"

using namespace sgb;

namespace {

thread_local std::string g_create_error;

int ensure_reduction_buffers(sgb_ctx* ctx, int grid) {
  CU(ctx->partials.reserve(reduction_partials_doubles(static_cast<size_t>(grid)) * sizeof(double)));
  const size_t ticket_bytes = reduction_tickets(static_cast<size_t>(grid)) * sizeof(unsigned int);
  if (ticket_bytes > ctx->ticket.cap) {  // the kernels leave the counters zeroed; only a fresh buffer needs clearing
    CU(ctx->ticket.reserve(ticket_bytes));
    CU(cudaMemsetAsync(ctx->ticket.p, 0, ctx->ticket.cap, ctx->stream));
  }
  return 0;
}

int upload_tree(sgb_ctx* ctx, const FlatTree& tree, const float* host_pts_xyzw) {
  // packet (BVH2) records of the same tree for the warp-cooperative search
  std::vector<PacketNode> pnodes;
  int pending = 1;
  build_packet_nodes(tree, host_pts_xyzw, pnodes, &pending);
  if (pending > 40) return fail(ctx, 1, "kd-tree too deep for the device traversal stack (depth > 40)");
  CU(ctx->tgt_pnodes.reserve(pnodes.size() * sizeof(PacketNode)));
  CU(cudaMemcpyAsync(ctx->tgt_pnodes.p, pnodes.data(), pnodes.size() * sizeof(PacketNode), cudaMemcpyHostToDevice, ctx->stream));
  CU(ctx->tgt_perm.reserve(tree.perm.size() * sizeof(uint32_t)));
#ifdef SGB_PROFILING  // the 8-byte kd nodes are only walked by the per-thread / fused A/B kernels
  CU(ctx->tgt_nodes.reserve(tree.nodes.size() * sizeof(FlatNode)));
  CU(cudaMemcpyAsync(ctx->tgt_nodes.p, tree.nodes.data(), tree.nodes.size() * sizeof(FlatNode), cudaMemcpyHostToDevice, ctx->stream));
#endif
  CU(cudaMemcpyAsync(ctx->tgt_perm.p, tree.perm.data(), tree.perm.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  if (int rc = gather_target_features(ctx, true)) return rc;
  // the host vectors go out of scope when the caller returns: make sure the async copies are done
  CU(cudaStreamSynchronize(ctx->stream));
  return install_tree(ctx, tree.depth, pnodes.size());
}

// the answer of linearize / error() over an empty cloud (helper_test.cpp:53-59: empty clouds must not crash): a sum over nothing
int zero_result(sgb_ctx* ctx, const double* T, double* d_out, bool linearize) {
  const size_t at = linearize ? 0 : 48, doubles = linearize ? 44 : 1;  // slots of the mapped host result (sgb_linearize / sgb_error)
  if (ctx->comm_world > 1) {  // an empty shard still takes part in the exchange: contribute zeros
    if (int rc = ensure_reduction_buffers(ctx, 1)) return rc;
    LinParams P0;
    fill_params(ctx, P0, T);
    P0.out = d_out;
    CU(launch_reduce_nothing(P0, linearize, ctx->stream));
    ctx->launches += 1;
  } else if (d_out == ctx->h_out_dev + at) {  // the mapped host slot: clear it from the host side, in stream order
    CU(cudaStreamSynchronize(ctx->stream));
    std::memset(ctx->h_out + at, 0, doubles * sizeof(double));
  } else {
    CU(cudaMemsetAsync(d_out, 0, doubles * sizeof(double), ctx->stream));
  }
  return 0;
}

// the single-source calls need one target: a multi-map voxel target serves the batched calls only
int single_target_check(sgb_ctx* ctx, const char* who) {
  if (ctx->tgt_state == TargetState::KdTrees)
    return fail(ctx, 1, std::string(who) + ": the target holds " + std::to_string(ctx->kt_maps) +
                            " kd-trees (sgb_target_build_kdtrees), which only the batched calls use; set a single target first");
  if (ctx->tgt_state != TargetState::VoxelMaps) return 0;
  return fail(ctx, 1, std::string(who) + ": the target holds " + std::to_string(ctx->vm_maps) +
                          " voxel maps (sgb_target_build_voxelmaps), which only the batched calls use; set a single target first");
}

void forget_linearisation(sgb_ctx* ctx) {
  ctx->have_lin = false;
  ctx->corr_seeds = false;
  ctx->b_view_ok = false;  // the target (or the pairing) it was built from may have changed
  ctx->b_dseed_ok = false;
  for (LoopGraph* g : {&ctx->align_loop, &ctx->joint_loop, &ctx->gnc_loop, &ctx->joint_gnc_loop, &ctx->joint_gnc_sync_loop})
    g->key.clear();  // every stream-ordered loop is rebuilt
}

}  // namespace

int sgb::fill_params(sgb_ctx* ctx, LinParams& P, const double* T_colmajor16) {
  std::memset(&P, 0, sizeof(P));
  P.tgt.pts = ctx->tgt_pts.as<float4>();
  P.tgt.normals = ctx->tgt_normals.as<float4>();
  P.tgt.covA = ctx->tgt_covA.as<float4>();
  P.tgt.covB = ctx->tgt_covB.as<float4>();
  P.tgt.nodes = ctx->tgt_nodes.as<KdNode>();
  P.tgt.centre = ctx->tgt_centre.as<double>();
  P.tgt.vox_table = ctx->vox_table.as<int4>();
  P.tgt.vox_mask = ctx->vox_mask;
  P.tgt.vox_num_offsets = ctx->vox_offsets;
  P.tgt.vox_inv_leaf = ctx->vox_inv_leaf;
  P.src.pts = ctx->src_pts.as<float4>();
  P.src.covA = ctx->src_covA.as<float4>();
  P.src.covB = ctx->src_covB.as<float4>();
  P.src.centre = ctx->src_centre.as<double>();
  P.src.n = static_cast<uint32_t>(ctx->n_src);
  P.src.run = ctx->src_run;
  pose_from_colmajor(T_colmajor16, P.T);
  P.corr = ctx->corr.as<uint32_t>();
  P.partials = ctx->partials.as<double>();
  P.ticket = ctx->ticket.as<unsigned int>();
  if (ctx->comm_world > 1) {  // the launch that finishes the reduction also exchanges it with the other ranks
    P.comm.world = ctx->comm_world;
    P.comm.rank = ctx->comm_rank;
    for (int p = 0; p < ctx->comm_world; p++) P.comm.mail[p] = ctx->comm_peers[p];
    P.comm.seq = ++ctx->comm_seq;  // exactly one reduction per fill_params (do_linearize / do_error)
    P.comm.timeout_ns = ctx->comm_timeout_ns;
    P.comm.status = ctx->comm_status.as<unsigned int>();
    P.comm.stamps = reinterpret_cast<unsigned long long*>(ctx->comm_status.as<unsigned char>() + 64);
  }
  return 0;
}

void sgb::pose_from_colmajor(const double* T, double out12[12]) {
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) out12[i * 3 + j] = T[j * 4 + i];
    out12[9 + i] = T[12 + i];
  }
}

// ---- transitions ----
int sgb::begin_point_target(sgb_ctx* ctx, size_t n, bool normals, bool covs, bool lo) {
  ctx->tgt_state = TargetState::Points;
  ctx->n_tgt = n;
  ctx->tgt_has_normals = normals;
  ctx->tgt_has_covs = covs;
  ctx->tgt_has_lo = lo;
  ctx->grid_ready = false;
  forget_linearisation(ctx);
  CU(ctx->tgt_centre.reserve(4 * sizeof(double)));
  CU(ctx->tgt_bounds.reserve(6 * sizeof(double)));
  return 0;
}

int sgb::begin_voxel_target(sgb_ctx* ctx, size_t n, bool covs, double leaf_size, int search_offsets, bool maps, size_t n_maps) {
  ctx->tgt_state = maps ? TargetState::VoxelMaps : TargetState::VoxelMap;
  ctx->vm_maps = maps ? n_maps : 0;
  ctx->n_tgt = n;
  ctx->tgt_has_normals = false;
  ctx->tgt_has_covs = covs;
  ctx->grid_ready = false;
  forget_linearisation(ctx);
  ctx->vox_offsets = search_offsets;
  ctx->vox_inv_leaf = 1.0 / leaf_size;
  CU(ctx->tgt_centre.reserve(4 * sizeof(double)));
  CU(ctx->tgt_bounds.reserve(6 * sizeof(double)));
  return 0;
}

int sgb::begin_forest_target(sgb_ctx* ctx, size_t n, bool normals, bool covs, size_t n_maps) {
  ctx->tgt_state = TargetState::KdTrees;
  ctx->kt_maps = n_maps;
  ctx->vm_maps = 0;
  ctx->n_tgt = n;
  ctx->tgt_has_normals = normals;
  ctx->tgt_has_covs = covs;
  ctx->tgt_has_lo = false;
  ctx->grid_ready = false;
  forget_linearisation(ctx);
  CU(ctx->tgt_centre.reserve(4 * sizeof(double)));
  CU(ctx->tgt_bounds.reserve(6 * sizeof(double)));
  return 0;
}

size_t sgb::target_maps(const sgb_ctx* ctx) {
  if (ctx->tgt_state == TargetState::VoxelMaps) return ctx->vm_maps;
  if (ctx->tgt_state == TargetState::KdTrees) return ctx->kt_maps;
  return 0;
}

int sgb::install_tree(sgb_ctx* ctx, int depth, size_t n_pnodes) {
  ctx->tgt_state = TargetState::Tree;
  ctx->tree_depth = depth;
  ctx->n_pnodes = n_pnodes;
  forget_linearisation(ctx);
  return build_grid(ctx);
}

void sgb::begin_source(sgb_ctx* ctx, SourceState state, size_t n, bool covs) {
  ctx->src_state = state;
  ctx->n_src = n;
  ctx->src_has_covs = covs;
  ctx->src_has_lo = ctx->src_tree_valid = ctx->src_cov_orig_valid = false;
  ctx->b_paired = ctx->b_pair_has_maps = ctx->b_submaps = false;
  ctx->b_pair_maps.clear();
  ctx->b_weighted = false;  // the weights belonged to the rows of the old members
  forget_linearisation(ctx);
}

void sgb::begin_pairs(sgb_ctx* ctx) {
  ctx->b_paired = true;
  ctx->b_pair_has_maps = ctx->b_submaps = false;
  ctx->b_pair_maps.clear();
  ctx->b_weighted = false;
  forget_linearisation(ctx);
}

void sgb::features_changed(sgb_ctx* ctx, bool target) {
  if (target)
    ctx->tgt_has_normals = ctx->tgt_has_covs = true;
  else
    ctx->src_has_covs = true;
  forget_linearisation(ctx);
}

// ---- steps shared by the entry points ----
int sgb::gather_target_features(sgb_ctx* ctx, bool points) {
  const size_t n = ctx->n_tgt;
  if (points) CU(ctx->tgt_pts.reserve(n * sizeof(float4)));
  if (ctx->tgt_has_normals) CU(ctx->tgt_normals.reserve(n * sizeof(float4)));
  if (ctx->tgt_has_covs) {
    CU(ctx->tgt_covA.reserve(n * sizeof(float4)));
    CU(ctx->tgt_covB.reserve(n * sizeof(float4)));
  }
  if (!points && !ctx->tgt_has_normals && !ctx->tgt_has_covs) return 0;
  CU(launch_gather(ctx->tgt_perm.as<uint32_t>(), n, points ? ctx->tgt_orig_pts.as<float4>() : nullptr, ctx->tgt_pts.as<float4>(),
                   ctx->tgt_has_normals ? ctx->tgt_orig_normals.as<float4>() : nullptr, ctx->tgt_normals.as<float4>(),
                   ctx->tgt_has_covs ? ctx->tgt_orig_covA.as<float4>() : nullptr, ctx->tgt_covA.as<float4>(),
                   ctx->tgt_has_covs ? ctx->tgt_orig_covB.as<float4>() : nullptr, ctx->tgt_covB.as<float4>(), ctx->sm_count, ctx->stream));
  ctx->launches += 1;
  return 0;
}

int sgb::reserve_query_scratch(sgb_ctx* ctx, size_t n) {
  CU(ctx->grid_state.reserve(n));
  const void* before = ctx->grid_pending.p;
  CU(ctx->grid_pending.reserve((n + 2) * sizeof(uint32_t)));
  if (ctx->grid_pending.p != before) ctx->pending_clean = false;
  CU(ctx->grid_pending_q.reserve(n * sizeof(float4)));
  before = ctx->chunk_lists.p;
  CU(ctx->chunk_lists.reserve((8 + static_cast<size_t>(kChunkClasses) * ((n + 31) / 32)) * sizeof(uint32_t)));
  if (ctx->chunk_lists.p != before) ctx->chunk_lists_clean = false;
  return 0;
}

// The n points at stage_pts[off..] become one source cloud: centred on its own box (centre / bounds), rounded to FP32 (tmp_pts[off..]:
// original order, w = index; lo: the rounding residuals, or nullptr), Hilbert-sorted within itself (src_perm[off..]: search order ->
// original index; sort_bytes of sort_temp suffice for n) and gathered into src_pts[off..].  With cov_chunks > 0 the covariances at
// stage_covs[off..] are packed into the search order in cov_chunks pieces, piece k once arrived[k] has fired (arrived = nullptr: they are
// already there).  run > 1 (profiling build only): the chunk-transposed order of the per-thread search.
int sgb::store_source(sgb_ctx* ctx, size_t off, size_t n, double* centre, double* bounds, float4* lo, size_t sort_bytes, uint32_t run, int cov_chunks,
                      const cudaEvent_t* arrived) {
  const double* pts = ctx->stage_pts.as<double>() + 4 * off;
  uint32_t* perm = ctx->src_perm.as<uint32_t>() + off;
  CU(launch_bounds_centre(pts, n, bounds, centre, ctx->sm_count, ctx->stream));
  CU(launch_convert(pts, nullptr, nullptr, n, centre, ctx->tmp_pts.as<float4>() + off, nullptr, nullptr, nullptr, ctx->keys_in.as<uint64_t>() + off,
                    ctx->vals_in.as<uint32_t>() + off, ctx->sm_count, ctx->stream, lo));
  // Hilbert order: consecutive lanes get spatially adjacent queries (coherent tree paths, coalesced gathers)
  CU(sort_pairs_u64_u32_bits(ctx->sort_temp.p, sort_bytes, ctx->keys_in.as<uint64_t>() + off, ctx->keys_out.as<uint64_t>() + off,
                             ctx->vals_in.as<uint32_t>() + off, perm, n, 63, ctx->stream));
#ifdef SGB_PROFILING
  // chunk-transposed order of the per-thread search (A/B): a lane walks K consecutive points of the curve, warp loads stay coalesced
  if (run > 1) {
    CU(launch_chunk_transpose(perm, ctx->vals_in.as<uint32_t>() + off, n, run, ctx->sm_count, ctx->stream));
    CU(cudaMemcpyAsync(perm, ctx->vals_in.as<uint32_t>() + off, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
    ctx->launches += 1;
  }
#else
  (void)run;
#endif
  CU(launch_gather(perm, n, ctx->tmp_pts.as<float4>() + off, ctx->src_pts.as<float4>() + off, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                   ctx->sm_count, ctx->stream));
  ctx->launches += 5;
  if (cov_chunks == 0) return 0;
  uint32_t* rank = ctx->src_rank.as<uint32_t>() + off;
  CU(launch_inverse_perm(perm, n, rank, ctx->sm_count, ctx->stream));
  ctx->launches += 1;
  const size_t per_chunk = (n + cov_chunks - 1) / cov_chunks;
  for (int k = 0; k < cov_chunks; k++) {
    const size_t first = static_cast<size_t>(k) * per_chunk, cnt = std::min(per_chunk, n - first);
    if (arrived) CU(cudaStreamWaitEvent(ctx->stream, arrived[k], 0));
    CU(launch_convert_cov_scatter(ctx->stage_covs.as<double>() + 16 * off, first, cnt, rank, ctx->src_covA.as<float4>() + off, ctx->src_covB.as<float4>() + off,
                                  nullptr, nullptr, ctx->sm_count, ctx->stream));
    ctx->launches += 1;
  }
  return 0;
}

int sgb::check_target(sgb_ctx* ctx, const char* who, int factor) {
  if (ctx->tgt_state != TargetState::Tree && ctx->tgt_state != TargetState::VoxelMap && ctx->tgt_state != TargetState::VoxelMaps &&
      ctx->tgt_state != TargetState::KdTrees)
    return fail(ctx, 1, std::string(who) + ": target has no search structure (call sgb_target_set_kdtree / _build_kdtree / _set_voxelmap)");
  if (factor == SGB_FACTOR_PLANE_ICP && (!ctx->tgt_has_normals || ctx->tgt_state == TargetState::VoxelMap || ctx->tgt_state == TargetState::VoxelMaps))
    return fail(ctx, 1, std::string(who) + ": point-to-plane needs target normals");
  if (factor == SGB_FACTOR_GICP && (!ctx->tgt_has_covs || !ctx->src_has_covs)) return fail(ctx, 1, std::string(who) + ": GICP needs target and source covariances");
  return 0;
}

float sgb::search_bound(int rejector, double max_dist_sq) {
  if (rejector != SGB_REJECT_DISTANCE) return FLT_MAX;
  const float bound = nextafterf(static_cast<float>(max_dist_sq * (1.0 + 4e-6) + 1e-12), INFINITY);
  return bound < FLT_MAX ? bound : FLT_MAX;
}

namespace {

int do_linearize_impl(sgb_ctx* ctx, int factor, int robust, double robust_c, int rejector, double max_dist_sq, const double* T, double* d_out) {
  if (factor < 0 || factor > 2 || robust < 0 || robust > 2 || rejector < 0 || rejector > 1) return fail(ctx, 1, "sgb_linearize: invalid factor/robust/rejector kind");
  if (!T) return fail(ctx, 1, "sgb_linearize: null pose");
  CU(cudaSetDevice(ctx->device));
  ctx->last_out = d_out;
  if (ctx->n_src == 0 || ctx->n_tgt == 0) {
    if (int rc = zero_result(ctx, T, d_out, true)) return rc;
    if (ctx->n_src) {
      CU(ctx->corr.reserve(ctx->n_src * sizeof(uint32_t)));
      CU(cudaMemsetAsync(ctx->corr.p, 0xFF, ctx->n_src * sizeof(uint32_t), ctx->stream));
    }
    ctx->have_lin = true;
    ctx->lin_factor = factor;
    ctx->lin_robust = robust;
    ctx->lin_c = robust_c;
    pose_from_colmajor(T, ctx->Tlin);
    return 0;
  }
  if (int rc = check_target(ctx, "sgb_linearize", factor)) return rc;
  const bool voxel = ctx->tgt_state == TargetState::VoxelMap;

  const int depth = voxel ? 0 : (ctx->tree_depth > 0 ? ctx->tree_depth : 1);
  const int grid = one_wave_grid(ctx->n_src, ctx->sm_count, linearize_occupancy(depth));
  // one allocation that serves every kernel that may finish the reduction (growing a buffer later would cudaFree, i.e.
  // synchronise the whole device in the middle of the call)
  if (int rc = ensure_reduction_buffers(ctx, std::max(grid, ctx->sm_count * 8))) return rc;
  CU(ctx->corr.reserve(ctx->n_src * sizeof(uint32_t)));

  LinParams P;
  fill_params(ctx, P, T);
  std::memcpy(P.Tlin, P.T, sizeof(P.T));
  // FP32 search bound a hair above the threshold; the rejector itself (d2 > max, rejector.hpp:24) is applied to the FP64 residual
  P.max_dist_sq = search_bound(rejector, max_dist_sq);
  P.max_dist_sq_d = rejector == SGB_REJECT_DISTANCE ? max_dist_sq : DBL_MAX;
  P.use_prev = (ctx->corr_seeds && !voxel) ? 1 : 0;
  P.robust_c = robust_c;
  P.out = d_out;
#ifdef SGB_PROFILING
  const bool split_path = ctx->search_mode != 0 && !voxel;
  const bool packet_path = ctx->search_mode == 2 && ctx->src_run == 1;
#else
  const bool split_path = !voxel;
  const bool packet_path = true;
#endif
  if (split_path) {
    // phase 1: search at high occupancy; phase 2: factor algebra + reduction (sgb_kernels_split.cu)
    if (packet_path) {
      if (int rc = launch_point_search(ctx, P, depth)) return rc;
    } else {
#ifdef SGB_PROFILING
      const uint32_t chunk_pts = 32u * ctx->src_run;
      const size_t n_chunks = (ctx->n_src + chunk_pts - 1) / chunk_pts;
      CU(launch_search(P, one_wave_grid(n_chunks * 32, ctx->sm_count, search_occupancy(depth)), depth, ctx->stream));
#endif
    }
    // exactly one wave of the factor kernel (its CTAs loop over tiles)
    const int fgrid = one_wave_grid(ctx->n_src, ctx->sm_count, factor_reduce_occupancy(factor, robust));
    if (int rc = ensure_reduction_buffers(ctx, fgrid)) return rc;
    P.partials = ctx->partials.as<double>();
    P.ticket = ctx->ticket.as<unsigned int>();
    CU(launch_factor_reduce(P, factor, robust, fgrid, ctx->stream));
    ctx->launches += 2;
  } else {
    CU(launch_linearize(P, factor, robust, voxel, grid, depth, ctx->stream));
    ctx->launches += 1;
  }
  ctx->have_lin = true;
  ctx->corr_seeds = true;
  ctx->lin_factor = factor;
  ctx->lin_robust = robust;
  ctx->lin_c = robust_c;
  std::memcpy(ctx->Tlin, P.T, sizeof(P.T));
  return 0;
}
}  // namespace

// The grid front end's parameters for n queries (grid_ready, the buffers sized for them): the chunk class lists with the counters of
// `parity`, and what the warp-per-query finish reads (pp.g: the cell grid of the probe).
void sgb::point_search_params(const sgb_ctx* ctx, size_t n, int parity, ChunkClasses& cc, PendingParams& pp) {
  GridParams g;
  for (int a = 0; a < 3; a++) g.origin[a] = ctx->grid_origin[a];
  g.inv_cell = ctx->grid_inv_cell;
  g.settle_d2 = ctx->grid_settle_d2;
  if (ctx->use_chunk_classes) {
    // work lists of the packet search by cost class; two sets of counters alternate like the pending counters
    uint32_t* cbase = ctx->chunk_lists.as<uint32_t>();
    cc.count = cbase + 4 * parity;
    cc.count_next = cbase + 4 * (parity ^ 1);
    cc.lists = cbase + 8;
    cc.n_chunks = static_cast<uint32_t>((n + 31) / 32);
    const float cell = ctx->grid_cell;
    cc.wide_r2 = ctx->class_wide_cells * ctx->class_wide_cells * cell * cell;  // search balls wider than two cells / one cell
    cc.mid_r2 = cell * cell;
    cc.fallback_pct = ctx->class_fallback_pct;
  }
  // the finishing kernel serves both regimes: few pending queries warp-per-query, many through the packet walk
  pp.list = ctx->grid_pending.as<uint32_t>() + 2;
  pp.q = ctx->grid_pending_q.as<float4>();
  pp.grid_pts = ctx->grid_pts.as<float4>();
  pp.table = ctx->use_ring ? ctx->grid_table.as<GridSlot>() : nullptr;
  pp.capacity = ctx->grid_capacity;
  pp.g = g;
}

// The search of a point target over P.src (P.src.n queries): grid probe, then the packet search / warp-per-query finish.  Fills P.corr.
int sgb::launch_point_search(sgb_ctx* ctx, const LinParams& P, int depth) {
  const size_t n = P.src.n;
  const int sgrid = one_wave_grid((n + 31) / 32 * 32, ctx->sm_count, packet_occupancy(depth));
  const uint8_t* settled = nullptr;
  const uint32_t* pending_count = nullptr;
  ChunkClasses cc = {};
  PendingParams pp = {};
  if (ctx->grid_ready) {
    // grid front end: settles every query whose nearest neighbour lies within half a cell (sgb_grid.cu)
    CU(ctx->grid_state.reserve(n));
    // [0], [1]: two pending counters that alternate between calls (each probe clears the other one), [2..]: the list
    const void* before = ctx->grid_pending.p;
    CU(ctx->grid_pending.reserve((n + 2) * sizeof(uint32_t)));
    if (ctx->grid_pending.p != before || !ctx->pending_clean) {
      CU(cudaMemsetAsync(ctx->grid_pending.p, 0, 2 * sizeof(uint32_t), ctx->stream));
      ctx->pending_clean = true;
    }
    if (ctx->use_chunk_classes) {  // (sized in sgb_source_set_points)
      const void* cb = ctx->chunk_lists.p;
      CU(ctx->chunk_lists.reserve((8 + static_cast<size_t>(kChunkClasses) * ((n + 31) / 32)) * sizeof(uint32_t)));
      if (ctx->chunk_lists.p != cb || !ctx->chunk_lists_clean) {
        CU(cudaMemsetAsync(ctx->chunk_lists.p, 0, 8 * sizeof(uint32_t), ctx->stream));
        ctx->chunk_lists_clean = true;
      }
    }
    CU(ctx->grid_pending_q.reserve(n * sizeof(float4)));
    point_search_params(ctx, n, ctx->pending_parity, cc, pp);
    uint32_t* pbase = ctx->grid_pending.as<uint32_t>();
    pending_count = pbase + ctx->pending_parity;
    settled = ctx->grid_state.as<uint8_t>();
    CU(launch_grid_probe(P, nullptr, ctx->grid_pts.as<float4>(), ctx->grid_table.as<GridSlot>(), ctx->grid_capacity, pp.g, ctx->grid_state.as<uint8_t>(),
                         pbase + ctx->pending_parity, pbase + 2, ctx->grid_pending_q.as<float4>(), pbase + (ctx->pending_parity ^ 1), cc, ctx->stream));
    ctx->pending_parity ^= 1;
    ctx->launches += 1;
  }
  // many pending queries: the packet search walks the tree
  uint32_t *queue = nullptr, *queue_next = nullptr;
  if (ctx->use_packet_queue) {
    if (!ctx->packet_queue.p) {  // first use: two zeroed counters (afterwards every launch clears the other one)
      CU(ctx->packet_queue.reserve(2 * sizeof(uint32_t)));
      CU(cudaMemsetAsync(ctx->packet_queue.p, 0, 2 * sizeof(uint32_t), ctx->stream));
    }
    queue = ctx->packet_queue.as<uint32_t>() + ctx->packet_parity;
    queue_next = ctx->packet_queue.as<uint32_t>() + (ctx->packet_parity ^ 1);
    ctx->packet_parity ^= 1;
  }
  CU(launch_packet_search(P, nullptr, ctx->tgt_pnodes.as<float4>(), sgrid, depth, settled, pending_count, static_cast<uint32_t>(ctx->pending_div), queue, queue_next,
                          cc, pp, ctx->tma_leaf, ctx->stream));
#ifdef SGB_PROFILING
  if (ctx->debug_pending && pending_count) {  // profiling aid: synchronises
    uint32_t h = 0;
    CU(cudaMemcpyAsync(&h, pending_count, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    std::fprintf(stderr, "[sgb] grid front end: %u of %zu queries pending (cell %.4g)\n", h, n, ctx->grid_cell);
  }
#endif
  return 0;
}

namespace {

int do_error_impl(sgb_ctx* ctx, const double* T, double* d_out) {
  if (!T) return fail(ctx, 1, "sgb_error: null pose");
  if (!ctx->have_lin) return fail(ctx, 1, "sgb_error: no preceding sgb_linearize (the correspondences are cached there)");
  CU(cudaSetDevice(ctx->device));
  if (ctx->n_src == 0 || ctx->n_tgt == 0) return zero_result(ctx, T, d_out, false);
  // point targets: the factor kernel's operand pipeline (one wave of CTAs looping over tiles); voxel-map targets and the profiling switch
  // SGB_ERROR_PIPE=0: the plain grid-stride kernel
  const bool pipelined = ctx->tgt_state != TargetState::VoxelMap && ctx->error_pipelined;
  const int grid = one_wave_grid(ctx->n_src, ctx->sm_count, pipelined ? error_pipelined_occupancy(ctx->lin_factor, ctx->lin_robust) : 8);
  if (int rc = ensure_reduction_buffers(ctx, grid)) return rc;
  LinParams P;
  fill_params(ctx, P, T);
  std::memcpy(P.Tlin, ctx->Tlin, sizeof(P.Tlin));
  P.robust_c = ctx->lin_c;
  P.out = d_out;
  if (pipelined)
    CU(launch_error_pipelined(P, ctx->lin_factor, ctx->lin_robust, grid, ctx->stream));
  else
    CU(launch_error(P, ctx->lin_factor, ctx->lin_robust, grid, ctx->stream));
  ctx->launches += 1;
  return 0;
}


// With the fused multi-GPU exchange every rank must issue the same sequence of collective reductions.  A call that fails on the
// host of ONE rank (bad argument, missing covariances, a CUDA error) before its reduction kernel was launched would leave that rank
// one sequence number behind its peers for good: they would spin into the timeout, and every later exchange would mismatch.
// The wrappers therefore make a failed call collective-safe: the rank still takes its sequence number and launches a one-CTA
// kernel that tells the peers "nothing valid from me" (kCommPoison) -- they get NaN + a non-zero status immediately instead of a
// timeout -- and the context refuses further work until sgb_comm_connect* is called again.
int comm_poison(sgb_ctx* ctx, const double* T, double* d_out, bool linearize) {
  static const double identity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  const std::string first_error = ctx->err;
  ctx->comm_failed = true;
  if (ensure_reduction_buffers(ctx, 1) == 0 && d_out) {
    LinParams P0;
    fill_params(ctx, P0, T ? T : identity);
    P0.comm.poison = 1;
    P0.out = d_out;
    if (launch_reduce_nothing(P0, linearize, ctx->stream) == cudaSuccess) ctx->launches += 1;
  }
  ctx->err = first_error + " [multi-GPU: the peers were told; call sgb_comm_connect again before the next collective call]";
  return 0;
}

int do_linearize(sgb_ctx* ctx, int factor, int robust, double robust_c, int rejector, double max_dist_sq, const double* T, double* d_out) {
  if (int rc = single_target_check(ctx, "sgb_linearize")) return rc;
  if (ctx->src_state == SourceState::Batch) return fail(ctx, 1, "sgb_linearize: the context holds a batch of sources (sgb_source_set_batch); use sgb_linearize_batch");
  if (ctx->comm_failed) return fail(ctx, 5, "sgb_linearize: an earlier multi-GPU exchange of this context failed; call sgb_comm_connect again");
  const unsigned long long seq0 = ctx->comm_seq;
  const int rc = do_linearize_impl(ctx, factor, robust, robust_c, rejector, max_dist_sq, T, d_out);
  if (rc != 0 && ctx->comm_world > 1 && ctx->comm_seq == seq0) comm_poison(ctx, T, d_out, true);
  return rc;
}

int do_error(sgb_ctx* ctx, const double* T, double* d_out) {
  if (int rc = single_target_check(ctx, "sgb_error")) return rc;
  if (ctx->src_state == SourceState::Batch) return fail(ctx, 1, "sgb_error: the context holds a batch of sources (sgb_source_set_batch); use sgb_error_batch");
  if (ctx->comm_failed) return fail(ctx, 5, "sgb_error: an earlier multi-GPU exchange of this context failed; call sgb_comm_connect again");
  const unsigned long long seq0 = ctx->comm_seq;
  const int rc = do_error_impl(ctx, T, d_out);
  if (rc != 0 && ctx->comm_world > 1 && ctx->comm_seq == seq0) comm_poison(ctx, T, d_out, false);
  return rc;
}

// after a host-visible result of a collective call has arrived: did the exchange behind it give up on / hear a failure from a peer?
int comm_check(sgb_ctx* ctx, const char* who) {
  if (ctx->comm_world <= 1) return 0;
  const unsigned int st = *reinterpret_cast<volatile unsigned int*>(ctx->h_out + 60);
  if (st == 0) return 0;
  ctx->comm_failed = true;
  return fail(ctx, 4, std::string(who) + ((st & 2u) ? ": a peer rank reported a failed call" : ": gave up waiting for a peer rank (timeout)") +
                          "; the sums are NaN -- call sgb_comm_connect again on every rank");
}

}  // namespace

// =============================================================================================
extern "C" {

int sgb_create(int device_id, sgb_ctx** out_ctx) {
  if (!out_ctx) return 1;
  *out_ctx = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    g_create_error = std::string("sgb_create: no CUDA device (") + (e != cudaSuccess ? cudaGetErrorString(e) : "count = 0") +
                     "); this library has no CPU fallback";
    return 3;
  }
  if (device_id < 0 || device_id >= count) {
    g_create_error = "sgb_create: device_id out of range";
    return 1;
  }
  e = cudaSetDevice(device_id);
  if (e != cudaSuccess) {
    g_create_error = std::string("cudaSetDevice: ") + cudaGetErrorString(e);
    return 2;
  }
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, device_id);
  if (e != cudaSuccess) {
    g_create_error = std::string("cudaGetDeviceProperties: ") + cudaGetErrorString(e);
    return 2;
  }
  if (prop.major != 9 || prop.minor != 0) {
    g_create_error = "sgb_create: kernels are built for sm_90a (H100) only; found sm_" + std::to_string(prop.major) + std::to_string(prop.minor);
    return 3;
  }
  sgb_ctx* ctx = new sgb_ctx();
  ctx->device = device_id;
  ctx->sm_count = prop.multiProcessorCount;
  e = cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_entry, cudaEventDisableTiming);
  for (int k = 0; k < sgb_ctx::kUploadChunks && e == cudaSuccess; k++) e = cudaEventCreateWithFlags(&ctx->ev_upload[k], cudaEventDisableTiming);
  // result slot in MAPPED page-locked host memory: the finishing CTA of a reduction writes H|b|e straight into it over PCIe, so the
  // host-returning calls (sgb_linearize / sgb_error) need no device-to-host copy behind the kernel, just the stream synchronisation
  if (e == cudaSuccess) e = cudaHostAlloc(reinterpret_cast<void**>(&ctx->h_out), 64 * sizeof(double), cudaHostAllocMapped);
  if (e == cudaSuccess) e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&ctx->h_out_dev), ctx->h_out, 0);
  if (e != cudaSuccess) {
    g_create_error = std::string("sgb_create: ") + cudaGetErrorString(e);
    delete ctx;
    return 2;
  }
  ctx->stream = ctx->own_stream;
#ifdef SGB_PROFILING  // libsgicp_b200_prof.so only: the A/B switches of the experiments (the product library reads no environment variable)
  if (const char* s = getenv("SGB_SEARCH")) ctx->search_mode = atoi(s);  // profiling switch: 0 fused, 1 per-thread, 2 packet
  if (const char* s = getenv("SGB_CURVE")) set_source_curve(atoi(s));     // profiling switch: 0 Morton, 1 Hilbert (default)
  if (const char* s = getenv("SGB_GRID")) ctx->use_grid = !(s[0] == '0');  // profiling switch: 0 = tree search only
  // profiling switches of the grid front end (A/B runs, variants exercised by tests/test_gpu_parity.py)
  if (const char* s = getenv("SGB_RING")) ctx->use_ring = !(s[0] == '0');                   // 0 = pending queries always walk the tree
  if (const char* s = getenv("SGB_PENDING_DIV")) ctx->pending_div = std::max(1, atoi(s));   // packet search when more than n / div queries are pending
  if (const char* s = getenv("SGB_GRID_CELL")) {                                            // cell edge in units of the median point spacing
    const double v = atof(s);
    if (v > 0.1 && v < 100.0) ctx->grid_cell_factor = v;
  }
  if (const char* s = getenv("SGB_PACKET_QUEUE")) ctx->use_packet_queue = !(s[0] == '0');   // 0 = chunks assigned to warps by a static stride
  if (const char* s = getenv("SGB_CHUNK_CLASSES")) ctx->use_chunk_classes = !(s[0] == '0');  // 0 = no work lists by cost class: chunks in curve order
  if (const char* s = getenv("SGB_KD_SMEM")) ctx->kd_smem_refine = !(s[0] == '0');  // 0 = kd refinement with one radix sort per level all the way down
  if (const char* s = getenv("SGB_ERROR_PIPE")) ctx->error_pipelined = !(s[0] == '0');  // 0 = Reduction::error through the plain grid-stride kernel
  if (const char* s = getenv("SGB_TMA_LEAF")) ctx->tma_leaf = (s[0] == '1');  // 1 = dense leaf scans read a cp.async.bulk (TMA) staged copy of the leaf
  if (const char* s = getenv("SGB_CLASS_FALLBACK_PCT")) ctx->class_fallback_pct = static_cast<uint32_t>(std::max(0, atoi(s)));
  if (const char* s = getenv("SGB_CLASS_WIDE")) ctx->class_wide_cells = static_cast<float>(atof(s));
  ctx->debug_pending = getenv("SGB_DEBUG_PENDING") != nullptr;
  if (const char* s = getenv("SGB_TREE")) {  // profiling switch: "host" = kd-tree built on the host, "lbvh" = Hilbert-order linear BVH without refinement
    ctx->host_tree = (s[0] == 'h');
    if (s[0] == 'l') ctx->tree_quality = 0;
  }
  if (ctx->search_mode != 2) ctx->host_tree = true;                        // the per-thread / fused kernels walk 8-byte kd nodes
#endif
  *out_ctx = ctx;
  return 0;
}

void sgb_destroy(sgb_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  sgb_comm_disconnect(ctx);  // unmaps the peers' mailboxes
  if (ctx->h_out) cudaFreeHost(ctx->h_out);
  if (ctx->copy_stream) {
    cudaStreamSynchronize(ctx->copy_stream);
    cudaStreamDestroy(ctx->copy_stream);
  }
  if (ctx->ev_entry) cudaEventDestroy(ctx->ev_entry);
  for (int k = 0; k < sgb_ctx::kUploadChunks; k++)
    if (ctx->ev_upload[k]) cudaEventDestroy(ctx->ev_upload[k]);
  if (ctx->cap_stream) cudaStreamDestroy(ctx->cap_stream);
  if (ctx->cap_stream_nested) cudaStreamDestroy(ctx->cap_stream_nested);
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  delete ctx;  // every DevBuf and LoopGraph member frees what it owns (the context's device is current)
}

const char* sgb_last_error(const sgb_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int sgb_set_stream(sgb_ctx* ctx, void* cuda_stream) {
  if (!ctx) return 1;
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->own_stream;
  return 0;
}

int sgb_synchronize(sgb_ctx* ctx) {
  if (!ctx) return 1;
  CU(cudaSetDevice(ctx->device));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

uint64_t sgb_kernel_launches(const sgb_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ---- multi-GPU exchange ----------------------------------------------------------------------
static int comm_ensure_mailbox(sgb_ctx* ctx) {
  if (ctx->comm_mail.p) return 0;
  CU(cudaSetDevice(ctx->device));
  CU(ctx->comm_mail.reserve(kMailBytes));
  CU(cudaMemset(ctx->comm_mail.p, 0, ctx->comm_mail.cap));  // flags = 0: no call has sequence number 0
  CU(ctx->comm_status.reserve(64 + kCommStampRing * sizeof(unsigned long long)));  // [0]: sticky status word, [64..]: wait-time ring
  CU(cudaMemset(ctx->comm_status.p, 0, ctx->comm_status.cap));
  return 0;
}

int sgb_comm_mailbox(sgb_ctx* ctx, void** out_device_ptr) {
  if (!ctx || !out_device_ptr) return 1;
  if (int rc = comm_ensure_mailbox(ctx)) return rc;
  *out_device_ptr = ctx->comm_mail.p;
  return 0;
}

int sgb_comm_handle(sgb_ctx* ctx, void* out_handle64) {
  if (!ctx || !out_handle64) return 1;
  static_assert(sizeof(cudaIpcMemHandle_t) == SGB_COMM_HANDLE_BYTES, "IPC handle size");
  if (int rc = comm_ensure_mailbox(ctx)) return rc;
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, ctx->comm_mail.p));
  std::memcpy(out_handle64, &h, sizeof(h));
  return 0;
}

int sgb_comm_disconnect(sgb_ctx* ctx) {
  if (!ctx) return 1;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  for (int p = 0; p < kMaxPeers; p++) {
    if (ctx->comm_ipc_opened[p] && ctx->comm_peers[p]) cudaIpcCloseMemHandle(ctx->comm_peers[p]);
    ctx->comm_ipc_opened[p] = false;
    ctx->comm_peers[p] = nullptr;
  }
  ctx->comm_world = 0;
  ctx->comm_rank = 0;
  ctx->comm_failed = false;
  return 0;
}

int sgb_comm_set_timeout_ms(sgb_ctx* ctx, int milliseconds) {
  if (!ctx) return 1;
  if (milliseconds < 1) return fail(ctx, 1, "sgb_comm_set_timeout_ms: need a positive time");
  ctx->comm_timeout_ns = static_cast<unsigned long long>(milliseconds) * 1000000ull;
  return 0;
}

int sgb_comm_status(sgb_ctx* ctx, int* out_status) {
  if (!ctx || !out_status) return 1;
  *out_status = 0;
  if (!ctx->comm_status.p) return 0;
  CU(cudaSetDevice(ctx->device));
  unsigned int st = 0;
  CU(cudaMemcpyAsync(&st, ctx->comm_status.p, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (st) ctx->comm_failed = true;
  *out_status = static_cast<int>(st);
  return 0;
}

int sgb_comm_wait_ns(sgb_ctx* ctx, uint64_t* out_ring64, uint64_t* out_calls) {
  if (!ctx || !out_ring64) return 1;
  std::memset(out_ring64, 0, kCommStampRing * sizeof(uint64_t));
  if (out_calls) *out_calls = ctx->comm_seq;
  if (!ctx->comm_status.p) return 0;
  CU(cudaSetDevice(ctx->device));
  CU(cudaMemcpyAsync(out_ring64, ctx->comm_status.as<unsigned char>() + 64, kCommStampRing * sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

int sgb_comm_connect_ptrs(sgb_ctx* ctx, int rank, int world, void* const* mailboxes) {
  if (!ctx) return 1;
  if (world < 1 || world > kMaxPeers || rank < 0 || rank >= world || !mailboxes) return fail(ctx, 1, "sgb_comm_connect: need 1 <= world <= 8, 0 <= rank < world");
  if (int rc = comm_ensure_mailbox(ctx)) return rc;
  sgb_comm_disconnect(ctx);
  for (int p = 0; p < world; p++) {
    if (!mailboxes[p]) return fail(ctx, 1, "sgb_comm_connect: null mailbox");
    ctx->comm_peers[p] = static_cast<unsigned char*>(mailboxes[p]);
  }
  if (ctx->comm_peers[rank] != ctx->comm_mail.p) return fail(ctx, 1, "sgb_comm_connect: mailboxes[rank] is not this context's mailbox");
  // a fresh epoch: clear the flags and restart the sequence (every rank does the same before its first exchange;
  // the caller separates connect from the first linearize by a barrier, as with any communicator construction)
  CU(cudaMemset(ctx->comm_mail.p, 0, ctx->comm_mail.cap));
  CU(cudaMemset(ctx->comm_status.p, 0, ctx->comm_status.cap));
  ctx->comm_failed = false;
  ctx->comm_seq = 0;
  ctx->comm_world = world;
  ctx->comm_rank = rank;
  return 0;
}

int sgb_comm_connect(sgb_ctx* ctx, int rank, int world, const void* handles) {
  if (!ctx) return 1;
  if (world < 1 || world > kMaxPeers || rank < 0 || rank >= world || !handles) return fail(ctx, 1, "sgb_comm_connect: need 1 <= world <= 8, 0 <= rank < world");
  if (int rc = comm_ensure_mailbox(ctx)) return rc;
  sgb_comm_disconnect(ctx);
  CU(cudaSetDevice(ctx->device));
  void* ptrs[kMaxPeers] = {};
  bool opened[kMaxPeers] = {};
  for (int p = 0; p < world; p++) {
    if (p == rank) {
      ptrs[p] = ctx->comm_mail.p;
      continue;
    }
    cudaIpcMemHandle_t h;
    std::memcpy(&h, static_cast<const unsigned char*>(handles) + static_cast<size_t>(p) * SGB_COMM_HANDLE_BYTES, sizeof(h));
    const cudaError_t e = cudaIpcOpenMemHandle(&ptrs[p], h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      for (int q = 0; q < p; q++)
        if (opened[q]) cudaIpcCloseMemHandle(ptrs[q]);
      return fail(ctx, 2, std::string("sgb_comm_connect: cudaIpcOpenMemHandle(rank ") + std::to_string(p) + "): " + cudaGetErrorString(e));
    }
    opened[p] = true;
  }
  if (int rc = sgb_comm_connect_ptrs(ctx, rank, world, ptrs)) {
    for (int p = 0; p < world; p++)
      if (opened[p]) cudaIpcCloseMemHandle(ptrs[p]);
    sgb_comm_disconnect(ctx);  // forget the (now unmapped) pointers
    return rc;
  }
  for (int p = 0; p < world; p++) ctx->comm_ipc_opened[p] = opened[p];
  return 0;
}
size_t sgb_target_size(const sgb_ctx* ctx) { return ctx ? ctx->n_tgt : 0; }
size_t sgb_source_size(const sgb_ctx* ctx) { return ctx ? ctx->n_src : 0; }

// ---------------------------------------------------------------------------------------------
int sgb_target_set_points(sgb_ctx* ctx, size_t n, const double* points, const double* normals, const double* covs) {
  if (!ctx) return 1;
  if (n && !points) return fail(ctx, 1, "sgb_target_set_points: null points");
  if (n >= (1ull << 31)) return fail(ctx, 1, "sgb_target_set_points: too many points");
  CU(cudaSetDevice(ctx->device));
  // without normals or covariances, features may still be estimated on the device (sgb_target_estimate_features): keep the rounding residuals
  const bool keep_lo = !normals || !covs;
  if (int rc = begin_point_target(ctx, n, normals != nullptr, covs != nullptr, keep_lo)) return rc;
  if (n == 0) return 0;
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  CU(cudaMemcpyAsync(ctx->stage_pts.p, points, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (normals) {
    CU(ctx->stage_normals.reserve(n * 4 * sizeof(double)));
    CU(cudaMemcpyAsync(ctx->stage_normals.p, normals, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
    CU(ctx->tgt_orig_normals.reserve(n * sizeof(float4)));
  }
  if (covs) {
    CU(ctx->stage_covs.reserve(n * 16 * sizeof(double)));
    CU(cudaMemcpyAsync(ctx->stage_covs.p, covs, n * 16 * sizeof(double), cudaMemcpyDefault, ctx->stream));
    CU(ctx->tgt_orig_covA.reserve(n * sizeof(float4)));
    CU(ctx->tgt_orig_covB.reserve(n * sizeof(float4)));
  }
  CU(ctx->tgt_orig_pts.reserve(n * sizeof(float4)));
  if (keep_lo) CU(ctx->tgt_orig_lo.reserve(n * sizeof(float4)));
  CU(launch_bounds_centre(ctx->stage_pts.as<double>(), n, ctx->tgt_bounds.as<double>(), ctx->tgt_centre.as<double>(), ctx->sm_count, ctx->stream));
  CU(launch_convert(ctx->stage_pts.as<double>(), normals ? ctx->stage_normals.as<double>() : nullptr, covs ? ctx->stage_covs.as<double>() : nullptr, n,
                    ctx->tgt_centre.as<double>(), ctx->tgt_orig_pts.as<float4>(), ctx->tgt_orig_normals.as<float4>(), ctx->tgt_orig_covA.as<float4>(),
                    ctx->tgt_orig_covB.as<float4>(), nullptr, nullptr, ctx->sm_count, ctx->stream, keep_lo ? ctx->tgt_orig_lo.as<float4>() : nullptr));
  ctx->launches += 4;
  // pageable host memory: the async copies above are staged synchronously, nothing else borrows the inputs
  return 0;
}

int sgb_target_set_kdtree(sgb_ctx* ctx, const void* nodes24, size_t n_nodes, uint32_t root, const uint64_t* indices) {
  if (!ctx) return 1;
  if (ctx->tgt_state == TargetState::VoxelMap || ctx->tgt_state == TargetState::VoxelMaps)
    return fail(ctx, 1, "sgb_target_set_kdtree: the target is a voxel map; call sgb_target_set_points first");
  if (ctx->tgt_state == TargetState::KdTrees)
    return fail(ctx, 1, "sgb_target_set_kdtree: the target holds many kd-trees (sgb_target_build_kdtrees); call sgb_target_set_points first");
  if (ctx->n_tgt == 0) {
    ctx->tgt_state = TargetState::Tree;  // nothing to search
    return 0;
  }
  if (!nodes24 || !indices) return fail(ctx, 1, "sgb_target_set_kdtree: null tree");
  CU(cudaSetDevice(ctx->device));
  double centre[4];
  CU(cudaMemcpyAsync(centre, ctx->tgt_centre.p, sizeof(centre), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  FlatTree tree;
  std::string err;
  if (!flatten_reference_tree(nodes24, n_nodes, root, indices, ctx->n_tgt, centre, tree, err)) return fail(ctx, 1, "sgb_target_set_kdtree: " + err);
  std::vector<float> pts(ctx->n_tgt * 4);  // centred FP32 points, for the children bounding boxes
  CU(cudaMemcpyAsync(pts.data(), ctx->tgt_orig_pts.p, ctx->n_tgt * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return upload_tree(ctx, tree, pts.data());
}

int sgb_target_build_kdtree(sgb_ctx* ctx, int max_leaf_size) {
  if (!ctx) return 1;
  if (ctx->tgt_state == TargetState::VoxelMap || ctx->tgt_state == TargetState::VoxelMaps)
    return fail(ctx, 1, "sgb_target_build_kdtree: the target is a voxel map; call sgb_target_set_points first");
  if (ctx->tgt_state == TargetState::KdTrees)
    return fail(ctx, 1, "sgb_target_build_kdtree: the target holds many kd-trees (sgb_target_build_kdtrees); call sgb_target_set_points first");
  if (ctx->n_tgt == 0) {
    ctx->tgt_state = TargetState::Tree;  // nothing to search
    return 0;
  }
  CU(cudaSetDevice(ctx->device));
#ifdef SGB_PROFILING
  const bool device_build = ctx->search_mode == 2 && !ctx->host_tree;
#else
  const bool device_build = true;
  (void)max_leaf_size;
#endif
  if (device_build) {
    // device-side construction (linear BVH over the Hilbert order, sgb_kernels.cu): no host round trip, fully asynchronous
    const size_t n = ctx->n_tgt;
    int depth = 1;
    if (int rc = build_lbvh(ctx, ctx->tgt_orig_pts.as<float4>(), n, ctx->tgt_centre.as<double>(), ctx->tgt_perm, ctx->tgt_pts, ctx->tgt_pnodes, &depth)) return rc;
    if (depth > 40) return fail(ctx, 1, "sgb_target_build_kdtree: tree too deep");
    if (int rc = gather_target_features(ctx, false)) return rc;
    return install_tree(ctx, depth, (static_cast<size_t>(1) << (depth - 1)) - 1);  // P - 1 records of the implicit tree (depth = log2(P) + 1)
  }
#ifndef SGB_PROFILING
  return fail(ctx, 1, "sgb_target_build_kdtree: unreachable");
#else
  std::vector<float> pts(ctx->n_tgt * 4);
  CU(cudaMemcpyAsync(pts.data(), ctx->tgt_orig_pts.p, ctx->n_tgt * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  FlatTree tree;
  std::string err;
  if (!build_flat_tree(pts.data(), ctx->n_tgt, max_leaf_size, tree, err)) return fail(ctx, 1, "sgb_target_build_kdtree: " + err);
  return upload_tree(ctx, tree, pts.data());
#endif
}

int sgb_target_set_voxelmap(sgb_ctx* ctx, double leaf_size, size_t n_voxels, const int32_t* coords, const double* means, const double* covs, int search_offsets) {
  if (!ctx) return 1;
  if (!(leaf_size > 0.0)) return fail(ctx, 1, "sgb_target_set_voxelmap: leaf_size must be positive");
  if (search_offsets != 1 && search_offsets != 7 && search_offsets != 27) search_offsets = 1;  // incremental_voxelmap.hpp:159-163
  if (n_voxels && (!coords || !means)) return fail(ctx, 1, "sgb_target_set_voxelmap: null input");
  if (n_voxels >= (1ull << 30)) return fail(ctx, 1, "sgb_target_set_voxelmap: too many voxels");
  CU(cudaSetDevice(ctx->device));
  if (int rc = begin_voxel_target(ctx, n_voxels, covs != nullptr, leaf_size, search_offsets)) return rc;
  if (n_voxels == 0) return 0;
  const size_t n = n_voxels;
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  CU(cudaMemcpyAsync(ctx->stage_pts.p, means, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (covs) {
    CU(ctx->stage_covs.reserve(n * 16 * sizeof(double)));
    CU(cudaMemcpyAsync(ctx->stage_covs.p, covs, n * 16 * sizeof(double), cudaMemcpyDefault, ctx->stream));
    CU(ctx->tgt_covA.reserve(n * sizeof(float4)));
    CU(ctx->tgt_covB.reserve(n * sizeof(float4)));
  }
  CU(ctx->tgt_pts.reserve(n * sizeof(float4)));
  CU(launch_bounds_centre(ctx->stage_pts.as<double>(), n, ctx->tgt_bounds.as<double>(), ctx->tgt_centre.as<double>(), ctx->sm_count, ctx->stream));
  CU(launch_convert(ctx->stage_pts.as<double>(), nullptr, covs ? ctx->stage_covs.as<double>() : nullptr, n, ctx->tgt_centre.as<double>(),
                    ctx->tgt_pts.as<float4>(), nullptr, ctx->tgt_covA.as<float4>(), ctx->tgt_covB.as<float4>(), nullptr, nullptr, ctx->sm_count, ctx->stream));
  ctx->launches += 4;
  // open-addressing table (x, y, z, voxel id), load factor <= 0.5, built on the host
  size_t capacity = 16;
  while (capacity < 2 * n) capacity <<= 1;
  std::vector<int32_t> table(capacity * 4, -1);
  const uint32_t mask = static_cast<uint32_t>(capacity - 1);
  for (size_t i = 0; i < n; i++) {
    const int x = coords[i * 3 + 0], y = coords[i * 3 + 1], z = coords[i * 3 + 2];
    uint32_t slot = vox_hash(x, y, z) & mask;
    while (table[slot * 4 + 3] >= 0) {
      if (table[slot * 4 + 0] == x && table[slot * 4 + 1] == y && table[slot * 4 + 2] == z) return fail(ctx, 1, "sgb_target_set_voxelmap: duplicate voxel coordinate");
      slot = (slot + 1) & mask;
    }
    table[slot * 4 + 0] = x;
    table[slot * 4 + 1] = y;
    table[slot * 4 + 2] = z;
    table[slot * 4 + 3] = static_cast<int32_t>(i);
  }
  CU(ctx->vox_table.reserve(capacity * sizeof(int4)));
  CU(cudaMemcpyAsync(ctx->vox_table.p, table.data(), capacity * sizeof(int4), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->vox_mask = mask;
  return 0;
}

// ---------------------------------------------------------------------------------------------
int sgb_source_set_points(sgb_ctx* ctx, size_t n, const double* points, const double* covs) {
  if (!ctx) return 1;
  if (n && !points) return fail(ctx, 1, "sgb_source_set_points: null points");
  if (n >= (1ull << 31)) return fail(ctx, 1, "sgb_source_set_points: too many points");
  CU(cudaSetDevice(ctx->device));
  begin_source(ctx, SourceState::Single, n, covs != nullptr);
  CU(ctx->src_centre.reserve(4 * sizeof(double)));
  CU(ctx->src_bounds.reserve(6 * sizeof(double)));
  if (n == 0) return 0;
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  if (covs) {
    CU(ctx->stage_covs.reserve(n * 16 * sizeof(double)));
    CU(ctx->src_covA.reserve(n * sizeof(float4)));
    CU(ctx->src_covB.reserve(n * sizeof(float4)));
  }
  CU(ctx->tmp_pts.reserve(n * sizeof(float4)));
  CU(ctx->src_pts.reserve(n * sizeof(float4)));
  CU(ctx->corr.reserve(n * sizeof(uint32_t)));
  if (int rc = reserve_query_scratch(ctx, n)) return rc;
  if (int rc = ensure_reduction_buffers(ctx, ctx->sm_count * 8)) return rc;
  // without covariances, they may still be estimated on the device (sgb_source_estimate_features): keep the rounding residuals
  if (!covs) CU(ctx->tmp_lo.reserve(n * sizeof(float4)));
  ctx->src_has_lo = !covs;
  CU(ctx->keys_in.reserve(n * sizeof(uint64_t)));
  CU(ctx->keys_out.reserve(n * sizeof(uint64_t)));
  CU(ctx->vals_in.reserve(n * sizeof(uint32_t)));
  CU(ctx->src_perm.reserve(n * sizeof(uint32_t)));
  CU(ctx->src_rank.reserve(n * sizeof(uint32_t)));
  size_t temp_bytes = 0;
  CU(sort_pairs_u64_u32_bits(nullptr, temp_bytes, ctx->keys_in.as<uint64_t>(), ctx->keys_out.as<uint64_t>(), ctx->vals_in.as<uint32_t>(),
                             ctx->src_perm.as<uint32_t>(), n, 63, ctx->stream));
  CU(ctx->sort_temp.reserve(temp_bytes));

  // The upload is a two-stream pipeline.  The reference layout is 160 B / point, 128 of them the 4x4 double covariance: the points
  // (32 B) go first on the context's stream and are centred, keyed, Hilbert-sorted and gathered WHILE the covariances travel in
  // kUploadChunks pieces on the copy stream; each piece is packed (6 floats) and written straight to its place in the search order
  // as soon as it has arrived, so that after the last byte only 1 / kUploadChunks of the conversion is left.  (Pageable host memory
  // makes cudaMemcpyAsync stage synchronously: same result, no overlap.)  Device pointers are accepted too (cudaMemcpyDefault).
  CU(cudaEventRecord(ctx->ev_entry, ctx->stream));           // everything queued so far (it may still read the staging buffers) ...
  CU(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_entry, 0));  // ... precedes the first chunk
  CU(cudaMemcpyAsync(ctx->stage_pts.p, points, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  const int n_chunks = covs ? static_cast<int>(std::min<size_t>(sgb_ctx::kUploadChunks, (n + 65535) / 65536)) : 0;
  const size_t per_chunk = n_chunks ? (n + n_chunks - 1) / n_chunks : 0;  // as store_source cuts them
  if (covs) {
    // the chunks queue up behind the points on the same DMA engine: wait for the points' copy to have been ISSUED first
    CU(cudaEventRecord(ctx->ev_entry, ctx->stream));
    CU(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_entry, 0));
    for (int k = 0; k < n_chunks; k++) {
      const size_t first = static_cast<size_t>(k) * per_chunk, cnt = std::min(per_chunk, n - first);
      CU(cudaMemcpyAsync(ctx->stage_covs.as<double>() + first * 16, covs + first * 16, cnt * 16 * sizeof(double), cudaMemcpyDefault, ctx->copy_stream));
      CU(cudaEventRecord(ctx->ev_upload[k], ctx->copy_stream));
    }
  }
  uint32_t K = 1;
#ifdef SGB_PROFILING
  if (const char* s = getenv("SGB_RUN")) K = static_cast<uint32_t>(atoi(s)) > 0 ? static_cast<uint32_t>(atoi(s)) : 1;
  while (K > 1 && n / (32ull * K) < static_cast<size_t>(ctx->sm_count) * 16) K >>= 1;
#endif
  ctx->src_run = K;
  return store_source(ctx, 0, n, ctx->src_centre.as<double>(), ctx->src_bounds.as<double>(), covs ? nullptr : ctx->tmp_lo.as<float4>(), temp_bytes, K,
                      n_chunks, ctx->ev_upload);
}

// ---------------------------------------------------------------------------------------------
int sgb_linearize_device(sgb_ctx* ctx, int factor, int robust, double robust_c, int rejector, double max_dist_sq, const double* T, double* d_out44) {
  if (!ctx) return 1;
  if (!d_out44) return fail(ctx, 1, "sgb_linearize_device: null output");
  return do_linearize(ctx, factor, robust, robust_c, rejector, max_dist_sq, T, d_out44);
}

int sgb_linearize(sgb_ctx* ctx, int factor, int robust, double robust_c, int rejector, double max_dist_sq, const double* T, double* out_Hbe43) {
  if (!ctx) return 1;
  if (!out_Hbe43) return fail(ctx, 1, "sgb_linearize: null output");
  CU(cudaSetDevice(ctx->device));
  // the finishing CTA writes H|b|e|inliers straight into the mapped host slot: no copy behind the kernel
  if (int rc = do_linearize(ctx, factor, robust, robust_c, rejector, max_dist_sq, T, ctx->h_out_dev)) return rc;
  if (ctx->comm_world > 1) CU(cudaMemcpyAsync(ctx->h_out + 60, ctx->comm_status.p, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (int rc = comm_check(ctx, "sgb_linearize")) return rc;
  std::memcpy(out_Hbe43, ctx->h_out, 43 * sizeof(double));
  return 0;
}

int sgb_error_device(sgb_ctx* ctx, const double* T, double* d_out1) {
  if (!ctx) return 1;
  if (!d_out1) return fail(ctx, 1, "sgb_error_device: null output");
  return do_error(ctx, T, d_out1);
}

int sgb_error(sgb_ctx* ctx, const double* T, double* out_e) {
  if (!ctx) return 1;
  if (!out_e) return fail(ctx, 1, "sgb_error: null output");
  CU(cudaSetDevice(ctx->device));
  double* d_e = ctx->h_out_dev + 48;  // mapped host slot; H|b|e|inliers of the last linearize stay intact in [0, 44)
  if (int rc = do_error(ctx, T, d_e)) return rc;
  if (ctx->comm_world > 1) CU(cudaMemcpyAsync(ctx->h_out + 60, ctx->comm_status.p, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (int rc = comm_check(ctx, "sgb_error")) return rc;
  *out_e = ctx->h_out[48];
  return 0;
}

int sgb_correspondences(sgb_ctx* ctx, uint64_t* target_index) {
  if (!ctx) return 1;
  if (int rc = single_target_check(ctx, "sgb_correspondences")) return rc;
  if (ctx->src_state == SourceState::Batch) return fail(ctx, 1, "sgb_correspondences: the context holds a batch of sources (sgb_source_set_batch); use sgb_correspondences_batch");
  if (!ctx->have_lin) return fail(ctx, 1, "sgb_correspondences: no preceding sgb_linearize");
  if (ctx->n_src == 0) return 0;
  if (!target_index) return fail(ctx, 1, "sgb_correspondences: null output");
  CU(cudaSetDevice(ctx->device));
  CU(ctx->corr64.reserve(ctx->n_src * sizeof(uint64_t)));
  CU(launch_correspondences(ctx->corr.as<uint32_t>(), ctx->src_perm.as<uint32_t>(), ctx->n_src, ctx->tgt_pts.as<float4>(),
                            ctx->tgt_state == TargetState::VoxelMap ? 1 : 0, ctx->corr64.as<uint64_t>(), ctx->sm_count, ctx->stream));
  ctx->launches += 1;
  CU(cudaMemcpyAsync(target_index, ctx->corr64.p, ctx->n_src * sizeof(uint64_t), cudaMemcpyDefault, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

int sgb_num_inliers(sgb_ctx* ctx, size_t* n) {
  if (!ctx || !n) return 1;
  if (int rc = single_target_check(ctx, "sgb_num_inliers")) return rc;
  if (ctx->src_state == SourceState::Batch) return fail(ctx, 1, "sgb_num_inliers: the context holds a batch of sources (sgb_source_set_batch); sgb_linearize_batch returns each member's count");
  if (!ctx->have_lin || !ctx->last_out) return fail(ctx, 1, "sgb_num_inliers: no preceding sgb_linearize");
  CU(cudaSetDevice(ctx->device));
  if (ctx->last_out == ctx->h_out_dev) {  // sgb_linearize left the count in the mapped host slot
    CU(cudaStreamSynchronize(ctx->stream));
    *n = static_cast<size_t>(ctx->h_out[43] + 0.5);
    return 0;
  }
  CU(cudaMemcpyAsync(ctx->h_out + 56, ctx->last_out + 43, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  *n = static_cast<size_t>(ctx->h_out[56] + 0.5);
  return 0;
}

int sgb_drop_seeds(sgb_ctx* ctx) {
  if (!ctx) return 1;
  ctx->corr_seeds = false;
  ctx->b_dseed_ok = false;
  return 0;
}

}  // extern "C"
