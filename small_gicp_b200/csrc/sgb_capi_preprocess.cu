// SPDX-License-Identifier: MIT
// C-ABI entry points of the per-cloud preparation steps (SURVEY.md §8(f)): normal / covariance estimation and
// voxel-grid down-sampling on the device.  Kernels: sgb_preprocess.cu.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <vector>

#include "../../include/sgicp_b200.h"
#include "sgb_context.hpp"
#include "sgb_forest.h"
#include "sgb_kdtree_host.hpp"
#include "sgb_kernels.h"

using namespace sgb;

namespace sgb {

/// Device-side construction of the search structure over `n` centred FP32 points (original order, w = index):
/// Hilbert keys -> radix sort -> leaf-ordered points -> leaf boxes -> one kernel per level of the implicit binary tree.
/// No host round trip, no synchronisation.  Outputs: perm (leaf order -> original index), leaf_pts, pnodes, depth.
int build_lbvh(sgb_ctx* ctx, const float4* d_orig_pts, size_t n, const double* d_centre4, DevBuf& perm, DevBuf& leaf_pts, DevBuf& pnodes, int* depth) {
  if (n >= (1ull << 30)) return fail(ctx, 1, "too many points for the device tree");
  // P leaf slots (power of two), leaf j = positions [floor(j n / P), floor((j+1) n / P)): at most 32 points each
  uint32_t P = 2;
  int d = 1;
  while (static_cast<uint64_t>(P) * kLbvhLeafPoints < n) {
    P <<= 1;
    d++;
  }
  CU(ctx->keys_in.reserve(n * sizeof(uint64_t)));
  CU(ctx->keys_out.reserve(n * sizeof(uint64_t)));
  CU(ctx->vals_in.reserve(n * sizeof(uint32_t)));
  CU(perm.reserve(n * sizeof(uint32_t)));
  CU(leaf_pts.reserve(n * sizeof(float4)));
  CU(pnodes.reserve(static_cast<size_t>(P - 1) * 64));
  CU(launch_curve_keys(d_orig_pts, n, d_centre4, ctx->keys_in.as<uint64_t>(), ctx->vals_in.as<uint32_t>(), ctx->sm_count, ctx->stream));
  size_t temp_bytes = 0;
  CU(sort_pairs_u64_u32_bits(nullptr, temp_bytes, ctx->keys_in.as<uint64_t>(), ctx->keys_out.as<uint64_t>(), ctx->vals_in.as<uint32_t>(), perm.as<uint32_t>(), n,
                             63, ctx->stream));
  CU(ctx->sort_temp.reserve(temp_bytes));
  CU(sort_pairs_u64_u32_bits(ctx->sort_temp.p, temp_bytes, ctx->keys_in.as<uint64_t>(), ctx->keys_out.as<uint64_t>(), ctx->vals_in.as<uint32_t>(),
                             perm.as<uint32_t>(), n, 63, ctx->stream));
  CU(launch_gather(perm.as<uint32_t>(), n, d_orig_pts, leaf_pts.as<float4>(), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, ctx->sm_count, ctx->stream));
  ctx->launches += 5;
  // (Skipping this refinement for small clouds -- its d radix sorts are pure launch latency at 15k points -- was measured and rejected:
  // the k = 20 searches of the covariance estimation in the unrefined tree cost more than the sorts save.)
  if (ctx->tree_quality >= 1) {
    // median-split refinement: level by level, sort every node's points along the widest axis of its box; the balanced
    // position boundaries of the next level are then exactly the median splits of a kd-tree (same quality as the host
    // builder, ~d radix sorts instead of a D2H + recursive host build + H2D)
    CU(ctx->pre_boxes.reserve(static_cast<size_t>(P) * 6 * sizeof(uint32_t)));
    // top levels (nodes larger than a shared-memory segment): one radix sort per level; every subtree below is refined by ONE launch
    const int level0 = ctx->kd_smem_refine ? static_cast<int>(kd_smem_first_level(static_cast<uint32_t>(n), static_cast<uint32_t>(d))) : d;
    for (int level = 0; level < level0; level++) {
      const uint32_t count = 1u << level;
      CU(launch_kd_level_keys(leaf_pts.as<float4>(), static_cast<uint32_t>(n), count, ctx->pre_boxes.as<uint32_t>(), ctx->keys_in.as<uint64_t>(), ctx->stream));
      CU(cudaMemcpyAsync(ctx->vals_in.p, perm.p, n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
      size_t tb = 0;
      CU(sort_pairs_u64_u32_bits(nullptr, tb, ctx->keys_in.as<uint64_t>(), ctx->keys_out.as<uint64_t>(), ctx->vals_in.as<uint32_t>(), perm.as<uint32_t>(), n,
                                 32 + level, ctx->stream));
      CU(ctx->sort_temp.reserve(tb));
      CU(sort_pairs_u64_u32_bits(ctx->sort_temp.p, tb, ctx->keys_in.as<uint64_t>(), ctx->keys_out.as<uint64_t>(), ctx->vals_in.as<uint32_t>(),
                                 perm.as<uint32_t>(), n, 32 + level, ctx->stream));
      CU(launch_gather(perm.as<uint32_t>(), n, d_orig_pts, leaf_pts.as<float4>(), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, ctx->sm_count,
                       ctx->stream));
      ctx->launches += 8;
    }
    if (level0 < d) {
      CU(launch_kd_refine_smem(leaf_pts.as<float4>(), perm.as<uint32_t>(), static_cast<uint32_t>(n), static_cast<uint32_t>(level0), static_cast<uint32_t>(d), ctx->stream));
      ctx->launches += 1;
    }
  }
  int launches = 0;
  CU(launch_lbvh_build(leaf_pts.as<float4>(), static_cast<uint32_t>(n), P, pnodes.as<float4>(), &launches, ctx->stream));
  ctx->launches += launches;
  *depth = d + 1;
  return 0;
}

/// Uniform grid over the leaf-ordered target points.  Cell edge = 3 x the median point spacing of the tree's leaves, so the
/// settle radius (half a cell) is ~3 mean nearest-neighbour distances of a surface sampled like the target.
int build_grid(sgb_ctx* ctx) {
  ctx->grid_ready = false;
  const size_t n = ctx->n_tgt;
  if (!ctx->use_grid || ctx->search_mode != 2 || ctx->tgt_state != TargetState::Tree || n < 1024 || ctx->n_pnodes == 0) return 0;
  // spacing estimate from the leaf boxes + the target box (one small D2H, construction is a per-target one-off)
  const size_t m = ctx->n_pnodes * 2;
  CU(ctx->grid_spacing.reserve(m * sizeof(float)));
  CU(launch_grid_spacing(ctx->tgt_pnodes.as<float4>(), static_cast<uint32_t>(ctx->n_pnodes), ctx->grid_spacing.as<float>(), ctx->stream));
  std::vector<float> sp(m);
  double bounds[6], centre[4];
  CU(cudaMemcpyAsync(sp.data(), ctx->grid_spacing.p, m * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(bounds, ctx->tgt_bounds.p, sizeof(bounds), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(centre, ctx->tgt_centre.p, sizeof(centre), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  size_t k = 0;
  for (size_t i = 0; i < m; i++)
    if (sp[i] > 0.f) sp[k++] = sp[i];
  if (k == 0) return 0;
  std::nth_element(sp.begin(), sp.begin() + k / 2, sp.begin() + k);
  double cell = ctx->grid_cell_factor * sp[k / 2];
  double ext = 0.0;
  for (int a = 0; a < 3; a++) ext = std::max(ext, bounds[3 + a] - bounds[a]);
  if (!(cell > 0.0) || !(ext > 0.0)) return 0;
  cell = std::max(cell, ext / 8000.0);  // cell indices < 2^13: FP32 cell coordinates stay accurate to 1e-3 cells (kGridSlack in sgb_grid.cu)
  GridParams g;
  for (int a = 0; a < 3; a++) g.origin[a] = static_cast<float>(bounds[a] - centre[a]);
  g.inv_cell = static_cast<float>(1.0 / cell);
  const double settle = (0.5 - 4e-3) * cell;  // margin for the FP32 cell-coordinate arithmetic (kGridSlack cells, sgb_grid.cu)
  g.settle_d2 = static_cast<float>(settle * settle);
  if (n >= (1ull << 28)) return 0;  // eight anchor entries per point must stay below 2^31
  // compact sort keys: B bits per axis hold every cell and anchor coordinate (-2 .. cells along the widest axis + 1, biased by 2) with the
  // all-ones pad left over; at most 13 bits (cell indices < 2^13)
  const double cells_axis = std::ceil(ext / cell) + 2.0;
  int bits = 1;
  while (static_cast<double>((1ull << bits) - 1ull) <= cells_axis + 4.0) bits++;
  const size_t m_ent = n * 8;  // anchor entries: eight per point, real ones at the first point of each cell
  CU(ctx->keys_in.reserve(m_ent * sizeof(uint64_t)));
  CU(ctx->keys_out.reserve(m_ent * sizeof(uint64_t)));
  CU(ctx->vals_in.reserve(m_ent * sizeof(uint32_t)));
  CU(ctx->pre_vals_out.reserve(m_ent * sizeof(uint32_t)));
  CU(ctx->pre_heads.reserve(n * sizeof(uint32_t)));
  CU(ctx->grid_pts.reserve(n * sizeof(float4)));
  CU(ctx->grid_pending.reserve(2 * sizeof(uint32_t)));
  size_t tb = 0;
  CU(sort_pairs_u64_u32_bits(nullptr, tb, ctx->keys_in.as<uint64_t>(), ctx->keys_out.as<uint64_t>(), ctx->vals_in.as<uint32_t>(), ctx->pre_vals_out.as<uint32_t>(),
                             m_ent, 3 * bits, ctx->stream));
  CU(ctx->sort_temp.reserve(tb));
  uint32_t* d_counters = ctx->grid_pending.as<uint32_t>();  // the two pending counters double as scratch during construction
  CU(launch_grid_build(ctx->tgt_pts.as<float4>(), static_cast<uint32_t>(n), g, bits, ctx->keys_in.as<uint64_t>(), ctx->keys_out.as<uint64_t>(),
                       ctx->vals_in.as<uint32_t>(), ctx->pre_vals_out.as<uint32_t>(), ctx->sort_temp.p, tb, ctx->grid_pts.as<float4>(), ctx->pre_heads.as<uint32_t>(),
                       d_counters, ctx->stream));
  ctx->pending_clean = false;  // the two counters of the construction live in the pending counters
  uint32_t counters[2] = {0, 0};  // distinct anchors (= non-empty blocks), largest block
  CU(cudaMemcpyAsync(counters, d_counters, sizeof(counters), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const uint32_t distinct = counters[0], max_block = counters[1];
  ctx->launches += 7;
  uint32_t capacity = 1024;
  while (capacity < 2ull * distinct) capacity <<= 1;  // load factor <= 1/2
  if (ctx->debug_pending)
    std::fprintf(stderr, "[sgb] grid front end: cell %.9g (origin %a %a %a, inv_cell %a), %d key bits, %u blocks, largest block %u points, %.1f B/point%s\n", cell,
                 g.origin[0], g.origin[1], g.origin[2], g.inv_cell, 3 * bits, distinct, max_block,
                 (16.0 * static_cast<double>(n) + static_cast<double>(capacity) * sizeof(GridSlot)) / static_cast<double>(n),
                 max_block > kGridMaxList ? ", dropped" : "");
  if (max_block > kGridMaxList) return 0;  // degenerate density (see kGridMaxList): the tree search alone stays exact and bounded
  // one slot per non-empty block
  CU(ctx->grid_table.reserve(static_cast<size_t>(capacity) * sizeof(GridSlot)));
  CU(launch_grid_fill(ctx->keys_out.as<uint64_t>(), ctx->pre_vals_out.as<uint32_t>(), static_cast<uint32_t>(m_ent), ctx->pre_heads.as<uint32_t>(), bits,
                      ctx->grid_table.as<GridSlot>(), capacity, ctx->stream));
  ctx->launches += 2;
  for (int a = 0; a < 3; a++) ctx->grid_origin[a] = g.origin[a];
  ctx->grid_inv_cell = g.inv_cell;
  ctx->grid_settle_d2 = g.settle_d2;
  ctx->grid_cell = static_cast<float>(cell);
  ctx->grid_capacity = capacity;
  ctx->grid_ready = true;
  return 0;
}

}  // namespace sgb

namespace {

// Sorts the n points at stage_pts into voxels of edge 1 / inv_leaf: keys_out / pre_vals_out = voxel keys / point indices in key order,
// pre_heads[j] = 1 where a voxel starts, pre_slots = their exclusive scan (pre_slots[n] = voxel count).  7 launches.
int sort_into_voxels(sgb_ctx* ctx, size_t n, double inv_leaf) {
  CU(ctx->keys_in.reserve(n * sizeof(uint64_t)));
  CU(ctx->keys_out.reserve(n * sizeof(uint64_t)));
  CU(ctx->vals_in.reserve(n * sizeof(uint32_t)));
  CU(ctx->pre_vals_out.reserve(n * sizeof(uint32_t)));
  CU(ctx->pre_heads.reserve((n + 1) * sizeof(uint32_t)));
  CU(ctx->pre_slots.reserve((n + 1) * sizeof(uint32_t)));
  CU(launch_voxel_keys(ctx->stage_pts.as<double>(), n, inv_leaf, ctx->keys_in.as<uint64_t>(), ctx->vals_in.as<uint32_t>(), ctx->sm_count, ctx->stream));
  size_t temp_bytes = 0, scan_bytes = 0;
  CU(sort_pairs_u64_u32_bits(nullptr, temp_bytes, ctx->keys_in.as<uint64_t>(), ctx->keys_out.as<uint64_t>(), ctx->vals_in.as<uint32_t>(),
                             ctx->pre_vals_out.as<uint32_t>(), n, 63, ctx->stream));
  CU(exclusive_sum_u32(nullptr, scan_bytes, ctx->pre_heads.as<uint32_t>(), ctx->pre_slots.as<uint32_t>(), n + 1, ctx->stream));
  CU(ctx->sort_temp.reserve(temp_bytes > scan_bytes ? temp_bytes : scan_bytes));
  CU(sort_pairs_u64_u32_bits(ctx->sort_temp.p, temp_bytes, ctx->keys_in.as<uint64_t>(), ctx->keys_out.as<uint64_t>(), ctx->vals_in.as<uint32_t>(),
                             ctx->pre_vals_out.as<uint32_t>(), n, 63, ctx->stream));
  CU(cudaMemsetAsync(ctx->pre_heads.p, 0, (n + 1) * sizeof(uint32_t), ctx->stream));
  CU(launch_voxel_heads(ctx->keys_out.as<uint64_t>(), n, ctx->pre_heads.as<uint32_t>(), ctx->sm_count, ctx->stream));
  CU(exclusive_sum_u32(ctx->sort_temp.p, scan_bytes, ctx->pre_heads.as<uint32_t>(), ctx->pre_slots.as<uint32_t>(), n + 1, ctx->stream));
  ctx->launches += 7;
  return 0;
}

// n_maps clouds (host offsets, checked; offsets[n_maps] = n > 0) at stage_pts sorted into per-cloud voxels of edge 1 / inv_leaf
// (sgb_preprocess.cu: voxelmaps_*): keys_in / vals_in = voxel keys (bit 63 = the parity of the cloud's rank among the clouds with points)
// / original indices in (cloud, valid, key) order, pre_heads[0, n] = voxel heads, pre_slots = their exclusive scan (pre_slots[n] = voxel
// count), regions[m].z / .w = cloud m's first voxel / voxel count, vm_caps[0, n_maps] = the table capacity of each cloud's voxel map.
// sort_temp holds cap_scan_bytes, enough for the scan of those capacities.  7 launches, none of them per cloud.
int sort_into_voxelmaps(sgb_ctx* ctx, size_t n_maps, const size_t* offsets, double inv_leaf, uint4* regions, size_t& cap_scan_bytes) {
  const size_t n = offsets[n_maps];
  const uint32_t maps = static_cast<uint32_t>(n_maps);
  // the point offsets, then per map the parity of its rank among the maps with points (bit 63 of its stored keys, sgb_preprocess.cu)
  std::vector<uint32_t> off32(offsets, offsets + n_maps + 1);
  off32.resize(2 * n_maps + 1);
  uint32_t rank = 0;
  for (size_t m = 0; m < n_maps; m++) {
    off32[n_maps + 1 + m] = rank & 1u;
    if (offsets[m + 1] > offsets[m]) rank++;
  }
  CU(ctx->vm_offsets.reserve(off32.size() * sizeof(uint32_t)));
  CU(ctx->vm_caps.reserve(2 * (n_maps + 1) * sizeof(uint32_t)));
  CU(ctx->vm_keys.reserve(n * sizeof(uint64_t)));
  CU(ctx->vm_vals.reserve(n * sizeof(uint32_t)));
  CU(cudaMemcpyAsync(ctx->vm_offsets.p, off32.data(), off32.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  CU(ctx->keys_in.reserve(n * sizeof(uint64_t)));
  CU(ctx->keys_out.reserve(n * sizeof(uint64_t)));
  CU(ctx->vals_in.reserve(n * sizeof(uint32_t)));
  CU(ctx->pre_vals_out.reserve(n * sizeof(uint32_t)));
  CU(ctx->pre_heads.reserve((n + 1) * sizeof(uint32_t)));
  CU(ctx->pre_slots.reserve((n + 1) * sizeof(uint32_t)));
  int map_bits = 1;  // (map << 1 | valid) < 2 n_maps
  while ((1ull << map_bits) < 2ull * n_maps) map_bits++;
  uint64_t* keys = ctx->keys_in.as<uint64_t>();
  uint32_t* vals = ctx->vals_in.as<uint32_t>();
  uint32_t* caps = ctx->vm_caps.as<uint32_t>();
  size_t sort_bytes = 0, map_sort_bytes = 0, scan_bytes = 0;
  cap_scan_bytes = 0;
  CU(sort_pairs_u64_u32_bits(nullptr, sort_bytes, keys, ctx->keys_out.as<uint64_t>(), vals, ctx->pre_vals_out.as<uint32_t>(), n, 63, ctx->stream));
  CU(sort_pairs_u64_u32_bits(nullptr, map_sort_bytes, keys, ctx->vm_keys.as<uint64_t>(), vals, ctx->vm_vals.as<uint32_t>(), n, map_bits, ctx->stream));
  CU(exclusive_sum_u32(nullptr, scan_bytes, ctx->pre_heads.as<uint32_t>(), ctx->pre_slots.as<uint32_t>(), n + 1, ctx->stream));
  CU(exclusive_sum_u32(nullptr, cap_scan_bytes, caps, caps + n_maps + 1, n_maps + 1, ctx->stream));
  CU(ctx->sort_temp.reserve(std::max(std::max(sort_bytes, map_sort_bytes), std::max(scan_bytes, cap_scan_bytes))));
  // (map, valid, key) order: the key sort, then a stable sort by (map, valid); keys_in / vals_in end up holding the ordered keys / indices
  CU(launch_voxel_keys(ctx->stage_pts.as<double>(), n, inv_leaf, keys, vals, ctx->sm_count, ctx->stream));
  CU(sort_pairs_u64_u32_bits(ctx->sort_temp.p, sort_bytes, keys, ctx->keys_out.as<uint64_t>(), vals, ctx->pre_vals_out.as<uint32_t>(), n, 63, ctx->stream));
  CU(launch_voxelmaps_sort_keys(ctx->keys_out.as<uint64_t>(), ctx->pre_vals_out.as<uint32_t>(), n, ctx->vm_offsets.as<uint32_t>(), maps, keys, vals, ctx->sm_count,
                                ctx->stream));
  CU(sort_pairs_u64_u32_bits(ctx->sort_temp.p, map_sort_bytes, keys, ctx->vm_keys.as<uint64_t>(), vals, ctx->vm_vals.as<uint32_t>(), n, map_bits, ctx->stream));
  CU(launch_voxelmaps_order(ctx->vm_keys.as<uint64_t>(), ctx->vm_vals.as<uint32_t>(), ctx->keys_out.as<uint64_t>(), ctx->pre_vals_out.as<uint32_t>(), n,
                            ctx->vm_offsets.as<uint32_t>() + n_maps + 1, keys,
                            vals, ctx->pre_heads.as<uint32_t>(), ctx->sm_count, ctx->stream));
  CU(exclusive_sum_u32(ctx->sort_temp.p, scan_bytes, ctx->pre_heads.as<uint32_t>(), ctx->pre_slots.as<uint32_t>(), n + 1, ctx->stream));
  // per map: voxels and table capacity
  CU(launch_voxelmaps_count(ctx->vm_offsets.as<uint32_t>(), maps, ctx->pre_slots.as<uint32_t>(), regions, caps, ctx->stream));
  ctx->launches += 7;
  return 0;
}

// The layout of a forest over n_maps clouds (host offsets, checked), as build_lbvh sizes one tree per map: P = 2^depth leaf slots of at
// most kLbvhLeafPoints points, P - 1 packet records, and the first level whose nodes fit a shared-memory segment.  tab: the uint32
// ForestTables (pt_off, slot_off, seg_off: n_maps + 1 each; node_base, depth, level0: n_maps each).
struct ForestPlan {
  std::vector<uint32_t> tab;
  uint32_t max_depth = 0, radix_levels = 0, n_segments = 0, n_slots = 0;
  size_t nodes = 0;
  int key_bits = 32;
};
void plan_forest(size_t n_maps, const size_t* offsets, ForestPlan& p) {
  p.tab.assign(3 * (n_maps + 1) + 3 * n_maps, 0);
  uint32_t* pt_off = p.tab.data();
  uint32_t* slot_off = pt_off + (n_maps + 1);
  uint32_t* seg_off = slot_off + (n_maps + 1);
  uint32_t* node_base = seg_off + (n_maps + 1);
  uint32_t* depth = node_base + n_maps;
  uint32_t* level0 = depth + n_maps;
  for (size_t m = 0; m < n_maps; m++) {
    const uint32_t nm = static_cast<uint32_t>(offsets[m + 1] - offsets[m]);
    pt_off[m] = static_cast<uint32_t>(offsets[m]);
    node_base[m] = static_cast<uint32_t>(p.nodes);
    uint32_t P = 0, d = 0, l0 = 0, segs = 0;
    if (nm) {
      P = 2;
      d = 1;
      while (static_cast<uint64_t>(P) * kLbvhLeafPoints < nm) {
        P <<= 1;
        d++;
      }
      l0 = kd_smem_first_level(nm, d);
      segs = 1u << l0;
      p.nodes += P - 1;
    }
    depth[m] = d;
    level0[m] = l0;
    slot_off[m + 1] = slot_off[m] + P;
    seg_off[m + 1] = seg_off[m] + segs;
    p.max_depth = std::max(p.max_depth, d);
    p.radix_levels = std::max(p.radix_levels, l0);
  }
  pt_off[n_maps] = static_cast<uint32_t>(offsets[n_maps]);
  p.n_segments = seg_off[n_maps];
  p.n_slots = slot_off[n_maps];
  p.key_bits = 32;
  while ((1ull << (p.key_bits - 32)) < p.n_segments) p.key_bits++;
}
// the device tables of a plan uploaded to tp
ForestTables forest_tables(const uint32_t* tp, size_t n_maps) {
  return ForestTables{tp, tp + (n_maps + 1), tp + 2 * (n_maps + 1), tp + 3 * (n_maps + 1), tp + 3 * (n_maps + 1) + n_maps,
                      tp + 3 * (n_maps + 1) + 2 * n_maps, static_cast<uint32_t>(n_maps)};
}

// offsets of n_clouds clouds (what: "map" or "cloud") as the many-cloud calls take them: n_clouds + 1 ascending entries from 0
int check_offsets(sgb_ctx* ctx, const std::string& who, size_t n_clouds, const size_t* offsets, const std::string& what) {
  if (n_clouds > SGB_BATCH_MAX_MEMBERS) return fail(ctx, 1, who + std::to_string(n_clouds) + " " + what + "s, at most " + std::to_string(SGB_BATCH_MAX_MEMBERS));
  if (!offsets) return fail(ctx, 1, who + "null offsets");
  if (offsets[0] != 0) return fail(ctx, 1, who + "offsets[0] must be 0");
  for (size_t m = 0; m < n_clouds; m++)
    if (offsets[m + 1] < offsets[m]) return fail(ctx, 1, who + "offsets must be ascending (" + what + " " + std::to_string(m) + ")");
  return 0;
}

}  // namespace

extern "C" {

int sgb_estimate_features(sgb_ctx* ctx, size_t n, const double* points, int num_neighbors, double* out_normals, double* out_covs) {
  if (!ctx) return 1;
  if (n && !points) return fail(ctx, 1, "sgb_estimate_features: null points");
  if (num_neighbors < 1 || num_neighbors > 32) return fail(ctx, 1, "sgb_estimate_features: num_neighbors must be in 1..32");
  if (n >= (1ull << 30)) return fail(ctx, 1, "sgb_estimate_features: too many points");
  if (n == 0 || (!out_normals && !out_covs)) return 0;
  CU(cudaSetDevice(ctx->device));
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  CU(cudaMemcpyAsync(ctx->stage_pts.p, points, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  CU(ctx->pre_centre.reserve(4 * sizeof(double)));
  CU(ctx->pre_bounds.reserve(6 * sizeof(double)));
  CU(ctx->pre_pts.reserve(n * sizeof(float4)));
  CU(ctx->pre_lo.reserve(n * sizeof(float4)));
  CU(launch_bounds_centre(ctx->stage_pts.as<double>(), n, ctx->pre_bounds.as<double>(), ctx->pre_centre.as<double>(), ctx->sm_count, ctx->stream));
  CU(launch_convert(ctx->stage_pts.as<double>(), nullptr, nullptr, n, ctx->pre_centre.as<double>(), ctx->pre_pts.as<float4>(), nullptr, nullptr, nullptr, nullptr,
                    nullptr, ctx->sm_count, ctx->stream, ctx->pre_lo.as<float4>()));
  ctx->launches += 4;
  int depth = 0;
  ctx->src_tree_valid = false;  // the scratch tree buffers are about to hold THIS cloud's tree
  if (int rc = build_lbvh(ctx, ctx->pre_pts.as<float4>(), n, ctx->pre_centre.as<double>(), ctx->pre_perm, ctx->pre_leaf_pts, ctx->pre_nodes, &depth)) return rc;
  if (out_normals) CU(ctx->pre_out_normals.reserve(n * 4 * sizeof(double)));
  if (out_covs) CU(ctx->pre_out_covs.reserve(n * 16 * sizeof(double)));
  const int mode = (out_normals ? 1 : 0) | (out_covs ? 2 : 0);
  CU(launch_features(ctx->pre_nodes.as<float4>(), ctx->pre_leaf_pts.as<float4>(), static_cast<uint32_t>(n), num_neighbors, ctx->pre_centre.as<double>(), mode,
                     nullptr, nullptr, nullptr, out_normals ? ctx->pre_out_normals.as<double>() : nullptr, out_covs ? ctx->pre_out_covs.as<double>() : nullptr,
                     depth, 0, ctx->stream, ctx->pre_lo.as<float4>()));
  ctx->launches += 1;
  if (out_normals) CU(cudaMemcpyAsync(out_normals, ctx->pre_out_normals.p, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (out_covs) CU(cudaMemcpyAsync(out_covs, ctx->pre_out_covs.p, n * 16 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

int sgb_target_estimate_features(sgb_ctx* ctx, int num_neighbors) {
  if (!ctx) return 1;
  if (num_neighbors < 1 || num_neighbors > 32) return fail(ctx, 1, "sgb_target_estimate_features: num_neighbors must be in 1..32");
  if (ctx->tgt_state != TargetState::Tree) return fail(ctx, 1, "sgb_target_estimate_features: needs a point target with its kd-tree (set points, then set/build the tree)");
  const size_t n = ctx->n_tgt;
  features_changed(ctx, true);
  if (n == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  CU(ctx->tgt_normals.reserve(n * sizeof(float4)));
  CU(ctx->tgt_covA.reserve(n * sizeof(float4)));
  CU(ctx->tgt_covB.reserve(n * sizeof(float4)));
  // the target's own tree and leaf-ordered points are already resident: write the features straight into the leaf-ordered streams
  CU(launch_features(ctx->tgt_pnodes.as<float4>(), ctx->tgt_pts.as<float4>(), static_cast<uint32_t>(n), num_neighbors, ctx->tgt_centre.as<double>(), 3,
                     ctx->tgt_normals.as<float4>(), ctx->tgt_covA.as<float4>(), ctx->tgt_covB.as<float4>(), nullptr, nullptr, ctx->tree_depth, 1, ctx->stream,
                     ctx->tgt_has_lo ? ctx->tgt_orig_lo.as<float4>() : nullptr));
  ctx->launches += 1;
  // keep the ORIGINAL-order copies in step (a later sgb_target_build_kdtree / _set_kdtree re-gathers the leaf-ordered streams from them)
  CU(ctx->tgt_orig_normals.reserve(n * sizeof(float4)));
  CU(ctx->tgt_orig_covA.reserve(n * sizeof(float4)));
  CU(ctx->tgt_orig_covB.reserve(n * sizeof(float4)));
  CU(launch_scatter(ctx->tgt_perm.as<uint32_t>(), n, ctx->tgt_normals.as<float4>(), ctx->tgt_orig_normals.as<float4>(), ctx->tgt_covA.as<float4>(),
                    ctx->tgt_orig_covA.as<float4>(), ctx->tgt_covB.as<float4>(), ctx->tgt_orig_covB.as<float4>(), ctx->sm_count, ctx->stream));
  ctx->launches += 1;
  return 0;
}

int sgb_source_estimate_features(sgb_ctx* ctx, int num_neighbors) {
  if (!ctx) return 1;
  if (num_neighbors < 1 || num_neighbors > 32) return fail(ctx, 1, "sgb_source_estimate_features: num_neighbors must be in 1..32");
  if (ctx->src_state == SourceState::Batch) return fail(ctx, 1, "sgb_source_estimate_features: the context holds a batch of sources; pass each member's covariances to sgb_source_set_batch");
  const size_t n = ctx->n_src;
  features_changed(ctx, false);
  if (n == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  // a single source of n > 0 points: tmp_pts holds it in ORIGINAL order (centred FP32, w = index)
  int depth = 0;
  ctx->src_tree_valid = false;
  if (int rc = build_lbvh(ctx, ctx->tmp_pts.as<float4>(), n, ctx->src_centre.as<double>(), ctx->pre_perm, ctx->pre_leaf_pts, ctx->pre_nodes, &depth)) return rc;
  ctx->src_tree_valid = true;  // kept: sgb_target_adopt_source turns this cloud, tree and covariances into the next target
  ctx->src_tree_depth = depth;
  ctx->src_cov_orig_valid = true;
  CU(ctx->tmp_covA.reserve(n * sizeof(float4)));
  CU(ctx->tmp_covB.reserve(n * sizeof(float4)));
  CU(ctx->src_covA.reserve(n * sizeof(float4)));
  CU(ctx->src_covB.reserve(n * sizeof(float4)));
  CU(launch_features(ctx->pre_nodes.as<float4>(), ctx->pre_leaf_pts.as<float4>(), static_cast<uint32_t>(n), num_neighbors, ctx->src_centre.as<double>(), 2, nullptr,
                     ctx->tmp_covA.as<float4>(), ctx->tmp_covB.as<float4>(), nullptr, nullptr, depth, 0, ctx->stream, ctx->src_has_lo ? ctx->tmp_lo.as<float4>() : nullptr));
  // original order -> the search order of the source (chunk-transposed Morton)
  CU(launch_gather(ctx->src_perm.as<uint32_t>(), n, ctx->tmp_covA.as<float4>(), ctx->src_covA.as<float4>(), ctx->tmp_covB.as<float4>(), ctx->src_covB.as<float4>(),
                   nullptr, nullptr, nullptr, nullptr, ctx->sm_count, ctx->stream));
  ctx->launches += 2;
  return 0;
}

int sgb_voxelgrid_sampling(sgb_ctx* ctx, size_t n, const double* points, double leaf_size, double* out_points, size_t* n_out) {
  if (!ctx || !n_out) return 1;
  *n_out = 0;
  if (n && (!points || !out_points)) return fail(ctx, 1, "sgb_voxelgrid_sampling: null buffer");
  if (!(leaf_size > 0.0)) return fail(ctx, 1, "sgb_voxelgrid_sampling: leaf_size must be positive");
  if (n >= (1ull << 31)) return fail(ctx, 1, "sgb_voxelgrid_sampling: too many points");
  if (n == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  CU(cudaMemcpyAsync(ctx->stage_pts.p, points, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (int rc = sort_into_voxels(ctx, n, 1.0 / leaf_size)) return rc;
  CU(ctx->stage_covs.reserve(n * 4 * sizeof(double)));  // output staging (re-uses a scratch buffer)
  CU(launch_voxel_means(ctx->keys_out.as<uint64_t>(), ctx->pre_vals_out.as<uint32_t>(), ctx->pre_heads.as<uint32_t>(), ctx->pre_slots.as<uint32_t>(), n,
                        ctx->stage_pts.as<double>(), ctx->stage_covs.as<double>(), ctx->sm_count, ctx->stream));
  ctx->launches += 1;
  uint32_t count = 0;
  CU(cudaMemcpyAsync(&count, ctx->pre_slots.as<uint32_t>() + n, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (count) {
    CU(cudaMemcpyAsync(out_points, ctx->stage_covs.p, static_cast<size_t>(count) * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  *n_out = count;
  return 0;
}

// Many clouds down-sampled in one pass: the (cloud, valid, key) order of sgb_target_build_voxelmaps (sort_into_voxelmaps), whose bit 63
// stops voxel_means_kernel's run over equal keys at every cloud boundary, so that cloud c's voxels are those of sgb_voxelgrid_sampling
// of cloud c alone, in the same ascending key order, with their sums in the same ascending original index order.
int sgb_voxelgrid_sampling_batch(sgb_ctx* ctx, size_t n_clouds, const size_t* offsets, const double* points, double leaf_size, double* out_points,
                                 size_t* out_offsets) {
  if (!ctx) return 1;
  const std::string who = "sgb_voxelgrid_sampling_batch: ";
  if (!out_offsets) return fail(ctx, 1, who + "null out_offsets");
  if (int rc = check_offsets(ctx, who, n_clouds, offsets, "cloud")) return rc;
  const size_t n = offsets[n_clouds];
  if (n >= (1ull << 31)) return fail(ctx, 1, who + "too many points (fewer than 2^31 in all)");
  if (n && (!points || !out_points)) return fail(ctx, 1, who + "null buffer");
  if (!(leaf_size > 0.0)) return fail(ctx, 1, who + "leaf_size must be positive");
  std::fill(out_offsets, out_offsets + n_clouds + 1, size_t{0});
  if (n == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  CU(cudaMemcpyAsync(ctx->stage_pts.p, points, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  CU(ctx->pre_regions.reserve(n_clouds * sizeof(uint4)));
  size_t cap_scan_bytes = 0;
  if (int rc = sort_into_voxelmaps(ctx, n_clouds, offsets, 1.0 / leaf_size, ctx->pre_regions.as<uint4>(), cap_scan_bytes)) return rc;
  // the means straight into a device-resident output (voxel ids are global, cloud after cloud); a host output goes through staging
  cudaPointerAttributes attr = {};
  CU(cudaPointerGetAttributes(&attr, out_points));
  const bool direct = attr.type == cudaMemoryTypeManaged || (attr.type == cudaMemoryTypeDevice && attr.device == ctx->device);
  if (!direct) CU(ctx->stage_covs.reserve(n * 4 * sizeof(double)));
  double* means = direct ? out_points : ctx->stage_covs.as<double>();
  CU(launch_voxel_means(ctx->keys_in.as<uint64_t>(), ctx->vals_in.as<uint32_t>(), ctx->pre_heads.as<uint32_t>(), ctx->pre_slots.as<uint32_t>(), n,
                        ctx->stage_pts.as<double>(), means, ctx->sm_count, ctx->stream));
  ctx->launches += 1;
  // the one synchronisation: every cloud's first voxel, and the voxel count
  std::vector<uint4> regions(n_clouds);
  uint32_t* h = reinterpret_cast<uint32_t*>(ctx->h_out + 56);
  CU(cudaMemcpyAsync(regions.data(), ctx->pre_regions.p, n_clouds * sizeof(uint4), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(h, ctx->pre_slots.as<uint32_t>() + n, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const uint32_t count = h[0];
  for (size_t c = 0; c < n_clouds; c++) out_offsets[c] = regions[c].z;
  out_offsets[n_clouds] = count;
  if (!direct && count) {
    CU(cudaMemcpyAsync(out_points, ctx->stage_covs.p, static_cast<size_t>(count) * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  return 0;
}

// Features of many clouds: a forest over them (launch_forest_build, as sgb_target_build_kdtrees builds it, here in the preprocessing
// scratch) and the single cloud's features body run on each point's own map (launch_forest_features).  Map m's tree is built from its own
// points alone, so a cloud's results do not depend on the rest of the batch.
int sgb_estimate_features_batch(sgb_ctx* ctx, size_t n_clouds, const size_t* offsets, const double* points, int num_neighbors, double* out_normals,
                                double* out_covs) {
  if (!ctx) return 1;
  const std::string who = "sgb_estimate_features_batch: ";
  if (int rc = check_offsets(ctx, who, n_clouds, offsets, "cloud")) return rc;
  const size_t n = offsets[n_clouds];
  if (num_neighbors < 1 || num_neighbors > 32) return fail(ctx, 1, who + "num_neighbors must be in 1..32");
  if (n >= (1ull << 30)) return fail(ctx, 1, who + "too many points (fewer than 2^30 in all)");
  if (n && !points) return fail(ctx, 1, who + "null points");
  if (n == 0 || (!out_normals && !out_covs)) return 0;
  CU(cudaSetDevice(ctx->device));
  ForestPlan plan;
  plan_forest(n_clouds, offsets, plan);
  const size_t T = plan.tab.size();
  CU(ctx->pre_tables.reserve(T * sizeof(uint32_t)));
  // pageable host memory: staged before cudaMemcpyAsync returns
  CU(cudaMemcpyAsync(ctx->pre_tables.p, plan.tab.data(), T * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  CU(cudaMemcpyAsync(ctx->stage_pts.p, points, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  CU(ctx->pre_centres.reserve(n_clouds * 4 * sizeof(double)));
  CU(ctx->pre_pts.reserve(n * sizeof(float4)));
  CU(ctx->pre_lo.reserve(n * sizeof(float4)));
  CU(ctx->pre_leaf_pts.reserve(n * sizeof(float4)));
  CU(ctx->pre_perm.reserve(n * sizeof(uint32_t)));
  CU(ctx->pre_nodes.reserve(std::max<size_t>(plan.nodes, 1) * 64));
  CU(ctx->pre_boxes.reserve(static_cast<size_t>(plan.n_segments) * 6 * sizeof(uint32_t)));
  CU(ctx->keys_in.reserve(n * sizeof(uint64_t)));
  CU(ctx->keys_out.reserve(n * sizeof(uint64_t)));
  CU(ctx->vals_in.reserve(n * sizeof(uint32_t)));
  size_t sort_bytes = 0;
  if (plan.radix_levels) {
    CU(sort_pairs_u64_u32_bits(nullptr, sort_bytes, ctx->keys_in.as<uint64_t>(), ctx->keys_out.as<uint64_t>(), ctx->vals_in.as<uint32_t>(),
                               ctx->pre_perm.as<uint32_t>(), n, plan.key_bits, ctx->stream));
    CU(ctx->sort_temp.reserve(sort_bytes));
  }
  ctx->src_tree_valid = false;  // the scratch tree buffers are about to hold this forest
  ForestBuild b = {};
  b.tables = forest_tables(ctx->pre_tables.as<uint32_t>(), n_clouds);
  b.n = static_cast<uint32_t>(n);
  b.n_segments = plan.n_segments;
  b.n_slots = plan.n_slots;
  b.radix_levels = plan.radix_levels;
  b.max_depth = plan.max_depth;
  b.key_bits = plan.key_bits;
  b.sm_count = ctx->sm_count;
  b.points = ctx->stage_pts.as<double>();
  b.centres = ctx->pre_centres.as<double>();
  b.orig_pts = ctx->pre_pts.as<float4>();
  b.orig_lo = ctx->pre_lo.as<float4>();
  b.leaf_pts = ctx->pre_leaf_pts.as<float4>();
  b.perm = ctx->pre_perm.as<uint32_t>();
  b.pnodes = ctx->pre_nodes.as<float4>();
  b.boxes = ctx->pre_boxes.as<uint32_t>();
  b.keys_in = ctx->keys_in.as<uint64_t>();
  b.keys_out = ctx->keys_out.as<uint64_t>();
  b.vals_in = ctx->vals_in.as<uint32_t>();
  b.sort_temp = ctx->sort_temp.p;
  b.sort_temp_bytes = sort_bytes;
  int launches = 0;
  CU(launch_forest_build(b, ctx->stream, &launches));
  ctx->launches += launches;
  if (out_normals) CU(ctx->pre_out_normals.reserve(n * 4 * sizeof(double)));
  if (out_covs) CU(ctx->pre_out_covs.reserve(n * 16 * sizeof(double)));
  const int mode = (out_normals ? 1 : 0) | (out_covs ? 2 : 0);
  CU(launch_forest_features(ctx->pre_nodes.as<float4>(), ctx->pre_leaf_pts.as<float4>(), static_cast<uint32_t>(n), num_neighbors, b.tables,
                            ctx->pre_centres.as<double>(), mode, out_normals ? ctx->pre_out_normals.as<double>() : nullptr,
                            out_covs ? ctx->pre_out_covs.as<double>() : nullptr, static_cast<int>(plan.max_depth) + 1, ctx->pre_lo.as<float4>(), ctx->stream));
  ctx->launches += 1;
  if (out_normals) CU(cudaMemcpyAsync(out_normals, ctx->pre_out_normals.p, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (out_covs) CU(cudaMemcpyAsync(out_covs, ctx->pre_out_covs.p, n * 16 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

// The frame-stream hand-over (odometry_benchmark_small_gicp_tbb.cpp:41-43: `target_points = points; target_tree = tree;`): the cloud that was
// the source of this align() is the target of the next one.  Everything that already exists on the device is taken over, not rebuilt.
int sgb_target_adopt_source(sgb_ctx* ctx) {
  if (!ctx) return 1;
  if (ctx->tgt_state == TargetState::KdTrees)
    return fail(ctx, 1, "sgb_target_adopt_source: the target holds many kd-trees (sgb_target_build_kdtrees); set a single target first");
  if (ctx->src_state != SourceState::Single || ctx->n_src == 0) return fail(ctx, 1, "sgb_target_adopt_source: no source points (call sgb_source_set_points first)");
  CU(cudaSetDevice(ctx->device));
  const size_t n = ctx->n_src;
  const bool covs = ctx->src_has_covs;
  // covariances in ORIGINAL order: either still there from the device-side estimation, or un-permuted from the search-ordered streams
  if (covs && !ctx->src_cov_orig_valid) {
    CU(ctx->tmp_covA.reserve(n * sizeof(float4)));
    CU(ctx->tmp_covB.reserve(n * sizeof(float4)));
    CU(launch_scatter(ctx->src_perm.as<uint32_t>(), n, ctx->src_covA.as<float4>(), ctx->tmp_covA.as<float4>(), ctx->src_covB.as<float4>(), ctx->tmp_covB.as<float4>(),
                      nullptr, nullptr, ctx->sm_count, ctx->stream));
    ctx->launches += 1;
  }
  ctx->tgt_orig_pts.swap(ctx->tmp_pts);
  if (ctx->src_has_lo) ctx->tgt_orig_lo.swap(ctx->tmp_lo);
  if (covs) {
    ctx->tgt_orig_covA.swap(ctx->tmp_covA);
    ctx->tgt_orig_covB.swap(ctx->tmp_covB);
  }
  ctx->tgt_centre.swap(ctx->src_centre);
  ctx->tgt_bounds.swap(ctx->src_bounds);
  CU(ctx->src_centre.reserve(4 * sizeof(double)));
  CU(ctx->src_bounds.reserve(6 * sizeof(double)));
  const bool src_tree = ctx->src_tree_valid;
  int depth = ctx->src_tree_depth;
  if (int rc = begin_point_target(ctx, n, false, covs, ctx->src_has_lo)) return rc;
  // the context has no source until the next sgb_source_set_points (its buffers now belong to the target)
  begin_source(ctx, SourceState::None, 0, false);
  if (src_tree) {
    ctx->tgt_perm.swap(ctx->pre_perm);
    ctx->tgt_pts.swap(ctx->pre_leaf_pts);
    ctx->tgt_pnodes.swap(ctx->pre_nodes);
  } else if (int rc = build_lbvh(ctx, ctx->tgt_orig_pts.as<float4>(), n, ctx->tgt_centre.as<double>(), ctx->tgt_perm, ctx->tgt_pts, ctx->tgt_pnodes, &depth)) {
    return rc;
  }
  if (depth > 40) return fail(ctx, 1, "sgb_target_adopt_source: tree too deep");
  if (int rc = gather_target_features(ctx, false)) return rc;
  return install_tree(ctx, depth, (static_cast<size_t>(1) << (depth - 1)) - 1);
}

// Gaussian voxel map built on the device (SURVEY §8f row 3): replaces IncrementalVoxelMap<GaussianVoxel>::insert
// (incremental_voxelmap.hpp:55-92) + GaussianVoxel::add / finalize (gaussian_voxelmap.hpp:30-62) for a one-shot map.
int sgb_target_build_voxelmap(sgb_ctx* ctx, size_t n, const double* points, const double* covs, double leaf_size, int search_offsets) {
  if (!ctx) return 1;
  if (!(leaf_size > 0.0)) return fail(ctx, 1, "sgb_target_build_voxelmap: leaf_size must be positive");
  if (n && !points) return fail(ctx, 1, "sgb_target_build_voxelmap: null points");
  if (n >= (1ull << 31)) return fail(ctx, 1, "sgb_target_build_voxelmap: too many points");
  if (search_offsets != 1 && search_offsets != 7 && search_offsets != 27) search_offsets = 1;  // incremental_voxelmap.hpp:159-163
  CU(cudaSetDevice(ctx->device));
  if (int rc = begin_voxel_target(ctx, 0, covs != nullptr, leaf_size, search_offsets)) return rc;  // n_tgt = the voxel count once known
  if (n == 0) return 0;
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  CU(cudaMemcpyAsync(ctx->stage_pts.p, points, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (covs) {
    CU(ctx->stage_covs.reserve(n * 16 * sizeof(double)));
    CU(cudaMemcpyAsync(ctx->stage_covs.p, covs, n * 16 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  }
  if (int rc = sort_into_voxels(ctx, n, 1.0 / leaf_size)) return rc;
  uint32_t n_vox = 0;
  CU(cudaMemcpyAsync(&n_vox, ctx->pre_slots.as<uint32_t>() + n, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (n_vox == 0) return 0;  // every point outside the 21-bit voxel range
  // per-voxel mean / covariance / integer coordinates (FP64), then the same device-side conversion as sgb_target_set_voxelmap
  CU(ctx->pre_out_normals.reserve(static_cast<size_t>(n_vox) * 4 * sizeof(double)));
  if (covs) CU(ctx->pre_out_covs.reserve(static_cast<size_t>(n_vox) * 16 * sizeof(double)));
  CU(ctx->pre_vox_coords.reserve(static_cast<size_t>(n_vox) * sizeof(int4)));
  CU(launch_voxel_stats(ctx->keys_out.as<uint64_t>(), ctx->pre_vals_out.as<uint32_t>(), ctx->pre_heads.as<uint32_t>(), ctx->pre_slots.as<uint32_t>(), n,
                        ctx->stage_pts.as<double>(), covs ? ctx->stage_covs.as<double>() : nullptr, ctx->pre_out_normals.as<double>(),
                        covs ? ctx->pre_out_covs.as<double>() : nullptr, ctx->pre_vox_coords.as<int4>(), ctx->sm_count, ctx->stream));
  CU(ctx->tgt_pts.reserve(static_cast<size_t>(n_vox) * sizeof(float4)));
  if (covs) {
    CU(ctx->tgt_covA.reserve(static_cast<size_t>(n_vox) * sizeof(float4)));
    CU(ctx->tgt_covB.reserve(static_cast<size_t>(n_vox) * sizeof(float4)));
  }
  CU(launch_bounds_centre(ctx->pre_out_normals.as<double>(), n_vox, ctx->tgt_bounds.as<double>(), ctx->tgt_centre.as<double>(), ctx->sm_count, ctx->stream));
  CU(launch_convert(ctx->pre_out_normals.as<double>(), nullptr, covs ? ctx->pre_out_covs.as<double>() : nullptr, n_vox, ctx->tgt_centre.as<double>(),
                    ctx->tgt_pts.as<float4>(), nullptr, ctx->tgt_covA.as<float4>(), ctx->tgt_covB.as<float4>(), nullptr, nullptr, ctx->sm_count, ctx->stream));
  uint32_t capacity = 16;
  while (capacity < 2ull * n_vox) capacity <<= 1;  // load factor <= 1/2
  CU(ctx->vox_table.reserve(static_cast<size_t>(capacity) * sizeof(int4)));
  CU(launch_vox_table_build(ctx->pre_vox_coords.as<int4>(), n_vox, ctx->vox_table.as<int4>(), capacity, ctx->stream));
  ctx->launches += 7;
  ctx->vox_mask = capacity - 1;
  ctx->n_tgt = n_vox;
  return 0;
}

// Many Gaussian voxel maps as one target of the batched calls, built in a fixed number of launches and one host synchronisation whatever
// the map count (sgb_preprocess.cu: voxelmaps_*).  Map m is stored as sgb_target_build_voxelmap stores it alone: its voxels in ascending key
// order (global ids first .. first + count), sums in ascending original index, FP32 about the centre of its own voxel means, and its own
// table region with the single map's capacity rule and hash.
int sgb_target_build_voxelmaps(sgb_ctx* ctx, size_t n_maps, const size_t* offsets, const double* points, const double* covs, double leaf_size,
                               int search_offsets) {
  if (!ctx) return 1;
  const std::string who = "sgb_target_build_voxelmaps: ";
  if (int rc = check_offsets(ctx, who, n_maps, offsets, "map")) return rc;
  const size_t n = offsets[n_maps];
  if (n >= (1ull << 31)) return fail(ctx, 1, who + "too many points");
  if (n && !points) return fail(ctx, 1, who + "null points");
  if (!(leaf_size > 0.0)) return fail(ctx, 1, who + "leaf_size must be positive");
  if (search_offsets != 1 && search_offsets != 7 && search_offsets != 27) return fail(ctx, 1, who + "search_offsets must be 1, 7 or 27");
  CU(cudaSetDevice(ctx->device));
  if (int rc = begin_voxel_target(ctx, 0, covs != nullptr, leaf_size, search_offsets, true, n_maps)) return rc;  // n_tgt = the voxel count once known
  const size_t M = std::max<size_t>(n_maps, 1);
  CU(ctx->vm_centres.reserve(M * 4 * sizeof(double)));
  CU(ctx->vm_regions.reserve(M * sizeof(uint4)));
  if (n == 0) return 0;
  const uint32_t maps = static_cast<uint32_t>(n_maps);
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  CU(cudaMemcpyAsync(ctx->stage_pts.p, points, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (covs) {
    CU(ctx->stage_covs.reserve(n * 16 * sizeof(double)));
    CU(cudaMemcpyAsync(ctx->stage_covs.p, covs, n * 16 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  }
  size_t cap_scan_bytes = 0;
  if (int rc = sort_into_voxelmaps(ctx, n_maps, offsets, 1.0 / leaf_size, ctx->vm_regions.as<uint4>(), cap_scan_bytes)) return rc;
  uint64_t* keys = ctx->keys_in.as<uint64_t>();
  uint32_t* vals = ctx->vals_in.as<uint32_t>();
  uint32_t* caps = ctx->vm_caps.as<uint32_t>();
  uint32_t* cap_scan = caps + n_maps + 1;
  // the table's layout
  CU(exclusive_sum_u32(ctx->sort_temp.p, cap_scan_bytes, caps, cap_scan, n_maps + 1, ctx->stream));
  ctx->launches += 1;
  // the one synchronisation: voxel count and table size (into the page-locked result slot)
  uint32_t* h = reinterpret_cast<uint32_t*>(ctx->h_out + 56);
  CU(cudaMemcpyAsync(h, ctx->pre_slots.as<uint32_t>() + n, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(h + 1, cap_scan + n_maps, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const uint32_t n_vox = h[0], table_slots = h[1];
  if (n_vox == 0) return 0;  // every point outside the 21-bit voxel range
  // the capacities sum to at most 4 n_vox + 16 n_maps: below 2^32 (the scan's type) with this bound
  if (n_vox > (1u << 29)) return fail(ctx, 1, who + "too many voxels");
  CU(ctx->pre_out_normals.reserve(static_cast<size_t>(n_vox) * 4 * sizeof(double)));
  if (covs) CU(ctx->pre_out_covs.reserve(static_cast<size_t>(n_vox) * 16 * sizeof(double)));
  CU(ctx->pre_vox_coords.reserve(static_cast<size_t>(n_vox) * sizeof(int4)));
  CU(ctx->tgt_pts.reserve(static_cast<size_t>(n_vox) * sizeof(float4)));
  if (covs) {
    CU(ctx->tgt_covA.reserve(static_cast<size_t>(n_vox) * sizeof(float4)));
    CU(ctx->tgt_covB.reserve(static_cast<size_t>(n_vox) * sizeof(float4)));
  }
  CU(ctx->vox_table.reserve(static_cast<size_t>(table_slots) * sizeof(int4)));
  CU(launch_voxel_stats(keys, vals, ctx->pre_heads.as<uint32_t>(), ctx->pre_slots.as<uint32_t>(), n, ctx->stage_pts.as<double>(),
                        covs ? ctx->stage_covs.as<double>() : nullptr, ctx->pre_out_normals.as<double>(), covs ? ctx->pre_out_covs.as<double>() : nullptr,
                        ctx->pre_vox_coords.as<int4>(), ctx->sm_count, ctx->stream));
  CU(launch_voxelmaps_centres(ctx->pre_out_normals.as<double>(), maps, ctx->vm_regions.as<uint4>(), cap_scan, ctx->vm_centres.as<double>(), ctx->stream));
  CU(launch_voxelmaps_table(ctx->pre_out_normals.as<double>(), covs ? ctx->pre_out_covs.as<double>() : nullptr, ctx->pre_vox_coords.as<int4>(), n_vox,
                            ctx->vm_regions.as<uint4>(), maps, ctx->vm_centres.as<double>(), ctx->tgt_pts.as<float4>(), ctx->tgt_covA.as<float4>(),
                            ctx->tgt_covB.as<float4>(), ctx->vox_table.as<int4>(), table_slots, ctx->stream));
  ctx->launches += 4;
  ctx->n_tgt = n_vox;
  return 0;
}

// Many point clouds with their kd-trees as one target of the batched calls (sgb_forest.cu).  Every size follows from the host offsets,
// so the build is launched without a host synchronisation, in a number of launches set by the largest map alone.  Map m is stored as
// sgb_target_set_points + sgb_target_build_kdtree store it alone: centred FP32 on its own box centre, w = index within the map, leaves
// of at most kLbvhLeafPoints points cut by median splits along the widest axis of every node.
int sgb_target_build_kdtrees(sgb_ctx* ctx, size_t n_maps, const size_t* offsets, const double* points, const double* normals, const double* covs) {
  if (!ctx) return 1;
  const std::string who = "sgb_target_build_kdtrees: ";
  if (int rc = check_offsets(ctx, who, n_maps, offsets, "map")) return rc;
  const size_t n = offsets[n_maps];
  if (n >= (1ull << 30)) return fail(ctx, 1, who + "too many points (fewer than 2^30 in all)");
  if (n && !points) return fail(ctx, 1, who + "null points");
  CU(cudaSetDevice(ctx->device));
  if (int rc = begin_forest_target(ctx, n, normals != nullptr, covs != nullptr, n_maps)) return rc;
  const size_t M = std::max<size_t>(n_maps, 1);
  CU(ctx->kt_centres.reserve(M * 4 * sizeof(double)));
  ctx->kt_depth = 1;
  if (n == 0) return 0;
  ForestPlan plan;
  plan_forest(n_maps, offsets, plan);
  const uint32_t max_depth = plan.max_depth, radix_levels = plan.radix_levels, n_segments = plan.n_segments, n_slots = plan.n_slots;
  const size_t nodes = plan.nodes;
  const int key_bits = plan.key_bits;
  if (max_depth + 1 > 40) return fail(ctx, 1, who + "tree too deep");
  const size_t T = plan.tab.size();
  CU(ctx->kt_tables.reserve(T * sizeof(uint32_t)));
  // pageable host memory: staged before cudaMemcpyAsync returns
  CU(cudaMemcpyAsync(ctx->kt_tables.p, plan.tab.data(), T * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  CU(cudaMemcpyAsync(ctx->stage_pts.p, points, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (normals) {
    CU(ctx->stage_normals.reserve(n * 4 * sizeof(double)));
    CU(cudaMemcpyAsync(ctx->stage_normals.p, normals, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
    CU(ctx->tgt_orig_normals.reserve(n * sizeof(float4)));
    CU(ctx->tgt_normals.reserve(n * sizeof(float4)));
  }
  if (covs) {
    CU(ctx->stage_covs.reserve(n * 16 * sizeof(double)));
    CU(cudaMemcpyAsync(ctx->stage_covs.p, covs, n * 16 * sizeof(double), cudaMemcpyDefault, ctx->stream));
    CU(ctx->tgt_orig_covA.reserve(n * sizeof(float4)));
    CU(ctx->tgt_orig_covB.reserve(n * sizeof(float4)));
    CU(ctx->tgt_covA.reserve(n * sizeof(float4)));
    CU(ctx->tgt_covB.reserve(n * sizeof(float4)));
  }
  CU(ctx->tgt_orig_pts.reserve(n * sizeof(float4)));
  CU(ctx->tgt_pts.reserve(n * sizeof(float4)));
  CU(ctx->tgt_perm.reserve(n * sizeof(uint32_t)));
  CU(ctx->tgt_pnodes.reserve(std::max<size_t>(nodes, 1) * 64));
  CU(ctx->pre_boxes.reserve(static_cast<size_t>(n_segments) * 6 * sizeof(uint32_t)));
  CU(ctx->keys_in.reserve(n * sizeof(uint64_t)));
  CU(ctx->keys_out.reserve(n * sizeof(uint64_t)));
  CU(ctx->vals_in.reserve(n * sizeof(uint32_t)));
  size_t sort_bytes = 0;
  if (radix_levels) {
    CU(sort_pairs_u64_u32_bits(nullptr, sort_bytes, ctx->keys_in.as<uint64_t>(), ctx->keys_out.as<uint64_t>(), ctx->vals_in.as<uint32_t>(),
                               ctx->tgt_perm.as<uint32_t>(), n, key_bits, ctx->stream));
    CU(ctx->sort_temp.reserve(sort_bytes));
  }
  ForestBuild b = {};
  b.tables = forest_tables(ctx->kt_tables.as<uint32_t>(), n_maps);
  b.n = static_cast<uint32_t>(n);
  b.n_segments = n_segments;
  b.n_slots = n_slots;
  b.radix_levels = radix_levels;
  b.max_depth = max_depth;
  b.key_bits = key_bits;
  b.sm_count = ctx->sm_count;
  b.points = ctx->stage_pts.as<double>();
  b.normals = normals ? ctx->stage_normals.as<double>() : nullptr;
  b.covs = covs ? ctx->stage_covs.as<double>() : nullptr;
  b.centres = ctx->kt_centres.as<double>();
  b.orig_pts = ctx->tgt_orig_pts.as<float4>();
  b.orig_normals = normals ? ctx->tgt_orig_normals.as<float4>() : nullptr;
  b.orig_covA = covs ? ctx->tgt_orig_covA.as<float4>() : nullptr;
  b.orig_covB = covs ? ctx->tgt_orig_covB.as<float4>() : nullptr;
  b.leaf_pts = ctx->tgt_pts.as<float4>();
  b.leaf_normals = ctx->tgt_normals.as<float4>();
  b.leaf_covA = ctx->tgt_covA.as<float4>();
  b.leaf_covB = ctx->tgt_covB.as<float4>();
  b.perm = ctx->tgt_perm.as<uint32_t>();
  b.pnodes = ctx->tgt_pnodes.as<float4>();
  b.boxes = ctx->pre_boxes.as<uint32_t>();
  b.keys_in = ctx->keys_in.as<uint64_t>();
  b.keys_out = ctx->keys_out.as<uint64_t>();
  b.vals_in = ctx->vals_in.as<uint32_t>();
  b.sort_temp = ctx->sort_temp.p;
  b.sort_temp_bytes = sort_bytes;
  int launches = 0;
  CU(launch_forest_build(b, ctx->stream, &launches));
  ctx->launches += launches;
  ctx->kt_depth = static_cast<int>(max_depth) + 1;
  ctx->n_pnodes = nodes;
  return 0;
}

// k nearest neighbours of arbitrary queries in the target's search structure (SURVEY §8f row 4: the batch NN API)
int sgb_target_batch_knn(sgb_ctx* ctx, size_t n_queries, const double* queries, int k, uint64_t* out_indices, double* out_sq_dists) {
  if (!ctx) return 1;
  if (k < 1 || k > 32) return fail(ctx, 1, "sgb_target_batch_knn: k must be in 1..32");
  if (n_queries && (!queries || !out_indices || !out_sq_dists)) return fail(ctx, 1, "sgb_target_batch_knn: null buffer");
  if (n_queries >= (1ull << 31) / static_cast<size_t>(k)) return fail(ctx, 1, "sgb_target_batch_knn: too many queries");
  if (ctx->tgt_state != TargetState::Tree) return fail(ctx, 1, "sgb_target_batch_knn: needs a point target with its kd-tree (set points, then set/build the tree)");
  if (n_queries == 0) return 0;
  CU(cudaSetDevice(ctx->device));
  const size_t n = n_queries, nk = n * static_cast<size_t>(k);
  if (ctx->n_tgt == 0) {  // nothing to find: KnnResult's initial state
    for (size_t j = 0; j < nk; j++) {
      out_indices[j] = ~0ull;
      out_sq_dists[j] = std::numeric_limits<double>::max();
    }
    return 0;
  }
  CU(ctx->stage_pts.reserve(n * 4 * sizeof(double)));
  CU(cudaMemcpyAsync(ctx->stage_pts.p, queries, n * 4 * sizeof(double), cudaMemcpyDefault, ctx->stream));
  CU(ctx->pre_out_covs.reserve(nk * sizeof(double)));
  CU(ctx->corr64.reserve(nk * sizeof(uint64_t)));
  CU(launch_batch_knn(ctx->tgt_pnodes.as<float4>(), ctx->tgt_pts.as<float4>(), ctx->stage_pts.as<double>(), static_cast<uint32_t>(n), k, ctx->tgt_centre.as<double>(),
                      ctx->corr64.as<unsigned long long>(), ctx->pre_out_covs.as<double>(), ctx->tree_depth, ctx->stream));
  ctx->launches += 1;
  CU(cudaMemcpyAsync(out_indices, ctx->corr64.p, nk * sizeof(uint64_t), cudaMemcpyDefault, ctx->stream));
  CU(cudaMemcpyAsync(out_sq_dists, ctx->pre_out_covs.p, nk * sizeof(double), cudaMemcpyDefault, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

}  // extern "C"
