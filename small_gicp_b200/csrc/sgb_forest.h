// SPDX-License-Identifier: MIT
// Many kd-trees as one target of the batched calls: device tables, build and search launchers (sgb_forest.cu; C-ABI
// sgb_target_build_kdtrees in sgb_capi_preprocess.cu, batched rounds in sgb_capi_batch.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sgb_batch.h"

namespace sgb {

/// Per-map tables on the device, all derived on the host from the map offsets.  Prefix arrays have n_maps + 1 entries.
struct ForestTables {
  const uint32_t* pt_off;     // first point of map m (points concatenated in map order)
  const uint32_t* slot_off;   // first leaf slot of map m (P_m = 2^depth slots, 0 for an empty map)
  const uint32_t* seg_off;    // first shared-memory segment of map m (2^level0 segments, 0 for an empty map)
  const uint32_t* node_base;  // [n_maps] first packet record of map m in the record array (P_m - 1 records)
  const uint32_t* depth;      // [n_maps] inner levels of map m's tree (0: empty map)
  const uint32_t* level0;     // [n_maps] first level whose nodes hold at most kKdSegMax points
  uint32_t n_maps;
};

/// What the search reads: the record blocks, each map's centre [4] and the tables above.
struct ForestView {
  const float4* pnodes;
  const double* centres;
  const uint32_t* pt_off;
  const uint32_t* node_base;
};

/// One build (device pointers; orig_* in original order, leaf_* in leaf order).
struct ForestBuild {
  ForestTables tables;
  uint32_t n, n_segments, n_slots, radix_levels, max_depth;
  int key_bits, sm_count;
  const double* points;   // n x 4
  const double* normals;  // n x 4 or null
  const double* covs;     // n x 16 or null
  double* centres;        // [n_maps][4]
  float4 *orig_pts, *orig_normals, *orig_covA, *orig_covB;
  float4 *leaf_pts, *leaf_normals, *leaf_covA, *leaf_covB;
  float4* orig_lo;        // null, or what the FP32 rounding of orig_pts dropped (convert_kernel's out_lo): feature estimation only
  uint32_t* perm;         // leaf position -> global original position
  float4* pnodes;
  uint32_t* boxes;        // n_segments x 6
  uint64_t *keys_in, *keys_out;
  uint32_t* vals_in;
  void* sort_temp;
  size_t sort_temp_bytes;
};

/// Launches the whole build on st (no host synchronisation); *launches = launches made (memory copies and radix sorts count one each).
cudaError_t launch_forest_build(const ForestBuild& b, cudaStream_t st, int* launches);
/// Exact nearest neighbour of every point of the call's tiles in its member's map; vcorr[vfirst + k] = global leaf position or kNone.
/// max_depth: stack entries per lane (inner levels of the deepest tree + 1, at most 40); bound: the FP32 search bound (search_bound).
/// round null: n_tiles tiles; else a round of sgb_align_batch_async: n_tiles CTAs, of which the first round->n_tiles search (none in an
/// error() round).
cudaError_t launch_forest_search(const BatchParams& B, const ForestView& F, const BatchRound* round, uint32_t n_tiles, int max_depth, float bound, uint32_t* vcorr,
                                 cudaStream_t st);
/// The same for submap members: the exact nearest neighbour of every point over ALL entries of its member's list, each entry's tree
/// walked in its own stored frame with the bound the earlier entries left; vcorr as above, S.centry[stored position] = the entry.
cudaError_t launch_submap_search(const BatchParams& B, const float4* pnodes, const SubmapView& S, const BatchRound* round, uint32_t n_tiles, int max_depth,
                                 float bound, uint32_t* vcorr, cudaStream_t st);
/// Normals (mode bit 0) / covariances (bit 1) of every point of a built forest from its k nearest neighbours in its own map, as
/// launch_features computes them for one cloud (sgb_preprocess.cu): one thread per leaf-ordered point, outputs in the double layout at
/// the point's global original position.  lo: the build's orig_lo, or null.  depth: stack entries (inner levels of the deepest tree + 1).
cudaError_t launch_forest_features(const float4* pnodes, const float4* leaf_pts, uint32_t n, int k, const ForestTables& F, const double* centres, int mode,
                                   double* out_normals_d, double* out_covs_d, int depth, const float4* lo, cudaStream_t st);

}  // namespace sgb
