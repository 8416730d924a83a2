// SPDX-License-Identifier: MIT
// Host-visible launchers of the kernels in sgb_kernels.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdlib>
#include <type_traits>

#include "sgb_device.cuh"

namespace sgb {

/// Launch `kernel` as a programmatic dependent of the previous kernel on `st` (its set-up overlaps the predecessor's tail;
/// the kernel itself waits with grid_dependency_wait()).  Profiling build: SGB_PDL=0 falls back to plain stream order (A/B switch).
inline bool pdl_enabled() {
#ifdef SGB_PROFILING
  static const bool on = !(std::getenv("SGB_PDL") && std::getenv("SGB_PDL")[0] == '0');
  return on;
#else
  return true;
#endif
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_dependent(void (*kernel)(KArgs...), int grid, int block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(grid));
  cfg.blockDim = dim3(static_cast<unsigned>(block));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

/// The factor x robust kernel pair as compile-time constants: returns fn(std::integral_constant<int, FACTOR>{},
/// std::integral_constant<int, ROBUST>{}) for factor, robust in 0..2, or `invalid` when factor * 3 + robust is outside 0..8.
template <typename Ret, typename Fn>
inline Ret dispatch_factor_robust(int factor, int robust, Ret invalid, Fn&& fn) {
  using F0 = std::integral_constant<int, 0>;
  using F1 = std::integral_constant<int, 1>;
  using F2 = std::integral_constant<int, 2>;
  switch (factor * 3 + robust) {
    case 0: return fn(F0{}, F0{});
    case 1: return fn(F0{}, F1{});
    case 2: return fn(F0{}, F2{});
    case 3: return fn(F1{}, F0{});
    case 4: return fn(F1{}, F1{});
    case 5: return fn(F1{}, F2{});
    case 6: return fn(F2{}, F0{});
    case 7: return fn(F2{}, F1{});
    case 8: return fn(F2{}, F2{});
    default: return invalid;
  }
}

/// Lets `kernel` launch on the current device with `bytes` of dynamic shared memory: the one place that sets its opt-in limit.  The limit is
/// per (device, kernel) and shared by every context of the process, so it is only ever raised, never lowered, under one mutex; a launch at or
/// below the size it allowed stays valid whatever other threads allow meanwhile.  Nothing to do up to 48 KiB.
cudaError_t allow_dynamic_smem(const void* kernel, size_t bytes);
template <typename... KArgs>
inline cudaError_t allow_dynamic_smem(void (*kernel)(KArgs...), size_t bytes) {
  return allow_dynamic_smem(reinterpret_cast<const void*>(kernel), bytes);
}
/// Resident CTAs per SM (at least 1) of `kernel` launched with `block` threads and `smem` bytes of dynamic shared memory, asked once per
/// device, kernel, block and smem.  Before the query: max_shared_carveout prefers the largest shared-memory carveout, smem_limit raises the
/// kernel's dynamic shared-memory limit to at least `smem` through allow_dynamic_smem.
int ctas_per_sm(const void* kernel, int block, size_t smem, bool max_shared_carveout, bool smem_limit);
template <typename... KArgs>
inline int ctas_per_sm(void (*kernel)(KArgs...), int block, size_t smem, bool max_shared_carveout, bool smem_limit) {
  return ctas_per_sm(reinterpret_cast<const void*>(kernel), block, smem, max_shared_carveout, smem_limit);
}
/// CTAs of kLinBlock threads for `threads` threads, at most one wave of `ctas_per_sm` CTAs on each of `sm_count` SMs
inline int one_wave_grid(size_t threads, int sm_count, int ctas_per_sm) {
  const size_t grid = (threads + kLinBlock - 1) / kLinBlock, cap = static_cast<size_t>(sm_count) * ctas_per_sm;
  return static_cast<int>(grid < cap ? grid : cap);
}

cudaError_t launch_linearize(const LinParams& P, int factor, int robust, bool voxel, int grid, int stack_depth, cudaStream_t st);
cudaError_t launch_error(const LinParams& P, int factor, int robust, int grid, cudaStream_t st);
cudaError_t launch_reduce_nothing(const LinParams& P, bool linearize, cudaStream_t st);
int linearize_occupancy(int stack_depth);
cudaError_t set_source_curve(int hilbert);
// sgb_kernels_split.cu
int search_occupancy(int stack_depth);
cudaError_t launch_search(const LinParams& P, int grid, int stack_depth, cudaStream_t st);
cudaError_t launch_factor_reduce(const LinParams& P, int factor, int robust, int grid, cudaStream_t st);
int factor_reduce_occupancy(int factor, int robust);
/// Reduction::error through the factor kernel's operand pipeline (one wave of CTAs looping over tiles)
cudaError_t launch_error_pipelined(const LinParams& P, int factor, int robust, int grid, cudaStream_t st);
int error_pipelined_occupancy(int factor, int robust);

cudaError_t launch_bounds_centre(const double* d_pts4, size_t n, double* d_bounds6, double* d_centre4, int sm_count, cudaStream_t st);
cudaError_t launch_convert(const double* d_pts4, const double* d_normals4, const double* d_covs16, size_t n, const double* d_centre4, float4* out_pts,
                           float4* out_normals, float4* out_covA, float4* out_covB, uint64_t* keys, uint32_t* vals, int sm_count, cudaStream_t st,
                           float4* out_lo = nullptr);
/// Many source clouds stored in one pass, each bit-identical to store_source of it alone (sgb_source_set_batch): cloud c = points
/// offsets[c] .. offsets[c+1] (device, uint32).  Per-cloud box and centre, FP32 conversion and curve keys, a stable key sort, a stable
/// sort by cloud (cloud_bits bits), then the points, search order -> index within the cloud, and covariances (covs or null) in
/// (cloud, key, index) order: the order of the per-cloud sorts.  6 launches (the two sorts count one each), whatever n_clouds is.
struct StoreClouds {
  uint32_t n, n_clouds;
  int cloud_bits, sm_count;
  const double* points;  // n x 4
  const double* covs;    // n x 16 or null
  const uint32_t* offsets;
  double *bounds, *centres;  // [n_clouds][6] / [n_clouds][4]
  float4* orig_pts;          // scratch: centred FP32 points in original order, w = index within the cloud
  uint64_t *keys_a, *keys_b;
  uint32_t *vals_a, *vals_b;
  void* sort_temp;
  size_t sort_temp_bytes;  // enough for both sorts of n pairs
  float4 *pts, *covA, *covB;
  uint32_t* perm;
};
cudaError_t launch_store_clouds(const StoreClouds& s, cudaStream_t st);
cudaError_t launch_inverse_perm(const uint32_t* perm, size_t n, uint32_t* rank, int sm_count, cudaStream_t st);
cudaError_t launch_convert_cov_scatter(const double* d_covs16, size_t first, size_t n, const uint32_t* rank, float4* outA, float4* outB, float4* origA,
                                       float4* origB, int sm_count, cudaStream_t st);
cudaError_t launch_gather(const uint32_t* perm, size_t n, const float4* in0, float4* out0, const float4* in1, float4* out1, const float4* in2, float4* out2,
                          const float4* in3, float4* out3, int sm_count, cudaStream_t st);
cudaError_t launch_scatter(const uint32_t* perm, size_t n, const float4* in0, float4* out0, const float4* in1, float4* out1, const float4* in2, float4* out2,
                           int sm_count, cudaStream_t st);
cudaError_t launch_correspondences(const uint32_t* corr, const uint32_t* perm, size_t n, const float4* tgt_pts, int voxel, uint64_t* out, int sm_count,
                                   cudaStream_t st);
cudaError_t launch_chunk_transpose(const uint32_t* in, uint32_t* out, size_t n, uint32_t K, int sm_count, cudaStream_t st);

/// Work lists of the packet search, filled by the probe (one warp of the probe = one 32-query chunk): chunk ids by cost class
/// (0 = widest search ball ... kChunkClasses - 1 = narrowest), so that the packet search can take the expensive walks first.
constexpr uint32_t kChunkClasses = 3;
struct ChunkClasses {
  uint32_t* count;       // [kChunkClasses] entries of each list (zero on entry: the previous probe cleared them)
  uint32_t* count_next;  // [kChunkClasses] the counters of the NEXT linearize (this probe clears them)
  uint32_t* lists;       // [kChunkClasses][n_chunks] chunk ids, or null: no lists (the packet search scans the settled flags itself)
  uint32_t n_chunks;
  float wide_r2, mid_r2;  // class boundaries on the squared search radius
  uint32_t fallback_pct;  // more than this share of all chunks listed (i.e. with pending lanes): the packet search ignores the lists (curve order)
};
// sgb_kernels_packet.cu
int packet_occupancy(int max_depth);
// sgb_grid.cu: uniform-grid front end of the search
struct GridParams {
  float origin[3];  // minimum corner of the target's box (centred frame)
  float inv_cell;   // 1 / cell edge
  float settle_d2;  // a candidate within this squared distance is provably the nearest neighbour ((cell/2 - margin)^2)
};
/// One slot of the block table = one 32-byte sector: the 2 x 2 x 2 block anchored at cell (x, y, z) is, in the raster-ordered copy
/// of the target, four contiguous runs -- run r = cells (x, y + (r & 1), z + (r >> 1)) and (x + 1, same y, same z).
struct __align__(32) GridSlot {
  unsigned long long key;  // packed anchor coordinates (grid_key), ~0 = empty
  uint32_t start[4];       // first point of each run (cell-ordered copy)
  uint16_t count[4];       // points of each run (a kept block holds at most kGridMaxList)
};
/// What the warp-per-query search of few pending queries needs (it runs inside packet_search_kernel; see sgb_grid.cuh)
struct PendingParams {
  const uint32_t* list;    // pending list (source positions)
  const float4* q;         // parallel: transformed query + squared distance of the probe's best candidate
  const float4* grid_pts;  // target points in cell (raster) order: (x, y, z, leaf position)
  const GridSlot* table;   // block table, or null: no ring phase
  uint32_t capacity;
  GridParams g;
};
/// queue / queue_next: two alternating zero-initialised counters of the dynamic chunk queue (this launch clears queue_next), or null = static stride.
/// pending_count <= P.src.n / pending_div: the launch finishes the pending queries warp-per-query (ring phase / tree walk); more: the packet walk.
/// n_queries non-null: a round of sgb_align_batch_async, *n_queries of the P.src.n queries (read on the device) in place of P.src.n.
cudaError_t launch_packet_search(const LinParams& P, const uint32_t* n_queries, const float4* pnodes, int grid, int max_depth, const uint8_t* settled,
                                 const uint32_t* pending_count, uint32_t pending_div, uint32_t* queue, uint32_t* queue_next, const ChunkClasses& cc,
                                 const PendingParams& pp, bool tma_leaf, cudaStream_t st);
cudaError_t launch_grid_spacing(const float4* pnodes, uint32_t n_inner, float* out, cudaStream_t st);
/// Cell-ordered points + block table (sgb_grid.cu), sorted by compact raster keys of 3 `bits` bits.  build: cell keys of the n
/// leaf-ordered points, radix sort, the points in cell order into grid_pts (n float4), cell sizes into cnt (n), the eight block anchors
/// of every cell (8 n entries, padded), radix sort; then d_counters[0] = distinct anchors, [1] = largest block (points).  keys_a / b and
/// vals_a / b hold 8 n entries; the sorted anchors end in keys_b / vals_b.  fill: table of `capacity` slots from the sorted anchors.
cudaError_t launch_grid_build(const float4* leaf_pts, uint32_t n, const GridParams& g, int bits, uint64_t* keys_a, uint64_t* keys_b, uint32_t* vals_a, uint32_t* vals_b,
                              void* sort_temp, size_t sort_temp_bytes, float4* grid_pts, uint32_t* cnt, uint32_t* d_counters, cudaStream_t st);
cudaError_t launch_grid_fill(const uint64_t* akeys, const uint32_t* avals, uint32_t m, const uint32_t* cnt, int bits, GridSlot* table, uint32_t capacity,
                             cudaStream_t st);
/// largest block (points, the sum of its four runs) the grid front end accepts: beyond it a single query's scan would dominate (a cluster of near-duplicate
/// points, or a few far outliers stretching the box so that the cell-count bound inflates the cell) and the exact tree search alone is used
constexpr uint32_t kGridMaxList = 2048;
/// n_queries non-null: a round of sgb_align_batch_async, a grid for P.src.n queries of which the first *n_queries (read on the device) are probed.
cudaError_t launch_grid_probe(const LinParams& P, const uint32_t* n_queries, const float4* grid_pts, const GridSlot* table, uint32_t capacity,
                              const GridParams& g, uint8_t* state, uint32_t* pending_count, uint32_t* pending_list, float4* pending_q, uint32_t* next_count,
                              const ChunkClasses& cc, cudaStream_t st);
/// what the 27-block ring is guaranteed to cover: squared radius ((2.5 - slack) cells)^2
inline float ring_cover_sq(float cell) {
  const float c = (2.5f - 4e-3f) * cell;
  return c * c;
}
// device-side tree construction (sgb_kernels.cu)
constexpr uint32_t kLbvhLeafPoints = 32;
cudaError_t launch_curve_keys(const float4* pts, size_t n, const double* centre4, uint64_t* keys, uint32_t* vals, int sm_count, cudaStream_t st);
cudaError_t launch_lbvh_build(const float4* leaf_pts, uint32_t n, uint32_t P, float4* pnodes, int* launches, cudaStream_t st);
cudaError_t launch_kd_level_keys(const float4* cur_pts, uint32_t n, uint32_t count, uint32_t* boxes, uint64_t* keys, cudaStream_t st);
uint32_t kd_smem_first_level(uint32_t n, uint32_t levels);
cudaError_t launch_kd_refine_smem(float4* leaf_pts, uint32_t* perm, uint32_t n, uint32_t level0, uint32_t levels, cudaStream_t st);
cudaError_t sort_pairs_u64_u32_bits(void* d_temp, size_t& temp_bytes, const uint64_t* keys_in, uint64_t* keys_out, const uint32_t* vals_in, uint32_t* vals_out,
                                    size_t n, int end_bit, cudaStream_t st);
// sgb_preprocess.cu
cudaError_t launch_features(const float4* pnodes, const float4* pts, uint32_t n, int k, const double* centre, int mode, float4* out_normals, float4* out_covA,
                            float4* out_covB, double* out_normals_d, double* out_covs_d, int depth, int leaf_order_out, cudaStream_t st,
                            const float4* lo_orig = nullptr);
cudaError_t launch_batch_knn(const float4* pnodes, const float4* pts, const double* queries4, uint32_t n, int k, const double* centre, unsigned long long* out_idx,
                             double* out_d, int depth, cudaStream_t st);
/// Query sets against a kd-tree forest (sgb_target_batch_knn_maps on many kd-trees, sgb_target_batch_knn_submaps): query i belongs to
/// set s = owner of i in query_off [n_sets + 1], and is searched in the union of entries entry_off[s] .. entry_off[s + 1] - 1 (entry_off
/// null: set s has the one entry s); entry e = map entry_maps[e] placed by the pose whose inverse is inv_poses[12 e ..] (row-major R | t;
/// null: identity).  pt_off / node_base / centres: the forest's tables (ForestTables, kt_centres).
struct ForestKnn {
  const float4* pnodes;
  const float4* pts;
  const double4* queries;
  const uint32_t* query_off;
  uint32_t n_sets;
  const uint32_t* entry_off;
  const uint32_t* entry_maps;
  const double* inv_poses;
  const uint32_t* pt_off;
  const uint32_t* node_base;
  const double* centres;
};
cudaError_t launch_forest_knn(const ForestKnn& P, uint32_t n, int k, unsigned long long* out_idx, double* out_d, int depth, cudaStream_t st);
/// Query sets against Gaussian voxel maps (sgb_target_batch_knn_maps): query i of set s in map set_maps[s], whose table region, voxels
/// and centre are regions[m] = (first slot, mask, first voxel, count), pts (voxel means, centred FP32) and centres[4 m ..].
struct VoxelKnn {
  const double4* queries;
  const uint32_t* query_off;
  uint32_t n_sets;
  const uint32_t* set_maps;
  const uint4* regions;
  const int4* table;
  const float4* pts;
  const double* centres;
  int num_offsets;
  double inv_leaf;
};
cudaError_t launch_voxel_knn(const VoxelKnn& P, uint32_t n, int k, unsigned long long* out_idx, double* out_d, cudaStream_t st);
cudaError_t launch_voxel_keys(const double* d_pts4, size_t n, double inv_leaf, uint64_t* keys, uint32_t* vals, int sm_count, cudaStream_t st);
cudaError_t launch_voxel_means(const uint64_t* keys, const uint32_t* vals, const uint32_t* heads, const uint32_t* slots, size_t n, const double* d_pts4,
                               double* d_out4, int sm_count, cudaStream_t st);
cudaError_t launch_voxel_stats(const uint64_t* keys, const uint32_t* vals, const uint32_t* heads, const uint32_t* slots, size_t n, const double* d_pts4,
                               const double* d_covs16, double* out_means4, double* out_covs16, int4* out_coords, int sm_count, cudaStream_t st);
// many Gaussian voxel maps in one pass (sgb_target_build_voxelmaps; sgb_preprocess.cu has the order they are stored in)
/// after the key sort (keys / vals = voxel keys / original indices): map_keys = (map << 1 | valid), pos = position, for the second sort
cudaError_t launch_voxelmaps_sort_keys(const uint64_t* keys, const uint32_t* vals, size_t n, const uint32_t* offsets, uint32_t n_maps, uint64_t* map_keys,
                                       uint32_t* pos, int sm_count, cudaStream_t st);
/// after the (map, valid) sort: keys (bit 63 = rank_parity[map], the parity of the map's rank among the maps with points) and original
/// indices in (map, valid, key) order, heads[0, n] of the voxels
cudaError_t launch_voxelmaps_order(const uint64_t* map_keys, const uint32_t* pos, const uint64_t* keys, const uint32_t* vals, size_t n,
                                   const uint32_t* rank_parity, uint64_t* out_keys, uint32_t* out_vals, uint32_t* heads, int sm_count, cudaStream_t st);
/// correspondences of a member of a multi-map target in the caller's order: out[perm[i]] = (id within its map) << 32 (tgt_pts[k].w holds it)
cudaError_t launch_voxelmaps_correspondences(const uint32_t* corr, const uint32_t* perm, size_t n, const float4* tgt_pts, uint64_t* out, int sm_count,
                                             cudaStream_t st);
/// regions[m] = (0, table mask, first voxel, voxel count) of every map, caps[0, n_maps] = table capacities (then 0) for their scan
cudaError_t launch_voxelmaps_count(const uint32_t* offsets, uint32_t n_maps, const uint32_t* slots, uint4* regions, uint32_t* caps, cudaStream_t st);
/// centres[4 m ..] = centre of map m's voxel means (as launch_bounds_centre), regions[m].x = cap_scan[m]
cudaError_t launch_voxelmaps_centres(const double* means4, uint32_t n_maps, uint4* regions, const uint32_t* cap_scan, double* centres, cudaStream_t st);
/// FP32 voxels about their map's centre, and every map's region of the table (table_slots slots in all)
cudaError_t launch_voxelmaps_table(const double* means4, const double* covs16, const int4* coords, uint32_t n_voxels, const uint4* regions, uint32_t n_maps,
                                   const double* centres, float4* out_pts, float4* out_covA, float4* out_covB, int4* table, uint32_t table_slots,
                                   cudaStream_t st);
cudaError_t exclusive_sum_u32(void* d_temp, size_t& temp_bytes, const uint32_t* in, uint32_t* out, size_t n, cudaStream_t st);

}  // namespace sgb
