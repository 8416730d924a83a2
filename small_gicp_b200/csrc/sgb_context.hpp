// SPDX-License-Identifier: MIT
// The context behind the opaque sgb_ctx handle of include/sgicp_b200.h (shared by sgb_capi.cu / sgb_capi_preprocess.cu / sgb_capi_batch.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

namespace sgb {

/// Grow-only device buffer (re-used across calls so that streams of similarly sized frames never reallocate).
/// Owns its allocation: freed with the context (sgb_destroy makes the context's device current first).
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    const size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <typename T>
  T* as() const {
    return static_cast<T*>(p);
  }
  void swap(DevBuf& o) {
    void* tp = p;
    p = o.p;
    o.p = tp;
    const size_t tc = cap;
    cap = o.cap;
    o.cap = tc;
  }
};

/// The instantiated graph of a stream-ordered align's device loop and the key it was built under (launch_loop in sgb_capi_batch.cu):
/// an empty key matches no call, so the next one rebuilds the graph.  Owns the graph: destroyed with the context.
struct LoopGraph {
  cudaGraphExec_t exec = nullptr;
  std::vector<unsigned char> key;
  LoopGraph() = default;
  LoopGraph(const LoopGraph&) = delete;
  LoopGraph& operator=(const LoopGraph&) = delete;
  ~LoopGraph() { drop(); }
  void drop() {
    if (exec) cudaGraphExecDestroy(exec);
    exec = nullptr;
    key.clear();
  }
};

/// The device side of a joint window align (JointParams in sgb_batch.h): the window / edge tables, the frames' poses, candidates and
/// steps, the edges' last sums, the windows' WindowState and phase
struct JointBufs {
  DevBuf tables, X, cand, delta, sums, state, phase;
};

/// What the target is.  Points: tgt_orig_* hold n_tgt points in original order, no search structure yet.  Tree: the points are still
/// resident, and tgt_perm / tgt_pts / tgt_pnodes (+ the grid front end when grid_ready) are their search structure.  VoxelMap: tgt_pts /
/// tgt_cov* hold n_tgt voxels and vox_table indexes them; tgt_orig_* belong to no one.  VoxelMaps: vm_maps voxel maps for batched calls
/// only (member m against map m): their voxels concatenated in map order in tgt_pts / tgt_cov*, one region of vox_table per map.
/// KdTrees: kt_maps point clouds with their kd-trees, for batched calls only (member m against map m): points and features concatenated
/// in map order in leaf order in tgt_pts / tgt_normals / tgt_cov*, each map's packet records at its own base in tgt_pnodes.
enum class TargetState { None, Points, Tree, VoxelMap, VoxelMaps, KdTrees };
/// What the source is.  Single: one cloud of n_src points.  Batch: b_offsets.size() - 1 members concatenated (n_src = 0).
enum class SourceState { None, Single, Batch };

}  // namespace sgb

struct sgb_ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;
  // second stream + events of the pipelined source upload (sgb_source_set_points): the covariance chunks travel on it while the
  // context's stream converts / orders the points and the chunks that have already arrived
  cudaStream_t copy_stream = nullptr;
  static constexpr int kUploadChunks = 8;
  cudaEvent_t ev_upload[kUploadChunks] = {};
  cudaEvent_t ev_entry = nullptr;
  std::string err;
  uint64_t launches = 0;
  // The product library has ONE search path (grid front end + packet / pending search, then the factor kernel).  The fields below that
  // select anything else are only ever changed by the profiling build (-DSGB_PROFILING, libsgicp_b200_prof.so: A/B runs).
  int search_mode = 2;  // 2: packet (warp-cooperative) search + factor kernel; [profiling build] 1: per-thread search + factor kernel; 0: single fused kernel

  // ---- target ----
  // tgt_state and src_state are written by the transitions in sgb_capi.cu (begin_point_target, begin_voxel_target, install_tree,
  // begin_source, features_changed), which are also the only places that drop the last linearisation (have_lin, corr_seeds).
  // (A tree over an empty target only sets tgt_state = Tree: there is nothing to install and nothing is dropped.)
  sgb::TargetState tgt_state = sgb::TargetState::None;
  size_t n_tgt = 0;
  bool tgt_has_normals = false, tgt_has_covs = false;
  sgb::DevBuf tgt_orig_pts, tgt_orig_normals, tgt_orig_covA, tgt_orig_covB;  // original order (Points / Tree)
  sgb::DevBuf tgt_orig_lo, tmp_lo, pre_lo;  // what the FP32 rounding of the coordinates dropped (target / source / scratch cloud, original order): feature estimation only
  sgb::DevBuf tgt_pts, tgt_normals, tgt_covA, tgt_covB;                      // leaf order (or voxel order)
  sgb::DevBuf tgt_nodes, tgt_perm, tgt_pnodes;  // kd nodes (8 B, profiling build only), leaf permutation, packet records (64 B / inner node)
  int tree_depth = 0;
  bool host_tree = false;   // profiling switch: sgb_target_build_kdtree builds a median-split kd-tree on the host
  int tree_quality = 1;     // device construction: 1 = Hilbert order + per-level median-split refinement (kd quality), 0 = Hilbert order only (linear BVH)
  sgb::DevBuf pre_boxes;
  size_t n_pnodes = 0;      // packet records of the current target tree
  // uniform-grid front end of the search (sgb_grid.cu)
  bool use_grid = true, grid_ready = false;  // the front end holds the cell-ordered points + block table (one lookup per query)
  sgb::DevBuf grid_pts, grid_table, grid_state, grid_spacing, grid_pending;  // grid_pending: [0], [1] = alternating counters, [2..] = pending query positions
  sgb::DevBuf grid_pending_q;  // parallel to the list: transformed query + squared distance of the probe's best candidate
  bool use_ring = true, debug_pending = false;  // profiling switches (sgb_create)
  int pending_div = 16;           // more than n_src / pending_div pending queries: packet search, else a warp per pending query
  double grid_cell_factor = 2.5;  // cell edge in units of the median point spacing (2 / 2.5 / 3 / 4 were compared)
  uint32_t grid_capacity = 0;
  bool pending_clean = false;  // both pending counters are zero / maintained by the probe kernels
  int pending_parity = 0;
  sgb::DevBuf packet_queue;      // two alternating chunk-queue counters of the packet search (each launch clears the other)
  sgb::DevBuf chunk_lists;       // [2 parities][3] class counters, then [3][n_chunks] chunk ids: the packet search's work lists, filled by the probe
  bool chunk_lists_clean = false;
  uint32_t class_fallback_pct = 85;  // more than this share of the chunks listed (pending lanes almost everywhere): curve order instead of the lists
  float class_wide_cells = 2.0f;     // search radius (in cells) from which a chunk counts as wide
  bool kd_smem_refine = true;    // subtrees of <= 2048 points refined in shared memory by one launch (profiling switch SGB_KD_SMEM=0: one radix sort per level)
  bool error_pipelined = true;   // Reduction::error through the factor kernel's cp.async operand pipeline (profiling switch SGB_ERROR_PIPE=0: plain kernel)
  bool tma_leaf = false;         // profiling switch SGB_TMA_LEAF=1 (A/B of the north-star's TMA leaf staging)
  bool use_chunk_classes = true; // profiling switch SGB_CHUNK_CLASSES=0: the packet search scans all chunks in curve order
  int packet_parity = 0;
  bool use_packet_queue = true;  // profiling switch SGB_PACKET_QUEUE=0: static stride
  float grid_origin[3] = {0, 0, 0}, grid_inv_cell = 1.f, grid_settle_d2 = 0.f, grid_cell = 0.f;
  sgb::DevBuf tgt_centre, tgt_bounds;  // 4 / 6 doubles
  sgb::DevBuf vox_table;
  uint32_t vox_mask = 0;
  int vox_offsets = 1;
  double vox_inv_leaf = 1.0;
  // multi-map voxel target (VoxelMaps, sgb_target_build_voxelmaps): per map its centre [4] and (first table slot, mask, first voxel,
  // voxel count); voxel ids in tgt_* / corr are global, map m's are first .. first + count
  size_t vm_maps = 0;
  sgb::DevBuf vm_centres, vm_regions;
  sgb::DevBuf vm_offsets, vm_caps, vm_keys, vm_vals;  // build scratch: point offsets, table capacities / their scan, the second sort
  // many kd-trees (KdTrees, sgb_target_build_kdtrees, sgb_forest.h): per map its centre [4] and the uint32 tables of ForestTables
  // (pt_off, slot_off, seg_off: n_maps + 1 each; node_base, depth, level0: n_maps each); kt_depth = stack entries of the search
  size_t kt_maps = 0;
  int kt_depth = 1;
  sgb::DevBuf kt_centres, kt_tables;

  // ---- source ----
  sgb::SourceState src_state = sgb::SourceState::None;
  size_t n_src = 0;
  bool src_has_covs = false;
  sgb::DevBuf src_pts, src_covA, src_covB, src_perm, src_rank, src_centre, src_bounds;  // search order (src_perm: search order -> original index)
  uint32_t src_run = 1;  // K of the chunk-transposed source layout (DevSource::run)
  // Buffers of the single source that outlive a call, read by sgb_source_estimate_features and taken over by sgb_target_adopt_source.
  // begin_source clears their flags; only sgb_estimate_features also writes one of them (its scratch tree goes to pre_*).
  sgb::DevBuf tmp_pts;  // the source in original order (centred FP32, w = index)
  bool tgt_has_lo = false, src_has_lo = false;  // tgt_orig_lo / tmp_lo hold the residuals of the current target / single source
  bool src_tree_valid = false;  // pre_perm / pre_leaf_pts / pre_nodes hold the source's tree (sgb_source_estimate_features built it), depth src_tree_depth
  sgb::DevBuf tmp_covA, tmp_covB;
  bool src_cov_orig_valid = false;  // tmp_covA / tmp_covB hold the source's covariances in original order (estimated on the device)
  int src_tree_depth = 0;

  // ---- scratch: contents do not outlive the call that writes them ----
  // raw double uploads, and the host poses and outputs of sgb_align_batch_gnc / sgb_align_joint_gnc staged in device memory (stage_pts)
  sgb::DevBuf stage_pts, stage_normals, stage_covs;
  sgb::DevBuf keys_in, keys_out, vals_in, sort_temp;
  sgb::DevBuf corr, partials, ticket, corr64;
  sgb::DevBuf knn_tables;  // the set / entry tables of sgb_target_batch_knn_maps / _submaps
  double* h_out = nullptr;      // page-locked AND mapped, 64 doubles: [0,44) H|b|e|inliers, [48] error(), [56] scratch, [60] comm status
  double* h_out_dev = nullptr;  // device address of the same memory (the reduction's finishing CTA writes into it)

  // ---- preprocessing scratch (sgb_capi_preprocess.cu) ----
  sgb::DevBuf pre_pts, pre_leaf_pts, pre_nodes, pre_perm, pre_centre, pre_bounds, pre_out_normals, pre_out_covs, pre_heads, pre_slots, pre_vals_out;
  sgb::DevBuf pre_vox_coords;  // integer voxel coordinates of sgb_target_build_voxelmap
  // many clouds (sgb_voxelgrid_sampling_batch / sgb_estimate_features_batch): per cloud its voxel region, and its centre [4] + the
  // ForestTables of the scratch forest (pre_pts / pre_leaf_pts / pre_perm / pre_nodes hold its points and records)
  sgb::DevBuf pre_regions, pre_centres, pre_tables;

  // ---- multi-GPU exchange fused into the reduction's finishing CTA (sgb_comm_*, CommParams in sgb_device.cuh) ----
  sgb::DevBuf comm_mail;                  // this rank's mailbox (zeroed at allocation)
  unsigned char* comm_peers[8] = {};      // mailbox of every rank as mapped into this process (own entry = comm_mail.p)
  bool comm_ipc_opened[8] = {};           // mapped by cudaIpcOpenMemHandle (to be closed)
  int comm_world = 0, comm_rank = 0;      // world <= 1: single GPU
  unsigned long long comm_seq = 0;        // collective calls issued so far
  unsigned long long comm_timeout_ns = 5000000000ull;  // a peer that has not arrived after 5 s (sgb_comm_set_timeout_ms) is given up on
  sgb::DevBuf comm_status;                // one sticky word: != 0 after an exchange gave up on a peer (read back with every host-visible result)
  bool comm_failed = false;               // host copy of that word: every later call of this context fails until sgb_comm_connect* is called again

  // ---- state of the last linearize (cached for error(), gicp_factor.hpp:94-96) ----
  bool have_lin = false;
  bool corr_seeds = false;  // corr[] holds correspondences of the current (target, tree, source) triple
  int lin_factor = 0, lin_robust = 0;
  double lin_c = 1.0;
  double Tlin[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
  const double* last_out = nullptr;  // device pointer holding H|b|e|inliers of the last linearize

  // ---- batch of sources (sgb_source_set_batch, sgb_capi_batch.cu): members concatenated in src_pts / src_covA / src_covB / src_perm ----
  std::vector<size_t> b_offsets;           // members + 1
  std::vector<uint8_t> b_lin, b_seeded;    // per member: linearised against the current target / correspondences usable as search seeds
  sgb::DevBuf b_centres, b_bounds;         // [members][4] / [members][6]
  sgb::DevBuf b_poses, b_lin_poses;        // [members][12]: this call's poses / each member's last linearisation pose
  sgb::DevBuf b_tiles, b_members;          // BatchTile / uint4 tables of the current call
  sgb::DevBuf b_corr;                      // per stored point: cached correspondence
  sgb::DevBuf b_vq, b_vcorr;               // virtual source of the search: transformed queries of the active members and what the search found
  sgb::DevBuf b_partials, b_out;           // per-tile partial sums, per-member results
  sgb::DevBuf b_state, b_phase;            // sgb_align_batch: per member MemberState / next round (kPhase*, one byte)
  sgb::DevBuf b_rows_e, b_rows_hb;         // sgb_*_batch_points: the per-point rows staged for outputs that are not device memory
  // sgb_source_set_weights: b_weighted = the batched calls scale each point's terms by b_weights (per stored point, stored order, every
  // one checked finite and >= 0); b_wnext / b_wbad = the gather's output and its first offending row, before the check lets it in force.
  // The source setters and pairings clear b_weighted (begin_source, begin_pairs); the buffer keeps its address while the count does.
  bool b_weighted = false;
  sgb::DevBuf b_weights, b_wnext, b_wbad;
  // sgb_align_batch_gnc, for the call's duration: b_wround = its rounds use b_wuse (null: unweighted) instead of the weights in force.
  // Its own grow-only buffers: g_w = the stage's weights (stored order), g_e = the reweighting linearize's e rows and then each point's g
  // (row layout), g_state = GncState [members] | live flags [members].
  bool b_wround = false;
  const double* b_wuse = nullptr;
  sgb::DevBuf g_w, g_e, g_state;
  // The clouds of sgb_source_set_batch are stored once (src_* and b_centres / b_bounds, cloud after cloud).  Without a pairing the
  // members are those clouds.  After sgb_source_set_pairs (b_paired) member p is a replica of one stored cloud in p_*, b_offsets are
  // the members' offsets, and b_pair_maps (empty: member m against map m) names each member's map.
  std::vector<size_t> b_cloud_offsets;     // clouds + 1
  sgb::DevBuf b_cloud_off;                 // the same as uint32, on the device
  bool b_paired = false;
  bool b_pair_has_maps = false;  // the pairing has a maps table (possibly of 0 members)
  std::vector<uint32_t> b_pair_maps;
  std::vector<uint32_t> b_pair_clouds;  // the cloud of each pair member
  uint32_t b_pair_max_map = 0;  // the largest map index the pairing names (b_pair_maps, or b_sub_maps of a submap pairing): the per-call check's fast path
  sgb::DevBuf p_tables;                    // uint32: member offsets [members + 1] | cloud of each member | map of each member
  sgb::DevBuf p_pts, p_covA, p_covB, p_perm, p_centres, p_bounds;
  // the many-maps target seen through b_pair_maps (PairView): rebuilt by the first batched call after the pairing or the target changed
  bool b_view_ok = false;
  sgb::DevBuf v_centres, v_tables, v_regions;  // [members][4] / pt_off [members + 1] | node_base [members] / [members]
  // After sgb_source_set_submaps (b_submaps; also b_paired, without a maps table) member p is aligned against the union of the entries
  // b_sub_off[p] .. b_sub_off[p + 1] - 1: entry j = map b_sub_maps[j] of a many-kd-trees target placed by a rigid pose.  s_tables is the
  // one upload of the lists (SubmapTables in sgb_capi_batch.cu), s_entries / s_centres the target seen through them (SubmapView,
  // rebuilt with b_view_ok), b_centry the entry of every cached correspondence (beside b_corr).
  bool b_submaps = false;
  std::vector<uint32_t> b_sub_off, b_sub_maps;
  sgb::DevBuf s_tables, s_entries, s_centres, b_centry;
  // sgb_align_batch_async: the round the planner made (BatchRound), the device's copy of b_seeded (b_dseed_ok: it never claims a seed
  // the host's flags would not allow; cleared with them) and the stream a round is captured on
  sgb::DevBuf b_round, b_dseed;
  bool b_dseed_ok = false;
  cudaStream_t cap_stream = nullptr;
  cudaStream_t cap_stream_nested = nullptr;  // the stream the body of a loop nested in a loop's body is captured on
  // sgb_align_joint and sgb_align_joint_gnc: the buffers of their JointParams.  sgb_align_joint_async and sgb_align_joint_gnc_async have
  // their own (joint_async), which no synchronous call writes: its tables are uploaded only when they differ from ja_tab, the host copy of
  // what joint_async.tables holds.
  sgb::JointBufs joint, joint_async;
  std::vector<uint32_t> ja_tab;
  // The instantiated loops of sgb_align_batch_async, sgb_align_joint_async and the loops of stages of both batch GNC aligns (gnc_loop: its
  // graph reads no caller pointer), of sgb_align_joint_gnc_async (on joint_async) and of sgb_align_joint_gnc (joint_gnc_sync_loop, on joint)
  sgb::LoopGraph align_loop, joint_loop, gnc_loop, joint_gnc_loop, joint_gnc_sync_loop;
};

namespace sgb {

inline int fail(sgb_ctx* c, int code, const std::string& msg) {
  if (c) c->err = msg;
  return code;
}

/// device-side tree construction (sgb_capi_preprocess.cu)
int build_lbvh(sgb_ctx* ctx, const float4* d_orig_pts, size_t n, const double* d_centre4, DevBuf& perm, DevBuf& leaf_pts, DevBuf& pnodes, int* depth);
/// uniform grid over the current (leaf-ordered) target for the search front end; no-op unless enabled
int build_grid(sgb_ctx* ctx);

// ---- transitions (sgb_capi.cu) ----
/// a target of n points (with normals / covariances / FP32 rounding residuals as flagged) replaces the target; no search structure yet
int begin_point_target(sgb_ctx* ctx, size_t n, bool normals, bool covs, bool lo);
/// a voxel map of n voxels (maps: n_maps voxel maps, VoxelMaps) replaces the target (the caller fills tgt_pts / tgt_cov*, vox_table and
/// for maps vm_centres / vm_regions)
int begin_voxel_target(sgb_ctx* ctx, size_t n, bool covs, double leaf_size, int search_offsets, bool maps = false, size_t n_maps = 0);
/// n_maps point clouds of n points in all (with normals / covariances as flagged) replace the target as many kd-trees (KdTrees); the
/// caller fills tgt_pts / tgt_normals / tgt_cov* / tgt_pnodes and kt_*
int begin_forest_target(sgb_ctx* ctx, size_t n, bool normals, bool covs, size_t n_maps);
/// the map count of a multi-map target (VoxelMaps or KdTrees), else 0
size_t target_maps(const sgb_ctx* ctx);
/// the point target's tree in tgt_perm / tgt_pts / tgt_pnodes (depth, n_pnodes packet records) becomes its search structure; builds the grid
int install_tree(sgb_ctx* ctx, int depth, size_t n_pnodes);
/// a single cloud of n points, a batch (n = 0) or nothing replaces the source (and forgets any pairing of a batch)
void begin_source(sgb_ctx* ctx, SourceState state, size_t n, bool covs);
/// the batch's members become pairs of its stored clouds (the caller fills b_offsets, b_pair_maps or the submap lists, and the replicas)
void begin_pairs(sgb_ctx* ctx);
/// normals and covariances (target) or covariances (source) were estimated on the device
void features_changed(sgb_ctx* ctx, bool target);

// ---- steps shared by the entry points (sgb_capi.cu) ----
void pose_from_colmajor(const double* T, double out12[12]);
/// gathers the target's normals / covariances (and with points its FP32 points) from original into leaf order: 0 or 1 launch
int gather_target_features(sgb_ctx* ctx, bool points);
/// sizes the per-query scratch of the search for n queries, so that the linearize calls never (re)allocate: a cudaFree there would
/// synchronise the device in the middle of an asynchronous call
int reserve_query_scratch(sgb_ctx* ctx, size_t n);
/// stores stage_pts[off, off + n) as one source cloud in src_*[off..] (see the definition); 5 launches, + 1 + cov_chunks with covariances
int store_source(sgb_ctx* ctx, size_t off, size_t n, double* centre, double* bounds, float4* lo, size_t sort_bytes, uint32_t run, int cov_chunks,
                 const cudaEvent_t* arrived);
/// the submap lists of sgb_source_set_submaps / sgb_target_batch_knn_submaps checked (messages start with who; what names a list's owner)
/// and laid out for the device: inverse entry poses [entries][12] | list_off [n_lists + 1] | entry_maps [entries] (sgb_capi_batch.cu)
int submap_lists(sgb_ctx* ctx, const std::string& who, const char* what, size_t n_lists, const size_t* list_off, const uint32_t* entry_maps,
                 const double* entry_poses16, std::vector<double>& tables, uint32_t* max_map);
/// the target can serve `factor` (who names the caller in the message)
int check_target(sgb_ctx* ctx, const char* who, int factor);
/// FP32 search bound a hair above the rejector's threshold (FLT_MAX without a distance rejector)
float search_bound(int rejector, double max_dist_sq);

struct LinParams;
struct ChunkClasses;
struct PendingParams;
/// kernel parameters of the current target and source at pose T (sgb_capi.cu)
int fill_params(sgb_ctx* ctx, LinParams& P, const double* T_colmajor16);
/// the grid front end's parameters of a point search over n queries with the class counters of `parity` (grid_ready; sgb_capi.cu)
void point_search_params(const sgb_ctx* ctx, size_t n, int parity, ChunkClasses& cc, PendingParams& pp);
/// nearest-neighbour search of the P.src.n queries of P.src in a point target: grid probe, then the packet search (sgb_capi.cu)
int launch_point_search(sgb_ctx* ctx, const LinParams& P, int depth);

}  // namespace sgb

#define CU(expr)                                                                                                 \
  do {                                                                                                           \
    cudaError_t _e = (expr);                                                                                     \
    if (_e != cudaSuccess) return sgb::fail(ctx, 2, std::string(#expr) + ": " + cudaGetErrorString(_e));        \
  } while (0)
