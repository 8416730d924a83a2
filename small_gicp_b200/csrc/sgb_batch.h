// SPDX-License-Identifier: MIT
// Batched registration: device-side layout and launchers (sgb_batch.cu; C-ABI in sgb_capi_batch.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sgb_device.cuh"

namespace sgb {

/// 128 consecutive points (or fewer, at the end of a member) of ONE member: `first` = position in the member-concatenated storage,
/// `vfirst` = position in the virtual source of this call (the active members' points, concatenated)
struct __align__(16) BatchTile {
  uint32_t member, first, count, vfirst;
};
/// per member: x = first tile of this call, y = tile count (0: inactive or empty), z = flags
constexpr uint32_t kMemberActive = 1u, kMemberSeeded = 2u;

struct BatchParams {
  DevTarget tgt;
  const float4* pts;   // members concatenated, each centred on its own box and in its own curve order (as sgb_source_set_points stores one cloud)
  const float4* covA;
  const float4* covB;
  const double* centres;  // [members][4]
  const double* poses;    // [members][12] row-major R | t of this call
  double* lin_poses;      // [members][12] pose of each member's last linearize
  const BatchTile* tiles;
  const uint4* members;
  uint32_t* corr;         // per stored point: leaf-order position / voxel id of its correspondence, or kNone
  double max_dist_sq_d;
  double robust_c;
  double* tile_partials;  // [tiles][kPartialStride]
};

/// Per-point rows of sgb_linearize_batch_points / sgb_error_batch_points, written by the factor kernel beside its sums: stored point i of
/// member m writes row batch_row(member_off, perm, m, i), the caller's order of sgb_correspondences_batch.  e: [points] the point's share
/// of the member's e (or null); Hb: [points][42] its H (36, row-major) | b (6) (or null; linearize only).  w: the weights in force
/// (sgb_source_set_weights), [points] in stored order, read by the weighted instantiations only (any mode, the rows' fields unused
/// without POINTS).  Kept out of BatchParams, which keys the cached graph of sgb_align_batch_async.
struct BatchRows {
  const uint32_t* perm;        // stored position -> original index within the member's cloud
  const uint32_t* member_off;  // [members + 1]
  double* e;
  double* Hb;
  const double* w;
};
/// the caller's row of stored point i of member m: the member's first row plus the point's original index within its cloud
__device__ __forceinline__ size_t batch_row(const uint32_t* __restrict__ member_off, const uint32_t* __restrict__ perm, uint32_t m, uint32_t i) {
  return static_cast<size_t>(__ldg(&member_off[m])) + __ldg(&perm[i]);
}
/// sgb_source_set_weights: the caller's weights (src, row layout) gathered into stored order (dst), n stored points of n_members members
/// (member_off / perm as BatchRows); the first row whose weight is not finite and >= 0 goes to *bad (atomicMin; ~0u: none)
struct WeightGather {
  uint32_t n, n_members;
  const uint32_t *member_off, *perm;
  const double* src;
  double* dst;
  uint32_t* bad;
};
cudaError_t launch_weight_gather(const WeightGather& g, int sm_count, cudaStream_t st);

/// Members as (cloud, map) pairs (sgb_source_set_pairs): member p = a replica of stored cloud clouds[p], at member_off[p] .. member_off[p+1]
/// of the member buffers; its centre and bounds too.  covA = null: no covariances.
struct PairGather {
  uint32_t n, n_members;  // member points, members
  const uint32_t *member_off, *clouds, *cloud_off;
  const float4 *pts, *covA, *covB;
  const uint32_t* perm;
  const double *centres, *bounds;
  float4 *out_pts, *out_covA, *out_covB;
  uint32_t* out_perm;
  double *out_centres, *out_bounds;
};
cudaError_t launch_pair_gather(const PairGather& g, int sm_count, cudaStream_t st);
/// What the round kernels read per map, indexed by member instead (member p -> map maps[p]): centres [members][4]; many kd-trees
/// (map_pt_off non-null): pt_off [members + 1] and node_base [members] of a ForestView; voxel maps (map_regions non-null): regions.
struct PairView {
  uint32_t n_members;
  const uint32_t* maps;
  const double* map_centres;
  const uint32_t *map_pt_off, *map_node_base;
  const uint4* map_regions;
  double* centres;
  uint32_t *pt_off, *node_base;
  uint4* regions;
};
cudaError_t launch_pair_view(const PairView& v, cudaStream_t st);
/// Submap members (sgb_source_set_submaps): member p is aligned against the union of its entries entry_off[p] .. entry_off[p + 1] - 1,
/// entry j = one map of a many-kd-trees target placed by a rigid pose.  Nothing of a map is transformed: the member's pose is carried
/// into each map's stored frame (relative_pose) instead.
struct SubmapView {
  const uint32_t* entry_off;  // [members + 1]
  const uint4* entries;       // per entry: first point of its map in tgt_pts, point count, first packet record, map
  const double* centres;      // [entries][4] the map's centre
  const double* inv_poses;    // [entries][12] inverse of the entry's placement, row-major R^T | -R^T t
  uint32_t* centry;           // per stored member point, beside BatchParams::corr: the entry (within the member's list) its correspondence lies in
};
/// The per-entry tables above from the target's per-map tables, one launch: entry j -> map entry_maps[j].
struct SubmapViewBuild {
  uint32_t n_entries;
  const uint32_t* entry_maps;
  const uint32_t *map_pt_off, *map_node_base;
  const double* map_centres;
  uint4* entries;
  double* centres;
};
cudaError_t launch_submap_view(const SubmapViewBuild& v, int sm_count, cudaStream_t st);
/// launch_correspondences for one submap member: out[perm[i]] = (entry << 32) | original index within the entry's map
cudaError_t launch_submap_correspondences(const uint32_t* corr, const uint32_t* centry, const uint32_t* perm, size_t n, const float4* tgt_pts, uint64_t* out,
                                          int sm_count, cudaStream_t st);
// ---- sgb_align_batch_async (DESIGN.md §11 "Asynchronous align"): the rounds planned and sized on the device ----
/// What a round does, written by batch_plan_kernel at its head and read by every kernel of the round.  lin: 1 = linearize of the members
/// in kPhaseLinearize, 0 = error() of the members in kPhaseTrial; n_tiles: tiles the factor kernel and the tile searches process;
/// n_search: queries of the virtual source (linearize rounds of a point target, else 0); n_clear: tiles whose points are left without a
/// correspondence (a linearize round against an empty target).
struct __align__(16) BatchRound {
  uint32_t lin, n_tiles, n_search, n_clear;
};
/// The planner's inputs: the host loop's rule and batch_tables' tables, built on the device by one CTA.
struct BatchPlan {
  uint32_t n_members;
  const uint32_t* member_off;  // [members + 1]
  const uint8_t* phase;        // [members] kPhase* after the last step
  uint8_t* seeded;             // [members] the device's copy of b_seeded: 1 = the member's cached correspondences may seed its search
  int seeds;                   // linearize rounds mark seeded members (point targets; voxel maps have no search to seed)
  int no_target;               // an empty target: no tiles to search or factor (the members still get zeros), n_clear instead
  BatchTile* tiles;
  uint4* members;
  BatchRound* round;
  uint32_t* zero[3];  // counters of the point search cleared at the head of every round (null: none)
  uint32_t zero_n[3];
  cudaGraphConditionalHandle loop;  // set to 0 here; the step kernel sets it to 1 while a member is still in a round
};
cudaError_t launch_batch_plan(const BatchPlan& p, cudaStream_t st);

// ---- one launcher per step of a round.  round = null: a round planned on the host, with exact grids (n_tiles tiles of the call, n_members
// members).  Else a round planned on the device (batch_plan_kernel): the grids are sized for every tile (n_tiles = the most a round can
// have), what the round does is read from `round`, and the CTAs beyond it exit at once. ----
/// The active members' queries as the virtual source of the point search (linearize rounds only)
cudaError_t launch_batch_transform(const BatchParams& B, const BatchRound* round, uint32_t n_tiles, float4* vq, uint32_t* vcorr, cudaStream_t st);
/// A linearize round against an empty target (planned on the device): every point of the active members is left without a correspondence
cudaError_t launch_batch_unmatch(const BatchParams& B, const BatchRound* round, uint32_t n_tiles, cudaStream_t st);
/// The factor kernel of the target's kind: 0 one point target (vcorr = the point search's result over the virtual source), 1 one voxel
/// map (the VGICP probe), 2 many voxel maps (member m against map m: map_centres [maps][4], map_regions [maps] = (first table slot, mask,
/// first voxel, voxel count) of each map), 3 many kd-trees (map_centres; vcorr = the forest search's result), 4 submaps (S; vcorr = the
/// submap search's result).  Linearize (err = false), error() with the cached correspondences (err = true), or with a round what it
/// says.  Point-to-plane only for kinds 0 and 3.  rows (null: none): every processed point's row too; with a round only unweighted and
/// without a robust kernel (the reweighting round of sgb_align_batch_gnc_async).  weights (null: none): each point's terms scaled by its
/// weight (stored order) before its row and the sums.
cudaError_t launch_batch_factor(const BatchParams& B, int kind, int factor, int robust, bool err, const BatchRound* round, uint32_t n_tiles, const uint32_t* vcorr,
                                const double* map_centres, const uint4* map_regions, const SubmapView& S, const BatchRows* rows, const double* weights,
                                cudaStream_t st);
/// out: [members][44] (linearize) or [members] (error)
cudaError_t launch_batch_segment(const BatchParams& B, uint32_t n_members, bool linearize, const BatchRound* round, double* out, cudaStream_t st);
/// batched align(): every member whose phase matches the round (linearize: kPhaseLinearize, else kPhaseTrial) takes its optimiser step
/// from `out` (what launch_batch_segment wrote); then every member's next pose (row-major R | t) goes to poses and its phase to phase.
/// With a round, the step sets `loop` to 1 while a member is still in a round.
cudaError_t launch_batch_step(const AlignOptions& o, uint32_t n_members, bool linearize, const BatchRound* round, cudaGraphConditionalHandle loop,
                              const double* out, MemberState* state, double* poses, uint8_t* phase, cudaStream_t st);
/// align_init of every member from its column-major initial pose: state, this call's pose and phase; seeded cleared unless keep_seeds
cudaError_t launch_batch_align_init(const AlignOptions& o, uint32_t n_members, const double* init_T16, MemberState* state, double* poses, uint8_t* phase,
                                    uint8_t* seeded, bool keep_seeds, cudaStream_t st);
/// sgb_align_batch's outputs from the members' final state: T (16, column-major), info (converged, iterations, inliers, error), H | b (or null)
cudaError_t launch_batch_align_finish(uint32_t n_members, const MemberState* state, double* out_T16, double* out_info4, double* out_Hb42, cudaStream_t st);

// ---- sgb_align_batch_gnc (DESIGN.md §11 "Graduated non-convexity"): the stages' reweighting between the stages' aligns ----
/// What the GNC kernels of one stage share.  The members in the stage are those with live[m] = 1.  e: [rows] in the row layout of BatchRows
/// (member_off, perm): the reweighting linearize's e rows in, each point's g of the stage out.  corr: BatchParams::corr after that
/// linearize.  w: the weights in force in stored order (null: none); wstage: [points] w_i g_i in stored order, the weights of the stage's align.
struct GncParams {
  uint32_t n, n_members;
  int kind;        // kGncGemanMcClure / kGncTls
  double c2;       // the noise bound c^2
  int max_stages, stage_iterations;
  const uint32_t *member_off, *perm;
  const uint32_t* corr;
  double* e;
  const double* w;
  double* wstage;
  GncState* gnc;   // [members]
  uint8_t* live;   // [members] in: in this stage; the init kernel leaves 1 for a member with a stage to go
};
/// stage 0: every member's largest r^2 = 2 e_i > 0 over its points with a correspondence (gnc[m].r2max, cleared by the caller).  Launched
/// at every stage of the device loop: the members that have begun no stage only
cudaError_t launch_gnc_rmax(const GncParams& p, int sm_count, cudaStream_t st);
/// one thread per member in the stage: gnc_stage_begin
cudaError_t launch_gnc_stage(const GncParams& p, cudaStream_t st);
/// one thread per stored point of a member in the stage: its g (0 without a correspondence) to e, w_i g_i to wstage, TLS's not_binary flag
cudaError_t launch_gnc_weight(const GncParams& p, int sm_count, cudaStream_t st);
/// one thread per member: a member in the stage ends GNC after it if the stage is its last (TLS: or its weights are all binary), adds
/// the previous stage's iterations and starts its align from its current pose (align_init of o with max_iterations = stage_iterations
/// unless last; pose and phase as the align's rounds read them); every other member is left done
cudaError_t launch_gnc_init(const GncParams& p, const AlignOptions& o, MemberState* state, double* poses, uint8_t* phase, cudaStream_t st);
/// launch_batch_step for a round of a GNC stage planned on the device: each member steps with its stage's max_iterations (as launch_gnc_init
/// chose), the round's kind read from `round`, `loop` set to 1 while a member has a round to go
cudaError_t launch_gnc_step(const GncParams& p, const AlignOptions& o, const BatchRound* round, cudaGraphConditionalHandle loop, const double* out,
                            MemberState* state, double* poses, uint8_t* phase, cudaStream_t st);

// ---- sgb_align_batch_gnc_async (DESIGN.md §11 "Asynchronous graduated non-convexity"): the stages and their rounds on the device ----
/// the head of a stage: phase[m] = kPhaseLinearize for the members still in GNC (live), kPhaseDone for the others; `rounds` set to 0
cudaError_t launch_gnc_reweigh(uint32_t n_members, const uint8_t* live, uint8_t* phase, cudaGraphConditionalHandle rounds, cudaStream_t st);
/// after launch_gnc_init: `stages` set to 1 if a member has a stage to go after this one (live), `rounds` to 1 if a member's align has a
/// round to go
cudaError_t launch_gnc_loops(uint32_t n_members, const uint8_t* live, const uint8_t* phase, cudaGraphConditionalHandle stages, cudaGraphConditionalHandle rounds,
                             cudaStream_t st);
/// after launch_batch_align_finish: info's iterations summed over the stages, and gnc2 (or null) = the stages run and the last stage's mu
cudaError_t launch_gnc_finish(uint32_t n_members, const MemberState* state, const GncState* gnc, double* out_info4, double* out_gnc2, cudaStream_t st);

// ---- sgb_align_joint (DESIGN.md §11 "Joint windows"): windows of frames, each edge a pair member ----
/// The call's tables (built once per call) and state.  Window w holds frames frame_off[w] .. frame_off[w + 1] - 1 and the edges
/// edge_off[w] .. edge_off[w + 1] - 1 of the edge list (member order within each window); edge q is member edge_member[q], cloud frame
/// edge_i[q] against map frame edge_j[q] (local to the window).  free[k]: index of frame k among its window's free frames, or -1.
struct JointParams {
  uint32_t n_windows, n_edges;
  const uint32_t *frame_off, *edge_off, *n_free, *edge_member, *edge_win;
  const int *edge_i, *edge_j, *free;
  double *X, *cand, *delta;  // [frames][16] / [frames][16] / [frames][6] (window w's steps from 6 frame_off[w])
  double* sums;              // [edges][44]: each edge's H | b | e | inliers of its last linearize
  WindowState* state;        // [windows]
  uint8_t* phase;            // [windows]
  double* poses;             // BatchParams::poses: [members][12]
};
/// the scratch of joint_step_kernel for windows of up to max_free free frames (dynamic shared memory)
inline size_t joint_step_smem(int max_free) { return static_cast<size_t>(joint_work_doubles(max_free)) * sizeof(double); }
/// every edge's pose X_j^-1 X_i (row-major R | t) from the frames' X
cudaError_t launch_joint_edge_poses(const JointParams& J, cudaStream_t st);
/// one CTA per window: every window in the round's phase (linearize: kPhaseLinearize, else kPhaseTrial) takes its step from `out` (what
/// launch_batch_segment wrote for the edges), then writes its edges' next poses and its phase.  With a round (planned on the device) the
/// kind is the round's, every stepped window's phase goes to its edges' member_phase too, and `loop` is set to 1 while a window still
/// has a round to go.
cudaError_t launch_joint_step(const AlignOptions& o, const JointParams& J, int max_free, bool linearize, const BatchRound* round, cudaGraphConditionalHandle loop,
                              uint8_t* member_phase, const double* out, cudaStream_t st);

// ---- sgb_align_joint_async (DESIGN.md §11 "Asynchronous joint windows"): the rounds of sgb_align_joint planned on the device ----
/// one CTA per window: joint_init, the frames' X from init_X16 (column-major), every edge's initial pose, its window's phase as its member
/// phase, and its seed flag cleared unless keep_seeds
cudaError_t launch_joint_align_init(const AlignOptions& o, const JointParams& J, const double* init_X16, uint8_t* member_phase, uint8_t* seeded, bool keep_seeds,
                                    cudaStream_t st);
/// sgb_align_joint's outputs from the windows' final state: X (16, column-major) per frame, fixed frames copied from init_X16; info
/// (converged, iterations, inliers, error) per window
cudaError_t launch_joint_align_finish(const JointParams& J, uint32_t n_frames, const double* init_X16, double* out_X16, double* out_info4, cudaStream_t st);

// ---- sgb_align_joint_gnc (DESIGN.md §11 "Graduated non-convexity for joint windows"): sgb_align_batch_gnc's stages with the window as the
// GNC unit.  GncState and live flags per window: p (the point kernels) has n_members = the edges, each point's window member_win[its edge];
// pw (the window kernels, and launch_gnc_stage) the same with n_members = the windows. ----
/// stage 0: every window's largest r^2 = 2 e_i > 0 over its edges' points with a correspondence (gnc[w].r2max, cleared by the caller).
/// Launched at every stage of the device loop: the windows that have begun no stage only
cudaError_t launch_joint_gnc_rmax(const GncParams& p, const uint32_t* member_win, int sm_count, cudaStream_t st);
/// launch_gnc_weight with each point's window's mu (TLS: not_binary per window)
cudaError_t launch_joint_gnc_weight(const GncParams& p, const uint32_t* member_win, int sm_count, cudaStream_t st);
/// launch_gnc_init per window: joint_init of a window in the stage from its current X (max_iterations = stage_iterations unless last),
/// its phase to J.phase; every other window is left done
cudaError_t launch_joint_gnc_init(const GncParams& pw, const AlignOptions& o, const JointParams& J, cudaStream_t st);
/// launch_joint_step for a round of a GNC stage planned on the device (member_phase, loop as there): each window steps with its stage's
/// max_iterations
cudaError_t launch_joint_gnc_step(const AlignOptions& o, const JointParams& J, int max_free, const double* out, const GncParams& pw, const BatchRound* round,
                                  cudaGraphConditionalHandle loop, uint8_t* member_phase, cudaStream_t st);

// ---- sgb_align_joint_gnc_async (DESIGN.md §11 "Asynchronous graduated non-convexity for joint windows"): the stages and their joint rounds
// on the device, the edges the members of the rounds ----
/// the head of a stage: member_phase of every edge of a window still in GNC (live) = kPhaseLinearize, of every other edge kPhaseDone;
/// `rounds` set to 0
cudaError_t launch_joint_gnc_reweigh(const JointParams& J, const uint8_t* live, uint8_t* member_phase, cudaGraphConditionalHandle rounds, cudaStream_t st);
/// after launch_joint_gnc_init: every edge's member_phase = its window's phase; `stages` set to 1 if a window has a stage to go after this
/// one (live), `rounds` to 1 if a window's joint align has a round to go
cudaError_t launch_joint_gnc_loops(const JointParams& J, const uint8_t* live, uint8_t* member_phase, cudaGraphConditionalHandle stages,
                                   cudaGraphConditionalHandle rounds, cudaStream_t st);
/// after launch_joint_align_finish: info's iterations summed over each window's stages, and gnc2 (or null) = the stages run and the last mu
cudaError_t launch_joint_gnc_finish(const JointParams& J, const GncState* gnc, double* out_info4, double* out_gnc2, cudaStream_t st);

}  // namespace sgb
