/* SPDX-License-Identifier: MIT
 *
 * sgicp_b200.h -- C-ABI of the H100-native small_gicp hot path (libsgicp_b200.so).
 *
 * One context = one GPU = one CUDA stream.  A context is NOT thread-safe; distinct contexts are
 * (the reference runs several align() calls concurrently from TBB flow-graph nodes,
 * src/benchmark/odometry_benchmark_small_gicp_tbb_flow.cpp:81-98 -- give each its own context).
 * Distinct contexts may also be on distinct devices of one process, used at the same time.
 *
 * Every entry point returns 0 on success and a non-zero code on failure; sgb_last_error() then
 * returns a description.  There is NO CPU fallback: without a CUDA device sgb_create() fails.
 *
 * All host input buffers are borrowed for the duration of the call only; the context owns all
 * device memory.  One exception, by CUDA's own rules: a cloud passed in PAGE-LOCKED host memory
 * (cudaMallocHost / cudaHostRegister / torch pin_memory) is copied asynchronously on the context's
 * stream, so sgb_{target,source}_set_points / sgb_target_set_voxelmap may return before it has been
 * read -- leave such a buffer unchanged until sgb_synchronize() or any call that returns results to
 * the host (sgb_linearize, sgb_error, sgb_correspondences, ...).  Pageable memory (std::vector,
 * numpy) is consumed when the call returns.  Every bulk input / output pointer (points, normals, covariances, queries, feature and
 * correspondence outputs) may also be a DEVICE pointer of the context's GPU (copies use cudaMemcpyDefault): a device-resident producer hands
 * its buffers over without a host round trip.  Host layouts are exactly the reference's in-memory layouts so that the header
 * glue (INTEGRATION.md) can pass `cloud.points[0].data()` etc. without repacking:
 *   points / normals : N x 4 doubles (x,y,z,1) / (nx,ny,nz,0)   -- std::vector<Eigen::Vector4d>,
 *                      include/small_gicp/points/point_cloud.hpp:69-70
 *   covariances      : N x 16 doubles, 4x4 with zero 4th row/col (symmetric, so row/col-major
 *                      agree)                                    -- point_cloud.hpp:71
 *   poses            : 16 doubles, COLUMN-major 4x4 = Eigen::Isometry3d::data()
 *   H | b | e        : 36 + 6 + 1 doubles (H symmetric)          -- the tuple returned by
 *                      Reduction::linearize, registration/reduction.hpp:20-27
 *
 * Non-finite points.  A point whose x, y or z is NaN or +-Inf (organized LiDAR clouds mark missing
 * returns so) is INERT, in every call that takes points:
 *   - box and storage: it takes no part in its cloud's box, centre, extent, curve keys, tree boxes or
 *     grid; every finite point is stored bit for bit as it is in the cloud without it;
 *   - sgb_voxelgrid_sampling(_batch) and sgb_target_build_voxelmap(s) drop it, as the reference does;
 *   - in a target (single kd-tree, many kd-trees, pairs, submaps, the grid front end) it is never a
 *     correspondence and never a k-NN entry (sgb_target_batch_knn, sgb_target_knn_maps / _submaps);
 *   - in a source (single, batch, pairs, submaps, joint frames) it has no correspondence and zero
 *     per-point rows: it adds nothing to H | b | e, the inlier count or error(); in GNC its weight is 0;
 *   - in sgb_estimate_features(_batch) it is never another point's neighbour, and its own row gets what a
 *     point with fewer than 5 neighbours gets (zero normal, identity covariance).
 * So the results for the finite rows equal the results for the cloud with the non-finite rows removed,
 * indices mapped back.  Non-finite normals, covariances or poses supplied by the caller are not covered:
 * they propagate, as in the reference.
 */
#ifndef SGICP_B200_H_
#define SGICP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sgb_ctx sgb_ctx;

/* Per-point factor evaluated by the kernel.
 * replaces ICPFactor::linearize/error          include/small_gicp/factors/icp_factor.hpp:20-64
 *          PointToPlaneICPFactor::linearize/.. include/small_gicp/factors/plane_icp_factor.hpp:20-69
 *          GICPFactor::linearize/error         include/small_gicp/factors/gicp_factor.hpp:35-89 */
enum sgb_factor_kind { SGB_FACTOR_ICP = 0, SGB_FACTOR_PLANE_ICP = 1, SGB_FACTOR_GICP = 2 };
/* RobustFactor<Huber|Cauchy, F>   include/small_gicp/factors/robust_kernel.hpp:11-106 */
enum sgb_robust_kind { SGB_ROBUST_NONE = 0, SGB_ROBUST_HUBER = 1, SGB_ROBUST_CAUCHY = 2 };
/* NullRejector / DistanceRejector include/small_gicp/registration/rejector.hpp:11-28 */
enum sgb_rejector_kind { SGB_REJECT_NONE = 0, SGB_REJECT_DISTANCE = 1 };

#define SGB_NO_CORRESPONDENCE UINT64_MAX /* std::numeric_limits<size_t>::max(), icp_factor.hpp:66 */

/* ---- context ------------------------------------------------------------------------------ */
int sgb_create(int device_id, sgb_ctx** out_ctx);
void sgb_destroy(sgb_ctx* ctx);
/* ctx may be NULL: returns the error of the last failed sgb_create() on this thread. */
const char* sgb_last_error(const sgb_ctx* ctx);
/* Run all work of this context on an existing cudaStream_t (e.g. the caller's / torch's current
 * stream) instead of the context's own.  Pass NULL to go back to the private stream. */
int sgb_set_stream(sgb_ctx* ctx, void* cuda_stream);
/* Block until everything queued by this context has finished. */
int sgb_synchronize(sgb_ctx* ctx);
/* Number of this library's kernels launched by the context since creation (bench.py gpu_launches). */
uint64_t sgb_kernel_launches(const sgb_ctx* ctx);

/* ---- multi-GPU (one process per GPU, source sharded, target replicated; SURVEY.md §8e).  The reference has no
 *      counterpart: its reductions (reduction_omp.hpp:24-58, reduction_tbb.hpp:70-92) sum within one process.  After
 *      sgb_comm_connect* every sgb_linearize* / sgb_error* of this context returns the SUM OVER ALL RANKS: the CTA that
 *      finishes the reduction writes its sums straight into the peers' mailboxes over NVLink and adds theirs (one kernel,
 *      no NCCL call, deterministic rank order).  All ranks must issue the same sequence of linearize / error calls. ---- */
#define SGB_COMM_HANDLE_BYTES 64
#define SGB_COMM_MAX_RANKS 8
/* CUDA IPC handle (64 bytes) of this context's mailbox; allocate it on first use. */
int sgb_comm_handle(sgb_ctx* ctx, void* out_handle64);
/* `handles` = world x 64 bytes, rank order, gathered by the caller (e.g. torch.distributed.all_gather). */
int sgb_comm_connect(sgb_ctx* ctx, int rank, int world, const void* handles);
/* Same wiring from raw device pointers (contexts of ONE process: tests, single-process multi-stream setups). */
int sgb_comm_mailbox(sgb_ctx* ctx, void** out_device_ptr);
int sgb_comm_connect_ptrs(sgb_ctx* ctx, int rank, int world, void* const* mailboxes);
int sgb_comm_disconnect(sgb_ctx* ctx);
/* How long a rank waits for a peer before it gives up on an exchange (default 5000 ms). */
int sgb_comm_set_timeout_ms(sgb_ctx* ctx, int milliseconds);
/* Failure handling of the fused exchange.  A rank that gives up on a peer (timeout), or that hears from a peer that its call failed on
 * the host, gets NaN sums AND a sticky status word: the host-returning calls (sgb_linearize, sgb_error) then return a non-zero code
 * (4), every later collective call of the context returns 5 until sgb_comm_connect* is called again.  Users of the *_device variants
 * read the status themselves: 0 = fine, bit 0 = timeout, bit 1 = a peer reported a failed call.  A call that fails on the host of one
 * rank (bad argument, missing covariances) still takes part in the exchange -- it tells the peers instead of leaving them waiting. */
int sgb_comm_status(sgb_ctx* ctx, int* out_status);
/* Diagnostics: nanoseconds this rank's finishing CTA waited for its slowest peer in each of the last 64 exchanges (ring indexed by
 * call number % 64; *out_calls = exchanges so far).  The rank that arrives last sees the bare transport latency, the first one skew
 * + transport: the minimum and maximum over the ranks separate the two (bench.py `comm_wait_us`). */
int sgb_comm_wait_ns(sgb_ctx* ctx, uint64_t* out_ring64, uint64_t* out_calls);

/* ---- target: replaces traits::point/normal/cov(target, k) (points/traits.hpp:38-54) and the
 *      target_tree argument of Reduction::linearize (reduction.hpp:23) -------------------------- */
int sgb_target_set_points(sgb_ctx* ctx, size_t n, const double* points_xyz1, const double* normals_xyz0 /*or NULL*/,
                          const double* covs_4x4 /*or NULL*/);
/* Adopt a tree built by the reference: `nodes24` = KdTree<PointCloud>::kdtree.nodes.data()
 * (KdTreeNode<AxisAlignedProjection>, 24 bytes, ann/kdtree.hpp:56-71), `indices` = ...kdtree.indices.data()
 * (ann/kdtree.hpp:237).  Any builder's node order is accepted (serial / OMP / TBB). Leaf scan order is
 * preserved, so exact-tie behaviour follows the reference's (ann/knn_result.hpp:80-83). */
int sgb_target_set_kdtree(sgb_ctx* ctx, const void* nodes24, size_t n_nodes, uint32_t root, const uint64_t* indices);
/* Or build this library's own kd-tree over the current target points ON THE DEVICE (replaces
 * KdTreeBuilder::build_tree, ann/kdtree.hpp:74-131, and the OMP / TBB builders): Hilbert-order sort, then one radix sort
 * per level along the widest axis of every node's box -- a balanced median-split kd-tree with at most 32 points per leaf
 * (one per lane of the warp-cooperative leaf scan; the reference's builder uses 20), stored implicitly.  Asynchronous on
 * the context's stream, no host round trip.  Exact nearest-neighbour results do not depend on the split choices (only
 * exact ties can).  max_leaf_size is accepted for source compatibility with KdTreeBuilder::max_leaf_size and ignored. */
int sgb_target_build_kdtree(sgb_ctx* ctx, int max_leaf_size);
/* Gaussian voxel map target (VGICP): replaces IncrementalVoxelMap<GaussianVoxel>::nearest_neighbor_search
 * (ann/incremental_voxelmap.hpp:99-119) and its point/cov traits (:207-222).  Voxel i of the arrays is
 * flat_voxels[i]; reported correspondences are (i << 32) like calc_index (:151).
 * search_offsets is 1, 7 or 27 (:157-186). */
int sgb_target_set_voxelmap(sgb_ctx* ctx, double leaf_size, size_t n_voxels, const int32_t* coords_xyz, const double* means_xyz1,
                            const double* covs_4x4, int search_offsets);
/* Build the Gaussian voxel map on the device from raw points (+ 4x4 covariances): replaces the one-shot use of
 * IncrementalVoxelMap<GaussianVoxel>::insert (ann/incremental_voxelmap.hpp:55-92) with GaussianVoxel::add / finalize
 * (ann/gaussian_voxelmap.hpp:30-62): voxel = floor(p / leaf_size), mean = sum p / n, cov = sum C / n.  Voxel ids are in
 * ascending key order (the reference numbers them in first-insertion order; only the ids differ). */
int sgb_target_build_voxelmap(sgb_ctx* ctx, size_t n, const double* points_xyz1, const double* covs_4x4 /*or NULL*/, double leaf_size,
                              int search_offsets);
/* n_maps Gaussian voxel maps as ONE target, for the batched calls only (member m is aligned against map m; see the batch section).
 * offsets: n_maps + 1 ascending entries, offsets[0] = 0; map m = points offsets[m] .. offsets[m+1] (empty maps allowed), covariances
 * likewise (or NULL).  Host, page-locked or device memory.  Map m is stored exactly as sgb_target_build_voxelmap would store it alone:
 * the same voxels in ascending key order, FP64 sums in ascending original index within a voxel, FP32 about the centre of its own voxel
 * means, points outside the 21-bit voxel range dropped; each map has its own region of the hash table, so a member can only ever match
 * its own map's voxels.  sgb_target_size returns the total voxel count.  A fixed number of launches and one host synchronisation
 * whatever n_maps is.  n_maps <= SGB_BATCH_MAX_MEMBERS, fewer than 2^31 points in all, leaf_size > 0, search_offsets 1, 7 or 27; at
 * most 2^29 voxels in all (the table regions are addressed with 32-bit slot numbers), else the call fails with a message. */
int sgb_target_build_voxelmaps(sgb_ctx* ctx, size_t n_maps, const size_t* offsets, const double* points_xyz1, const double* covs_4x4 /*or NULL*/,
                               double leaf_size, int search_offsets);
/* n_maps point clouds, each with its own kd-tree, as ONE target for the batched calls only (member m is aligned against map m; see the
 * batch section).  offsets, points, normals and covariances as for sgb_target_build_voxelmaps (host, page-locked or device memory; empty
 * maps allowed).  Map m is stored as sgb_target_set_points + sgb_target_build_kdtree would store it alone: FP32 about the box centre of
 * its own points, leaves of at most 32 points cut by median splits along the widest axis; a member can only ever match its own map's
 * points.  The launch count depends on the size of the largest map only, never on n_maps, and there is no host synchronisation.
 * n_maps <= SGB_BATCH_MAX_MEMBERS and fewer than 2^30 points in all, else the call fails with a message. */
int sgb_target_build_kdtrees(sgb_ctx* ctx, size_t n_maps, const size_t* offsets, const double* points_xyz1, const double* normals_xyz0 /*or NULL*/,
                             const double* covs_4x4 /*or NULL*/);
/* k nearest neighbours (1 <= k <= 32) of arbitrary query points in the target's kd-tree: replaces KdTree::knn_search /
 * nearest_neighbor_search (ann/kdtree.hpp:165-189,254-274) and the batch_knn_search / batch_nearest_neighbor_search of the
 * Python binding (src/python/kdtree.cpp).  out_indices / out_sq_dists: n_queries x k, original target indices.  The distance reported
 * and ranked is the FP64 squared distance between the target point as stored (centred on the target's box, rounded to FP32) and the
 * FP64 query; rows are non-decreasing in it.  The search itself runs in FP32 and keeps 4 spare candidates, so the set is the exact k
 * nearest except among points within ~2e-6 relative of the k-th distance.  UINT64_MAX / DBL_MAX pad when the target has fewer than k
 * points (knn_result.hpp:60-66).  It needs a point target with its tree and fails with a message on any other target, many maps and
 * many kd-trees included: sgb_target_batch_knn_maps / _submaps below query those. */
int sgb_target_batch_knn(sgb_ctx* ctx, size_t n_queries, const double* queries_xyz1, int k, uint64_t* out_indices, double* out_sq_dists);
/* k nearest neighbours of query SETS, each in one map of the target: a keyframe database's overlap and chamfer checks without rebuilding
 * any map as a target of its own.  Conventions of both query-set calls: k in 1..32; query_offsets has n_sets + 1 ascending entries from 0,
 * set s = queries query_offsets[s] .. query_offsets[s+1] - 1 of queries_xyz1 (N x 4 doubles (x, y, z, 1), N = query_offsets[n_sets]);
 * out_indices / out_sq_dists: N x k, each row non-decreasing in the reported FP64 squared distance, UINT64_MAX / DBL_MAX padding where
 * fewer than k neighbours exist.  Queries and outputs in host, page-locked or device memory; index arrays and poses in host memory.
 * n_sets <= SGB_BATCH_MAX_MEMBERS and fewer than 2^31 / k queries in all, else the call fails with a message.  One search launch
 * whatever the set, map or entry counts, plus the copies, and one host synchronisation.  Neither call changes the target, the source,
 * a batch, a pairing or submap lists, seeds or the cached linearisation.
 * Set s is searched in map maps[s] (maps == NULL: map s, which needs n_sets == the map count), its queries given in the frame in which
 * that map's points were given.  Many kd-trees (sgb_target_build_kdtrees): the k nearest points of the map as sgb_target_batch_knn finds
 * them in a context holding that map alone (the query centred on the map's own centre, FP32 search with 4 spare candidates, the FP64
 * distance to the stored point reported and ranked); index = original index within the map.  The one kd-tree: map 0, bit for bit
 * sgb_target_batch_knn.  Many voxel maps (sgb_target_build_voxelmaps) or the one voxel map (map 0): IncrementalVoxelMap::knn_search
 * (incremental_voxelmap.hpp:99-148): the means of the query's voxel (floor(q / leaf_size)) and of its other search_offsets - 1 offset
 * voxels, ranked by the FP64 distance to the stored mean, the first found winning exact ties; at most search_offsets voxels per row;
 * index = voxel id within the map << 32, as correspondences report it.  Any other target, or a maps[s] beyond the map count, fails with
 * a message. */
int sgb_target_batch_knn_maps(sgb_ctx* ctx, size_t n_sets, const size_t* query_offsets, const uint32_t* maps /*or NULL*/, const double* queries_xyz1, int k,
                              uint64_t* out_indices, double* out_sq_dists);
/* k nearest neighbours of query sets, each in the UNION of posed maps of a many-kd-trees target: set s against entries list_off[s] ..
 * list_off[s+1] - 1, entry j = map entry_maps[j] placed by the rigid pose entry_poses16[16 j ..] (map -> common frame, column-major;
 * NULL = identity), the lists meaning exactly what they mean in sgb_source_set_submaps; queries in the common frame.  Nothing of a map is
 * transformed: per entry the FP64 query is carried into the map's stored frame (P_j^-1 q), centred on the map and its tree walked in
 * FP32, one candidate list of k + 4 carried from entry to entry; the candidates are then ranked by the FP64 distance, each in its own
 * entry's frame, an exact tie going to the earlier entry.  index = (entry within the set's list) << 32 | original index within the map.
 * A map listed twice holds two copies of its points (both can appear in one row); an empty list gives a padded row.  A one-entry
 * identity list is sgb_target_batch_knn_maps on that map, bit for bit.  Conventions and limits of sgb_target_batch_knn_maps, fewer than
 * 2^31 entries, every pose rigid (as for sgb_source_set_submaps), every map in range, a many-kd-trees target (voxel maps fail), else the
 * call fails with a message. */
int sgb_target_batch_knn_submaps(sgb_ctx* ctx, size_t n_sets, const size_t* query_offsets, const size_t* list_off, const uint32_t* entry_maps,
                                 const double* entry_poses16 /*or NULL*/, const double* queries_xyz1, int k, uint64_t* out_indices, double* out_sq_dists);
size_t sgb_target_size(const sgb_ctx* ctx);

/* ---- source: replaces traits::point/cov(source, i) ------------------------------------------- */
int sgb_source_set_points(sgb_ctx* ctx, size_t n, const double* points_xyz1, const double* covs_4x4 /*or NULL*/);
size_t sgb_source_size(const sgb_ctx* ctx);

/* ---- the hot path ------------------------------------------------------------------------------
 * sgb_linearize replaces {Serial,ParallelReductionOMP,ParallelReductionTBB}::linearize
 * (registration/reduction.hpp:20-47, reduction_omp.hpp:24-59, reduction_tbb.hpp:117-131): for every
 * source point transform -> nearest neighbour -> reject -> factor -> sum.  out_Hbe = H(36) | b(6) | e(1).
 * The correspondences (and, for GICP, the linearisation pose from which the fused precision matrix is
 * re-derived) stay cached in the context for sgb_error(), as the reference caches them in its factor
 * vector (gicp_factor.hpp:94-96). */
int sgb_linearize(sgb_ctx* ctx, int factor_kind, int robust_kind, double robust_c, int rejector_kind, double max_dist_sq,
                  const double* T_colmajor16, double* out_Hbe43);
/* replaces {...}::error (reduction.hpp:55-62, reduction_omp.hpp:61-70, reduction_tbb.hpp:133-138):
 * sum of factor errors at a trial pose with the cached correspondences (no new search). */
int sgb_error(sgb_ctx* ctx, const double* T_colmajor16, double* out_e);
/* Same, but asynchronous on the context's stream with the result left in DEVICE memory
 * (d_out44 = H|b|e|num_inliers as doubles; d_out1 = e) -- for multi-GPU all-reduce without a host hop. */
int sgb_linearize_device(sgb_ctx* ctx, int factor_kind, int robust_kind, double robust_c, int rejector_kind, double max_dist_sq,
                         const double* T_colmajor16, double* d_out44);
int sgb_error_device(sgb_ctx* ctx, const double* T_colmajor16, double* d_out1);

/* Forget the correspondences of the previous linearize as search seeds: the next sgb_linearize searches like the first iteration of a
 * fresh align() (the seeds only ever prune -- results are identical with or without them; this exists so that a benchmark can time an
 * unseeded first iteration without re-uploading the source). */
int sgb_drop_seeds(sgb_ctx* ctx);

/* factors[i].target_index of the last linearize, in the caller's source order
 * (SGB_NO_CORRESPONDENCE = rejected; icp_factor.hpp:66-69). */
int sgb_correspondences(sgb_ctx* ctx, uint64_t* target_index);
/* count_if(factors, inlier()) of the last linearize (registration/optimizer.hpp:60,146). */
int sgb_num_inliers(sgb_ctx* ctx, size_t* n);

/* ---- batched registration: many sources against the one target, each at its own pose --------------
 * The context holds EITHER one source (sgb_source_set_points) OR a batch of sources ("members"); each setter replaces the other.
 * While a batch is set, sgb_linearize, sgb_error, sgb_correspondences, sgb_num_inliers and the _device variants fail with a
 * message, and the _batch calls fail while a single source is set.  The batch calls are single-GPU: they fail while
 * sgb_comm_connect* is active.  Every member is stored exactly as sgb_source_set_points would store it alone (centred on its own
 * box, FP32, its own curve order), and its results -- H | b | e | inliers, error(), correspondences -- are bit-identical whatever
 * else is in the batch, wherever it sits and whichever other members are inactive, EXCEPT at exact FP32 distance ties between two
 * target points: the search returns an exact nearest neighbour, but which of two equidistant ones it returns depends on the
 * traversal, and that may depend on the other queries of a 32-query chunk (members are not padded to chunks) and on the batch's
 * total pending count.  sgb_drop_seeds applies to every member.
 * The upload is batched: sgb_source_set_batch stores all clouds in 6 launches whatever their count (with or without covariances),
 * each bit-identical to sgb_source_set_points of that cloud alone.
 * Many targets: after sgb_target_build_voxelmaps, member m is paired with map m -- sgb_linearize_batch, sgb_error_batch,
 * sgb_align_batch and sgb_correspondences_batch work as against one voxel map (same launches per round), and fail with a message while
 * the member count differs from the map count.  Each member's results are bit-identical to a context holding its map alone and that
 * member as a batch of one; its correspondences are voxel ids within its own map (id << 32).  On such a target the single-source calls
 * (sgb_linearize, sgb_error, their _device variants, sgb_correspondences, sgb_num_inliers) and sgb_target_batch_knn,
 * sgb_target_estimate_features, sgb_target_set_kdtree / _build_kdtree fail with a message (sgb_target_batch_knn_maps queries the maps).
 * Pair one source with many maps, many
 * sources with one map, or a cloud with several initial poses through sgb_source_set_pairs below: each cloud is stored once and
 * each map built once.  A source against the union of several posed kd-tree maps: sgb_source_set_submaps.
 * Many kd-trees: after sgb_target_build_kdtrees, member m is paired with map m in the same way, for ICP, point-to-plane (the maps need
 * normals) and GICP (covariances).  A linearize round is 3 launches (search, factor, per-member sums) and an error round 2, whatever the
 * member count.  The calls fail with a message while the member count differs from the map count.  Each member's results are
 * bit-identical to a context holding its map alone (sgb_target_set_points + sgb_target_build_kdtree) and that member as a batch of one,
 * except at exact FP32 distance ties; and they are bit-identical whatever else is in the batch INCLUDING at exact ties, since a member is
 * searched by warps of its own points only.  Its correspondences are original indices within its own map.  sgb_target_size returns
 * the total point count.  On such a target the single-source calls (sgb_linearize, sgb_error, their _device variants,
 * sgb_correspondences, sgb_num_inliers), sgb_target_batch_knn, sgb_target_estimate_features, sgb_target_set_kdtree / _build_kdtree
 * and sgb_target_adopt_source fail with a message (sgb_target_batch_knn_maps / _submaps query the maps and unions of them). */
#define SGB_BATCH_MAX_MEMBERS 65536
/* offsets: n_members + 1 ascending entries, offsets[0] = 0; member m = points offsets[m] .. offsets[m+1] (empty members allowed).
 * points / covariances: all members concatenated, in the layouts above (host, page-locked or device memory). */
int sgb_source_set_batch(sgb_ctx* ctx, size_t n_members, const size_t* offsets, const double* points_xyz1, const double* covs_4x4 /*or NULL*/);
/* The batch's members become n_members (cloud, map) pairs drawn from the clouds of the last sgb_source_set_batch: member p is a copy of
 * cloud clouds[p] as stored (or cloud p when clouds == NULL, which needs n_members == the cloud count), aligned against map maps[p] of a
 * many-maps / many-kd-trees target (maps == NULL: against map p, or the one target; S copies of a cloud against one target are S
 * starts).  Index arrays in host memory.  No upload, no re-sort: 1 launch whatever n_members is, plus 1 at the first batched call after
 * the pairing or the target changed (the maps seen through the pairing).  Afterwards sgb_linearize_batch, sgb_error_batch,
 * sgb_align_batch, sgb_correspondences_batch and sgb_drop_seeds work on the pair members (poses, outputs and correspondences per member,
 * in pair order; correspondences in its cloud's original order), each bit-identical to that cloud uploaded again as a member paired
 * with that map; the per-member state starts afresh as after sgb_source_set_batch.  Calling it again re-pairs the same clouds;
 * sgb_source_set_batch or sgb_source_set_points forgets the pairing.  Every batched call checks maps against the current target: a
 * maps[p] beyond its map count, or a maps table with a target that is not many maps or many kd-trees, fails with a message (without a
 * maps table the member count must equal the map count, as without pairs).  n_members <= SGB_BATCH_MAX_MEMBERS, fewer than 2^31 member
 * points in all, every clouds[p] below the cloud count, a batch set, else the call fails with a message; n_members = 0: an empty batch. */
int sgb_source_set_pairs(sgb_ctx* ctx, size_t n_members, const uint32_t* clouds /*or NULL*/, const uint32_t* maps /*or NULL*/);
/* Submaps: the batch's members become n_members (cloud, submap) pairs.  Member p = stored cloud clouds[p] (NULL: cloud p) against the UNION
 * of its entries j = list_off[p] .. list_off[p+1] - 1 (list_off: n_members + 1 ascending, list_off[0] = 0): entry j = map entry_maps[j] of a
 * many-kd-trees target (sgb_target_build_kdtrees), placed by the rigid pose entry_poses16[16 j ..] (map -> common frame, column-major
 * 4x4; NULL = all identity).  A scan against a local map of several keyframes each at its own pose, or against the few tiles of a tiled
 * map around it, without building or storing a tree of the union: every map is built once, whatever lists name it and however often the
 * poses change.  Nothing of a map is transformed.  Rigid motions preserve distances, so the nearest neighbour in the placed union is the
 * nearest over the entries of the nearest in each map's own frame at the member's pose carried into that frame (P_j^-1 T), and the ICP and
 * GICP terms r^T (C_t + R C_s R^T)^-1 r with their derivatives by the right perturbation of T are the same in either frame: each point
 * is linearised against its correspondence's map as stored.  Point-to-plane is not (the reference's residual is the element-wise n o r):
 * SGB_FACTOR_PLANE_ICP fails with a message.  The poses, init_T16xB and out_T16xB of the batched calls are source -> common frame.
 * It is a pairing like sgb_source_set_pairs: index arrays and poses in host memory, one copy of the lists and 1 launch whatever the
 * counts, plus 1 at the first batched call after it or after the target changed; the per-member state starts afresh; calling it again
 * re-pairs or changes the poses: no map is rebuilt and no cloud uploaded, but the call is a full pairing even if only poses changed
 * (the replicas are gathered again, 1 launch over all member points, and every member's cached correspondences and seeds are dropped);
 * sgb_source_set_batch, sgb_source_set_pairs or sgb_source_set_points forgets it.
 * A linearize round stays 3 launches and an error round 2.  The same map may appear in many lists and, at different poses, several times
 * in one; an empty list gives the member no correspondences and zero sums.  At an exact FP32 distance tie between two entries the earlier
 * entry wins (a search seed aside, as in one tree); a member's results depend on its own points, pose, list and seeds only.
 * sgb_correspondences_batch reports (entry index within the member's list) << 32 | original index within that entry's map.  Every batched
 * call checks the lists against the current target: a target that is not many kd-trees (voxel maps included), or an entry_maps[j] beyond
 * its map count, fails with a message.  Limits of sgb_source_set_pairs, fewer than 2^31 entries in all, and every pose rigid (rotation
 * block orthonormal to 1e-6, determinant > 0, last row 0 0 0 1), else the call fails with a message. */
int sgb_source_set_submaps(sgb_ctx* ctx, size_t n_members, const uint32_t* clouds /*or NULL*/, const size_t* list_off, const uint32_t* entry_maps,
                           const double* entry_poses16 /*or NULL*/);
/* One linearize per member at its pose T_colmajor16xB[16 m ..]: out44xB[44 m ..] = H(36) | b(6) | e | num_inliers.  active (or NULL =
 * all): an inactive member costs no search or factor work, gets zeros and keeps its cached correspondences and linearisation pose.
 * out44xB may be host or device memory; the call returns when the results are there. */
int sgb_linearize_batch(sgb_ctx* ctx, int factor_kind, int robust_kind, double robust_c, int rejector_kind, double max_dist_sq,
                        const double* T_colmajor16xB, const uint8_t* active /*or NULL*/, double* out44xB);
/* error() of every active member at its trial pose with its cached correspondences; GICP precision matrices re-derived from THAT
 * member's last linearisation pose.  Inactive members: 0. */
int sgb_error_batch(sgb_ctx* ctx, const double* T_colmajor16xB, const uint8_t* active /*or NULL*/, double* out_e);
/* Correspondences of every member's last linearize, concatenated in the caller's order (offsets of sgb_source_set_batch), original
 * target indices; SGB_NO_CORRESPONDENCE = rejected or never linearised. */
int sgb_correspondences_batch(sgb_ctx* ctx, uint64_t* out);
/* Per-point terms: sgb_linearize_batch / sgb_error_batch that also return every source point's share of its member's sums, e.g. to flag
 * points whose error stays large after an align, to score an alignment per member, or to weight the points in a solver of one's own.
 *   - Each call does exactly what the plain call does (search, correspondences, seeds, cached linearisation and the state it leaves) and
 *     out44xB / out_e are bit-identical to it.  sgb_kernel_launches counts the same launches: the factor kernel writes the rows itself.
 *   - One row per source point, in the layout of sgb_correspondences_batch: members concatenated (pair and submap members in the
 *     pairing's member order), each in its cloud's original order.
 *   - out_point_e[i]: the point's share of its member's e.  linearize: w e as RobustFactor::linearize returns it; error(): Factor::error
 *     at the trial pose with the cached correspondence (GICP: the precision matrix of the member's linearisation pose), robust-weighted.
 *   - out_point_Hb42[42 i ..]: the point's H (36, row-major, symmetric) | b (6).  A member's rows add up to its H | b | e.
 *   - Zero rows: rejected points, points without a correspondence, every point of an inactive member, and every point against an
 *     empty target.
 *   - Outputs in host, page-locked or device memory; the call returns when the results are there.  Device memory of the context's GPU is
 *     written by the kernel directly, any other memory through one copy.
 *   - They fail where the plain calls fail, and also when out_point_e and out_point_Hb42 are both NULL (linearize) or out_point_e is
 *     NULL (error). */
int sgb_linearize_batch_points(sgb_ctx* ctx, int factor_kind, int robust_kind, double robust_c, int rejector_kind, double max_dist_sq,
                               const double* T_colmajor16xB, const uint8_t* active /*or NULL*/, double* out44xB, double* out_point_e /*or NULL*/,
                               double* out_point_Hb42 /*or NULL*/);
int sgb_error_batch_points(sgb_ctx* ctx, const double* T_colmajor16xB, const uint8_t* active /*or NULL*/, double* out_e, double* out_point_e);
/* Per-point weights: the caller's weight w_i on every source point's terms in every batched call, e.g. to suppress points of moving
 * objects flagged by their per-point error, to apply semantic or intensity confidences or overlap masks, or to run IRLS / graduated
 * non-convexity with a robust kernel of one's own (align, read the rows of sgb_error_batch_points, compute weights, align again).
 *   - weights: one double per member point in the row layout of sgb_correspondences_batch and the _points calls (member m's rows are its
 *     offsets' range, in its cloud's original order; pair and submap members in the pairing's member order, so two members of one cloud
 *     may carry different weights).  The count is the batch's point count.  Host, page-locked or device memory of the context's GPU.
 *     NULL clears the weights: the batched calls are unweighted again.
 *   - Meaning: after the factor and the robust kernel, each of a point's terms (H, b and e of a linearize, its error() share) is
 *     multiplied by w_i, one FP64 multiply per term; the robust weight is still computed from the unweighted residual.  The correspondence
 *     search, the rejector and num_inliers do not change: a zero-weight point that has a correspondence still counts as an inlier.  The
 *     rows of the _points calls are the weighted terms, the exact summands of the member sums.  With all weights 1 every result is
 *     bit-identical to an unweighted call.
 *   - Honoured by sgb_linearize_batch, sgb_error_batch, both _points calls, sgb_align_batch, sgb_align_batch_async, sgb_align_joint and
 *     sgb_align_joint_async, against every target kind; not by the single-source calls (sgb_linearize, sgb_error, their _device variants)
 *     nor the k-NN calls.
 *   - Every weight must be finite and >= 0 (-0.0 passes).  The weights are gathered into the stored order and checked in 1 launch, and the
 *     call synchronises once to read the check: a failing weight fails the call with a message naming its row, and the weights in force
 *     stay.  Fails with a message too without a batch and while the context's stream is being captured.  The batched calls never check
 *     again, and keep their launch counts.  Weights set again with the same count keep their device address, so a cached or captured
 *     asynchronous align reads the new ones at its next launch or replay.
 *   - sgb_source_set_batch, sgb_source_set_pairs, sgb_source_set_submaps and sgb_source_set_points clear the weights; target changes and
 *     sgb_drop_seeds keep them. */
int sgb_source_set_weights(sgb_ctx* ctx, const double* weights /*or NULL*/);

/* Batched align(): Registration<Factor, ..., GeneralFactor, Rejector, Optimizer>::align (registration.hpp:17-54, optimizer.hpp:10-158) of
 * every member from its own initial pose, in lockstep.  A round is one sgb_linearize_batch over the members still iterating or, for
 * Levenberg-Marquardt, one sgb_error_batch over the members with a pending trial (until none has one), followed by one kernel in which
 * each member solves its damped 6x6 system, updates its pose, lambda and convergence exactly as the reference's optimizer does, and
 * writes its next pose on the device.  Per round the host reads one byte per member.  A member's results depend only on its own cloud,
 * initial pose and the options (the exact-FP32-tie caveat above applies).  Afterwards sgb_correspondences_batch returns each member's
 * correspondences of its last linearize. */
enum sgb_optimizer_kind { SGB_OPT_GAUSS_NEWTON = 0, SGB_OPT_LEVENBERG_MARQUARDT = 1 };
typedef struct sgb_align_options {
  int factor_kind, robust_kind; /* sgb_factor_kind, sgb_robust_kind */
  double robust_c;
  int rejector_kind; /* sgb_rejector_kind */
  double max_dist_sq;
  int optimizer_kind;       /* sgb_optimizer_kind */
  int max_iterations;       /* 20 */
  double gn_lambda;         /* 1e-6: GaussNewtonOptimizer::lambda */
  int max_inner_iterations; /* 10 */
  double init_lambda, lambda_factor; /* 1e-3, 10 */
  double rotation_eps, translation_eps; /* 0.1 deg [rad], 1e-3 [m]: TerminationCriteria */
  double dof_mask[6]; /* RestrictDoFFactor (rx ry rz tx ty tz; 0 = frozen): H(i,i) += 1e9 |mask_i - 1|.  All 1 = NullFactor */
} sgb_align_options;
/* init_T16xB / out_T16xB: column-major 4x4 per member; inputs and outputs in host memory.  out_info4xB = converged, iterations, num_inliers, error per member;
 * out_Hb42xB (or NULL) = H(36) | b(6) per member (RegistrationResult).  max_iterations <= 0 returns the initial poses, not converged. */
int sgb_align_batch(sgb_ctx* ctx, const sgb_align_options* options, const double* init_T16xB, double* out_T16xB, double* out_info4xB,
                    double* out_Hb42xB /*or NULL*/);
/* Graduated non-convexity (GNC; Yang, Antonante, Tzoumas, Carlone, RA-L 2020): outlier-robust batched align, for moving objects, partial
 * overlap, clutter or wrong loop-closure candidates, where a fixed-width robust kernel breaks down.  Each member alternates a weighted
 * sgb_align_batch with a closed-form update of its per-point weights, annealing a surrogate of the Geman-McClure or truncated-least-squares
 * cost from convex to the true cost; the weights stay on the device.  Per member, stage s (s = 0, 1, ...) from its current pose T_s (T_0 =
 * its initial pose):
 *   1. Reweighting linearize: one unweighted linearize at T_s with the options' factor and rejector and no robust kernel.  A point with a
 *      correspondence has r_i^2 = 2 e_i (e_i: its row of sgb_linearize_batch_points without weights; c^2 is on this scale: ICP m^2, GICP
 *      Mahalanobis); a point without one gets g_i = 0 for the stage.
 *   2. Stage 0: r_max^2 = the member's largest r_i^2 (0 without any).  GM: mu = 2 r_max^2 / c^2, or 1 if that is <= 1.  TLS: if
 *      2 r_max^2 <= c^2 the member has no outliers: every point with a correspondence gets g_i = 1, this stage is its last, and its mu is
 *      reported as 0; else mu = c^2 / (2 r_max^2 - c^2).  Later stages: GM mu = max(mu / 1.4, 1), TLS mu = 1.4 mu.
 *   3. Weights: GM g = (mu c^2 / (r^2 + mu c^2))^2; TLS g = 1 if r^2 <= mu / (mu + 1) c^2, 0 if r^2 >= (mu + 1) / mu c^2, else
 *      c / r sqrt(mu (mu + 1)) - mu (clamped to [0, 1]).  The stage's align uses w_i g_i, w_i = the weight in force (1 without).  Every
 *      formula is FP64 with a fixed operation order and no contraction (sgb_math.cuh): numpy reproduces every bit.
 *   4. The stage is the member's last when GM's mu is 1, when TLS's weights are all binary (every g in {0, 1}), or at s = max_stages - 1.
 *   5. Weighted align: sgb_align_batch's algorithm from T_s (a fresh start, the options as given) with the stage's weights and max_iterations
 *      = stage_iterations, or options->max_iterations at the last stage; its result is T_{s+1}.
 * Outputs (host memory; out_point_w may also be device memory of the context's GPU): T, H | b and info of the last stage's align (converged,
 * iterations summed over all stages, inliers and the weighted error), out_gnc2xB = the stages run and the last stage's mu, out_point_w =
 * each point's final g (without the weights in force) in the row layout of sgb_correspondences_batch.  Each member's results are
 * bit-identical to this loop driven from the host on a context holding that member alone: sgb_source_set_weights(NULL),
 * sgb_linearize_batch_points, the formulas, sgb_source_set_weights(w * g), sgb_align_batch (the exact-FP32-tie caveat above applies).
 * Afterwards the context is as sgb_align_batch leaves it after each member's last stage (sgb_correspondences_batch, sgb_error_batch), and
 * the weights in force are unchanged: the stage weights live in a buffer of the call.
 * The call runs sgb_align_batch_gnc_async on its poses and outputs staged in device memory: every stage and round on the device, one
 * upload of the poses, one copy of the outputs and one host synchronisation per call.  So it needs conditional graph nodes (CUDA 12.4 or
 * later, driver included) as that call does, and keeps the device's seed flags as it does (a call after they were cleared starts
 * unseeded; the exact-FP32-tie caveat above applies).  sgb_kernel_launches counts 4 per call (initial state, one launch of the graph, two
 * for the outputs), whatever the stage and round counts, plus 1 when the pairing's view of the target is rebuilt.
 * Fails with a message, enqueuing nothing, for robust_kind != SGB_ROBUST_NONE (the GNC weights are the robust kernel), an invalid kind,
 * noise_bound_sq not finite or <= 0, max_stages < 1, stage_iterations < 1, while the context's stream is being captured (the call
 * synchronises), and for everything sgb_align_batch refuses. */
enum sgb_gnc_kind { SGB_GNC_GEMAN_MCCLURE = 0, SGB_GNC_TLS = 1 };
typedef struct sgb_gnc_options {
  int kind;               /* sgb_gnc_kind */
  double noise_bound_sq;  /* c^2, on the factor's own r^2 = 2 e scale (ICP: m^2; GICP: Mahalanobis) */
  int max_stages;         /* hard bound on the stage count, >= 1 */
  int stage_iterations;   /* max_iterations of every stage but the last (>= 1); the last uses options->max_iterations */
} sgb_gnc_options;
int sgb_align_batch_gnc(sgb_ctx* ctx, const sgb_align_options* options, const sgb_gnc_options* gnc, const double* init_T16xB, double* out_T16xB,
                        double* out_info4xB, double* out_Hb42xB /*or NULL*/, double* out_gnc2xB /*or NULL*/, double* out_point_w /*or NULL*/);
/* Joint window registration: every frame pose of a window of scans solved against all the window's pairwise edges at once, many windows
 * per call.  Frame k is cloud k of the last sgb_source_set_batch with map k of a many-kd-trees or many-voxel-maps target, both in frame k's
 * own coordinates (cloud count == map count).  The edges are the members of the pairing of sgb_source_set_pairs with a maps table: member
 * p is the edge "cloud clouds[p] against map maps[p]" (clouds[p] != maps[p]).  Windows partition the frames: window_off has n_windows + 1
 * ascending entries from 0 to the frame count, at most 32 frames per window; both frames of an edge lie in one window.  fixed[k] = 1 holds
 * frame k at its initial pose (NULL: the first frame of each window); a window with an edge needs a fixed frame.
 *   - Each window minimises E(X) = sum over its edges (i, j) of the factor error of the edge at T_e = X_j^-1 X_i (factor, robust kernel and
 *     rejector of the options).  With the right perturbations X <- X exp(delta), delta_e = delta_i + A_e delta_j, A_e = -Ad(T_e^-1), and
 *     the window's system over its free frames is assembled from the edges' H | b (H_ii += H_e, H_ij += H_e A_e, H_jj += A_e^T H_e A_e,
 *     b_i += b_e, b_j += A_e^T b_e, in member order), plus 1e9 |mask - 1| on every free frame's diagonal.  The step (H + lambda I) delta = -b
 *     updates every free frame at once: Gauss-Newton with gn_lambda, or Levenberg-Marquardt with the reference's lambda schedule on the
 *     window's summed error().  Converged: the termination criteria hold for every free frame's step.
 *   - init_X16xK / out_X16xK: column-major 4x4 per frame, host memory; fixed frames come back bit for bit.  out_info4xW: per window
 *     converged, iterations, num_inliers, error (both summed over its edges), as sgb_align_batch's per member.  A window without an edge or
 *     without a free frame returns its initial poses, not converged, 0 iterations; a free frame without an edge stays put.
 *   - Rounds as sgb_align_batch's, per window: a round is the pairs round of the active edges (those of the windows in that round's phase)
 *     plus one joint_step_kernel launch, whatever the counts of windows, frames and edges; plus 1 set-up launch for the initial edge poses
 *     (and 1 when the pairing's view of the target is rebuilt).  The context is left as sgb_align_batch leaves it: sgb_correspondences_batch
 *     gives each edge's correspondences of its last linearize, and the batched calls work on the edges afterwards.
 *   - Fails with a message, the context still usable, on: no batch, no pairing with a maps table or a submap pairing, a target that is not
 *     many maps, cloud count != map count, a self-edge, an edge across windows, a window with edges but no fixed frame, a window of more than
 *     32 frames, window_off not ascending from 0 to the frame count, more than SGB_BATCH_MAX_MEMBERS windows, and wherever sgb_align_batch
 *     fails. */
int sgb_align_joint(sgb_ctx* ctx, const sgb_align_options* options, size_t n_windows, const size_t* window_off, const uint8_t* fixed /*or NULL*/,
                    const double* init_X16xK, double* out_X16xK, double* out_info4xW);
/* The edge poses sgb_align_joint linearises at: per member p of the pairing (in member order), T_p = X_j^-1 X_i for its cloud i and map
 * j, column-major 4x4 into out_T16xE, computed on the device by the joint align's own kernel and tables, so its bits are those of the
 * poses the joint align and sgb_align_joint_gnc use (a host X_j^-1 X_i differs in the last bits).  The layout of the poses that
 * sgb_linearize_batch_points takes.  X16xK and out_T16xE are host memory.  Checks and messages as sgb_align_joint's for the windows and
 * the pairing (fixed frames do not enter); no pairing member: nothing to do.  1 launch. */
int sgb_joint_edge_poses(sgb_ctx* ctx, size_t n_windows, const size_t* window_off, const double* X16xK, double* out_T16xE);
/* Graduated non-convexity for joint windows: sgb_align_batch_gnc's stages with the window as the GNC unit, one mu annealing the window's
 * whole objective.  Frames, windows, fixed flags, edges, targets and options as sgb_align_joint; gnc as sgb_align_batch_gnc.  Per window,
 * stage s (s = 0, 1, ...) from its frames X_s (X_0 = init_X16xK):
 *   1. Edge poses: every edge's T_e from X_s (sgb_joint_edge_poses' bits).
 *   2. Reweighting linearize: one unweighted linearize of the window's edges at those poses, the options' factor and rejector, no robust
 *      kernel.  A point with a correspondence has r_i^2 = 2 e_i; one without gets g_i = 0 for the stage.
 *   3. Stage 0: r_max^2 = the largest r_i^2 over all the window's edges; mu_0 from it as in sgb_align_batch_gnc (TLS without outliers,
 *      2 r_max^2 <= c^2, per window).  Later stages: the schedule's next mu.
 *   4. Weights g_i of sgb_align_batch_gnc's formulas with the window's mu; the stage's align uses w_i g_i (w_i: the weight in force).
 *   5. The stage is the window's last when GM's mu is 1, when TLS's weights are all binary over the whole window or it has no outliers, or
 *      at s = max_stages - 1.
 *   6. Joint align: sgb_align_joint's algorithm from X_s (a fresh start, lambda = init_lambda) with the stage's weights and max_iterations
 *      = stage_iterations, or options->max_iterations at the last stage; its frames are X_{s+1}.
 * Outputs (host memory; out_point_w may also be device memory of the context's GPU): out_X16xK the frames after the last stage (fixed
 * frames bit for bit); out_info4xW per window converged, iterations summed over all stages, inliers and weighted error (summed over its
 * edges) of the last stage; out_gnc2xW the stages run and the last mu; out_point_w each edge point's final g (without the weights in
 * force) in the row layout of sgb_correspondences_batch.  Each window's results are bit-identical to this loop driven from the host on a
 * context holding that window alone: sgb_source_set_weights(NULL), sgb_joint_edge_poses, sgb_linearize_batch_points at those poses (no
 * robust kernel), the formulas, sgb_source_set_weights(w * g), sgb_align_joint (the exact-FP32-tie caveat above applies).  A window with
 * no edge, which no such context can hold, returns its initial poses, not converged, 0 iterations, and the stage count and mu of r_max^2 =
 * 0 (GM: 1 stage, mu 1; TLS: 1 stage, mu 0).  Afterwards the context is as sgb_align_joint leaves it after each window's last stage
 * (sgb_correspondences_batch, sgb_error_batch on the edges), and the weights in force are unchanged.
 * The call runs sgb_align_joint_gnc_async on its frames and outputs staged in device memory, with window tables of its own (uploaded at
 * every call, never those the asynchronous calls cache): every stage and joint round on the device, one copy of the outputs and one host
 * synchronisation per call.  So it needs conditional graph nodes (CUDA 12.4 or later, driver included) as that call does, and keeps the
 * device's seed flags as it does (the exact-FP32-tie caveat above applies).  sgb_kernel_launches counts 3 per call with at least one
 * edge (one launch of the graph, two for the outputs) and 4 without (the stage kernels of the one stage, two for the outputs), whatever
 * the stage and round counts, plus 1 when the pairing's view of the target is rebuilt.
 * Fails with a message, enqueuing nothing, where sgb_align_batch_gnc refuses its GNC options (robust_kind != SGB_ROBUST_NONE, an invalid
 * kind, noise_bound_sq not finite or <= 0, max_stages < 1, stage_iterations < 1), while the context's stream is being captured, and for
 * everything sgb_align_joint refuses. */
int sgb_align_joint_gnc(sgb_ctx* ctx, const sgb_align_options* options, const sgb_gnc_options* gnc, size_t n_windows, const size_t* window_off,
                        const uint8_t* fixed /*or NULL*/, const double* init_X16xK, double* out_X16xK, double* out_info4xW, double* out_gnc2xW /*or NULL*/,
                        double* out_point_w /*or NULL*/);
/* sgb_align_batch enqueued on the context's stream (sgb_set_stream) with no host involvement after the call: the rounds are planned on
 * the device and driven by a CUDA graph whose conditional WHILE node repeats one round (planner, search, factor, per-member sums, step)
 * until no member has a round to go.  No host synchronisation, no device-to-host copy, no upload from pageable memory: the call returns
 * once the work is enqueued, and a torch op (or any work) queued after it on the same stream sees the results.
 *   - Inputs and outputs as sgb_align_batch (same layouts), but all of them device memory of the context's GPU; host, page-locked or
 *     managed pointers fail with a message and nothing is enqueued.  Per member, T, info and H | b are bit-identical to sgb_align_batch with
 *     the same options, poses, batch, pairing or submap lists and target, and the context is left as sgb_align_batch leaves it
 *     (sgb_correspondences_batch, sgb_error_batch and sgb_linearize_batch behave alike afterwards).
 *   - It fails with a message where sgb_align_batch does (no batch, connected comm, invalid kinds, point-to-plane on submaps, missing
 *     normals or covariances), and where the driver has no conditional graph nodes.  Errors of the enqueued work surface at the next
 *     synchronising call of the context (as for sgb_linearize_device).
 *   - While the context's stream is being captured (cudaStreamIsCapturing, e.g. inside torch.cuda.graph) the align is added to the
 *     capture instead: each replay re-runs it from what d_init_T16xB holds at replay time.  The captured work is only valid while the
 *     context's batch, pairing, target and buffers are those of the capture; call it once outside the capture first (the first batched
 *     call of a context allocates).  Outside a capture the loop's instantiated graph is cached in the context and rebuilt when the options,
 *     the batch, the pairing, the target or any buffer it uses changes.
 *   - sgb_kernel_launches counts 3 per call with max_iterations > 0 (initial state, one launch of the loop graph, outputs) and 2 without,
 *     whatever the round count, plus 1 when the pairing's view of the target is rebuilt (as for sgb_align_batch); captured work counts
 *     the same at capture and nothing at replay. */
int sgb_align_batch_async(sgb_ctx* ctx, const sgb_align_options* options, const double* d_init_T16xB, double* d_out_T16xB, double* d_out_info4xB,
                          double* d_out_Hb42xB /*or NULL*/);
/* sgb_align_joint enqueued on the context's stream with no host involvement after the call, as sgb_align_batch_async enqueues
 * sgb_align_batch: the edges are the members of the device loop's rounds, each edge's phase its window's, and one joint step per round
 * (one CTA per window) writes the windows' new phases to their edges and keeps the loop running while a window has a round to go.
 *   - Arguments, checks, messages and results as sgb_align_joint: for the same inputs out_X16xK and out_info4xW are bit-identical to it,
 *     fixed frames come back bit for bit from d_init_X16xK, and the context is left as sgb_align_joint leaves it (sgb_correspondences_batch,
 *     sgb_error_batch and sgb_linearize_batch on the edges afterwards).  window_off and fixed are host memory, read during the call; poses
 *     and outputs are device memory of the context's GPU (host, page-locked or managed pointers fail with a message, nothing enqueued).
 *   - The window tables built from window_off, fixed and the pairing are cached in the context, apart from sgb_align_joint's: a call whose
 *     tables are unchanged uploads nothing; one whose tables changed uploads them once.
 *   - While the context's stream is being captured the align is added to the capture (each replay re-runs it from what d_init_X16xK holds
 *     then); a call that would have to allocate or to upload its window tables fails with a message instead: call it once outside the
 *     capture first.  The captured work is only valid while the context's batch, pairing, target, windows and fixed flags are those of
 *     the capture.  Outside a capture the loop's instantiated graph is cached and rebuilt when anything it captured changes.
 *   - sgb_kernel_launches counts 3 per call with max_iterations > 0 and at least one edge (initial state, one launch of the loop graph,
 *     outputs) and 2 otherwise, whatever the round count, plus 1 when the pairing's view of the target is rebuilt; captured work counts at
 *     capture, not at replay.  A call with no window enqueues nothing. */
int sgb_align_joint_async(sgb_ctx* ctx, const sgb_align_options* options, size_t n_windows, const size_t* window_off, const uint8_t* fixed /*or NULL*/,
                          const double* d_init_X16xK, double* d_out_X16xK, double* d_out_info4xW);
/* sgb_align_batch_gnc enqueued on the context's stream with no host involvement after the call, as sgb_align_batch_async enqueues
 * sgb_align_batch: a CUDA graph whose outer WHILE node runs one GNC stage per iteration (the reweighting linearize of the members still
 * in GNC, planned on the device; the stage's mu, weights and align_init) and whose body holds an inner WHILE node repeating the stage's
 * align rounds (planner, search, factor with the stage's weights, per-member sums, step) until no member has a round to go.  Members run
 * their stages in lockstep in sgb_align_batch_gnc's order.
 *   - Arguments, checks, messages and results as sgb_align_batch_gnc, except that every pose and output is device memory of the context's
 *     GPU (host, page-locked or managed pointers fail with a message, nothing enqueued).  For the same inputs T, info, H | b, gnc2 and
 *     out_point_w are bit-identical to it, the context is left as it leaves it (sgb_correspondences_batch, sgb_error_batch and
 *     sgb_linearize_batch behave alike afterwards), and the weights in force are unchanged.  Errors of the enqueued work surface at the next
 *     synchronising call of the context.
 *   - While the context's stream is being captured the whole GNC is added to the capture: each replay re-runs it from what d_init_T16xB
 *     and the weights in force hold at replay time.  A call that would have to allocate (the GNC buffers for the batch, the first batched
 *     call's search queue, the capture streams) fails with a message instead: call it once outside the capture first.  The captured work
 *     is only valid while the context's batch, pairing, target and buffers are those of the capture.  Outside a capture the instantiated
 *     graph is cached in the context and rebuilt when the align or GNC options, the batch, the pairing, the target or any buffer it uses
 *     changes.
 *   - sgb_kernel_launches counts 4 per call (initial state, one launch of the graph, two for the outputs), whatever the stage and round
 *     counts, plus 1 when the pairing's view of the target is rebuilt; captured work counts at capture, not at replay. */
int sgb_align_batch_gnc_async(sgb_ctx* ctx, const sgb_align_options* options, const sgb_gnc_options* gnc, const double* d_init_T16xB, double* d_out_T16xB,
                              double* d_out_info4xB, double* d_out_Hb42xB /*or NULL*/, double* d_out_gnc2xB /*or NULL*/, double* d_out_point_w /*or NULL*/);
/* sgb_align_joint_gnc enqueued on the context's stream with no host involvement after the call, as sgb_align_batch_gnc_async enqueues
 * sgb_align_batch_gnc: a CUDA graph whose outer WHILE node runs one GNC stage per iteration (every edge's pose from its window's X, the
 * reweighting linearize of the edges of the windows still in GNC, planned on the device; the stage's mu, weights and joint_init per
 * window) and whose body holds an inner WHILE node repeating the stage's joint rounds (planner, search, factor with the stage's weights,
 * per-edge sums, one joint step per window) until no window has a round to go.  Windows run their stages in lockstep in
 * sgb_align_joint_gnc's order.
 *   - Arguments, checks, messages and results as sgb_align_joint_gnc, except that the poses and every output are device memory of the
 *     context's GPU (host, page-locked or managed pointers fail with a message, nothing enqueued); window_off and fixed are host memory,
 *     read during the call.  For the same inputs X, info, gnc2 and out_point_w are bit-identical to it (a window with no edge, and a call
 *     with no edge at all, included; a call made from other seeds -- the correspondences an earlier call left -- may differ at exact FP32
 *     distance ties, as above), fixed frames come back bit for bit from d_init_X16xK, the context is left as it leaves it
 *     (sgb_correspondences_batch, sgb_error_batch and sgb_linearize_batch on the edges behave alike afterwards), and the weights in force
 *     are unchanged.  Errors of the enqueued work surface at the next synchronising call of the context.
 *   - The window tables are those of sgb_align_joint_async, cached in the context once for both calls and apart from the synchronous
 *     joint calls': a call whose tables are unchanged uploads nothing; one whose tables changed uploads them once.
 *   - While the context's stream is being captured the whole GNC is added to the capture: each replay re-runs it from what d_init_X16xK
 *     and the weights in force hold at replay time.  A call that would have to allocate or upload (the GNC buffers for its windows, the
 *     first batched call's search queue, the capture streams, window tables that differ from the cached ones) fails with a message
 *     instead: call it once outside the capture first.  The captured work is only valid while the context's batch, pairing, target,
 *     windows, fixed flags and buffers are those of the capture.  Outside a capture the instantiated graph is cached in the context and
 *     rebuilt when the align or GNC options, the windows, the batch, the pairing, the target or any buffer it uses changes.
 *   - sgb_kernel_launches counts 3 per call with at least one edge (one launch of the graph, two for the outputs) and 4 without (the stage
 *     kernels of the one stage, two for the outputs), whatever the stage and round counts, plus 1 when the pairing's view of the target
 *     is rebuilt; captured work counts at capture, not at replay.  A call with no window enqueues nothing. */
int sgb_align_joint_gnc_async(sgb_ctx* ctx, const sgb_align_options* options, const sgb_gnc_options* gnc, size_t n_windows, const size_t* window_off,
                              const uint8_t* fixed /*or NULL*/, const double* d_init_X16xK, double* d_out_X16xK, double* d_out_info4xW,
                              double* d_out_gnc2xW /*or NULL*/, double* d_out_point_w /*or NULL*/);

/* ---- per-cloud preparation on the device (SURVEY.md §8(f); not per-iteration) --------------------
 * sgb_estimate_features replaces estimate_normals / estimate_covariances / estimate_normals_covariances and
 * their _omp / _tbb variants (include/small_gicp/util/normal_estimation.hpp:12-140, normal_estimation_omp.hpp:9-60):
 * k nearest neighbours of every point in the cloud's own kd-tree (the point itself included), local covariance,
 * smallest-eigenvalue direction -> normal (flipped toward the origin, w = 0) and covariance with eigenvalues replaced
 * by (1e-3, 1, 1); fewer than 5 neighbours -> zero normal / identity covariance.  Either output may be NULL.
 * num_neighbors in 1..32. */
int sgb_estimate_features(sgb_ctx* ctx, size_t n, const double* points_xyz1, int num_neighbors, double* out_normals_xyz0 /*or NULL*/,
                          double* out_covs_4x4 /*or NULL*/);
/* Device-resident variants: fill the normals + covariances of the CURRENT target (after its kd-tree is set/built) or
 * the covariances of the CURRENT source without any host round trip (frame streams, benchmark_odom.hpp:59 +
 * odometry_benchmark_small_gicp_tbb.cpp:26-27). */
int sgb_target_estimate_features(sgb_ctx* ctx, int num_neighbors);
int sgb_source_estimate_features(sgb_ctx* ctx, int num_neighbors);
/* Frame streams (odometry_benchmark_small_gicp_tbb.cpp:41-43: `target_points = points; target_tree = tree;`): the CURRENT SOURCE becomes the
 * target -- its points, the kd-tree sgb_source_estimate_features built over them and its covariances are taken over on the device (a tree
 * is built only if none exists; host-supplied covariances are taken over too), the grid front end is built, and the context has no source
 * until the next sgb_source_set_points.  No normals: call sgb_target_estimate_features for point-to-plane. */
int sgb_target_adopt_source(sgb_ctx* ctx);
/* replaces voxelgrid_sampling{,_omp,_tbb} (include/small_gicp/util/downsampling.hpp:22-78): one output point per occupied
 * voxel = mean of its points, voxels ordered by the reference's 63-bit key (x | y<<21 | z<<42 of floor(p/leaf)+2^20);
 * points whose voxel coordinate leaves the 21-bit range are dropped.  out_points_xyz1 must hold n points. */
int sgb_voxelgrid_sampling(sgb_ctx* ctx, size_t n, const double* points_xyz1, double leaf_size, double* out_points_xyz1, size_t* n_out);
/* Many clouds at once, for preparing a sequence of frames: the outputs feed sgb_target_build_kdtrees / sgb_target_build_voxelmaps /
 * sgb_source_set_batch.  offsets: n_clouds + 1 ascending entries, offsets[0] = 0; cloud c = points offsets[c] .. offsets[c+1] (empty clouds
 * allowed); host, page-locked or device memory.  Neither call changes the context's target, source, batch, seeds or linearisation cache.
 * sgb_voxelgrid_sampling_batch: cloud c's output is sgb_voxelgrid_sampling of cloud c alone, bit for bit, at out_points_xyz1[out_offsets[c]
 * .. out_offsets[c+1]) (out_points_xyz1 must hold offsets[n_clouds] points; out_offsets: host memory, n_clouds + 1 entries).  A launch
 * count independent of n_clouds and one host synchronisation (a host out_points_xyz1 adds the copy of the means).  n_clouds <=
 * SGB_BATCH_MAX_MEMBERS, fewer than 2^31 points in all, leaf_size > 0, else the call fails with a message. */
int sgb_voxelgrid_sampling_batch(sgb_ctx* ctx, size_t n_clouds, const size_t* offsets, const double* points_xyz1, double leaf_size,
                                 double* out_points_xyz1, size_t* out_offsets);
/* sgb_estimate_features_batch: cloud c's normals / covariances are those of sgb_estimate_features of cloud c alone, in the caller's
 * concatenated order, EXCEPT where exact FP32 distance ties among a point's k + 4 nearest candidates are ranked differently (cloud c's
 * kd-tree is built as sgb_target_build_kdtrees builds map c, without the single call's curve pre-sort, so equal coordinates may sit in
 * another order); a cloud's results are bit-identical whatever else is in the batch, ties included.  Either output may be NULL.
 * num_neighbors in 1..32, n_clouds <= SGB_BATCH_MAX_MEMBERS, fewer than 2^30 points in all, else the call fails with a message.  The
 * launch count depends on the size of the largest cloud only; one host synchronisation at the end, as sgb_estimate_features. */
int sgb_estimate_features_batch(sgb_ctx* ctx, size_t n_clouds, const size_t* offsets, const double* points_xyz1, int num_neighbors,
                                double* out_normals_xyz0 /*or NULL*/, double* out_covs_4x4 /*or NULL*/);

#ifdef __cplusplus
}
#endif
#endif /* SGICP_B200_H_ */
