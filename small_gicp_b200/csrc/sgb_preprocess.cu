// SPDX-License-Identifier: MIT
// Per-cloud preparation on the device (SURVEY.md §8(f) rows 1 and 3):
//   * k-nearest-neighbour search of every cloud point in its own kd-tree + local covariance + closed-form 3x3
//     symmetric eigen-decomposition -> normal and regularised covariance
//       replaces estimate_normals / estimate_covariances / estimate_normals_covariances{,_omp,_tbb}
//       (/root/reference/include/small_gicp/util/normal_estimation.hpp:12-140, normal_estimation_omp.hpp:9-60)
//   * voxel-grid down-sampling: 3 x 21-bit voxel key, radix sort, segmented mean
//       replaces voxelgrid_sampling{,_omp,_tbb} (.../util/downsampling.hpp:22-78)
//   * many clouds at once: the features body over a forest of kd-trees (forest_features_kernel), and the voxel means over the
//     (cloud, valid, key) order of the many-maps sort (sgb_capi_preprocess.cu)
#include <cfloat>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "sgb_device.cuh"
#include "sgb_forest.h"
#include "sgb_kernels.h"

namespace sgb {

// ---------------------------------------------------------------------------------------------
// k-NN with a register-resident sorted candidate list (ann/knn_result.hpp:80-101 semantics: only strictly
// closer candidates enter, equal distances keep their arrival order).  Empty slots: the type's maximum distance and index ~0.
// ---------------------------------------------------------------------------------------------
template <int KMAX, typename D = float, typename I = uint32_t>
struct KnnList {
  D d[KMAX];
  I i[KMAX];
  D worst;
  int k;
  __device__ __forceinline__ void init(int k_) {
    const D big = sizeof(D) == sizeof(double) ? DBL_MAX : FLT_MAX;
    k = k_;
#pragma unroll
    for (int j = 0; j < KMAX; j++) {
      d[j] = big;
      i[j] = ~I(0);
    }
    worst = big;
  }
  __device__ __forceinline__ void offer(D v, I vi) {
    if (!(v < worst)) return;
#pragma unroll
    for (int j = 0; j < KMAX; j++) {
      if (j < k && v < d[j]) {
        const D td = d[j];
        const I ti = i[j];
        d[j] = v;
        i[j] = vi;
        v = td;
        vi = ti;
      }
    }
#pragma unroll
    for (int j = 0; j < KMAX; j++)
      if (j == k - 1) worst = d[j];
  }
};

/// Exact k-NN of one query per thread in the packet (BVH2) records of the cloud's tree (sgb_kernels_packet.cu has the
/// record layout): near child first, the far child is kept pending only while its box is closer than the k-th distance.
/// stack entry s of thread t: desc[s * kLinBlock + t] (child descriptor) and dist[s * kLinBlock + t] (its box distance).
/// A candidate enters L as tag | its leaf position: tag tells the trees of one list apart (forest_knn_kernel).
template <int KMAX, typename I = uint32_t>
__device__ __forceinline__ void bvh_knn(const float4* __restrict__ pnodes, const float4* __restrict__ pts, float qx, float qy, float qz,
                                        KnnList<KMAX, float, I>& L, uint2* desc, float* dist, I tag = 0) {
  if (!(isfinite(qx) && isfinite(qy) && isfinite(qz))) return;  // a non-finite query has no neighbours: no walk
  int sp = 0;
  uint2* my_desc = desc + threadIdx.x;
  float* my_dist = dist + threadIdx.x;
  uint32_t cur = 0;
  bool expand = true;
  uint2 leaf = make_uint2(0u, 0u);
  for (;;) {
    if (expand) {
      const float4 n0 = __ldg(&pnodes[cur * 4 + 0]), n1 = __ldg(&pnodes[cur * 4 + 1]);
      const float4 n2 = __ldg(&pnodes[cur * 4 + 2]), n3 = __ldg(&pnodes[cur * 4 + 3]);
      const float dl = box_dist2(qx, qy, qz, n0, n1), dr = box_dist2(qx, qy, qz, n2, n3);
      const bool left_first = dl <= dr;
      const float dn = left_first ? dl : dr, df = left_first ? dr : dl;
      const uint2 cn = left_first ? make_uint2(__float_as_uint(n0.w), __float_as_uint(n1.w)) : make_uint2(__float_as_uint(n2.w), __float_as_uint(n3.w));
      const uint2 cf = left_first ? make_uint2(__float_as_uint(n2.w), __float_as_uint(n3.w)) : make_uint2(__float_as_uint(n0.w), __float_as_uint(n1.w));
      if (df < L.worst) {
        my_desc[sp * kLinBlock] = cf;
        my_dist[sp * kLinBlock] = df;
        sp++;
      }
      if (!(dn < L.worst)) {
        expand = false;
        continue;
      }
      if (cn.y == 0u) {
        cur = cn.x;
        continue;
      }
      leaf = cn;
    } else {
      bool got = false;
      while (sp > 0) {
        sp--;
        if (my_dist[sp * kLinBlock] < L.worst) {  // worst_distance() > lower bound of the subtree (ann/kdtree.hpp:228 analogue)
          leaf = my_desc[sp * kLinBlock];
          got = true;
          break;
        }
      }
      if (!got) break;
      if (leaf.y == 0u) {
        cur = leaf.x;
        expand = true;
        continue;
      }
    }
    for (uint32_t j = 0; j < leaf.y; j++) {
      const float4 t = __ldg(&pts[leaf.x + j]);
      const float dx = t.x - qx, dy = t.y - qy, dz = t.z - qz;
      L.offer(dx * dx + dy * dy + dz * dz, tag | static_cast<I>(leaf.x + j));
    }
    expand = false;
  }
}

/// The features of the point at leaf position i (features_kernel, forest_features_kernel).  mode bit 0: normals, bit 1: covariances.
/// The cloud's points and its lo residuals are indexed by base + w (w = pts[].w, the index within the cloud); outputs are written at
/// base + w (or at i with leaf_order_out): device layout (float4 streams) and / or the reference's double layout.
///
/// Neighbour sets.  The search runs on the centred FP32 coordinates (rounded by up to ~2 um at 50 m), the reference on doubles: at the
/// k-th neighbour a near-tie could swap one point of the set -- rare (0.5 % of the points), but a different covariance where it happens.
/// So the search collects k + kFeatExtra candidates, and the k nearest of them are picked by their distance on the EXACT coordinates
/// (hi + lo, lo = what the FP32 rounding dropped, kept in original order): the set is then the reference's unless two candidates are
/// equidistant to ~1e-12 m^2, and the covariance sums use the exact coordinates as well.  lo == nullptr: FP32 coordinates throughout.
constexpr int kFeatExtra = 4;
template <int KMAX>
__device__ __forceinline__ void features_point(const float4* __restrict__ pnodes, const float4* __restrict__ pts, uint32_t i, uint32_t base, int k,
                                               const double* __restrict__ centre, int mode, float4* out_normals, float4* out_covA, float4* out_covB,
                                               double* out_normals_d, double* out_covs_d, int leaf_order_out, int depth, const float4* __restrict__ lo,
                                               uint2* s_stack) {
  constexpr int KC = KMAX + kFeatExtra;
  const float4 q = __ldg(&pts[i]);
  KnnList<KC> L;
  const int kc = lo ? k + kFeatExtra : k;
  L.init(kc);
  bvh_knn<KC>(pnodes, pts, q.x, q.y, q.z, L, s_stack, reinterpret_cast<float*>(s_stack + static_cast<size_t>(depth) * kLinBlock));
  const uint32_t qo = base + static_cast<uint32_t>(__float_as_int(q.w));
  double qx = q.x, qy = q.y, qz = q.z;
  if (lo) {
    const float4 l = __ldg(&lo[qo]);
    qx += l.x; qy += l.y; qz += l.z;
  }
  // exact offset of candidate j from the query (hi + lo of both)
  auto offset = [&](int j, double& x, double& y, double& z) {
    const float4 t = __ldg(&pts[L.i[j]]);
    double tx = t.x, ty = t.y, tz = t.z;
    if (lo) {
      const float4 l = __ldg(&lo[base + static_cast<uint32_t>(__float_as_int(t.w))]);
      tx += l.x; ty += l.y; tz += l.z;
    }
    x = tx - qx; y = ty - qy; z = tz - qz;
  };
  // exact squared distances of the candidates (-1 = no candidate / dropped)
  double d2[KC];
  int found = 0;
#pragma unroll
  for (int j = 0; j < KC; j++) {
    d2[j] = -1.0;
    if (j < kc && L.i[j] != kNone) {
      double x, y, z;
      offset(j, x, y, z);
      d2[j] = x * x + y * y + z * z;
      found++;
    }
  }
  // drop the (found - k) farthest candidates (exact distances; among exact ties the later arrival goes, knn_result.hpp:88-101)
  for (int drop = found - k; drop > 0; drop--) {
    double worst = -1.0;
    int wj = -1;
#pragma unroll
    for (int j = 0; j < KC; j++)
      if (d2[j] >= worst && d2[j] >= 0.0) {
        worst = d2[j];
        wj = j;
      }
#pragma unroll
    for (int j = 0; j < KC; j++)
      if (j == wj) d2[j] = -1.0;
    found--;
  }
  // sums relative to the query point (covariance is translation invariant; keeps the FP64 sums well conditioned); the offsets are
  // re-derived rather than kept: 3 x KC doubles of registers would spill
  double s[3] = {0, 0, 0}, ss[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
  for (int j = 0; j < KC; j++) {
    if (d2[j] >= 0.0) {
      double x, y, z;
      offset(j, x, y, z);
      s[0] += x; s[1] += y; s[2] += z;
      ss[0] += x * x; ss[1] += x * y; ss[2] += x * z; ss[3] += y * y; ss[4] += y * z; ss[5] += z * z;
    }
  }
  const uint32_t orig = leaf_order_out ? i : qo;
  double nrm[3] = {0.0, 0.0, 0.0};
  double cov[6] = {1.0, 0.0, 0.0, 1.0, 0.0, 1.0};  // < 5 neighbours: identity covariance, zero normal (normal_estimation.hpp:33-37,71-75)
  if (found >= 5) {
    const double inv_n = 1.0 / found;
    const double mx = s[0] * inv_n, my = s[1] * inv_n, mz = s[2] * inv_n;
    // cov = (sum_cross - mean * sum^T) / n   (normal_estimation.hpp:85-86)
    const double c00 = (ss[0] - mx * s[0]) * inv_n, c01 = (ss[1] - mx * s[1]) * inv_n, c02 = (ss[2] - mx * s[2]) * inv_n;
    const double c11 = (ss[3] - my * s[1]) * inv_n, c12 = (ss[4] - my * s[2]) * inv_n, c22 = (ss[5] - mz * s[2]) * inv_n;
    double v[3];
    smallest_eigenvector(c00, c01, c02, c11, c12, c22, v);
    // V diag(1e-3, 1, 1) V^T = I - (1 - 1e-3) v v^T for orthonormal V
    const double w = 1.0 - 1e-3;
    cov[0] = 1.0 - w * v[0] * v[0]; cov[1] = -w * v[0] * v[1]; cov[2] = -w * v[0] * v[2];
    cov[3] = 1.0 - w * v[1] * v[1]; cov[4] = -w * v[1] * v[2]; cov[5] = 1.0 - w * v[2] * v[2];
    // flip the normal toward the origin of the cloud's own frame (normal_estimation.hpp:19-23)
    const double px = qx + centre[0], py = qy + centre[1], pz = qz + centre[2];
    const double sgn = (px * v[0] + py * v[1] + pz * v[2]) > 0.0 ? -1.0 : 1.0;
    nrm[0] = sgn * v[0]; nrm[1] = sgn * v[1]; nrm[2] = sgn * v[2];
  }
  if (mode & 1) {
    if (out_normals) out_normals[orig] = make_float4((float)nrm[0], (float)nrm[1], (float)nrm[2], 0.f);
    if (out_normals_d) {
      double* o = out_normals_d + static_cast<size_t>(orig) * 4;
      o[0] = nrm[0]; o[1] = nrm[1]; o[2] = nrm[2]; o[3] = 0.0;
    }
  }
  if (mode & 2) {
    if (out_covA) {
      out_covA[orig] = make_float4((float)cov[0], (float)cov[1], (float)cov[2], (float)cov[3]);
      out_covB[orig] = make_float4((float)cov[4], (float)cov[5], 0.f, 0.f);
    }
    if (out_covs_d) {
      double* o = out_covs_d + static_cast<size_t>(orig) * 16;
      o[0] = cov[0]; o[1] = cov[1]; o[2] = cov[2]; o[3] = 0.0;
      o[4] = cov[1]; o[5] = cov[3]; o[6] = cov[4]; o[7] = 0.0;
      o[8] = cov[2]; o[9] = cov[4]; o[10] = cov[5]; o[11] = 0.0;
      o[12] = 0.0; o[13] = 0.0; o[14] = 0.0; o[15] = 0.0;
    }
  }
}

/// One thread per point of the cloud in LEAF order (neighbouring threads query neighbouring points); outputs in ORIGINAL order
/// (w = index) unless leaf_order_out.
template <int KMAX>
__global__ void __launch_bounds__(kLinBlock) features_kernel(const float4* __restrict__ pnodes, const float4* __restrict__ pts, uint32_t n, int k,
                                                             const double* __restrict__ centre, int mode, float4* out_normals, float4* out_covA,
                                                             float4* out_covB, double* out_normals_d, double* out_covs_d, int leaf_order_out, int depth,
                                                             const float4* __restrict__ lo) {
  extern __shared__ uint2 s_stack[];  // [depth][kLinBlock] descriptors, then [depth][kLinBlock] distances
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  features_point<KMAX>(pnodes, pts, i, 0u, k, centre, mode, out_normals, out_covA, out_covB, out_normals_d, out_covs_d, leaf_order_out, depth, lo, s_stack);
}

/// The forest of many clouds (launch_forest_features): one thread per leaf-ordered point of any map.  Map m's points occupy leaf and
/// original positions pt_off[m] .. pt_off[m+1] with w = the index within the map, its records start at node_base[m] and hold global
/// leaf positions, so the single cloud's body runs unchanged on map m's records, centre and base pt_off[m].
template <int KMAX>
__global__ void __launch_bounds__(kLinBlock) forest_features_kernel(const float4* __restrict__ pnodes, const float4* __restrict__ pts, uint32_t n, int k,
                                                                    const uint32_t* __restrict__ pt_off, const uint32_t* __restrict__ node_base,
                                                                    uint32_t n_maps, const double* __restrict__ centres, int mode, double* out_normals_d,
                                                                    double* out_covs_d, int depth, const float4* __restrict__ lo) {
  extern __shared__ uint2 s_stack[];  // [depth][kLinBlock] descriptors, then [depth][kLinBlock] distances
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t m = owner_of(pt_off, n_maps, i);
  features_point<KMAX>(pnodes + 4 * static_cast<size_t>(__ldg(&node_base[m])), pts, i, __ldg(&pt_off[m]), k, centres + 4 * static_cast<size_t>(m), mode,
                       nullptr, nullptr, nullptr, out_normals_d, out_covs_d, 0, depth, lo, s_stack);
}

template <int KMAX>
static cudaError_t launch_forest_features_t(const float4* pnodes, const float4* pts, uint32_t n, int k, const ForestTables& F, const double* centres, int mode,
                                            double* ond, double* ocd, int depth, const float4* lo, cudaStream_t st) {
  if (depth < 1) depth = 1;
  const size_t smem = static_cast<size_t>(depth) * kLinBlock * (sizeof(uint2) + sizeof(float));
  const cudaError_t e = allow_dynamic_smem(forest_features_kernel<KMAX>, smem);
  if (e != cudaSuccess) return e;
  const int grid = static_cast<int>((n + kLinBlock - 1) / kLinBlock);
  forest_features_kernel<KMAX><<<grid, kLinBlock, smem, st>>>(pnodes, pts, n, k, F.pt_off, F.node_base, F.n_maps, centres, mode, ond, ocd, depth, lo);
  return cudaGetLastError();
}

cudaError_t launch_forest_features(const float4* pnodes, const float4* leaf_pts, uint32_t n, int k, const ForestTables& F, const double* centres, int mode,
                                   double* out_normals_d, double* out_covs_d, int depth, const float4* lo, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  if (k <= 10) return launch_forest_features_t<10>(pnodes, leaf_pts, n, k, F, centres, mode, out_normals_d, out_covs_d, depth, lo, st);
  if (k <= 20) return launch_forest_features_t<20>(pnodes, leaf_pts, n, k, F, centres, mode, out_normals_d, out_covs_d, depth, lo, st);
  if (k <= 32) return launch_forest_features_t<32>(pnodes, leaf_pts, n, k, F, centres, mode, out_normals_d, out_covs_d, depth, lo, st);
  return cudaErrorInvalidValue;
}

template <int KMAX>
static cudaError_t launch_features_t(const float4* nodes, const float4* pts, uint32_t n, int k, const double* centre, int mode, float4* on, float4* oa, float4* ob,
                                     double* ond, double* ocd, int depth, int leaf_order_out, cudaStream_t st, const float4* lo) {
  if (depth < 1) depth = 1;
  const size_t smem = static_cast<size_t>(depth) * kLinBlock * (sizeof(uint2) + sizeof(float));
  const cudaError_t e = allow_dynamic_smem(features_kernel<KMAX>, smem);
  if (e != cudaSuccess) return e;
  const int grid = static_cast<int>((n + kLinBlock - 1) / kLinBlock);
  features_kernel<KMAX><<<grid, kLinBlock, smem, st>>>(nodes, pts, n, k, centre, mode, on, oa, ob, ond, ocd, leaf_order_out, depth, lo);
  return cudaGetLastError();
}

cudaError_t launch_features(const float4* nodes, const float4* pts, uint32_t n, int k, const double* centre, int mode, float4* out_normals, float4* out_covA,
                            float4* out_covB, double* out_normals_d, double* out_covs_d, int depth, int leaf_order_out, cudaStream_t st, const float4* lo_orig) {
  if (n == 0) return cudaSuccess;
  if (k <= 10) return launch_features_t<10>(nodes, pts, n, k, centre, mode, out_normals, out_covA, out_covB, out_normals_d, out_covs_d, depth, leaf_order_out, st, lo_orig);
  if (k <= 20) return launch_features_t<20>(nodes, pts, n, k, centre, mode, out_normals, out_covA, out_covB, out_normals_d, out_covs_d, depth, leaf_order_out, st, lo_orig);
  if (k <= 32) return launch_features_t<32>(nodes, pts, n, k, centre, mode, out_normals, out_covA, out_covB, out_normals_d, out_covs_d, depth, leaf_order_out, st, lo_orig);
  return cudaErrorInvalidValue;
}

// ---------------------------------------------------------------------------------------------
// k-NN of arbitrary query points in the target's search structure (KdTree::knn_search, ann/kdtree.hpp:165-189;
// batch_knn_search / batch_nearest_neighbor_search of the Python binding): one query per thread, results ascending.
// The search runs on the FP32 centred coordinates; what is reported, and what ranks the results, is the FP64 squared distance between
// the stored (FP32 centred) target point and the FP64 centred query.  The two orders disagree on near-ties -- ranking by the FP32
// distance and reporting the FP64 one gave rows that were not ascending -- so the search collects k + kFeatExtra candidates and the k
// nearest of them by the FP64 distance are reported in its order (equal FP64 distances keep the FP32 search's order).
// ---------------------------------------------------------------------------------------------
/// The FP64 re-rank of the candidates: candidate j < kc (d2 = its FP64 squared distance, DBL_MAX / ~0 for an empty slot) goes to
/// slot rank(j) of the query's row = the number of candidates before it in (FP64 distance, [BY_ENTRY: entry = idx >> 32,] candidate
/// order), a permutation of 0 .. kc - 1 computed without indexing the register arrays by a run-time value; ranks >= k are dropped.
template <int KC, bool BY_ENTRY>
__device__ __forceinline__ void knn_store_ranked(const double* d2, const unsigned long long* idx, int kc, int k, uint32_t i, unsigned long long* out_idx,
                                                 double* out_d) {
#pragma unroll
  for (int j = 0; j < KC; j++) {
    if (j < kc) {
      int rank = 0;
#pragma unroll
      for (int m = 0; m < KC; m++) {
        if constexpr (BY_ENTRY) {
          const uint32_t em = static_cast<uint32_t>(idx[m] >> 32), ej = static_cast<uint32_t>(idx[j] >> 32);
          if (m < kc && (d2[m] < d2[j] || ((em < ej || (em == ej && m < j)) && d2[m] == d2[j]))) rank++;
        } else {
          if (m < kc && (d2[m] < d2[j] || (m < j && d2[m] == d2[j]))) rank++;
        }
      }
      if (rank < k) {
        out_idx[static_cast<size_t>(i) * k + rank] = idx[j];
        out_d[static_cast<size_t>(i) * k + rank] = d2[j];
      }
    }
  }
}

template <int KMAX>
__global__ void __launch_bounds__(kLinBlock) batch_knn_kernel(const float4* __restrict__ pnodes, const float4* __restrict__ pts, const double4* __restrict__ queries,
                                                              uint32_t n, int k, const double* __restrict__ centre, unsigned long long* out_idx, double* out_d,
                                                              int depth) {
  extern __shared__ uint2 s_stack[];  // [depth][kLinBlock] descriptors, then [depth][kLinBlock] distances
  constexpr int KC = KMAX + kFeatExtra;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double4 q = queries[i];
  const double qx = q.x - centre[0], qy = q.y - centre[1], qz = q.z - centre[2];
  const int kc = k + kFeatExtra;
  KnnList<KC> L;
  L.init(kc);
  bvh_knn<KC>(pnodes, pts, static_cast<float>(qx), static_cast<float>(qy), static_cast<float>(qz), L, s_stack,
              reinterpret_cast<float*>(s_stack + static_cast<size_t>(depth) * kLinBlock));
  // fewer candidates than slots: size_t(-1) / max() like KnnResult's initial state (knn_result.hpp:60-66); they rank last
  double d2[KC];
  unsigned long long idx[KC];
#pragma unroll
  for (int j = 0; j < KC; j++) {
    d2[j] = DBL_MAX;
    idx[j] = ~0ull;
    if (j < kc && L.i[j] != kNone) {
      const float4 t = __ldg(&pts[L.i[j]]);
      const double dx = static_cast<double>(t.x) - qx, dy = static_cast<double>(t.y) - qy, dz = static_cast<double>(t.z) - qz;
      idx[j] = static_cast<uint32_t>(__float_as_int(t.w));
      d2[j] = dx * dx + dy * dy + dz * dz;
    }
  }
  knn_store_ranked<KC, false>(d2, idx, kc, k, i, out_idx, out_d);
}

// ---------------------------------------------------------------------------------------------
// k-NN of query sets in many-maps targets (sgb_target_batch_knn_maps / _submaps): one query per thread, its set from the query offsets.
// ---------------------------------------------------------------------------------------------
/// The FP64 query q of entry e (map m) centred on map m, in map m's stored frame: P_e^-1 q - c_m (the placement's inverse carried as a
/// pose with the query as its "source centre"), or q - c_m without placements, as batch_knn_kernel centres it.
__device__ __forceinline__ double3 forest_knn_query(const ForestKnn& P, uint32_t e, uint32_t m, const double4& q) {
  const double* c = P.centres + 4 * static_cast<size_t>(m);
  if (!P.inv_poses) return make_double3(q.x - c[0], q.y - c[1], q.z - c[2]);
  return centred_translation(P.inv_poses + 12 * static_cast<size_t>(e), q.x, q.y, q.z, c);
}

/// Query i of set s against the union of entries e0 .. e1 - 1 of a kd-tree forest: the one candidate list of k + kFeatExtra FP32
/// candidates carried from entry to entry (each tree walked with its own FP32 query, the bound the list's k-th distance so far), a
/// candidate tagged (entry - e0) << 32 | leaf position, so that two entries of one map stay apart.  Then batch_knn_kernel's FP64 re-rank,
/// each candidate's distance in its own entry's frame, exact ties by entry, then candidate order.  Reported index: (entry within the
/// list) << 32 | original index within the map (w); without an entry table (the maps call) the entry is always 0.
template <int KMAX>
__global__ void __launch_bounds__(kLinBlock) forest_knn_kernel(const __grid_constant__ ForestKnn P, uint32_t n, int k, unsigned long long* out_idx, double* out_d,
                                                               int depth) {
  extern __shared__ uint2 s_stack[];  // [depth][kLinBlock] descriptors, then [depth][kLinBlock] distances
  constexpr int KC = KMAX + kFeatExtra;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t s = owner_of(P.query_off, P.n_sets, i);
  const uint32_t e0 = P.entry_off ? __ldg(&P.entry_off[s]) : s, e1 = P.entry_off ? __ldg(&P.entry_off[s + 1]) : s + 1;
  const double4 q = P.queries[i];
  const int kc = k + kFeatExtra;
  KnnList<KC, float, unsigned long long> L;
  L.init(kc);
  for (uint32_t e = e0; e < e1; e++) {
    const uint32_t m = __ldg(&P.entry_maps[e]);
    if (__ldg(&P.pt_off[m + 1]) == __ldg(&P.pt_off[m])) continue;  // an empty map
    const double3 c = forest_knn_query(P, e, m, q);
    bvh_knn<KC, unsigned long long>(P.pnodes + 4 * static_cast<size_t>(__ldg(&P.node_base[m])), P.pts, static_cast<float>(c.x), static_cast<float>(c.y),
                                    static_cast<float>(c.z), L, s_stack, reinterpret_cast<float*>(s_stack + static_cast<size_t>(depth) * kLinBlock),
                                    static_cast<unsigned long long>(e - e0) << 32);
  }
  double d2[KC];
  unsigned long long idx[KC];
#pragma unroll
  for (int j = 0; j < KC; j++) {
    d2[j] = DBL_MAX;
    idx[j] = ~0ull;
    if (j < kc && L.i[j] != ~0ull) {
      const uint32_t e = e0 + static_cast<uint32_t>(L.i[j] >> 32);
      const double3 c = forest_knn_query(P, e, __ldg(&P.entry_maps[e]), q);
      const float4 t = __ldg(&P.pts[static_cast<uint32_t>(L.i[j])]);
      const double dx = static_cast<double>(t.x) - c.x, dy = static_cast<double>(t.y) - c.y, dz = static_cast<double>(t.z) - c.z;
      idx[j] = (L.i[j] & 0xFFFFFFFF00000000ull) | static_cast<uint32_t>(__float_as_int(t.w));
      d2[j] = dx * dx + dy * dy + dz * dz;
    }
  }
  knn_store_ranked<KC, true>(d2, idx, kc, k, i, out_idx, out_d);
}

/// IncrementalVoxelMap::knn_search (incremental_voxelmap.hpp:99-148) of query i of set s in voxel map maps[s]: the voxel of the FP64
/// query as given (fast_floor(q * inv_leaf)), its 1 / 7 / 27 offset voxels in vox_offset's order, their means ranked by the FP64
/// distance to the centred query, the first found winning exact ties (KnnList).  Reported index: the voxel id within its map << 32.
template <int KMAX>
__global__ void __launch_bounds__(kLinBlock) voxel_knn_kernel(const __grid_constant__ VoxelKnn P, uint32_t n, int k, unsigned long long* out_idx, double* out_d) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t m = __ldg(&P.set_maps[owner_of(P.query_off, P.n_sets, i)]);
  const uint4 r = P.regions[m];
  const double* c = P.centres + 4 * static_cast<size_t>(m);
  const double4 q = P.queries[i];
  const int cx = static_cast<int>(floor(q.x * P.inv_leaf)), cy = static_cast<int>(floor(q.y * P.inv_leaf)), cz = static_cast<int>(floor(q.z * P.inv_leaf));
  const double qx = q.x - c[0], qy = q.y - c[1], qz = q.z - c[2];
  KnnList<KMAX, double, uint32_t> L;
  L.init(k);
  for (int o = 0; o < P.num_offsets; o++) {
    int ox, oy, oz;
    vox_offset(P.num_offsets, o, ox, oy, oz);
    const int id = vox_find(P.table + r.x, r.y, cx + ox, cy + oy, cz + oz);
    if (id >= 0) {
      const float4 t = __ldg(&P.pts[id]);
      const double dx = static_cast<double>(t.x) - qx, dy = static_cast<double>(t.y) - qy, dz = static_cast<double>(t.z) - qz;
      L.offer(dx * dx + dy * dy + dz * dz, static_cast<uint32_t>(id) - r.z);
    }
  }
#pragma unroll
  for (int j = 0; j < KMAX; j++) {
    if (j < k) {
      out_idx[static_cast<size_t>(i) * k + j] = L.i[j] == kNone ? ~0ull : static_cast<unsigned long long>(L.i[j]) << 32;
      out_d[static_cast<size_t>(i) * k + j] = L.d[j];
    }
  }
}

template <int KMAX>
static cudaError_t launch_batch_knn_t(const float4* pnodes, const float4* pts, const double* queries4, uint32_t n, int k, const double* centre,
                                      unsigned long long* out_idx, double* out_d, int depth, cudaStream_t st) {
  if (depth < 1) depth = 1;
  const size_t smem = static_cast<size_t>(depth) * kLinBlock * (sizeof(uint2) + sizeof(float));
  const cudaError_t e = allow_dynamic_smem(batch_knn_kernel<KMAX>, smem);
  if (e != cudaSuccess) return e;
  batch_knn_kernel<KMAX><<<(n + kLinBlock - 1) / kLinBlock, kLinBlock, smem, st>>>(pnodes, pts, reinterpret_cast<const double4*>(queries4), n, k, centre, out_idx,
                                                                                  out_d, depth);
  return cudaGetLastError();
}

cudaError_t launch_batch_knn(const float4* pnodes, const float4* pts, const double* queries4, uint32_t n, int k, const double* centre, unsigned long long* out_idx,
                             double* out_d, int depth, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  if (k <= 1) return launch_batch_knn_t<1>(pnodes, pts, queries4, n, k, centre, out_idx, out_d, depth, st);
  if (k <= 10) return launch_batch_knn_t<10>(pnodes, pts, queries4, n, k, centre, out_idx, out_d, depth, st);
  if (k <= 20) return launch_batch_knn_t<20>(pnodes, pts, queries4, n, k, centre, out_idx, out_d, depth, st);
  if (k <= 32) return launch_batch_knn_t<32>(pnodes, pts, queries4, n, k, centre, out_idx, out_d, depth, st);
  return cudaErrorInvalidValue;
}

template <int KMAX>
static cudaError_t launch_forest_knn_t(const ForestKnn& P, uint32_t n, int k, unsigned long long* out_idx, double* out_d, int depth, cudaStream_t st) {
  if (depth < 1) depth = 1;
  const size_t smem = static_cast<size_t>(depth) * kLinBlock * (sizeof(uint2) + sizeof(float));
  const cudaError_t e = allow_dynamic_smem(forest_knn_kernel<KMAX>, smem);
  if (e != cudaSuccess) return e;
  forest_knn_kernel<KMAX><<<(n + kLinBlock - 1) / kLinBlock, kLinBlock, smem, st>>>(P, n, k, out_idx, out_d, depth);
  return cudaGetLastError();
}

cudaError_t launch_forest_knn(const ForestKnn& P, uint32_t n, int k, unsigned long long* out_idx, double* out_d, int depth, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  if (k <= 1) return launch_forest_knn_t<1>(P, n, k, out_idx, out_d, depth, st);
  if (k <= 10) return launch_forest_knn_t<10>(P, n, k, out_idx, out_d, depth, st);
  if (k <= 20) return launch_forest_knn_t<20>(P, n, k, out_idx, out_d, depth, st);
  if (k <= 32) return launch_forest_knn_t<32>(P, n, k, out_idx, out_d, depth, st);
  return cudaErrorInvalidValue;
}

cudaError_t launch_voxel_knn(const VoxelKnn& P, uint32_t n, int k, unsigned long long* out_idx, double* out_d, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  const unsigned grid = (n + kLinBlock - 1) / kLinBlock;
  if (k <= 1) voxel_knn_kernel<1><<<grid, kLinBlock, 0, st>>>(P, n, k, out_idx, out_d);
  else if (k <= 10) voxel_knn_kernel<10><<<grid, kLinBlock, 0, st>>>(P, n, k, out_idx, out_d);
  else if (k <= 20) voxel_knn_kernel<20><<<grid, kLinBlock, 0, st>>>(P, n, k, out_idx, out_d);
  else if (k <= 32) voxel_knn_kernel<32><<<grid, kLinBlock, 0, st>>>(P, n, k, out_idx, out_d);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// voxel-grid down-sampling
// ---------------------------------------------------------------------------------------------
__global__ void voxel_keys_kernel(const double4* __restrict__ pts, size_t n, double inv_leaf, uint64_t* keys, uint32_t* vals) {
  constexpr int coord_bit_size = 21;
  constexpr int64_t coord_bit_mask = (1 << 21) - 1;
  constexpr int coord_offset = 1 << (coord_bit_size - 1);
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const double4 p = pts[i];
    const int64_t cx = static_cast<int64_t>(floor(p.x * inv_leaf)) + coord_offset;
    const int64_t cy = static_cast<int64_t>(floor(p.y * inv_leaf)) + coord_offset;
    const int64_t cz = static_cast<int64_t>(floor(p.z * inv_leaf)) + coord_offset;
    // out of the 21-bit range, or non-finite (the reference's fast_floor gives INT_MIN there; the cast here gives 0 for NaN): dropped
    // (downsampling.hpp:41-45 warns and marks them invalid)
    uint64_t key = ~0ull;
    if (point_is_finite(p.x, p.y, p.z) && cx >= 0 && cy >= 0 && cz >= 0 && cx <= coord_bit_mask && cy <= coord_bit_mask && cz <= coord_bit_mask)
      key = static_cast<uint64_t>(cx) | (static_cast<uint64_t>(cy) << coord_bit_size) | (static_cast<uint64_t>(cz) << (2 * coord_bit_size));
    keys[i] = key;
    vals[i] = static_cast<uint32_t>(i);
  }
}

// one thread per segment head: mean of the segment's points in sorted (= original index) order, FP64
__global__ void voxel_means_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, const uint32_t* __restrict__ heads,
                                   const uint32_t* __restrict__ slots, size_t n, const double4* __restrict__ pts, double4* out) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    if (!heads[i]) continue;
    const uint64_t k = keys[i];
    double sx = 0, sy = 0, sz = 0, cnt = 0;
    for (size_t j = i; j < n && keys[j] == k; j++) {
      const double4 p = pts[vals[j]];
      sx += p.x; sy += p.y; sz += p.z; cnt += 1.0;
    }
    out[slots[i]] = make_double4(sx / cnt, sy / cnt, sz / cnt, 1.0);
  }
}

static int vgrid(size_t n, int cap) {
  size_t g = (n + 255) / 256;
  if (g < 1) g = 1;
  if (g > static_cast<size_t>(cap)) g = cap;
  return static_cast<int>(g);
}

cudaError_t launch_voxel_keys(const double* d_pts4, size_t n, double inv_leaf, uint64_t* keys, uint32_t* vals, int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  voxel_keys_kernel<<<vgrid(n, sm_count * 8), 256, 0, st>>>(reinterpret_cast<const double4*>(d_pts4), n, inv_leaf, keys, vals);
  return cudaGetLastError();
}
cudaError_t launch_voxel_means(const uint64_t* keys, const uint32_t* vals, const uint32_t* heads, const uint32_t* slots, size_t n, const double* d_pts4,
                               double* d_out4, int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  voxel_means_kernel<<<vgrid(n, sm_count * 8), 256, 0, st>>>(keys, vals, heads, slots, n, reinterpret_cast<const double4*>(d_pts4),
                                                             reinterpret_cast<double4*>(d_out4));
  return cudaGetLastError();
}
// ---------------------------------------------------------------------------------------------
// Gaussian voxel map construction (incremental_voxelmap.hpp:55-92 with GaussianVoxel::add / finalize,
// gaussian_voxelmap.hpp:30-62): one thread per voxel adds its points and covariances in original-index order
// (the order the reference's insert loop meets them) and divides by the count.
// ---------------------------------------------------------------------------------------------
__global__ void voxel_stats_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, const uint32_t* __restrict__ heads,
                                   const uint32_t* __restrict__ slots, size_t n, const double4* __restrict__ pts, const double* __restrict__ covs,
                                   double4* out_means, double* out_covs, int4* out_coords) {
  constexpr int coord_bit_size = 21;
  constexpr uint64_t coord_bit_mask = (1ull << 21) - 1;
  constexpr int coord_offset = 1 << (coord_bit_size - 1);
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    if (!heads[i]) continue;
    const uint64_t k = keys[i];
    double sx = 0, sy = 0, sz = 0, cnt = 0;
    double c[16];
#pragma unroll
    for (int a = 0; a < 16; a++) c[a] = 0.0;
    for (size_t j = i; j < n && keys[j] == k; j++) {
      const uint32_t v = vals[j];
      const double4 p = pts[v];
      sx += p.x;
      sy += p.y;
      sz += p.z;
      cnt += 1.0;
      if (covs) {
        const double* cv = covs + static_cast<size_t>(v) * 16;
#pragma unroll
        for (int a = 0; a < 16; a++) c[a] += cv[a];
      }
    }
    const uint32_t id = slots[i];
    out_means[id] = make_double4(sx / cnt, sy / cnt, sz / cnt, 1.0);
    if (covs) {
#pragma unroll
      for (int a = 0; a < 16; a++) out_covs[static_cast<size_t>(id) * 16 + a] = c[a] / cnt;
    }
    out_coords[id] = make_int4(static_cast<int>(k & coord_bit_mask) - coord_offset, static_cast<int>((k >> coord_bit_size) & coord_bit_mask) - coord_offset,
                               static_cast<int>((k >> (2 * coord_bit_size)) & coord_bit_mask) - coord_offset, static_cast<int>(id));
  }
}

__global__ void vox_table_clear_kernel(int4* table, uint32_t capacity) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < capacity) table[i] = make_int4(0, 0, 0, -1);
}

cudaError_t launch_voxel_stats(const uint64_t* keys, const uint32_t* vals, const uint32_t* heads, const uint32_t* slots, size_t n, const double* d_pts4,
                               const double* d_covs16, double* out_means4, double* out_covs16, int4* out_coords, int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  voxel_stats_kernel<<<vgrid(n, sm_count * 8), 256, 0, st>>>(keys, vals, heads, slots, n, reinterpret_cast<const double4*>(d_pts4), d_covs16,
                                                             reinterpret_cast<double4*>(out_means4), out_covs16, out_coords);
  return cudaGetLastError();
}
// ---------------------------------------------------------------------------------------------
// Many Gaussian voxel maps in one pass (sgb_target_build_voxelmaps).  The points are ordered by (map, valid, voxel key), ascending
// original index within a voxel: the key sort, then a stable sort by (map, valid).  Each map's points keep their slots
// offsets[m] .. offsets[m+1] of that order, its dropped points (key ~0) first.  The stored key carries in bit 63 (outside the 63-bit
// key, ignored when the coordinates are decoded) the parity of the map's rank among the maps that have points: maps next to each other
// in this order -- empty maps hold no slots, so maps 0 and 2 are neighbours when map 1 is empty -- always differ in it, so that
// voxel_stats_kernel's run over equal keys cannot run from one map's last voxel into the next map's first voxel or dropped points.
// ---------------------------------------------------------------------------------------------
// after the key sort: (map << 1 | valid) of every point in key order, and its position
__global__ void voxelmaps_sort_keys_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, size_t n, const uint32_t* __restrict__ offsets,
                                           uint32_t n_maps, uint64_t* map_keys, uint32_t* pos) {
  for (size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; j < n; j += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const uint32_t m = owner_of(offsets, n_maps, vals[j]);
    map_keys[j] = (static_cast<uint64_t>(m) << 1) | (keys[j] != ~0ull ? 1u : 0u);
    pos[j] = static_cast<uint32_t>(j);
  }
}

// after the (map, valid) sort: the points' keys (bit 63 = rank_parity[map]) and original indices in (map, valid, key) order, and the
// voxel heads: a valid point whose predecessor is invalid, of another map or of another voxel
__global__ void voxelmaps_order_kernel(const uint64_t* __restrict__ map_keys, const uint32_t* __restrict__ pos, const uint64_t* __restrict__ keys,
                                       const uint32_t* __restrict__ vals, size_t n, const uint32_t* __restrict__ rank_parity, uint64_t* out_keys,
                                       uint32_t* out_vals, uint32_t* heads) {
  for (size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; j < n; j += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const uint64_t mk = map_keys[j], k = keys[pos[j]];
    const uint64_t parity = static_cast<uint64_t>(rank_parity[mk >> 1] & 1u) << 63;
    const bool valid = (mk & 1ull) != 0;
    out_keys[j] = valid ? (k | parity) : ((~0ull >> 1) | parity);
    out_vals[j] = vals[pos[j]];
    heads[j] = valid && (j == 0 || map_keys[j - 1] != mk || keys[pos[j - 1]] != k) ? 1u : 0u;
    if (j == 0) heads[n] = 0u;
  }
}

// one thread per map: its voxels (slots[offsets[m]] .. slots[offsets[m+1]]) and its table capacity, sgb_target_build_voxelmap's rule
// (a power of two >= 16 and >= twice the voxel count); caps[n_maps] = 0 closes the scan of the capacities
__global__ void voxelmaps_count_kernel(const uint32_t* __restrict__ offsets, uint32_t n_maps, const uint32_t* __restrict__ slots, uint4* regions, uint32_t* caps) {
  const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m == 0) caps[n_maps] = 0u;
  if (m >= n_maps) return;
  const uint32_t first = slots[offsets[m]], count = slots[offsets[m + 1]] - first;
  uint32_t capacity = 16;
  while (capacity < 2ull * count) capacity <<= 1;
  regions[m] = make_uint4(0u, capacity - 1u, first, count);
  caps[m] = capacity;
}

// one CTA per map: the centre of its voxel means, and the map's first table slot from the scan of the capacities
__global__ void __launch_bounds__(kBoxBlock) voxelmaps_centre_kernel(const double4* __restrict__ means, uint4* regions, const uint32_t* __restrict__ cap_scan,
                                                                    double* centres) {
  const uint32_t m = blockIdx.x;
  const uint4 r = regions[m];
  cta_box_centre(means, r.z, r.z + r.w, nullptr, centres + 4 * static_cast<size_t>(m));
  if (threadIdx.x == 0) regions[m].x = cap_scan[m];
}

// one thread per voxel: FP32 mean / covariance about its map's centre (convert_kernel's rounding), w = its id within the map, and its
// entry (x, y, z, global id) in its map's region of the table: voxel coordinates are distinct, so an insert only has to find a free slot
// of its probe sequence
__global__ void voxelmaps_convert_insert_kernel(const double4* __restrict__ means, const double* __restrict__ covs, const int4* __restrict__ coords,
                                                uint32_t n_voxels, const uint4* __restrict__ regions, uint32_t n_maps, const double* __restrict__ centres,
                                                float4* out_pts, float4* out_covA, float4* out_covB, int4* table) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_voxels) return;
  const uint32_t m = owner_of<4>(&regions[0].z, n_maps, i);  // the map whose voxels are first .. first + count - 1 (regions[m].z / .w)
  const uint4 r = regions[m];
  const double* c = centres + 4 * static_cast<size_t>(m);
  const double4 p = means[i];
  const double x = p.x - c[0], y = p.y - c[1], z = p.z - c[2];
  out_pts[i] = make_float4((float)x, (float)y, (float)z, __int_as_float(static_cast<int>(i - r.z)));
  if (covs) {
    out_covA[i] = pack_covA(covs + static_cast<size_t>(i) * 16);
    out_covB[i] = pack_covB(covs + static_cast<size_t>(i) * 16);
  }
  const int4 v = coords[i];
  int4* region = table + r.x;
  uint32_t slot = vox_hash(v.x, v.y, v.z) & r.y;
  for (;;) {
    if (atomicCAS(&region[slot].w, -1, v.w) == -1) {
      region[slot].x = v.x;
      region[slot].y = v.y;
      region[slot].z = v.z;
      return;
    }
    slot = (slot + 1u) & r.y;
  }
}

cudaError_t launch_voxelmaps_sort_keys(const uint64_t* keys, const uint32_t* vals, size_t n, const uint32_t* offsets, uint32_t n_maps, uint64_t* map_keys,
                                       uint32_t* pos, int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  voxelmaps_sort_keys_kernel<<<vgrid(n, sm_count * 8), 256, 0, st>>>(keys, vals, n, offsets, n_maps, map_keys, pos);
  return cudaGetLastError();
}
cudaError_t launch_voxelmaps_order(const uint64_t* map_keys, const uint32_t* pos, const uint64_t* keys, const uint32_t* vals, size_t n,
                                   const uint32_t* rank_parity, uint64_t* out_keys, uint32_t* out_vals, uint32_t* heads, int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  voxelmaps_order_kernel<<<vgrid(n, sm_count * 8), 256, 0, st>>>(map_keys, pos, keys, vals, n, rank_parity, out_keys, out_vals, heads);
  return cudaGetLastError();
}
cudaError_t launch_voxelmaps_count(const uint32_t* offsets, uint32_t n_maps, const uint32_t* slots, uint4* regions, uint32_t* caps, cudaStream_t st) {
  voxelmaps_count_kernel<<<(n_maps + 256u) / 256u, 256, 0, st>>>(offsets, n_maps, slots, regions, caps);
  return cudaGetLastError();
}
cudaError_t launch_voxelmaps_centres(const double* means4, uint32_t n_maps, uint4* regions, const uint32_t* cap_scan, double* centres, cudaStream_t st) {
  if (!n_maps) return cudaSuccess;
  voxelmaps_centre_kernel<<<n_maps, kBoxBlock, 0, st>>>(reinterpret_cast<const double4*>(means4), regions, cap_scan, centres);
  return cudaGetLastError();
}
cudaError_t launch_voxelmaps_table(const double* means4, const double* covs16, const int4* coords, uint32_t n_voxels, const uint4* regions, uint32_t n_maps,
                                   const double* centres, float4* out_pts, float4* out_covA, float4* out_covB, int4* table, uint32_t table_slots,
                                   cudaStream_t st) {
  vox_table_clear_kernel<<<(table_slots + 255u) / 256u, 256, 0, st>>>(table, table_slots);
  if (n_voxels)
    voxelmaps_convert_insert_kernel<<<(n_voxels + 255u) / 256u, 256, 0, st>>>(reinterpret_cast<const double4*>(means4), covs16, coords, n_voxels, regions,
                                                                             n_maps, centres, out_pts, out_covA, out_covB, table);
  return cudaGetLastError();
}

cudaError_t exclusive_sum_u32(void* d_temp, size_t& temp_bytes, const uint32_t* in, uint32_t* out, size_t n, cudaStream_t st) {
  return cub::DeviceScan::ExclusiveSum(d_temp, temp_bytes, in, out, static_cast<int>(n), st);
}

}  // namespace sgb
