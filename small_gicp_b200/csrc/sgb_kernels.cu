// SPDX-License-Identifier: MIT
// Hot-path kernels (sm_90a): fused transform -> kd-tree NN -> reject -> factor -> reduction, the
// error() kernel for the LM inner loop, and the one-off layout kernels (upload conversion, Morton
// ordering of the source, leaf ordering of the target).  See DESIGN.md §4 for the roofline of each.
#include "sgb_device.cuh"
#include "sgb_kernels.h"

#include <cfloat>
#include <cub/device/device_radix_sort.cuh>
#include <map>
#include <mutex>
#include <tuple>

namespace sgb {

// =============================================================================================
// linearize: one thread per source point (grid-stride, Morton-ordered so a warp's queries share
// their path through the tree), FP32 search on FP32 coordinates, FP64 factor algebra and sums.
// =============================================================================================
#ifdef SGB_PROFILING  // single fused kernel (SGB_SEARCH=0): the round-1 starting point, kept for A/B runs only
template <int FACTOR, int ROBUST>
__global__ void __launch_bounds__(kLinBlock) linearize_kd_kernel(const __grid_constant__ LinParams P) {
  extern __shared__ uint2 s_stack[];
  double acc[kAcc + 1];
#pragma unroll
  for (int k = 0; k <= kAcc; k++) acc[k] = 0.0;

  const double* R = P.T;
  const double csx = P.src.centre[0], csy = P.src.centre[1], csz = P.src.centre[2];
  const double3 tp = centred_translation(P.T, csx, csy, csz, P.tgt.centre);

  // Work unit = chunk of 32*K source positions per warp; lane l handles positions base + k*32 + l, k = 0..K-1,
  // which are K consecutive points along the Morton curve: the previous result of the lane is a tight search
  // seed for the next query, and so is the previous linearize's correspondence of the same point.
  const uint32_t K = P.src.run, chunk_pts = 32u * K;
  const uint32_t n_chunks = (P.src.n + chunk_pts - 1) / chunk_pts;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t chunk = warp; chunk < n_chunks; chunk += n_warps) {
    uint32_t chain = kNone;
    for (uint32_t k = 0; k < K; k++) {
      const uint32_t i = chunk * chunk_pts + k * 32u + lane;
      if (i >= P.src.n) break;
      const float4 sp = __ldg(&P.src.pts[i]);
      const double sx = sp.x, sy = sp.y, sz = sp.z;
      const double3 q = centred_query(R, tp, sp);
      const double qx = q.x, qy = q.y, qz = q.z;
      const float fx = static_cast<float>(qx), fy = static_cast<float>(qy), fz = static_cast<float>(qz);

      float best_d = P.max_dist_sq;
      uint32_t best = kNone;
      {  // seeds
        const uint32_t prev = P.use_prev ? P.corr[i] : kNone;
        if (prev != kNone) {
          const float4 t = __ldg(&P.tgt.pts[prev]);
          const float dx = t.x - fx, dy = t.y - fy, dz = t.z - fz;
          const float d = dx * dx + dy * dy + dz * dz;
          if (d < best_d) {
            best_d = d;
            best = prev;
          }
        }
        if (chain != kNone && chain != prev) {
          const float4 t = __ldg(&P.tgt.pts[chain]);
          const float dx = t.x - fx, dy = t.y - fy, dz = t.z - fz;
          const float d = dx * dx + dy * dy + dz * dz;
          if (d < best_d) {
            best_d = d;
            best = chain;
          }
        }
      }
      best = kd_nearest(P.tgt.nodes, P.tgt.pts, fx, fy, fz, best_d, best, s_stack);
      if (best != kNone) chain = best;

      double rx = 0.0, ry = 0.0, rz = 0.0;
      if (best != kNone) {
        const float4 tq = __ldg(&P.tgt.pts[best]);
        rx = static_cast<double>(tq.x) - qx;
        ry = static_cast<double>(tq.y) - qy;
        rz = static_cast<double>(tq.z) - qz;
        if (rx * rx + ry * ry + rz * rz > P.max_dist_sq_d) best = kNone;  // DistanceRejector on the FP64 residual (rejector.hpp:24)
      }
      P.corr[i] = best;
      if (best == kNone) continue;

      Sym3 M;
      if (FACTOR == 0) {
        M = Sym3{1.0, 0.0, 0.0, 1.0, 0.0, 1.0};
      } else if (FACTOR == 1) {
        const float4 n = __ldg(&P.tgt.normals[best]);
        M = Sym3{static_cast<double>(n.x) * n.x, 0.0, 0.0, static_cast<double>(n.y) * n.y, 0.0, static_cast<double>(n.z) * n.z};
      } else {
        M = gicp_precision(R, __ldg(&P.src.covA[i]), __ldg(&P.src.covB[i]), __ldg(&P.tgt.covA[best]), __ldg(&P.tgt.covB[best]));
      }
      accumulate_factor<ROBUST>(R, M, rx, ry, rz, csx + sx, csy + sy, csz + sz, P.robust_c, acc);
      acc[kAcc] += 1.0;
    }
  }
  block_reduce_and_finish<kAcc + 1, true>(acc, P.partials, P.ticket, P.out, P.comm);
}

#endif  // SGB_PROFILING

// Gaussian-voxel-map target (VGICP): the nearest voxel mean of every point (vox_nearest, sgb_device.cuh), factor, reduction.
template <int FACTOR, int ROBUST>
__global__ void __launch_bounds__(kLinBlock) linearize_vox_kernel(const __grid_constant__ LinParams P) {
  double acc[kAcc + 1];
#pragma unroll
  for (int k = 0; k <= kAcc; k++) acc[k] = 0.0;
  const double* R = P.T;
  const double csx = P.src.centre[0], csy = P.src.centre[1], csz = P.src.centre[2];
  const double ctx = P.tgt.centre[0], cty = P.tgt.centre[1], ctz = P.tgt.centre[2];
  const double3 tp = centred_translation(P.T, csx, csy, csz, P.tgt.centre);
  const double max_d = P.max_dist_sq_d;

  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < P.src.n; i += stride) {
    const float4 sp = __ldg(&P.src.pts[i]);
    const double sx = sp.x, sy = sp.y, sz = sp.z;
    const double3 q = centred_query(R, tp, sp);
    double brx = 0, bry = 0, brz = 0;
    const uint32_t best = vox_nearest(P.tgt, q.x, q.y, q.z, ctx, cty, ctz, max_d, brx, bry, brz);
    P.corr[i] = best;
    if (best == kNone) continue;
    Sym3 M;
    if (FACTOR == 2) {
      M = gicp_precision(R, __ldg(&P.src.covA[i]), __ldg(&P.src.covB[i]), __ldg(&P.tgt.covA[best]), __ldg(&P.tgt.covB[best]));
    } else {
      M = Sym3{1.0, 0.0, 0.0, 1.0, 0.0, 1.0};
    }
    accumulate_factor<ROBUST>(R, M, brx, bry, brz, csx + sx, csy + sy, csz + sz, P.robust_c, acc);
    acc[kAcc] += 1.0;
  }
  block_reduce_and_finish<kAcc + 1, true>(acc, P.partials, P.ticket, P.out, P.comm);
}

// =============================================================================================
// error(): cached correspondences, trial pose T, GICP precision matrix re-derived from the pose of
// the last linearize (gicp_factor.hpp:81-89).  Pure streaming + gather.
// =============================================================================================
template <int FACTOR, int ROBUST>
__global__ void __launch_bounds__(kLinBlock) error_kernel(const __grid_constant__ LinParams P) {
  double acc[1] = {0.0};
  const double* R = P.T;
  const double3 tp = centred_translation(P.T, P.src.centre[0], P.src.centre[1], P.src.centre[2], P.tgt.centre);
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < P.src.n; i += stride) {
    const uint32_t k = __ldg(&P.corr[i]);
    if (k == kNone) continue;
    const float4 sp = __ldg(&P.src.pts[i]);
    const float4 tq = __ldg(&P.tgt.pts[k]);
    float4 sA = make_float4(0.f, 0.f, 0.f, 0.f), sB = sA, t1 = sA, t2 = sA;
    if (FACTOR == 1) t1 = __ldg(&P.tgt.normals[k]);
    if (FACTOR == 2) {
      sA = __ldg(&P.src.covA[i]);
      sB = __ldg(&P.src.covB[i]);
      t1 = __ldg(&P.tgt.covA[k]);
      t2 = __ldg(&P.tgt.covB[k]);
    }
    const double e = point_error<FACTOR, ROBUST>(R, tp.x, tp.y, tp.z, P.Tlin, P.robust_c, sp, sA, sB, tq, t1, t2);
    acc[0] += e;
  }
  block_reduce_and_finish<1, false>(acc, P.partials, P.ticket, P.out, P.comm);
}

// ---------------------------------------------------------------------------------------------
template <int FACTOR, int ROBUST>
static cudaError_t launch_lin(const LinParams& P, bool voxel, int grid, size_t smem, cudaStream_t st) {
  if (voxel) {
    if (FACTOR == 1) return cudaErrorInvalidValue;
    linearize_vox_kernel<(FACTOR == 1 ? 0 : FACTOR), ROBUST><<<grid, kLinBlock, 0, st>>>(P);
  } else {
#ifdef SGB_PROFILING
    const cudaError_t e = allow_dynamic_smem(linearize_kd_kernel<FACTOR, ROBUST>, smem);
    if (e != cudaSuccess) return e;
    linearize_kd_kernel<FACTOR, ROBUST><<<grid, kLinBlock, smem, st>>>(P);
#else
    return cudaErrorNotSupported;  // point targets go through the search + factor kernels (sgb_grid.cu, sgb_kernels_packet.cu, sgb_kernels_split.cu)
#endif
  }
  return cudaGetLastError();
}

cudaError_t launch_linearize(const LinParams& P, int factor, int robust, bool voxel, int grid, int stack_depth, cudaStream_t st) {
  const size_t smem = voxel ? 0 : static_cast<size_t>(stack_depth) * kLinBlock * sizeof(uint2);
  return dispatch_factor_robust(factor, robust, cudaErrorInvalidValue, [&](auto f, auto r) { return launch_lin<f, r>(P, voxel, grid, smem, st); });
}
cudaError_t launch_error(const LinParams& P, int factor, int robust, int grid, cudaStream_t st) {
  return dispatch_factor_robust(factor, robust, cudaErrorInvalidValue, [&](auto f, auto r) {
    error_kernel<f, r><<<grid, kLinBlock, 0, st>>>(P);
    return cudaGetLastError();
  });
}

// A rank whose shard is empty still has to take part in the fused exchange: one CTA that reduces nothing.
template <int NACC, bool EXPAND>
__global__ void __launch_bounds__(kLinBlock) reduce_nothing_kernel(const __grid_constant__ LinParams P) {
  double acc[NACC];
#pragma unroll
  for (int k = 0; k < NACC; k++) acc[k] = 0.0;
  block_reduce_and_finish<NACC, EXPAND>(acc, P.partials, P.ticket, P.out, P.comm);
}
cudaError_t launch_reduce_nothing(const LinParams& P, bool linearize, cudaStream_t st) {
  if (linearize)
    reduce_nothing_kernel<kAcc + 1, true><<<1, kLinBlock, 0, st>>>(P);
  else
    reduce_nothing_kernel<1, false><<<1, kLinBlock, 0, st>>>(P);
  return cudaGetLastError();
}

int linearize_occupancy(int stack_depth) {
#ifdef SGB_PROFILING
  if (stack_depth > 0) {
    const size_t smem = static_cast<size_t>(stack_depth) * kLinBlock * sizeof(uint2);
    return ctas_per_sm(linearize_kd_kernel<2, 0>, kLinBlock, smem, false, smem > 48 * 1024);
  }
#endif
  (void)stack_depth;  // resident CTAs of the voxel-map kernel (VGICP): its grid-stride loop is sized to one wave
  return ctas_per_sm(linearize_vox_kernel<2, 0>, kLinBlock, 0, false, false);
}

// Kernel attributes belong to the kernel on a device, not to a context: every context of the process on that device shares them.  One mutex
// guards both caches below, and the dynamic shared-memory limit only ever grows, so a launch at or below the limit it asked for can never be
// undercut by another thread lowering it between that thread's set and its launch.
static std::mutex g_attr_mu;
static std::map<std::pair<int, const void*>, size_t> g_smem_limit;  // (device, kernel) -> largest opt-in limit set so far

static cudaError_t allow_dynamic_smem_locked(int device, const void* kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return cudaSuccess;  // within every kernel's default limit
  size_t& limit = g_smem_limit[std::make_pair(device, kernel)];
  if (bytes <= limit) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
  if (e == cudaSuccess) limit = bytes;
  return e;
}

cudaError_t allow_dynamic_smem(const void* kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return cudaSuccess;
  int device = 0;
  cudaError_t e = cudaGetDevice(&device);
  if (e != cudaSuccess) return e;
  const std::lock_guard<std::mutex> lock(g_attr_mu);
  return allow_dynamic_smem_locked(device, kernel, bytes);
}

int ctas_per_sm(const void* kernel, int block, size_t smem, bool max_shared_carveout, bool smem_limit) {
  static std::map<std::tuple<int, const void*, int, size_t>, int> cache;
  int device = 0;
  cudaGetDevice(&device);
  const auto key = std::make_tuple(device, kernel, block, smem);
  const std::lock_guard<std::mutex> lock(g_attr_mu);
  const auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  if (max_shared_carveout) cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (smem_limit) allow_dynamic_smem_locked(device, kernel, smem);
  int nb = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, block, smem) != cudaSuccess || nb < 1) nb = 1;
  cache.emplace(key, nb);
  return nb;
}

// =============================================================================================
// One-off layout kernels
// =============================================================================================
// min/max of N x 4 doubles (xyz used) -> bounds[6] via ordered-int atomics on doubles
__device__ __forceinline__ void atomic_min_double(double* addr, double v) {
  unsigned long long* a = reinterpret_cast<unsigned long long*>(addr);
  unsigned long long old = *a, assumed;
  do {
    assumed = old;
    if (__longlong_as_double(assumed) <= v) break;
    old = atomicCAS(a, assumed, static_cast<unsigned long long>(__double_as_longlong(v)));
  } while (assumed != old);
}
__device__ __forceinline__ void atomic_max_double(double* addr, double v) {
  unsigned long long* a = reinterpret_cast<unsigned long long*>(addr);
  unsigned long long old = *a, assumed;
  do {
    assumed = old;
    if (__longlong_as_double(assumed) >= v) break;
    old = atomicCAS(a, assumed, static_cast<unsigned long long>(__double_as_longlong(v)));
  } while (assumed != old);
}

__global__ void bounds_init_kernel(double* bounds) {
  if (threadIdx.x < 3) bounds[threadIdx.x] = DBL_MAX;
  if (threadIdx.x >= 3 && threadIdx.x < 6) bounds[threadIdx.x] = -DBL_MAX;
}

__global__ void bounds_kernel(const double4* __restrict__ pts, size_t n, double* bounds) {
  double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, hi[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const double4 p = pts[i];
    if (!point_is_finite(p.x, p.y, p.z)) continue;  // inert: no part in the box
    lo[0] = fmin(lo[0], p.x); lo[1] = fmin(lo[1], p.y); lo[2] = fmin(lo[2], p.z);
    hi[0] = fmax(hi[0], p.x); hi[1] = fmax(hi[1], p.y); hi[2] = fmax(hi[2], p.z);
  }
#pragma unroll
  for (int d = 0; d < 3; d++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[d] = fmin(lo[d], __shfl_down_sync(0xffffffffu, lo[d], o));
      hi[d] = fmax(hi[d], __shfl_down_sync(0xffffffffu, hi[d], o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int d = 0; d < 3; d++) {
      atomic_min_double(&bounds[d], lo[d]);
      atomic_max_double(&bounds[3 + d], hi[d]);
    }
  }
}

// centre = box centre ; also emit the Morton scale
__global__ void centre_kernel(const double* bounds, double* centre) {
  if (threadIdx.x < 3) {
    const double lo = bounds[threadIdx.x], hi = bounds[3 + threadIdx.x];
    centre[threadIdx.x] = (lo <= hi) ? 0.5 * (lo + hi) : 0.0;
  }
  if (threadIdx.x == 3) {
    double ext = 0.0;
    for (int d = 0; d < 3; d++) ext = fmax(ext, bounds[3 + d] - bounds[d]);
    centre[3] = ext > 0.0 ? ext : 1.0;  // largest extent
  }
}

__device__ int d_use_hilbert = 1;  // space-filling curve of the source order: 1 Hilbert, 0 Morton (profiling switch)
cudaError_t set_source_curve(int hilbert) { return cudaMemcpyToSymbol(d_use_hilbert, &hilbert, sizeof(int)); }

__device__ __forceinline__ uint64_t spread21(uint64_t x) {  // 21 bits -> every third bit
  x &= 0x1fffffull;
  x = (x | x << 32) & 0x1f00000000ffffull;
  x = (x | x << 16) & 0x1f0000ff0000ffull;
  x = (x | x << 8) & 0x100f00f00f00f00full;
  x = (x | x << 4) & 0x10c30c30c30c30c3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}


/// 63-bit space-filling-curve key of a finite centred point (h = half extent of the cloud's box, inv_ext = (2^21 - 1) / extent).
__device__ __forceinline__ uint64_t curve_key_finite(double x, double y, double z, double h, double inv_ext) {
  const uint64_t kx = static_cast<uint64_t>(fmin(fmax((x + h) * inv_ext, 0.0), 2097151.0));
  const uint64_t ky = static_cast<uint64_t>(fmin(fmax((y + h) * inv_ext, 0.0), 2097151.0));
  const uint64_t kz = static_cast<uint64_t>(fmin(fmax((z + h) * inv_ext, 0.0), 2097151.0));
  if (!d_use_hilbert) return spread21(kx) | (spread21(ky) << 1) | (spread21(kz) << 2);  // Morton
  // Hilbert index (Skilling's transpose algorithm, 21 bits x 3): unlike the Z-curve it has no jumps, so 32 consecutive
  // points form a tighter patch
  uint32_t X[3] = {static_cast<uint32_t>(kx), static_cast<uint32_t>(ky), static_cast<uint32_t>(kz)};
  const uint32_t M = 1u << 20;
  for (uint32_t Q = M; Q > 1; Q >>= 1) {
    const uint32_t Pm = Q - 1;
#pragma unroll
    for (int a = 0; a < 3; a++) {
      if (X[a] & Q) {
        X[0] ^= Pm;
      } else {
        const uint32_t t = (X[0] ^ X[a]) & Pm;
        X[0] ^= t;
        X[a] ^= t;
      }
    }
  }
  X[1] ^= X[0];
  X[2] ^= X[1];
  uint32_t t = 0;
  for (uint32_t Q = M; Q > 1; Q >>= 1)
    if (X[2] & Q) t ^= Q - 1;
  X[0] ^= t;
  X[1] ^= t;
  X[2] ^= t;
  return (spread21(X[0]) << 2) | (spread21(X[1]) << 1) | spread21(X[2]);
}
/// The sort key of a point: a non-finite point gets the largest 63-bit key and every finite point a smaller one, so that the stable
/// sort stores the non-finite points after every finite point of their cloud, and the finite points at the positions they have in the
/// cloud without them.
constexpr uint64_t kCurveKeyNonFinite = (1ull << 63) - 1ull;
__device__ __forceinline__ uint64_t curve_key(double x, double y, double z, double h, double inv_ext) {
  if (!point_is_finite(x, y, z)) return kCurveKeyNonFinite;
  const uint64_t k = curve_key_finite(x, y, z, h, inv_ext);
  return k < kCurveKeyNonFinite ? k : kCurveKeyNonFinite - 1ull;
}

// raw (double AoS) -> centred float4 in ORIGINAL order (w = index), optional features, optional curve key
__global__ void convert_kernel(const double4* __restrict__ pts, const double4* __restrict__ normals, const double* __restrict__ covs, size_t n,
                               const double* __restrict__ centre, float4* out_pts, float4* out_normals, float4* out_covA, float4* out_covB,
                               uint64_t* keys, uint32_t* vals, float4* out_lo) {
  const double cx = centre[0], cy = centre[1], cz = centre[2];
  const double inv_ext = 2097151.0 / centre[3];
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const double4 p = pts[i];
    const double x = p.x - cx, y = p.y - cy, z = p.z - cz;
    out_pts[i] = centred_store_point(p, x, y, z, static_cast<uint32_t>(i));
    // what the rounding to FP32 dropped (hi + lo carries ~48 bits of x - c): the feature estimation ranks its neighbour candidates and
    // sums its covariances on the exact coordinates, so that its neighbour SETS are the reference's, not FP32 near-tie variants of them
    if (out_lo) out_lo[i] = make_float4((float)(x - (double)(float)x), (float)(y - (double)(float)y), (float)(z - (double)(float)z), 0.f);
    if (normals) {
      const double4 nn = normals[i];
      out_normals[i] = make_float4((float)nn.x, (float)nn.y, (float)nn.z, 0.f);
    }
    if (covs) {
      const double* c = covs + i * 16;
      out_covA[i] = pack_covA(c);
      out_covB[i] = pack_covB(c);
    }
    if (keys) {
      keys[i] = curve_key(x, y, z, 0.5 * centre[3], inv_ext);
      vals[i] = static_cast<uint32_t>(i);
    }
  }
}

// rank[perm[j]] = j: where the point with original index i ends up in the search order
__global__ void inverse_perm_kernel(const uint32_t* __restrict__ perm, size_t n, uint32_t* rank) {
  for (size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; j < n; j += static_cast<size_t>(gridDim.x) * blockDim.x) rank[perm[j]] = static_cast<uint32_t>(j);
}

// one CHUNK of raw 4x4 double covariances (original indices first .. first + n) -> packed floats written straight to their place in
// the search order (and, optionally, to the original-order copy): the chunk is converted while the next one is still on the PCIe bus
__global__ void convert_cov_scatter_kernel(const double* __restrict__ covs, size_t first, size_t n, const uint32_t* __restrict__ rank, float4* outA,
                                           float4* outB, float4* origA, float4* origB) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const double* c = covs + (first + i) * 16;
    const float4 a = pack_covA(c), b = pack_covB(c);
    const uint32_t r = rank[first + i];
    outA[r] = a;
    outB[r] = b;
    if (origA) {
      origA[first + i] = a;
      origB[first + i] = b;
    }
  }
}

// ---- many source clouds stored in one pass (sgb_source_set_batch): cloud c = points off[c] .. off[c+1], each stored exactly as
// store_source stores it alone.  Here because the curve (curve_key, d_use_hilbert) must have one definition per library.
// One CTA per cloud: its bounds [6] and centre [4]
__global__ void __launch_bounds__(kBoxBlock) clouds_box_kernel(const double4* __restrict__ pts, const uint32_t* __restrict__ off, double* bounds, double* centres) {
  const uint32_t c = blockIdx.x;
  cta_box_centre(pts, off[c], off[c + 1], bounds + 6 * static_cast<size_t>(c), centres + 4 * static_cast<size_t>(c));
}

// convert_kernel's arithmetic about each point's own cloud centre: centred FP32 point in original order (w = index within the cloud),
// curve key, vals = global position
__global__ void clouds_convert_kernel(const double4* __restrict__ pts, uint32_t n, const uint32_t* __restrict__ off, uint32_t n_clouds,
                                      const double* __restrict__ centres, float4* out_pts, uint64_t* keys, uint32_t* vals) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t c = owner_of(off, n_clouds, i);
    const double* centre = centres + 4 * static_cast<size_t>(c);
    const double cx = centre[0], cy = centre[1], cz = centre[2];
    const double inv_ext = 2097151.0 / centre[3];
    const double4 p = pts[i];
    const double x = p.x - cx, y = p.y - cy, z = p.z - cz;
    out_pts[i] = centred_store_point(p, x, y, z, i - off[c]);
    keys[i] = curve_key(x, y, z, 0.5 * centre[3], inv_ext);
    vals[i] = i;
  }
}

// after the stable key sort (vals = global positions in key order): the cloud of each, the key of the stable sort by cloud
__global__ void clouds_ids_kernel(const uint32_t* __restrict__ vals, uint32_t n, const uint32_t* __restrict__ off, uint32_t n_clouds, uint64_t* keys) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) keys[j] = owner_of(off, n_clouds, vals[j]);
}

// order = global positions in (cloud, key, index) order, the per-cloud sort's order: every cloud's search-order points, the
// search order -> index within the cloud (the converted point's w), covariances packed into that order
__global__ void clouds_store_kernel(const uint32_t* __restrict__ order, uint32_t n, const float4* __restrict__ orig, const double* __restrict__ covs, float4* pts,
                                    uint32_t* perm, float4* covA, float4* covB) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const uint32_t g = order[j];
    const float4 f = orig[g];
    pts[j] = f;
    perm[j] = static_cast<uint32_t>(__float_as_int(f.w));
    if (covs) {
      const double* c = covs + static_cast<size_t>(g) * 16;
      covA[j] = pack_covA(c);
      covB[j] = pack_covB(c);
    }
  }
}

// curve keys of points that are already on the device in centred FP32 form (target: device-side tree construction)
__global__ void curve_keys_kernel(const float4* __restrict__ pts, size_t n, const double* __restrict__ centre, uint64_t* keys, uint32_t* vals) {
  const double inv_ext = 2097151.0 / centre[3], h = 0.5 * centre[3];
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 p = pts[i];
    keys[i] = curve_key(p.x, p.y, p.z, h, inv_ext);
    vals[i] = static_cast<uint32_t>(i);
  }
}

// ---------------------------------------------------------------------------------------------
// Device-side construction of the search structure (replaces KdTreeBuilder::build_tree, ann/kdtree.hpp:74-131, and its
// OMP / TBB variants).  Exact nearest-neighbour results do not depend on how the hierarchy is formed, so instead of
// recursive median splits the tree is a linear BVH: points sorted along the Hilbert curve, leaves = runs of kLbvhLeaf
// consecutive points, hierarchy = the implicit perfect binary tree over P = 2^ceil(log2(#leaves)) leaf slots (node i has
// children 2i+1, 2i+2; missing leaves are empty boxes that no query ever enters).  Every step is a data-parallel kernel;
// the output is the same 64-byte packet record array the search kernel consumes.
// The helpers and the bodies of the shared-memory refinement and of the record kernels are in sgb_device.cuh, which the many-tree
// build (sgb_forest.cu) shares.
// ---------------------------------------------------------------------------------------------
// ---- median-split refinement (device-side kd construction): one pass per level ------------------------------------
__global__ void kd_boxes_init_kernel(uint32_t* boxes, uint32_t count) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < count * 6u) boxes[t] = (t % 6u) < 3u ? 0xFFFFFFFFu : 0u;
}

__global__ void kd_boxes_kernel(const float4* __restrict__ pts, uint32_t n, uint32_t count, uint32_t* boxes) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = i < n;
  const uint32_t idx = valid ? i : n - 1u;
  const float4 p = pts[idx];
  const uint32_t node = tree_node_of(idx, count, n);
  uint32_t v[6] = {box_lo_word(p.x), box_lo_word(p.y), box_lo_word(p.z), box_hi_word(p.x), box_hi_word(p.y), box_hi_word(p.z)};
  // pre-reduction: whole CTA in one node (upper levels: otherwise thousands of atomics hit the same six words), else
  // whole warp in one node, else per-thread atomics (deepest levels, little contention)
  __shared__ uint32_t s_box[6];
  __shared__ uint32_t s_first_node, s_last_node;
  if (threadIdx.x == 0) s_first_node = node;
  if (threadIdx.x == blockDim.x - 1) s_last_node = node;
  if (threadIdx.x < 6) s_box[threadIdx.x] = threadIdx.x < 3 ? 0xFFFFFFFFu : 0u;
  __syncthreads();
  const bool cta_uniform = s_first_node == s_last_node;  // positions are contiguous: equal ends => one node
  const uint32_t node0 = __shfl_sync(0xffffffffu, node, 0);
  if (__all_sync(0xffffffffu, node == node0)) {
#pragma unroll
    for (int a = 0; a < 3; a++) {
      v[a] = __reduce_min_sync(0xffffffffu, v[a]);
      v[3 + a] = __reduce_max_sync(0xffffffffu, v[3 + a]);
    }
    if ((threadIdx.x & 31u) == 0) {
      uint32_t* dst = cta_uniform ? s_box : &boxes[node * 6];
#pragma unroll
      for (int a = 0; a < 3; a++) {
        atomicMin(&dst[a], v[a]);
        atomicMax(&dst[3 + a], v[3 + a]);
      }
    }
    if (cta_uniform) {
      __syncthreads();
      if (threadIdx.x < 3) atomicMin(&boxes[node * 6 + threadIdx.x], s_box[threadIdx.x]);
      if (threadIdx.x >= 3 && threadIdx.x < 6) atomicMax(&boxes[node * 6 + threadIdx.x], s_box[threadIdx.x]);
    }
  } else if (valid) {
#pragma unroll
    for (int a = 0; a < 3; a++) {
      atomicMin(&boxes[node * 6 + a], v[a]);
      atomicMax(&boxes[node * 6 + 3 + a], v[3 + a]);
    }
  }
}

// key = (node << 32) | coordinate along the node's widest axis: sorting by it orders every node's points along its split
// axis, and the balanced position boundaries of the next level then ARE the median splits
__global__ void kd_keys_kernel(const float4* __restrict__ pts, uint32_t n, uint32_t count, const uint32_t* __restrict__ boxes, uint64_t* keys) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t node = tree_node_of(i, count, n);
  const float ex = float_unflip(boxes[node * 6 + 3]) - float_unflip(boxes[node * 6 + 0]);
  const float ey = float_unflip(boxes[node * 6 + 4]) - float_unflip(boxes[node * 6 + 1]);
  const float ez = float_unflip(boxes[node * 6 + 5]) - float_unflip(boxes[node * 6 + 2]);
  const float4 p = pts[i];
  const float c = ex >= ey ? (ex >= ez ? p.x : p.z) : (ey >= ez ? p.y : p.z);
  keys[i] = (static_cast<uint64_t>(node) << 32) | float_flip(c);
}

// The same median-split refinement for every subtree of at most kKdSegMax points in ONE launch: CTA b refines node b of level `level0`
// in shared memory (kd_refine_segment).  Above level0 a level is ~12 launches (boxes, keys, radix sort, gather); for a 16k-point frame
// that was 9 levels = ~110 launches of pure launch latency, now 3 levels + this kernel.
__global__ void __launch_bounds__(1024) kd_refine_smem_kernel(float4* __restrict__ leaf_pts, uint32_t* __restrict__ perm, uint32_t n, uint32_t level0, uint32_t levels) {
  kd_refine_segment(leaf_pts, perm, 0u, blockIdx.x, n, level0, levels);
}

// one warp per leaf slot: bounding box of its (at most 32) consecutive points -> the parent's child record
__global__ void lbvh_leaf_kernel(const float4* __restrict__ leaf_pts, uint32_t n, uint32_t P, float4* pnodes) {
  const uint32_t slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (slot >= P) return;
  const uint32_t first = tree_bound(slot, P, n), last = tree_bound(slot + 1u, P, n);
  float lo[3], hi[3];
  lbvh_leaf_box(leaf_pts, 0u, first, last, lane, lo, hi);
  if (lane == 0) {
    const uint32_t cnt = last - first;
    lbvh_store_child(pnodes, (P - 1u) + slot, lo, hi, cnt ? first : 0u, cnt);  // cnt == 0: inverted box, never entered
  }
}

// one thread per inner node of a level (children records complete): union box -> the parent's child record
__global__ void lbvh_level_kernel(uint32_t level_first, uint32_t level_count, float4* pnodes) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= level_count) return;
  lbvh_inner_record(pnodes, level_first + t);
}

cudaError_t launch_curve_keys(const float4* pts, size_t n, const double* centre4, uint64_t* keys, uint32_t* vals, int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  size_t g = (n + 255) / 256;
  if (g > static_cast<size_t>(sm_count) * 8) g = static_cast<size_t>(sm_count) * 8;
  curve_keys_kernel<<<static_cast<int>(g), 256, 0, st>>>(pts, n, centre4, keys, vals);
  return cudaGetLastError();
}

/// pnodes: (P - 1) * 4 float4 records, P = number of leaf slots (power of two >= 2).  Returns the number of launches in *launches.
cudaError_t launch_lbvh_build(const float4* leaf_pts, uint32_t n, uint32_t P, float4* pnodes, int* launches, cudaStream_t st) {
  const uint32_t warps_per_block = 8;
  lbvh_leaf_kernel<<<(P + warps_per_block - 1) / warps_per_block, warps_per_block * 32, 0, st>>>(leaf_pts, n, P, pnodes);
  int count = 1;
  for (uint32_t level_count = P >> 1; level_count >= 2; level_count >>= 1) {  // deepest inner level first; the root (level_count 1) has no parent
    const uint32_t level_first = level_count - 1u;
    lbvh_level_kernel<<<(level_count + 255) / 256, 256, 0, st>>>(level_first, level_count, pnodes);
    count++;
  }
  if (launches) *launches = count;
  return cudaGetLastError();
}

/// One level of the median-split refinement: boxes of the `count` nodes of this level over the points in their current
/// order, then the sort keys.  The caller sorts (keys, perm) and re-gathers the points.
cudaError_t launch_kd_level_keys(const float4* cur_pts, uint32_t n, uint32_t count, uint32_t* boxes, uint64_t* keys, cudaStream_t st) {
  kd_boxes_init_kernel<<<(count * 6u + 255u) / 256u, 256, 0, st>>>(boxes, count);
  kd_boxes_kernel<<<(n + 255u) / 256u, 256, 0, st>>>(cur_pts, n, count, boxes);
  kd_keys_kernel<<<(n + 255u) / 256u, 256, 0, st>>>(cur_pts, n, count, boxes, keys);
  return cudaGetLastError();
}

/// first level whose nodes hold at most kKdSegMax points (from there on kd_refine_smem_kernel refines whole subtrees in shared memory)
uint32_t kd_smem_first_level(uint32_t n, uint32_t levels) {
  uint32_t l = 0;
  while (l < levels && (static_cast<uint64_t>(n) + (1ull << l) - 1ull) / (1ull << l) > kKdSegMax) l++;
  return l;
}
cudaError_t launch_kd_refine_smem(float4* leaf_pts, uint32_t* perm, uint32_t n, uint32_t level0, uint32_t levels, cudaStream_t st) {
  if (level0 >= levels) return cudaSuccess;
  const cudaError_t e = allow_dynamic_smem(kd_refine_smem_kernel, kKdRefineSmem);
  if (e != cudaSuccess) return e;
  kd_refine_smem_kernel<<<1u << level0, 1024, kKdRefineSmem, st>>>(leaf_pts, perm, n, level0, levels);
  return cudaGetLastError();
}

cudaError_t sort_pairs_u64_u32_bits(void* d_temp, size_t& temp_bytes, const uint64_t* keys_in, uint64_t* keys_out, const uint32_t* vals_in, uint32_t* vals_out,
                                    size_t n, int end_bit, cudaStream_t st) {
  return cub::DeviceRadixSort::SortPairs(d_temp, temp_bytes, keys_in, keys_out, vals_in, vals_out, static_cast<int>(n), 0, end_bit, st);
}

// out[j] = in[perm[j]] for up to four float4 streams (leaf ordering of the target / Morton ordering of the source)
__global__ void gather_kernel(const uint32_t* __restrict__ perm, size_t n, const float4* __restrict__ in0, float4* out0, const float4* __restrict__ in1,
                              float4* out1, const float4* __restrict__ in2, float4* out2, const float4* __restrict__ in3, float4* out3) {
  for (size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; j < n; j += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const uint32_t s = perm[j];
    if (in0) out0[j] = in0[s];
    if (in1) out1[j] = in1[s];
    if (in2) out2[j] = in2[s];
    if (in3) out3[j] = in3[s];
  }
}

// out[perm[j]] = in[j]: leaf order -> original order (features estimated on the device in leaf order)
__global__ void scatter_kernel(const uint32_t* __restrict__ perm, size_t n, const float4* __restrict__ in0, float4* out0, const float4* __restrict__ in1,
                               float4* out1, const float4* __restrict__ in2, float4* out2) {
  for (size_t j = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; j < n; j += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const uint32_t d = perm[j];
    if (in0) out0[d] = in0[j];
    if (in1) out1[d] = in1[j];
    if (in2) out2[d] = in2[j];
  }
}

// Morton-rank order -> chunk-transposed order (see LinParams / DevSource::run): out[p] = in[rank(p)]
__global__ void chunk_transpose_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, size_t n, uint32_t K) {
  const size_t chunk_pts = 32ull * K;
  for (size_t p = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; p < n; p += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t chunk = p / chunk_pts, r = p % chunk_pts;
    size_t m = p;
    if ((chunk + 1) * chunk_pts <= n) m = chunk * chunk_pts + (r % 32) * K + r / 32;  // full chunks only; the ragged tail keeps Morton order
    out[p] = in[m];
  }
}

// correspondences in the caller's order: out[perm[i]] = original target index (or voxel id << 32)
__global__ void correspondences_kernel(const uint32_t* __restrict__ corr, const uint32_t* __restrict__ perm, size_t n, const float4* __restrict__ tgt_pts,
                                       int voxel, uint64_t* out) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const uint32_t k = corr[i];
    uint64_t v = ~0ull;
    if (k != kNone) v = voxel ? (static_cast<uint64_t>(k) << 32) : static_cast<uint64_t>(static_cast<uint32_t>(__float_as_int(tgt_pts[k].w)));
    out[perm[i]] = v;
  }
}

// the same for a member of a multi-map voxel target: out[perm[i]] = (voxel id within its map) << 32, the id stored in tgt_pts[k].w
__global__ void voxelmaps_correspondences_kernel(const uint32_t* __restrict__ corr, const uint32_t* __restrict__ perm, size_t n,
                                                 const float4* __restrict__ tgt_pts, uint64_t* out) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const uint32_t k = corr[i];
    out[perm[i]] = k == kNone ? ~0ull : static_cast<uint64_t>(static_cast<uint32_t>(__float_as_int(tgt_pts[k].w))) << 32;
  }
}

static int grid_for(size_t n, int block, int cap) {
  size_t g = (n + block - 1) / block;
  if (g < 1) g = 1;
  if (g > static_cast<size_t>(cap)) g = cap;
  return static_cast<int>(g);
}

cudaError_t launch_bounds_centre(const double* d_pts4, size_t n, double* d_bounds6, double* d_centre4, int sm_count, cudaStream_t st) {
  bounds_init_kernel<<<1, 32, 0, st>>>(d_bounds6);
  if (n) bounds_kernel<<<grid_for(n, 256, sm_count * 8), 256, 0, st>>>(reinterpret_cast<const double4*>(d_pts4), n, d_bounds6);
  centre_kernel<<<1, 32, 0, st>>>(d_bounds6, d_centre4);
  return cudaGetLastError();
}

cudaError_t launch_convert(const double* d_pts4, const double* d_normals4, const double* d_covs16, size_t n, const double* d_centre4, float4* out_pts,
                           float4* out_normals, float4* out_covA, float4* out_covB, uint64_t* keys, uint32_t* vals, int sm_count, cudaStream_t st, float4* out_lo) {
  if (!n) return cudaSuccess;
  convert_kernel<<<grid_for(n, 256, sm_count * 8), 256, 0, st>>>(reinterpret_cast<const double4*>(d_pts4), reinterpret_cast<const double4*>(d_normals4), d_covs16,
                                                                 n, d_centre4, out_pts, out_normals, out_covA, out_covB, keys, vals, out_lo);
  return cudaGetLastError();
}

cudaError_t launch_inverse_perm(const uint32_t* perm, size_t n, uint32_t* rank, int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  inverse_perm_kernel<<<grid_for(n, 256, sm_count * 8), 256, 0, st>>>(perm, n, rank);
  return cudaGetLastError();
}

cudaError_t launch_convert_cov_scatter(const double* d_covs16, size_t first, size_t n, const uint32_t* rank, float4* outA, float4* outB, float4* origA,
                                       float4* origB, int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  convert_cov_scatter_kernel<<<grid_for(n, 256, sm_count * 8), 256, 0, st>>>(d_covs16, first, n, rank, outA, outB, origA, origB);
  return cudaGetLastError();
}

cudaError_t launch_gather(const uint32_t* perm, size_t n, const float4* in0, float4* out0, const float4* in1, float4* out1, const float4* in2, float4* out2,
                          const float4* in3, float4* out3, int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  gather_kernel<<<grid_for(n, 256, sm_count * 8), 256, 0, st>>>(perm, n, in0, out0, in1, out1, in2, out2, in3, out3);
  return cudaGetLastError();
}

cudaError_t launch_scatter(const uint32_t* perm, size_t n, const float4* in0, float4* out0, const float4* in1, float4* out1, const float4* in2, float4* out2,
                           int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  scatter_kernel<<<grid_for(n, 256, sm_count * 8), 256, 0, st>>>(perm, n, in0, out0, in1, out1, in2, out2);
  return cudaGetLastError();
}

cudaError_t launch_correspondences(const uint32_t* corr, const uint32_t* perm, size_t n, const float4* tgt_pts, int voxel, uint64_t* out, int sm_count,
                                   cudaStream_t st) {
  if (!n) return cudaSuccess;
  correspondences_kernel<<<grid_for(n, 256, sm_count * 8), 256, 0, st>>>(corr, perm, n, tgt_pts, voxel, out);
  return cudaGetLastError();
}

cudaError_t launch_voxelmaps_correspondences(const uint32_t* corr, const uint32_t* perm, size_t n, const float4* tgt_pts, uint64_t* out, int sm_count,
                                             cudaStream_t st) {
  if (!n) return cudaSuccess;
  voxelmaps_correspondences_kernel<<<grid_for(n, 256, sm_count * 8), 256, 0, st>>>(corr, perm, n, tgt_pts, out);
  return cudaGetLastError();
}

cudaError_t launch_store_clouds(const StoreClouds& s, cudaStream_t st) {
  const uint32_t n = s.n;
  clouds_box_kernel<<<s.n_clouds, 256, 0, st>>>(reinterpret_cast<const double4*>(s.points), s.offsets, s.bounds, s.centres);
  const int g = grid_for(n, 256, s.sm_count * 8);
  clouds_convert_kernel<<<g, 256, 0, st>>>(reinterpret_cast<const double4*>(s.points), n, s.offsets, s.n_clouds, s.centres, s.orig_pts, s.keys_a, s.vals_a);
  size_t tb = s.sort_temp_bytes;
  cudaError_t e = sort_pairs_u64_u32_bits(s.sort_temp, tb, s.keys_a, s.keys_b, s.vals_a, s.vals_b, n, 63, st);
  if (e != cudaSuccess) return e;
  clouds_ids_kernel<<<g, 256, 0, st>>>(s.vals_b, n, s.offsets, s.n_clouds, s.keys_a);
  tb = s.sort_temp_bytes;
  if ((e = sort_pairs_u64_u32_bits(s.sort_temp, tb, s.keys_a, s.keys_b, s.vals_b, s.vals_a, n, s.cloud_bits, st)) != cudaSuccess) return e;
  clouds_store_kernel<<<g, 256, 0, st>>>(s.vals_a, n, s.orig_pts, s.covs, s.pts, s.perm, s.covA, s.covB);
  return cudaGetLastError();
}

cudaError_t launch_chunk_transpose(const uint32_t* in, uint32_t* out, size_t n, uint32_t K, int sm_count, cudaStream_t st) {
  if (!n) return cudaSuccess;
  chunk_transpose_kernel<<<grid_for(n, 256, sm_count * 8), 256, 0, st>>>(in, out, n, K);
  return cudaGetLastError();
}

}  // namespace sgb
