// SPDX-License-Identifier: MIT
// The factor / reduction phase of linearize, and the per-thread search kept as a profiling switch (DESIGN.md §4):
//   nn_search_kernel      (SGB_SEARCH=1) transform + exact kd-tree NN, one query per thread -- the product path searches
//                         with sgb_grid.cu + sgb_kernels_packet.cu instead
//   factor_reduce_kernel  streams source + correspondences, gathers the matched target point / covariance with cp.async two
//                         tiles ahead, FP64 rejector + factor algebra (source frame), block reduction, ticket-tree finish
//                         and -- with several GPUs -- the exchange of the sums over the peers' mailboxes
// Search and factor phases run back to back on the context's stream; the only extra traffic is the 4-byte correspondence
// per point that sgb_error()/sgb_correspondences() need anyway.
#include <cfloat>
#include <cstdlib>

#include "sgb_device.cuh"
#include "sgb_kernels.h"

namespace sgb {

#ifdef SGB_PROFILING
// ---------------------------------------------------------------------------------------------------------------
// Phase 1.  Every lane owns a run of K consecutive points of the Morton curve (chunk-transposed layout) and walks
// it INDEPENDENTLY of the other lanes: a lane that finishes a query starts its next one in the same iteration of the
// warp loop instead of idling until the slowest query of the warp is done.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLinBlock) nn_search_kernel(const __grid_constant__ LinParams P) {
  extern __shared__ uint2 s_stack[];
  const double* R = P.T;
  const double csx = P.src.centre[0], csy = P.src.centre[1], csz = P.src.centre[2];
  const double tpx = R[0] * csx + R[1] * csy + R[2] * csz + P.T[9] - P.tgt.centre[0];
  const double tpy = R[3] * csx + R[4] * csy + R[5] * csz + P.T[10] - P.tgt.centre[1];
  const double tpz = R[6] * csx + R[7] * csy + R[8] * csz + P.T[11] - P.tgt.centre[2];
  // the FP32 query is the FP64 transform rounded once (same value phase 2 derives its residual from)
  const KdNode* __restrict__ nodes = P.tgt.nodes;
  const float4* __restrict__ pts = P.tgt.pts;

  const uint32_t K = P.src.run, chunk_pts = 32u * K;
  const uint32_t n_chunks = (P.src.n + chunk_pts - 1) / chunk_pts;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  uint2* my_stack = s_stack + threadIdx.x;

  for (uint32_t chunk = warp; chunk < n_chunks; chunk += n_warps) {
    uint32_t k = 0, chain = kNone;
    bool active = false;
    uint32_t i = 0, node = 0, best = kNone;
    int sp = 0;
    float fx = 0.f, fy = 0.f, fz = 0.f, best_d = 0.f;
    for (;;) {
      if (!active) {  // start the lane's next query
        i = chunk * chunk_pts + k * 32u + lane;
        if (k >= K || i >= P.src.n) break;
        const float4 s = __ldg(&P.src.pts[i]);
        const double sx = s.x, sy = s.y, sz = s.z;
        fx = static_cast<float>(R[0] * sx + R[1] * sy + R[2] * sz + tpx);
        fy = static_cast<float>(R[3] * sx + R[4] * sy + R[5] * sz + tpy);
        fz = static_cast<float>(R[6] * sx + R[7] * sy + R[8] * sz + tpz);
        best_d = P.max_dist_sq;
        best = kNone;
        const uint32_t prev = P.use_prev ? P.corr[i] : kNone;
        if (prev != kNone) {
          const float4 t = __ldg(&pts[prev]);
          const float dx = t.x - fx, dy = t.y - fy, dz = t.z - fz;
          const float d = dx * dx + dy * dy + dz * dz;
          if (d < best_d) {
            best_d = d;
            best = prev;
          }
        }
        if (chain != kNone && chain != prev) {
          const float4 t = __ldg(&pts[chain]);
          const float dx = t.x - fx, dy = t.y - fy, dz = t.z - fz;
          const float d = dx * dx + dy * dy + dz * dz;
          if (d < best_d) {
            best_d = d;
            best = chain;
          }
        }
        node = 0;
        sp = 0;
        active = true;
      }
      // descend to a leaf
      KdNode nd = __ldg(&nodes[node]);
      uint32_t kind = nd.y & 3u;
      while (kind != 3u) {
        const float qv = kind == 0u ? fx : (kind == 1u ? fy : fz);
        const float diff = qv - __uint_as_float(nd.x);
        const uint32_t right = nd.y >> 2, left = node + 1u;
        const bool go_left = diff < 0.0f;
        const float cut = diff * diff;
        if (cut < best_d) {
          my_stack[sp * kLinBlock] = make_uint2(go_left ? right : left, __float_as_uint(cut));
          sp++;
        }
        node = go_left ? left : right;
        nd = __ldg(&nodes[node]);
        kind = nd.y & 3u;
      }
      {  // scan the leaf
        const uint32_t first = nd.x, cnt = nd.y >> 2;
        const float4* lp = pts + first;
        for (uint32_t j = 0; j < cnt; j++) {
          const float4 t = __ldg(&lp[j]);
          const float dx = t.x - fx, dy = t.y - fy, dz = t.z - fz;
          const float d = dx * dx + dy * dy + dz * dz;
          if (d < best_d) {
            best_d = d;
            best = first + j;
          }
        }
      }
      // next pending subtree that can still hold a closer point, else the query is finished
      bool resumed = false;
      while (sp > 0) {
        sp--;
        const uint2 e = my_stack[sp * kLinBlock];
        if (__uint_as_float(e.y) < best_d) {
          node = e.x;
          resumed = true;
          break;
        }
      }
      if (!resumed) {
        P.corr[i] = best;
        if (best != kNone) chain = best;
        k++;
        active = false;
      }
    }
  }
}

#endif  // SGB_PROFILING

// ---------------------------------------------------------------------------------------------------------------
// Phase 2.  One point per thread per tile of kLinBlock points.  The gather of the matched target point / covariance
// depends on the correspondence index, and the FP64 factor algebra holds ~128 registers (4 CTAs / SM), so plain loads
// left the kernel latency-bound (few issue slots used, far from the HBM bandwidth).  The loads are therefore issued two
// tiles ahead with cp.async into a per-thread landing zone in shared memory:
//   A(t+2): correspondence index + source point / covariance (coalesced)
//   B(t+1): target point / normal / covariance gathered through the index A(t+1) brought in
//   C(t)  : FP64 rejector + factor algebra on the operands that landed during the previous tile's arithmetic
// Every thread only reads what it copied itself, so the pipeline needs no barrier, just cp.async.wait_group.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem));
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

template <int FACTOR>
struct FactorFields {
  // landing-zone slots (float4 each): source point [+ source covariance], target point [+ normal | covariance]
  static constexpr int kSrc = FACTOR == 2 ? 3 : 1;
  static constexpr int kAll = FACTOR == 2 ? 6 : (FACTOR == 1 ? 3 : 2);
};
constexpr int kFactorStages = 3;

// NREG: register budget per thread = resident CTAs per SM (128 -> 4 CTAs x 4 warps, no spills; 96 -> 5 CTAs; 80 -> 6, both with spills and slower): the algebra is a chain of
// dependent FP64 operations and the kernel is short of warps, not of FP64 pipe.
// ERR: the same operand pipeline evaluating Reduction::error instead (cached correspondences, trial pose P.T, GICP precision matrix re-derived
// from the linearisation pose P.Tlin, one sum): the LM inner loop's kernel.  The plain grid-stride version of it (error_kernel, sgb_kernels.cu)
// waited on two dependent load round trips per point with nothing in flight: longer than the whole linearize algebra.
template <int FACTOR, int ROBUST, int NREG, bool ERR = false>
__global__ void __maxnreg__(NREG) factor_reduce_kernel(const __grid_constant__ LinParams P) {
  using F = FactorFields<FACTOR>;
  extern __shared__ float4 s_zone[];  // [kFactorStages][F::kAll][kLinBlock]
  __shared__ uint32_t s_corr[kFactorStages][kLinBlock];
  constexpr int NACC = ERR ? 1 : kAcc + 1;
  double acc[NACC];
#pragma unroll
  for (int k = 0; k < NACC; k++) acc[k] = 0.0;
  const double* R = P.T;
  const double csx = P.src.centre[0], csy = P.src.centre[1], csz = P.src.centre[2];
  const double tpx = R[0] * csx + R[1] * csy + R[2] * csz + P.T[9] - P.tgt.centre[0];
  const double tpy = R[3] * csx + R[4] * csy + R[5] * csz + P.T[10] - P.tgt.centre[1];
  const double tpz = R[6] * csx + R[7] * csy + R[8] * csz + P.T[11] - P.tgt.centre[2];
  const uint32_t n = P.src.n, n_tiles = (n + kLinBlock - 1u) / kLinBlock, tid = threadIdx.x;
  float4* zone = s_zone + tid;
  auto slot = [&](int stage, int f) { return zone + (stage * F::kAll + f) * kLinBlock; };
  auto issue_a = [&](uint32_t tile, int stage) {
    const uint32_t i = tile * kLinBlock + tid;
    if (tile < n_tiles && i < n) {
      cp_async4(&s_corr[stage][tid], &P.corr[i]);
      cp_async16(slot(stage, 0), &P.src.pts[i]);
      if (FACTOR == 2) {
        cp_async16(slot(stage, 1), &P.src.covA[i]);
        cp_async16(slot(stage, 2), &P.src.covB[i]);
      }
    } else {
      s_corr[stage][tid] = kNone;
    }
  };
  auto issue_b = [&](int stage) {
    const uint32_t best = s_corr[stage][tid];
    if (best == kNone) return;
    cp_async16(slot(stage, F::kSrc), &P.tgt.pts[best]);
    if (FACTOR == 1) cp_async16(slot(stage, F::kSrc + 1), &P.tgt.normals[best]);
    if (FACTOR == 2) {
      cp_async16(slot(stage, F::kSrc + 1), &P.tgt.covA[best]);
      cp_async16(slot(stage, F::kSrc + 2), &P.tgt.covB[best]);
    }
  };

  grid_dependency_wait();  // the search kernels wrote the correspondences
  const uint32_t G = gridDim.x;
  uint32_t tile = blockIdx.x;
  issue_a(tile, 0);
  cp_async_commit();
  cp_async_wait_all();
  issue_b(0);
  issue_a(tile + G, 1);
  cp_async_commit();
  int st = 0;
  for (; tile < n_tiles; tile += G) {
    cp_async_wait_all();  // B(tile) and A(tile + G) have landed
    const int st1 = st == kFactorStages - 1 ? 0 : st + 1, st2 = st1 == kFactorStages - 1 ? 0 : st1 + 1;
    issue_b(st1);
    issue_a(tile + 2u * G, st2);
    cp_async_commit();
    const uint32_t best = s_corr[st][tid];
    if (best != kNone) {
      const uint32_t i = tile * kLinBlock + tid;
      // operands out of this thread's landing zone; the per-point arithmetic is point_linearize_source / point_error (sgb_math.cuh)
      const float4 sp = *slot(st, 0);
      const float4 tq = *slot(st, F::kSrc);
      if (ERR) {
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        acc[0] += point_error<FACTOR, ROBUST>(R, tpx, tpy, tpz, P.Tlin, P.robust_c, sp, FACTOR == 2 ? *slot(st, 1) : z, FACTOR == 2 ? *slot(st, 2) : z, tq,
                                              FACTOR >= 1 ? *slot(st, F::kSrc + 1) : z, FACTOR == 2 ? *slot(st, F::kSrc + 2) : z);
      } else if (!point_linearize_source<FACTOR, ROBUST>(R, tpx, tpy, tpz, csx, csy, csz, P.max_dist_sq_d, P.robust_c, sp, slot(st, 1), slot(st, 2), tq,
                                                         slot(st, F::kSrc + 1), slot(st, F::kSrc + 2), acc)) {
        P.corr[i] = kNone;  // rejected: error() and sgb_correspondences() must not see it
      }
    }
    st = st1;
  }
  cp_async_wait_all();
  block_reduce_and_finish<NACC, !ERR>(acc, P.partials, P.ticket, P.out, P.comm);
}

constexpr int kFactorRegs = 128;  // 4 CTAs x 128 threads x 128 registers = the whole register file, no spills (120 left 32 B on the stack)
#ifdef SGB_PROFILING
static int factor_regs_switch() {  // SGB_FACTOR_REGS=96 / 80: GICP without robust kernel only (the bench workload)
  static const int v = std::getenv("SGB_FACTOR_REGS") ? std::atoi(std::getenv("SGB_FACTOR_REGS")) : kFactorRegs;
  return v;
}
#endif
template <int FACTOR, int ROBUST>
static cudaError_t launch_factor(const LinParams& P, int grid, cudaStream_t st) {
  const size_t smem = static_cast<size_t>(kFactorStages) * FactorFields<FACTOR>::kAll * kLinBlock * sizeof(float4);
#ifdef SGB_PROFILING
  if (FACTOR == 2 && ROBUST == 0 && factor_regs_switch() == 96) return launch_dependent(factor_reduce_kernel<2, 0, 96>, grid, kLinBlock, smem, st, P);
  if (FACTOR == 2 && ROBUST == 0 && factor_regs_switch() == 80) return launch_dependent(factor_reduce_kernel<2, 0, 80>, grid, kLinBlock, smem, st, P);
  if (FACTOR == 2 && ROBUST == 0 && factor_regs_switch() == 120) return launch_dependent(factor_reduce_kernel<2, 0, 120>, grid, kLinBlock, smem, st, P);
#endif
  return launch_dependent(factor_reduce_kernel<FACTOR, ROBUST, kFactorRegs>, grid, kLinBlock, smem, st, P);
}

template <int FACTOR, int ROBUST>
static cudaError_t launch_error_pipe(const LinParams& P, int grid, cudaStream_t st) {
  const size_t smem = static_cast<size_t>(kFactorStages) * FactorFields<FACTOR>::kAll * kLinBlock * sizeof(float4);
  factor_reduce_kernel<FACTOR, ROBUST, kFactorRegs, true><<<grid, kLinBlock, smem, st>>>(P);
  return cudaGetLastError();
}
template <int FACTOR, int ROBUST>
static int error_ctas_per_sm() {
  static int cached = 0;
  if (cached) return cached;
  const size_t smem = static_cast<size_t>(kFactorStages) * FactorFields<FACTOR>::kAll * kLinBlock * sizeof(float4);
  cudaFuncSetAttribute(factor_reduce_kernel<FACTOR, ROBUST, kFactorRegs, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  int nb = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, factor_reduce_kernel<FACTOR, ROBUST, kFactorRegs, true>, kLinBlock, smem) != cudaSuccess || nb < 1) nb = 1;
  cached = nb;
  return nb;
}

// resident CTAs per SM of one instantiation (the grid is sized to exactly one wave: a partial second wave of this
// register-heavy kernel runs one CTA per SM for a good part of the kernel's duration)
template <int FACTOR, int ROBUST>
static int factor_ctas_per_sm() {
  static int cached = 0;
  if (cached) return cached;
  const size_t smem = static_cast<size_t>(kFactorStages) * FactorFields<FACTOR>::kAll * kLinBlock * sizeof(float4);
  int nb = 0;
#ifdef SGB_PROFILING
  if (FACTOR == 2 && ROBUST == 0 && (factor_regs_switch() == 96 || factor_regs_switch() == 80)) {
    if (factor_regs_switch() == 96) {
      cudaFuncSetAttribute(factor_reduce_kernel<2, 0, 96>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
      cudaFuncSetAttribute(factor_reduce_kernel<2, 0, 96>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, factor_reduce_kernel<2, 0, 96>, kLinBlock, smem) != cudaSuccess || nb < 1) nb = 1;
    } else {
      cudaFuncSetAttribute(factor_reduce_kernel<2, 0, 80>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
      cudaFuncSetAttribute(factor_reduce_kernel<2, 0, 80>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, factor_reduce_kernel<2, 0, 80>, kLinBlock, smem) != cudaSuccess || nb < 1) nb = 1;
    }
    cached = nb;
    return nb;
  }
#endif
  cudaFuncSetAttribute(factor_reduce_kernel<FACTOR, ROBUST, kFactorRegs>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, factor_reduce_kernel<FACTOR, ROBUST, kFactorRegs>, kLinBlock, smem) != cudaSuccess || nb < 1) nb = 1;
  cached = nb;
  return nb;
}

#define SGB_SPLIT_DISPATCH(FN, ...)                                \
  switch (factor * 3 + robust) {                                   \
    case 0: return FN<0, 0>(__VA_ARGS__);                          \
    case 1: return FN<0, 1>(__VA_ARGS__);                          \
    case 2: return FN<0, 2>(__VA_ARGS__);                          \
    case 3: return FN<1, 0>(__VA_ARGS__);                          \
    case 4: return FN<1, 1>(__VA_ARGS__);                          \
    case 5: return FN<1, 2>(__VA_ARGS__);                          \
    case 6: return FN<2, 0>(__VA_ARGS__);                          \
    case 7: return FN<2, 1>(__VA_ARGS__);                          \
    case 8: return FN<2, 2>(__VA_ARGS__);                          \
  }
cudaError_t launch_error_pipelined(const LinParams& P, int factor, int robust, int grid, cudaStream_t st) {
  SGB_SPLIT_DISPATCH(launch_error_pipe, P, grid, st)
  return cudaErrorInvalidValue;
}
int error_pipelined_occupancy(int factor, int robust) {
  SGB_SPLIT_DISPATCH(error_ctas_per_sm)
  return 1;
}

int factor_reduce_occupancy(int factor, int robust) {
  switch (factor * 3 + robust) {
    case 0: return factor_ctas_per_sm<0, 0>();
    case 1: return factor_ctas_per_sm<0, 1>();
    case 2: return factor_ctas_per_sm<0, 2>();
    case 3: return factor_ctas_per_sm<1, 0>();
    case 4: return factor_ctas_per_sm<1, 1>();
    case 5: return factor_ctas_per_sm<1, 2>();
    case 6: return factor_ctas_per_sm<2, 0>();
    case 7: return factor_ctas_per_sm<2, 1>();
    case 8: return factor_ctas_per_sm<2, 2>();
    default: return 1;
  }
}

#ifdef SGB_PROFILING
int search_occupancy(int stack_depth) {
  int nb = 0;
  const size_t smem = static_cast<size_t>(stack_depth) * kLinBlock * sizeof(uint2);
  if (smem > 48 * 1024) cudaFuncSetAttribute(nn_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, nn_search_kernel, kLinBlock, smem) != cudaSuccess) return 1;
  return nb > 0 ? nb : 1;
}

cudaError_t launch_search(const LinParams& P, int grid, int stack_depth, cudaStream_t st) {
  const size_t smem = static_cast<size_t>(stack_depth) * kLinBlock * sizeof(uint2);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(nn_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
  }
  nn_search_kernel<<<grid, kLinBlock, smem, st>>>(P);
  return cudaGetLastError();
}

#endif  // SGB_PROFILING

cudaError_t launch_factor_reduce(const LinParams& P, int factor, int robust, int grid, cudaStream_t st) {
  switch (factor * 3 + robust) {
    case 0: return launch_factor<0, 0>(P, grid, st);
    case 1: return launch_factor<0, 1>(P, grid, st);
    case 2: return launch_factor<0, 2>(P, grid, st);
    case 3: return launch_factor<1, 0>(P, grid, st);
    case 4: return launch_factor<1, 1>(P, grid, st);
    case 5: return launch_factor<1, 2>(P, grid, st);
    case 6: return launch_factor<2, 0>(P, grid, st);
    case 7: return launch_factor<2, 1>(P, grid, st);
    case 8: return launch_factor<2, 2>(P, grid, st);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace sgb
