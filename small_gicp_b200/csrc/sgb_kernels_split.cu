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
  const double3 tp = centred_translation(P.T, P.src.centre[0], P.src.centre[1], P.src.centre[2], P.tgt.centre);
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
        const float3 f = centred_query_f32(R, tp, __ldg(&P.src.pts[i]));
        fx = f.x;
        fy = f.y;
        fz = f.z;
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
// depends on the correspondence index and the FP64 factor algebra is a chain of dependent operations: the kernel is bound
// by latency, neither by HBM bandwidth nor by the FP64 pipe, and needs many warps in flight.  The loads are issued two
// tiles ahead with cp.async into a per-thread landing zone in shared memory:
//   A(t+2): correspondence index + source point / covariance (coalesced)
//   B(t+1): target point / normal / covariance gathered through the index A(t+1) brought in
//   C(t)  : FP64 rejector + factor algebra on the operands that landed during the previous tile's arithmetic
// Every thread only reads what it copied itself, so the pipeline needs no barrier, just cp.async.wait_group.
// linearize sums every tile across the warp as it computes the terms (warp_sum_transposed, eight sums at a time) and keeps
// ONE running FP64 sum per lane (lane k: sum k), not 29 per thread: 80 registers without spills.  With a covariance's
// second float4 landed as the 8 bytes it carries (yz, zz), 80 B per point and stage, that is 6 CTAs of 128 threads per SM.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem));
}
__device__ __forceinline__ void cp_async8(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem));
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

template <int FACTOR, bool NARROW>
struct FactorFields {
  // landing-zone float4 slots: source point [+ source covariance], target point [+ normal | covariance].  NARROW (GICP): a
  // covariance's second float4 carries only (yz, zz); those 8 bytes land in float2 slots (source, target) after the float4 slots
  static constexpr int kCov = FACTOR == 2 ? (NARROW ? 1 : 2) : 0;  // float4 slots per covariance
  static constexpr int kSrc = 1 + kCov;                            // first target slot
  static constexpr int kQuads = FACTOR == 1 ? 3 : 2 * kSrc;
  static constexpr int kPairs = FACTOR == 2 && NARROW ? 2 : 0;
};
constexpr int kFactorStages = 3;

// NREG: register budget per thread.  TILES (linearize): the per-tile warp sums above.  Otherwise every thread keeps its own running
// sums over its tiles and the CTA reduces them at the end: the ERR instantiations (one sum), and the 29 sums of linearize in the
// profiling build's A/B kernel (SGB_FACTOR_TILES=0: 128 registers, 4 CTAs per SM).
// ERR: the same operand pipeline evaluating Reduction::error instead (cached correspondences, trial pose P.T, GICP precision matrix re-derived
// from the linearisation pose P.Tlin, one sum): the LM inner loop's kernel.  The plain grid-stride version of it (error_kernel, sgb_kernels.cu)
// waited on two dependent load round trips per point with nothing in flight: longer than the whole linearize algebra.  It keeps the full float4
// landing zone: its occupancy, hence its grid and the order of error()'s additions, stay those of that layout.
template <int FACTOR, int ROBUST, int NREG, bool ERR = false, bool TILES = !ERR>
__global__ void __maxnreg__(NREG) factor_reduce_kernel(const __grid_constant__ LinParams P) {
  using F = FactorFields<FACTOR, TILES>;
  extern __shared__ float4 s_zone[];  // [kFactorStages][F::kQuads][kLinBlock] float4, then [kFactorStages][F::kPairs][kLinBlock] float2
  __shared__ uint32_t s_corr[kFactorStages][kLinBlock];
  constexpr int NACC = ERR || TILES ? 1 : kAcc + 1;
  double acc[NACC];
#pragma unroll
  for (int k = 0; k < NACC; k++) acc[k] = 0.0;
  const double* R = P.T;
  const double csx = P.src.centre[0], csy = P.src.centre[1], csz = P.src.centre[2];
  const double3 tp = centred_translation(P.T, csx, csy, csz, P.tgt.centre);
  const uint32_t n = P.src.n, n_tiles = (n + kLinBlock - 1u) / kLinBlock, tid = threadIdx.x;
  float4* zone = s_zone + tid;
  float2* pairs = reinterpret_cast<float2*>(s_zone + kFactorStages * F::kQuads * kLinBlock) + tid;
  auto slot = [&](int stage, int f) { return zone + (stage * F::kQuads + f) * kLinBlock; };
  auto pair = [&](int stage, int f) { return pairs + (stage * F::kPairs + f) * kLinBlock; };
  auto issue_a = [&](uint32_t tile, int stage) {
    const uint32_t i = tile * kLinBlock + tid;
    if (tile < n_tiles && i < n) {
      cp_async4(&s_corr[stage][tid], &P.corr[i]);
      cp_async16(slot(stage, 0), &P.src.pts[i]);
      if (FACTOR == 2) {
        cp_async16(slot(stage, 1), &P.src.covA[i]);
        if (F::kPairs)
          cp_async8(pair(stage, 0), &P.src.covB[i]);
        else
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
      if (F::kPairs)
        cp_async8(pair(stage, 1), &P.tgt.covB[best]);
      else
        cp_async16(slot(stage, F::kSrc + 2), &P.tgt.covB[best]);
    }
  };
  // NARROW: the (yz, zz) of the source (f = 0) / target (f = 1) covariance as the float4 the algebra takes (.z, .w unused)
  auto cov_b = [&](int stage, int f) {
    const float2 c = *pair(stage, f);
    return make_float4(c.x, c.y, 0.f, 0.f);
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
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    // operands out of this thread's landing zone; the per-point arithmetic is point_linearize_source / point_error (sgb_math.cuh)
    if (TILES) {
      // every lane takes part in the warp sums: rejected points and the padding of a partial tile give exact zero terms
      Sym3 D{0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      double rs[3] = {0.0, 0.0, 0.0}, p[3] = {0.0, 0.0, 0.0};
      bool inlier = false;
      if (best != kNone) {
        const float4 sB = FACTOR == 2 ? cov_b(st, 0) : z, tB = FACTOR == 2 ? cov_b(st, 1) : z;
        inlier = point_weight_source<FACTOR>(R, tp.x, tp.y, tp.z, csx, csy, csz, P.max_dist_sq_d, *slot(st, 0), slot(st, 1), &sB, *slot(st, F::kSrc),
                                             slot(st, F::kSrc + 1), &tB, D, rs, p);
        if (!inlier) P.corr[tile * kLinBlock + tid] = kNone;  // rejected: error() and sgb_correspondences() must not see it
      }
      double t[kAcc + 1];  // c = 1 where there is no inlier: a robust weight of a zero residual that stays finite whatever P.robust_c is
      factor_terms_source<ROBUST>(D, rs[0], rs[1], rs[2], p[0], p[1], p[2], inlier ? P.robust_c : 1.0, t);
      t[kAcc] = inlier ? 1.0 : 0.0;
      acc[0] += warp_sum_transposed<kAcc + 1>(t);
    } else if (best != kNone) {
      const uint32_t i = tile * kLinBlock + tid;
      const float4 sp = *slot(st, 0);
      const float4 tq = *slot(st, F::kSrc);
      if (ERR) {
        acc[0] += point_error<FACTOR, ROBUST>(R, tp.x, tp.y, tp.z, P.Tlin, P.robust_c, sp, FACTOR == 2 ? *slot(st, 1) : z, FACTOR == 2 ? *slot(st, 2) : z, tq,
                                              FACTOR >= 1 ? *slot(st, F::kSrc + 1) : z, FACTOR == 2 ? *slot(st, F::kSrc + 2) : z);
      } else if (!point_linearize_source<FACTOR, ROBUST>(R, tp.x, tp.y, tp.z, csx, csy, csz, P.max_dist_sq_d, P.robust_c, sp, slot(st, 1), slot(st, 2), tq,
                                                         slot(st, F::kSrc + 1), slot(st, F::kSrc + 2), acc)) {
        P.corr[i] = kNone;
      }
    }
    st = st1;
  }
  cp_async_wait_all();
  block_reduce_and_finish<TILES ? kAcc + 1 : NACC, !ERR, TILES>(acc, P.partials, P.ticket, P.out, P.comm);
}

constexpr int kFactorRegs = 80;  // linearize: 6 CTAs x 128 threads x 80 registers fit the register file (88 do not); no spills
constexpr int kFactorSumRegs = 128;  // per-thread sums (ERR, the A/B kernel): 4 CTAs x 128 threads x 128 registers = the whole register file
#ifdef SGB_PROFILING
static bool factor_tiles_switch() {  // SGB_FACTOR_TILES=0: per-thread sums instead (GICP without robust kernel only, the bench workload)
  static const bool v = !std::getenv("SGB_FACTOR_TILES") || std::atoi(std::getenv("SGB_FACTOR_TILES")) != 0;
  return v;
}
#endif
/// dynamic shared memory of factor_reduce_kernel: its operand landing zones
template <int FACTOR, bool NARROW>
constexpr size_t factor_smem() {
  using F = FactorFields<FACTOR, NARROW>;
  return static_cast<size_t>(kFactorStages) * kLinBlock * (F::kQuads * sizeof(float4) + F::kPairs * sizeof(float2));
}
template <int FACTOR, int ROBUST>
static cudaError_t launch_factor(const LinParams& P, int grid, cudaStream_t st) {
#ifdef SGB_PROFILING
  if (FACTOR == 2 && ROBUST == 0 && !factor_tiles_switch())
    return launch_dependent(factor_reduce_kernel<2, 0, kFactorSumRegs, false, false>, grid, kLinBlock, factor_smem<2, false>(), st, P);
#endif
  return launch_dependent(factor_reduce_kernel<FACTOR, ROBUST, kFactorRegs>, grid, kLinBlock, factor_smem<FACTOR, true>(), st, P);
}

// resident CTAs per SM of one instantiation (the grid is sized to exactly one wave: a partial second wave of this
// register-heavy kernel runs one CTA per SM for a good part of the kernel's duration)
template <int FACTOR, int ROBUST>
static int factor_ctas_per_sm() {
#ifdef SGB_PROFILING
  if (FACTOR == 2 && ROBUST == 0 && !factor_tiles_switch())
    return ctas_per_sm(factor_reduce_kernel<2, 0, kFactorSumRegs, false, false>, kLinBlock, factor_smem<2, false>(), true, false);
#endif
  return ctas_per_sm(factor_reduce_kernel<FACTOR, ROBUST, kFactorRegs>, kLinBlock, factor_smem<FACTOR, true>(), true, false);
}

cudaError_t launch_factor_reduce(const LinParams& P, int factor, int robust, int grid, cudaStream_t st) {
  return dispatch_factor_robust(factor, robust, cudaErrorInvalidValue, [&](auto f, auto r) { return launch_factor<f, r>(P, grid, st); });
}
int factor_reduce_occupancy(int factor, int robust) {
  return dispatch_factor_robust(factor, robust, 1, [](auto f, auto r) { return factor_ctas_per_sm<f, r>(); });
}

cudaError_t launch_error_pipelined(const LinParams& P, int factor, int robust, int grid, cudaStream_t st) {
  return dispatch_factor_robust(factor, robust, cudaErrorInvalidValue, [&](auto f, auto r) {
    factor_reduce_kernel<f, r, kFactorSumRegs, true><<<grid, kLinBlock, factor_smem<f, false>(), st>>>(P);
    return cudaGetLastError();
  });
}
int error_pipelined_occupancy(int factor, int robust) {
  return dispatch_factor_robust(factor, robust, 1, [](auto f, auto r) {
    return ctas_per_sm(factor_reduce_kernel<f, r, kFactorSumRegs, true>, kLinBlock, factor_smem<f, false>(), true, false);
  });
}

#ifdef SGB_PROFILING
int search_occupancy(int stack_depth) {
  const size_t smem = static_cast<size_t>(stack_depth) * kLinBlock * sizeof(uint2);
  return ctas_per_sm(nn_search_kernel, kLinBlock, smem, false, smem > 48 * 1024);
}

cudaError_t launch_search(const LinParams& P, int grid, int stack_depth, cudaStream_t st) {
  const size_t smem = static_cast<size_t>(stack_depth) * kLinBlock * sizeof(uint2);
  const cudaError_t e = allow_dynamic_smem(nn_search_kernel, smem);
  if (e != cudaSuccess) return e;
  nn_search_kernel<<<grid, kLinBlock, smem, st>>>(P);
  return cudaGetLastError();
}

#endif  // SGB_PROFILING

}  // namespace sgb
