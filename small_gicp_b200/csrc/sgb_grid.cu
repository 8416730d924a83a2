// SPDX-License-Identifier: MIT
// Uniform-grid front end of the exact nearest-neighbour search.
//
// In a registration that is not wildly misaligned almost every query's nearest neighbour is a fraction of the point
// spacing away.  The 2 x 2 x 2 block of grid cells (cell edge c) anchored at floor(u - 1/2) covers the cube
// [q - c/2, q + c/2]^3, i.e. it holds EVERY target point within c/2 of q: if the closest point of the block is within c/2
// it is the exact nearest neighbour and the query is finished -- no tree walk, no dependent pointer chasing.
// BLOCK LISTS: every target point is stored under the eight blocks that contain its cell, so a block is ONE hash lookup and ONE
// contiguous run of points (grid_probe_blocks_kernel); 8x the point storage buys the removal of seven lookups and of divergent per-cell
// scans.  The runs are stored as 32-byte PAIR RECORDS (sgb_grid.cuh: GridPair): two points per sector.
// Queries the probe cannot settle (nothing within c/2: misaligned first iterations, holes, outliers) are appended to a
// compact pending list -- with the best candidate found so far as an upper bound -- and finished exactly by packet_search_kernel:
//   * few of them: a warp per query (pending_search_body, sgb_grid.cuh): ring search over the 27 blocks at stride 2 around the query
//     (everything within 2.5 c), then, only if that radius does not decide it, a walk of the packet tree;
//   * many of them: the packet walk (sgb_kernels_packet.cu) over the chunk-ordered queries, settled lanes idle.
// Which of the two runs is decided on the device from the pending counter.  Results are identical to a pure tree search
// (exact ties aside; tests/test_gpu_parity.py::test_search_structures_agree).
#include <cfloat>
#include <cstdlib>
#include <cub/device/device_radix_sort.cuh>

#include "sgb_device.cuh"
#include "sgb_grid.cuh"
#include "sgb_kernels.h"

namespace sgb {

// Morton (Z-order) code of the three 21-bit offset coordinates: the ORDER in which the lists are laid out in memory.  The table is keyed
// by the plain packed coordinates (grid_key); only the sort uses the curve, so that the lists a warp of Hilbert-ordered queries needs --
// a compact patch of ~11 neighbouring blocks -- are neighbours in memory too (DRAM pages, L2 sectors, TLB) instead of being strung along
// x only (it matters most for the probe at 10M points and more).
__device__ __forceinline__ uint64_t grid_spread21(uint64_t x) {
  x &= 0x1fffffull;
  x = (x | x << 32) & 0x1f00000000ffffull;
  x = (x | x << 16) & 0x1f0000ff0000ffull;
  x = (x | x << 8) & 0x100f00f00f00f00full;
  x = (x | x << 4) & 0x10c30c30c30c30c3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}
__device__ __forceinline__ uint64_t grid_compact21(uint64_t x) {
  x &= 0x1249249249249249ull;
  x = (x | x >> 2) & 0x10c30c30c30c30c3ull;
  x = (x | x >> 4) & 0x100f00f00f00f00full;
  x = (x | x >> 8) & 0x1f0000ff0000ffull;
  x = (x | x >> 16) & 0x1f00000000ffffull;
  x = (x | x >> 32) & 0x1fffffull;
  return x;
}
__device__ __forceinline__ uint64_t grid_order_key(int ix, int iy, int iz, bool curve) {
  if (!curve) return grid_key(ix, iy, iz);
  return grid_spread21(static_cast<uint32_t>(ix + (1 << 20))) | (grid_spread21(static_cast<uint32_t>(iy + (1 << 20))) << 1) |
         (grid_spread21(static_cast<uint32_t>(iz + (1 << 20))) << 2);
}
/// sort key -> table key (packed coordinates)
__device__ __forceinline__ uint64_t grid_table_key(uint64_t k, bool curve) {
  if (!curve) return k;
  return grid_compact21(k) | (grid_compact21(k >> 1) << 21) | (grid_compact21(k >> 2) << 42);
}

// cell key of every target point (leaf-ordered, centred FP32); value = leaf position.
// BLOCKS: every point is entered under the eight 2 x 2 x 2 cell blocks that contain its cell (block anchor = lowest cell),
// so that a query finds every point of the block around it in ONE contiguous run (8x the points, one lookup, one loop).
__global__ void grid_keys_kernel(const float4* __restrict__ pts, uint32_t n, GridParams g, uint64_t* keys, uint32_t* vals, bool curve) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t i = t >> 3, o = t & 7u;
  if (i >= n) return;
  const float4 p = pts[i];
  const int ix = __float2int_rd((p.x - g.origin[0]) * g.inv_cell), iy = __float2int_rd((p.y - g.origin[1]) * g.inv_cell),
            iz = __float2int_rd((p.z - g.origin[2]) * g.inv_cell);
  keys[t] = grid_order_key(ix - static_cast<int>(o & 1u), iy - static_cast<int>((o >> 1) & 1u), iz - static_cast<int>(o >> 2), curve);
  vals[t] = i;
}

// after the sort: one table entry per run of equal keys, and the run's points as PAIR RECORDS (sgb_grid.cuh: GridPair).
// pass 1 (heads): length of every run -> its number of records at the head's position (0 elsewhere); counters[0] = number of runs
// (sizes the hash table and, with m, the record array), counters[1] = longest run
__global__ void grid_heads_kernel(const uint64_t* __restrict__ keys, uint32_t m, uint32_t* pairs, uint32_t* counters) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t np = 0;
  bool head = false;
  if (i < m) {
    const uint64_t k = keys[i];
    head = i == 0 || keys[i - 1] != k;
    if (head) {
      uint32_t cnt = 1;
      // (a run longer than the front end accepts is only measured up to the limit: build_grid drops the grid before anything reads the records)
      while (i + cnt < m && cnt <= kGridMaxList && keys[i + cnt] == k) cnt++;
      np = (cnt + 1u) >> 1;
      atomicMax(counters + 1, cnt);  // longest list: build_grid drops the front end when one query would have to scan thousands of points
    }
    pairs[i] = np;
  }
  const unsigned b = __ballot_sync(0xffffffffu, head);
  if ((threadIdx.x & 31u) == 0 && b) atomicAdd(counters, static_cast<uint32_t>(__popc(b)));
}
// pass 2 (after an exclusive scan of `pairs` -> first record of every run): the head of a run writes its records -- two points per
// record, components interleaved; an odd run is padded with a point at infinity that can never be nearest -- and claims the table slot
__global__ void grid_fill_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ leaf_pos, const float4* __restrict__ leaf_pts, uint32_t m,
                                 const uint32_t* __restrict__ pair_start, GridPair* grid_pairs, GridSlot* table, uint32_t mask, bool curve) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint64_t k = keys[i];
  if (i != 0 && keys[i - 1] == k) return;
  uint32_t cnt = 1;
  while (i + cnt < m && keys[i + cnt] == k) cnt++;
  const uint32_t first = pair_start[i];
  for (uint32_t e = 0; e < cnt; e += 2u) {
    const uint32_t l0 = leaf_pos[i + e];
    const float4 p0 = leaf_pts[l0];
    float4 p1 = make_float4(kGridPadCoord, kGridPadCoord, kGridPadCoord, 0.f);
    uint32_t l1 = kNone;
    if (e + 1u < cnt) {
      l1 = leaf_pos[i + e + 1u];
      p1 = leaf_pts[l1];
    }
    GridPair r;
    r.a = make_float4(p0.x, p1.x, p0.y, p1.y);
    r.b = make_float4(p0.z, p1.z, __uint_as_float(l0), __uint_as_float(l1));
    grid_pairs[first + (e >> 1)] = r;
  }
  const uint64_t tk = grid_table_key(k, curve);
  uint32_t slot = grid_hash_of_key(tk) & mask;
  for (;;) {
    const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(&table[slot].key), ~0ull, static_cast<unsigned long long>(tk));
    if (prev == ~0ull) break;
    slot = (slot + 1u) & mask;
  }
  table[slot].start = first;  // in records
  table[slot].count = cnt;    // in points
}

__global__ void grid_table_init_kernel(GridSlot* table, uint32_t capacity) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < capacity) {
    table[i].key = ~0ull;
    table[i].start = 0u;
    table[i].count = 0u;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// probe, block lists: the block anchored at floor(u - 1/2) covers [q - c/2, q + c/2]^3; one lookup, one contiguous scan
// ---------------------------------------------------------------------------------------------------------------
// UNROLL pairs of the scan loop are in flight per thread (2: 32 registers = 8 CTAs of 256 threads = full occupancy);
// PREFETCH: the whole list is requested into L2 as soon as its table slot is known.  MIN_CTAS / UNROLL / PREFETCH other than the defaults
// exist in the profiling library only (SGB_PROBE_CTAS, SGB_PROBE_UNROLL, SGB_PROBE_PREFETCH).
template <int MIN_CTAS, int UNROLL = 2, bool PREFETCH = true>
__global__ void __launch_bounds__(256, MIN_CTAS) grid_probe_blocks_kernel(const __grid_constant__ LinParams P, const GridPair* __restrict__ grid_pairs,
                                                               const GridSlot* __restrict__ table, uint32_t mask, GridParams g, uint8_t* state,
                                                               uint32_t* pending_count, uint32_t* pending_list, float4* pending_q, uint32_t* next_count,
                                                               ChunkClasses cc) {
  const uint32_t gi = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in_range = gi < P.src.n;
  if (gi == 0u) *next_count = 0u;  // the counter of the NEXT linearize (two counters alternate: no memset between launches)
  if (gi < kChunkClasses && cc.count_next) cc.count_next[gi] = 0u;
  const uint32_t i = in_range ? gi : P.src.n - 1u;
  const double* R = P.T;
  const double csx = P.src.centre[0], csy = P.src.centre[1], csz = P.src.centre[2];
  const double tpx = R[0] * csx + R[1] * csy + R[2] * csz + P.T[9] - P.tgt.centre[0];
  const double tpy = R[3] * csx + R[4] * csy + R[5] * csz + P.T[10] - P.tgt.centre[1];
  const double tpz = R[6] * csx + R[7] * csy + R[8] * csz + P.T[11] - P.tgt.centre[2];
  const float4 s = __ldg(&P.src.pts[i]);
  const double sx = s.x, sy = s.y, sz = s.z;
  const float fx = static_cast<float>(R[0] * sx + R[1] * sy + R[2] * sz + tpx);
  const float fy = static_cast<float>(R[3] * sx + R[4] * sy + R[5] * sz + tpy);
  const float fz = static_cast<float>(R[6] * sx + R[7] * sy + R[8] * sz + tpz);
  float best_d = P.max_dist_sq;
  uint32_t best = kNone;
  const float ax = floorf((fx - g.origin[0]) * g.inv_cell - 0.5f), ay = floorf((fy - g.origin[1]) * g.inv_cell - 0.5f),
              az = floorf((fz - g.origin[2]) * g.inv_cell - 0.5f);
  // queries far outside the target's box cannot be settled anyway; clamping keeps the integer cell coordinates in range
  const int bx = static_cast<int>(fminf(fmaxf(ax, -1e5f), 1e5f)), by = static_cast<int>(fminf(fmaxf(ay, -1e5f), 1e5f)),
            bz = static_cast<int>(fminf(fmaxf(az, -1e5f), 1e5f));
  const uint2 e = grid_lookup(table, mask, bx, by, bz);
  {
    // The list is a contiguous run of ceil(e.y / 2) PAIR RECORDS (32 B: two points, components interleaved), read by two 128-bit
    // loads of one sector (load_pair).  The squared distance is fma(dz, dz, fma(dy, dy, dx * dx)) in FP32 with round-to-nearest for
    // each point, so the candidate and its distance are bit-identical to a packed f32x2 evaluation of the same expression.
    const GridPair* __restrict__ rec = grid_pairs + e.x;
    const uint32_t npairs = (e.y + 1u) >> 1;
    // pull all of its lines into L2 at once (the scan would otherwise pay one DRAM round trip per batch of loads)
    const char* lp = reinterpret_cast<const char*>(rec);
    const uint32_t bytes = npairs * 32u;
    if (PREFETCH)
      for (uint32_t off = 128u; off < bytes; off += 128u) asm volatile("prefetch.global.L2 [%0];" ::"l"(lp + off));
    if (PREFETCH && bytes > 128u) asm volatile("prefetch.global.L2 [%0];" ::"l"(lp + bytes - 32u));  // last line of a run that is not 128 B aligned
#pragma unroll UNROLL
    for (uint32_t j = 0; j < npairs; j++) {
      const GridPair t = load_pair(rec + j);
      const float dx0 = __fsub_rn(t.a.x, fx), dy0 = __fsub_rn(t.a.z, fy), dz0 = __fsub_rn(t.b.x, fz);
      const float dx1 = __fsub_rn(t.a.y, fx), dy1 = __fsub_rn(t.a.w, fy), dz1 = __fsub_rn(t.b.y, fz);
      const float d0 = __fmaf_rn(dz0, dz0, __fmaf_rn(dy0, dy0, __fmul_rn(dx0, dx0)));
      const float d1 = __fmaf_rn(dz1, dz1, __fmaf_rn(dy1, dy1, __fmul_rn(dx1, dx1)));
      if (d0 < best_d) {  // first point of the pair first: ties keep the scan order
        best_d = d0;
        best = __float_as_uint(t.b.z);
      }
      if (d1 < best_d) {  // (the pad of an odd list sits at 1e18: ~3e36, never nearest)
        best_d = d1;
        best = __float_as_uint(t.b.w);
      }
    }
  }
  const bool settled = best != kNone && best_d <= g.settle_d2;
  if (!settled && P.use_prev) {  // keep the better of (grid candidate, previous correspondence) as the tree search's seed
    const uint32_t prev = P.corr[i];
    if (prev != kNone) {
      const float4 t = __ldg(&P.tgt.pts[prev]);
      const float dx = t.x - fx, dy = t.y - fy, dz = t.z - fz;
      const float d = dx * dx + dy * dy + dz * dz;
      if (d < best_d) {  // (a seed beyond the rejector's bound is no use: best_d starts there)
        best = prev;
        best_d = d;
      }
    }
  }
  if (in_range) {
    P.corr[i] = best;
    state[i] = settled ? 1 : 0;
  }
  // Pending queries go to a compact list, and -- for the packet search -- the CHUNK (one warp here = one 32-query chunk there) goes into
  // the work list of its cost class = how far its widest search ball reaches (best_d is the squared radius a pending lane starts its
  // walk with).  The packet search takes the wide classes first, so that what is left when the GPU drains are the cheap walks
  // (otherwise a long tail of late-starting heavy chunks); chunks without a pending lane are in no list.
  // Both appends are aggregated over the CTA's eight warps: at most four atomics per CTA -- one per warp and list made the hot
  // counters the probe's own tail at the identity pose.
  const bool pend = in_range && !settled;
  const unsigned m = __ballot_sync(0xffffffffu, pend);
  const uint32_t lane = threadIdx.x & 31u, wib = threadIdx.x >> 5;
  __shared__ uint32_t s_cnt[8], s_cls[8], s_base[8];
  {
    const uint32_t r2 = __reduce_max_sync(0xffffffffu, pend ? __float_as_uint(best_d) : 0u);  // non-negative floats order like their bits
    if (lane == 0) {
      const float r = __uint_as_float(r2);
      s_cnt[wib] = static_cast<uint32_t>(__popc(m));
      s_cls[wib] = !m ? kChunkClasses : (r >= cc.wide_r2 ? 0u : (r >= cc.mid_r2 ? 1u : 2u));
    }
  }
  __syncthreads();
  if (wib == 0) {
    const uint32_t nw = blockDim.x >> 5;
    const uint32_t cnt = lane < nw ? s_cnt[lane] : 0u, cls = lane < nw ? s_cls[lane] : kChunkClasses;
    uint32_t incl = cnt;  // inclusive prefix over the warps
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= static_cast<uint32_t>(o)) incl += t;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 7);
    uint32_t pbase = 0;
    if (lane == 0 && total) pbase = atomicAdd(pending_count, total);
    pbase = __shfl_sync(0xffffffffu, pbase, 0);
    if (lane < nw) s_base[lane] = pbase + incl - cnt;
    if (cc.lists) {
#pragma unroll
      for (uint32_t c = 0; c < kChunkClasses; c++) {
        const unsigned mc = __ballot_sync(0xffffffffu, cls == c);
        if (!mc) continue;
        uint32_t cb = 0;
        if (lane == static_cast<uint32_t>(__ffs(mc) - 1)) cb = atomicAdd(&cc.count[c], static_cast<uint32_t>(__popc(mc)));
        cb = __shfl_sync(0xffffffffu, cb, __ffs(mc) - 1);
        if (cls == c) cc.lists[static_cast<size_t>(c) * cc.n_chunks + cb + __popc(mc & ((1u << lane) - 1u))] = (blockIdx.x * blockDim.x >> 5) + lane;
      }
    }
  }
  __syncthreads();
  if (pend) {  // the pending record: who, where (transformed query) and how far its best candidate is -- the finishing kernel needs nothing else
    const uint32_t slot = s_base[wib] + __popc(m & ((1u << lane) - 1u));
    pending_list[slot] = i;
    pending_q[slot] = make_float4(fx, fy, fz, best_d);
  }
}

// per-leaf spacing estimate from the packet records (two largest box extents / count) for the choice of the cell size
__global__ void grid_spacing_kernel(const float4* __restrict__ pnodes, uint32_t n_inner, float* out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_inner * 2u) return;
  const float4 lo = pnodes[(t >> 1) * 4 + (t & 1u) * 2 + 0], hi = pnodes[(t >> 1) * 4 + (t & 1u) * 2 + 1];
  const uint32_t cnt = __float_as_uint(hi.w);
  float v = -1.0f;
  if (cnt >= 4u && hi.x >= lo.x) {
    float e0 = hi.x - lo.x, e1 = hi.y - lo.y, e2 = hi.z - lo.z;
    const float mn = fminf(e0, fminf(e1, e2));
    const float area = (e0 * e1 * e2 > 0.f && mn > 0.f) ? (e0 * e1 * e2 / mn) : fmaxf(e0 * e1, fmaxf(e0 * e2, e1 * e2));
    v = sqrtf(area / static_cast<float>(cnt));
  }
  out[t] = v;
}

// ---------------------------------------------------------------------------------------------------------------
cudaError_t launch_grid_spacing(const float4* pnodes, uint32_t n_inner, float* out, cudaStream_t st) {
  if (!n_inner) return cudaSuccess;
  grid_spacing_kernel<<<(n_inner * 2u + 255u) / 256u, 256, 0, st>>>(pnodes, n_inner, out);
  return cudaGetLastError();
}

cudaError_t launch_grid_sort(const float4* leaf_pts, uint32_t n, const GridParams& g, uint64_t* keys_in, uint64_t* keys_out, uint32_t* vals_in, uint32_t* vals_out,
                             void* sort_temp, size_t sort_temp_bytes, uint32_t* d_counters, bool curve, cudaStream_t st) {
  const uint32_t m = n * 8u;
  grid_keys_kernel<<<(m + 255u) / 256u, 256, 0, st>>>(leaf_pts, n, g, keys_in, vals_in, curve);
  cudaError_t e = cub::DeviceRadixSort::SortPairs(sort_temp, sort_temp_bytes, keys_in, keys_out, vals_in, vals_out, static_cast<int>(m), 0, 63, st);
  if (e != cudaSuccess) return e;
  e = cudaMemsetAsync(d_counters, 0, 2 * sizeof(uint32_t), st);
  if (e != cudaSuccess) return e;
  grid_heads_kernel<<<(m + 255u) / 256u, 256, 0, st>>>(keys_out, m, vals_in, d_counters);  // the sort's value input is free again: records per run
  return cudaGetLastError();
}

cudaError_t launch_grid_fill(const uint64_t* keys_sorted, const uint32_t* vals_sorted, const float4* leaf_pts, uint32_t m, const uint32_t* pairs, uint32_t* pair_start,
                             void* scan_temp, size_t scan_temp_bytes, float4* grid_pts, GridSlot* table, uint32_t capacity, bool curve, cudaStream_t st) {
  size_t need = 0;
  cudaError_t e = exclusive_sum_u32(nullptr, need, pairs, pair_start, m, st);
  if (e != cudaSuccess) return e;
  if (need > scan_temp_bytes) return cudaErrorInvalidValue;  // (the radix sort's scratch, which the caller hands over, is far larger)
  e = exclusive_sum_u32(scan_temp, need, pairs, pair_start, m, st);
  if (e != cudaSuccess) return e;
  grid_table_init_kernel<<<(capacity + 255u) / 256u, 256, 0, st>>>(table, capacity);
  grid_fill_kernel<<<(m + 255u) / 256u, 256, 0, st>>>(keys_sorted, vals_sorted, leaf_pts, m, pair_start, reinterpret_cast<GridPair*>(grid_pts), table, capacity - 1u, curve);
  return cudaGetLastError();
}

cudaError_t launch_grid_probe(const LinParams& P, const float4* grid_pts, const GridSlot* table, uint32_t capacity, const GridParams& g, uint8_t* state,
                              uint32_t* pending_count, uint32_t* pending_list, float4* pending_q, uint32_t* next_count, const ChunkClasses& cc, cudaStream_t st) {
  // *pending_count must be zero on entry: the previous probe (or the context) cleared it
  const uint32_t grid = (P.src.n + 255u) / 256u;
  const GridPair* pairs = reinterpret_cast<const GridPair*>(grid_pts);
#ifdef SGB_PROFILING
  static const int ctas = std::getenv("SGB_PROBE_CTAS") ? std::atoi(std::getenv("SGB_PROBE_CTAS")) : 5;
  static const int unroll = std::getenv("SGB_PROBE_UNROLL") ? std::atoi(std::getenv("SGB_PROBE_UNROLL")) : 2;
#define SGB_PROBE_VARIANT(C, U)                                                                                                                        \
  if (ctas == C && unroll == U) {                                                                                                                      \
    grid_probe_blocks_kernel<C, U><<<grid, 256, 0, st>>>(P, pairs, table, capacity - 1u, g, state, pending_count, pending_list, pending_q, next_count, cc); \
    return cudaGetLastError();                                                                                                                         \
  }
  static const bool prefetch = !(std::getenv("SGB_PROBE_PREFETCH") && std::getenv("SGB_PROBE_PREFETCH")[0] == '0');
  if (!prefetch) {
    grid_probe_blocks_kernel<5, 2, false><<<grid, 256, 0, st>>>(P, pairs, table, capacity - 1u, g, state, pending_count, pending_list, pending_q, next_count, cc);
    return cudaGetLastError();
  }
  SGB_PROBE_VARIANT(5, 1) SGB_PROBE_VARIANT(5, 3) SGB_PROBE_VARIANT(5, 4) SGB_PROBE_VARIANT(6, 1) SGB_PROBE_VARIANT(6, 2) SGB_PROBE_VARIANT(6, 3) SGB_PROBE_VARIANT(8, 2)
#undef SGB_PROBE_VARIANT
#endif
  grid_probe_blocks_kernel<5><<<grid, 256, 0, st>>>(P, pairs, table, capacity - 1u, g, state, pending_count, pending_list, pending_q, next_count, cc);
  return cudaGetLastError();
}

}  // namespace sgb
