// SPDX-License-Identifier: MIT
// Uniform-grid front end of the exact nearest-neighbour search.
//
// In a registration that is not wildly misaligned almost every query's nearest neighbour is a fraction of the point
// spacing away.  The 2 x 2 x 2 block of grid cells (cell edge c) anchored at floor(u - 1/2) covers the cube
// [q - c/2, q + c/2]^3, i.e. it holds EVERY target point within c/2 of q: if the closest point of the block is within c/2
// it is the exact nearest neighbour and the query is finished -- no tree walk, no dependent pointer chasing.
// CELL ORDER + BLOCK TABLE: the target is held once more, sorted by cell in raster order (x fastest), one float4 per point
// (x, y, z, leaf position).  In that order the block anchored at (x, y, z) is exactly FOUR contiguous runs, one per (y, z) row pair,
// each run being cells x and x + 1; a table slot per non-empty block (one 32-byte sector: sgb_kernels.h GridSlot) holds the four
// runs, so a block is ONE hash lookup and four independent scans (grid_probe_blocks_kernel).  Every point is stored once (16 B)
// and the blocks of neighbouring queries share their points in L2.
// Queries the probe cannot settle (nothing within c/2: misaligned first iterations, holes, outliers) are appended to a
// compact pending list -- with the best candidate found so far as an upper bound -- and finished exactly by packet_search_kernel:
//   * few of them: a warp per query (pending_search_body, sgb_grid.cuh): ring search over the 27 blocks at stride 2 around the query
//     (everything within 2.5 c), then, only if that radius does not decide it, a walk of the packet tree;
//   * many of them: the packet walk (sgb_kernels_packet.cu) over the chunk-ordered queries, settled lanes idle.
// Which of the two runs is decided on the device from the pending counter.  Results are identical to a pure tree search
// (exact ties aside; tests/test_gpu_parity.py::test_search_structures_agree).
#include <cfloat>
#include <cub/device/device_radix_sort.cuh>

#include "sgb_device.cuh"
#include "sgb_grid.cuh"
#include "sgb_kernels.h"

namespace sgb {

// Construction sorts by a COMPACT raster key: B bits per axis (build_grid picks B from the number of cells along the widest axis),
// coordinate + 2, x in the lowest bits -- the same order as grid_key, in 3 B bits instead of 63, so the radix sorts make fewer passes.
// All-ones (grid_sort_pad) is never a real cell or anchor: it pads the anchor entries of points that do not start a cell.
__device__ __forceinline__ uint64_t grid_sort_key(int ix, int iy, int iz, int bits) {
  return static_cast<uint64_t>(ix + 2) | (static_cast<uint64_t>(iy + 2) << bits) | (static_cast<uint64_t>(iz + 2) << (2 * bits));
}
__device__ __forceinline__ void grid_sort_coords(uint64_t k, int bits, int& ix, int& iy, int& iz) {
  const uint64_t m = (1ull << bits) - 1ull;
  ix = static_cast<int>(k & m) - 2;
  iy = static_cast<int>((k >> bits) & m) - 2;
  iz = static_cast<int>((k >> (2 * bits)) & m) - 2;
}
__device__ __forceinline__ uint64_t grid_sort_pad(int bits) { return (1ull << (3 * bits)) - 1ull; }

// cell key of every target point (leaf-ordered, centred FP32); value = leaf position.  A stored non-finite point (NaN) gets the pad:
// it sorts after every cell and is in no block
__global__ void grid_cell_keys_kernel(const float4* __restrict__ pts, uint32_t n, GridParams g, int bits, uint64_t* keys, uint32_t* vals) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = pts[i];
  const int ix = __float2int_rd((p.x - g.origin[0]) * g.inv_cell), iy = __float2int_rd((p.y - g.origin[1]) * g.inv_cell),
            iz = __float2int_rd((p.z - g.origin[2]) * g.inv_cell);
  keys[i] = isnan(p.x) || isnan(p.y) || isnan(p.z) ? grid_sort_pad(bits) : grid_sort_key(ix, iy, iz, bits);
  vals[i] = i;
}

// after the (stable) sort: the points in cell order -- within a cell in ascending leaf position -- and, at position j, the eight
// anchor entries of the cell that starts at j: every cell c is part of the blocks anchored at c - o, o in {0, 1}^3, in run
// r = oy + 2 oz of each (value 4 j + r).  cnt[j] = points of that cell (measured up to kGridMaxList + 1: beyond it build_grid drops
// the front end anyway).  Positions that start no cell, and the non-finite points at the end, write eight pads.
__global__ void grid_cell_heads_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ leaf_pos, const float4* __restrict__ leaf_pts, uint32_t n,
                                       int bits, float4* grid_pts, uint32_t* cnt, uint64_t* akeys, uint32_t* avals) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t l = leaf_pos[j];
  const float4 p = leaf_pts[l];
  grid_pts[j] = make_float4(p.x, p.y, p.z, __uint_as_float(l));
  const uint64_t k = keys[j];
  if ((j != 0 && keys[j - 1] == k) || k == grid_sort_pad(bits)) {  // not the head of a cell, or a non-finite point
#pragma unroll
    for (uint32_t o = 0; o < 8u; o++) {
      akeys[8u * j + o] = grid_sort_pad(bits);
      avals[8u * j + o] = 0u;
    }
    return;
  }
  uint32_t c = 1;
  while (j + c < n && c <= kGridMaxList && keys[j + c] == k) c++;
  cnt[j] = c;
  int ix, iy, iz;
  grid_sort_coords(k, bits, ix, iy, iz);
#pragma unroll
  for (uint32_t o = 0; o < 8u; o++) {
    akeys[8u * j + o] = grid_sort_key(ix - static_cast<int>(o & 1u), iy - static_cast<int>((o >> 1) & 1u), iz - static_cast<int>(o >> 2), bits);
    avals[8u * j + o] = 4u * j + ((o >> 1) & 3u);
  }
}

// after sorting the anchor entries (pads last): the first entry of every distinct anchor adds up its block (at most 8 cells);
// counters[0] = distinct anchors (sizes the table), counters[1] = largest block (build_grid drops the front end beyond kGridMaxList)
__global__ void grid_anchor_heads_kernel(const uint64_t* __restrict__ akeys, const uint32_t* __restrict__ avals, uint32_t m, const uint32_t* __restrict__ cnt,
                                         int bits, uint32_t* counters) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool head = false;
  if (i < m) {
    const uint64_t k = akeys[i];
    head = k != grid_sort_pad(bits) && (i == 0 || akeys[i - 1] != k);
    if (head) {
      uint32_t total = 0;
      for (uint32_t e = i; e < m && akeys[e] == k; e++) total += cnt[avals[e] >> 2];
      atomicMax(counters + 1, total);
    }
  }
  const unsigned b = __ballot_sync(0xffffffffu, head);
  if ((threadIdx.x & 31u) == 0 && b) atomicAdd(counters, static_cast<uint32_t>(__popc(b)));
}

// the first entry of every distinct anchor writes its slot: run r holds the cells with ox = 0 then ox = 1 (adjacent in raster
// order, so the run starts at the first point of whichever is non-empty and counts both)
__global__ void grid_fill_kernel(const uint64_t* __restrict__ akeys, const uint32_t* __restrict__ avals, uint32_t m, const uint32_t* __restrict__ cnt, int bits,
                                 GridSlot* table, uint32_t mask) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint64_t k = akeys[i];
  if (k == grid_sort_pad(bits) || (i != 0 && akeys[i - 1] == k)) return;
  uint32_t start[4] = {~0u, ~0u, ~0u, ~0u}, count[4] = {0u, 0u, 0u, 0u};
  for (uint32_t e = i; e < m && akeys[e] == k; e++) {
    const uint32_t v = avals[e], s = v >> 2, r = v & 3u;
    start[r] = min(start[r], s);
    count[r] += cnt[s];
  }
  int ix, iy, iz;
  grid_sort_coords(k, bits, ix, iy, iz);
  const unsigned long long tk = grid_key(ix, iy, iz);
  uint32_t slot = grid_hash(ix, iy, iz) & mask;
  for (;;) {
    const unsigned long long prev = atomicCAS(&table[slot].key, ~0ull, tk);
    if (prev == ~0ull) break;
    slot = (slot + 1u) & mask;
  }
  uint4* w = reinterpret_cast<uint4*>(&table[slot]);
  // (the key half of the first 16 bytes is already in place; an empty run keeps start 0)
  w[0].z = count[0] ? start[0] : 0u;
  w[0].w = count[1] ? start[1] : 0u;
  w[1] = make_uint4(count[2] ? start[2] : 0u, count[3] ? start[3] : 0u, count[0] | (count[1] << 16), count[2] | (count[3] << 16));
}

__global__ void grid_table_init_kernel(GridSlot* table, uint32_t capacity) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < capacity) {
    uint4* w = reinterpret_cast<uint4*>(&table[i]);
    w[0] = make_uint4(~0u, ~0u, 0u, 0u);
    w[1] = make_uint4(0u, 0u, 0u, 0u);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// probe: the block anchored at floor(u - 1/2) covers [q - c/2, q + c/2]^3; one lookup, then its four contiguous runs
// ---------------------------------------------------------------------------------------------------------------
// 32 registers, no spills: 8 CTAs of 256 threads = full occupancy.  ROUND (a round of sgb_align_batch_async): the first *n_queries of the
// grid's queries (written on the device by the round's planner), the CTAs beyond them exit at once; the planner cleared both pending
// counters and the class counters at the head of the round.  The count read from memory does not fit 32 registers (at 8 or 7 CTAs of
// 256 threads it spills 4 bytes): 39 registers, 6 CTAs.
template <bool ROUND>
__global__ void __launch_bounds__(256, ROUND ? 6 : 8) grid_probe_blocks_kernel(const __grid_constant__ LinParams P, const float4* __restrict__ grid_pts,
                                                                               const GridSlot* __restrict__ table, uint32_t mask, GridParams g, uint8_t* state,
                                                                               uint32_t* pending_count, uint32_t* pending_list, float4* pending_q,
                                                                               uint32_t* next_count, ChunkClasses cc, const uint32_t* __restrict__ n_queries) {
  uint32_t n = P.src.n;
  if constexpr (ROUND) {
    n = *n_queries;
    if (blockIdx.x * blockDim.x >= n) return;
  }
  const uint32_t gi = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in_range = gi < n;
  if (gi == 0u) *next_count = 0u;  // the counter of the NEXT linearize (two counters alternate: no memset between launches)
  if (gi < kChunkClasses && cc.count_next) cc.count_next[gi] = 0u;
  const uint32_t i = in_range ? gi : n - 1u;
  const double3 tp = centred_translation(P.T, P.src.centre[0], P.src.centre[1], P.src.centre[2], P.tgt.centre);
  const float3 f = centred_query_f32(P.T, tp, __ldg(&P.src.pts[i]));
  const float fx = f.x, fy = f.y, fz = f.z;
  const float ax = floorf((fx - g.origin[0]) * g.inv_cell - 0.5f), ay = floorf((fy - g.origin[1]) * g.inv_cell - 0.5f),
              az = floorf((fz - g.origin[2]) * g.inv_cell - 0.5f);
  // queries far outside the target's box cannot be settled anyway; clamping keeps the integer cell coordinates in range
  const int bx = static_cast<int>(fminf(fmaxf(ax, -1e5f), 1e5f)), by = static_cast<int>(fminf(fmaxf(ay, -1e5f), 1e5f)),
            bz = static_cast<int>(fminf(fmaxf(az, -1e5f), 1e5f));
  const GridRuns e = grid_lookup(table, mask, bx, by, bz);
  // The four runs are scanned as one sequence (run r starts at position p_r = count[0] + ... + count[r - 1], and o_r maps a position
  // of run r to its point), unrolled by four so that four independent loads are in flight per thread.  The squared distance is
  // fma(dz, dz, fma(dy, dy, dx * dx)) in FP32 with round-to-nearest, and the candidate is the lexicographic minimum of (distance, leaf
  // position) -- within one block the same point the scan of a leaf-position-ordered list with a strict < keeps.
  uint64_t best_key = grid_cand_key(P.max_dist_sq, 0u);
  {
    const uint32_t p1 = e.count[0], p2 = p1 + e.count[1], p3 = p2 + e.count[2], total = p3 + e.count[3];
    const uint32_t o0 = e.start[0], o1 = e.start[1] - p1, o2 = e.start[2] - p2, o3 = e.start[3] - p3;
#pragma unroll 4
    for (uint32_t j = 0; j < total; j++) {
      const uint32_t idx = j + (j >= p3 ? o3 : j >= p2 ? o2 : j >= p1 ? o1 : o0);
      const float4 t = __ldg(&grid_pts[idx]);
      const float dx = __fsub_rn(t.x, fx), dy = __fsub_rn(t.y, fy), dz = __fsub_rn(t.z, fz);
      const uint64_t key = grid_cand_key(__fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx))), __float_as_uint(t.w));
      best_key = key < best_key ? key : best_key;
    }
  }
  float best_d = P.max_dist_sq;
  uint32_t best = kNone;
  if (best_key != grid_cand_key(P.max_dist_sq, 0u)) {
    best_d = __uint_as_float(static_cast<uint32_t>(best_key >> 32));
    best = static_cast<uint32_t>(best_key);
  }
  // a stored non-finite point (NaN query) is settled without a correspondence: no walk ever starts for it
  const bool settled = (best != kNone && best_d <= g.settle_d2) || isnan(fx);
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

cudaError_t launch_grid_build(const float4* leaf_pts, uint32_t n, const GridParams& g, int bits, uint64_t* keys_a, uint64_t* keys_b, uint32_t* vals_a, uint32_t* vals_b,
                              void* sort_temp, size_t sort_temp_bytes, float4* grid_pts, uint32_t* cnt, uint32_t* d_counters, cudaStream_t st) {
  const int end_bit = 3 * bits;
  const uint32_t m = n * 8u;
  grid_cell_keys_kernel<<<(n + 255u) / 256u, 256, 0, st>>>(leaf_pts, n, g, bits, keys_a, vals_a);
  cudaError_t e = cub::DeviceRadixSort::SortPairs(sort_temp, sort_temp_bytes, keys_a, keys_b, vals_a, vals_b, static_cast<int>(n), 0, end_bit, st);
  if (e != cudaSuccess) return e;
  // the cell-sorted keys / positions are read from keys_b / vals_b; the anchor entries go to keys_a / vals_a and are sorted back into b
  grid_cell_heads_kernel<<<(n + 255u) / 256u, 256, 0, st>>>(keys_b, vals_b, leaf_pts, n, bits, grid_pts, cnt, keys_a, vals_a);
  e = cub::DeviceRadixSort::SortPairs(sort_temp, sort_temp_bytes, keys_a, keys_b, vals_a, vals_b, static_cast<int>(m), 0, end_bit, st);
  if (e != cudaSuccess) return e;
  e = cudaMemsetAsync(d_counters, 0, 2 * sizeof(uint32_t), st);
  if (e != cudaSuccess) return e;
  grid_anchor_heads_kernel<<<(m + 255u) / 256u, 256, 0, st>>>(keys_b, vals_b, m, cnt, bits, d_counters);
  return cudaGetLastError();
}

cudaError_t launch_grid_fill(const uint64_t* akeys, const uint32_t* avals, uint32_t m, const uint32_t* cnt, int bits, GridSlot* table, uint32_t capacity,
                             cudaStream_t st) {
  grid_table_init_kernel<<<(capacity + 255u) / 256u, 256, 0, st>>>(table, capacity);
  grid_fill_kernel<<<(m + 255u) / 256u, 256, 0, st>>>(akeys, avals, m, cnt, bits, table, capacity - 1u);
  return cudaGetLastError();
}

cudaError_t launch_grid_probe(const LinParams& P, const uint32_t* n_queries, const float4* grid_pts, const GridSlot* table, uint32_t capacity,
                              const GridParams& g, uint8_t* state, uint32_t* pending_count, uint32_t* pending_list, float4* pending_q, uint32_t* next_count,
                              const ChunkClasses& cc, cudaStream_t st) {
  // *pending_count must be zero on entry: the previous probe (or the context) cleared it
  const uint32_t grid = (P.src.n + 255u) / 256u;  // with n_queries: P.src.n = the most queries a round can have
  if (n_queries)
    grid_probe_blocks_kernel<true><<<grid, 256, 0, st>>>(P, grid_pts, table, capacity - 1u, g, state, pending_count, pending_list, pending_q, next_count, cc, n_queries);
  else
    grid_probe_blocks_kernel<false><<<grid, 256, 0, st>>>(P, grid_pts, table, capacity - 1u, g, state, pending_count, pending_list, pending_q, next_count, cc, nullptr);
  return cudaGetLastError();
}

}  // namespace sgb
