// SPDX-License-Identifier: MIT
// Device-side pieces of the grid front end that more than one kernel uses: the block-table lookup and the warp-per-query search of
// the pending queries (ring phase over the block table, then -- only beyond the ring's reach -- a warp-cooperative walk of the packet
// records).  The latter runs inside packet_search_kernel (sgb_kernels_packet.cu), which picks the regime from the probe's counter:
// one launch for both, where round 1 launched two kernels of which one exited at once.
#pragma once
#include "sgb_device.cuh"
#include "sgb_kernels.h"

namespace sgb {

// slack (in cells) for the FP32 cell-coordinate arithmetic: cell indices stay below 2^13 (build_grid), so a coordinate
// in cell units carries < 1e-3 of rounding error
constexpr float kGridSlack = 4e-3f;

__device__ __forceinline__ uint64_t grid_key(int ix, int iy, int iz) {
  return (static_cast<uint64_t>(static_cast<uint32_t>(ix + (1 << 20)) & 0x1fffffu)) | (static_cast<uint64_t>(static_cast<uint32_t>(iy + (1 << 20)) & 0x1fffffu) << 21) |
         (static_cast<uint64_t>(static_cast<uint32_t>(iz + (1 << 20)) & 0x1fffffu) << 42);
}
__device__ __forceinline__ uint32_t grid_hash(int ix, int iy, int iz) {
  uint32_t h = static_cast<uint32_t>(ix) * 73856093u ^ static_cast<uint32_t>(iy) * 19349663u ^ static_cast<uint32_t>(iz) * 83492791u;
  h ^= h >> 15;
  return h;
}

/// The four runs of one block (sgb_kernels.h: GridSlot); all counts zero when the block is empty.
struct GridRuns {
  uint32_t start[4], count[4];
};

/// One slot = one sector, read by two 128-bit loads issued together.
__device__ __forceinline__ GridRuns grid_lookup(const GridSlot* __restrict__ table, uint32_t mask, int ix, int iy, int iz) {
  const uint64_t k = grid_key(ix, iy, iz);
  uint32_t slot = grid_hash(ix, iy, iz) & mask;
  GridRuns r;
  for (;;) {
    const uint4* p = reinterpret_cast<const uint4*>(&table[slot]);
    const uint4 a = __ldg(p), b = __ldg(p + 1);
    const uint64_t ek = static_cast<uint64_t>(a.x) | (static_cast<uint64_t>(a.y) << 32);
    if (ek == k) {
      r.start[0] = a.z;
      r.start[1] = a.w;
      r.start[2] = b.x;
      r.start[3] = b.y;
      r.count[0] = b.z & 0xffffu;
      r.count[1] = b.z >> 16;
      r.count[2] = b.w & 0xffffu;
      r.count[3] = b.w >> 16;
      return r;
    }
    if (ek == ~0ull) {
#pragma unroll
      for (int j = 0; j < 4; j++) r.start[j] = r.count[j] = 0u;
      return r;
    }
    slot = (slot + 1u) & mask;
  }
}

/// Lexicographic minimum of (squared distance, leaf position): the key of a candidate is its distance's bits (non-negative floats
/// order like their bits) above its leaf position.  Starting from (bits(bound), 0) only points strictly closer than the bound enter.
__device__ __forceinline__ uint64_t grid_cand_key(float d, uint32_t pos) { return (static_cast<uint64_t>(__float_as_uint(d)) << 32) | pos; }

// ---------------------------------------------------------------------------------------------------------------
// Few pending queries (holes, outliers, borders: a few per mille to a few per cent, scattered): one WARP per query.
// Ring phase first (block table): 27 lookups in parallel, their 108 runs scanned as one flattened run over all lanes, a
// hardware min -- a handful of memory round trips.  Only if the ring's radius (2.5 cells) does not decide the query does
// the warp walk the packet records: every step of a single walk is a dependent load, so a thread per query would be
// pure latency; with a warp per query a leaf's points are fetched by one coalesced
// load and reduced by a hardware min, and thousands of walks are in flight at once.  Runs (inside packet_search_kernel) when at most N / pending_div queries
// are pending; with more, the packet search over the chunk-ordered queries takes them.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kPendWarps = kLinBlock / 32;
constexpr int kPendStack = 40;

__device__ __forceinline__ float grid_box_dist2(float qx, float qy, float qz, const float4& lo, const float4& hi) {
  const float dx = fmaxf(fmaxf(lo.x - qx, qx - hi.x), 0.0f);
  const float dy = fmaxf(fmaxf(lo.y - qy, qy - hi.y), 0.0f);
  const float dz = fmaxf(fmaxf(lo.z - qz, qz - hi.z), 0.0f);
  return dx * dx + dy * dy + dz * dz;
}

/// What the warp-per-query search needs besides LinParams (filled by the host, see launch_packet_search).
struct RingParams {
  const uint32_t* list;     // pending list: source positions, [*count] entries
  const float4* q;          // parallel to it: transformed query (x, y, z) and the squared distance of the probe's best candidate (w)
  const float4* grid_pts;   // target points in cell (raster) order: (x, y, z, leaf position)
  const GridSlot* table;    // block table (null: no ring phase, every pending query walks the tree)
  uint32_t mask;
  GridParams g;
  float cell;
};

/// desc / dist: this warp's pending-subtree stack in shared memory (kPendStack entries each)
__device__ __forceinline__ void pending_search_body(const LinParams& P, const float4* __restrict__ pnodes, uint32_t count, const RingParams& R, uint2* desc, float* dist) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  const float4* __restrict__ pts = P.tgt.pts;
  for (uint32_t k = warp; k < count; k += n_warps) {
    // everything below is warp-uniform except the leaf scan.  The probe left the transformed query and the squared distance of its
    // best candidate in the pending record (corr[i] already holds that candidate): no source load, no seed gather on this chain.
    const uint32_t i = R.list[k];
    const float4 rec = __ldg(&R.q[k]);
    const float qx = rec.x, qy = rec.y, qz = rec.z;
    float best_d = rec.w;
    uint32_t best = kNone;  // "nothing closer than the probe's candidate found (yet)"
    if (R.table) {
      // Ring phase (block table): the 3 x 3 x 3 blocks at stride 2 around the query's own block tile the cells
      // [a - 2, a + 4)^3, i.e. they hold every target point within 2.5 cells of q.  One lookup per lane, all 27 in parallel, their
      // 4 runs each scanned together, then a warp min: a handful of memory round trips instead of the ~45 of a tree walk.
      const float ux = (qx - R.g.origin[0]) * R.g.inv_cell, uy = (qy - R.g.origin[1]) * R.g.inv_cell, uz = (qz - R.g.origin[2]) * R.g.inv_cell;
      const int ax = static_cast<int>(fminf(fmaxf(floorf(ux - 0.5f), -1e5f), 1e5f)), ay = static_cast<int>(fminf(fmaxf(floorf(uy - 0.5f), -1e5f), 1e5f)),
                az = static_cast<int>(fminf(fmaxf(floorf(uz - 0.5f), -1e5f), 1e5f));
      GridRuns e;
#pragma unroll
      for (int r = 0; r < 4; r++) e.start[r] = e.count[r] = 0u;
      if (lane < 27u) {
        const int bx = ax + 2 * (static_cast<int>(lane % 3u) - 1), by = ay + 2 * (static_cast<int>((lane / 3u) % 3u) - 1),
                  bz = az + 2 * (static_cast<int>(lane / 9u) - 1);
        const float ex = fmaxf(fmaxf(static_cast<float>(bx) - ux, ux - static_cast<float>(bx + 2)) - kGridSlack, 0.0f);
        const float ey = fmaxf(fmaxf(static_cast<float>(by) - uy, uy - static_cast<float>(by + 2)) - kGridSlack, 0.0f);
        const float ez = fmaxf(fmaxf(static_cast<float>(bz) - uz, uz - static_cast<float>(bz + 2)) - kGridSlack, 0.0f);
        if ((ex * ex + ey * ey + ez * ez) * R.cell * R.cell < best_d) e = grid_lookup(R.table, R.mask, bx, by, bz);
      }
      // The (typically ~9 non-empty) blocks' up to 108 runs are scanned as ONE flattened run spread over all 32 lanes: point j of the
      // concatenation goes to lane j mod 32, which finds the block by a shuffle binary search over the exclusive prefix sums of the
      // blocks' sizes, then the run within it from the block's partial sums.  off[r] = start of run r minus the points before it.
      const uint32_t p1 = e.count[0], p2 = p1 + e.count[1], p3 = p2 + e.count[2], np = p3 + e.count[3];
      const uint32_t off0 = e.start[0], off1 = e.start[1] - p1, off2 = e.start[2] - p2, off3 = e.start[3] - p3;  // (mod 2^32)
      uint32_t incl = np;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= static_cast<uint32_t>(o)) incl += t;
      }
      const uint32_t excl = incl - np, total = __shfl_sync(0xffffffffu, incl, 31);
      const uint64_t bound = grid_cand_key(best_d, 0u);
      uint64_t mine = bound;
#pragma unroll 2
      for (uint32_t base = 0; base < total; base += 32u) {
        const uint32_t j = base + lane;
        uint32_t owner = 0;  // largest lane whose exclusive prefix is <= j (empty blocks share their successor's prefix and lose)
#pragma unroll
        for (uint32_t step = 16u; step >= 1u; step >>= 1) {
          const uint32_t cand = owner + step;
          const uint32_t ex = __shfl_sync(0xffffffffu, excl, cand & 31u);
          if (cand < 32u && ex <= j) owner = cand;
        }
        const uint32_t ex0 = __shfl_sync(0xffffffffu, excl, owner);
        const uint32_t q1 = __shfl_sync(0xffffffffu, p1, owner), q2 = __shfl_sync(0xffffffffu, p2, owner), q3 = __shfl_sync(0xffffffffu, p3, owner);
        const uint32_t o0 = __shfl_sync(0xffffffffu, off0, owner), o1 = __shfl_sync(0xffffffffu, off1, owner);
        const uint32_t o2 = __shfl_sync(0xffffffffu, off2, owner), o3 = __shfl_sync(0xffffffffu, off3, owner);
        if (j < total) {
          const uint32_t local = j - ex0;
          const uint32_t idx = local + (local >= q3 ? o3 : local >= q2 ? o2 : local >= q1 ? o1 : o0);
          const float4 t = __ldg(&R.grid_pts[idx]);
          const float dx = t.x - qx, dy = t.y - qy, dz = t.z - qz;
          const uint64_t key = grid_cand_key(dx * dx + dy * dy + dz * dz, __float_as_uint(t.w));
          mine = key < mine ? key : mine;
        }
      }
      // warp minimum of (distance, leaf position): the smallest distance first, then the lowest position among the lanes holding it
      const uint32_t dbits = mine != bound ? static_cast<uint32_t>(mine >> 32) : 0x7f800000u;
      const uint32_t dmin = __reduce_min_sync(0xffffffffu, dbits);
      if (dmin != 0x7f800000u) {
        best = __reduce_min_sync(0xffffffffu, dbits == dmin ? static_cast<uint32_t>(mine) : kNone);
        best_d = __uint_as_float(dmin);
      }
      const float cover = (2.5f - kGridSlack) * R.cell;
      if (best_d <= cover * cover) {  // everything within sqrt(best_d) of q has been examined: exact (or exactly nothing)
        if (lane == 0 && best != kNone) P.corr[i] = best;
        continue;
      }
    }
    int sp = 0;
    uint32_t cur = 0;
    bool expand = true;
    uint2 leaf = make_uint2(0u, 0u);
    for (;;) {
      if (expand) {
        const float4 n0 = __ldg(&pnodes[cur * 4 + 0]), n1 = __ldg(&pnodes[cur * 4 + 1]);
        const float4 n2 = __ldg(&pnodes[cur * 4 + 2]), n3 = __ldg(&pnodes[cur * 4 + 3]);
        const float dl = grid_box_dist2(qx, qy, qz, n0, n1), dr = grid_box_dist2(qx, qy, qz, n2, n3);
        const bool left_first = dl <= dr;
        const float dn = left_first ? dl : dr, df = left_first ? dr : dl;
        const uint2 cl = make_uint2(__float_as_uint(n0.w), __float_as_uint(n1.w)), cr = make_uint2(__float_as_uint(n2.w), __float_as_uint(n3.w));
        const uint2 cn = left_first ? cl : cr, cf = left_first ? cr : cl;
        if (df < best_d && sp < kPendStack) {
          if (lane == 0) {
            desc[sp] = cf;
            dist[sp] = df;
          }
          sp++;
        }
        if (!(dn < best_d)) {
          expand = false;
          continue;
        }
        if (cn.y == 0u) {
          cur = cn.x;
          continue;
        }
        leaf = cn;
      } else {
        // Every popped descriptor is read (volatile) before the test.  When the read sits behind the test, ptxas of CUDA 12.9 for sm_90a
        // sinks it out of the loop and addresses desc[sp - 1] -- the entry below, at sp == 0 the bytes before this warp's stack.
        bool got = false;
        __syncwarp();
        while (sp > 0) {
          sp--;
          const volatile uint2* e = desc + sp;
          const uint2 c = make_uint2(e->x, e->y);
          if (dist[sp] < best_d) {
            leaf = c;
            got = true;
            break;
          }
        }
        __syncwarp();
        if (!got) break;
        if (leaf.y == 0u) {
          cur = leaf.x;
          expand = true;
          continue;
        }
      }
      // leaf: lane j takes point j, the nearest comes out of one hardware min (non-negative floats order like their bits)
      for (uint32_t base = 0; base < leaf.y; base += 32u) {
        const uint32_t j = base + lane;
        uint32_t dbits = 0x7f800000u;
        if (j < leaf.y) {
          const float4 t = __ldg(&pts[leaf.x + j]);
          const float dx = t.x - qx, dy = t.y - qy, dz = t.z - qz;
          dbits = __float_as_uint(dx * dx + dy * dy + dz * dz);
        }
        const uint32_t dmin = __reduce_min_sync(0xffffffffu, dbits);
        const float d = __uint_as_float(dmin);
        if (d < best_d) {
          const unsigned who = __ballot_sync(0xffffffffu, dbits == dmin);  // lowest lane = first point in scan order
          best_d = d;
          best = leaf.x + base + (__ffs(who) - 1);
        }
      }
      expand = false;
    }
    if (lane == 0 && best != kNone) P.corr[i] = best;
  }
}


}  // namespace sgb
