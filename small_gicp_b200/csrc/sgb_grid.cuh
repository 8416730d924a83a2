// SPDX-License-Identifier: MIT
// Device-side pieces of the grid front end that more than one kernel uses: the block-table lookup and the warp-per-query search of
// the pending queries (ring phase over the block lists, then -- only beyond the ring's reach -- a warp-cooperative walk of the packet
// records).  The latter runs inside packet_search_kernel (sgb_kernels_packet.cu), which picks the regime from the probe's counter:
// one launch for both, where round 1 launched two kernels of which one exited at once.
#pragma once
#include "sgb_device.cuh"
#include "sgb_kernels.h"

namespace sgb {

// slack (in cells) for the FP32 cell-coordinate arithmetic: cell indices stay below 2^13 (build_grid), so a coordinate
// in cell units carries < 1e-3 of rounding error
constexpr float kGridSlack = 4e-3f;

// One entry of a block list: TWO points in one 32-byte sector, components interleaved: a = (x0, x1, y0, y1), b = (z0, z1, leaf
// position 0, leaf position 1).  A list with an odd number of points ends in a pad: coordinates kGridPadCoord (squared distance ~3e36:
// farther than anything real, still finite), position kNone.
struct __align__(32) GridPair {
  float4 a, b;
};
constexpr float kGridPadCoord = 1e18f;

// sm_90 has no 256-bit load: the record is two 128-bit read-only loads (LDG.E.128.CONSTANT) of the same sector
__device__ __forceinline__ GridPair load_pair(const GridPair* p) {
  GridPair r;
  r.a = __ldg(&p->a);
  r.b = __ldg(&p->b);
  return r;
}

__device__ __forceinline__ uint64_t grid_key(int ix, int iy, int iz) {
  return (static_cast<uint64_t>(static_cast<uint32_t>(ix + (1 << 20)) & 0x1fffffu)) | (static_cast<uint64_t>(static_cast<uint32_t>(iy + (1 << 20)) & 0x1fffffu) << 21) |
         (static_cast<uint64_t>(static_cast<uint32_t>(iz + (1 << 20)) & 0x1fffffu) << 42);
}
__device__ __forceinline__ uint32_t grid_hash(int ix, int iy, int iz) {
  uint32_t h = static_cast<uint32_t>(ix) * 73856093u ^ static_cast<uint32_t>(iy) * 19349663u ^ static_cast<uint32_t>(iz) * 83492791u;
  h ^= h >> 15;
  return h;
}
__device__ __forceinline__ uint32_t grid_hash_of_key(uint64_t k) {
  const int ix = static_cast<int>(k & 0x1fffffu) - (1 << 20), iy = static_cast<int>((k >> 21) & 0x1fffffu) - (1 << 20),
            iz = static_cast<int>((k >> 42) & 0x1fffffu) - (1 << 20);
  return grid_hash(ix, iy, iz);
}

__device__ __forceinline__ uint2 grid_lookup(const GridSlot* __restrict__ table, uint32_t mask, int ix, int iy, int iz) {
  const uint64_t k = grid_key(ix, iy, iz);
  uint32_t slot = grid_hash(ix, iy, iz) & mask;
  for (;;) {
    const uint4 e = __ldg(reinterpret_cast<const uint4*>(&table[slot]));
    const uint64_t ek = static_cast<uint64_t>(e.x) | (static_cast<uint64_t>(e.y) << 32);
    if (ek == k) return make_uint2(e.z, e.w);
    if (ek == ~0ull) return make_uint2(0u, 0u);
    slot = (slot + 1u) & mask;
  }
}


// ---------------------------------------------------------------------------------------------------------------
// Few pending queries (holes, outliers, borders: a few per mille to a few per cent, scattered): one WARP per query.
// Ring phase first (block lists): 27 lookups in parallel, the lists scanned as one flattened run over all lanes, a
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
  const GridPair* grid_pairs;  // block lists (pair records)
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
      // Ring phase (block lists): the 3 x 3 x 3 blocks at stride 2 around the query's own block tile the cells
      // [a - 2, a + 4)^3, i.e. they hold every target point within 2.5 cells of q.  One lookup and one list scan per lane,
      // all 27 in parallel, then a warp min: a handful of memory round trips instead of the ~45 of a tree walk.
      const float ux = (qx - R.g.origin[0]) * R.g.inv_cell, uy = (qy - R.g.origin[1]) * R.g.inv_cell, uz = (qz - R.g.origin[2]) * R.g.inv_cell;
      const int ax = static_cast<int>(fminf(fmaxf(floorf(ux - 0.5f), -1e5f), 1e5f)), ay = static_cast<int>(fminf(fmaxf(floorf(uy - 0.5f), -1e5f), 1e5f)),
                az = static_cast<int>(fminf(fmaxf(floorf(uz - 0.5f), -1e5f), 1e5f));
      uint2 e = make_uint2(0u, 0u);
      if (lane < 27u) {
        const int bx = ax + 2 * (static_cast<int>(lane % 3u) - 1), by = ay + 2 * (static_cast<int>((lane / 3u) % 3u) - 1),
                  bz = az + 2 * (static_cast<int>(lane / 9u) - 1);
        const float ex = fmaxf(fmaxf(static_cast<float>(bx) - ux, ux - static_cast<float>(bx + 2)) - kGridSlack, 0.0f);
        const float ey = fmaxf(fmaxf(static_cast<float>(by) - uy, uy - static_cast<float>(by + 2)) - kGridSlack, 0.0f);
        const float ez = fmaxf(fmaxf(static_cast<float>(bz) - uz, uz - static_cast<float>(bz + 2)) - kGridSlack, 0.0f);
        if ((ex * ex + ey * ey + ez * ez) * R.cell * R.cell < best_d) e = grid_lookup(R.table, R.mask, bx, by, bz);
      }
      // The (typically ~9 non-empty) lists are scanned as ONE flattened run spread over all 32 lanes: point j of the
      // concatenation (of pair records) goes to lane j mod 32, which finds its list by a shuffle binary search over the exclusive prefix
      // sums of the counts.  A lane per list would walk up to ~40 points in dependent batches; this is ~7 loads per lane.
      const uint32_t np = (e.y + 1u) >> 1;  // records of this lane's list (two points each)
      uint32_t incl = np;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= static_cast<uint32_t>(o)) incl += t;
      }
      const uint32_t excl = incl - np, total = __shfl_sync(0xffffffffu, incl, 31);
      float my_d = best_d;
      uint32_t my_best = kNone;
#pragma unroll 2
      for (uint32_t base = 0; base < total; base += 32u) {
        const uint32_t j = base + lane;
        uint32_t owner = 0;  // largest lane whose exclusive prefix is <= j (empty lists share their successor's prefix and lose)
#pragma unroll
        for (uint32_t step = 16u; step >= 1u; step >>= 1) {
          const uint32_t cand = owner + step;
          const uint32_t ex = __shfl_sync(0xffffffffu, excl, cand & 31u);
          if (cand < 32u && ex <= j) owner = cand;
        }
        const uint32_t st = __shfl_sync(0xffffffffu, e.x, owner), ex0 = __shfl_sync(0xffffffffu, excl, owner);
        if (j < total) {
          const GridPair t = load_pair(R.grid_pairs + st + (j - ex0));
          const float dx0 = t.a.x - qx, dy0 = t.a.z - qy, dz0 = t.b.x - qz;
          const float dx1 = t.a.y - qx, dy1 = t.a.w - qy, dz1 = t.b.y - qz;
          const float d0 = dx0 * dx0 + dy0 * dy0 + dz0 * dz0, d1 = dx1 * dx1 + dy1 * dy1 + dz1 * dz1;
          if (d0 < my_d) {
            my_d = d0;
            my_best = __float_as_uint(t.b.z);
          }
          if (d1 < my_d) {  // (a pad never is: ~3e36)
            my_d = d1;
            my_best = __float_as_uint(t.b.w);
          }
        }
      }
      const uint32_t dbits = my_best != kNone ? __float_as_uint(my_d) : 0x7f800000u;
      const uint32_t dmin = __reduce_min_sync(0xffffffffu, dbits);
      if (dmin != 0x7f800000u) {
        const unsigned who = __ballot_sync(0xffffffffu, dbits == dmin);
        best = __shfl_sync(0xffffffffu, my_best, __ffs(who) - 1);
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
