// SPDX-License-Identifier: MIT
// Warp-cooperative ("packet") exact nearest-neighbour search -- the search phase of linearize.
//
// A warp owns 32 CONSECUTIVE source points of the Morton order, i.e. 32 queries that sit within a small patch of the
// surface.  Instead of 32 divergent per-thread walks (a third of the lanes active, every lane issuing its own
// node and point loads), the warp walks the tree ONCE with a single shared traversal stack:
//   * every control-flow decision is a warp vote, so the instruction stream never diverges;
//   * node and leaf-point addresses are warp-uniform: one 64 B node / one 16 B point is fetched per warp and broadcast;
//   * each lane keeps only its own query, best distance and best index; a subtree is entered when ANY lane's search
//     ball reaches its bounding box, and every lane tests every point of an entered leaf (a superset of what it would
//     test alone -- the result is still its exact nearest neighbour).
// The tree is the kd-tree (same leaves, same permutation) with each inner node carrying the tight bounding boxes of its two
// children (64 B, "BVH2" layout):  float4[4] = {L.lo|L.a, L.hi|L.b, R.lo|R.a, R.hi|R.b} where a child is a leaf
// (a = first point, b = count > 0) or an inner node (a = node index, b = 0).
// forest_search_kernel (sgb_forest.cu) copies this walk for a batch over many trees, one member per warp.  One kernel serves the search
// of linearize and, with ROUND, the rounds of sgb_align_batch_async, whose query count is read from the device.
#include <algorithm>
#include <cfloat>
#include <cstdlib>

#include "sgb_device.cuh"
#include "sgb_grid.cuh"
#include "sgb_kernels.h"

namespace sgb {

constexpr int kPktWarps = kLinBlock / 32;
// a leaf wanted by more lanes than this is scanned by all lanes (10 instr / point); otherwise the interested lanes are
// served one by one by the whole warp (~16 instr / lane): break-even ~ points_per_leaf * 10 / 16
constexpr int kPacketDenseLanes = 18;
// resident CTAs per SM the kernel is compiled for: the compiler's own 48 registers -> 10 CTAs x 4 warps.  Forcing 12 (40 registers, 8 B
// of spills) is the profiling library's A/B (SGB_PACKET_CTAS=12).
constexpr int kPacketCtas = 10;

// ---- TMA staging of a leaf's point block (BASELINE north_star: "TMA bulk loads for the leaf point blocks") ----------------------
// One elected lane arms the warp's mbarrier with the byte count and issues ONE cp.async.bulk (SASS UBLKCP) for the leaf's contiguous
// <= 32 x 16 B; the warp waits on the barrier's phase and then reads the points from shared memory.  TMA_LEAF is a compile-time A/B:
// kept in the profiling library (the broadcast __ldg path below serves an L1-resident leaf in ~32 cycles per load, pipelined; the bulk copy
// always makes the round trip through L2) -- DESIGN.md §4 says which variant ships.
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(bar))), "r"(count));
}
__device__ __forceinline__ void bulk_load_leaf(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  const uint32_t b = static_cast<uint32_t>(__cvta_generic_to_shared(bar)), d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(d), "l"(gsrc), "r"(bytes), "r"(b) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  const uint32_t b = static_cast<uint32_t>(__cvta_generic_to_shared(bar));
  uint32_t done = 0;
  while (!done) {
    asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(done)
      : "r"(b), "r"(phase)
      : "memory");
  }
}

// ROUND (a round of sgb_align_batch_async): *n_queries queries (written on the device by the round's planner), the regime picked from
// n_queries / pending_div as launch_packet_search picks it on the host; the planner cleared the queue counters.
template <bool TMA_LEAF, int MIN_CTAS, bool ROUND>
__global__ void __launch_bounds__(kLinBlock, MIN_CTAS) packet_search_kernel(const __grid_constant__ LinParams P, const float4* __restrict__ pnodes, int max_depth,
                                                                  const uint8_t* __restrict__ settled, const uint32_t* __restrict__ pending_count,
                                                                  uint32_t min_pending, uint32_t* queue, uint32_t* queue_next, ChunkClasses cc, RingParams ring,
                                                                  const uint32_t* __restrict__ n_queries, uint32_t pending_div) {
  const uint32_t n_src = ROUND ? *n_queries : P.src.n;
  if constexpr (ROUND) {
    if (n_src == 0) return;
    min_pending = n_src / pending_div;
  }
  // Work distribution: chunks (32 consecutive queries) differ wildly in cost -- all lanes settled by the grid probe, or 32
  // tree walks through a misaligned wall -- and a static stride left a third of the warps idle for the second half of the
  // kernel (achieved occupancy far below the theoretical).  With `queue` the warps take their first chunk by rank and
  // every further one from a global counter.  Two counters alternate between launches: this launch clears the next one's
  // (launches of one context are stream-ordered, the next user is the packet search of the NEXT linearize).
  if (queue_next && blockIdx.x == 0 && threadIdx.x == 0) *queue_next = 0u;
  grid_dependency_wait();  // probe / pending search wrote corr[], the settled flags and the pending counter
  extern __shared__ float s_dist[];  // [max_depth][kLinBlock] per-lane box distance of each pending subtree
  __shared__ uint2 s_child[kPktWarps][40];  // per-warp: the pending subtrees themselves (warp-uniform)
  __shared__ __align__(128) float4 s_leaf[TMA_LEAF ? kPktWarps : 1][32];  // TMA landing zone of the warp's current leaf
  __shared__ __align__(8) uint64_t s_bar[TMA_LEAF ? kPktWarps : 1];
  // Two regimes, picked from the probe's counter: FEW pending queries (holes, borders, outliers at an aligned pose) -> a warp per query
  // (ring phase over the block table, tree walk only beyond its reach: sgb_grid.cuh); MANY (a misaligned first iteration) -> the packet
  // walk below.  One launch serves both (two kernels, one of which exits at once, cost a launch per linearize).
  if (pending_count) {
    const uint32_t pc = *pending_count;
    if (pc <= min_pending) {
      if (pc) pending_search_body(P, pnodes, pc, ring, s_child[threadIdx.x >> 5], s_dist + (threadIdx.x >> 5) * kPendStack);
      return;
    }
  }
  uint32_t tma_phase = 0;
  if (TMA_LEAF) {
    if ((threadIdx.x & 31u) == 0) mbar_init(&s_bar[threadIdx.x >> 5], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();
  }
  const double* R = P.T;
  const double3 tp = centred_translation(P.T, P.src.centre[0], P.src.centre[1], P.src.centre[2], P.tgt.centre);
  const float4* __restrict__ pts = P.tgt.pts;
  const uint32_t lane = threadIdx.x & 31u, wib = threadIdx.x >> 5;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  float* my_dist = s_dist + threadIdx.x;
  uint2* my_child = s_child[wib];
  // What there is to do: with the probe's class lists (cc.lists) the work items are the chunks that have a pending lane, the widest
  // search balls first -- positions [0, n0) of the virtual sequence are class 0, [n0, n0 + n1) class 1, ... -- so that the GPU drains
  // on cheap walks; without lists every chunk of the source is an item and the settled flags are consulted here.
  uint32_t c0 = 0, c1 = 0, n_items = (n_src + 31u) >> 5;
  if (cc.lists) {
    c0 = cc.count[0];
    c1 = c0 + cc.count[1];
    // The lists are in the order the probe's warps happened to finish: neighbouring items are NOT neighbouring chunks, so the warps of
    // an SM no longer share tree nodes through L1.  When nearly every chunk has pending lanes anyway (a grossly misaligned first
    // iteration: nothing to skip, no cheap tail to save for the end) the curve order wins (threshold: class_fallback_pct).
    const uint32_t listed = c1 + cc.count[2];
    if (listed * 100u > n_items * cc.fallback_pct) cc.lists = nullptr;
    else n_items = listed;
  }

  for (uint32_t item = warp; item < n_items;) {
    uint32_t chunk = item;
    if (cc.lists) chunk = item < c0 ? cc.lists[item] : (item < c1 ? cc.lists[cc.n_chunks + (item - c0)] : cc.lists[2u * cc.n_chunks + (item - c1)]);
    const uint32_t i = chunk * 32u + lane;
    // the item after this one: from the queue (dynamic) or by stride (static)
    uint32_t next_item = item + n_warps;
    if (queue) {
      if (lane == 0) next_item = n_warps + atomicAdd(queue, 1u);
      next_item = __shfl_sync(0xffffffffu, next_item, 0);
    }
    // with the grid front end (sgb_grid.cu) most queries are already settled; only the pending ones walk the tree,
    // seeded with the candidate the grid probe left in corr[]
    const bool valid = i < n_src && !(settled && settled[i]);
    if (!__any_sync(0xffffffffu, valid)) {
      item = next_item;
      continue;
    }
    float fx = 0.f, fy = 0.f, fz = 0.f;
    float best_d = -1.0f;  // an idle lane is never interested in anything
    uint32_t best = kNone;
    if (valid) {
      const float3 f = centred_query_f32(R, tp, __ldg(&P.src.pts[i]));
      fx = f.x;
      fy = f.y;
      fz = f.z;
      best_d = isnan(fx) ? -1.0f : P.max_dist_sq;  // a stored non-finite point (NaN query): no search, as an idle lane
      const uint32_t prev = (P.use_prev || settled) ? P.corr[i] : kNone;  // seed: an upper bound only prunes
      if (prev != kNone) {
        const float4 t = __ldg(&pts[prev]);
        const float dx = t.x - fx, dy = t.y - fy, dz = t.z - fz;
        const float d = dx * dx + dy * dy + dz * dz;
        if (d < best_d) {
          best_d = d;
          best = prev;
        }
      }
    }

    int sp = 0;
    uint32_t cur = 0;      // inner node being expanded
    bool expand = true;    // false: nothing to expand, take the next pending subtree
    uint32_t leaf_first = 0, leaf_cnt = 0;
    float leaf_d = 0.f;  // this lane's distance to the box of the leaf about to be scanned
    for (;;) {
      if (expand) {
        const float4 n0 = __ldg(&pnodes[cur * 4 + 0]), n1 = __ldg(&pnodes[cur * 4 + 1]);
        const float4 n2 = __ldg(&pnodes[cur * 4 + 2]), n3 = __ldg(&pnodes[cur * 4 + 3]);
        const float dl = box_dist2(fx, fy, fz, n0, n1), dr = box_dist2(fx, fy, fz, n2, n3);
        const bool wl = dl < best_d, wr = dr < best_d;
        const unsigned ml = __ballot_sync(0xffffffffu, wl), mr = __ballot_sync(0xffffffffu, wr);
        uint32_t ca, cb;  // descriptor of the child to enter now
        if (ml && mr) {
          // enter the child most interested lanes are closer to, keep the other pending
          const unsigned closer_l = __ballot_sync(0xffffffffu, (wl || wr) && dl <= dr);
          const bool left_first = 2 * __popc(closer_l) >= __popc(ml | mr);
          my_dist[sp * kLinBlock] = left_first ? dr : dl;
          if (lane == 0) my_child[sp] = left_first ? make_uint2(__float_as_uint(n2.w), __float_as_uint(n3.w)) : make_uint2(__float_as_uint(n0.w), __float_as_uint(n1.w));
          sp++;
          ca = left_first ? __float_as_uint(n0.w) : __float_as_uint(n2.w);
          cb = left_first ? __float_as_uint(n1.w) : __float_as_uint(n3.w);
          leaf_d = left_first ? dl : dr;
        } else if (ml) {
          ca = __float_as_uint(n0.w);
          cb = __float_as_uint(n1.w);
          leaf_d = dl;
        } else if (mr) {
          ca = __float_as_uint(n2.w);
          cb = __float_as_uint(n3.w);
          leaf_d = dr;
        } else {
          expand = false;
          continue;
        }
        if (cb == 0u) {  // inner child
          cur = ca;
          continue;
        }
        leaf_first = ca;
        leaf_cnt = cb;
      } else {
        // next pending subtree some lane still cares about
        bool got = false;
        uint2 c = make_uint2(0u, 0u);
        while (sp > 0) {
          sp--;
          const float d = my_dist[sp * kLinBlock];
          if (__any_sync(0xffffffffu, d < best_d)) {
            __syncwarp();  // lane 0's push of this entry is visible
            c = my_child[sp];
            __syncwarp();  // ... and every lane has read it before lane 0 may push over it (entries popped unread need neither)
            leaf_d = d;
            got = true;
            break;
          }
        }
        if (!got) break;
        if (c.y == 0u) {
          cur = c.x;
          expand = true;
          continue;
        }
        leaf_first = c.x;
        leaf_cnt = c.y;
      }
      // ---- leaf ----
      // Only the lanes whose ball reaches this leaf's box need its points; typically a handful of the 32.
      unsigned want = __ballot_sync(0xffffffffu, leaf_d < best_d);
      if (__popc(want) > kPacketDenseLanes) {
        // many interested lanes: every lane tests every point (uniform addresses -> one broadcast load per point)
        const float4* lp = pts + leaf_first;
        if (TMA_LEAF && leaf_cnt <= 32u) {
          __syncwarp();  // everybody is done with the previous leaf in the landing zone
          if (lane == 0) bulk_load_leaf(s_leaf[wib], lp, leaf_cnt * 16u, &s_bar[wib]);
          mbar_wait(&s_bar[wib], tma_phase);
          tma_phase ^= 1u;
          lp = s_leaf[wib];
        }
#pragma unroll 4
        for (uint32_t j = 0; j < leaf_cnt; j++) {
          const float4 t = (TMA_LEAF && leaf_cnt <= 32u) ? lp[j] : __ldg(&lp[j]);
          const float dx = t.x - fx, dy = t.y - fy, dz = t.z - fz;
          const float d = dx * dx + dy * dy + dz * dz;
          if (d < best_d) {
            best_d = d;
            best = leaf_first + j;
          }
        }
      } else {
        // few interested lanes: serve them one at a time with the WHOLE warp -- lane j holds point j of the leaf, the
        // query is broadcast by shuffle, the nearest point comes out of one hardware min-reduction (squared distances
        // are non-negative floats, so their bit patterns order like unsigned integers)
        for (uint32_t base = 0; base < leaf_cnt; base += 32u) {
          const uint32_t j = base + lane;
          float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
          if (j < leaf_cnt) t = __ldg(&pts[leaf_first + j]);
          unsigned todo = want;
          while (todo) {
            const int src = __ffs(todo) - 1;
            todo &= todo - 1;
            const float qx = __shfl_sync(0xffffffffu, fx, src), qy = __shfl_sync(0xffffffffu, fy, src), qz = __shfl_sync(0xffffffffu, fz, src);
            const float dx = t.x - qx, dy = t.y - qy, dz = t.z - qz;
            const uint32_t dbits = j < leaf_cnt ? __float_as_uint(dx * dx + dy * dy + dz * dz) : 0x7f800000u;
            const uint32_t dmin = __reduce_min_sync(0xffffffffu, dbits);
            const unsigned who = __ballot_sync(0xffffffffu, dbits == dmin);  // lowest lane = first point in scan order
            if (static_cast<int>(lane) == src) {
              const float d = __uint_as_float(dmin);
              if (d < best_d) {
                best_d = d;
                best = leaf_first + base + (__ffs(who) - 1);
              }
            }
          }
        }
      }
      expand = false;
    }
    __syncwarp();
    if (valid) P.corr[i] = best;
    item = next_item;
  }
}

int packet_occupancy(int max_depth) {
  const size_t smem = std::max(static_cast<size_t>(max_depth > 0 ? max_depth : 1) * kLinBlock, static_cast<size_t>(kPktWarps) * kPendStack) * sizeof(float);
  return ctas_per_sm(packet_search_kernel<false, kPacketCtas, false>, kLinBlock, smem, false, false);
}

namespace {
RingParams ring_params(const PendingParams& pp) {
  RingParams ring;
  ring.list = pp.list;
  ring.q = pp.q;
  ring.grid_pts = pp.grid_pts;
  ring.table = pp.table;
  ring.mask = pp.capacity ? pp.capacity - 1u : 0u;
  ring.g = pp.g;
  ring.cell = pp.g.inv_cell > 0.f ? 1.0f / pp.g.inv_cell : 0.f;
  return ring;
}
}  // namespace

cudaError_t launch_packet_search(const LinParams& P, const uint32_t* n_queries, const float4* pnodes, int grid, int max_depth, const uint8_t* settled,
                                 const uint32_t* pending_count, uint32_t pending_div, uint32_t* queue, uint32_t* queue_next, const ChunkClasses& cc,
                                 const PendingParams& pp, bool tma_leaf, cudaStream_t st) {
  if (max_depth > 40 || pending_div == 0) return cudaErrorInvalidValue;
  // per-lane box distances of the packet walk; the warp-per-query regime uses the first kPktWarps x kPendStack floats of it
  const size_t smem = std::max(static_cast<size_t>(max_depth > 0 ? max_depth : 1) * kLinBlock, static_cast<size_t>(kPktWarps) * kPendStack) * sizeof(float);
  const RingParams ring = ring_params(pp);
  if (n_queries) {
    packet_search_kernel<false, kPacketCtas, true><<<grid, kLinBlock, smem, st>>>(P, pnodes, max_depth, settled, pending_count, 0u, queue, queue_next, cc, ring,
                                                                                   n_queries, pending_div);
    return cudaGetLastError();
  }
  // more pending queries than this: packet search over the chunk-ordered queries, else a warp per pending query
  const uint32_t min_pending = P.src.n / pending_div;
  const uint32_t* none = nullptr;
#ifdef SGB_PROFILING
  if (tma_leaf) {  // A/B (SGB_TMA_LEAF=1): leaf blocks staged by cp.async.bulk + mbarrier
    if (!settled) {
      packet_search_kernel<true, kPacketCtas, false><<<grid, kLinBlock, smem, st>>>(P, pnodes, max_depth, settled, pending_count, min_pending, queue, queue_next, cc,
                                                                                    ring, none, 0u);
      return cudaGetLastError();
    }
    return launch_dependent(packet_search_kernel<true, kPacketCtas, false>, grid, kLinBlock, smem, st, P, pnodes, max_depth, settled, pending_count, min_pending,
                            queue, queue_next, cc, ring, none, 0u);
  }
#endif
#ifdef SGB_PROFILING
  static const bool twelve = std::getenv("SGB_PACKET_CTAS") && std::atoi(std::getenv("SGB_PACKET_CTAS")) == 12;  // A/B: 40 registers, 12 CTAs / SM
  if (twelve && settled)
    return launch_dependent(packet_search_kernel<false, 12, false>, grid, kLinBlock, smem, st, P, pnodes, max_depth, settled, pending_count, min_pending, queue,
                            queue_next, cc, ring, none, 0u);
#endif
  if (!settled) {  // no grid front end: nothing on the stream this launch could overlap with
    packet_search_kernel<false, kPacketCtas, false><<<grid, kLinBlock, smem, st>>>(P, pnodes, max_depth, settled, pending_count, min_pending, queue, queue_next, cc,
                                                                                   ring, none, 0u);
    return cudaGetLastError();
  }
  (void)tma_leaf;
  return launch_dependent(packet_search_kernel<false, kPacketCtas, false>, grid, kLinBlock, smem, st, P, pnodes, max_depth, settled, pending_count, min_pending,
                          queue, queue_next, cc, ring, none, 0u);
}

}  // namespace sgb
