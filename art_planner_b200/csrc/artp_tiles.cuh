// art_planner_b200/csrc/artp_tiles.cuh
// Stage B of the pose-validity pipeline: one WARP per queued box, the box's zone staged in shared memory by TMA.
//
// Every queued box needs the heights of its zone -- the sub-rectangle of the heightfield its AABB overlaps, ~9 x 9
// vertices for a reach box, ~40 x 40 for the torso (heightfield.cpp:1880-1892) -- several times: vertex scan, corner
// candidates, merge screen. The warp copies the zone into shared memory as ONE 2-D TMA tile
// (cp.async.bulk.tensor.2d with the tensor map of the layer; tile origin = zone origin rounded down to a multiple of 4
// columns because TMA needs 16-byte aligned row starts -- an unaligned inner coordinate traps as "illegal instruction",
// profiles/tma_probe.cu; out-of-map elements are zero-filled and never read) and double-buffers: while box i is decided
// out of tile slot i & 1, the tile of box i + 1 is already in flight into the other slot (one mbarrier per slot).
// No address arithmetic, L1 wavefronts or registers are spent on the gather, and all later reads are shared-memory reads.
//
// Three queues feed three launches: box_tiles_warp_kernel once over the big-tile queue (torso boxes; one tile slot per
// warp) and once over the reach boxes that need the merge screen or the zone reduction (small tiles, two slots), and
// reach_groups_kernel over the other reach boxes (merge-free, with or without -inf: four boxes per warp, below). A box
// whose zone does not fit its tile (cannot happen for the sizes the tiles are derived from) goes to the exact grouping stage.
// Queue records are claimed with guided chunk sizes (a share of what is left), one claim ahead of the work.
// Round 2 also tried one THREAD per reach box over the staged tiles (no cross-lane traffic at all): SIMT divergence
// left 8-10 of 32 lanes busy and it was slower (profiles/r02_v1_reach_*).
#pragma once

#include <cuda.h>

#include "artp_kernels.cuh"

namespace artp {

constexpr uint32_t kDeferReachBit = 0x80000000u;   // defer-list entry refers to the reach-box queue
constexpr int kTileChunk = 8;                      // most records claimed per atomic (the tile pipeline restarts per claim)

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "TWAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra TWAIT_DONE;\n\t"
      "bra TWAIT_LOOP;\n\t"
      "TWAIT_DONE:\n\t"
      "}" ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_tile_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_addr(dst)),
      "l"(map), "r"(smem_addr(bar)), "r"(c0), "r"(c1)
      : "memory");
}

constexpr int kMaxTileWarps = 8;

// This warp's `n` tile slots of tc.stride bytes in the dynamic shared memory (TMA destinations: 128-byte aligned), with
// its two mbarriers (one per slot parity) initialised.
__device__ __forceinline__ unsigned char* warp_tile_slots(unsigned char* smem, const TileCfg& tc, int n, uint64_t bars[2]) {
  const int wid = threadIdx.x >> 5;
  unsigned char* slots = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem) + 127) & ~(uintptr_t)127) +
                         (size_t)wid * n * tc.stride;
  if ((threadIdx.x & 31) == 0) { mbar_init(&bars[0], 1); mbar_init(&bars[1], 1); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncwarp();
  return slots;
}

// map0 / map1: tiles of `elevation` / `elevation_masked` (same tile extent). queue_bit tags defer-list entries.
__global__ void __launch_bounds__(kMaxTileWarps * 32, 3)
box_tiles_warp_kernel(const Checker c, const __grid_constant__ CUtensorMap map0, const __grid_constant__ CUtensorMap map1,
                      const TileCfg tc, const Work w, const BoxRec* __restrict__ recs, const uint32_t* __restrict__ rec_count,
                      uint32_t* __restrict__ work_counter, uint32_t* __restrict__ defer_count, uint32_t* __restrict__ defer_list,
                      uint32_t queue_bit, int force_defer) {
  extern __shared__ __align__(128) unsigned char tile_smem[];
  __shared__ WarpScratch ws_all[kMaxTileWarps];
  __shared__ uint64_t bars[kMaxTileWarps][2];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  WarpScratch& ws = ws_all[wid];
  unsigned char* slots = warp_tile_slots(tile_smem, tc, tc.slots, bars[wid]);
  uint32_t phase[2] = {0u, 0u};
  const uint32_t total = *rec_count;
  // lane 0 starts the copy of record ri's zone into tile slot `slot`
  auto prefetch = [&](uint32_t ri, int slot) {
    const int x0 = rec_x0(recs + ri), z0 = rec_z0(recs + ri);
    const uint32_t fl = rec_flags(recs + ri);
    if (lane == 0) {
      mbar_expect_tx(&bars[wid][slot], tc.bytes);
      tma_tile_2d(slots + (size_t)slot * tc.stride, (fl & 7u) ? &map1 : &map0, &bars[wid][slot], (x0 & ~3) - tc.x_off, z0);
    }
  };
  // Guided claims: a share of what is left (1 .. kTileChunk records), so that a short queue spreads over all warps
  // instead of keeping a few of them busy with kTileChunk boxes each (one box is ~5 us of dependent latency); the next
  // claim is issued before the current one is worked on, so its round trip hides behind the boxes.
  const uint32_t nwarps2 = 2u * gridDim.x * (blockDim.x >> 5);
  uint32_t next_r0 = 0, next_n = 0;     // lane 0's
  // (a long queue keeps fixed claims: measured, the guided sizes cost this kernel 15-20 % there -- a claim restarts the
  //  tile pipeline -- while they halve its time on short queues)
  const uint32_t first_seen = *(volatile const uint32_t*)work_counter;   // ~ where this launch's share of the queue begins
  const bool fixed_claims = total - min(first_seen, total) >= (nwarps2 >> 2) * (uint32_t)kTileChunk;
  auto claim = [&]() {
    if (lane == 0) {
      next_n = (uint32_t)kTileChunk;
      if (!fixed_claims) {
        const uint32_t cur = *(volatile const uint32_t*)work_counter;   // fresh: a stale value would hand out big claims at the end
        next_n = cur < total ? min(max((total - cur) / nwarps2, 1u), (uint32_t)kTileChunk) : 1u;
      }
      next_r0 = atomicAdd(work_counter, next_n);
    }
  };
  // guided claims are issued one ahead (their round trip hides behind the boxes; the sizes account for the chunk in hand),
  // fixed ones when needed (a warp holding two 8-box chunks would unbalance a queue of a few boxes per warp)
  if (!fixed_claims) claim();
  for (;;) {
    if (fixed_claims) claim();
    const uint32_t r0 = __shfl_sync(kFull, next_r0, 0), nclaim = __shfl_sync(kFull, next_n, 0);
    if (r0 >= total) break;
    if (!fixed_claims) claim();
    const uint32_t r1 = min(r0 + nclaim, total);
    if (force_defer) {
      if (lane == 0) for (uint32_t ri = r0; ri < r1; ++ri) defer_list[atomicAdd(defer_count, 1u)] = ri | queue_bit;
      continue;
    }
    for (uint32_t ri = r0; ri < r1; ++ri) {
      const int slot = (int)(ri - r0) & (tc.slots - 1);
      if (tc.slots == 1 || ri == r0) { __syncwarp(); prefetch(ri, slot); }   // every lane is done with the slot
      const BoxRec r = load_rec(recs + ri);   // every lane reads the whole record itself (broadcast loads)
      if (tc.slots == 2 && ri + 1 < r1) { __syncwarp(); prefetch(ri + 1, slot ^ 1); }   // the other slot's box (ri - 1) is finished
      const uint32_t slot_item = r.item;
      const bool foot = (r.flags & 7) != 0;
      // another box of the item (or state of the edge) already failed: nothing can change the verdict (perf only)
      int dead = 0;
      if (lane == 0) dead = (*(volatile const uint8_t*)(w.valid + slot_item) == 0);
      dead = __shfl_sync(kFull, dead, 0);
      mbar_wait(&bars[wid][slot], phase[slot]);       // the tile must land before its slot can be reused
      phase[slot] ^= 1u;
      if (dead) continue;
      BoxCtx b;
      rec_to_ctx(c, r, b);
      int res;
      if ((b.x1 - b.x0) + 4 > tc.tw || (b.z1 - b.z0) + 1 > tc.th) {
        res = R_DEFER;                                // zone larger than the tile: exact grouping stage
      } else {
        const ZoneView zv{reinterpret_cast<const float*>(slots + (size_t)slot * tc.stride) + (b.x0 & 3), tc.tw};
        res = box_collide_warp<true>(foot ? c.f[1] : c.f[0], b, zv, ws, lane, c.cell_margin, (r.flags & REC_NEEDS_REDUCE) != 0,
                                     (r.flags & REC_ALLFINITE) != 0, (r.flags & REC_MERGEFREE) != 0);
      }
      if (lane == 0) {
        if (res == R_DEFER) defer_list[atomicAdd(defer_count, 1u)] = ri | queue_bit;
        else if (box_fails(foot, res)) w.valid[slot_item] = 0;
      }
    }
  }
}

// -------------------------------------------------------------------------------------------------------------------
// Reach boxes of a merge-free zone (no screen, no grouping) reduced by the tables, with or without -inf heights. A reach
// box's 81 vertices / 8 corners do not fill a warp (the one-warp-per-box kernel above runs them at 20 of 32 lanes and pays
// its per-box overhead 1 : 1), so here a warp decides FOUR boxes at a time, 8 lanes each: lane = vertex in the vertex
// stage, lane = corner when the candidate cells are collected; the candidate (cell, triangle) tasks of the four boxes are
// then POOLED: lane = one task of any of the four boxes (its box read from shared memory), so the test loop runs
// ceil(total / 32) times instead of as long as the longest of four 8-lane lists.
// The vertex and collection stages run the four groups in lock-step through the same loops (trip counts = the maximum over
// the groups, finished groups predicated off), so every ballot is a full-warp ballot and a group's result is a byte of it.
// Every warp-wide exchange here must be executed by all 32 lanes: never inside a short-circuit && / || or a ?: arm.
// -------------------------------------------------------------------------------------------------------------------
constexpr int kGroupRounds = 8;      // a warp claims 4 * kGroupRounds records per atomic
constexpr int kGroupTasks = 64;      // candidate (cell, triangle) tasks per box: 8 corners x 4 cells x 2

__global__ void __launch_bounds__(kMaxTileWarps * 32, 3)
reach_groups_kernel(const Checker c, const __grid_constant__ CUtensorMap map1, const TileCfg tc, const Work w,
                    const BoxRec* __restrict__ recs, const uint32_t* __restrict__ rec_count, uint32_t* __restrict__ work_counter) {
  extern __shared__ __align__(128) unsigned char tile_smem[];
  __shared__ uint64_t bars[kMaxTileWarps][2];
  __shared__ uint16_t tasks_all[kMaxTileWarps][4][kGroupTasks];
  __shared__ __align__(16) float ctx_all[kMaxTileWarps][4][16];   // per box of the round: R1[9], P[3], minB, x0, z0 (task stage)
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, g = lane >> 3, gl = lane & 7;
  const Field& f = c.f[1];
  unsigned char* slots = warp_tile_slots(tile_smem, tc, 8, bars[wid]);   // [slot 0/1][group 0..3]
  uint16_t* tasks = tasks_all[wid][g];
  uint32_t phase = 0u;                     // bit s: parity of tile slot s's barrier (a bit mask, not an indexed array)
  const uint32_t total = *rec_count;
  const unsigned gshift = (unsigned)g * 8u;
  // lanes 0, 8, 16, 24 read the zone origins of the four records of a round, lane 0 starts their copies
  auto prefetch = [&](uint32_t first, int slot) {
    const uint32_t ri = first + (uint32_t)g;
    int x0 = 0, z0 = 0;
    const bool act = ri < total;
    if (act && gl == 0) { x0 = rec_x0(recs + ri); z0 = rec_z0(recs + ri); }
    const int nact = (int)min(4u, total - first);
    if (lane == 0) mbar_expect_tx(&bars[wid][slot], (uint32_t)nact * tc.bytes);
#pragma unroll 1
    for (int q = 0; q < nact; ++q) {
      const int sx = __shfl_sync(kFull, x0, q * 8), sz = __shfl_sync(kFull, z0, q * 8);
      if (lane == 0) tma_tile_2d(slots + (size_t)(slot * 4 + q) * tc.stride, &map1, &bars[wid][slot], (sx & ~3) - tc.x_off, sz);
    }
  };
  // guided, software-pipelined claims (1 .. kGroupRounds rounds of four records), see box_tiles_warp_kernel
  const uint32_t nwarps8 = 8u * gridDim.x * (blockDim.x >> 5);
  uint32_t next_r0 = 0, next_n = 0;     // lane 0's
  auto claim = [&]() {
    if (lane == 0) {
      const uint32_t cur = *(volatile const uint32_t*)work_counter;
      next_n = 4u * (cur < total ? min(max((total - cur) / nwarps8, 1u), (uint32_t)kGroupRounds) : 1u);
      next_r0 = atomicAdd(work_counter, next_n);
    }
  };
  claim();
  for (;;) {
    const uint32_t r0 = __shfl_sync(kFull, next_r0, 0), nclaim = __shfl_sync(kFull, next_n, 0);
    if (r0 >= total) break;
    claim();
    const int nrounds = (int)((min(r0 + nclaim, total) - r0 + 3u) / 4u);
    __syncwarp();                          // every lane is done with both slots
    prefetch(r0, 0);
#pragma unroll 1
    for (int round = 0; round < nrounds; ++round) {
      const int slot = round & 1;
      const uint32_t ri = r0 + 4u * (uint32_t)round + (uint32_t)g;
      const bool act = ri < total;
      BoxRec r = {};
      if (act) r = load_rec(recs + ri);
      if (round + 1 < nrounds) { __syncwarp(); prefetch(r0 + 4u * (uint32_t)(round + 1), slot ^ 1); }
      int alive = 0;
      if (act && gl == 0) alive = (*(volatile const uint8_t*)(w.valid + r.item) != 0);
      alive = __shfl_sync(kFull, alive, 0, 8);
      mbar_wait(&bars[wid][slot], (phase >> slot) & 1u);
      phase ^= 1u << slot;
      __syncwarp();                        // lanes leave the barrier poll at different times
      bool gdone = !(act && alive);        // group-uniform
      BoxCtx b;
      rec_to_ctx(c, r, b);                 // an all-zero record for idle groups: every field defined
      if (gdone) { b.x0 = b.z0 = 0; b.x1 = b.z1 = 1; }
      if (gl == 0) {          // the box as the pooled task stage reads it (any lane may test any group's task)
        float* cx = ctx_all[wid][g];
#pragma unroll
        for (int i = 0; i < 9; ++i) cx[i] = b.R1[i];
        cx[9] = b.P[0]; cx[10] = b.P[1]; cx[11] = b.P[2]; cx[12] = b.minB;
        cx[13] = __int_as_float(b.x0); cx[14] = __int_as_float(b.z0);
      }
      const float* tile = reinterpret_cast<const float*>(slots + (size_t)(slot * 4 + g) * tc.stride) + (b.x0 & 3);
      const float top = b.maxB + (1e-4f + 4e-6f * fabsf(b.maxB));
      bool ghit = false;
      const bool allFinite = (r.flags & REC_ALLFINITE) != 0;   // group-uniform
      // vertex stage, lane = vertex. Only the vertices inside the box's own xz extent are scanned: a point inside the box
      // has |x - P.x| <= xr = sum_j |R1[0][j]| side_j / 2 (and likewise in z), while the zone is that extent padded to whole
      // cells on every side (heightfield.cpp:1880-1892) -- its outer ring, 81 -> ~49 vertices for a reach box, cannot hold
      // one (margin 1e-4 m, far above the rounding of the fp32 inside test). In a zone with -inf heights a vertex inside the
      // box counts only if the collider tests it (vertex_in_kept_triangle): checked for the rare hit, not for every vertex.
      {
        const float xr = box_half_extent(b.R1, b.side, 0) + 1e-4f, zr = box_half_extent(b.R1, b.side, 2) + 1e-4f;
        const int vx0 = max(b.x0, (int)ceilf((b.P[0] - xr) * f.iW)), vx1 = min(b.x1, (int)floorf((b.P[0] + xr) * f.iW));
        const int vz0 = max(b.z0, (int)ceilf((b.P[2] - zr) * f.iD)), vz1 = min(b.z1, (int)floorf((b.P[2] + zr) * f.iD));
        const int nXi = max(vx1 - vx0 + 1, 0), nZi = max(vz1 - vz0 + 1, 0), nVi = nXi * nZi;
        const float* tin = tile + (vz0 - b.z0) * tc.tw + (vx0 - b.x0);
        int maxNV = gdone ? 0 : nVi;
        maxNV = __reduce_max_sync(kFull, maxNV);
        const uint32_t magicX = magic_for(nXi);
#pragma unroll 1
        for (int t0 = 0; t0 < maxNV; t0 += 8) {
          const int t = t0 + gl;
          bool hit = false;
          if (!gdone && t < nVi) {
            const int zi = (nXi > 1) ? (int)__umulhi((uint32_t)t, magicX) : t, xi = t - zi * nXi;
            const float h = tin[zi * tc.tw + xi];
            hit = h > b.minB && h < top && vertex_inside(b, (vx0 + xi) * f.sW, h, (vz0 + zi) * f.sD);
            if (hit && !allFinite)
              hit = vertex_in_kept_triangle<true>(ZoneView{tile, tc.tw}, b.x1 - b.x0 + 1, b.z1 - b.z0 + 1, vx0 - b.x0 + xi,
                                                  vz0 - b.z0 + zi, b.minB);
          }
          if ((__ballot_sync(kFull, hit) >> gshift) & 0xffu) { ghit = true; gdone = true; }
          if (__all_sync(kFull, gdone)) break;
        }
      }
      __syncwarp();
      // plane stage: collect the candidate (cell, triangle) tasks, lane = corner
      int nt = 0;
      {
        float pc[3];
        box_corner(b, gl, pc);
        const float gx = pc[0] * f.iW, gz = pc[2] * f.iD;
        const int cxl = (int)floorf(gx - c.cell_margin), cxh = (int)floorf(gx + c.cell_margin);
        const int czl = (int)floorf(gz - c.cell_margin), czh = (int)floorf(gz + c.cell_margin);
        // an upright box projects its top corners into the cells of the bottom corners: the same cells twice
        // (four unconditional exchanges: inside a short-circuit && the later ones would run in only some of the lanes)
        const int oxl = __shfl_xor_sync(kFull, cxl, 4), oxh = __shfl_xor_sync(kFull, cxh, 4);
        const int ozl = __shfl_xor_sync(kFull, czl, 4), ozh = __shfl_xor_sync(kFull, czh, 4);
        const bool same = (oxl == cxl) & (oxh == cxh) & (ozl == czl) & (ozh == czh);
        // the (up to four) cells of this corner that lie inside the zone: sub-cell s uses cxh for s & 1, czh for s & 2
        const bool mine = !gdone && !((gl & 4) && same);
        bool ok[4];
#pragma unroll
        for (int sub = 0; sub < 4; ++sub) {
          const int ccx = (sub & 1) ? cxh : cxl, ccz = (sub & 2) ? czh : czl;
          ok[sub] = mine && !((sub & 1) && cxh == cxl) && !((sub & 2) && czh == czl) && ccx >= b.x0 && ccx < b.x1 && ccz >= b.z0 &&
                    ccz < b.z1;
        }
        // task slots by ballots (order within the list is irrelevant): sub-cell s of lane gl sits behind all sub-cells < s
        // of the group and behind sub-cell s of the lower lanes
        int base = 0;
#pragma unroll
        for (int sub = 0; sub < 4; ++sub) {
          const unsigned gm = (__ballot_sync(kFull, ok[sub]) >> gshift) & 0xffu;
          if (ok[sub]) {
            const int slot_i = base + __popc(gm & ((1u << gl) - 1u));
            const int ccx = (sub & 1) ? cxh : cxl, ccz = (sub & 2) ? czh : czl;
            const int code = (((ccx - b.x0) << 8) | (ccz - b.z0)) << 1;
            tasks[2 * slot_i] = (uint16_t)code; tasks[2 * slot_i + 1] = (uint16_t)(code | 1);
          }
          base += __popc(gm);
        }
        nt = 2 * base;      // <= 64
      }
      __syncwarp();
      // ... and test them, lane = task, the four lists pooled: a round's ~40 tasks fill the warp once or twice, where four
      // separate 8-lane loops ran as long as the longest list (measured: 12 of 32 lanes). The task's box comes from ctx_all.
      {
        const int n0 = __shfl_sync(kFull, nt, 0), n1 = __shfl_sync(kFull, nt, 8), n2 = __shfl_sync(kFull, nt, 16), n3 = __shfl_sync(kFull, nt, 24);
        const int o1 = n0, o2 = n0 + n1, o3 = o2 + n2, NT = o3 + n3;
        unsigned hit_groups = 0u;
#pragma unroll 1
        for (int j0 = 0; j0 < NT; j0 += 32) {
          const int j = j0 + lane;
          if (j < NT) {
            const int gi = (j >= o1) + (j >= o2) + (j >= o3);
            const int q = j - (gi == 0 ? 0 : gi == 1 ? o1 : gi == 2 ? o2 : o3);
            const int tk = tasks_all[wid][gi][q];
            const float4* cx = reinterpret_cast<const float4*>(ctx_all[wid][gi]);
            const float4 c0 = cx[0], c1 = cx[1], c2 = cx[2], c3 = cx[3];
            BoxCtx tb;
            tb.R1[0] = c0.x; tb.R1[1] = c0.y; tb.R1[2] = c0.z; tb.R1[3] = c0.w; tb.R1[4] = c1.x; tb.R1[5] = c1.y; tb.R1[6] = c1.z;
            tb.R1[7] = c1.w; tb.R1[8] = c2.x; tb.P[0] = c2.y; tb.P[1] = c2.z; tb.P[2] = c2.w; tb.minB = c3.x;
            tb.side[0] = c.side[1][0]; tb.side[1] = c.side[1][1]; tb.side[2] = c.side[1][2];
            const int tx0 = __float_as_int(c3.y), tz0 = __float_as_int(c3.z);
            const bool isUp = (tk & 1) == 0;
            const int lx = tk >> 9, lz = (tk >> 1) & 0xff, ccx = tx0 + lx, ccz = tz0 + lz;
            const float* p = reinterpret_cast<const float*>(slots + (size_t)(slot * 4 + gi) * tc.stride) + (tx0 & 3) + lz * tc.tw + lx;
            const float hA = p[0], hB = p[1], hC = p[tc.tw], hD = p[tc.tw + 1];
            if (tri_kept(isUp, hA, hB, hC, hD, tb.minB)) {
              float pl[4], cxs[4], czs[4];
              cell_plane(f, isUp, ccx, ccz, hA, hB, hC, hD, pl);
              const int nc = box_plane(tb, pl, 4, cxs, czs);
              const int tcx = isUp ? ccx : ccx + 1, tcz = isUp ? ccz : ccz + 1;
              bool hit = false;
              // unrolled over box_plane's four contacts, the count as a predicate: with constant indices the contacts stay in
              // registers (a loop over nc put them, and this stage's loads and stores, in local memory)
#pragma unroll
              for (int i = 0; i < 4; ++i) hit = hit || (i < nc && on_tri(f, isUp, tcx, tcz, cxs[i], czs[i]));
              if (hit) hit_groups |= 1u << gi;
            }
          }
        }
        __syncwarp();
        hit_groups = __reduce_or_sync(kFull, hit_groups);
        if ((hit_groups >> g) & 1u) ghit = true;
      }
      if (gl == 0 && act && alive && box_fails(true, ghit ? R_HIT : R_FREE)) w.valid[r.item] = 0;
      __syncwarp();
    }
  }
}

}  // namespace artp
