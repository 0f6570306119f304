// art_planner_b200/csrc/artp_kernels.cuh
// Pose-validity kernels (StateValidityChecker::isValid, validity_checker.cpp:39-45, on top of the ODE
// box-vs-heightfield decision, heightfield.cpp:973-1964) for sm_90a, as a three-stage pipeline:
//
//   A  classify_items_kernel     one THREAD per work item (pose / interpolated edge state): quaternion -> R,
//      dxOrthogonalizeR, the five box centres / map-inside tests / AABBs / zones, the zone min/max/all-finite from
//      exact range tables (no zone scan), and the collider's four early-outs. Items decided here (the majority)
//      never touch the heightfield; every box that needs the vertex / plane tests becomes a BoxRec in a queue.
//   B  box_tiles_warp_kernel (artp_tiles.cuh)   one WARP per queued box, the box's zone staged in shared memory by TMA:
//      vertex-in-box and plane tests by warp ballots. The reference's O(T^2) plane grouping is replaced by an
//      exact shortcut: only triangles under one of the 8 box corners can own a plane-contact point, so only those
//      "candidate" planes are built; a bloom filter on the (approximate) normal finds any earlier triangle that
//      could epsilon-merge with a live candidate. None => every candidate is its own group base (exact);
//      otherwise the box is deferred to C.
//   C  box_items_block_kernel    one CTA per deferred box: the full decision including the reference's greedy,
//      order-dependent epsilon grouping, with all planes staged in shared memory.
// The pose result is a pure AND over its boxes (torso free, every reach box touching), so B and C only ever
// clear the provisional 1 that A wrote. All three are bit-exact against oracle/ (tests/test_pose_gpu.py).
// Each stage also has an explain form (kWhy, WhyWork): every box of every item is decided and records its own bit.
#pragma once

#include <type_traits>

#include "artp_device.cuh"

namespace artp {

constexpr int kWarpsPerCta = 8;
constexpr int kMaxCand = 32;          // live candidates kept per box (more -> the box goes to the grouping stage)
constexpr int kBloomWords = 128;      // 4096-bit filter per warp
constexpr unsigned kFull = 0xffffffffu;

enum { R_FREE = 0, R_HIT = 1, R_DEFER = 2 };

// Whether a box's decided result r fails its item (validity_checker.cpp:39-45): the torso must be free, every reach box
// must touch. Any other r (undecided, deferred) fails nothing yet.
__device__ __forceinline__ bool box_fails(bool foot, int r) { return foot ? r == R_FREE : r == R_HIT; }

struct WarpScratch {
  float cpl[kMaxCand][4];   // candidate planes (exact)
  int cidx[kMaxCand];       // emission index of a LIVE candidate, -1 otherwise
  uint32_t bloom[kBloomWords];    // level 1: approximate (n0, n2)
  uint32_t bloom2[kBloomWords];   // level 2: exact (n0, n2, d)
  uint32_t cand_bits[kBloomWords];   // bit i: triangle i of the zone is a live candidate
};

// Work description shared by K1/K2. EDGE mode: item w -> edge e = w / (steps+1), j = w % (steps+1);
// j == 0 checks s2, j >= 1 checks interp(s1, s2, j/(steps+1)) (OMPL SE3 interpolation, SURVEY 8a-a14).
struct Work {
  const double* s1 = nullptr;    // EDGE: start states; POSE: unused
  const double* s2 = nullptr;    // EDGE: end states;   POSE: the states
  const float* s2f = nullptr;    // POSE only: states already cast to float (exactly what Pose3FromSE3 does first); else null
  uint8_t* valid = nullptr;      // per pose / per edge
  uint32_t item_base = 0;        // first work item of this launch (chunked calls)
  uint32_t n_items = 0;          // one past the last work item of this launch
  int steps = 0;                 // EDGE: interior steps; POSE: 0
  int edge_mode = 0;
  // INTERIOR mode (edge_mode == 0, item_off != null): item i is interior state j = i - item_off[e] + 1 of edge e at
  // t = j * (1.0 / (n_e + 1)), n_e = item_off[e+1] - item_off[e]  (prm_motion_cost.cpp:345-353); valid[] is per item.
  const uint32_t* item_off = nullptr;   // n_edges + 1 exclusive prefix sums of the per-edge interior-state counts
  uint32_t n_edges = 0;
  // SEGMENT mode (item_off != null, quotient = 1): OMPL DiscreteMotionValidator over nd_e = item_off[e+1] - item_off[e]
  // segments: item k of edge e is interpolate(s1, s2, (k + 1) / nd_e) for k < nd_e - 1 and s2 itself for k = nd_e - 1.
  int quotient = 0;
};

// The explain form of the pose pipeline (artp_box_verdicts, POSE mode only): instead of one verdict byte per item, why[i]
// receives the item's ARTP_BOX_* word -- bit k when box k fails, bit 8 + k when box k's centre is off the map -- with
// every box decided (no item leaves the pipeline at its first failing box). valid is not used.
struct WhyWork : Work {
  uint16_t* why = nullptr;
};
template <bool kWhy>
using WorkOf = std::conditional_t<kWhy, WhyWork, Work>;

// Sets bit k of a why word. The boxes of one item are decided by different threads, possibly in kernels that run side
// by side: a 16-bit compare-and-swap loop (one per failing box), so no store reaches past the caller's buffer.
__device__ __forceinline__ void why_set(uint16_t* why, uint32_t slot, int k) {
  unsigned short* p = reinterpret_cast<unsigned short*>(why + slot);
  unsigned short old = *(volatile unsigned short*)p, seen;
  do {
    seen = old;
    old = atomicCAS(p, seen, (unsigned short)(seen | (1u << k)));
  } while (old != seen);
}

__device__ __forceinline__ uint32_t bloom_hash(int kx, int kz) {
  return (((uint32_t)kx * 0x9E3779B1u) ^ ((uint32_t)kz * 0x85EBCA77u)) >> 20;   // 12 bits
}
// ceil(2^32 / n) for the flattened-index division t / n = umulhi(t, magic) (exact while t * n < 2^32).
struct MagicTab {
  uint32_t v[129];
  constexpr MagicTab() : v() {
    for (int i = 2; i < 129; ++i) v[i] = 0xFFFFFFFFu / (uint32_t)i + 1u;
  }
};
__constant__ MagicTab kMagicTab = MagicTab();
__device__ __forceinline__ uint32_t magic_for(int n) {
  return n <= 1 ? 0u : (n <= 128 ? kMagicTab.v[n] : 0xFFFFFFFFu / (uint32_t)n + 1u);
}

// EDGE-mode state j of the edge (s1, s2) with `steps` interior steps: s2 itself for j == 0, else
// interpolate(s1, s2, j / (steps + 1)).
__device__ __forceinline__ void edge_state(const double* s1, const double* s2, uint32_t j, int steps, double s[7]) {
  double b[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) b[k] = s2[k];
  if (j == 0) {
#pragma unroll
    for (int k = 0; k < 7; ++k) s[k] = b[k];
  } else {
    double a[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) a[k] = s1[k];
    se3_interpolate(a, b, (double)j / (double)((uint32_t)steps + 1u), s);
  }
}

__device__ __forceinline__ void load_item_state(const Work& w, uint32_t item, double s[7]) {
  if (w.item_off) {
    const uint32_t lo = edge_of_item<true>(w.item_off, w.n_edges, item);
    const uint32_t o0 = __ldg(w.item_off + lo), o1 = __ldg(w.item_off + lo + 1);
    const int n_e = (int)(o1 - o0), step = (int)(item - o0) + 1;
    double a[7], b[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) { a[k] = w.s1[(size_t)lo * 7 + k]; b[k] = w.s2[(size_t)lo * 7 + k]; }
    if (w.quotient) segment_state(a, b, step, n_e, s);
    else interior_state(a, b, step, n_e, s);
    return;
  }
  if (!w.edge_mode) {
    // Each state is read once: streaming loads (evict first in L1 and L2), so the pose stream does not push the range
    // tables that classify reads at random out of L2. (Edge mode keeps the default: every step of an edge reads its
    // endpoints again.)
    if (w.s2f) {
#pragma unroll
      for (int k = 0; k < 7; ++k) s[k] = (double)__ldcs(w.s2f + (size_t)item * 7 + k);   // exact; cast back to float downstream
    } else {
#pragma unroll
      for (int k = 0; k < 7; ++k) s[k] = __ldcs(w.s2 + (size_t)item * 7 + k);
    }
    return;
  }
  const uint32_t per = (uint32_t)w.steps + 1u;
  const uint32_t e = item / per, j = item - e * per;
  edge_state(w.s1 + (size_t)e * 7, w.s2 + (size_t)e * 7, j, w.steps, s);
}

__device__ __forceinline__ uint32_t item_slot(const Work& w, uint32_t item) {
  return w.edge_mode ? item / ((uint32_t)w.steps + 1u) : item;
}

// The collider's rules for one cell (heightfield.cpp:1306-1441) against a box bottom minB: a vertex collides when it is
// finite and above minB; the Up (A, B, C) / Down (D, B, C) triangle is kept when its vertices are finite and one of them
// collides; vertex v (0 A, 1 B, 2 C, 3 D) is tested when it collides and belongs to a kept triangle.
// tri_kept is the triangle rule: with no NaN (heights are finite or -inf), "all three finite and one above minB" is
// "lowest > -inf, highest < +inf and highest > minB".
__device__ __forceinline__ bool tri_kept(bool isUp, float hA, float hB, float hC, float hD, float minB) {
  const float h0 = isUp ? hA : hD;
  const float lo = fminf(h0, fminf(hB, hC)), hi = fmaxf(h0, fmaxf(hB, hC));
  return lo > -CUDART_INF_F && hi < CUDART_INF_F && hi > minB;
}
struct CellKeep {
  bool up, dn, cA, cB, cC, cD;
  __device__ __forceinline__ bool tested(int v) const {
    return v == 0 ? (up && cA) : v == 1 ? ((up || dn) && cB) : v == 2 ? ((up || dn) && cC) : (dn && cD);
  }
};
__device__ __forceinline__ CellKeep cell_keep(float hA, float hB, float hC, float hD, float minB) {
  CellKeep k;
  k.cA = finitef(hA) && hA > minB; k.cB = finitef(hB) && hB > minB;
  k.cC = finitef(hC) && hC > minB; k.cD = finitef(hD) && hD > minB;
  k.up = tri_kept(true, hA, hB, hC, hD, minB);
  k.dn = tri_kept(false, hA, hB, hC, hD, minB);
  return k;
}

// -------------------------------------------------------------------------------------------------
// K1: warp-level box-vs-heightfield decision. Returns R_FREE / R_HIT / R_DEFER (warp-uniform).
// -------------------------------------------------------------------------------------------------

// Early outs of dCollideHeightfieldZone (heightfield.cpp:1027-1064, 1139-1160) given the zone reductions.
// Returns R_FREE / R_HIT, or -1 if the vertex / plane stages are needed.
__device__ __forceinline__ int zone_early_out(const BoxCtx& b, float maxY, float minY, bool allFinite) {
  if (b.minB - maxY > -ARTP_EPS) return R_FREE;                                            // above
  if (minY - b.maxB > -ARTP_EPS) return R_FREE;                                            // under (art_planner mod)
  if (allFinite && minY - b.minB > -ARTP_EPS && b.maxB - maxY > -ARTP_EPS) return R_HIT;   // spans
  if (allFinite && maxY - minY < ARTP_EPS) {                                               // single plane
    const float pl[4] = {0.0f, 1.0f, 0.0f, minY};
    float cx[4], cz[4];
    return box_plane(b, pl, 1, cx, cz) > 0 ? R_HIT : R_FREE;
  }
  if (b.x1 - b.x0 < 1 || b.z1 - b.z0 < 1) return R_FREE;                                   // no cell, no triangle
  return -1;
}

// zone_early_out on the compact tables' intervals: maxY in [dec(cM - 1), dec(cM)], minY in [dec(cm), dec(cm + 1)].
// Every subtraction and comparison of the tests is monotone in maxY and minY, so each test is evaluated at the interval
// ends as true, false or unknown, in zone_early_out's order. Returns its answer when the first test that is not false is
// true (or all are false), kZoneUnknown when an unknown comes first -- always for the single-plane test, which needs
// the exact minY -- and for zones without a finite height (reserved codes).
constexpr int kZoneUnknown = -4;
__device__ __forceinline__ int zone_early_out_codes(const Field& f, const BoxCtx& b, uint32_t cM, uint32_t cm,
                                                    bool allFinite) {
  if (cM == 0 || cM == kCodeNone || cm == kCodeNone) return kZoneUnknown;
  const float mxLo = code_dec(f.cbase, f.cstep, cM - 1), mxHi = code_dec(f.cbase, f.cstep, cM);
  const float mnLo = code_dec(f.cbase, f.cstep, cm), mnHi = code_dec(f.cbase, f.cstep, cm + 1);
  if (b.minB - mxHi > -ARTP_EPS) return R_FREE;                                            // above
  if (!(b.minB - mxLo > -ARTP_EPS)) {
    if (mnLo - b.maxB > -ARTP_EPS) return R_FREE;                                          // under
    if (!(mnHi - b.maxB > -ARTP_EPS)) {
      if (allFinite) {
        if (mnLo - b.minB > -ARTP_EPS && b.maxB - mxHi > -ARTP_EPS) return R_HIT;           // spans
        if (!(mnHi - b.minB > -ARTP_EPS && b.maxB - mxLo > -ARTP_EPS) && !(mxLo - mnHi < ARTP_EPS)) {   // single plane
          if (b.x1 - b.x0 < 1 || b.z1 - b.z0 < 1) return R_FREE;
          return -1;
        }
      } else {
        if (b.x1 - b.x0 < 1 || b.z1 - b.z0 < 1) return R_FREE;
        return -1;
      }
    }
  }
  return kZoneUnknown;
}

// The zone as the warp stage reads it: element (xi, zi) -- vertex (x0 + xi, z0 + zi) -- at p[zi * stride + xi]; either the
// heightfield itself (p = H + z0 * pitch + x0, stride = pitch) or a shared-memory tile the zone was copied into by TMA.
struct ZoneView { const float* p; int stride; };
template <bool SMEM>
__device__ __forceinline__ float zload(const ZoneView& v, int xi, int zi) {
  const float* q = v.p + zi * v.stride + xi;
  return SMEM ? *q : __ldg(q);
}
template <bool SMEM>
__device__ __forceinline__ void zcell(const ZoneView& v, int lx, int lz, float& hA, float& hB, float& hC, float& hD) {
  const float* q = v.p + lz * v.stride + lx;
  if (SMEM) { hA = q[0]; hB = q[1]; hC = q[v.stride]; hD = q[v.stride + 1]; }
  else { hA = __ldg(q); hB = __ldg(q + 1); hC = __ldg(q + v.stride); hD = __ldg(q + v.stride + 1); }
}

// cell_keep's vertex rule, per vertex: a colliding vertex (xi, zi) of an nX x nZ zone is tested when one of the up to six triangles
// around it is kept (tri_kept: with the vertex above minB, when its three vertices are finite). Cell c of the four around
// it holds the vertex as its D (c = 0, Down only), C (1), B (2) or A (3, Up only).
template <bool SMEM>
__device__ __forceinline__ bool vertex_in_kept_triangle(const ZoneView& zv, int nX, int nZ, int xi, int zi, float minB) {
  bool kept = false;
#pragma unroll 1
  for (int c = 0; c < 4 && !kept; ++c) {
    const int cxi = xi - 1 + (c & 1), czi = zi - 1 + (c >> 1);
    if (cxi < 0 || czi < 0 || cxi >= nX - 1 || czi >= nZ - 1) continue;
    float hA, hB, hC, hD;
    zcell<SMEM>(zv, cxi, czi, hA, hB, hC, hD);
    kept = (c != 0 && tri_kept(true, hA, hB, hC, hD, minB)) || (c != 3 && tri_kept(false, hA, hB, hC, hD, minB));
  }
  return kept;
}

// Bloom keys of the merge screen. Level 1 (cheap, every kept triangle): buckets of the APPROXIMATE normal (n0, n2);
// level 2 (flagged triangles only): buckets of the EXACT plane (n0, n2, d).
__device__ __forceinline__ uint32_t bloom_hash3(int kx, int kz, int kd) {
  return ((((uint32_t)kx * 0x9E3779B1u) ^ ((uint32_t)kz * 0x85EBCA77u)) + (uint32_t)kd * 0xC2B2AE3Du) >> 20;   // 12 bits
}

// Warp-level decision for one box; the zone is read through `zv`. Returns R_FREE / R_HIT / R_DEFER (warp-uniform).
//   (3) vertex stage: lane = vertex. Big all-finite zones (the torso's ~40 x 40 vertices) are walked window by window:
//       the level-3 range table holds the maximum of every 8 x 8 vertex window, and a window whose maximum does not
//       exceed the box bottom holds neither a colliding vertex nor a kept triangle, so it is skipped in the vertex
//       stage AND in the merge screen -- on rough terrain most torso boxes hover over all but a few peaks.
//   (4) plane stage: a plane contact point is always a box corner (up to a few ulps), so only the triangles in the
//       cells under the 8 corners (+- cell_margin) can report one: <= 64 candidates, lane = candidate.
//   (5) merge screen: does an EARLIER kept triangle epsilon-match a live candidate (greedy grouping,
//       heightfield.cpp:1511-1556)? Two bloom levels: the approximate normal of every kept triangle against the
//       candidates' (n0, n2) buckets; a flagged lane builds its exact plane and tests the (n0, n2, d) buckets -- matching
//       planes need |d_m - d_c| < eps, which on non-degenerate terrain never happens, so the exact compare against the
//       candidate list (shared memory) is reached only on flat / terraced ground. Live candidates themselves are
//       skipped by the screen (a bitmap over the triangle indices); candidate-vs-candidate matches are caught when the
//       level-2 keys are inserted. Any match => R_DEFER (exact stage C).
// Code size matters here (round 2: a 5 400-instruction version stalled on instruction fetch, `no_instruction` 9 of 16
// cycles per issue): one region loop serves both the windowed and the flat case, nothing is unrolled.
template <bool SMEM>
__device__ int box_collide_warp(const Field& f, const BoxCtx& b, const ZoneView& zv, WarpScratch& ws, int lane,
                                float cell_margin, bool needs_reduce, bool all_finite_known, bool merge_free) {
  const int nX = b.x1 - b.x0 + 1, nZ = b.z1 - b.z0 + 1;
  const int nV = nX * nZ;

  // (1)+(2) zone reductions and early outs -- normally already done by stage A
  bool allFinite = all_finite_known;
  if (needs_reduce) {
    const uint32_t magicX = magic_for(nX);
    float mx = -CUDART_INF_F, mn = CUDART_INF_F;
    bool fin = true;
#pragma unroll 1
    for (int t = lane; t < nV; t += 32) {
      const int zi = (nX > 1) ? (int)__umulhi((uint32_t)t, magicX) : t;
      const float h = zload<SMEM>(zv, t - zi * nX, zi);
      mx = fmaxf(mx, h);
      if (finitef(h)) mn = fminf(mn, h); else fin = false;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mx = fmaxf(mx, __shfl_xor_sync(kFull, mx, o));
      mn = fminf(mn, __shfl_xor_sync(kFull, mn, o));
    }
    allFinite = __all_sync(kFull, fin);
    const int e = zone_early_out(b, mx, mn, allFinite);
    if (e >= 0) return e;
  }

  const int nCZ = nZ - 1;
  // A vertex strictly inside the box lies within the box's vertical extent: h >= maxB + slack cannot be inside
  // (slack = 1e-4 + 4e-6 |maxB|: > 10x the rounding of the rotated coordinates and of maxB itself).
  const float top = b.maxB + (1e-4f + 4e-6f * fabsf(b.maxB));

  // Regions: the active 8 x 8-vertex windows of a big all-finite zone (bit w of `act`), else the whole zone.
  const int nWx = (nX + 5) / 7, nWz = (nZ + 5) / 7;       // windows advance by 7 cells
  const bool windowed = allFinite && nV > 256 && f.kmax >= 3 && nX >= 8 && nZ >= 8 && nWx * nWz <= 64;
  // ... and, for the vertex stage only, `actv`: the windows that can hold a vertex INSIDE the box. A window is the
  // axis-aligned block [xs, xs+7] x [min h, max h] x [zs, zs+7] (level-3 table: max and min of its 64 heights); if
  // that block lies entirely beyond one of the box's six faces -- its extent along the face normal, evaluated at the
  // block's corners, stays outside +-side/2 by more than 2 mm (>> the rounding of vertex_inside's fp32 arithmetic at
  // map coordinates of a few hundred metres) -- no vertex of it passes dGeomBoxPointDepth. For a tilted torso over rough
  // ground this is far tighter than "window max > box bottom": the AABB bottom lies below most of the zone, the
  // box's own bottom face does not. Kept triangles are a different question (h > minB): the plane stage keeps `act`.
  unsigned long long act = 1ull, actv = 1ull;
  if (windowed) {
    const float2* __restrict__ T3 = f.T[3];
    act = 0ull; actv = 0ull;
    const uint32_t magicWx = magic_for(nWx);
    // per face axis j: centre offset and the block's half extents along it (the x / z half extents are the same for
    // every window: 3.5 cells), in centre / radius form
    const float hx = 3.5f * f.sW, hz = 3.5f * f.sD;
    const float rxz0 = fabsf(b.R1[0]) * hx + fabsf(b.R1[6]) * hz, rxz1 = fabsf(b.R1[1]) * hx + fabsf(b.R1[7]) * hz,
                rxz2 = fabsf(b.R1[2]) * hx + fabsf(b.R1[8]) * hz;
    const float lim0 = 0.5f * b.side[0] + 2e-3f, lim1 = 0.5f * b.side[1] + 2e-3f, lim2 = 0.5f * b.side[2] + 2e-3f;
#pragma unroll 1
    for (int w0 = 0; w0 < nWx * nWz; w0 += 32) {
      const int wi = w0 + lane;
      bool a = false, av = false;
      if (wi < nWx * nWz) {
        const int wz = (nWx > 1) ? (int)__umulhi((uint32_t)wi, magicWx) : wi, wx = wi - wz * nWx;
        const int xs = min(b.x0 + 7 * wx, b.x1 - 7), zs = min(b.z0 + 7 * wz, b.z1 - 7);
        const float2 mm = __ldg(T3 + (size_t)zs * f.pitch + xs);
        a = mm.x > b.minB;
        if (a) {
          const float dx = ((float)xs + 3.5f) * f.sW - b.P[0], dz = ((float)zs + 3.5f) * f.sD - b.P[2];
          const float dy = 0.5f * (mm.x + mm.y) - b.P[1], hy = 0.5f * (mm.x - mm.y);
          const float c0 = b.R1[0] * dx + b.R1[3] * dy + b.R1[6] * dz, c1 = b.R1[1] * dx + b.R1[4] * dy + b.R1[7] * dz,
                      c2 = b.R1[2] * dx + b.R1[5] * dy + b.R1[8] * dz;
          const bool sep = fabsf(c0) - (rxz0 + fabsf(b.R1[3]) * hy) > lim0 || fabsf(c1) - (rxz1 + fabsf(b.R1[4]) * hy) > lim1 ||
                           fabsf(c2) - (rxz2 + fabsf(b.R1[5]) * hy) > lim2;
          av = !sep;
        }
      }
      act |= (unsigned long long)__ballot_sync(kFull, a) << w0;
      actv |= (unsigned long long)__ballot_sync(kFull, av) << w0;
    }
    if (act == 0ull) return R_FREE;   // no vertex above the box bottom: no colliding vertex, no kept triangle
  }
  // neighbouring windows share a row / column of vertices: when most of them are active one pass over the zone is cheaper
  const bool by_window = windowed && 3 * __popcll(act) <= 2 * nWx * nWz;
  const bool by_window_v = windowed && 3 * __popcll(actv) <= 2 * nWx * nWz;
  if (!by_window) act = 1ull;
  if (!by_window_v) actv = 1ull;          // (windowed && actv == 0 stays 0: the vertex stage has nothing to scan)
  // region r of the walk: origin (lx0, lz0) and extent (rw, rh) in vertices
  auto region = [&](bool by_window, int wi, int& lx0, int& lz0, int& rw, int& rh) {
    if (by_window) {
      const int wz = wi / nWx, wx = wi - wz * nWx;
      lx0 = min(7 * wx, nX - 8); lz0 = min(7 * wz, nZ - 8); rw = 8; rh = 8;
    } else { lx0 = 0; lz0 = 0; rw = nX; rh = nZ; }
  };

  // (3) vertex-in-box test of every colliding vertex of a kept triangle (heightfield.cpp:1306-1441)
  if (allFinite) {
    // every colliding vertex belongs to some kept triangle (all finite, >= 1 cell)
    if (nV > 128 && actv != 0ull) {
      // Probe pass: one vertex per lane on an 8 x 4 lattice over the box footprint (a hit anywhere in the zone is the
      // reference's answer) -- finds most intersecting torso boxes in one step.
      const float u0 = (((float)(lane & 7) + 0.5f) * 0.25f - 1.0f) * (0.5f * b.side[0]);
      const float u1 = (((float)(lane >> 3) + 0.5f) * 0.5f - 1.0f) * (0.5f * b.side[1]);
      const float qx = b.P[0] + u0 * b.R1[0] + u1 * b.R1[1], qz = b.P[2] + u0 * b.R1[6] + u1 * b.R1[7];
      const int vx = min(max(__float2int_rn(qx * f.iW), b.x0), b.x1), vz = min(max(__float2int_rn(qz * f.iD), b.z0), b.z1);
      const float h = zload<SMEM>(zv, vx - b.x0, vz - b.z0);
      const bool hit = h > b.minB && h < top && vertex_inside(b, vx * f.sW, h, vz * f.sD);
      if (__any_sync(kFull, hit)) return R_HIT;
    }
    // the whole-zone walk covers only the box's own xz extent: a point inside the box has |x - P.x| <= sum_j |R1[0][j]|
    // side_j / 2 (likewise z); the zone is that extent padded to whole cells, its outer ring cannot hold an inside vertex
    int ix0 = 0, iz0 = 0, iw = nX, ih = nZ;
    if (!by_window_v) {
      const float xr = box_half_extent(b.R1, b.side, 0) + 1e-4f, zr = box_half_extent(b.R1, b.side, 2) + 1e-4f;
      const int vx0 = max(b.x0, (int)ceilf((b.P[0] - xr) * f.iW)), vx1 = min(b.x1, (int)floorf((b.P[0] + xr) * f.iW));
      const int vz0 = max(b.z0, (int)ceilf((b.P[2] - zr) * f.iD)), vz1 = min(b.z1, (int)floorf((b.P[2] + zr) * f.iD));
      ix0 = vx0 - b.x0; iz0 = vz0 - b.z0; iw = max(vx1 - vx0 + 1, 0); ih = max(vz1 - vz0 + 1, 0);
    }
#pragma unroll 1
    for (unsigned long long m = actv; m; m &= m - 1) {
      int lx0, lz0, rw, rh;
      region(by_window_v, __ffsll((long long)m) - 1, lx0, lz0, rw, rh);
      if (!by_window_v) { lx0 = ix0; lz0 = iz0; rw = iw; rh = ih; }
      const uint32_t magicW = magic_for(rw);
      const int n = rw * rh;
#pragma unroll 1
      for (int t0 = 0; t0 < n; t0 += 32) {
        const int t = t0 + lane;
        bool hit = false;
        if (t < n) {
          const int q = (rw > 1) ? (int)__umulhi((uint32_t)t, magicW) : t;
          const int xi = lx0 + t - q * rw, zi = lz0 + q;
          const float h = zload<SMEM>(zv, xi, zi);
          hit = h > b.minB && h < top && vertex_inside(b, (b.x0 + xi) * f.sW, h, (b.z0 + zi) * f.sD);
        }
        if (__any_sync(kFull, hit)) return R_HIT;
      }
    }
  } else {
    const int nCX = nX - 1, nC = nCX * nCZ;
    const uint32_t magicC = magic_for(nCX);
#pragma unroll 1
    for (int t0 = 0; t0 < nC; t0 += 32) {
      const int t = t0 + lane;
      bool hit = false;
      if (t < nC) {
        const int czi = (nCX > 1) ? (int)__umulhi((uint32_t)t, magicC) : t;   // flattened, x fastest
        const int cxi = t - czi * nCX;
        const int cx = b.x0 + cxi, cz = b.z0 + czi;
        float hA, hB, hC, hD;
        zcell<SMEM>(zv, cxi, czi, hA, hB, hC, hD);
        const CellKeep ck = cell_keep(hA, hB, hC, hD, b.minB);
#pragma unroll 1
        for (int v = 0; v < 4 && !hit; ++v) {
          if (ck.tested(v)) hit = vertex_inside(b, (cx + (v & 1)) * f.sW, v == 0 ? hA : v == 1 ? hB : v == 2 ? hC : hD, (cz + (v >> 1)) * f.sD);
        }
      }
      if (__any_sync(kFull, hit)) return R_HIT;
    }
  }

  // (4) plane stage (heightfield.cpp:1474-1617)
  const int T = 2 * (nX - 1) * nCZ;                      // triangles of the zone
  const bool use_bits = T <= 32 * kBloomWords;           // candidate bitmap over the triangle indices
  // merge_free: the map's plane tables (artp_set_map) say that no two triangles of this zone lie in one plane (within
  // eps): every kept triangle is its own group, no screen is needed -- the normal case on natural terrain.
  __syncwarp();   // the previous box's reads of this warp's scratch are done (no WAR across boxes)
  if (!merge_free) {
#pragma unroll 1
    for (int i = lane; i < kBloomWords; i += 32) { ws.bloom[i] = 0u; ws.bloom2[i] = 0u; ws.cand_bits[i] = 0u; }
  }
  __syncwarp();
  // Task t = lane + 32 * pass: corner (t >> 1) & 7, triangle t & 1 (Up / Down of a cell on neighbouring lanes), sub-cell
  // t >> 4. A corner has a second / third / fourth candidate cell only when it lies within cell_margin of a cell
  // boundary, so pass 0 is normally 16 busy lanes and pass 1 is skipped by the whole warp.
  const int corner = (lane >> 1) & 7, u = lane & 1;
  float pc[3];
  box_corner(b, corner, pc);
  // Height of this lane's corner (the lower one of the vertical pair that may be folded into one lane below). Every
  // contact dCollideBoxPlane returns is a box corner lying BELOW the plane; if it also lies on the triangle, the plane
  // there is no higher than the triangle's highest vertex. So in a merge-free zone (each triangle is tested against its
  // own plane only) a candidate triangle whose vertices all lie more than 1 mm below the corner that selected it
  // cannot be hit through that corner -- and the lane of any other corner over the same cell tests it for itself.
  // A torso hovering over rough ground keeps nearly all candidates by the h > minB rule (its AABB bottom is low) and
  // drops nearly all of them by this one.
  const float py_pair = fminf(pc[1], __shfl_xor_sync(kFull, pc[1], 8));
  const float gx = pc[0] * f.iW, gz = pc[2] * f.iD;
  const int cxl = (int)floorf(gx - cell_margin), cxh = (int)floorf(gx + cell_margin);
  const int czl = (int)floorf(gz - cell_margin), czh = (int)floorf(gz + cell_margin);
  bool hit_own = false, pair_possible = false;
  int nLive = 0, max_live = -1;
#pragma unroll 1
  for (int pass = 0; pass < 2; ++pass) {
    const int sub = 2 * pass + (lane >> 4);
    const int ccx = (sub & 1) ? cxh : cxl, ccz = (sub & 2) ? czh : czl;
    bool actc = !((sub & 1) && cxh == cxl) && !((sub & 2) && czh == czl);
    actc = actc && ccx >= b.x0 && ccx < b.x1 && ccz >= b.z0 && ccz < b.z1;
    if (!__any_sync(kFull, actc)) continue;
    // an upright box projects its top corners into the cells of the bottom corners: the same triangle twice
    {
      const int pcx = __shfl_xor_sync(kFull, ccx, 8), pcz = __shfl_xor_sync(kFull, ccz, 8);
      const bool pact = __shfl_xor_sync(kFull, actc, 8);
      if ((corner & 4) && pact && pcx == ccx && pcz == ccz) actc = false;
    }
    bool live = false;
    float pl[4] = {0.f, 0.f, 0.f, 0.f};
    int idx = -1;
    if (actc) {
      float hA, hB, hC, hD;
      zcell<SMEM>(zv, ccx - b.x0, ccz - b.z0, hA, hB, hC, hD);
      const bool isUp = (u == 0);
      bool keep = tri_kept(isUp, hA, hB, hC, hD, b.minB);
      if (merge_free && keep) {
        const float hT = isUp ? fmaxf(hA, fmaxf(hB, hC)) : fmaxf(hD, fmaxf(hB, hC));
        keep = hT > py_pair - 1e-3f;
      }
      if (keep) {
        cell_plane(f, isUp, ccx, ccz, hA, hB, hC, hD, pl);
        // Liveness: any plane within eps of this one changes the box-plane depth by far less than tau.
        const float Q1 = pl[0] * b.R1[0] + pl[1] * b.R1[3] + pl[2] * b.R1[6];
        const float Q2 = pl[0] * b.R1[1] + pl[1] * b.R1[4] + pl[2] * b.R1[7];
        const float Q3 = pl[0] * b.R1[2] + pl[1] * b.R1[5] + pl[2] * b.R1[8];
        const float B1 = fabsf(b.side[0] * Q1), B2 = fabsf(b.side[1] * Q2), B3 = fabsf(b.side[2] * Q3);
        const float depth = pl[3] + 0.5f * (B1 + B2 + B3) - (pl[0] * b.P[0] + pl[1] * b.P[1] + pl[2] * b.P[2]);
        const float tau = 16.0f * ARTP_EPS * (1.0f + b.side[0] + b.side[1] + b.side[2] + fabsf(b.P[0]) +
                                              fabsf(b.P[1]) + fabsf(b.P[2]) + fabsf(pl[3]));
        if (depth >= -tau) {   // else dead: no plane of its would-be group can touch the box
          live = true;
          idx = ((ccx - b.x0) * nCZ + (ccz - b.z0)) * 2 + u;   // emission order: x outer, z inner, Up, Down
          if (!merge_free) {
          if (use_bits) atomicOr(&ws.cand_bits[idx >> 5], 1u << (idx & 31));
          // level-1 keys: every bucket the approximate normal of an eps-matching triangle may fall into;
          // level-2 keys: every bucket its exact (n0, n2, d) may fall into. The candidate's own level-2 bucket goes in
          // last (after every candidate of the pass has inserted its neighbour buckets): finding it occupied means
          // another live candidate may match this one.
          const int kxc = nkey(pl[0]), kzc = nkey(pl[2]), kdc = dkey(pl[3]);
          const int kx0 = nkey(pl[0] - kKeyMargin), kx1 = nkey(pl[0] + kKeyMargin);
          const int kz0 = nkey(pl[2] - kKeyMargin), kz1 = nkey(pl[2] + kKeyMargin);
          const int kd0 = dkey(pl[3] - 2.0f * ARTP_EPS), kd1 = dkey(pl[3] + 2.0f * ARTP_EPS);
#pragma unroll 1
          for (int kx = kx0; kx <= kx1; ++kx)
#pragma unroll 1
            for (int kz = kz0; kz <= kz1; ++kz) {
              const uint32_t hsh = bloom_hash(kx, kz);
              atomicOr(&ws.bloom[hsh >> 5], 1u << (hsh & 31));
#pragma unroll 1
              for (int kd = kd0; kd <= kd1; ++kd) {
                if (kx == kxc && kz == kzc && kd == kdc) continue;
                const uint32_t h3 = bloom_hash3(kx, kz, kd);
                atomicOr(&ws.bloom2[h3 >> 5], 1u << (h3 & 31));
              }
            }
          }
          // contact points with the triangle's OWN plane (valid if it turns out to be its group base)
          float cx[4], cz[4];
          const int nc = box_plane(b, pl, 4, cx, cz);
          const int tcx = isUp ? ccx : ccx + 1, tcz = isUp ? ccz : ccz + 1;
#pragma unroll 1
          for (int i = 0; i < nc; ++i) hit_own = hit_own || on_tri(f, isUp, tcx, tcz, cx[i], cz[i]);
        }
      }
    }
    __syncwarp();
    if (live && !merge_free) {
      const uint32_t h3 = bloom_hash3(nkey(pl[0]), nkey(pl[2]), dkey(pl[3]));
      if ((atomicOr(&ws.bloom2[h3 >> 5], 1u << (h3 & 31)) >> (h3 & 31)) & 1u) pair_possible = true;
    }
    // append this pass's live candidates to the list
    const unsigned lm = __ballot_sync(kFull, live);
    if (nLive + __popc(lm) > kMaxCand) return R_DEFER;   // exact fallback (not seen in practice)
    if (live) {
      const int p = nLive + __popc(lm & ((1u << lane) - 1u));
      ws.cpl[p][0] = pl[0]; ws.cpl[p][1] = pl[1]; ws.cpl[p][2] = pl[2]; ws.cpl[p][3] = pl[3];
      ws.cidx[p] = idx;
    }
    nLive += __popc(lm);
    max_live = max(max_live, idx);
  }
  if (nLive == 0) return R_FREE;
  if (merge_free) return __any_sync(kFull, hit_own) ? R_HIT : R_FREE;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) max_live = max(max_live, __shfl_xor_sync(kFull, max_live, o));
  __syncwarp();
  if (!use_bits) pair_possible = true;
  if (__any_sync(kFull, pair_possible)) {
    // candidate against candidate, exactly: any two matching live candidates => one may absorb the other
    bool merge = false;
    if (lane < nLive) {
#pragma unroll 1
      for (int j = 0; j < nLive; ++j)
        if (ws.cidx[j] != ws.cidx[lane] && plane_match(ws.cpl[lane], ws.cpl[j])) merge = true;
    }
    if (__any_sync(kFull, merge)) return R_DEFER;
  }

  // (5) merge screen over the regions: one cell per lane
#pragma unroll 1
  for (unsigned long long m = act; m; m &= m - 1) {
    int lx0, lz0, rw, rh;
    region(by_window, __ffsll((long long)m) - 1, lx0, lz0, rw, rh);
    if ((lx0 * nCZ + lz0) * 2 >= max_live) continue;       // the whole region is emitted after the last live candidate
    const int cw = rw - 1, n = cw * (rh - 1);
    const uint32_t magicW = magic_for(cw);
#pragma unroll 1
    for (int t0 = 0; t0 < n; t0 += 32) {
      const int t = t0 + lane;
      bool merge = false;
      if (t < n) {
        const int q = (cw > 1) ? (int)__umulhi((uint32_t)t, magicW) : t;
        const int cxi = lx0 + t - q * cw, czi = lz0 + q;
        const int cell_idx = (cxi * nCZ + czi) * 2;
        if (cell_idx < max_live) {   // only triangles emitted before the last live candidate can absorb one
          const int cx = b.x0 + cxi, cz = b.z0 + czi;
          float hA, hB, hC, hD;
          zcell<SMEM>(zv, cxi, czi, hA, hB, hC, hD);
          const CellKeep ck = cell_keep(hA, hB, hC, hD, b.minB);
          if (ck.up || ck.dn) {
            const float xA = cx * f.sW, xB = (cx + 1) * f.sW, zA = cz * f.sD, zC = (cz + 1) * f.sD;
#pragma unroll 1
            for (int uu = 0; uu < 2; ++uu) {
              const int idx = cell_idx + uu;
              if (!(uu == 0 ? ck.up : ck.dn) || idx >= max_live) continue;
              if (use_bits && ((ws.cand_bits[idx >> 5] >> (idx & 31)) & 1u)) continue;   // live candidates: handled above
              // approximate normal (cross product value-identical to tri_plane's, zero terms dropped):
              // Up (A,B,C): E1 = C-A, E2 = B-A, c = E1 x E2;  Down (D,B,C): E1 = C-D, E2 = B-D, c = E2 x E1
              const float ey = uu == 0 ? hC - hA : hB - hD, ez = uu == 0 ? zC - zA : zA - zC;
              const float gx2 = uu == 0 ? xB - xA : xA - xB, gy = uu == 0 ? hB - hA : hC - hD;
              const float c0 = -(ez * gy), c1 = ez * gx2, c2 = -(ey * gx2);
              const float r = rsqrtf(c0 * c0 + c1 * c1 + c2 * c2);
              const uint32_t hsh = bloom_hash(nkey(c0 * r), nkey(c2 * r));
              if (ws.bloom[hsh >> 5] & (1u << (hsh & 31))) {
                float plm[4];   // flagged: exact plane, level-2 buckets
                cell_plane(f, uu == 0, cx, cz, hA, hB, hC, hD, plm);
                const uint32_t h3 = bloom_hash3(nkey(plm[0]), nkey(plm[2]), dkey(plm[3]));
                if (ws.bloom2[h3 >> 5] & (1u << (h3 & 31))) {
#pragma unroll 1
                  for (int sidx = 0; sidx < nLive; ++sidx)
                    if (ws.cidx[sidx] > idx && plane_match(plm, ws.cpl[sidx])) merge = true;
                }
              }
            }
          }
        }
      }
      if (__any_sync(kFull, merge)) return R_DEFER;
    }
  }
  const int res = __any_sync(kFull, hit_own) ? R_HIT : R_FREE;
  __syncwarp();   // scratch is reused by the next box
  return res;
}

// One queued box (80 bytes): everything stage B/C need, so nothing is recomputed.
struct alignas(16) BoxRec {
  float R1[9];
  float P[3];
  float minB, maxB;
  int x0, x1, z0, z1;
  uint32_t item;     // verdict slot of the work item (pose index / edge index / interior-state index)
  uint32_t flags;    // bits 0-2: box (0 torso, 1..4 feet); bit 3: zone all finite; bit 4: zone not reduced yet;
                     // bit 5: no mergeable triangle pair in the zone (plane tables, artp_set_map)
};
static_assert(sizeof(BoxRec) == 80, "BoxRec is read as five 16-byte words");
enum { REC_ALLFINITE = 8, REC_NEEDS_REDUCE = 16, REC_MERGEFREE = 32 };

// The whole record, as five 16-byte loads.
__device__ __forceinline__ BoxRec load_rec(const BoxRec* p) {
  BoxRec r;
  const uint4* rp = reinterpret_cast<const uint4*>(p);
  uint4* dst = reinterpret_cast<uint4*>(&r);
#pragma unroll
  for (int i = 0; i < 5; ++i) dst[i] = __ldg(rp + i);
  return r;
}
// One 4-byte field of a record, at byte offset `off`, out of the 16-byte word that holds it: the tile kernels read a
// record's zone origin and flags to start its tile copy before they load the whole record.
__device__ __forceinline__ uint32_t rec_field(const BoxRec* p, size_t off) {
  const uint4 q = __ldg(reinterpret_cast<const uint4*>(p) + off / 16);
  const size_t i = off % 16 / 4;
  return i == 0 ? q.x : i == 1 ? q.y : i == 2 ? q.z : q.w;
}
__device__ __forceinline__ int rec_x0(const BoxRec* p) { return (int)rec_field(p, offsetof(BoxRec, x0)); }
__device__ __forceinline__ int rec_z0(const BoxRec* p) { return (int)rec_field(p, offsetof(BoxRec, z0)); }
__device__ __forceinline__ uint32_t rec_flags(const BoxRec* p) { return rec_field(p, offsetof(BoxRec, flags)); }
static_assert(offsetof(BoxRec, x0) % 4 == 0 && offsetof(BoxRec, z0) % 4 == 0 && offsetof(BoxRec, flags) % 4 == 0,
              "rec_field reads whole 4-byte words");

__device__ __forceinline__ void rec_to_ctx(const Checker& c, const BoxRec& r, BoxCtx& b) {
#pragma unroll
  for (int i = 0; i < 9; ++i) b.R1[i] = r.R1[i];
  b.P[0] = r.P[0]; b.P[1] = r.P[1]; b.P[2] = r.P[2];
  b.minB = r.minB; b.maxB = r.maxB;
  b.x0 = r.x0; b.x1 = r.x1; b.z0 = r.z0; b.z1 = r.z1;
  const int w = (r.flags & 7) ? 1 : 0;
  b.side[0] = c.side[w][0]; b.side[1] = c.side[w][1]; b.side[2] = c.side[w][2];
}

// One box of one item in the classify stage, in three steps that the classify kernel runs as separate waves:
//   box_geometry   box pose, map-inside test, AABB and zone: pure arithmetic on the item's pose, so the record emission
//                  recomputes it bit for bit instead of keeping it;
//   zone_classify  range-table reductions and the collider's early outs;
//   vertex_probe   the probe vertices of an all-finite zone that the early outs left open (probe_applies).
constexpr int kBoxOutside = -2;
constexpr int kBoxOutsideWindow = -3;   // map shards (artp_set_map_window): the item is reported invalid + sticky error

// Returns -1 with b complete, R_FREE when the AABB misses the map, kBoxOutside when the box centre is outside the map
// (the caller applies the outside-map rule), kBoxOutsideWindow when the zone leaves the handle's map window.
__device__ __forceinline__ int box_geometry(const Checker& c, const float R[9], const float R1[9], const float t[3], int k,
                                            BoxCtx& b) {
  const Field& g = c.f[0];      // both layers share the map geometry
  const bool foot = k > 0;
  const int fk = k - 1;
  const float ox = foot ? ((fk & 2) ? -c.feet_ox : c.feet_ox) : c.torso_off[0];
  const float oy = foot ? ((fk & 1) ? -c.feet_oy : c.feet_oy) : c.torso_off[1];
  const float oz = foot ? 0.0f : c.torso_off[2];
  const float sd[3] = {foot ? c.side[1][0] : c.side[0][0], foot ? c.side[1][1] : c.side[0][1],
                       foot ? c.side[1][2] : c.side[0][2]};
  float tt[3];
  compose_translation(R, t, ox, oy, oz, tt);
  if (!is_inside(c, tt[0], tt[1])) return kBoxOutside;   // validity_checker_body.cpp:29-32, validity_checker_feet.cpp:34-37
  // dCollideHeightfield prologue (heightfield.cpp:1841-1892) + dxBox::computeAABB: P = Rf^T (centre - field position),
  // Rf = rows [-1,0,0], [0,0,1], [0,1,-0] (the literal products with 0 / +-1 only change signs of zeros, which no
  // comparison sees). The caller passes R1 = Rf^T Rb.
  const float d0 = tt[0] - g.px, d1 = tt[1] - g.py, d2 = tt[2] - 0.0f;
  b.P[0] = -d0 + g.hW; b.P[1] = d2; b.P[2] = d1 + g.hD;
  const float xr = box_half_extent(R1, sd, 0), yr = box_half_extent(R1, sd, 1), zr = box_half_extent(R1, sd, 2);
  const float a0 = b.P[0] - xr, a1 = b.P[0] + xr, a4 = b.P[2] - zr, a5 = b.P[2] + zr;
  b.minB = b.P[1] - yr; b.maxB = b.P[1] + yr;
  if ((a0 > g.W || a4 > g.D) || (a1 < 0.0f || a5 < 0.0f)) return R_FREE;   // dCollide returns 0 (heightfield.cpp:1870-1876)
  b.x0 = max((int)floorf(next_down(a0 * g.iW)), 0);
  b.x1 = min((int)ceilf(next_up(a1 * g.iW)), g.nx - 1);
  b.z0 = max((int)floorf(next_down(a4 * g.iD)), 0);
  b.z1 = min((int)ceilf(next_up(a5 * g.iD)), g.nz - 1);
  if (b.x0 < g.x_lo || b.x1 > g.x_hi) return kBoxOutsideWindow;   // the zone leaves this handle's map window
#pragma unroll
  for (int i = 0; i < 9; ++i) b.R1[i] = R1[i];
  b.side[0] = sd[0]; b.side[1] = sd[1]; b.side[2] = sd[2];
  return -1;
}

// Whether a box that box_geometry placed outside (kBoxOutside / kBoxOutsideWindow) fails its item. Outside the map only a
// reach box does, and only when unknown space is untraversable; a zone that leaves the handle's map window always does
// (fail closed), and `raise` then sets the sticky error word.
__device__ __forceinline__ bool outside_fails(const Checker& c, bool foot, int r, bool raise) {
  if (r == kBoxOutsideWindow) {
    if (raise) *(volatile uint32_t*)c.err_word = 2u;
    return true;
  }
  return foot && c.unknown_untraversable;
}

// Zone of a box that box_geometry placed on the map: R_FREE / R_HIT when the early outs decide it, else -1. fl receives
// the record flags (box index, REC_*).
__device__ __forceinline__ int zone_classify(const Checker& c, const BoxCtx& b, int k, int force_all, uint32_t& fl) {
  const bool foot = k > 0;
  int r;                        // R_FREE / R_HIT / -1 undecided
  fl = (uint32_t)k;
  {
    // zone reductions from the range tables (exact: max/min/or are idempotent, windows may overlap)
    const Field& f = foot ? c.f[1] : c.f[0];
    const int nX = b.x1 - b.x0 + 1, nZ = b.z1 - b.z0 + 1;
    const int kk = 31 - __clz(min(nX, nZ));
    const int cx = (nX + (1 << kk) - 1) >> kk, cz = (nZ + (1 << kk) - 1) >> kk;
    if (force_all || kk < 1 || kk > f.kmax || cx * cz > 32) {
      r = -1; fl |= REC_NEEDS_REDUCE;
    } else {
      // Zone codes and flags from the compact tables first (one word per window, half the bytes of T: they stay in L2);
      // the exact T entries are read only when the codes' intervals leave a test open.
      const uint32_t* __restrict__ C = f.C[kk];
      const int sW = 1 << kk;
      const int xs1 = b.x1 - sW + 1, zs1 = b.z1 - sW + 1;   // the last window starts
      uint32_t wmax = 0, wmin = 0xFFFFFFFFu, wor = 0;
      if (cx * cz <= 8) {
        // The short side of the zone holds at most two windows (kk is the floor of its log2), so the windows start on a
        // 4 x 2 grid (8 x 1 when the short side holds one), long side first. All eight words are requested before any
        // is used; a start past the zone's last window clamps to that window (max, min and OR are idempotent).
        const bool zlong = cz > cx;
        const int sh = min(cx, cz) - 1;
        uint32_t wv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int a = j >> sh, s = j & sh;   // window along the long / short side
          const int ix = zlong ? s : a, iz = zlong ? a : s;
          wv[j] = __ldg(C + (size_t)min(b.z0 + iz * sW, zs1) * f.pitch + min(b.x0 + ix * sW, xs1));
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) { wmax = max(wmax, wv[j]); wmin = min(wmin, code_min_key(wv[j])); wor |= wv[j]; }
      } else {
        for (int iz = 0; iz < cz; ++iz) {
          const int zs = min(b.z0 + iz * sW, zs1);
          for (int ix = 0; ix < cx; ++ix) {
            const uint32_t wv = __ldg(C + (size_t)zs * f.pitch + min(b.x0 + ix * sW, xs1));
            wmax = max(wmax, wv); wmin = min(wmin, code_min_key(wv)); wor |= wv;
          }
        }
      }
      const uint32_t cM = code_max(wmax), cm = code_min(wmin), nf = code_flags(wor);
      const bool allFinite = (nf & 1) == 0;
      r = zone_early_out_codes(f, b, cM, cm, allFinite);
      if (r == kZoneUnknown) {
        // exact zone max / min (the max and min codes commute with the reductions; the exact values do too)
        const float2* __restrict__ T = f.T[kk];
        float mx = -CUDART_INF_F, mn = CUDART_INF_F;
#pragma unroll 1
        for (int iz = 0; iz < cz; ++iz) {
          const int zs = min(b.z0 + iz * sW, b.z1 - sW + 1);
#pragma unroll 1
          for (int ix = 0; ix < cx; ++ix) {
            const float2 v = __ldg(T + (size_t)zs * f.pitch + min(b.x0 + ix * sW, b.x1 - sW + 1));
            mx = fmaxf(mx, v.x); mn = fminf(mn, v.y);
          }
        }
        r = zone_early_out(b, mx, mn, allFinite);
      }
      if (allFinite) fl |= REC_ALLFINITE;
      if ((nf & 2) == 0) fl |= REC_MERGEFREE;   // no two triangles of the zone lie in one plane: greedy grouping is the identity
    }
  }
  return r;
}

// Vertex probes of a box zone_classify left undecided. In an all-finite zone every vertex with h > minB belongs to a kept
// triangle, and the collider returns 1 as soon as ANY such vertex lies inside the box (heightfield.cpp:1344-1441), so a hit
// found here is exactly the reference's answer; a miss decides nothing and the box is queued.
// Reach box: the cell under the box centre; torso: a 3x3 pattern across the footprint.
// (measured: 3x3 / 5x5 reach-box patterns remove another 25 % of the queue but cost the classify stage twice what the warp
// stage saves -- one thread walks them serially)
__device__ __forceinline__ bool probe_applies(const BoxCtx& b, uint32_t fl) {
  return (fl & REC_ALLFINITE) && b.x1 - b.x0 >= 1 && b.z1 - b.z0 >= 1;
}
__device__ __forceinline__ bool vertex_probe(const Checker& c, const BoxCtx& b, bool foot) {
  const Field& g = c.f[0];
  const Field& f = foot ? c.f[1] : c.f[0];
  const int np = foot ? 1 : 9;
  const float h0 = 0.5f * b.side[0], h1 = 0.5f * b.side[1];
  for (int pi = 0; pi < np; ++pi) {
    const float u0 = foot ? 0.0f : 0.7f * (float)(pi % 3 - 1), u1 = foot ? 0.0f : 0.7f * (float)(pi / 3 - 1);
    const float qx = b.P[0] + (u0 * h0) * b.R1[0] + (u1 * h1) * b.R1[1];
    const float qz = b.P[2] + (u0 * h0) * b.R1[6] + (u1 * h1) * b.R1[7];
    const int pcx = min(max((int)floorf(qx * g.iW), b.x0), b.x1 - 1);
    const int pcz = min(max((int)floorf(qz * g.iD), b.z0), b.z1 - 1);
    float hA, hB, hC, hD;
    load_cell(f, pcx, pcz, hA, hB, hC, hD);
    const float xA = pcx * f.sW, xB = (pcx + 1) * f.sW, zA = pcz * f.sD, zC = (pcz + 1) * f.sD;
    if ((hA > b.minB && vertex_inside(b, xA, hA, zA)) || (hB > b.minB && vertex_inside(b, xB, hB, zA)) ||
        (hC > b.minB && vertex_inside(b, xA, hC, zC)) || (hD > b.minB && vertex_inside(b, xB, hD, zC)))
      return true;
  }
  return false;
}

// All three steps for one box (the latency path): R_FREE / R_HIT when decided, -1 when the box needs the vertex / plane
// stages (b and fl are then complete), kBoxOutside / kBoxOutsideWindow as box_geometry.
__device__ __forceinline__ int classify_box(const Checker& c, const float R[9], const float R1[9], const float t[3], int k,
                                            int force_all, BoxCtx& b, uint32_t& fl) {
  fl = (uint32_t)k;
  const int g = box_geometry(c, R, R1, t, k, b);
  if (g != -1) return g;
  const int r = zone_classify(c, b, k, force_all, fl);
  return (r == -1 && probe_applies(b, fl) && vertex_probe(c, b, k > 0)) ? R_HIT : r;
}

// ---------------------------------------------------------------------------------------------
// Stage A: a CTA classifies kClassifyItems items box by box.
//   pose phase   one thread per item: state -> t, R, R1 (orthogonalised) into shared memory.
//   box waves    reach boxes 1..4, then the torso: a wave takes only the items that are still valid (this stage can only
//                INVALIDATE an item through a reach box that touches nothing, and a torso box is decided free here or
//                queued, so on an invalid pose the torso is usually never looked at). Lane j of the CTA classifies live
//                item j; the reach boxes that get past the early outs are compacted again and probed densely. (A thread
//                walking all five boxes of its item kept every warp on its slowest lane's path.)
//   emission     the undecided boxes of the items still valid, one thread per record: a block scan and one atomicAdd
//                per CTA and queue. A record's geometry is recomputed from the pose (box_geometry is pure arithmetic,
//                compiled without FMA contraction, so it is bit-identical); only its flag byte is kept.
// Records land in their queues in CTA order; the box kernels and the grouping stage only ever clear verdicts, so the
// order within a queue does not matter.
// ---------------------------------------------------------------------------------------------
// 64 items per CTA, 16 CTAs per SM (64 registers, no spills). Measured on the bench workload, H100 80GB HBM3 at 400 W:
// 256-item CTAs classified in 0.315 ms, 128-item CTAs in 0.244 ms, 64-item CTAs in 0.234 ms; small CTAs wait less at
// the waves' barriers.
constexpr int kClassifyItems = 64;                        // items (and threads) per CTA
constexpr int kClassifyWarps = kClassifyItems / 32;
constexpr int kPoseWords = 21;                            // t[3], R[9], R1[9]
// pending byte of an (item, box): REC_* flags and box index in bits 0-5, queue in bits 6-7 (0: decided)
enum { PEND_BIG = 1, PEND_REACH = 2, PEND_GROUP = 3 };

struct ClassifyShared {
  float pose[kPoseWords][kClassifyItems];
  float probe_f[4][kClassifyItems];                       // P, minB of a reach box to be probed, by wave lane
  int probe_i[4][kClassifyItems];                         // its zone x0, x1, z0, z1
  uint8_t valid[kClassifyItems];                          // 1 valid so far, 0 invalid (or out of range)
  uint8_t pend[5][kClassifyItems];
  uint16_t live[kClassifyItems];                          // items still valid at a wave
  uint16_t probe[kClassifyItems];                         // wave lanes whose reach box is probed
  uint16_t emit[5 * kClassifyItems];                      // (box << 8) | item of every record, grouped by queue
  unsigned long long warp_sum[kClassifyWarps];
  int warp_count[kClassifyWarps];
  uint32_t base[3];
};
static_assert(kClassifyItems <= 256, "emit packs the item index into 8 bits");
struct ClassifySharedWhy : ClassifyShared {               // the explain form: each item's word of the boxes decided here
  uint16_t why[kClassifyItems];
};

__device__ __forceinline__ void load_pose(const ClassifyShared& s, int i, float t[3], float R[9], float R1[9]) {
#pragma unroll
  for (int j = 0; j < 3; ++j) t[j] = s.pose[j][i];
#pragma unroll
  for (int j = 0; j < 9; ++j) { R[j] = s.pose[3 + j][i]; R1[j] = s.pose[12 + j][i]; }
}

// Exclusive CTA-wide scan of v (sums of fields that cannot overflow into each other); `total` receives the sum over the
// CTA. Uses s.warp_sum: consecutive calls must be separated by a barrier.
__device__ __forceinline__ unsigned long long cta_scan(ClassifyShared& s, unsigned long long v, unsigned long long& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned long long incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(kFull, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) s.warp_sum[wid] = incl;
  __syncthreads();
  unsigned long long before = 0;
  total = 0;
#pragma unroll
  for (int q = 0; q < kClassifyWarps; ++q) {
    const unsigned long long x = s.warp_sum[q];
    if (q < wid) before += x;
    total += x;
  }
  return before + incl - v;
}

// Writes the entries of the threads with `pred` to list in thread order; returns the list length. The list is written
// after a barrier and read after a second one, so every read of the list before the call is done before it changes.
__device__ __forceinline__ int cta_compact(ClassifyShared& s, uint16_t* list, bool pred, int entry) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(kFull, pred);
  if (lane == 0) s.warp_count[wid] = __popc(m);
  __syncthreads();
  int before = 0, total = 0;
#pragma unroll
  for (int q = 0; q < kClassifyWarps; ++q) {
    const int x = s.warp_count[q];
    before += q < wid ? x : 0;
    total += x;
  }
  if (pred) list[before + __popc(m & ((1u << lane) - 1u))] = (uint16_t)entry;
  __syncthreads();
  return total;
}

// Explain form (kWhy): s.valid stays 1 for every item in range, so every wave takes every item and every undecided box is
// queued; a decided box sets its bits in s.why instead of clearing s.valid, and the word goes to w.why.
template <bool kWhy>
__global__ void __launch_bounds__(kClassifyItems, 16)
classify_items_kernel(const Checker c, const WorkOf<kWhy> w, BoxRec* __restrict__ recs_w, BoxRec* __restrict__ recs_f,
                      BoxRec* __restrict__ recs_g, uint32_t* __restrict__ count_w, uint32_t* __restrict__ count_f,
                      uint32_t* __restrict__ count_g, int force_all) {   // force_all: every in-map box goes to the grouping stage (artp_set_mode 1)
  __shared__ std::conditional_t<kWhy, ClassifySharedWhy, ClassifyShared> s;
  const int tid = threadIdx.x;
  const uint32_t item0 = w.item_base + blockIdx.x * kClassifyItems;
  const bool in_range = item0 + tid < w.n_items;
  if (in_range) {
    double st[7];
    load_item_state(w, item0 + tid, st);
    float t[3], R[9], Rb[9];
    pose3_from_se3(st, t, R);
#pragma unroll
    for (int i = 0; i < 9; ++i) Rb[i] = R[i];
    orthogonalize_r(Rb);          // dBodySetRotation of the same matrix for all five boxes
#pragma unroll
    for (int j = 0; j < 3; ++j) s.pose[j][tid] = t[j];
#pragma unroll
    for (int j = 0; j < 9; ++j) s.pose[3 + j][tid] = R[j];
#pragma unroll
    for (int j = 0; j < 3; ++j) { s.pose[12 + j][tid] = -Rb[j]; s.pose[15 + j][tid] = Rb[6 + j]; s.pose[18 + j][tid] = Rb[3 + j]; }
  }
  s.valid[tid] = in_range ? 1 : 0;
  if constexpr (kWhy) s.why[tid] = 0;
#pragma unroll
  for (int k = 0; k < 5; ++k) s.pend[k][tid] = 0;

#pragma unroll 1
  for (int kk = 0; kk < 5; ++kk) {
    const int k = kk == 4 ? 0 : kk + 1;
    const bool foot = k > 0;
    const int n_live = cta_compact(s, s.live, s.valid[tid] != 0, tid);
    bool probe = false;
    if (tid < n_live) {
      const int i = s.live[tid];
      float t[3], R[9], R1[9];
      load_pose(s, i, t, R, R1);
      BoxCtx b;
      uint32_t fl = 0;
      int r = box_geometry(c, R, R1, t, k, b);
      if (r == -1) r = zone_classify(c, b, k, force_all, fl);
      if (r == kBoxOutside || r == kBoxOutsideWindow) {
        if constexpr (kWhy) s.why[i] |= (uint16_t)((1u << (8 + k)) | (outside_fails(c, foot, r, true) ? 1u << k : 0u));
        else if (outside_fails(c, foot, r, true)) s.valid[i] = 0;
      } else if (r == -1) {
        // reach boxes go to their own queue (small TMA tiles); the torso -- and a reach box whose zone would not fit the
        // small tile -- to the big-tile queue
        const bool thread_path = foot && (b.x1 - b.x0) + 4 <= c.reach_tw && (b.z1 - b.z0) + 1 <= c.reach_th;
        // ... and of those, the merge-free ones reduced by the tables (no merge screen, no zone reduction; a zone with -inf
        // heights too) to the 8-lane-group kernel
        const bool group_path = thread_path && recs_g != nullptr && (fl & (REC_MERGEFREE | REC_NEEDS_REDUCE)) == REC_MERGEFREE;
        s.pend[k][i] = (uint8_t)(fl | (uint32_t)(group_path ? PEND_GROUP : thread_path ? PEND_REACH : PEND_BIG) << 6);
        // Vertex probes here only for reach boxes (one cell); an undecided torso is rare and its probes run lane-parallel
        // at the head of the warp stage instead. Classify without the probes measured slower: the boxes they decide
        // land in the queues.
        probe = foot && probe_applies(b, fl);
        if (probe) {
          s.probe_f[0][tid] = b.P[0]; s.probe_f[1][tid] = b.P[1]; s.probe_f[2][tid] = b.P[2]; s.probe_f[3][tid] = b.minB;
          s.probe_i[0][tid] = b.x0; s.probe_i[1][tid] = b.x1; s.probe_i[2][tid] = b.z0; s.probe_i[3][tid] = b.z1;
        }
      } else if (box_fails(foot, r)) {
        if constexpr (kWhy) s.why[i] |= (uint16_t)(1u << k);
        else s.valid[i] = 0;
      }
    }
    if (!foot) break;
    const int n_probe = cta_compact(s, s.probe, probe, tid);
    if (tid < n_probe) {
      const int p = s.probe[tid], i = s.live[p];
      BoxCtx b;
      b.P[0] = s.probe_f[0][p]; b.P[1] = s.probe_f[1][p]; b.P[2] = s.probe_f[2][p]; b.minB = s.probe_f[3][p];
      b.x0 = s.probe_i[0][p]; b.x1 = s.probe_i[1][p]; b.z0 = s.probe_i[2][p]; b.z1 = s.probe_i[3][p];
#pragma unroll
      for (int j = 0; j < 9; ++j) b.R1[j] = s.pose[12 + j][i];
      b.side[0] = c.side[1][0]; b.side[1] = c.side[1][1]; b.side[2] = c.side[1][2];
      if (vertex_probe(c, b, true)) s.pend[k][i] = 0;           // the reach box touches: decided
    }
  }
  __syncthreads();

  // provisional result; the later stages clear it if an undecided box fails
  const bool valid = s.valid[tid] != 0;
  if (in_range) {
    const uint32_t slot = item_slot(w, item0 + tid);
    if constexpr (kWhy) w.why[slot] = s.why[tid];
    else if (w.edge_mode) { if (!valid) w.valid[slot] = 0; }
    else w.valid[slot] = (uint8_t)valid;
  }
  // records of the undecided boxes of valid items: per queue, 21-bit counts packed into one scan
  unsigned long long cnt = 0;
  if (valid) {
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const int q = s.pend[k][tid] >> 6;
      if (q) cnt += 1ull << (21 * (q - 1));
    }
  }
  unsigned long long tot;
  unsigned long long off = cta_scan(s, cnt, tot);
  if (tot == 0) return;
  const uint32_t n_w = (uint32_t)(tot & 0x1FFFFF), n_f = (uint32_t)((tot >> 21) & 0x1FFFFF), n_g = (uint32_t)(tot >> 42);
  if (tid == 0) {
    s.base[0] = n_w ? atomicAdd(count_w, n_w) : 0u;
    s.base[1] = n_f ? atomicAdd(count_f, n_f) : 0u;
    s.base[2] = n_g ? atomicAdd(count_g, n_g) : 0u;
  }
  if (cnt) {   // the list holds the big-tile records, then the reach-box records, then the group records
    uint32_t pw = (uint32_t)(off & 0x1FFFFF), pf = n_w + (uint32_t)((off >> 21) & 0x1FFFFF), pg = n_w + n_f + (uint32_t)(off >> 42);
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const int q = s.pend[k][tid] >> 6;
      const uint16_t e = (uint16_t)((k << 8) | tid);
      if (q == PEND_BIG) s.emit[pw++] = e;
      else if (q == PEND_REACH) s.emit[pf++] = e;
      else if (q == PEND_GROUP) s.emit[pg++] = e;
    }
  }
  __syncthreads();
  const uint32_t n_rec = n_w + n_f + n_g;
#pragma unroll 1
  for (uint32_t j = tid; j < n_rec; j += kClassifyItems) {
    const int e = s.emit[j], i = e & 0xFF, k = e >> 8;
    float t[3], R[9], R1[9];
    load_pose(s, i, t, R, R1);
    BoxCtx b;
    box_geometry(c, R, R1, t, k, b);
    BoxRec o;
#pragma unroll
    for (int m = 0; m < 9; ++m) o.R1[m] = R1[m];
    o.P[0] = b.P[0]; o.P[1] = b.P[1]; o.P[2] = b.P[2];
    o.minB = b.minB; o.maxB = b.maxB;
    o.x0 = b.x0; o.x1 = b.x1; o.z0 = b.z0; o.z1 = b.z1;
    o.item = item_slot(w, item0 + i);   // later stages only need the verdict slot
    o.flags = s.pend[k][i] & 0x3Fu;
    if (j < n_w) recs_w[s.base[0] + j] = o;
    else if (j < n_w + n_f) recs_f[s.base[1] + (j - n_w)] = o;
    else recs_g[s.base[2] + (j - n_w - n_f)] = o;
  }
}

// -------------------------------------------------------------------------------------------------
// K2: block-level exact decision including the greedy epsilon grouping.
// Shared memory: planes[T][4] floats, group[T] ints, state[T] bytes, T = 2 * max cells of a zone.
// -------------------------------------------------------------------------------------------------
struct BlockShared {
  float* planes;     // [T][4]
  int* group;        // [T] base index (== own index for bases); -1 for not-kept
  uint8_t* state;    // [T] 1 = assigned
  int T_cap;
};
// The store carved from dynamic shared memory of T_cap * 21 bytes: planes, then group, then state.
__device__ __forceinline__ BlockShared block_shared(unsigned char* smem, int T_cap) {
  BlockShared sh;
  sh.T_cap = T_cap;
  sh.planes = reinterpret_cast<float*>(smem);
  sh.group = reinterpret_cast<int*>(smem + (size_t)T_cap * 16);
  sh.state = reinterpret_cast<uint8_t*>(smem + (size_t)T_cap * 20);
  return sh;
}

__device__ __forceinline__ float block_reduce_max(float v, float* red, bool is_max) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float a = __shfl_xor_sync(kFull, v, o);
    v = is_max ? ((v > a) ? v : a) : ((v > a) ? a : v);
  }
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float r = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) {
    const float a = red[i];
    r = is_max ? ((r > a) ? r : a) : ((r > a) ? a : r);
  }
  return r;
}

// Returns R_FREE / R_HIT, or R_DEFER if the zone does not fit the shared-memory plane store (host
// sizes it so that this cannot happen for the configured boxes).
__device__ int box_collide_block(const Field& f, const BoxCtx& b, const BlockShared& sh, float* red, int* s_next) {
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int nX = b.x1 - b.x0 + 1, nZ = b.z1 - b.z0 + 1, nV = nX * nZ;
  const float* base = f.H + (size_t)b.z0 * f.pitch + b.x0;
  float mx = -CUDART_INF_F, mn = CUDART_INF_F;
  int fin = 1;
  for (int t = tid; t < nV; t += nthr) {
    const int zi = t / nX, xi = t - zi * nX;
    const float h = __ldg(base + (size_t)zi * f.pitch + xi);
    mx = (mx > h) ? mx : h;
    if (finitef(h)) mn = (mn > h) ? h : mn; else fin = 0;
  }
  const float maxY = block_reduce_max(mx, red, true);
  const float minY = block_reduce_max(mn, red, false);
  const bool allFinite = __syncthreads_and(fin) != 0;
  const int e = zone_early_out(b, maxY, minY, allFinite);
  if (e >= 0) return e;
  const int nCX = nX - 1, nCZ = nZ - 1, nC = nCX * nCZ, T = 2 * nC;
  if (T > sh.T_cap) return R_DEFER;
  // triangles in emission order (x outer, z inner, Up then Down): vertex tests + planes
  int hit = 0;
  for (int t = tid; t < nC; t += nthr) {
    const int cxi = t / nCZ, czi = t - cxi * nCZ;          // emission order index t = cxi*nCZ + czi
    const int cx = b.x0 + cxi, cz = b.z0 + czi;
    float hA, hB, hC, hD;
    load_cell(f, cx, cz, hA, hB, hC, hD);
    const CellKeep ck = cell_keep(hA, hB, hC, hD, b.minB);
    const float xA = cx * f.sW, xB = (cx + 1) * f.sW, zA = cz * f.sD, zC = (cz + 1) * f.sD;
    if (ck.tested(0)) hit |= vertex_inside(b, xA, hA, zA);
    if (ck.tested(1)) hit |= vertex_inside(b, xB, hB, zA);
    if (ck.tested(2)) hit |= vertex_inside(b, xA, hC, zC);
    if (ck.tested(3)) hit |= vertex_inside(b, xB, hD, zC);
    const int i0 = 2 * t;
    sh.state[i0] = 0; sh.state[i0 + 1] = 0;
    sh.group[i0] = -1; sh.group[i0 + 1] = -1;
    if (ck.up) { cell_plane(f, true, cx, cz, hA, hB, hC, hD, sh.planes + 4 * i0); sh.group[i0] = i0; }
    if (ck.dn) { cell_plane(f, false, cx, cz, hA, hB, hC, hD, sh.planes + 4 * (i0 + 1)); sh.group[i0 + 1] = i0 + 1; }
  }
  if (__syncthreads_or(hit)) return R_HIT;
  // Singleton screen. The greedy grouping below is sequential in the number of groups (~T when nothing merges:
  // 2000 block-wide steps, 60 us for a torso zone). A triangle can absorb or be absorbed only if some OTHER kept
  // triangle epsilon-matches it, and matching planes have normals within eps, i.e. the other's (n0, n2) bucket lies in
  // this one's +-kKeyMargin neighbourhood. Two bit tables over the hashed buckets (occupied, occupied twice) find the
  // triangles that cannot have a partner: they are their own group, marked assigned up front; the sequential loop only
  // walks the rest (normally none).
  {
    __shared__ uint32_t occ1[kBloomWords], occ2[kBloomWords];
    for (int i = tid; i < kBloomWords; i += nthr) { occ1[i] = 0u; occ2[i] = 0u; }
    __syncthreads();
    for (int m = tid; m < T; m += nthr) {
      if (sh.group[m] < 0) continue;
      const float* pm = sh.planes + 4 * m;
      const uint32_t hsh = bloom_hash(nkey(pm[0]), nkey(pm[2]));
      const uint32_t bit = 1u << (hsh & 31);
      if (atomicOr(&occ1[hsh >> 5], bit) & bit) atomicOr(&occ2[hsh >> 5], bit);
    }
    __syncthreads();
    int any_pot = 0;
    for (int m = tid; m < T; m += nthr) {
      if (sh.group[m] < 0) continue;
      const float* pm = sh.planes + 4 * m;
      const int kxc = nkey(pm[0]), kzc = nkey(pm[2]);
      const int kx0 = nkey(pm[0] - kKeyMargin), kx1 = nkey(pm[0] + kKeyMargin);
      const int kz0 = nkey(pm[2] - kKeyMargin), kz1 = nkey(pm[2] + kKeyMargin);
      bool pot = false;
      for (int kx = kx0; kx <= kx1; ++kx)
        for (int kz = kz0; kz <= kz1; ++kz) {
          const uint32_t hsh = bloom_hash(kx, kz);
          const uint32_t* tab = (kx == kxc && kz == kzc) ? occ2 : occ1;   // own bucket: someone else must be there too
          pot = pot || ((tab[hsh >> 5] >> (hsh & 31)) & 1u);
        }
      if (pot) any_pot = 1; else sh.state[m] = 1;
    }
    any_pot = __syncthreads_or(any_pot);
    if (!any_pot) goto groups_done;
  }
  // greedy grouping (heightfield.cpp:1511-1556)
  {
  int k = -1;
  for (;;) {
    if (tid == 0) {
      int q = k + 1;
      while (q < T && (sh.group[q] < 0 || sh.state[q])) ++q;
      *s_next = q;
    }
    __syncthreads();
    k = *s_next;
    if (k >= T) break;
    const float* pk = sh.planes + 4 * k;
    const float p0 = pk[0], p1 = pk[1], p2 = pk[2], p3 = pk[3];
    for (int m = k + 1 + tid; m < T; m += nthr) {
      if (sh.group[m] < 0 || sh.state[m]) continue;
      const float* pm = sh.planes + 4 * m;
      if (fabsf(p1 - pm[1]) < ARTP_EPS && fabsf(p3 - pm[3]) < ARTP_EPS && fabsf(p0 - pm[0]) < ARTP_EPS &&
          fabsf(p2 - pm[2]) < ARTP_EPS) {
        sh.state[m] = 1;
        sh.group[m] = k;
      }
    }
    if (tid == 0) sh.state[k] = 1;
    __syncthreads();
  }
  }
groups_done:
  // per-group plane contacts vs member triangles (heightfield.cpp:1573-1617), evaluated per member
  hit = 0;
  for (int m = tid; m < T; m += nthr) {
    const int g = sh.group[m];
    if (g < 0) continue;
    float cx[4], cz[4];
    const int nc = box_plane(b, sh.planes + 4 * g, 4, cx, cz);
    if (nc == 0) continue;
    const int t = m >> 1;
    const int cxi = t / nCZ, czi = t - cxi * nCZ;
    const bool isUp = (m & 1) == 0;
    const int tcx = b.x0 + cxi + (isUp ? 0 : 1), tcz = b.z0 + czi + (isUp ? 0 : 1);
    for (int i = 0; i < nc; ++i) hit |= on_tri(f, isUp, tcx, tcz, cx[i], cz[i]);
  }
  return __syncthreads_or(hit) ? R_HIT : R_FREE;
}

constexpr int kBlockStageThreads = 256;   // threads per deferred box in the grouping stage
template <bool kWhy>
__global__ void __launch_bounds__(kBlockStageThreads)
box_items_block_kernel(const Checker c, const WorkOf<kWhy> w, const BoxRec* __restrict__ recs, const BoxRec* __restrict__ recs_f,
                       const uint32_t* __restrict__ defer_count, const uint32_t* __restrict__ defer_list, int T_cap,
                       uint32_t* __restrict__ overflow) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float red[kBlockStageThreads / 32];
  __shared__ int s_next;
  const BlockShared sh = block_shared(smem_raw, T_cap);
  const uint32_t count = *defer_count;
  for (uint32_t q = blockIdx.x; q < count; q += gridDim.x) {
    const uint32_t e = defer_list[q];     // bit 31: record of the reach-box queue
    const BoxRec r = (e & 0x80000000u) ? recs_f[e & 0x7fffffffu] : recs[e];
    const uint32_t slot = r.item;
    const bool foot = (r.flags & 7) != 0;
    BoxCtx b;
    rec_to_ctx(c, r, b);
    const int res = box_collide_block(foot ? c.f[1] : c.f[0], b, sh, red, &s_next);
    if (threadIdx.x == 0) {
      // a zone that does not fit the plane store cannot be decided: fail closed (item invalid) and raise the sticky
      // error word (mapped host memory; the host returns ARTP_E_LIMIT from the call / artp_poll_error)
      if constexpr (kWhy) {
        if (res == R_DEFER) *(volatile uint32_t*)overflow = 1u;
        if (res == R_DEFER || box_fails(foot, res)) why_set(w.why, slot, (int)(r.flags & 7));
      } else {
        if (res == R_DEFER) { *(volatile uint32_t*)overflow = 1u; w.valid[slot] = 0; }
        else if (box_fails(foot, res)) w.valid[slot] = 0;
      }
    }
    __syncthreads();
  }
}

// -------------------------------------------------------------------------------------------------
// Latency path: the planner's one-state-at-a-time isValid calls (ompl::base::StateValidityChecker::isValid). One launch
// does everything for up to kSmallBatch poses -- the states travel in the kernel parameter block and the verdicts are
// written straight to mapped host memory, so a call is one launch + one stream synchronise instead of memset, H2D,
// three launches and D2H. One CTA per pose: threads 0..4 classify the five boxes, warps 0..4 run the warp-stage
// decision of the undecided ones, the whole CTA handles a deferred box with the grouping-stage code.
// -------------------------------------------------------------------------------------------------
constexpr int kSmallBatch = 64;
struct SmallBatch {
  double s[kSmallBatch][7];
};

// The decision of one pose by one CTA of 256 threads, the latency path's routine: threads 0..4 fill the pose's state with
// load_state(st) and classify the five boxes, warps 0..4 run the warp-stage decision of the undecided ones, and the whole
// CTA runs a deferred box through the grouping stage. The verdict goes to out[blockIdx.x].
template <typename LoadState>
__device__ __forceinline__ void pose_cta_decide(const Checker& c, int T_cap, uint32_t* overflow, int force_all, uint8_t* out,
                                                LoadState load_state) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float red[8];
  __shared__ int s_next;
  __shared__ BoxCtx s_box[5];
  __shared__ uint32_t s_fl[5];
  __shared__ int s_res[5];    // per box after classify: -1 undecided, R_FREE / R_HIT decided, kBoxOutside(Window)
  __shared__ int s_res2[5];   // warp-stage result of an undecided box (separate: other warps may still read s_res)
  __shared__ WarpScratch s_ws[5];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid < 5) {
    double st[7];
    load_state(st);
    float t[3], R[9], Rb[9], R1[9];
    pose3_from_se3(st, t, R);
#pragma unroll
    for (int i = 0; i < 9; ++i) Rb[i] = R[i];
    orthogonalize_r(Rb);
#pragma unroll
    for (int j = 0; j < 3; ++j) { R1[j] = -Rb[j]; R1[3 + j] = Rb[6 + j]; R1[6 + j] = Rb[3 + j]; }
    BoxCtx b;
    uint32_t fl = 0;
    const int r = classify_box(c, R, R1, t, tid, force_all, b, fl);
    s_res[tid] = r;
    if (r == -1) { s_box[tid] = b; s_fl[tid] = fl; }
  }
  __syncthreads();
  // item verdict from the decided boxes
  bool valid = true;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const int r = s_res[k];
    if (r == kBoxOutside || r == kBoxOutsideWindow) { if (outside_fails(c, k > 0, r, tid == 0)) valid = false; }
    else if (box_fails(k > 0, r)) valid = false;
  }
  if (valid && !force_all && wid < 5 && s_res[wid] == -1) {
    const bool foot = wid > 0;
    const Field& fw = foot ? c.f[1] : c.f[0];
    const ZoneView zv{fw.H + (size_t)s_box[wid].z0 * fw.pitch + s_box[wid].x0, fw.pitch};   // straight from the heightfield
    const int res = box_collide_warp<false>(fw, s_box[wid], zv, s_ws[wid], lane, c.cell_margin,
                                            (s_fl[wid] & REC_NEEDS_REDUCE) != 0, (s_fl[wid] & REC_ALLFINITE) != 0,
                                            (s_fl[wid] & REC_MERGEFREE) != 0);
    if (lane == 0) s_res2[wid] = res;
  }
  __syncthreads();
  if (valid) {
    const BlockShared sh = block_shared(smem_raw, T_cap);
#pragma unroll 1
    for (int k = 0; k < 5; ++k) {
      int r = s_res[k];   // block-uniform
      if (r == -1 && !force_all) r = s_res2[k];
      if (r == -1 || r == R_DEFER) {   // -1 only in force_all mode
        r = box_collide_block(k > 0 ? c.f[1] : c.f[0], s_box[k], sh, red, &s_next);
        if (r == R_DEFER) { if (tid == 0) *(volatile uint32_t*)overflow = 1u; valid = false; }   // fail closed
        __syncthreads();
      }
      if (box_fails(k > 0, r)) valid = false;
    }
  }
  if (tid == 0) out[blockIdx.x] = valid ? 1 : 0;
}

__global__ void __launch_bounds__(256)
pose_small_kernel(const Checker c, const SmallBatch sb, uint8_t* __restrict__ out, int T_cap, uint32_t* __restrict__ overflow,
                  int force_all, int steps) {   // steps < 0: CTA b checks sb.s[b]; else edges: see below
  pose_cta_decide(c, T_cap, overflow, force_all, out, [&](double st[7]) {
    if (steps < 0) {
#pragma unroll
      for (int i = 0; i < 7; ++i) st[i] = sb.s[blockIdx.x][i];
    } else {
      // edge e = (s1 = sb.s[2e], s2 = sb.s[2e+1]); CTA e*(steps+1)+j checks its EDGE-mode state j
      const uint32_t per = (uint32_t)steps + 1u, e = blockIdx.x / per;
      edge_state(sb.s[2 * e], sb.s[2 * e + 1], blockIdx.x - e * per, steps, st);
    }
  });
}

// The roadmap's interior states (artp_roadmap.cu): CTA b decides states[b] for b < *count (an upper bound sizes the grid;
// the CTAs past the count exit) into verdict[b]. Nothing to do once *stop is set.
__global__ void __launch_bounds__(256)
pose_states_kernel(const Checker c, const double* __restrict__ states, const uint32_t* __restrict__ count,
                   const uint32_t* __restrict__ stop, uint8_t* __restrict__ verdict, int T_cap, uint32_t* __restrict__ overflow) {
  if (*stop || blockIdx.x >= *count) return;
  pose_cta_decide(c, T_cap, overflow, 0, verdict, [&](double st[7]) {
#pragma unroll
    for (int i = 0; i < 7; ++i) st[i] = states[(size_t)blockIdx.x * 7 + i];
  });
}

}  // namespace artp
