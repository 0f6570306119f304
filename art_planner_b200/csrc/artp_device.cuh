// art_planner_b200/csrc/artp_device.cuh
// Exact fp32 building blocks of the box-vs-heightfield decision, shared by the warp kernel, the
// block-level grouping kernel and the map's plane tables (artp_map.cu). Arithmetic contract (SURVEY.md
// Appendix A): IEEE fp32, round-to-nearest, NO FMA contraction, left-to-right association exactly as the
// reference's ODE source writes it.
// This translation unit is compiled with -fmad=false and default -prec-div/-prec-sqrt/-ftz=false;
// 1/sqrt is spelled as two correctly rounded operations (ode/include/ode/common.h:285).
#pragma once

#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include <cmath>

#include "../../include/artp.h"

#define ARTP_EPS 1.1920928955078125e-07f  // dEpsilon = FLT_EPSILON (ode/ode/src/common.h:42)

namespace artp {

// One heightfield layer as ODE sees it (dxHeightfieldData::SetData, ode/ode/src/heightfield.cpp:130-169).
constexpr int kMaxLevel = 6;   // range tables for windows up to 64 x 64 vertices

struct Field {
  const float* H;  // H[x + z*pitch] = layer(x, nz-1-z): column-reversed copy (height_map_box_checker.cpp:44)
  int nx, nz;      // m_nWidthSamples (rows), m_nDepthSamples (cols)
  int pitch;       // row stride in floats (multiple of 4 -> 16 B aligned rows)
  // Range tables (exact, idempotent reductions): level k holds, for every (x,z), the reduction over the
  // 2^k x 2^k vertex window starting there: T[k][x + z*pitch] = (max h, min over finite h or +inf). Built at
  // artp_set_map, k = 1..kmax.
  const float2* T[kMaxLevel + 1];
  // Conservative copies of T[k] at half the size that also carry the window's flags (the classify stage's random lookups
  // then stay in L2, one load per window): C[k][i] = (maxCode << 17) | (minCode << 2) | flags (see code_max / code_min /
  // code_flags) with max in [dec(maxCode - 1), dec(maxCode)] and min in [dec(minCode), dec(minCode + 1)],
  // dec(c) = cbase + c * cstep (code_dec). Finite heights take max codes 1..kCodeMax and min codes 0..kCodeMax; a window
  // without a finite height has max code 0 (max -inf) and min code kCodeNone (min +inf). Flag bit 0 = the window holds a
  // non-finite height, bit 1 = a cell starting in the window has a triangle whose plane matches (within eps) the plane of
  // another triangle of the map. Same pitch and row shift as T.
  const uint32_t* C[kMaxLevel + 1];
  float cbase, cstep;   // smallest finite height of the stored window; a power of two
  int kmax;
  float W, D, hW, hD, sW, sD, asp, iW, iD;
  float px, py;    // heightfield body position (float casts of the map centre)
  // Map window (artp_set_map_window): only vertices x in [x_lo, x_hi] are stored (H, T, C are shifted by -x_lo so that
  // global indices keep working); nx and all geometry are those of the full map. Whole map: 0, nx - 1.
  int x_lo, x_hi;
};

struct Checker {
  Field f[2];             // 0: `elevation` (torso), 1: `elevation_masked` (feet)
  float side[2][3];       // torso box, reach box
  float torso_off[3];     // (off.x, off.y, float(off.z - feet.off.z)), validity_checker.cpp:41-43
  float feet_ox, feet_oy;
  int unknown_untraversable;
  double Lx, Ly, cx, cy;  // grid_map length / position (doubles) for isInside
  float cell_margin;      // candidate-cell search margin in cells (plane stage)
  uint32_t* err_word;     // sticky error word (mapped host memory): bit 0 plane-store overflow, bit 1 box outside the map window
  // extent of the reach-box queue's TMA tile in floats (artp_tiles.cuh; 0: no such queue). The tile starts at column
  // x0 & ~3, so a zone may be at most reach_tw - 3 wide.
  int reach_tw, reach_th;
};

// TMA tile of a box queue (artp_tiles.cuh).
struct TileCfg {
  int tw, th;              // tile extent in floats (tw a multiple of 4; a zone may be at most tw - 3 wide, th high)
  uint32_t bytes, stride;  // tw * th * 4, and that rounded up to 128 bytes
  int x_off;               // first stored vertex column of the layer (map window), a multiple of 4
  int slots;               // tile slots per warp: 2 = the next box's tile is prefetched while this one is decided, 1 = none
};
struct SamplerDev {
  const float* elevation_rev;   // Field::H of the elevation layer: H[x + z*pitch] = layer(x, cols-1-z)
  int pitch;
  const float* normal_x;        // grid_map layout: (row, col) at row + col*rows
  const float* normal_y;
  const float* normal_z;
  const float* std_dev;
  const float* cum_prob;        // may be null (uniform mode)
  const float* cum_row;         // rows floats
  int rows, cols;
  double res, cx, cy;
  double max_roll_pert, max_pitch_pert;
  int from_distribution;
  double low[2], high[2];
  double reach_z;
};

// OMPL 1.4.2 SE3StateSpace::interpolate (RealVector lerp + SO3 slerp), double.
__device__ __forceinline__ void se3_interpolate(const double* a, const double* b, double t, double* out) {
  for (int i = 0; i < 3; ++i) out[i] = a[i] + (b[i] - a[i]) * t;
  const double dq = a[3] * b[3] + a[4] * b[4] + a[5] * b[5] + a[6] * b[6];
  const double dqa = fabs(dq);
  const double theta = (dqa > 1.0 - 1e-9) ? 0.0 : acos(dqa);
  if (theta > 2.220446049250313e-16) {
    const double d = 1.0 / sin(theta);
    const double s0 = sin((1.0 - t) * theta);
    double s1 = sin(t * theta);
    if (dq < 0) s1 = -s1;
    out[3] = (a[3] * s0 + b[3] * s1) * d;
    out[4] = (a[4] * s0 + b[4] * s1) * d;
    out[5] = (a[5] * s0 + b[5] * s1) * d;
    out[6] = (a[6] * s0 + b[6] * s1) * d;
  } else {
    out[3] = a[3]; out[4] = a[4]; out[5] = a[5]; out[6] = a[6];
  }
}

// OMPL 1.4.2 SE3StateSpace::distance = RealVectorStateSpace::distance (sqrt of the running sum of squares) + 1.0 *
// SO3StateSpace::distance (arcLength: acos(|q1.q2|), 0 above 1 - MAX_QUATERNION_NORM_ERROR = 1 - 1e-9), in double.
__device__ __forceinline__ double se3_distance(const double* a, const double* b) {
  double r = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double d = a[i] - b[i];
    r += d * d;
  }
  const double dq = fabs(a[3] * b[3] + a[4] * b[4] + a[5] * b[5] + a[6] * b[6]);
  const double so3 = dq > 1.0 - 1e-9 ? 0.0 : acos(dq);
  return sqrt(r) + so3;
}

// ---- Edge discretisation ---------------------------------------------------------------------------------------------
// How an edge (a, b) is cut into the states a check visits or into the pieces the learned cost prices. Every unit that
// uses these is compiled without FMA contraction (build.py), so a __host__ __device__ body does the same arithmetic on
// both sides.

// Longest valid segment of the R^3 and SO(3) parts of an SE(3) space: maximum extent * longestValidSegmentFraction, with
// the extents |high - low| and pi/2 (OMPL 1.4.2 StateSpace.cpp).
struct SegLen { double r3, so3; };
// The segment lengths of sp (fraction 0.01 when sp's is not positive); false for a space whose R^3 length is not > 0.
inline bool segment_lengths(const artp_se3_space& sp, SegLen& out) {
  const double frac = sp.longest_valid_segment_fraction > 0 ? sp.longest_valid_segment_fraction : 0.01;
  double e2 = 0;
  for (int i = 0; i < 3; ++i) e2 += (sp.high[i] - sp.low[i]) * (sp.high[i] - sp.low[i]);
  out.r3 = std::sqrt(e2) * frac;
  out.so3 = 0.5 * 3.14159265358979323846 * frac;
  return out.r3 > 0;
}

// ompl::base::CompoundStateSpace::validSegmentCount for SE3: the larger of (unsigned)ceil(distance / segment length) over
// the R^3 part (Euclidean distance) and the SO(3) part (arc length acos(|q1.q2|), 0 above 1 - 1e-9). 0 for identical states.
__host__ __device__ __forceinline__ uint32_t valid_segment_count(const double* a, const double* b, SegLen seg) {
  const double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
  const double d3 = sqrt(dx * dx + dy * dy + dz * dz);
  const double dq = fabs(a[3] * b[3] + a[4] * b[4] + a[5] * b[5] + a[6] * b[6]);
  const double ds = dq > 1.0 - 1e-9 ? 0.0 : acos(dq);
  const unsigned n3 = (unsigned)ceil(d3 / seg.r3), ns = (unsigned)ceil(ds / seg.so3);
  return n3 > ns ? n3 : ns;
}
// The segments DiscreteMotionValidator::checkMotion walks: at least one, so identical states check s2 only.
__host__ __device__ __forceinline__ uint32_t segment_count(const double* a, const double* b, SegLen seg) {
  const uint32_t nd = valid_segment_count(a, b, seg);
  return nd > 1u ? nd : 1u;
}

// lateralDistance (utils.h:52-61) from a to b over a length L.
__host__ __device__ __forceinline__ double lateral_ratio(const double* a, const double* b, double L) {
  const double dx = b[0] - a[0], dy = b[1] - a[1];
  return sqrt(dx * dx + dy * dy) / L;
}
// Interior states of a roadmap connection: (unsigned)(lateralDistance / L), L = kMaxDist (prm_motion_cost.cpp:340-343).
__host__ __device__ __forceinline__ uint32_t lateral_count(const double* a, const double* b, double L) {
  return (unsigned)lateral_ratio(a, b, L);
}
// Pieces MotionCostObjective::motionCost splits an edge into: (unsigned)(lateralDistance / max_query_edge_length) + 1
// (motion_cost_objective.cpp:40-45); 0 when that quotient does not fit 32 bits or is not finite.
__host__ __device__ __forceinline__ uint64_t cost_pieces(const double* a, const double* b, double L) {
  const double q = lateral_ratio(a, b, L);
  if (!(q < 4294967296.0)) return 0;
  return (uint64_t)(unsigned int)q + 1;
}

// Interior state j (1 .. n) of an edge with n interior states: interpolate(a, b, j * (1.0 / (n + 1))), the product form
// of prm_motion_cost.cpp:345-353 and motion_cost_objective.cpp:49-67 (not OMPL's j / nd quotient).
template <typename I>   // the caller's index type; j and n + 1 convert to double exactly either way
__device__ __forceinline__ void interior_state(const double* a, const double* b, I j, I n, double* s) {
  const double n_interp_div = 1.0 / (double)(n + 1);
  se3_interpolate(a, b, (double)j * n_interp_div, s);
}
// State j (1 .. nd) DiscreteMotionValidator::checkMotion visits on nd segments: interpolate(a, b, j / nd), and b itself
// for j = nd.
template <typename I>
__device__ __forceinline__ void segment_state(const double* a, const double* b, I j, I nd, double* s) {
  if (j == nd) {
#pragma unroll
    for (int k = 0; k < 7; ++k) s[k] = b[k];
  } else {
    se3_interpolate(a, b, (double)j / (double)nd, s);
  }
}

// The edge that flat index `item` belongs to, over the exclusive prefix sums off[0 .. n] of the edges' item counts: the
// largest e < n with off[e] <= item (off is non-decreasing, off[0] = 0). Ldg reads off through the read-only cache, which
// is only right when nothing writes off during the kernel.
template <bool Ldg>
__device__ __forceinline__ uint32_t edge_of_item(const uint32_t* off, uint32_t n, uint32_t item) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if ((Ldg ? __ldg(off + mid) : off[mid]) <= item) lo = mid; else hi = mid;
  }
  return lo;
}

// The number of leading valid verdicts among an edge's n (n when the whole edge is valid).
__device__ __forceinline__ uint32_t leading_valid(const uint8_t* valid, uint32_t n) {
  uint32_t p = 0;
  while (p < n && valid[p]) ++p;
  return p;
}

// ---- Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11) -------------------------
__host__ __device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k0, n1 = (uint32_t)p1;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k1, n3 = (uint32_t)p0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}

// getYawFromSO3 (utils.h:80-88) of the quaternion of SE(3) state s: double atan2, returned as `Scalar` = float. On the host
// atan2 is libm's, on the device CUDA's.
__host__ __device__ __forceinline__ float so3_yaw(const double* s) {
  return (float)atan2(2 * (s[6] * s[5] + s[3] * s[4]), 1 - 2 * (s[4] * s[4] + s[5] * s[5]));
}

// Box pose in heightfield space + AABB + zone.
struct BoxCtx {
  float R1[9];   // rows: -R.row0, R.row2, R.row1 of the orthogonalised box rotation (3x3, row-major)
  float P[3];    // box centre in heightfield space
  float side[3];
  float minB, maxB;
  int x0, x1, z0, z1;
};

// Height of code c of the compact range tables. The host builds the codes with this same function (both sides are
// compiled without FMA contraction): c * step is exact, and the rounded sum is non-decreasing in c, so every bound
// the codes state holds by construction.
constexpr uint32_t kCodeMax = 32765;    // largest code of a finite max; the host picks cstep so that dec(kCodeMax) >= max
constexpr uint32_t kCodeNone = 32767;   // reserved: a max above dec(kCodeMax) / a window without a finite min
__host__ __device__ __forceinline__ float code_dec(float base, float step, uint32_t c) { return base + (float)c * step; }
__host__ __device__ __forceinline__ uint32_t code_word(uint32_t cM, uint32_t cm, uint32_t flags) {
  return (cM << 17) | (cm << 2) | flags;
}
// A zone's codes from its windows' words: the max code is the top field, so it is the top field of the words' unsigned max;
// the min code over the words' low 17 bits (min code and flags) is the min code of their minimum; the flags reduce by OR.
__device__ __forceinline__ uint32_t code_max(uint32_t max_of_words) { return max_of_words >> 17; }
__device__ __forceinline__ uint32_t code_min_key(uint32_t w) { return w & 0x1FFFFu; }
__device__ __forceinline__ uint32_t code_min(uint32_t min_of_keys) { return min_of_keys >> 2; }
__device__ __forceinline__ uint32_t code_flags(uint32_t or_of_words) { return or_of_words & 3u; }

// nextafterf(x, -inf) / nextafterf(x, +inf) for finite x (dNextAfter, ode/include/ode/common.h:296), as integer ops.
__device__ __forceinline__ float next_down(float x) {
  if (x == 0.0f) return __int_as_float(0x80000001);
  return __int_as_float(__float_as_int(x) + ((x > 0.0f) ? -1 : 1));
}
__device__ __forceinline__ float next_up(float x) {
  if (x == 0.0f) return __int_as_float(0x00000001);
  return __int_as_float(__float_as_int(x) + ((x > 0.0f) ? 1 : -1));
}

// 1.0f / sqrtf(x) as two correctly rounded operations; __frcp_rn(y) is the correctly rounded 1/y, i.e. bit-identical to
// __fdiv_rn(1.0f, y), in fewer instructions.
__device__ __forceinline__ float rsqrt_exact(float x) { return __frcp_rn(__fsqrt_rn(x)); }

// dxSafeNormalize3, ode/ode/src/odemath.cpp:95-161: scale by the largest component m, then u = lower-index other
// component / m, v = higher-index other component / m, l = 1 / sqrt(1 + u*u + v*v). Written without a branch per
// largest-component case (which component is largest depends on the yaw, so a warp would run all three copies): the
// operands are selected, the arithmetic is the same sequence of correctly rounded operations.
__device__ __forceinline__ void safe_normalize3(float& a0, float& a1, float& a2) {
  const float b0 = fabsf(a0), b1 = fabsf(a1), b2 = fabsf(a2);
  int idx;
  if (b1 > b0) idx = (b2 > b1) ? 2 : 1;
  else if (b2 > b0) idx = 2;
  else { if (!(b0 > 0.0f)) return; idx = 0; }
  const float bm = idx == 0 ? b0 : (idx == 1 ? b1 : b2);
  const float am = idx == 0 ? a0 : (idx == 1 ? a1 : a2);
  const float au = idx == 0 ? a1 : a0, av = idx == 2 ? a1 : a2;
  const float r = __fdiv_rn(1.0f, bm);
  const float u = au * r, v = av * r;
  const float l = rsqrt_exact(1.0f + u * u + v * v);
  const float nu = u * l, nv = v * l, nm = copysignf(l, am);
  a0 = idx == 0 ? nm : nu;
  a1 = idx == 1 ? nm : (idx == 0 ? nu : nv);
  a2 = idx == 2 ? nm : nv;
}

// dBodySetRotation -> dxOrthogonalizeR (ode/ode/src/ode.cpp:358-374, odemath.cpp:260-313) on the 3x3
// row-major m; quirk kept: with proj != 0 the Gram-Schmidt row goes to a temporary, stored row 1 untouched.
__device__ __forceinline__ void orthogonalize_r(float m[9]) {
  if (!(m[0] != 0.0f || m[1] != 0.0f || m[2] != 0.0f)) return;
  const float n0 = m[0] * m[0] + m[1] * m[1] + m[2] * m[2];
  float r0 = m[3], r1 = m[4], r2 = m[5];
  const float proj = m[0] * m[3] + m[1] * m[4] + m[2] * m[5];
  const bool tmp = (proj != 0.0f);
  if (tmp) {
    const float pd = __fdiv_rn(proj, n0);
    r0 = m[3] - pd * m[0];
    r1 = m[4] - pd * m[1];
    r2 = m[5] - pd * m[2];
  }
  if (!(r0 != 0.0f || r1 != 0.0f || r2 != 0.0f)) return;
  if (n0 != 1.0f) safe_normalize3(m[0], m[1], m[2]);
  const float n1 = r0 * r0 + r1 * r1 + r2 * r2;
  if (n1 != 1.0f) safe_normalize3(r0, r1, r2);
  if (!tmp) { m[3] = r0; m[4] = r1; m[5] = r2; }   // alias case: row 1 normalised in place
  m[6] = m[1] * r2 - m[2] * r1;                      // dCalcVectorCross3(row2, row0, row1')
  m[7] = m[2] * r0 - m[0] * r2;
  m[8] = m[0] * r1 - m[1] * r0;
}

// Eigen::Quaternion<float>(w,x,y,z).toRotationMatrix() on double->float casts (utils.h:25-38).
__device__ __forceinline__ void pose3_from_se3(const double* __restrict__ s, float t[3], float R[9]) {
  t[0] = (float)s[0]; t[1] = (float)s[1]; t[2] = (float)s[2];
  const float x = (float)s[3], y = (float)s[4], z = (float)s[5], w = (float)s[6];
  const float tx = 2.0f * x, ty = 2.0f * y, tz = 2.0f * z;
  const float twx = tx * w, twy = ty * w, twz = tz * w;
  const float txx = tx * x, txy = ty * x, txz = tz * x;
  const float tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1.0f - (tyy + tzz); R[1] = txy - twz;          R[2] = txz + twy;
  R[3] = txy + twz;          R[4] = 1.0f - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;          R[7] = tyz + twx;          R[8] = 1.0f - (txx + tyy);
}

// (pose * Pose3FromXYZ(o)).translation(): R*o + t, 3-term dot reduced as a0 + (a1 + a2) (Eigen redux).
__device__ __forceinline__ void compose_translation(const float R[9], const float t[3], float o0, float o1,
                                                    float o2, float out[3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float a0 = R[3 * i] * o0, a1 = R[3 * i + 1] * o1, a2 = R[3 * i + 2] * o2;
    out[i] = (a0 + (a1 + a2)) + t[i];
  }
}

// grid_map checkIfPositionWithinMap (double).
__device__ __forceinline__ bool is_inside(const Checker& c, float px, float py) {
  const double tx = -(((double)px - c.cx) - 0.5 * c.Lx);
  const double ty = -(((double)py - c.cy) - 0.5 * c.Ly);
  return tx >= 0.0 && ty >= 0.0 && tx < c.Lx && ty < c.Ly;
}

// Half extent of a box along heightfield axis a (0 x, 1 y, 2 z): row a of R1 against the sides (dxBox::computeAABB,
// box.cpp:60-77).
__device__ __forceinline__ float box_half_extent(const float R1[9], const float side[3], int a) {
  return 0.5f * (fabsf(R1[3 * a] * side[0]) + fabsf(R1[3 * a + 1] * side[1]) + fabsf(R1[3 * a + 2] * side[2]));
}

// Corner `corner` of the box in heightfield space: bit j of `corner` picks +side_j / 2 (set) or -side_j / 2 along box
// axis j, added to the centre axis by axis.
__device__ __forceinline__ void box_corner(const BoxCtx& b, int corner, float p[3]) {
  float px = b.P[0], py = b.P[1], pz = b.P[2];
  const float h0 = 0.5f * b.side[0], h1 = 0.5f * b.side[1], h2 = 0.5f * b.side[2];
  if (corner & 1) { px += h0 * b.R1[0]; py += h0 * b.R1[3]; pz += h0 * b.R1[6]; } else { px -= h0 * b.R1[0]; py -= h0 * b.R1[3]; pz -= h0 * b.R1[6]; }
  if (corner & 2) { px += h1 * b.R1[1]; py += h1 * b.R1[4]; pz += h1 * b.R1[7]; } else { px -= h1 * b.R1[1]; py -= h1 * b.R1[4]; pz -= h1 * b.R1[7]; }
  if (corner & 4) { px += h2 * b.R1[2]; py += h2 * b.R1[5]; pz += h2 * b.R1[8]; } else { px -= h2 * b.R1[2]; py -= h2 * b.R1[5]; pz -= h2 * b.R1[8]; }
  p[0] = px; p[1] = py; p[2] = pz;
}

// dGeomBoxPointDepth(v) > dEpsilon (ode/ode/src/box.cpp:109-173): depth > eps  <=>  all six face
// distances > eps (outside => depth <= 0; inside => depth = min of the six).
__device__ __forceinline__ bool vertex_inside(const BoxCtx& b, float vx, float vy, float vz) {
  const float p0 = vx - b.P[0], p1 = vy - b.P[1], p2 = vz - b.P[2];
  const float q0 = b.R1[0] * p0 + b.R1[3] * p1 + b.R1[6] * p2;   // dMultiply1_331
  const float q1 = b.R1[1] * p0 + b.R1[4] * p1 + b.R1[7] * p2;
  const float q2 = b.R1[2] * p0 + b.R1[5] * p1 + b.R1[8] * p2;
  const float s0 = b.side[0] * 0.5f, s1 = b.side[1] * 0.5f, s2 = b.side[2] * 0.5f;
  return (s0 - q0 > ARTP_EPS) && (s0 + q0 > ARTP_EPS) && (s1 - q1 > ARTP_EPS) && (s1 + q1 > ARTP_EPS) &&
         (s2 - q2 > ARTP_EPS) && (s2 + q2 > ARTP_EPS);
}

// Plane of a heightfield triangle (ode/ode/src/heightfield.cpp:1474-1501).
// v0 = vertices[0], v1 = vertices[1], v2 = vertices[2]; Up: (A,B,C), Down: (D,B,C).
__device__ __forceinline__ void tri_plane(bool isUp, float v0x, float v0y, float v0z, float v1x, float v1y,
                                          float v1z, float v2x, float v2y, float v2z, float pl[4]) {
  const float e1x = v2x - v0x, e1y = v2y - v0y, e1z = v2z - v0z;   // Edge1 = v2 - v0
  const float e2x = v1x - v0x, e2y = v1y - v0y, e2z = v1z - v0z;   // Edge2 = v1 - v0
  float ax, ay, az, bx, by, bz;
  if (isUp) { ax = e1x; ay = e1y; az = e1z; bx = e2x; by = e2y; bz = e2z; }
  else      { ax = e2x; ay = e2y; az = e2z; bx = e1x; by = e1y; bz = e1z; }
  float c0 = ay * bz - az * by;
  float c1 = az * bx - ax * bz;
  float c2 = ax * by - ay * bx;
  const float inv = rsqrt_exact(c0 * c0 + c1 * c1 + c2 * c2);
  c0 *= inv; c1 *= inv; c2 *= inv;
  pl[0] = c0; pl[1] = c1; pl[2] = c2;
  pl[3] = c0 * v0x + c1 * v0y + c2 * v0z;
}

__device__ __forceinline__ bool plane_match(const float a[4], const float b[4]) {   // heightfield.cpp:1541-1546
  return fabsf(a[1] - b[1]) < ARTP_EPS && fabsf(a[3] - b[3]) < ARTP_EPS && fabsf(a[0] - b[0]) < ARTP_EPS &&
         fabsf(a[2] - b[2]) < ARTP_EPS;
}

// dCollideBoxPlane (ode/ode/src/box.cpp:745-878) with maxc clamped to `maxc` (1 or 4): contact positions.
// cx/cz receive the X and Z of each contact (Y is never used by IsOnHeightfield2).
__device__ __forceinline__ int box_plane(const BoxCtx& b, const float n[4], int maxc, float cx[4], float cz[4]) {
  const float* R = b.R1;
  const float Q1 = n[0] * R[0] + n[1] * R[3] + n[2] * R[6];
  const float Q2 = n[0] * R[1] + n[1] * R[4] + n[2] * R[7];
  const float Q3 = n[0] * R[2] + n[1] * R[5] + n[2] * R[8];
  const float A1 = b.side[0] * Q1, A2 = b.side[1] * Q2, A3 = b.side[2] * Q3;
  const float B1 = fabsf(A1), B2 = fabsf(A2), B3 = fabsf(A3);
  const float depth = n[3] + 0.5f * (B1 + B2 + B3) - (n[0] * b.P[0] + n[1] * b.P[1] + n[2] * b.P[2]);
  if (depth < 0.0f) return 0;
  float px = b.P[0], pz = b.P[2];
  {
    const float h0 = 0.5f * b.side[0], h1 = 0.5f * b.side[1], h2 = 0.5f * b.side[2];
    if (A1 > 0.0f) { px -= h0 * R[0]; pz -= h0 * R[6]; } else { px += h0 * R[0]; pz += h0 * R[6]; }
    if (A2 > 0.0f) { px -= h1 * R[1]; pz -= h1 * R[7]; } else { px += h1 * R[1]; pz += h1 * R[7]; }
    if (A3 > 0.0f) { px -= h2 * R[2]; pz -= h2 * R[8]; } else { px += h2 * R[2]; pz += h2 * R[8]; }
  }
  cx[0] = px; cz[0] = pz;
  int ret = 1;
  if (maxc == 1) return ret;
  int first, second;
  if (B1 < B2) {
    if (B3 < B1) { first = 2; second = 0; }
    else         { first = 0; second = (B2 < B3) ? 1 : 2; }
  } else {
    if (B3 < B2) { first = 2; second = 1; }
    else         { first = 1; second = (B1 < B3) ? 0 : 2; }
  }
  float d1 = 0.0f, d2 = 0.0f;
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const int j = (c == 0) ? first : second;
    const float Bj = (j == 0) ? B1 : (j == 1 ? B2 : B3);
    const float Aj = (j == 0) ? A1 : (j == 1 ? A2 : A3);
    const float sj = (j == 0) ? b.side[0] : (j == 1 ? b.side[1] : b.side[2]);
    const float rx = (j == 0) ? R[0] : (j == 1 ? R[1] : R[2]);
    const float rz = (j == 0) ? R[6] : (j == 1 ? R[7] : R[8]);
    if (depth - Bj < 0.0f) break;
    if (Aj > 0.0f) { cx[ret] = px + sj * rx; cz[ret] = pz + sj * rz; }
    else           { cx[ret] = px - sj * rx; cz[ret] = pz - sj * rz; }
    if (c == 0) d1 = depth - Bj; else d2 = depth - Bj;
    ret++;
  }
  if (ret == 3) {
    const float d4 = d1 + d2 - depth;
    if (d4 > 0.0f) {
      cx[3] = cx[1] + cx[2] - px;
      cz[3] = cz[1] + cz[2] - pz;
      ret++;
    }
  }
  return ret;
}

// dxHeightfieldData::IsOnHeightfield2 (ode/ode/src/heightfield.cpp:264-321). (cx,cz): integer coords of the
// triangle's first vertex (A for Up, D for Down).
__device__ __forceinline__ bool on_tri(const Field& f, bool isUp, int cx, int cz, float X, float Z) {
  // Up:   MinX = cx*sW,     MaxX = (cx+1)*sW, ... inside && (MaxZ - Z) >  (X - MinX) * asp
  // Down: MinX = (cx-1)*sW, MaxX = cx*sW,     ... inside && (MaxZ - Z) <= (X - MinX) * asp
  // written without an isUp branch (same products, same comparisons) so mixed warps do not diverge.
  const int lx = isUp ? cx : cx - 1, lz = isUp ? cz : cz - 1;
  const float MinX = lx * f.sW, MaxX = (lx + 1) * f.sW, MinZ = lz * f.sD, MaxZ = (lz + 1) * f.sD;
  const bool inside = (X >= MinX) && (X < MaxX) && (Z >= MinZ) && (Z < MaxZ);
  const bool above = (MaxZ - Z) > (X - MinX) * f.asp;
  return inside && (isUp ? above : !above);
}

__device__ __forceinline__ bool finitef(float h) { return fabsf(h) < CUDART_INF_F; }   // no NaN by contract

// Heights of the four corners of cell (cx, cz): A(x,z) B(x+1,z) C(x,z+1) D(x+1,z+1).
__device__ __forceinline__ void load_cell(const Field& f, int cx, int cz, float& hA, float& hB, float& hC, float& hD) {
  const float* p = f.H + (size_t)cz * f.pitch + cx;
  hA = __ldg(p); hB = __ldg(p + 1); hC = __ldg(p + f.pitch); hD = __ldg(p + f.pitch + 1);
}

// Exact plane of the Up / Down triangle of cell (cx, cz).
__device__ __forceinline__ void cell_plane(const Field& f, bool isUp, int cx, int cz, float hA, float hB, float hC,
                                           float hD, float pl[4]) {
  const float xA = cx * f.sW, xB = (cx + 1) * f.sW, zA = cz * f.sD, zC = (cz + 1) * f.sD;
  // (A, B, C) or (D, B, C): one instruction stream for both (lanes holding an Up and a Down triangle do not diverge)
  tri_plane(isUp, isUp ? xA : xB, isUp ? hA : hD, isUp ? zA : zC, xB, hB, zA, xA, hC, zC, pl);
}

// Bucket keys of the plane screens and of the map's plane tables: nkey buckets a normal component (n0 or n2, in [-1, 1]),
// dkey a plane offset d. A key shifted by a margin is the key of the shifted component, e.g. nkey(n0 - kKeyMargin).
constexpr float kKeyScale = 16384.0f;   // bucket width 2^-14 on n0, n2 in [-1, 1]
constexpr float kKeyMargin = 4e-6f;     // > eps + rsqrt.approx error + quantisation error (see DESIGN.md)
constexpr float kDScale = 524288.0f;    // bucket width 2^-19 on d (> 2 eps, so |d_m - d_c| < eps spans <= 2 buckets)
__device__ __forceinline__ int nkey(float n) { return (int)floorf((n + 1.0f) * kKeyScale); }
__device__ __forceinline__ int dkey(float d) { return (int)floorf(fminf(fmaxf(d, -2000.0f), 2000.0f) * kDScale); }

}  // namespace artp
