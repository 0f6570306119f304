// artp_sampler.cuh -- SE3FromSE2Sampler::sampleUniform (art_planner/src/sampler.cpp:40-131) on the device.
//
// The reference draws one state at a time from OMPL's RNG (std::mt19937) and walks the two CDF layers linearly.
// Here one thread produces one candidate from six uniform01 variates, either given by the caller (parity tests feed
// the same variates to the CPU oracle) or generated in place by a counter-based generator (Philox4x32-10 keyed by
// (seed, sample index)), so that sample -> check -> compact runs without any host->device pose stream.
//
// All arithmetic is double, in the order the reference (and Eigen's Quaternion code it calls) evaluates it; this
// translation unit is compiled with -fmad=false. sin/cos/acos/atan2 are CUDA's (<= 2 ulp from libm), so states agree
// with the CPU restatement to ~1e-15 relative, the sampled cell (row, col) exactly.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "artp_device.cuh"

namespace artp {

constexpr uint32_t kSamplerTag = 0x41525450u;   // "ARTP": separates this stream from any other use of the key

// The six uniform01 doubles of sample `idx` under `seed`: words of Philox blocks (idx, b), b = 0..2; each double is
// the top 53 bits of (w[2k+1] << 32 | w[2k]) scaled by 2^-53 -> [0, 1).
__host__ __device__ __forceinline__ void sampler_uniforms(uint64_t seed, uint64_t idx, double u[6]) {
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    uint32_t c[4] = {(uint32_t)idx, (uint32_t)(idx >> 32), (uint32_t)b, kSamplerTag};
    philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
    u[2 * b] = (double)((((uint64_t)c[1] << 32) | c[0]) >> 11) * (1.0 / 9007199254740992.0);
    u[2 * b + 1] = (double)((((uint64_t)c[3] << 32) | c[2]) >> 11) * (1.0 / 9007199254740992.0);
  }
}

// First index i in [0, n-2] with (double)c[i*stride] > u, else n-1: what the linear scans of sampler.cpp:66-71 return.
// c is non-decreasing or entirely NaN (validated by artp_set_sampler), so a binary search finds the same index.
__device__ __forceinline__ int cdf_search(const float* __restrict__ c, size_t stride, int n, double u) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if ((double)__ldg(c + (size_t)mid * stride) > u) hi = mid; else lo = mid + 1;
  }
  return lo;
}

__device__ __forceinline__ void cross3d(const double a[3], const double b[3], double o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

// grid_map::getIndexFromPosition + checkIfPositionWithinMap (sampler.cpp:91, map.cpp:78): the cell (row, col) of a
// position; false when the position lies outside the map or its index out of range.
__device__ __forceinline__ bool map_cell(const SamplerDev& m, double px, double py, int& row, int& col) {
  const double Lx = m.rows * m.res, Ly = m.cols * m.res;
  const double vx = ((px - 0.5 * Lx) - m.cx) / m.res, vy = ((py - 0.5 * Ly) - m.cy) / m.res;
  row = (int)(-vx);
  col = (int)(-vy);
  const double tx = -((px - m.cx) - 0.5 * Lx), ty = -((py - m.cy) - 0.5 * Ly);
  const bool inside = tx >= 0.0 && ty >= 0.0 && tx < Lx && ty < Ly;
  return inside && row >= 0 && col >= 0 && row < m.rows && col < m.cols;
}

// The elevation of cell (row, col) (map.cpp getHeightAtIndex, sampler.cpp:93-95).
__device__ __forceinline__ double cell_height(const SamplerDev& m, int row, int col) {
  return (double)__ldg(m.elevation_rev + (size_t)row + (size_t)(m.cols - 1 - col) * m.pitch);
}

// Quaterniond(AngleAxisd(yaw, UnitZ)).inverse() * normal_w (sampler.cpp:118-121, map.cpp:84-87), in the order Eigen
// evaluates it.
__device__ __forceinline__ void normal_in_yaw_frame(double yaw, const double nw[3], double nb[3]) {
  double sn, cs;
  sincos(0.5 * yaw, &sn, &cs);
  const double q[4] = {sn * 0.0, sn * 0.0, sn * 1.0, cs};
  const double n2 = (q[0] * q[0] + q[2] * q[2]) + (q[1] * q[1] + q[3] * q[3]);
  const double qi[3] = {-q[0] / n2, -q[1] / n2, -q[2] / n2}, qw = q[3] / n2;
  double uv[3], t2[3];
  cross3d(qi, nw, uv);
  uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
  cross3d(qi, uv, t2);
#pragma unroll
  for (int k = 0; k < 3; ++k) nb[k] = (nw[k] + qw * uv[k]) + t2[k];
}

// setSO3FromRPY (utils.h:101-115): q = (qx, qy, qz, qw), the state's fields 3..6.
__device__ __forceinline__ void so3_from_rpy(double roll, double pitch, double yaw, double q[4]) {
  double cr, sr, cp, sp, cy, sy;
  sincos(roll * 0.5, &sr, &cr);
  sincos(pitch * 0.5, &sp, &cp);
  sincos(yaw * 0.5, &sy, &cy);
  q[3] = cy * cp * cr + sy * sp * sr;
  q[0] = cy * cp * sr - sy * sp * cr;
  q[1] = sy * cp * sr + cy * sp * cr;
  q[2] = sy * cp * cr - cy * sp * sr;
}

// One candidate. Returns false (state = NaN, row = col = -1) when the position is outside the map: only possible in
// uniform mode, where the reference loop (sampler.cpp:46-50) would draw again.
__device__ __forceinline__ bool sample_state(const SamplerDev& m, const double u[6], double s[7], int& row, int& col) {
  double pos[2];
  const double Lx = m.rows * m.res, Ly = m.cols * m.res;
  if (m.from_distribution) {                                   // samplePositionInMapFromDist, sampler.cpp:54-77
    const int r = cdf_search(m.cum_row, 1, m.rows, u[1]);
    const int c = cdf_search(m.cum_prob + r, (size_t)m.rows, m.cols, u[0]);
    // grid_map::getPositionFromIndex
    pos[0] = (m.cx + (0.5 * Lx - 0.5 * m.res)) + m.res * (-(double)r);
    pos[1] = (m.cy + (0.5 * Ly - 0.5 * m.res)) + m.res * (-(double)c);
  } else {                                                     // samplePositionInMap: uniformReal(a,b) = (b-a)*u + a
    pos[0] = (m.high[0] - m.low[0]) * u[0] + m.low[0];
    pos[1] = (m.high[1] - m.low[1]) * u[1] + m.low[1];
  }
  if (!map_cell(m, pos[0], pos[1], row, col)) {
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);
#pragma unroll
    for (int k = 0; k < 7; ++k) s[k] = qnan;
    row = col = -1;
    return false;
  }
  const size_t at = (size_t)row + (size_t)col * m.rows;
  double x = pos[0], y = pos[1];
  double z = cell_height(m, row, col);
  const double nw[3] = {(double)__ldg(m.normal_x + at), (double)__ldg(m.normal_y + at), (double)__ldg(m.normal_z + at)};
  const float sd = __ldg(m.std_dev + at);
  const double pert = ((2.0 * u[2] + -1.0) * (double)(sd < 0.5f ? sd : 0.5f)) * m.reach_z;          // :103
  x += nw[0] * pert; y += nw[1] * pert; z += nw[2] * pert;
  // RNG::eulerRPY (OMPL RandomNumbers.cpp)
  const double pi = 3.14159265358979323846;
  double v0 = pi * (-2.0 * u[3] + 1.0);
  double v1 = acos(1.0 - 2.0 * u[4]) - pi / 2.0;
  const double v2 = pi * (-2.0 * u[5] + 1.0);
  double nb[3];
  normal_in_yaw_frame(v2, nw, nb);
  v0 = -atan2(nb[1], nb[2]) + v0 * m.max_roll_pert / 1.57079632679489661923;      // :123-124 (M_PI_2)
  v1 = atan2(nb[0], nb[2]) + v1 * m.max_pitch_pert / 0.78539816339744830962;      // :125-126 (M_PI_4)
  s[0] = x; s[1] = y; s[2] = z;
  so3_from_rpy(v0, v1, v2, s + 3);
  return true;
}

// Map::get3DPoseFrom2D as Planner::plan applies it to the goal (planner.cpp:223-237, map.cpp:77-90): for a state whose
// (x, y) lies on the map, z = the cell's elevation, roll / pitch from the cell's normal seen in the state's yaw frame,
// yaw = getYawFromSO3 (utils.h:80-88: double atan2 returned as float); x and y stay. Other states pass unchanged.
__device__ __forceinline__ bool pose_from_2d(const SamplerDev& m, const double in[7], double out[7]) {
#pragma unroll
  for (int k = 0; k < 7; ++k) out[k] = in[k];
  int row, col;
  if (!map_cell(m, in[0], in[1], row, col)) return false;
  const size_t at = (size_t)row + (size_t)col * m.rows;
  const double nw[3] = {(double)__ldg(m.normal_x + at), (double)__ldg(m.normal_y + at), (double)__ldg(m.normal_z + at)};
  const double yaw = (double)so3_yaw(in);
  double nb[3];
  normal_in_yaw_frame(yaw, nw, nb);
  out[2] = cell_height(m, row, col);
  so3_from_rpy(-atan2(nb[1], nb[2]), atan2(nb[0], nb[2]), yaw, out + 3);
  return true;
}

__global__ void pose_from_2d_kernel(SamplerDev m, const double* __restrict__ in, size_t n, double* __restrict__ out,
                                    uint8_t* __restrict__ inside) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    double s[7], o[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) s[k] = in[i * 7 + k];
    const bool ok = pose_from_2d(m, s, o);
#pragma unroll
    for (int k = 0; k < 7; ++k) out[i * 7 + k] = o[k];
    if (inside) inside[i] = ok ? 1 : 0;
  }
}

// ---- StartState / GoalStateRegion::sampleGoal (start.cpp:7-41, goal.cpp:11-41) --------------------------------------
// The reference repairs a start or goal by rejection sampling in a disc: candidate 0 is the centre, candidate k = 1..n_iter
// the centre moved by the k-th offset of rng_.uniformInBall(radius) in x and y (z and the rotation stay), and the first
// valid candidate wins. OMPL's stream (a serial mt19937) cannot be reproduced here, so offsets are either given or drawn
// from the counter-based stream Philox4x32-10(key = seed, counter = (draw lo, draw hi, query, "ARTB")): the same
// distribution as uniformInBall in 2-D (uniform direction, radius r * sqrt(u)), not the same numbers.
constexpr uint32_t kBallTag = 0x41525442u;   // "ARTB"

// Offset of draw `draw` (the stream position) of query q: u0, u1 from one Philox block as in sampler_uniforms.
__host__ __device__ __forceinline__ void ball_offset(uint64_t seed, uint64_t draw, uint32_t q, double r, double off[2]) {
  uint32_t c[4] = {(uint32_t)draw, (uint32_t)(draw >> 32), q, kBallTag};
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  const double u0 = (double)((((uint64_t)c[1] << 32) | c[0]) >> 11) * (1.0 / 9007199254740992.0);
  const double u1 = (double)((((uint64_t)c[3] << 32) | c[2]) >> 11) * (1.0 / 9007199254740992.0);
  const double rr = r * sqrt(u1);
  double sn, cs;
  sincos(2.0 * 3.14159265358979323846 * u0, &sn, &cs);
  off[0] = rr * cs;
  off[1] = rr * sn;
}

// Per-call parameters of the disc search: n queries of n_iter + 1 candidates each (candidate k of query q is item
// q * (n_iter + 1) + k). offsets != null: n x n_iter x 2 given offsets; else the Philox stream from first_draw.
struct BallSearch {
  const double* centres;   // n x 7
  const double* radius;    // n
  const double* offsets;   // n x n_iter x 2, or null
  uint64_t seed, first_draw;
  uint32_t n_iter;
};

// Candidate k of query q: the centre, or the centre moved by offset k (a double add in x and y).
__device__ __forceinline__ void ball_candidate(const BallSearch& b, uint32_t q, uint32_t k, double s[7]) {
#pragma unroll
  for (int j = 0; j < 7; ++j) s[j] = b.centres[(size_t)q * 7 + j];
  if (k == 0) return;
  double off[2];
  if (b.offsets) {
    const size_t at = ((size_t)q * b.n_iter + (k - 1)) * 2;
    off[0] = b.offsets[at]; off[1] = b.offsets[at + 1];
  } else {
    ball_offset(b.seed, b.first_draw + (k - 1), q, b.radius[q], off);
  }
  s[0] = s[0] + off[0];
  s[1] = s[1] + off[1];
}

// The candidates [c0, c0 + m) as float states (the cast Pose3FromSE3 applies first), the form the pipeline consumes.
__global__ void ball_candidates_kernel(BallSearch b, uint64_t c0, size_t m, float* __restrict__ states_f32) {
  const uint64_t per = (uint64_t)b.n_iter + 1;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < m; i += (size_t)gridDim.x * blockDim.x) {
    const uint64_t g = c0 + i;
    double s[7];
    ball_candidate(b, (uint32_t)(g / per), (uint32_t)(g % per), s);
#pragma unroll
    for (int k = 0; k < 7; ++k) states_f32[i * 7 + k] = (float)s[k];
  }
}

// First valid candidate per query: the smallest valid k wins, whichever chunk it came from.
__global__ void ball_first_valid_kernel(const uint8_t* __restrict__ valid, uint64_t c0, size_t m, uint32_t n_iter,
                                        uint32_t* __restrict__ best) {
  const uint64_t per = (uint64_t)n_iter + 1;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < m; i += (size_t)gridDim.x * blockDim.x) {
    if (!valid[i]) continue;
    const uint64_t g = c0 + i;
    atomicMin(best + g / per, (uint32_t)(g % per));
  }
}

// The chosen candidate of each query, or candidate n_iter (the last one drawn, which the reference leaves in the state
// when no candidate is valid) with index -1.
__global__ void ball_result_kernel(BallSearch b, size_t n, const uint32_t* __restrict__ best, double* __restrict__ states,
                                   int32_t* __restrict__ index) {
  for (size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x; q < n; q += (size_t)gridDim.x * blockDim.x) {
    const uint32_t k = best[q];
    const bool found = k <= b.n_iter;
    double s[7];
    ball_candidate(b, (uint32_t)q, found ? k : b.n_iter, s);
#pragma unroll
    for (int j = 0; j < 7; ++j) states[q * 7 + j] = s[j];
    index[q] = found ? (int32_t)k : -1;
  }
}

__global__ void ball_offsets_kernel(uint64_t seed, uint64_t first_draw, size_t n, uint32_t n_iter, const double* __restrict__ radius,
                                    double* __restrict__ out) {
  const size_t total = n * (size_t)n_iter;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t q = i / n_iter, k = i - q * n_iter;
    ball_offset(seed, first_draw + k, (uint32_t)q, radius[q], out + 2 * i);
  }
}

__global__ void sampler_uniforms_kernel(uint64_t seed, uint64_t first, size_t n, double* __restrict__ u_out) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    double u[6];
    sampler_uniforms(seed, first + i, u);
#pragma unroll
    for (int k = 0; k < 6; ++k) u_out[i * 6 + k] = u[k];
  }
}

// u_in != null: variates from the caller; else Philox(seed, first + i). rowcol (nullable): n x 2 ints.
// states_f32 (nullable): the same states cast to float, the form the validity pipeline consumes.
__global__ void sample_states_kernel(SamplerDev m, const double* __restrict__ u_in, uint64_t seed, uint64_t first, size_t n,
                                     double* __restrict__ states, float* __restrict__ states_f32, int32_t* __restrict__ rowcol) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    double u[6], s[7];
    if (u_in) {
#pragma unroll
      for (int k = 0; k < 6; ++k) u[k] = u_in[i * 6 + k];
    } else {
      sampler_uniforms(seed, first + i, u);
    }
    int row, col;
    sample_state(m, u, s, row, col);
    if (states) {
#pragma unroll
      for (int k = 0; k < 7; ++k) states[i * 7 + k] = s[k];
    }
    if (states_f32) {
#pragma unroll
      for (int k = 0; k < 7; ++k) states_f32[i * 7 + k] = (float)s[k];
    }
    if (rowcol) { rowcol[2 * i] = row; rowcol[2 * i + 1] = col; }
  }
}

// A rejected candidate (NaN state) must not reach the validity pipeline as "valid": clear its flag.
__global__ void reject_nan_kernel(const double* __restrict__ states, size_t n, uint8_t* __restrict__ valid) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    if (states[i * 7] != states[i * 7]) valid[i] = 0;
}

// ---- art_planner::estimateNormals (art_planner/src/utils.cpp:213-324) ------------------------------------------
// One thread per cell (row index fastest -> coalesced in the column-major layers). float arithmetic exactly as Eigen
// evaluates the reference's expressions on 3-vectors (not vectorised): cross = (a1*b2 - a2*b1, ...), squaredNorm =
// x*x + (y*y + z*z), normalized() divides by sqrtf when the squared norm is > 0. Built with -fmad=false; sqrtf and
// the divisions are IEEE (nvcc defaults), so the result is bit-identical to the CPU restatement.
struct F3 { float x, y, z; };

__device__ __forceinline__ void en_accumulate(const F3& a, const F3& b, F3& sum) {
  float c0 = a.y * b.z - a.z * b.y;
  float c1 = a.z * b.x - a.x * b.z;
  float c2 = a.x * b.y - a.y * b.x;
  const float z = c0 * c0 + (c1 * c1 + c2 * c2);
  if (z > 0.0f) { const float n = sqrtf(z); c0 /= n; c1 /= n; c2 /= n; }
  sum.x += c0; sum.y += c1; sum.z += c2;
}

__global__ void estimate_normals_kernel(const float* __restrict__ H_rev, int pitch, int rows, int cols, double res, double cx,
                                        double cy, int r_cells, int r_diag, float* __restrict__ nx, float* __restrict__ ny,
                                        float* __restrict__ nz, float* __restrict__ sd) {
  const size_t total = (size_t)rows * cols;
  const double offx = 0.5 * (rows * res) - 0.5 * res, offy = 0.5 * (cols * res) - 0.5 * res;
  for (size_t at = blockIdx.x * (size_t)blockDim.x + threadIdx.x; at < total; at += (size_t)gridDim.x * blockDim.x) {
    const int j = (int)(at / rows), i = (int)(at - (size_t)j * rows);
    // map_3d (:236-249): grid_map::getPosition cast to float, elevation as stored
    auto P = [&](int ii, int jj) {
      F3 p;
      p.x = (float)((cx + offx) + res * (-(double)ii));
      p.y = (float)((cy + offy) + res * (-(double)jj));
      p.z = __ldg(H_rev + (size_t)ii + (size_t)(cols - 1 - jj) * pitch);
      return p;
    };
    const F3 c = P(i, j);
    F3 sum = {0.0f, 0.0f, 0.0f};
    unsigned int n_vec = 0;
    float max_z_diff = 0.0f;
    auto pair = [&](int i1, int j1, int i2, int j2) {
      const F3 p1 = P(i1, j1), p2 = P(i2, j2);
      const F3 vx = {p1.x - c.x, p1.y - c.y, p1.z - c.z}, vy = {p2.x - c.x, p2.y - c.y, p2.z - c.z};
      if (fabsf(vx.z) > max_z_diff) max_z_diff = fabsf(vx.z);
      if (fabsf(vy.z) > max_z_diff) max_z_diff = fabsf(vy.z);
      en_accumulate(vx, vy, sum);
      ++n_vec;
    };
    for (int o = 1; o < r_cells; ++o) {                                  // :260-271
      if (i + o >= rows || j + o >= cols) continue;
      pair(i + o, j, i, j + o);
    }
    for (int o = 1; o < r_cells; ++o) {                                  // :272-282
      if (i - o < 0 || j - o < 0) continue;
      pair(i - o, j, i, j - o);
    }
    for (int o = 1; o < r_diag; ++o) {                                   // :283-297
      if (i + o >= rows || j + o >= cols || i - o < 0) continue;
      pair(i + o, j + o, i - o, j + o);
    }
    for (int o = 1; o < r_diag; ++o) {                                   // :298-312
      if (i - o < 0 || j - o < 0 || i + o >= rows) continue;
      pair(i - o, j - o, i + o, j - o);
    }
    if (n_vec > 0) { const float d = (float)n_vec; sum.x /= d; sum.y /= d; sum.z /= d; }   // :315-317
    sd[at] = max_z_diff;
    const float z = sum.x * sum.x + (sum.y * sum.y + sum.z * sum.z);     // normalize(), :320
    if (z > 0.0f) { const float n = sqrtf(z); sum.x /= n; sum.y /= n; sum.z /= n; }
    nx[at] = sum.x; ny[at] = sum.y; nz[at] = sum.z;
  }
}

// ---- computeCumulativeProbabilityDistribution (probability_distribution.cpp:20-46) ---------------------------
// One thread per row walks its columns left to right (the order of the reference's rowwise sum and of its column-by-
// column cumulation); neighbouring threads touch neighbouring rows of the column-major layer, so every step is one
// coalesced access. row_sum[i] receives the row's probability mass.
__global__ void cdf_rows_kernel(const float* __restrict__ prob, int rows, int cols, float* __restrict__ cum_prob,
                                float* __restrict__ row_sum) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += gridDim.x * blockDim.x) {
    float s = prob[i];
    for (int j = 1; j < cols; ++j) s = s + prob[i + (size_t)j * rows];
    row_sum[i] = s;
    float run = prob[i] / s;
    cum_prob[i] = run;
    for (int j = 1; j < cols; ++j) {
      run = prob[i + (size_t)j * rows] / s + run;
      cum_prob[i + (size_t)j * rows] = run;
    }
  }
}

// Row distribution: sums / total, cumulated (sequential by definition; rows <= a few thousand). One thread.
__global__ void cdf_rowwise_kernel(float* __restrict__ row, int rows) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  float total = row[0];
  for (int i = 1; i < rows; ++i) total = total + row[i];
  float run = row[0] / total;
  row[0] = run;
  for (int i = 1; i < rows; ++i) { run = row[i] / total + run; row[i] = run; }
}

// Every CDF row must be non-decreasing and finite, or entirely NaN (a row without probability mass:
// probability_distribution.cpp:28 divides 0 by 0). bad[0] counts violations. One thread per row / for the row CDF.
__global__ void validate_cdf_kernel(const float* __restrict__ c, int rows, int cols, size_t stride_in_row, size_t stride_row,
                                    unsigned int* __restrict__ bad) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    const float* p = c + (size_t)r * stride_row;
    const float first = p[0];
    bool ok = true;
    if (first != first) {
      for (int k = 1; k < cols && ok; ++k) { const float v = p[(size_t)k * stride_in_row]; ok = (v != v); }
    } else {
      float prev = first;
      ok = isfinite(first);
      for (int k = 1; k < cols && ok; ++k) {
        const float v = p[(size_t)k * stride_in_row];
        ok = isfinite(v) && v >= prev;
        prev = v;
      }
    }
    if (!ok) atomicAdd(bad, 1u);
  }
}

}  // namespace artp
