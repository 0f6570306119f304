// art_planner_b200/csrc/artp_distribution.cuh
// The sampler's probability layer on the device, as Planner::setUpMapProcessors chains it (planner.cpp:39-58) and
// PRMMotionCostMaintainer::sampleGraph re-applies it (prm_motion_cost.cpp:190-193):
//   computeInverseSampleDensity (sample_density.cpp:12-43): vertex histogram, Gaussian blur, max - n
//   applyBaseSampleDistribution (probability_distribution.cpp:9-16): x traversability_sample_filter
//   applyMaxUnknownProbability  (probability_distribution.cpp:50-91): the unknown-space cap
// The traversability sample filter (basic.cpp:110-125) is morph_kernel (artp_basic.cuh); the CDF that follows is
// cdf_rows_kernel / cdf_rowwise_kernel (artp_sampler.cuh).
// Layers are grid_map matrices: column-major rows x cols floats, element (i, j) at [i + j * rows]. This translation unit
// is compiled with -fmad=false: every float / double expression rounds once per operation, in the order written.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "artp_sampler.cuh"

namespace artp {

constexpr int kMaxGaussTaps = 1023;   // largest Gaussian kernel (cells), i.e. half width 511

// getGaussianKernel(ksize, sigma, CV_32F) by distance from the centre: w[t] = coefficient of the taps at -t and +t.
struct GaussTaps {
  int half;
  float w[kMaxGaussTaps / 2 + 1];
};

// grid_map getIndex (isInside + getIndexFromPosition, the same map_cell the sampler uses) of every vertex's (x, y);
// +1 in n_samples (sample_density.cpp:24-31). Off-map and NaN positions are skipped. Counts are exact integers below 2^24,
// so the result does not depend on the order of the atomics.
__global__ void vertex_histogram_kernel(SamplerDev m, const double* __restrict__ states, size_t n, float* __restrict__ n_samples) {
  for (size_t v = blockIdx.x * (size_t)blockDim.x + threadIdx.x; v < n; v += (size_t)gridDim.x * blockDim.x) {
    int row, col;
    if (map_cell(m, states[v * 7], states[v * 7 + 1], row, col)) atomicAdd(n_samples + (size_t)row + (size_t)col * m.rows, 1.0f);
  }
}

// cv::borderInterpolate for BORDER_REFLECT_101, reflecting as often as needed (a map can be smaller than the kernel).
__device__ __forceinline__ int reflect101(int p, int len) {
  if (len == 1) return 0;
  while ((unsigned)p >= (unsigned)len) p = p < 0 ? -p : 2 * len - 2 - p;
  return p;
}

// One pass of the separable blur along one axis of the layer: AXIS 0 along i (contiguous; OpenCV's row filter on the
// cols x rows image the reference hands it, utils.cpp:93-96), AXIS 1 along j. dst = w0 * S0 + sum_{t=1..half} w[t] * (S[t] + S[-t]),
// accumulated in float in increasing t.
template <int AXIS>
__global__ void gauss_pass_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows, int cols, const GaussTaps k) {
  const size_t n = (size_t)rows * cols;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < n; idx += (size_t)gridDim.x * blockDim.x) {
    const int j = (int)(idx / rows), i = (int)(idx - (size_t)j * rows);
    float s = k.w[0] * src[idx];
    for (int t = 1; t <= k.half; ++t) {
      float a, b;
      if (AXIS == 0) {
        a = src[(size_t)j * rows + reflect101(i + t, rows)];
        b = src[(size_t)j * rows + reflect101(i - t, rows)];
      } else {
        a = src[(size_t)reflect101(j + t, cols) * rows + i];
        b = src[(size_t)reflect101(j - t, cols) * rows + i];
      }
      s = s + k.w[t] * (a + b);
    }
    dst[idx] = s;
  }
}

// *max_bits = bits of max |x| (non-negative floats order like their bit patterns). The blurred counts are sums of
// products of non-negative numbers, so this is also max(x), and max |x| <= 1e-5 is Eigen's isZero().
__global__ void abs_max_kernel(const float* __restrict__ x, size_t n, unsigned int* __restrict__ max_bits) {
  unsigned int m = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    m = max(m, __float_as_uint(fabsf(x[i])));
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(max_bits, m);
}

// sample_density.cpp:39-42 + probability_distribution.cpp:10-15: prob = max(n) - n unless n isZero() (then, and without a
// density, the uniform 1); times the filter where one is set.
__global__ void combine_kernel(const float* __restrict__ n_blur, const unsigned int* __restrict__ max_bits,
                               const float* __restrict__ filter, size_t n, float* __restrict__ prob) {
  const float mx = n_blur ? __uint_as_float(*max_bits) : 0.0f;
  const bool density = n_blur && !(mx <= 1e-5f);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float p = density ? mx - n_blur[i] : 1.0f;
    if (filter) p = p * filter[i];
    prob[i] = p;
  }
}

// probability_distribution.cpp:57-71 in a fixed order: per row, the double sums of prob over observed > 0 (known) and
// over the other cells (unknown), left to right. One thread per row.
__global__ void cap_rows_kernel(const float* __restrict__ prob, const float* __restrict__ observed, int rows, int cols,
                                double* __restrict__ known, double* __restrict__ unknown) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += gridDim.x * blockDim.x) {
    double k = 0.0, u = 0.0;
    for (int j = 0; j < cols; ++j) {
      const size_t at = (size_t)i + (size_t)j * rows;
      if (observed[at] > 0.0f) k += (double)prob[at]; else u += (double)prob[at];
    }
    known[i] = k;
    unknown[i] = u;
  }
}

// :73-87: the row sums added in row order, the three-way condition and the two multipliers (double, cast to float as the
// float "prob_unknown_mult" layer stores them): mult[0] known, mult[1] unknown; both 1 when the cap does not apply.
__global__ void cap_mult_kernel(const double* __restrict__ known, const double* __restrict__ unknown, int rows, double max_unknown,
                                float* __restrict__ mult) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  double k = 0.0, u = 0.0;
  for (int i = 0; i < rows; ++i) { k += known[i]; u += unknown[i]; }
  const double base = u / (k + u);
  if (k > 0 && u > 0 && base > max_unknown) {
    mult[0] = (float)((1 - max_unknown) / k);
    mult[1] = (float)(max_unknown / u);
  } else {
    mult[0] = 1.0f;
    mult[1] = 1.0f;
  }
}

// :90: prob *= prob_unknown_mult, in float.
__global__ void cap_apply_kernel(float* __restrict__ prob, const float* __restrict__ observed, const float* __restrict__ mult, size_t n) {
  const float km = mult[0], um = mult[1];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    prob[i] = prob[i] * (observed[i] > 0.0f ? km : um);
}

}  // namespace artp
