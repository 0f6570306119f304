// art_planner_b200/csrc/artp_sampling.cu -- the sampling half of the C ABI (include/artp.h): normals and the CDF, the
// sampler (SE3FromSE2Sampler::sampleUniform) with its fused sample -> check -> compact path, the start / goal search,
// poseFrom2D with the valid-heading and box-verdict layers, Basic's masking and the sampler's distribution. It reaches the
// validity pipeline through check_states_f32 and box_verdicts_f32 (artp_internal.h).
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "artp_internal.h"
#include "artp_sampler.cuh"
#include "artp_basic.cuh"
#include "artp_distribution.cuh"

namespace artp_api {

template <typename T> struct Buf { T* p = nullptr; size_t cap = 0; ~Buf() { cudaFree(p); } };   // for grow / carve; cap counts T

struct Sampling {
  // What belongs to the current map: sampling_forget_map resets it.
  struct MapFlags {
    bool has_sampler = false;
    bool has_device_normals = false;  // artp_estimate_normals filled the normal-plane layers for this map
    bool has_device_cdf = false;      // artp_compute_sample_cdf filled cum_prob / cum_row for this map
    bool has_normals = false;         // the normal-plane layers hold this map's normals (device-estimated or the caller's)
    bool has_sample_filter = false;   // dist_layers holds this map's traversability_sample_filter ...
    bool has_dist_observed = false;   // ... and observed layer
  } map;
  artp::SamplerDev samp{};            // the sampler's view (arm_sampler)
  Buf<float> samp_layers;             // layers kNormalX .. kCumRow
  Buf<char> samp_scratch;             // the fused sample -> check -> compact path and the start / goal search
  Buf<float> dist_layers;             // layers kFilter, kObserved
  Buf<char> dist_scratch;             // the sample filter's and the distribution's chains
  // The Basic-keep state is keyed by the layers' size, not by the map: a new map does not reset it.
  Buf<float> basic_keep;              // layers kBasicObserved, kThresholded
  int basic_rows = 0, basic_cols = 0;
  bool has_basic_layers = false, has_basic_observed = false;
};

}  // namespace artp_api

using namespace artp_api;

namespace {

// A buffer of per-cell layers, ncell floats each in the order of its enum below: L[k] is layer k.
struct Layers {
  float* base; size_t ncell;
  float* operator[](int k) const { return base + k * ncell; }
};
// Sampling::samp_layers: the normal-plane layers, cum_prob, then cum_row (rows floats), with 64 floats of slack.
enum { kNormalX, kNormalY, kNormalZ, kStdDev, kCumProb, kCumRow };
size_t samp_layers_floats(int rows, int cols) { return kCumRow * (size_t)rows * cols + (size_t)rows + 64; }
// Sampling::dist_layers: the current map's traversability_sample_filter and observed layer (artp_set_sample_filter).
enum { kFilter, kObserved, kDistLayers };
// Sampling::basic_keep: the last artp_process_basic's observed and traversability_thresholded layers.
enum { kBasicObserved, kThresholded, kBasicLayers };

Sampling& sampling(Handle* h) {
  if (!h->sampling) h->sampling = new Sampling();
  return *h->sampling;
}
Layers sampler_layers(Handle* h) { return {sampling(h).samp_layers.p, (size_t)h->rows * h->cols}; }

// ---------------------------------------------------------------------------------------------------------------
// Sampler: SE3FromSE2Sampler::sampleUniform on the device (artp_sampler.cuh)
// ---------------------------------------------------------------------------------------------------------------
int ensure_sampler_layers(Handle* h) {
  Sampling& S = sampling(h);
  const size_t need = samp_layers_floats(h->rows, h->cols);
  if (S.samp_layers.cap < need)   // the layers computed on the device go with the old buffer
    S.map.has_device_normals = S.map.has_device_cdf = S.map.has_normals = false;
  return grow(h, S.samp_layers.p, S.samp_layers.cap, need);
}

// The map fields of the sampler's view (geometry, elevation, the normal-plane layers).
void sampler_map_view(Handle* h, artp::SamplerDev& m) {
  const Layers L = sampler_layers(h);
  m.elevation_rev = h->d_H[0]; m.pitch = h->pitch;
  m.normal_x = L[kNormalX]; m.normal_y = L[kNormalY]; m.normal_z = L[kNormalZ]; m.std_dev = L[kStdDev];
  m.rows = h->rows; m.cols = h->cols;
  m.res = h->chk.Lx / h->rows; m.cx = h->chk.cx; m.cy = h->chk.cy;
}

// computeCumulativeProbabilityDistribution of a device-resident probability layer into cum_prob / cum_row
// (ensure_sampler_layers first). Two launches on s.
int launch_sample_cdf(Handle* h, const float* d_prob, cudaStream_t s) {
  const Layers L = sampler_layers(h);
  TRY(launch(h, artp::cdf_rows_kernel, (h->rows + 63) / 64, 64, 0, s, d_prob, h->rows, h->cols, L[kCumProb], L[kCumRow]));
  return launch(h, artp::cdf_rowwise_kernel, 1, 32, 0, s, L[kCumRow], h->rows);
}

// running total += chunk count (device-side, stream ordered)
__global__ void add_count_kernel(uint32_t* total, const uint32_t* chunk) { *total += *chunk; }

// out + 7 * (*total) .. : ordered gather of this chunk's valid candidates behind the previous chunks'
__global__ void gather_chunk_kernel(const double* __restrict__ states, const int64_t* __restrict__ idx,
                                    const uint32_t* __restrict__ chunk_count, const uint32_t* __restrict__ total_before,
                                    size_t capacity, double* __restrict__ out) {
  const size_t before = *total_before;
  const size_t room = capacity > before ? capacity - before : 0;
  const size_t cc = *chunk_count;
  const size_t keep = cc < room ? cc : room;
  const size_t n = keep * 7;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t k = i / 7, c = i - k * 7;
    out[before * 7 + i] = states[(size_t)idx[k] * 7 + c];
  }
}

// draws + (*total) .. : the draw index of each state gather_chunk_kernel keeps, first_draw + its index in the chunk
__global__ void gather_draws_kernel(const int64_t* __restrict__ idx, const uint32_t* __restrict__ chunk_count,
                                    const uint32_t* __restrict__ total_before, size_t capacity, uint64_t first_draw,
                                    uint64_t* __restrict__ draws) {
  const size_t before = *total_before;
  const size_t room = capacity > before ? capacity - before : 0;
  const size_t cc = *chunk_count;
  const size_t keep = cc < room ? cc : room;
  for (size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x; k < keep; k += (size_t)gridDim.x * blockDim.x)
    draws[before + k] = first_draw + (uint64_t)idx[k];
}

constexpr size_t kSampleChunk = (size_t)1 << 21;

// ---------------------------------------------------------------------------------------------------------------
// Start / goal repair: StartState / GoalStateRegion::sampleGoal (start.cpp:7-41, goal.cpp:11-41), and the goal's
// projection onto the map (planner.cpp:223-237, map.cpp:77-90)
// ---------------------------------------------------------------------------------------------------------------
// Argument checks shared by both forms; `radius` only when it is a host buffer.
int ball_search_args(Handle* h, size_t n, uint32_t n_iter, const double* radius) {
  TRY(require_map(h));
  if ((uint64_t)n >= (1ull << 32) || n * ((uint64_t)n_iter + 1) >= (1ull << 32)) {
    h->err = "n * (n_iter + 1) candidates must be < 2^32"; return ARTP_E_INVALID;
  }
  if (radius)
    for (size_t q = 0; q < n; ++q)
      if (!(radius[q] >= 0.0 && std::isfinite(radius[q]))) { h->err = "radius must be finite and >= 0"; return ARTP_E_INVALID; }
  return ARTP_OK;
}

// The search of n > 0 queries on s, in chunks of kSampleChunk candidates; arguments checked by ball_search_args.
int find_valid_near(Handle* h, const double* d_centres, size_t n, const double* d_radius, uint32_t n_iter, const double* d_offsets,
                    uint64_t seed, uint64_t first_draw, double* d_states_out, int32_t* d_index, cudaStream_t s) {
  const uint64_t total = n * ((uint64_t)n_iter + 1);
  const size_t chunk = (size_t)std::min<uint64_t>(total, kSampleChunk);
  char* r[3];   // candidate states f32 | verdicts | first valid candidate per query
  Buf<char>& scratch = sampling(h).samp_scratch;
  TRY(carve(h, scratch.p, scratch.cap, {chunk * 7 * sizeof(float), chunk, n * sizeof(uint32_t)}, r));
  float* d_sf = (float*)r[0];
  uint8_t* d_val = (uint8_t*)r[1];
  uint32_t* d_best = (uint32_t*)r[2];
  artp::BallSearch b{d_centres, d_radius, d_offsets, seed, first_draw, n_iter};
  CU_TRY(h, cudaMemsetAsync(d_best, 0xFF, n * sizeof(uint32_t), s));
  for (uint64_t c0 = 0; c0 < total; c0 += chunk) {
    const size_t m = (size_t)std::min<uint64_t>(chunk, total - c0);
    TRY(launch(h, artp::ball_candidates_kernel, grid_for(h, m, 128), 128, 0, s, b, c0, m, d_sf));
    TRY(check_states_f32(h, d_sf, m, d_val, s));
    TRY(launch(h, artp::ball_first_valid_kernel, grid_for(h, m, 256), 256, 0, s, d_val, c0, m, n_iter, d_best));
  }
  return launch(h, artp::ball_result_kernel, grid_for(h, n, 128), 128, 0, s, b, n, d_best, d_states_out, d_index);
}

// ---------------------------------------------------------------------------------------------------------------
// The valid-heading layer: isValid of the goal projection (planner.cpp:223-237) of every cell centre at each heading
// ---------------------------------------------------------------------------------------------------------------
// What the goal projection (poseFrom2D and the layers built on it) needs: the whole map, with its normals.
int projection_map_args(Handle* h) {
  TRY(require_whole_map(h));
  if (!sampling(h).map.has_normals) {
    h->err = "no normal layers for this map (artp_estimate_normals or artp_set_sampler after artp_set_map)"; return ARTP_E_INVALID;
  }
  return ARTP_OK;
}

// Argument checks shared by both forms, before any device work; the headings as the kernels take them into *hd.
int heading_args(Handle* h, const double* yaw, int n_yaw, const uint32_t* mask, artp::Headings* hd) {
  TRY(projection_map_args(h));
  if (n_yaw < 1 || n_yaw > artp::kMaxHeadings) { h->err = "n_yaw must lie in 1..32"; return ARTP_E_INVALID; }
  if (!yaw || !mask) return null_buffer(h);
  std::memset(hd, 0, sizeof(*hd));
  for (int k = 0; k < n_yaw; ++k) {
    if (!std::isfinite(yaw[k])) { h->err = "yaw must be finite"; return ARTP_E_INVALID; }
    hd->yaw[k] = (float)yaw[k];
  }
  hd->n = n_yaw;
  return ARTP_OK;
}

// The layer of the current map into d_mask (rows x cols words) on s, in chunks of whole cells of at most kSampleChunk
// poses each; arguments checked by heading_args.
int valid_heading_layer(Handle* h, const artp::Headings& hd, uint32_t* d_mask, cudaStream_t s) {
  const size_t ncell = (size_t)h->rows * h->cols;
  const size_t chunk_cells = std::min(ncell, kSampleChunk / hd.n);
  char* r[2];   // states f32 | verdicts
  Buf<char>& scratch = sampling(h).samp_scratch;
  TRY(carve(h, scratch.p, scratch.cap, {chunk_cells * hd.n * 7 * sizeof(float), chunk_cells * hd.n}, r));
  float* d_sf = (float*)r[0];
  uint8_t* d_val = (uint8_t*)r[1];
  artp::SamplerDev m{};
  sampler_map_view(h, m);
  for (size_t c0 = 0; c0 < ncell; c0 += chunk_cells) {
    const size_t cells = std::min(chunk_cells, ncell - c0), n = cells * hd.n;
    TRY(launch(h, artp::heading_poses_kernel, grid_for(h, n, 128), 128, 0, s, m, hd, c0, n, d_sf));
    TRY(check_states_f32(h, d_sf, n, d_val, s));
    TRY(launch(h, artp::heading_pack_kernel, grid_for(h, cells, 256), 256, 0, s, d_val, hd.n, c0, cells, d_mask));
  }
  return ARTP_OK;
}

// The box-verdict layer: the ARTP_BOX_* word of the same goal projection at one heading. The argument checks of both
// forms, before any device work; the heading as heading_poses_kernel takes it into *hd.
int box_layer_args(Handle* h, double yaw, const uint16_t* out, artp::Headings* hd) {
  TRY(projection_map_args(h));
  if (!std::isfinite(yaw)) { h->err = "yaw must be finite"; return ARTP_E_INVALID; }
  if (!out) return null_buffer(h);
  std::memset(hd, 0, sizeof(*hd));
  hd->yaw[0] = (float)yaw;
  hd->n = 1;
  return ARTP_OK;
}

// The layer of the current map into d_out (rows x cols words) on s: one pose per cell, cell-major as the layer, in
// chunks of at most kSampleChunk cells, each chunk's words written in place; arguments checked by box_layer_args.
int box_verdict_layer(Handle* h, const artp::Headings& hd, uint16_t* d_out, cudaStream_t s) {
  const size_t ncell = (size_t)h->rows * h->cols;
  const size_t chunk = std::min(ncell, kSampleChunk);
  char* r[1];   // states f32
  Buf<char>& scratch = sampling(h).samp_scratch;
  TRY(carve(h, scratch.p, scratch.cap, {chunk * 7 * sizeof(float)}, r));
  float* d_sf = (float*)r[0];
  artp::SamplerDev m{};
  sampler_map_view(h, m);
  for (size_t c0 = 0; c0 < ncell; c0 += chunk) {
    const size_t n = std::min(chunk, ncell - c0);
    TRY(launch(h, artp::heading_poses_kernel, grid_for(h, n, 128), 128, 0, s, m, hd, c0, n, d_sf));
    TRY(box_verdicts_f32(h, d_sf, n, d_out + c0, s));
  }
  return ARTP_OK;
}

// cv::circle(kernel, (r, r), r, 255, FILLED) on a size x size zero image, r = size / 2 (utils.cpp:106-111): OpenCV's
// integer midpoint circle (imgproc/src/drawing.cpp, Circle()): for every step (dx, dy) of the octant walk the rows
// cy -+ dy get the span cx -+ dx and the rows cy -+ dx the span cx -+ dy, everything clipped to the image.
artp::MorphKernel make_circular_kernel(int size) {
  artp::MorphKernel k;
  std::memset(&k, 0, sizeof(k));
  if (size <= 0) {   // empty element: cv::erode / cv::dilate fall back to the 3 x 3 box, anchor (1, 1)
    k.size = 3; k.anchor = 1;
    for (int r = 0; r < 3; ++r) { k.lo[r] = 0; k.hi[r] = 2; }
    return k;
  }
  k.size = size; k.anchor = size / 2;
  for (int r = 0; r < size; ++r) { k.lo[r] = 127; k.hi[r] = -1; }
  const int radius = size / 2, cx = radius, cy = radius;
  auto span = [&](int y, int x0, int x1) {
    if (y < 0 || y >= size) return;
    x0 = std::max(x0, 0); x1 = std::min(x1, size - 1);
    if (x0 > x1) return;
    k.lo[y] = (int8_t)std::min<int>(k.lo[y], x0); k.hi[y] = (int8_t)std::max<int>(k.hi[y], x1);
  };
  int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
  while (dx >= dy) {
    span(cy - dy, cx - dx, cx + dx); span(cy + dy, cx - dx, cx + dx);
    span(cy - dx, cx - dy, cx + dy); span(cy + dx, cx - dy, cx + dy);
    dy++; err += plus; plus += 2;
    const int mask = (err <= 0) - 1;
    err -= minus & mask; dx += mask; minus -= mask & 2;
  }
  return k;
}

// cv::dilate / cv::erode of a rows x cols layer with getCircularKernel(size), one launch on s.
int launch_morph(Handle* h, bool dilate, const float* src, float* dst, int rows, int cols, int size, unsigned grid, cudaStream_t s) {
  const artp::MorphKernel k = make_circular_kernel(size);
  if (dilate) return launch(h, artp::morph_kernel<true>, grid, 256, 0, s, src, dst, rows, cols, k);
  return launch(h, artp::morph_kernel<false>, grid, 256, 0, s, src, dst, rows, cols, k);
}

// ---------------------------------------------------------------------------------------------------------------
// The sampler's distribution (artp_distribution.cuh): Basic::setTraversabilityFilter, then computeInverseSampleDensity ->
// applyBaseSampleDistribution -> applyMaxUnknownProbability -> computeCumulativeProbabilityDistribution
// (planner.cpp:39-58), the chain sampleGraph re-applies every recompute_density_after_n_samples vertices.
// ---------------------------------------------------------------------------------------------------------------
// getGaussianKernel(ksize, sigma, CV_32F) for sigma > 0: exp(-x^2 / (2 sigma^2)) at x = i - (ksize - 1) / 2, normalised
// by the double sum, then cast to float -- equal to OpenCV's coefficients (tests/test_sample_distribution_cpu.py).
artp::GaussTaps gauss_taps(int ksize, double sigma) {
  artp::GaussTaps k;
  std::memset(&k, 0, sizeof(k));
  std::vector<double> v(ksize);
  const double scale2X = -0.5 / (sigma * sigma);
  double sum = 0.0;
  for (int i = 0; i < ksize; ++i) {
    const double x = i - (ksize - 1) * 0.5;
    v[i] = std::exp(scale2X * (x * x));
    sum += v[i];
  }
  const double inv = 1.0 / sum;
  k.half = ksize / 2;
  for (int t = 0; t <= k.half; ++t) k.w[t] = (float)(v[k.half + t] * inv);
  return k;
}

// The map chain's size rules at resolution res: ARTP_E_LIMIT past a kernel's limit, else the sizes into `out` if given.
// The blur's kernel size and sigma in cells (sample_density.cpp:33-35), at most 1023 taps.
struct Blur { int ksize = 0; double sigma = 0.0; };
int blur_size(Handle* h, double radius, double res, Blur* out = nullptr) {
  const double cells = 6 * radius / res;   // the size is the odd one of (int)cells and (int)cells + 1
  if (!(cells < artp::kMaxGaussTaps + 1) || ((int)cells | 1) > artp::kMaxGaussTaps) {
    h->err = "Gaussian kernel larger than 1023 cells"; return ARTP_E_LIMIT;
  }
  if (out) *out = {(int)cells | 1, radius / res};
  return ARTP_OK;
}

// basic.cpp:116-122, with the implicit double -> int conversions of the int size parameters: at most 64 cells
struct FilterElements { int reach, wall; };
int sample_filter_sizes(Handle* h, double res, FilterElements* out = nullptr) {
  const artp_params& p = h->p;
  const FilterElements f{(int)(std::sqrt(p.reach_x * p.reach_x + p.reach_y * p.reach_y) / res),
                         (int)(std::min((p.torso_length - p.reach_x) * 0.5, (p.torso_width - p.reach_y) * 0.5) / res)};
  if (std::max(f.reach, f.wall) > artp::kMaxMorph) { h->err = "structuring element larger than 64 cells"; return ARTP_E_LIMIT; }
  if (out) *out = f;
  return ARTP_OK;
}

// basic.cpp:65-74: Basic's structuring elements, at most 64 cells
struct BasicElements { int foothold, margin, hole, search; };
int basic_elements(Handle* h, const artp_basic_params* bp, double res, BasicElements* out = nullptr) {
  const BasicElements e{(int)std::ceil(bp->foothold_size / res), (int)std::ceil(2 * bp->foothold_margin / res),
                        (int)std::floor(bp->foothold_margin_max_hole_size / res),
                        (int)std::ceil(2 * bp->foothold_margin_max_drop_search_radius / res)};
  if (std::max({e.foothold, e.margin, e.hole, e.search}) > artp::kMaxMorph) {
    h->err = "structuring element larger than 64 cells"; return ARTP_E_LIMIT;
  }
  if (out) *out = e;
  return ARTP_OK;
}

// Argument checks shared by both forms; the blur's size into `blur` unless it is null.
int distribution_args(Handle* h, const artp_sample_distribution_params* dp, Blur* blur = nullptr) {
  TRY(require_whole_map(h));
  if (!dp) { h->err = "null distribution params"; return ARTP_E_INVALID; }
  if (dp->use_inverse_vertex_density) {
    if (!(dp->density_blur_radius > 0.0 && std::isfinite(dp->density_blur_radius))) {
      h->err = "density_blur_radius must be finite and > 0"; return ARTP_E_INVALID;
    }
    TRY(blur_size(h, dp->density_blur_radius, h->res, blur));
  }
  if (dp->use_max_prob_unknown_samples) {
    if (!(dp->max_prob_unknown_samples >= 0.0 && dp->max_prob_unknown_samples <= 1.0)) {
      h->err = "max_prob_unknown_samples must lie in [0, 1]"; return ARTP_E_INVALID;
    }
    if (!sampling(h).map.has_dist_observed) {
      h->err = "the unknown-space cap needs the observed layer (artp_set_sample_filter after artp_set_map)"; return ARTP_E_INVALID;
    }
  }
  return ARTP_OK;
}

// The chain on s into sample_probability (*d_prob, in dist_scratch) and the sampler's CDF layers; arguments checked by
// distribution_args, which gave the blur's size.
int update_distribution(Handle* h, const artp_sample_distribution_params* dp, const Blur& blur, const double* d_states, size_t n,
                        cudaStream_t s, float** d_prob = nullptr) {
  TRY(ensure_sampler_layers(h));
  Sampling& S = sampling(h);
  const int rows = h->rows, cols = h->cols;
  const size_t ncell = (size_t)rows * cols, lb = ncell * sizeof(float), rb = (size_t)rows * sizeof(double);
  char* r[7];   // n_samples | blur pass | sample_probability | known row sums | unknown row sums | max bits | cap multipliers
  TRY(carve(h, S.dist_scratch.p, S.dist_scratch.cap, {lb, lb, lb, rb, rb, sizeof(unsigned int), 2 * sizeof(float)}, r));
  float *n_samples = (float*)r[0], *pass = (float*)r[1], *prob = (float*)r[2], *mult = (float*)r[6];
  double *known = (double*)r[3], *unknown = (double*)r[4];
  unsigned int* max_bits = (unsigned int*)r[5];
  const unsigned grid = grid_for(h, ncell, 256);
  const float* n_blur = nullptr;
  if (dp->use_inverse_vertex_density) {                                          // sample_density.cpp:21-42
    CU_TRY(h, cudaMemsetAsync(n_samples, 0, ncell * sizeof(float), s));
    CU_TRY(h, cudaMemsetAsync(max_bits, 0, sizeof(unsigned int), s));
    if (n) {
      artp::SamplerDev m{};
      sampler_map_view(h, m);
      TRY(launch(h, artp::vertex_histogram_kernel, grid_for(h, n, 256), 256, 0, s, m, d_states, n, n_samples));
    }
    const artp::GaussTaps k = gauss_taps(blur.ksize, blur.sigma);
    TRY(launch(h, artp::gauss_pass_kernel<0>, grid, 256, 0, s, n_samples, pass, rows, cols, k));
    TRY(launch(h, artp::gauss_pass_kernel<1>, grid, 256, 0, s, pass, n_samples, rows, cols, k));
    TRY(launch(h, artp::abs_max_kernel, grid, 256, 0, s, n_samples, ncell, max_bits));
    n_blur = n_samples;
  }
  const Layers D{S.dist_layers.p, ncell};
  TRY(launch(h, artp::combine_kernel, grid, 256, 0, s, n_blur, max_bits, S.map.has_sample_filter ? D[kFilter] : nullptr, ncell,
      prob));
  if (dp->use_max_prob_unknown_samples) {                                        // probability_distribution.cpp:50-91
    const float* obs = D[kObserved];
    TRY(launch(h, artp::cap_rows_kernel, (rows + 63) / 64, 64, 0, s, prob, obs, rows, cols, known, unknown));
    TRY(launch(h, artp::cap_mult_kernel, 1, 32, 0, s, known, unknown, rows, dp->max_prob_unknown_samples, mult));
    TRY(launch(h, artp::cap_apply_kernel, grid, 256, 0, s, prob, obs, mult, ncell));
  }
  TRY(launch_sample_cdf(h, prob, s));
  S.map.has_device_cdf = true;
  S.map.has_sampler = false;      // the sampler must be (re)armed with artp_set_sampler
  if (d_prob) *d_prob = prob;
  return ARTP_OK;
}

// Basic::setTraversabilityFilter on s from the DEVICE layer d_thr (NULL: the last Basic's), with the HOST observed layer
// (NULL: the last Basic's, when it had one) kept for the unknown-space cap. Scratch: dist_scratch.
// basic_fits: the last Basic ran on a map of this size.
int sample_filter(Handle* h, const float* d_thr, const float* observed, bool basic_fits, cudaStream_t s) {
  FilterElements f;
  TRY(sample_filter_sizes(h, h->res, &f));
  Sampling& S = sampling(h);
  const int rows = h->rows, cols = h->cols;
  const bool basic_observed = !observed && basic_fits && S.has_basic_observed;
  const size_t n = (size_t)rows * cols, lb = n * sizeof(float);
  char* r[2];   // dilated | closed
  TRY(carve(h, S.dist_scratch.p, S.dist_scratch.cap, {lb, lb}, r));
  S.map.has_sample_filter = S.map.has_dist_observed = false;
  TRY(grow(h, S.dist_layers.p, S.dist_layers.cap, kDistLayers * n));
  const Layers D{S.dist_layers.p, n};
  const Layers B{S.basic_keep.p, n};
  float *filter = D[kFilter], *obs = D[kObserved];
  const float* thr = d_thr ? d_thr : B[kThresholded];
  if (observed) CU_TRY(h, cudaMemcpyAsync(obs, observed, lb, cudaMemcpyHostToDevice, s));
  if (basic_observed) CU_TRY(h, cudaMemcpyAsync(obs, B[kBasicObserved], lb, cudaMemcpyDeviceToDevice, s));
  const unsigned grid = grid_for(h, n, 256);
  TRY(launch_morph(h, true, thr, (float*)r[0], rows, cols, f.reach, grid, s));          // dilateAndErode: step over small obstacles
  TRY(launch_morph(h, false, (float*)r[0], (float*)r[1], rows, cols, f.reach, grid, s));
  TRY(launch_morph(h, false, (float*)r[1], filter, rows, cols, f.wall, grid, s));         // erode: keep away from walls
  S.map.has_sample_filter = true;
  S.map.has_dist_observed = observed || basic_observed;
  return ARTP_OK;
}

}  // namespace

int artp_api::set_sample_filter_basic(Handle* h, cudaStream_t s) { return sample_filter(h, nullptr, nullptr, true, s); }

int artp_api::map_chain_limits(Handle* h, const artp_basic_params* bp, double res, bool distribution, bool inverse_density) {
  TRY(basic_elements(h, bp, res));
  if (!distribution) return ARTP_OK;
  TRY(sample_filter_sizes(h, res));
  return inverse_density ? blur_size(h, density_blur_radius(h->p), res) : ARTP_OK;
}

int artp_api::process_basic(Handle* h, float* L, int rows, int cols, double res, const artp_basic_params* bp, bool has_observed,
                            cudaStream_t s) {
  BasicElements e;
  TRY(basic_elements(h, bp, res, &e));
  Sampling& S = sampling(h);
  const size_t n = (size_t)rows * cols, lb = n * sizeof(float);
  S.has_basic_layers = false;
  TRY(grow(h, S.basic_keep.p, S.basic_keep.cap, kBasicLayers * n));
  const Layers keep{S.basic_keep.p, n};
  // L: 0 elev, 1 trav, 2 observed, 3 T0, 4 A, 5 B, 6 elev eroded, 7 elev dilated, 8 out
  const unsigned grid = grid_for(h, n, 256);
  auto morph = [&](bool dil, const float* src, float* dst, int size) { return launch_morph(h, dil, src, dst, rows, cols, size, grid, s); };
  float *E = L, *T0 = L + 3 * n, *A = L + 4 * n, *B = L + 5 * n, *Elo = L + 6 * n, *Ehi = L + 7 * n, *O = L + 8 * n;
  const float drop = (float)bp->foothold_margin_max_drop, step = (float)bp->foothold_margin_min_step;
  TRY(launch(h, artp::basic_threshold_kernel, grid, 256, 0, s, L + n, L + 2 * n, bp->unknown_space_untraversable ? 1 : 0,
             bp->traversability_thres, n, T0));
  TRY(morph(true, T0, A, e.hole)); TRY(morph(false, A, B, e.hole));       // dilateAndErode: close holes (:72)
  TRY(morph(false, E, Elo, e.search));                                    // elevation - erode(elevation) (:75-77)
  TRY(morph(true, E, Ehi, e.margin));                                     // dilate(elevation) - elevation (:84)
  TRY(launch(h, artp::basic_select_kernel, grid, 256, 0, s, 0, E, Elo, Ehi, T0, B, drop, step, n, A));
  TRY(morph(false, A, B, e.margin));                                      // erode by the safety margin (:90)
  TRY(launch(h, artp::basic_select_kernel, grid, 256, 0, s, 1, E, Elo, Ehi, T0, B, drop, step, n, A));
  TRY(morph(false, A, B, e.foothold)); TRY(morph(true, B, A, e.foothold));   // erodeAndDilate: remove small patches (:95)
  TRY(launch(h, artp::basic_final_kernel, grid, 256, 0, s, E, T0, A, n, B, O));
  // kept for artp_set_sample_filter(h, NULL, NULL, ...)
  if (has_observed) CU_TRY(h, cudaMemcpyAsync(keep[kBasicObserved], L + 2 * n, lb, cudaMemcpyDeviceToDevice, s));
  CU_TRY(h, cudaMemcpyAsync(keep[kThresholded], B, lb, cudaMemcpyDeviceToDevice, s));
  S.basic_rows = rows; S.basic_cols = cols;
  S.has_basic_layers = true;
  S.has_basic_observed = has_observed;
  return ARTP_OK;
}

int artp_api::sampler_armed(Handle* h) {
  TRY(require_map(h));
  if (!sampling(h).map.has_sampler) { h->err = "no sampler layers set (artp_set_sampler after artp_set_map)"; return ARTP_E_NOMAP; }
  return ARTP_OK;
}

int artp_api::estimate_normals(Handle* h, double estimation_radius, cudaStream_t s) {
  TRY(ensure_sampler_layers(h));
  const Layers L = sampler_layers(h);
  const double res = h->chk.Lx / h->rows;
  const int r_cells = (int)(estimation_radius / res), r_diag = (int)(estimation_radius * 0.70710678118 / res);   // utils.cpp:226-227
  TRY(launch(h, artp::estimate_normals_kernel, grid_for(h, L.ncell, 128, 32), 128, 0, s, h->d_H[0], h->pitch, h->rows,
      h->cols, res, h->chk.cx, h->chk.cy, r_cells, r_diag, L[kNormalX], L[kNormalY], L[kNormalZ], L[kStdDev]));
  Sampling::MapFlags& f = sampling(h).map;
  f.has_device_normals = f.has_normals = true;
  f.has_sampler = false;      // the sampler must be (re)armed with artp_set_sampler
  return ARTP_OK;
}

int artp_api::ball_search(Handle* h, const double* d_centres, size_t n, const double* d_radius, uint32_t n_iter, uint64_t seed,
                          uint64_t first_draw, double* d_states_out, int32_t* d_index, cudaStream_t s) {
  TRY(ball_search_args(h, n, n_iter, nullptr));
  return find_valid_near(h, d_centres, n, d_radius, n_iter, nullptr, seed, first_draw, d_states_out, d_index, s);
}

int artp_api::pose_from_2d(Handle* h, const double* d_in, size_t n, double* d_out, uint8_t* d_inside, cudaStream_t s) {
  artp::SamplerDev m{};
  sampler_map_view(h, m);
  return launch(h, artp::pose_from_2d_kernel, grid_for(h, n, 128), 128, 0, s, m, d_in, n, d_out, d_inside);
}

// Without sp only the CDF pointers are set, to what an arming with sp gives them: null unless it samples from the
// distribution, else the resident layers, which stay put while the map does (they grow only for a larger map).
void artp_api::arm_sampler(Handle* h, const artp_sampler_params* sp) {
  Sampling& S = sampling(h);
  artp::SamplerDev& m = S.samp;
  if (sp) {
    sampler_map_view(h, m);
    m.max_roll_pert = sp->max_roll_pert; m.max_pitch_pert = sp->max_pitch_pert;
    m.from_distribution = sp->sample_from_distribution ? 1 : 0;
    m.low[0] = sp->low[0]; m.low[1] = sp->low[1]; m.high[0] = sp->high[0]; m.high[1] = sp->high[1];
    m.reach_z = h->p.reach_z;
  }
  const Layers L = sampler_layers(h);
  m.cum_prob = m.from_distribution ? L[kCumProb] : nullptr;
  m.cum_row = m.from_distribution ? L[kCumRow] : nullptr;
  S.map.has_sampler = true;
}

// Sample -> check -> compact on s, in chunks of kSampleChunk draws: the valid states of draws first_sample ..
// first_sample + n_draw - 1 in draw order into d_states_out (at most `capacity` of them), their number into *d_count;
// with d_draws, the draw index of each kept state too.
int artp_api::sample_valid_draws(Handle* h, uint64_t seed, uint64_t first_sample, size_t n_draw, double* d_states_out,
                                 uint64_t* d_draws, size_t capacity, uint32_t* d_count, cudaStream_t s) {
  CU_TRY(h, cudaMemsetAsync(d_count, 0, sizeof(uint32_t), s));
  if (n_draw == 0) return ARTP_OK;
  Sampling& S = sampling(h);
  const size_t chunk = std::min(n_draw, kSampleChunk);
  char* r[5];   // states f64 | states f32 | indices | valid | chunk count
  TRY(carve(h, S.samp_scratch.p, S.samp_scratch.cap,
             {chunk * 7 * sizeof(double), chunk * 7 * sizeof(float), chunk * sizeof(int64_t), chunk, sizeof(uint32_t)}, r));
  double* d_st = (double*)r[0];
  float* d_sf = (float*)r[1];
  int64_t* d_idx = (int64_t*)r[2];
  uint8_t* d_val = (uint8_t*)r[3];
  uint32_t* d_cnt = (uint32_t*)r[4];
  for (size_t done = 0; done < n_draw; done += chunk) {
    const size_t m = std::min(chunk, n_draw - done);
    TRY(launch(h, artp::sample_states_kernel, grid_for(h, m, 128), 128, 0, s, S.samp, nullptr, seed, first_sample + done, m,
        d_st, d_sf, nullptr));
    TRY(check_states_f32(h, d_sf, m, d_val, s));
    // rejected (outside-map) candidates carry NaN states
    if (!S.samp.from_distribution) TRY(launch(h, artp::reject_nan_kernel, grid_for(h, m, 256), 256, 0, s, d_st, m, d_val));
    TRY(compact_valid(h, d_val, m, 0, d_idx, d_cnt, s));
    TRY(launch(h, gather_chunk_kernel, grid_for(h, m * 7, 256), 256, 0, s, d_st, d_idx, d_cnt, d_count, capacity,
        d_states_out));
    if (d_draws)
      TRY(launch(h, gather_draws_kernel, grid_for(h, m, 256), 256, 0, s, d_idx, d_cnt, d_count, capacity, first_sample + done,
          d_draws));
    TRY(launch(h, add_count_kernel, 1, 1, 0, s, d_count, d_cnt));
  }
  return ARTP_OK;
}

int artp_api::check_distribution_args(Handle* h, const artp_sample_distribution_params* dp) { return distribution_args(h, dp); }

int artp_api::update_distribution_rearm(Handle* h, const artp_sample_distribution_params* dp, const double* d_states, size_t n,
                                        cudaStream_t s) {
  Blur blur;
  TRY(distribution_args(h, dp, &blur));
  TRY(update_distribution(h, dp, blur, d_states, n, s));
  arm_sampler(h, nullptr);   // artp_set_sampler(h, sp, ..., NULL, NULL): the CDF rows just computed are cumulative
  return ARTP_OK;
}

extern "C" {

int artp_estimate_normals(artp_handle* hh, double estimation_radius, float* normal_x, float* normal_y, float* normal_z,
                          float* plane_fit_std_dev) {
  LOCK_CALL(h, hh);
  TRY(require_whole_map(h));
  if (!(estimation_radius >= 0.0)) { h->err = "estimation_radius < 0"; return ARTP_E_INVALID; }
  TRY(host_call_begin(h));
  TRY(artp_api::estimate_normals(h, estimation_radius, h->stream));
  const Layers L = sampler_layers(h);
  float* dst[4] = {normal_x, normal_y, normal_z, plane_fit_std_dev};
  for (int k = 0; k < 4; ++k)
    if (dst[k]) CU_TRY(h, cudaMemcpyAsync(dst[k], L[k], L.ncell * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

int artp_compute_sample_cdf(artp_handle* hh, const float* sample_probability, float* cum_prob, float* cum_prob_rowwise) {
  LOCK_CALL(h, hh);
  TRY(require_whole_map(h));
  if (!sample_probability) return null_buffer(h);
  const size_t ncell = (size_t)h->rows * h->cols;
  char* d_prob;
  TRY(host_call_begin(h, {ncell * sizeof(float)}, &d_prob));
  TRY(ensure_sampler_layers(h));
  const Layers L = sampler_layers(h);
  CU_TRY(h, cudaMemcpyAsync(d_prob, sample_probability, ncell * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  TRY(launch_sample_cdf(h, (const float*)d_prob, h->stream));
  if (cum_prob) CU_TRY(h, cudaMemcpyAsync(cum_prob, L[kCumProb], ncell * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if (cum_prob_rowwise)
    CU_TRY(h, cudaMemcpyAsync(cum_prob_rowwise, L[kCumRow], (size_t)h->rows * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  TRY(host_call_end(h));
  sampling(h).map.has_device_cdf = true;
  sampling(h).map.has_sampler = false;      // the sampler must be (re)armed with artp_set_sampler
  return ARTP_OK;
}

int artp_set_sampler(artp_handle* hh, const artp_sampler_params* sp, const float* normal_x, const float* normal_y,
                     const float* normal_z, const float* plane_fit_std_dev, const float* cum_prob,
                     const float* cum_prob_rowwise) {
  LOCK_CALL(h, hh);
  TRY(require_whole_map(h));
  const bool host_normals = normal_x && normal_y && normal_z && plane_fit_std_dev;
  if (!sp) { h->err = "null sampler params"; return ARTP_E_INVALID; }
  if (!host_normals && (normal_x || normal_y || normal_z || plane_fit_std_dev)) {
    h->err = "pass all four normal / plane-fit layers or none"; return ARTP_E_INVALID;
  }
  Sampling& S = sampling(h);
  if (!host_normals && !S.map.has_device_normals) {
    h->err = "no normal layers: pass them or call artp_estimate_normals after artp_set_map"; return ARTP_E_INVALID;
  }
  const bool host_cdf = cum_prob && cum_prob_rowwise;
  if (sp->sample_from_distribution && !host_cdf && !(S.map.has_device_cdf && !cum_prob && !cum_prob_rowwise)) {
    h->err = "sample_from_distribution needs the cum_prob layers (pass both, or call artp_compute_sample_cdf first)";
    return ARTP_E_INVALID;
  }
  if (!sp->sample_from_distribution && !(sp->high[0] > sp->low[0] && sp->high[1] > sp->low[1])) {
    h->err = "empty sampling bounds"; return ARTP_E_INVALID;
  }
  char* d_bad_word;   // the CDF check's verdict
  TRY(host_call_begin(h, {sizeof(uint32_t)}, &d_bad_word));
  TRY(ensure_sampler_layers(h));
  const Layers L = sampler_layers(h);
  if (host_normals) {
    const float* src[4] = {normal_x, normal_y, normal_z, plane_fit_std_dev};
    for (int k = 0; k < 4; ++k)
      CU_TRY(h, cudaMemcpyAsync(L[k], src[k], L.ncell * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    S.map.has_device_normals = false;   // overwritten by the caller's layers
    S.map.has_normals = true;
  }
  uint32_t bad = 0;
  if (sp->sample_from_distribution) {
    if (host_cdf) {
      CU_TRY(h, cudaMemcpyAsync(L[kCumProb], cum_prob, L.ncell * sizeof(float), cudaMemcpyHostToDevice, h->stream));
      CU_TRY(h, cudaMemcpyAsync(L[kCumRow], cum_prob_rowwise, (size_t)h->rows * sizeof(float), cudaMemcpyHostToDevice,
                                h->stream));
      S.map.has_device_cdf = false;   // overwritten by the caller's layers
    }
    // the binary searches need monotone (or all-NaN) CDF rows: refuse anything else
    uint32_t* d_bad = (uint32_t*)d_bad_word;
    CU_TRY(h, cudaMemsetAsync(d_bad, 0, sizeof(uint32_t), h->stream));
    TRY(launch(h, artp::validate_cdf_kernel, (h->rows + 127) / 128, 128, 0, h->stream, L[kCumProb], h->rows, h->cols,
        (size_t)h->rows, 1, d_bad));
    TRY(launch(h, artp::validate_cdf_kernel, 1, 32, 0, h->stream, L[kCumRow], 1, h->rows, 1, 0, d_bad));
    CU_TRY(h, cudaMemcpyAsync(&bad, d_bad, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  }
  TRY(host_call_end(h));
  if (bad) { h->err = "cum_prob layers are not cumulative distributions (rows must be non-decreasing or all NaN)"; return ARTP_E_INVALID; }
  arm_sampler(h, sp);
  return ARTP_OK;
}

int artp_sampler_uniforms(artp_handle* hh, uint64_t seed, uint64_t first_sample, size_t n, double* u) {
  LOCK_CALL(h, hh);
  if (n == 0) return ARTP_OK;
  if (!u) return null_buffer(h);
  char* d_u;
  TRY(host_call_begin(h, {n * 6 * sizeof(double)}, &d_u));
  TRY(launch(h, artp::sampler_uniforms_kernel, grid_for(h, n, 256), 256, 0, h->stream, seed, first_sample, n, (double*)d_u));
  CU_TRY(h, cudaMemcpyAsync(u, d_u, n * 6 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

int artp_sample_states_device(artp_handle* hh, const double* d_u, uint64_t seed, uint64_t first_sample, size_t n,
                              double* d_states, int32_t* d_rowcol, void* stream) {
  LOCK_CALL(h, hh);
  TRY(sampler_armed(h));
  if (n == 0) return ARTP_OK;
  if (!d_states) return null_buffer(h);
  CU_TRY(h, cudaSetDevice(h->device));
  return launch(h, artp::sample_states_kernel, grid_for(h, n, 128), 128, 0, (cudaStream_t)stream, sampling(h).samp, d_u, seed, first_sample, n,
                d_states, nullptr, d_rowcol);
}

int artp_sample_states(artp_handle* hh, const double* u, uint64_t seed, uint64_t first_sample, size_t n, double* states,
                       int32_t* rowcol) {
  LOCK_CALL(h, hh);
  TRY(sampler_armed(h));
  if (n == 0) return ARTP_OK;
  if (!states) return null_buffer(h);
  char* r[3];   // u | states | rowcol
  TRY(host_call_begin(h, {n * 6 * sizeof(double), n * 7 * sizeof(double), n * 2 * sizeof(int32_t)}, r));
  if (u) CU_TRY(h, cudaMemcpyAsync(r[0], u, n * 6 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  TRY(launch(h, artp::sample_states_kernel, grid_for(h, n, 128), 128, 0, h->stream, sampling(h).samp, u ? (const double*)r[0] : nullptr,
      seed, first_sample, n, (double*)r[1], nullptr, rowcol ? (int32_t*)r[2] : nullptr));
  CU_TRY(h, cudaMemcpyAsync(states, r[1], n * 7 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (rowcol) CU_TRY(h, cudaMemcpyAsync(rowcol, r[2], n * 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

int artp_sample_valid_device(artp_handle* hh, uint64_t seed, uint64_t first_sample, size_t n_draw, double* d_states_out,
                             size_t capacity, uint32_t* d_count, void* stream) {
  LOCK_CALL(h, hh);
  TRY(sampler_armed(h));
  if (!d_count || (capacity && !d_states_out)) return null_buffer(h);
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  return sample_valid_draws(h, seed, first_sample, n_draw, d_states_out, nullptr, capacity, d_count, s);
}

int artp_sample_valid(artp_handle* hh, uint64_t seed, uint64_t first_sample, size_t n_draw, double* states, size_t capacity,
                      size_t* n_valid) {
  LOCK_CALL(h, hh);
  const size_t cap = std::min(capacity, n_draw);
  TRY(sampler_armed(h));
  if (!n_valid || (cap && !states)) return null_buffer(h);
  char* r[2];   // states | count
  TRY(host_call_begin(h, {cap * 7 * sizeof(double), sizeof(uint32_t)}, r));
  TRY(sample_valid_draws(h, seed, first_sample, n_draw, (double*)r[0], nullptr, cap, (uint32_t*)r[1], h->stream));
  uint32_t cnt = 0;
  CU_TRY(h, cudaMemcpyAsync(&cnt, r[1], sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  const int rc = host_call_end(h, true);
  if (rc == ARTP_E_CUDA) return rc;
  const size_t keep = std::min<size_t>(cnt, cap);
  if (keep) {   // the copy's size is the count: it follows the call's end (d_stage is still ours: the lock is held)
    CU_TRY(h, cudaMemcpyAsync(states, r[0], keep * 7 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(h, cudaStreamSynchronize(h->stream));
  }
  *n_valid = cnt;      // > capacity means the output was truncated to `capacity` states
  return rc;
}

int artp_find_valid_near_device(artp_handle* hh, const double* d_centres, size_t n, const double* d_radius, uint32_t n_iter,
                                const double* d_offsets, uint64_t seed, uint64_t first_draw, double* d_states_out,
                                int32_t* d_index, void* stream) {
  LOCK_CALL(h, hh);
  TRY(ball_search_args(h, n, n_iter, nullptr));
  if (n == 0) return ARTP_OK;
  if (!d_centres || !d_radius || !d_states_out || !d_index) return null_buffer(h);
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  return find_valid_near(h, d_centres, n, d_radius, n_iter, d_offsets, seed, first_draw, d_states_out, d_index, s);
}

int artp_find_valid_near(artp_handle* hh, const double* centres, size_t n, const double* radius, uint32_t n_iter,
                         const double* offsets, uint64_t seed, uint64_t first_draw, double* states_out, int32_t* index) {
  LOCK_CALL(h, hh);
  if (n && (!centres || !radius || !states_out || !index)) return null_buffer(h);
  TRY(ball_search_args(h, n, n_iter, radius));
  if (n == 0) return ARTP_OK;
  const size_t sb = n * 7 * sizeof(double), ob = offsets ? n * (size_t)n_iter * 2 * sizeof(double) : 0;
  char* r[5];   // centres | radius | offsets | states | index
  TRY(host_call_begin(h, {sb, n * sizeof(double), ob, sb, n * sizeof(int32_t)}, r));
  CU_TRY(h, cudaMemcpyAsync(r[0], centres, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], radius, n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  if (ob) CU_TRY(h, cudaMemcpyAsync(r[2], offsets, ob, cudaMemcpyHostToDevice, h->stream));
  TRY(find_valid_near(h, (const double*)r[0], n, (const double*)r[1], n_iter, offsets ? (const double*)r[2] : nullptr, seed,
      first_draw, (double*)r[3], (int32_t*)r[4], h->stream));
  CU_TRY(h, cudaMemcpyAsync(states_out, r[3], sb, cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(h, cudaMemcpyAsync(index, r[4], n * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h, true);
}

int artp_ball_offsets(artp_handle* hh, uint64_t seed, uint64_t first_draw, size_t n, uint32_t n_iter, const double* radius,
                      double* offsets) {
  LOCK_CALL(h, hh);
  const size_t total = n * (size_t)n_iter;
  if (total == 0) return ARTP_OK;
  if (!radius || !offsets) return null_buffer(h);
  if ((uint64_t)n >= (1ull << 32)) { h->err = "n must be < 2^32"; return ARTP_E_INVALID; }
  char* r[2];   // radius | offsets
  TRY(host_call_begin(h, {n * sizeof(double), total * 2 * sizeof(double)}, r));
  CU_TRY(h, cudaMemcpyAsync(r[0], radius, n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  TRY(launch(h, artp::ball_offsets_kernel, grid_for(h, total, 256), 256, 0, h->stream, seed, first_draw, n, n_iter,
      (const double*)r[0], (double*)r[1]));
  CU_TRY(h, cudaMemcpyAsync(offsets, r[1], total * 2 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

int artp_pose_from_2d(artp_handle* hh, const double* states_in, size_t n, double* states_out, uint8_t* inside) {
  LOCK_CALL(h, hh);
  TRY(projection_map_args(h));
  if (n == 0) return ARTP_OK;
  if (!states_in || !states_out) return null_buffer(h);
  char* r[3];   // states in | states out | inside
  TRY(host_call_begin(h, {n * 7 * sizeof(double), n * 7 * sizeof(double), n}, r));
  CU_TRY(h, cudaMemcpyAsync(r[0], states_in, n * 7 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  TRY(artp_api::pose_from_2d(h, (const double*)r[0], n, (double*)r[1], (uint8_t*)r[2], h->stream));
  CU_TRY(h, cudaMemcpyAsync(states_out, r[1], n * 7 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (inside) CU_TRY(h, cudaMemcpyAsync(inside, r[2], n, cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

int artp_valid_heading_layer(artp_handle* hh, const double* yaw, int n_yaw, uint32_t* mask) {
  LOCK_CALL(h, hh);
  artp::Headings hd;
  TRY(heading_args(h, yaw, n_yaw, mask, &hd));
  const size_t bytes = (size_t)h->rows * h->cols * sizeof(uint32_t);
  char* d_mask;
  TRY(host_call_begin(h, {bytes}, &d_mask));
  TRY(valid_heading_layer(h, hd, (uint32_t*)d_mask, h->stream));
  CU_TRY(h, cudaMemcpyAsync(mask, d_mask, bytes, cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h, true);
}

int artp_valid_heading_layer_device(artp_handle* hh, const double* yaw, int n_yaw, uint32_t* d_mask, void* stream) {
  LOCK_CALL(h, hh);
  artp::Headings hd;
  TRY(heading_args(h, yaw, n_yaw, d_mask, &hd));
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  return valid_heading_layer(h, hd, d_mask, s);
}

int artp_box_verdict_layer(artp_handle* hh, double yaw, uint16_t* out) {
  LOCK_CALL(h, hh);
  artp::Headings hd;
  TRY(box_layer_args(h, yaw, out, &hd));
  const size_t bytes = (size_t)h->rows * h->cols * sizeof(uint16_t);
  char* d_out;
  TRY(host_call_begin(h, {bytes}, &d_out));
  TRY(box_verdict_layer(h, hd, (uint16_t*)d_out, h->stream));
  TRY(copy_async(h, out, d_out, bytes, cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h, true);
}

int artp_box_verdict_layer_device(artp_handle* hh, double yaw, uint16_t* d_out, void* stream) {
  LOCK_CALL(h, hh);
  artp::Headings hd;
  TRY(box_layer_args(h, yaw, d_out, &hd));
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  return box_verdict_layer(h, hd, d_out, s);
}

int artp_debug_circular_kernel(int size, uint8_t* out) {   // test hook: the size x size element as 0 / 1 bytes (row-major)
  if (size > artp::kMaxMorph || !out) return ARTP_E_INVALID;
  const artp::MorphKernel k = make_circular_kernel(size);
  for (int r = 0; r < k.size; ++r) for (int c = 0; c < k.size; ++c) out[r * k.size + c] = (c >= k.lo[r] && c <= k.hi[r]) ? 1 : 0;
  return k.size;
}

int artp_process_basic(artp_handle* hh, const float* elevation, const float* traversability, const float* observed, int rows,
                       int cols, double res, const artp_basic_params* bp, float* elevation_masked, float* traversability_thresholded) {
  LOCK_CALL(h, hh);
  if (!elevation || !traversability || !bp || !elevation_masked || rows < 1 || cols < 1 || !(res > 0)) {
    h->err = "bad arguments"; return ARTP_E_INVALID;
  }
  if (bp->unknown_space_untraversable && !observed) { h->err = "unknown_space_untraversable needs the observed layer"; return ARTP_E_INVALID; }
  TRY(artp_api::map_chain_limits(h, bp, res, false, false));
  const size_t n = (size_t)rows * cols, lb = n * sizeof(float);
  char* stage;
  TRY(host_call_begin(h, {9 * lb}, &stage));
  float* L = (float*)stage;
  cudaStream_t s = h->stream;
  CU_TRY(h, cudaMemcpyAsync(L, elevation, lb, cudaMemcpyHostToDevice, s));
  CU_TRY(h, cudaMemcpyAsync(L + n, traversability, lb, cudaMemcpyHostToDevice, s));
  if (observed) CU_TRY(h, cudaMemcpyAsync(L + 2 * n, observed, lb, cudaMemcpyHostToDevice, s));
  TRY(artp_api::process_basic(h, L, rows, cols, res, bp, observed != nullptr, s));
  CU_TRY(h, cudaMemcpyAsync(elevation_masked, L + 8 * n, lb, cudaMemcpyDeviceToHost, s));
  if (traversability_thresholded) CU_TRY(h, cudaMemcpyAsync(traversability_thresholded, L + 5 * n, lb, cudaMemcpyDeviceToHost, s));
  return host_call_end(h);
}

int artp_set_sample_filter(artp_handle* hh, const float* traversability_thresholded, const float* observed,
                           float* traversability_sample_filter) {
  LOCK_CALL(h, hh);
  TRY(require_whole_map(h));
  const int rows = h->rows, cols = h->cols;
  const Sampling& S = sampling(h);
  const bool basic_fits = S.has_basic_layers && S.basic_rows == rows && S.basic_cols == cols;
  if (!traversability_thresholded && !basic_fits) {
    h->err = "no traversability_thresholded layer: pass it, or run artp_process_basic on a map of this size first";
    return ARTP_E_INVALID;
  }
  TRY(sample_filter_sizes(h, h->res));
  const size_t n = (size_t)rows * cols, lb = n * sizeof(float);
  char* r[1];   // caller's traversability_thresholded
  TRY(host_call_begin(h, {lb}, r));
  if (traversability_thresholded) CU_TRY(h, cudaMemcpyAsync(r[0], traversability_thresholded, lb, cudaMemcpyHostToDevice, h->stream));
  TRY(sample_filter(h, traversability_thresholded ? (const float*)r[0] : nullptr, observed, basic_fits, h->stream));
  if (traversability_sample_filter)
    CU_TRY(h, cudaMemcpyAsync(traversability_sample_filter, Layers{S.dist_layers.p, n}[kFilter], lb, cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

int artp_debug_gaussian_kernel(int ksize, double sigma, float* out) {   // test hook: the ksize coefficients
  if (ksize < 1 || ksize > artp::kMaxGaussTaps || !(ksize & 1) || !(sigma > 0) || !out) return ARTP_E_INVALID;
  const artp::GaussTaps k = gauss_taps(ksize, sigma);
  for (int i = 0; i < ksize; ++i) out[i] = k.w[std::abs(i - k.half)];
  return ksize;
}

int artp_update_sample_distribution_device(artp_handle* hh, const artp_sample_distribution_params* dp,
                                           const double* d_vertex_states, size_t n, void* stream) {
  LOCK_CALL(h, hh);
  Blur blur;
  TRY(distribution_args(h, dp, &blur));
  if (n && !d_vertex_states) return null_buffer(h);
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  return update_distribution(h, dp, blur, d_vertex_states, n, s);
}

int artp_update_sample_distribution(artp_handle* hh, const artp_sample_distribution_params* dp, const double* vertex_states,
                                    size_t n, float* sample_probability, float* cum_prob, float* cum_prob_rowwise) {
  LOCK_CALL(h, hh);
  Blur blur;
  TRY(distribution_args(h, dp, &blur));
  if (n && !vertex_states) return null_buffer(h);
  const size_t sb = n * 7 * sizeof(double), ncell = (size_t)h->rows * h->cols;
  char* r[1];
  TRY(host_call_begin(h, {sb}, r));
  if (n) CU_TRY(h, cudaMemcpyAsync(r[0], vertex_states, sb, cudaMemcpyHostToDevice, h->stream));
  float* d_prob;
  TRY(update_distribution(h, dp, blur, (const double*)r[0], n, h->stream, &d_prob));
  if (sample_probability)
    CU_TRY(h, cudaMemcpyAsync(sample_probability, d_prob, ncell * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  const Layers L = sampler_layers(h);
  if (cum_prob) CU_TRY(h, cudaMemcpyAsync(cum_prob, L[kCumProb], ncell * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if (cum_prob_rowwise)
    CU_TRY(h, cudaMemcpyAsync(cum_prob_rowwise, L[kCumRow], (size_t)h->rows * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

}  // extern "C"

void artp_api::sampling_forget_map(Handle* h) { sampling(h).map = Sampling::MapFlags{}; }

void artp_api::sampling_free(Handle* h) { delete h->sampling; }
