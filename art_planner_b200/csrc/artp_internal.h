// art_planner_b200/csrc/artp_internal.h -- what the units of the C ABI share (not installed). The units and what each owns:
//   artp_capi.cu           the handle's lifecycle, errors, stats and timing, and the validity pipeline (Pipeline): pose /
//                          motion / edge checks, box verdicts, compaction and bit packing
//   artp_map.cu            the installed map (MapStore): its layers, range tables and plane tables, artp_set_map[_window],
//                          and the reductions over a layer (finite range, non-finite cells)
//   artp_sampling.cu       normals and the CDF, the sampler, start / goal search, poseFrom2D, the valid-heading and
//                          box-verdict layers, Basic, the sample distribution (Sampling)
//   artp_cost.cu           path length, the edge matrix, the learned motion cost of edge rows, states and split edges
//   artp_cnn.cu            the motion-cost network: its weights, features, mode and timing, the trunk and the head (CostNet)
//   artp_inpaint.cu        inpaintMatrix and the cost server's map preparation of a raw layer, on the device
//   artp_roadmap.cu        the PRM roadmap: growth, edge upkeep and the solve (Roadmap)
//   artp_path_simplify.cu  artp_simplify_path: PathSimplifier::simplifyMax on the device (Simplify)
//   artp_planner.cu        artp_planner_set_map / artp_plan: the replan, over the other units' lock-free bodies (PlannerState)
// This header holds the handle and its lock, launch and call bookkeeping, scratch regions, argument checks, and the
// functions one unit calls in another, each under the unit that defines it. It includes no kernel header: each of those
// defines kernels and is compiled into exactly one unit.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <initializer_list>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/artp.h"
#include "artp_device.cuh"

namespace artp_api {

// Host <-> device traffic and host synchronisations of the calls that count them (artp_plan reports its own).
struct Traffic { uint64_t h2d = 0, d2h = 0; uint32_t syncs = 0; };

// The installed map as the other units read it. Only artp_map.cu writes it (upload_map), together with the map fields of
// Handle::chk.
struct MapView {
  bool has_map = false;
  int rows = 0, cols = 0;           // full map
  int pitch = 0;                    // row stride of the layers in floats
  int win_row0 = 0, win_rows = 0;   // rows held by this handle (artp_set_map_window); whole map: 0, rows
  double res = 0.0;                 // map resolution as artp_set_map received it
  // elevation, elevation_masked: the stored win_rows x cols layers (artp::Field::H), not shifted by win_row0
  const float* H[2] = {nullptr, nullptr};
};

// Each unit's state, created by the first call that needs it (Pipeline by artp_create) and released by artp_destroy.
struct Pipeline;       // the validity pipeline's queues, launch shapes, streams and events (artp_capi.cu)
struct MapStore;       // the map's layers, range tables and compact codes (artp_map.cu)
struct Sampling;       // the sampler, the distribution, their layers and what the map has of them (artp_sampling.cu)
struct CostNet;        // the motion-cost network's weights, activations, features, mode and timing (artp_cnn.cu)
struct Roadmap;        // the PRM roadmap store and its query buffers (artp_roadmap.cu)
struct Simplify;       // artp_simplify_path's state pool, path and round buffers (artp_path_simplify.cu)
struct PlannerState;   // artp_planner_set_map / artp_plan (artp_planner.cu)

struct Handle {
  artp_params p;
  int device = 0;
  int sm_count = 0;
  artp::Checker chk;
  char* d_stage = nullptr;          // device staging for the host-buffer API
  size_t stage_cap = 0;
  cudaStream_t stream = nullptr;    // internal compute stream for the host-buffer API
  // Cross-stream ordering of the per-handle scratch (ADVICE r1): calls may come on different streams; every call that
  // uses a scratch group first makes its stream wait for the previous user of that group, and records an event after.
  // group 0: the pipeline's counters and queues / d_stage / the sampling unit's scratch (check, sampler, distribution);
  // group 1: the pipeline's compaction state
  cudaEvent_t chain_ev[2] = {nullptr, nullptr};
  cudaStream_t chain_stream[2] = {nullptr, nullptr};
  bool chain_busy[2] = {false, false};
  // Sticky error word in mapped pinned host memory: the plane-grouping stage sets it when a zone does not fit its
  // shared-memory store (the item is then marked INVALID -- fail closed). Host-buffer calls return ARTP_E_LIMIT from the
  // call that caused it; device-buffer (asynchronous) calls surface it through artp_poll_error().
  uint32_t* h_err = nullptr;        // host view
  uint32_t* d_err = nullptr;        // device view of the same word
  Traffic traffic;
  artp_stats stats{};
  std::string err;
  std::mutex mtx;
  MapView map;
  bool planner_map = false;         // the current map was installed by artp_planner_set_map
  // the units' state
  Pipeline* pipe = nullptr;
  MapStore* map_store = nullptr;
  Sampling* sampling = nullptr;
  CostNet* cost_net = nullptr;
  Roadmap* roadmap = nullptr;
  Simplify* simplify = nullptr;
  PlannerState* planner = nullptr;
};

#define CU_TRY(h, expr)                                                                          \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      (h)->err = std::string(#expr) + ": " + cudaGetErrorString(_e);                             \
      return ARTP_E_CUDA;                                                                        \
    }                                                                                            \
  } while (0)

// Returns the error of a step that failed (ARTP_OK is 0).
#define TRY(expr)                                                                                \
  do {                                                                                           \
    if (const int _rc = (expr)) return _rc;                                                      \
  } while (0)

// Opens an entry point that takes a handle: a null handle is ARTP_E_INVALID; otherwise `h` is the handle, and its lock is
// held until the entry point returns. Entry points never call one another, so no call takes the lock twice.
#define LOCK_HANDLE(h, hh)                                                                       \
  if (!(hh)) return ARTP_E_INVALID;                                                              \
  Handle* h = reinterpret_cast<Handle*>(hh);                                                     \
  std::lock_guard<std::mutex> h##_lock(h->mtx)

// Set up by LOCK_CALL: on every return path of the call it sets stats.last_launches to the number of kernels the call
// launched.
struct CallScope {
  Handle* h;
  uint64_t launches0;
  explicit CallScope(Handle* h_) : h(h_), launches0(h_->stats.kernel_launches) {}
  ~CallScope() { h->stats.last_launches = (uint32_t)(h->stats.kernel_launches - launches0); }
};
// LOCK_HANDLE for the entry points that launch kernels.
#define LOCK_CALL(h, hh)                                                                         \
  LOCK_HANDLE(h, hh);                                                                            \
  CallScope h##_call(h)

// Checks the kernel launch just issued and counts it in stats.kernel_launches.
inline int count_launch(Handle* h) {
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 1;
  return ARTP_OK;
}

// kernel<<<grid, block, smem, s>>>(args...), checked and counted.
template <typename... P, typename... A>
int launch(Handle* h, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, A&&... args) {
  kernel<<<grid, block, smem, s>>>(std::forward<A>(args)...);
  return count_launch(h);
}

// Grid-stride launches: enough blocks for n items, at most `per_sm` blocks per SM.
inline unsigned grid_for(const Handle* h, size_t n, int block, size_t per_sm = 16) {
  return (unsigned)std::min<size_t>((n + block - 1) / block, (size_t)h->sm_count * per_sm);
}

inline int require_map(Handle* h) {
  if (!h->map.has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  return ARTP_OK;
}
// The calls over whole-map layers (sampler, normals, distribution, features) refuse a map window.
inline int require_whole_map(Handle* h) {
  TRY(require_map(h));
  if (h->map.win_rows != h->map.rows) { h->err = "not available on a map window (artp_set_map_window)"; return ARTP_E_INVALID; }
  return ARTP_OK;
}
inline int null_buffer(Handle* h) {
  h->err = "null buffer";
  return ARTP_E_INVALID;
}

// Grow a per-handle device buffer to hold `count` elements (cap counts them too); the contents are not kept. Rare (growth
// only): the device is synchronised before the free, because a call on any stream may still read the old buffer.
template <typename T>
int grow(Handle* h, T*& buf, size_t& cap, size_t count) {
  if (cap >= count) return ARTP_OK;
  CU_TRY(h, cudaDeviceSynchronize());
  cudaFree(buf);
  buf = nullptr;
  cap = 0;
  CU_TRY(h, cudaMalloc(&buf, count * sizeof(T)));
  cap = count;
  return ARTP_OK;
}

// Scratch regions: grows `buf` (contents not kept) to hold region[i] = bytes[i] bytes, each at a 256-byte boundary.
inline int carve(Handle* h, char*& buf, size_t& cap, std::initializer_list<size_t> bytes, char** region) {
  size_t end = 0;
  for (size_t b : bytes) end = ((end + 255) & ~(size_t)255) + b;
  TRY(grow(h, buf, cap, end));
  end = 0;
  for (size_t b : bytes) {
    end = (end + 255) & ~(size_t)255;
    *region++ = buf + end;
    end += b;
  }
  return ARTP_OK;
}

// Scratch-group ordering across streams (see Handle::chain_ev): a call on stream s that uses group g waits for the
// group's previous user, and records itself as the next one when it ends.
inline int chain_begin(Handle* h, int g, cudaStream_t s) {
  if (h->chain_busy[g] && h->chain_stream[g] != s) CU_TRY(h, cudaStreamWaitEvent(s, h->chain_ev[g], 0));
  return ARTP_OK;
}
inline int chain_end(Handle* h, int g, cudaStream_t s) {
  CU_TRY(h, cudaEventRecord(h->chain_ev[g], s));
  h->chain_stream[g] = s;
  h->chain_busy[g] = true;
  return ARTP_OK;
}
struct ChainScope {   // begin on construction, end on destruction (every return path)
  Handle* h; int g; cudaStream_t s; int rc;
  ChainScope(Handle* h_, int g_, cudaStream_t s_) : h(h_), g(g_), s(s_), rc(chain_begin(h_, g_, s_)) {}
  ~ChainScope() { if (rc == ARTP_OK) chain_end(h, g, s); }
};

// Sticky plane-grouping overflow (set by the device, see Handle::h_err): read and clear (artp_capi.cu).
int take_sticky_error(Handle* h);

// Copies and synchronisations counted in Handle::traffic (the paths artp_plan takes use these).
inline int copy_async(Handle* h, void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, cudaStream_t s) {
  CU_TRY(h, cudaMemcpyAsync(dst, src, bytes, kind, s));
  if (kind == cudaMemcpyHostToDevice) h->traffic.h2d += bytes;
  if (kind == cudaMemcpyDeviceToHost) h->traffic.d2h += bytes;
  return ARTP_OK;
}
inline int sync_stream(Handle* h, cudaStream_t s) {
  CU_TRY(h, cudaStreamSynchronize(s));
  h->traffic.syncs += 1;
  return ARTP_OK;
}

// Host-buffer calls run on h->stream as users of scratch group 0. host_call_begin waits for the group's previous user and
// hands out region[i] = bytes[i] bytes of d_stage (carve). host_call_end waits for the call's work, after which the group
// is idle. For a call that ran the validity pipeline (`pipeline`) it then returns the sticky device error (Handle::h_err)
// of the call; the verdicts are complete (fail closed) then, so only ARTP_E_CUDA from host_call_end means the call's
// outputs are not there.
inline int host_call_begin(Handle* h, std::initializer_list<size_t> bytes = {}, char** region = nullptr) {
  CU_TRY(h, cudaSetDevice(h->device));
  TRY(chain_begin(h, 0, h->stream));
  return carve(h, h->d_stage, h->stage_cap, bytes, region);
}
inline int host_call_end(Handle* h, bool pipeline = false) {
  TRY(sync_stream(h, h->stream));
  h->chain_busy[0] = false;
  return pipeline ? take_sticky_error(h) : ARTP_OK;
}
// Device-buffer calls that use scratch group 0 run on the caller's stream: device_call sets the device, then returns
// run(s) on that stream s as the group's user (ChainScope, so the group's next user waits for run's work).
template <class Run>
int device_call(Handle* h, void* stream, Run run) {
  CU_TRY(h, cudaSetDevice(h->device));
  const cudaStream_t s = (cudaStream_t)stream;
  const ChainScope cs(h, 0, s);
  return cs.rc ? cs.rc : run(s);
}

// Functions one unit calls in another, by the unit that defines them. A function named after an entry point is that entry
// point's body without the lock; artp_planner_set_map and artp_plan chain them.

// ---- artp_capi.cu: the validity pipeline ----
// The validity pipeline over n float states on the device (Pose3FromSE3's cast already applied) into d_valid, on s.
int check_states_f32(Handle* h, const float* d_states, size_t n, uint8_t* d_valid, cudaStream_t s);
// Its explain form: the ARTP_BOX_* word of each state into d_why (artp_box_verdicts), on s.
int box_verdicts_f32(Handle* h, const float* d_states, size_t n, uint16_t* d_why, cudaStream_t s);
// Ordered compaction of the n flags d_valid (bit-packed with `bits`) into the indices base + i of the set ones and their
// count, int64_t indices or, with `u32`, uint32_t ones. Uses scratch group 1.
int compact_valid(Handle* h, const uint8_t* d_valid, size_t n, int64_t base, void* d_indices, uint32_t* d_count, cudaStream_t s,
                  bool bits = false, bool u32 = false);
// The latency path's per-pose routine, one CTA per state, over the device states 0 .. *d_count - 1 (at most max_n, which
// sizes the grid) into d_valid, on s; nothing once *d_stop is set (the roadmap's interior states).
int check_states_cta(Handle* h, const double* d_states, const uint32_t* d_count, const uint32_t* d_stop, size_t max_n,
                     uint8_t* d_valid, cudaStream_t s);
// For upload_map, before any of its work: the grouping stage's plane store for zones of at most tcap triangles. Applies
// the artp_debug_set_group_capacity hook and the rounding to tcap and gives the store's bytes; ARTP_E_LIMIT when the
// store does not fit the stage's shared memory.
int plane_store(Handle* h, int& tcap, int& store);
// For upload_map, once the map is installed (Handle::map, chk): the box kernels' launch shapes from each box's zone
// bound span and the plane store: occupancy grids, tile maps, chk's reach tile.
int set_shapes(Handle* h, const int span[2][2], int tcap, int store);

// ---- artp_map.cu: the installed map ----
// artp_set_map_window's work. device_src: the two layers are DEVICE pointers (rows x cols, grid_map layout) and the
// compact-code scales come from a device reduction instead of a host pass.
int upload_map(Handle* h, const float* elevation, const float* elevation_masked, bool device_src, int rows, int cols,
               double res, double cx, double cy, int row0, int nrows);
// Finite minimum and maximum of n floats (-0 counted as +0) on s: d_out = {key(min), key(max), finite count} with
// order-preserving keys; key_float turns a key back into its float.
int finite_min_max(Handle* h, const float* d_layer, size_t n, uint32_t* d_out, cudaStream_t s);
float key_float(uint32_t key);
// Whether any of n floats is NaN or +-inf (d_out[0]) and whether any is +-inf (d_out[1]), 0 or 1, on s.
int nonfinite_any(Handle* h, const float* d_layer, size_t n, uint32_t* d_out, cudaStream_t s);
void map_free(Handle* h);

// ---- artp_sampling.cu: the sampler, the distribution and the map-derived layers ----
// upload_map forgets what the unit derived from the previous map; artp_destroy frees the rest.
void sampling_forget_map(Handle* h);
void sampling_free(Handle* h);
// The density blur radius of the reference's Planner (planner.cpp:48).
inline double density_blur_radius(const artp_params& p) { return (p.torso_length + p.torso_width) * 0.25; }
// For the roadmap: a map and an armed sampler (ARTP_E_NOMAP otherwise).
int sampler_armed(Handle* h);
// artp_sample_valid_device's work on s, with the draw index of every kept state into d_draws (capacity entries).
int sample_valid_draws(Handle* h, uint64_t seed, uint64_t first_sample, size_t n_draw, double* d_states_out, uint64_t* d_draws,
                       size_t capacity, uint32_t* d_count, cudaStream_t s);
// artp_update_sample_distribution_device's argument checks and work (n vertex states on the device, NaN ones not
// counted) on s; the sampler is re-armed on the new CDF.
int check_distribution_args(Handle* h, const artp_sample_distribution_params* dp);
int update_distribution_rearm(Handle* h, const artp_sample_distribution_params* dp, const double* d_states, size_t n,
                              cudaStream_t s);
// Basic over the device layers L[0, n) elevation, L[n, 2n) traversability, L[2n, 3n) observed (read when has_observed)
// with 6 more layers of scratch behind them; elevation_masked ends at L + 8n, traversability_thresholded at L + 5n, and
// both Basic layers are kept for set_sample_filter_basic. Structuring elements above 64 cells: ARTP_E_LIMIT.
int process_basic(Handle* h, float* L, int rows, int cols, double res, const artp_basic_params* bp, bool has_observed,
                  cudaStream_t s);
// The size limits the map chain would hit at resolution res (ARTP_E_LIMIT): Basic's structuring elements, and with
// `distribution` the sample filter's and (inverse_density) the density blur's.
int map_chain_limits(Handle* h, const artp_basic_params* bp, double res, bool distribution, bool inverse_density);
int estimate_normals(Handle* h, double estimation_radius, cudaStream_t s);
int set_sample_filter_basic(Handle* h, cudaStream_t s);   // artp_set_sample_filter(h, NULL, NULL, NULL)
// Points the sampler at the resident layers (the CDF too when it samples from the distribution): with sp, as
// artp_set_sampler(h, sp, NULL x 6) without its CDF validation; without, keeping its view and parameters.
void arm_sampler(Handle* h, const artp_sampler_params* sp);
int ball_search(Handle* h, const double* d_centres, size_t n, const double* d_radius, uint32_t n_iter, uint64_t seed,
                uint64_t first_draw, double* d_states_out, int32_t* d_index, cudaStream_t s);
int pose_from_2d(Handle* h, const double* d_in, size_t n, double* d_out, uint8_t* d_inside, cudaStream_t s);

// ---- artp_cost.cu: path length and the learned motion cost ----
// The loaded network's weights of roadmap edges on s, from the store's states and (u, v) pairs into d_ecost / d_eflag:
// edges 0 .. n-1 in their stored direction, feasible ones marked valid (updateEdges), or, with d_list, the first *d_count
// (at most n) listed edges in the listed direction, validity untouched (computeCostForVertexEdges). d_rows: n x 6 floats,
// d_cost3: n x 3 floats of scratch. ARTP_E_NOWEIGHTS without weights and features.
int price_store_edges(Handle* h, const double* d_states, const uint32_t* d_edges, const uint32_t* d_list,
                      const uint32_t* d_count, size_t n, float* d_rows, float* d_cost3, double* d_ecost, uint8_t* d_eflag,
                      cudaStream_t s);
// PathLengthObjective::motionCost of n edges (d_s1[i] -> d_s2[i]) into d_cost on s.
int path_length_cost(Handle* h, const double* d_s1, const double* d_s2, size_t n, double* d_cost, cudaStream_t s);
// MotionCostObjective::motionCost of n edges with the piece offsets d_piece_off (n + 1, total_pieces in all) on s: piece
// rows, the head, the per-edge reduction (artp_motion_cost_split_device's work).
int motion_cost_split(Handle* h, const double* d_s1, const double* d_s2, size_t n, const uint32_t* d_piece_off,
                      size_t total_pieces, float* d_rows, float* d_cost3, double* d_cost, cudaStream_t s);
// The piece offsets of motionCost's split of the n HOST edges (s1 + 7 e, s2 + 7 e) at max_query_edge_length: off (n + 1
// entries, exclusive, then the total) and *total. ARTP_E_INVALID when an edge or the total has 2^32 pieces or more.
int cost_piece_offsets(Handle* h, const double* s1, const double* s2, size_t n, double max_query_edge_length,
                       std::vector<uint32_t>& off, size_t* total);
// The same offsets of the n - 1 edges of the DEVICE path d_states (n entries, exclusive, then the total) on s; *total is
// read back (one synchronisation). ARTP_E_INVALID for an edge of 2^32 pieces or more.
int piece_offsets(Handle* h, const double* d_states, size_t n, double max_query_edge_length, uint32_t* d_off, size_t* total,
                  cudaStream_t s);

// ---- artp_cnn.cu: the motion-cost network ----
// The loaded network (ARTP_COST_NET_*), -1 without weights. check_cost_weights: ARTP_E_NOWEIGHTS without weights;
// check_cost_net: without weights and features.
int cost_network(const Handle* h);
int check_cost_weights(Handle* h);
int check_cost_net(Handle* h);
// CostPredictor.updateFeatures after check_cost_weights: the trunk over the rows x cols heightfield layer d_layer (as
// artp_set_map stores one, at `pitch`) on s, one synchronisation of s; the head then reads the map's geometry res, cx,
// cy. map_features: over the installed map's elevation on h->stream.
int update_features(Handle* h, const float* d_layer, int rows, int cols, int pitch, double res, double cx, double cy,
                    cudaStream_t s);
int map_features(Handle* h);
// The head over n edge rows d_edges (n x 6) into d_cost3 (n x 3) on s, after check_cost_net: one launch, none for n = 0.
int cost_head(Handle* h, const float* d_edges, size_t n, float* d_cost3, cudaStream_t s);
void cost_net_free(Handle* h);

// ---- artp_inpaint.cu: inpaintMatrix and the cost server's map preparation ----
// inpaintMatrix (artp_inpaint.cuh) of the rows x cols column-major layer d_in into d_out on s; d_mm holds the layer's
// finite_min_max words (at least one finite cell). Scratch is stream-ordered (cudaMallocAsync).
int inpaint_layer(Handle* h, const float* d_in, int rows, int cols, const uint32_t* d_mm, float* d_out, cudaStream_t s);
// The cost server's map preparation (artp_inpaint.cuh). The words of a layer are
// {finite_min_max's three, nonfinite_any's two}: cost_map_scan enqueues them into d_w on s, and cost_map_verdict, on
// their host copy, refuses the layers the server cannot prepare (ARTP_E_INVALID, artp.h). cost_map_layer then prepares the
// rows x cols column-major layer d_in into d_out (its grid_map layout, or with reverse_cols the trunk's heightfield layout
// at pitch rows); cost_map_features prepares it and runs the trunk on it (update_features's geometry and codes).
// Scratch is stream-ordered.
constexpr int kCostMapWords = 5;
int cost_map_scan(Handle* h, const float* d_in, size_t n, uint32_t* d_w, cudaStream_t s);
int cost_map_verdict(Handle* h, const uint32_t* w);
int cost_map_layer(Handle* h, const float* d_in, int rows, int cols, const uint32_t* d_w, bool holes, bool reverse_cols,
                   float* d_out, cudaStream_t s);
int cost_map_features(Handle* h, const float* d_in, int rows, int cols, const uint32_t* d_w, bool holes, double res,
                      double cx, double cy, cudaStream_t s);

// ---- artp_roadmap.cu: the PRM roadmap ----
int roadmap_clear(Handle* h, size_t vertex_capacity, size_t edge_capacity);
bool has_roadmap(const Handle* h);
int roadmap_sample_graph(Handle* h, const artp_roadmap_params* rp, const artp_sample_distribution_params* dp, uint64_t seed,
                         uint64_t first_sample, uint64_t* draws_used);
int roadmap_update_edges(Handle* h);
void roadmap_counts(const Handle* h, size_t* nv, size_t* ne);
// artp_roadmap_solve's work; with d_sg (DEVICE: start then goal, 14 doubles) the endpoints are not read on the host: a
// device check gives their bounds verdict and (x, y), and d_path_out (DEVICE, path_capacity x 7) receives the path instead
// of path_states.
int roadmap_solve(Handle* h, const double* start, const double* goal, const double* d_sg, const artp_se3_space* space,
                  double* path_states, double* d_path_out, size_t path_capacity, size_t* n_path, double* cost,
                  artp_roadmap_solve_info* info);
void roadmap_free(Handle* h);

// ---- artp_path_simplify.cu: the path simplifier ----
// artp_simplify_path's work; with d_path (DEVICE, n states) the pool is seeded on the device and the learned cost's piece
// offsets are computed there.
int simplify_path(Handle* h, const double* path, const double* d_path, size_t n, const artp_se3_space* space, int objective,
                  double max_query_edge_length, uint64_t seed, double* out, size_t capacity, size_t* n_out,
                  artp_simplify_info* info);
void simplify_free(Handle* h);

// ---- artp_planner.cu: the replan ----
void planner_free(Handle* h);

}  // namespace artp_api
