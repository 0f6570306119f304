// art_planner_b200/csrc/artp_planner.cu -- Planner::setMap and Planner::plan + getSolutionPath for prm_motion_cost
// (art_planner/src/planner.cpp:135-298) as two calls of the C ABI (include/artp.h): artp_planner_set_map and artp_plan.
// The stages are the ones the public entry points run (their bodies without the lock, artp_internal.h); between them every
// layer, state and path stays in device memory. The kernels here are the planner's own: the "observed" layer and the
// goal's bounds clip.
#include <cfloat>
#include <cmath>

#include "artp_internal.h"

using namespace artp_api;

namespace artp_api {

struct PlannerState {
  float* d_layers = nullptr;         // raw elevation | raw traversability | Basic's 9 layers (artp_api::process_basic)
  size_t layers_cap = 0;             // floats
  double* d_q = nullptr;             // query block (QB_* offsets)
  double* d_path = nullptr;          // the solved path (vertex capacity x 7)
  size_t path_cap = 0;               // states
  artp_se3_space space{};
  uint64_t generation = 0;           // map generation: stands in for the grid_map timestamp sampleGraph compares
  uint64_t sampled_generation = 0;   // the generation the last sampleGraph saw
  bool seeded = false;
  uint64_t seed = 0, next_sample = 0, start_draw = 0, goal_draw = 0, simplify_calls = 0;
  cudaEvent_t ev[6] = {};
};

}  // namespace artp_api

namespace {

// Offsets (in doubles) of the query block d_q.
enum : size_t {
  QB_START = 0, QB_GOAL = 7, QB_CLIPPED = 14, QB_PROJECTED = 21, QB_REPAIRED = 28 /* start, goal: 14 */, QB_RADIUS = 42,
  QB_FLAGS = 44 /* inside byte, clipped byte, two int32 ball indices */, QB_MINMAX = 46, QB_SIZE = 64
};

// addKnownCells (basic.cpp:25-38): observed = 1 where every basic layer ({elevation, traversability}, map.cpp:16) is finite
// (grid_map's isValid). A missing traversability layer is checkTraversability's 1.0 (basic.cpp:13-21), written to trav_fill.
__global__ void observed_kernel(const float* __restrict__ elevation, const float* __restrict__ traversability, size_t n,
                                float* __restrict__ observed, float* __restrict__ trav_fill) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    bool ok = fabsf(elevation[i]) < CUDART_INF_F;
    if (traversability) ok = ok && fabsf(traversability[i]) < CUDART_INF_F;
    else trav_fill[i] = 1.0f;
    observed[i] = ok ? 1.0f : 0.0f;
  }
}

constexpr double kQuatNormError = 1e-9;   // SO3StateSpace's MAX_QUATERNION_NORM_ERROR

// Planner::plan :207-221: satisfiesBounds, else enforceBounds, of the SE(3) goal. R3: RealVectorStateSpace's test with the
// DBL_EPSILON slack, then the clamp. SO3: satisfiesBounds is |norm - 1| < 1e-9; enforceBounds normalises when the SQUARED
// norm differs from 1 by more than DBL_EPSILON, to the identity when the norm is below DBL_EPSILON.
__global__ void goal_clip_kernel(const double* __restrict__ in, artp_se3_space sp, double* __restrict__ out,
                                 uint8_t* __restrict__ clipped) {
  double s[7];
  for (int k = 0; k < 7; ++k) s[k] = in[k];
  bool ok = true;
  for (int i = 0; i < 3; ++i)
    if (s[i] - DBL_EPSILON > sp.high[i] || s[i] + DBL_EPSILON < sp.low[i]) ok = false;
  const double nrm_sq = s[3] * s[3] + s[4] * s[4] + s[5] * s[5] + s[6] * s[6];
  const double norm = sqrt(nrm_sq);
  if (!(fabs(norm - 1.0) < kQuatNormError)) ok = false;
  if (!ok) {
    for (int i = 0; i < 3; ++i) {
      if (s[i] > sp.high[i]) s[i] = sp.high[i];
      else if (s[i] < sp.low[i]) s[i] = sp.low[i];
    }
    if (fabs(nrm_sq - 1.0) > DBL_EPSILON) {
      if (norm < DBL_EPSILON) { s[3] = s[4] = s[5] = 0.0; s[6] = 1.0; }
      else for (int k = 3; k < 7; ++k) s[k] /= norm;
    }
  }
  for (int k = 0; k < 7; ++k) out[k] = s[k];
  *clipped = ok ? 0 : 1;
}

int planner_status(int32_t solve_status) {   // planner.cpp:254-261
  switch (solve_status) {
    case ARTP_SOLVE_SOLVED: return ARTP_PLANNER_SOLVED;
    case ARTP_SOLVE_NOT_CONNECTED: case ARTP_SOLVE_NO_FEASIBLE_PATH: return ARTP_PLANNER_NOT_SOLVED;
    case ARTP_SOLVE_INVALID_START: return ARTP_PLANNER_INVALID_START;
    case ARTP_SOLVE_INVALID_GOAL: return ARTP_PLANNER_INVALID_GOAL;
    default: return ARTP_PLANNER_UNKNOWN;
  }
}

PlannerState* planner_of(Handle* h) {
  if (!h->planner) h->planner = new PlannerState();
  return h->planner;
}

artp_sample_distribution_params dist_params(const Handle* h, const artp_planner_params* pp) {
  artp_sample_distribution_params dp{};
  dp.use_inverse_vertex_density = pp->use_inverse_vertex_density;
  dp.density_blur_radius = density_blur_radius(h->p);
  dp.use_max_prob_unknown_samples = pp->use_max_prob_unknown_samples;
  dp.max_prob_unknown_samples = pp->max_prob_unknown_samples;
  return dp;
}

int plan_args(Handle* h, const artp_planner_params* pp) {
  if (!pp) return null_buffer(h);
  if (!(pp->start_radius >= 0.0 && std::isfinite(pp->start_radius) && pp->goal_radius >= 0.0 && std::isfinite(pp->goal_radius))) {
    h->err = "start_radius and goal_radius must be finite and >= 0"; return ARTP_E_INVALID;
  }
  if (pp->max_n_vertices >= 0xFFFFFFFFull || pp->max_n_edges >= 0xFFFFFFFFull ||
      pp->recompute_density_after_n_samples >= 0xFFFFFFFFull) {
    h->err = "roadmap caps must be < 2^32"; return ARTP_E_INVALID;
  }
  if (pp->vertex_capacity == 0 || pp->edge_capacity == 0 || pp->vertex_capacity >= 0x7FFFFFFFull || pp->edge_capacity >= 0x7FFFFFFFull) {
    h->err = "roadmap capacities must be > 0 and < 2^31"; return ARTP_E_INVALID;
  }
  if (pp->n_iter >= 0xFFFFFFFFu) { h->err = "n_iter must be < 2^32 - 1"; return ARTP_E_INVALID; }
  if (pp->simplify && !(pp->max_query_edge_length > 0.0)) { h->err = "max_query_edge_length must be > 0"; return ARTP_E_INVALID; }
  if (pp->use_max_prob_unknown_samples && !(pp->max_prob_unknown_samples >= 0.0 && pp->max_prob_unknown_samples <= 1.0)) {
    h->err = "max_prob_unknown_samples must lie in [0, 1]"; return ARTP_E_INVALID;
  }
  if (pp->cost_map_from_raw != 0 && pp->cost_map_from_raw != 1) { h->err = "cost_map_from_raw must be 0 or 1"; return ARTP_E_INVALID; }
  return ARTP_OK;
}

int record(Handle* h, PlannerState* st, int i) {
  CU_TRY(h, cudaEventRecord(st->ev[i], h->stream));
  return ARTP_OK;
}

}  // namespace

void artp_api::planner_free(Handle* h) {
  PlannerState* st = h->planner;
  if (!st) return;
  cudaFree(st->d_layers); cudaFree(st->d_q); cudaFree(st->d_path);
  for (cudaEvent_t e : st->ev) if (e) cudaEventDestroy(e);
  delete st;
  h->planner = nullptr;
}

namespace {

// artp_planner_set_map's body. raw: the inpainted layers are made on the device from the uploaded raw ones (the
// *_inpainted arguments are unused).
// The two layers' marches are independent: the traversability's runs on a second stream beside the elevation's, which
// matters when one giant component leaves most SMs idle. d_mm: the elevation's min / max words, the traversability's at +4.
int inpaint_both(Handle* h, const float* raw_e, const float* raw_t, int rows, int cols, const uint32_t* d_mm, float* L,
                 cudaStream_t s) {
  if (!raw_t) return inpaint_layer(h, raw_e, rows, cols, d_mm, L, s);
  const size_t n = (size_t)rows * cols;
  cudaStream_t s2 = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  int rc = ARTP_OK;
  auto cu = [&](cudaError_t e) { if (rc == ARTP_OK && e != cudaSuccess) { h->err = cudaGetErrorString(e); rc = ARTP_E_CUDA; } };
  cu(cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking));
  for (auto& e : ev) cu(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  cu(cudaEventRecord(ev[0], s));
  cu(cudaStreamWaitEvent(s2, ev[0], 0));
  if (rc == ARTP_OK) rc = inpaint_layer(h, raw_t, rows, cols, d_mm + 4, L + n, s2);
  if (rc == ARTP_OK) rc = inpaint_layer(h, raw_e, rows, cols, d_mm, L, s);
  cu(cudaEventRecord(ev[1], s2));
  cu(cudaStreamWaitEvent(s, ev[1], 0));
  for (auto e : ev) if (e) cudaEventDestroy(e);
  if (s2) cudaStreamDestroy(s2);   // released once its work is done
  return rc;
}

int set_map(Handle* h, const artp_planner_params* pp, const float* elevation, const float* traversability,
            const float* elevation_inpainted, const float* traversability_inpainted, bool raw, int rows, int cols,
            double res, double cx, double cy, artp_planner_map_info* info) {
  // every check before any work: a refused map leaves the previous one installed
  if (!pp || !elevation || (!raw && !elevation_inpainted)) return null_buffer(h);
  if (!raw && !traversability != !traversability_inpainted) {
    h->err = "pass both traversability layers (raw and inpainted) or neither"; return ARTP_E_INVALID;
  }
  if (raw && (size_t)rows * cols >= 0x7FFFFFFFull) { h->err = "inpaint: rows * cols must be < 2^31"; return ARTP_E_INVALID; }
  if (rows < 2 || cols < 2 || !(res > 0) || !std::isfinite(cx) || !std::isfinite(cy)) { h->err = "bad map arguments"; return ARTP_E_INVALID; }
  TRY(plan_args(h, pp));
  TRY(map_chain_limits(h, &pp->basic, res, pp->sample_from_distribution != 0, pp->use_inverse_vertex_density != 0));
  PlannerState* st = planner_of(h);
  const size_t n = (size_t)rows * cols, lb = n * sizeof(float);
  const Traffic t0 = h->traffic;
  TRY(host_call_begin(h));
  cudaStream_t s = h->stream;
  TRY(grow(h, st->d_layers, st->layers_cap, 11 * n));
  float *raw_e = st->d_layers, *raw_t = st->d_layers + n, *L = st->d_layers + 2 * n;
  TRY(copy_async(h, raw_e, elevation, lb, cudaMemcpyHostToDevice, s));
  if (!raw) TRY(copy_async(h, L, elevation_inpainted, lb, cudaMemcpyHostToDevice, s));
  if (traversability) {
    TRY(copy_async(h, raw_t, traversability, lb, cudaMemcpyHostToDevice, s));
    if (!raw) TRY(copy_async(h, L + n, traversability_inpainted, lb, cudaMemcpyHostToDevice, s));
  }
  // observed, and the SE(3) bounds from the RAW elevation (planner.cpp:146-156)
  TRY(launch(h, observed_kernel, grid_for(h, n, 256), 256, 0, s, raw_e, traversability ? raw_t : nullptr, n, L + 2 * n, L + n));
  if (!st->d_q) CU_TRY(h, cudaMalloc(&st->d_q, QB_SIZE * sizeof(double)));
  uint32_t* d_mm = reinterpret_cast<uint32_t*>(st->d_q + QB_MINMAX);
  TRY(finite_min_max(h, raw_e, n, d_mm, s));
  const bool raw_t_inpaint = raw && traversability;
  if (raw_t_inpaint) TRY(finite_min_max(h, raw_t, n, d_mm + 4, s));   // inpaintMatrix's range of the traversability
  const bool cost_map = pp->cost_map_from_raw != 0;
  if (cost_map) TRY(cost_map_scan(h, raw_e, n, d_mm + 8, s));        // the cost server's preparation of the elevation
  uint32_t mm[8 + kCostMapWords];
  TRY(copy_async(h, mm, d_mm, (cost_map ? 8 + kCostMapWords : raw_t_inpaint ? 8 : 3) * sizeof(uint32_t),
                 cudaMemcpyDeviceToHost, s));
  TRY(host_call_end(h));
  if (!mm[2]) { h->err = "the elevation layer has no finite cell"; return ARTP_E_INVALID; }
  if (raw_t_inpaint && !mm[6]) { h->err = "the traversability layer has no finite cell"; return ARTP_E_INVALID; }
  if (cost_map) TRY(cost_map_verdict(h, mm + 8));
  artp_se3_space sp{};
  const double Lx = rows * res, Ly = cols * res;   // grid_map getLength: the FULL length, not half of it
  sp.low[0] = cx - Lx; sp.high[0] = cx + Lx;
  sp.low[1] = cy - Ly; sp.high[1] = cy + Ly;
  sp.low[2] = (double)key_float(mm[0]) - h->p.reach_z / 2;
  sp.high[2] = (double)key_float(mm[1]) + h->p.reach_z / 2;
  sp.longest_valid_segment_fraction = 0.01;
  // processors::Basic, then the upload of the elevation and the masked layer straight from device memory. From here on a
  // failure (only a CUDA error can remain) leaves no planner map.
  h->planner_map = false;
  TRY(host_call_begin(h));
  if (raw) {   // processors::Basic's inpaintMatrix calls (basic.cpp:42-45), from the raw layers already on the device
    TRY(inpaint_both(h, raw_e, traversability ? raw_t : nullptr, rows, cols, d_mm, L, s));
  }
  TRY(process_basic(h, L, rows, cols, res, &pp->basic, true, s));
  TRY(host_call_end(h));
  TRY(upload_map(h, L, L + 8 * n, true, rows, cols, res, cx, cy, 0, rows));
  // the rest of the new-map chain (planner.cpp:39-58): normals, sample filter, distribution without vertices, CDF, sampler
  TRY(host_call_begin(h));
  TRY(estimate_normals(h, (h->p.torso_length + h->p.torso_width) * 0.25, s));
  artp_sampler_params smp{};
  smp.max_roll_pert = pp->max_roll_pert; smp.max_pitch_pert = pp->max_pitch_pert;
  smp.sample_from_distribution = pp->sample_from_distribution;
  smp.low[0] = sp.low[0]; smp.low[1] = sp.low[1]; smp.high[0] = sp.high[0]; smp.high[1] = sp.high[1];
  if (pp->sample_from_distribution) {
    TRY(set_sample_filter_basic(h, s));
    const artp_sample_distribution_params dp = dist_params(h, pp);
    TRY(update_distribution_rearm(h, &dp, nullptr, 0, s));
  }
  arm_sampler(h, &smp);
  TRY(host_call_end(h));
  // CostPredictor.updateFeatures, when a network is loaded: on the uploaded elevation, or with cost_map_from_raw on the
  // cost server's preparation of the raw one
  if (cost_network(h) >= 0) {
    CU_TRY(h, cudaSetDevice(h->device));
    if (cost_map) TRY(cost_map_features(h, raw_e, rows, cols, d_mm + 8, mm[8 + 3] != 0, h->map.res, h->chk.cx, h->chk.cy, h->stream));
    else TRY(map_features(h));
  }
  st->space = sp;
  st->generation += 1;
  h->planner_map = true;
  if (info) {
    CU_TRY(h, cudaStreamSynchronize(h->stream));   // the features' kernels are part of the call
    info->host_syncs = h->traffic.syncs - t0.syncs + 1;
    info->bytes_h2d = h->traffic.h2d - t0.h2d;
    info->bytes_d2h = h->traffic.d2h - t0.d2h;
  }
  return ARTP_OK;
}

}  // namespace

extern "C" {

int artp_planner_set_map(artp_handle* hh, const artp_planner_params* pp, const float* elevation, const float* traversability,
                         const float* elevation_inpainted, const float* traversability_inpainted, int rows, int cols,
                         double res, double cx, double cy, artp_planner_map_info* info) {
  LOCK_CALL(h, hh);
  return set_map(h, pp, elevation, traversability, elevation_inpainted, traversability_inpainted, false, rows, cols, res,
                 cx, cy, info);
}

int artp_planner_set_map_raw(artp_handle* hh, const artp_planner_params* pp, const float* elevation,
                             const float* traversability, int rows, int cols, double res, double cx, double cy,
                             artp_planner_map_info* info) {
  LOCK_CALL(h, hh);
  return set_map(h, pp, elevation, traversability, nullptr, nullptr, true, rows, cols, res, cx, cy, info);
}

int artp_planner_get_space(artp_handle* hh, artp_se3_space* out) {
  LOCK_HANDLE(h, hh);
  if (!out) return null_buffer(h);
  if (!h->planner_map) { h->err = "no map set by artp_planner_set_map"; return ARTP_E_NOMAP; }
  *out = h->planner->space;
  return ARTP_OK;
}

int artp_plan(artp_handle* hh, const artp_planner_params* pp, const double* start, const double* goal, double* path,
              size_t capacity, size_t* n_path, artp_plan_info* info) {
  LOCK_CALL(h, hh);
  if (!start || !goal) return null_buffer(h);
  TRY(plan_args(h, pp));
  for (int i = 0; i < 7; ++i)
    if (!std::isfinite(start[i]) || !std::isfinite(goal[i])) { h->err = "non-finite start or goal"; return ARTP_E_INVALID; }
  if (n_path) *n_path = 0;
  artp_plan_info o{};
  o.solve.path_vertices = info ? info->solve.path_vertices : nullptr;
  o.start_index = o.goal_index = -1;
  if (h->map.has_map && h->map.win_rows != h->map.rows) {
    h->err = "not available on a map window (artp_set_map_window)"; return ARTP_E_INVALID;
  }
  if (!h->planner_map) {                                   // planner.cpp:197-200
    o.status = ARTP_PLANNER_NO_MAP;
    if (info) *info = o;
    return ARTP_OK;
  }
  TRY(check_cost_net(h));                                  // the learned objective prices the edges
  const artp_sample_distribution_params dp = dist_params(h, pp);
  if (pp->sample_from_distribution) TRY(check_distribution_args(h, &dp));   // sampleGraph's recomputes: their limits first
  PlannerState* st = h->planner;
  const Traffic t0 = h->traffic;
  for (auto& e : st->ev)
    if (!e) CU_TRY(h, cudaEventCreate(&e));
  if (!st->seeded || st->seed != pp->seed) {   // a new seed starts every stream at its beginning
    st->seeded = true; st->seed = pp->seed;
    st->next_sample = st->start_draw = st->goal_draw = st->simplify_calls = 0;
  }
  cudaStream_t s = h->stream;
  // PRMMotionCost::clear (the ROS node's ss_->clear(), planner_ros.cpp:359,373), or the first roadmap of this handle
  if (pp->clear_roadmap || !has_roadmap(h)) TRY(roadmap_clear(h, pp->vertex_capacity, pp->edge_capacity));
  size_t nv = 0, ne = 0;
  // PRMMotionCost::solve -> sampleGraph: sample and updateEdges only when the map changed (prm_motion_cost.cpp:146-153)
  TRY(record(h, st, 0));
  o.first_sample = st->next_sample;
  if (st->sampled_generation != st->generation) {
    artp_roadmap_params rp{pp->max_n_vertices, pp->max_n_edges, pp->recompute_density_after_n_samples, pp->max_draws};
    uint64_t used = 0;
    TRY(roadmap_sample_graph(h, &rp, pp->sample_from_distribution ? &dp : nullptr, pp->seed, st->next_sample, &used));
    TRY(record(h, st, 1));
    TRY(roadmap_update_edges(h));
    st->sampled_generation = st->generation;
    st->next_sample += used;
    o.sampled = 1;
    o.draws_used = used;
  } else {
    TRY(record(h, st, 1));
  }
  TRY(host_call_begin(h));
  TRY(record(h, st, 2));
  // the goal: clip (:207-221), projection when on the map (:223-237); then setStartAndGoal's two searches (:167-189)
  double* q = st->d_q;
  uint8_t* flags = reinterpret_cast<uint8_t*>(q + QB_FLAGS);
  int32_t* idx = reinterpret_cast<int32_t*>(q + QB_FLAGS) + 1;
  double hq[14 + 2];
  std::copy_n(start, 7, hq); std::copy_n(goal, 7, hq + 7);
  hq[14] = pp->start_radius; hq[15] = pp->goal_radius;
  TRY(copy_async(h, q + QB_START, hq, 14 * sizeof(double), cudaMemcpyHostToDevice, s));
  TRY(copy_async(h, q + QB_RADIUS, hq + 14, 2 * sizeof(double), cudaMemcpyHostToDevice, s));
  TRY(launch(h, goal_clip_kernel, 1, 1, 0, s, (const double*)(q + QB_GOAL), st->space, q + QB_CLIPPED, flags + 1));
  TRY(pose_from_2d(h, q + QB_CLIPPED, 1, q + QB_PROJECTED, flags, s));
  o.start_draw = st->start_draw; o.goal_draw = st->goal_draw;
  TRY(ball_search(h, q + QB_START, 1, q + QB_RADIUS, pp->n_iter, pp->seed, st->start_draw, q + QB_REPAIRED, idx, s));
  TRY(ball_search(h, q + QB_PROJECTED, 1, q + QB_RADIUS + 1, pp->n_iter, ~pp->seed, st->goal_draw, q + QB_REPAIRED + 7, idx + 1, s));
  TRY(record(h, st, 3));
  TRY(host_call_end(h, true));
  // baseSolve on the device roadmap with the device endpoints
  if (st->path_cap < pp->vertex_capacity) {
    cudaFree(st->d_path); st->d_path = nullptr; st->path_cap = 0;
    CU_TRY(h, cudaMalloc(&st->d_path, pp->vertex_capacity * 7 * sizeof(double)));
    st->path_cap = pp->vertex_capacity;
  }
  size_t n_solved = 0;
  double cost = 0.0;
  TRY(roadmap_solve(h, nullptr, nullptr, q + QB_REPAIRED, &st->space, nullptr, st->d_path, st->path_cap, &n_solved, &cost, &o.solve));
  TRY(record(h, st, 4));
  o.status = planner_status(o.solve.status);
  o.path_cost = cost;
  size_t n_out = 0;
  int rc = ARTP_OK;
  if (o.status == ARTP_PLANNER_SOLVED && pp->simplify) {   // getSolutionPath(true) under MotionCostObjective
    o.simplify_seed = pp->seed + st->simplify_calls;
    st->simplify_calls += 1;
    rc = simplify_path(h, nullptr, st->d_path, n_solved, &st->space, ARTP_OBJ_LEARNED, pp->max_query_edge_length, o.simplify_seed,
                       path, capacity, &n_out, &o.simplify);
  } else if (o.status == ARTP_PLANNER_SOLVED) {
    n_out = n_solved;
    if (n_out > capacity) { h->err = "capacity too small"; rc = ARTP_E_LIMIT; }
    else if (path) {
      TRY(copy_async(h, path, st->d_path, n_out * 7 * sizeof(double), cudaMemcpyDeviceToHost, s));
      TRY(sync_stream(h, s));
    }
  }
  // the record of the query: endpoints, ball indices, flags (one copy at the end)
  TRY(host_call_begin(h));
  TRY(record(h, st, 5));
  double qb[QB_MINMAX];
  TRY(copy_async(h, qb, q, sizeof(qb), cudaMemcpyDeviceToHost, s));
  TRY(host_call_end(h));
  const uint8_t* fb = reinterpret_cast<const uint8_t*>(qb + QB_FLAGS);
  const int32_t* ib = reinterpret_cast<const int32_t*>(qb + QB_FLAGS) + 1;
  o.goal_inside = fb[0]; o.goal_clipped = fb[1];
  o.start_index = ib[0]; o.goal_index = ib[1];
  std::copy_n(qb + QB_CLIPPED, 7, o.goal_clipped_state);
  std::copy_n(qb + QB_PROJECTED, 7, o.goal_projected);
  std::copy_n(qb + QB_REPAIRED, 7, o.start_repaired);
  std::copy_n(qb + QB_REPAIRED + 7, 7, o.goal_repaired);
  // the searches' streams advance by what the reference's loops draw (StartState.sampleGoal's mirror)
  st->start_draw += o.start_index >= 0 ? (uint64_t)o.start_index : pp->n_iter;
  st->goal_draw += o.goal_index >= 0 ? (uint64_t)o.goal_index : pp->n_iter;
  float* ms[5] = {&o.ms_sample_graph, &o.ms_update_edges, &o.ms_endpoints, &o.ms_solve, &o.ms_simplify};
  const int from[5] = {0, 1, 2, 3, 4}, to[5] = {1, 2, 3, 4, 5};
  for (int k = 0; k < 5; ++k) CU_TRY(h, cudaEventElapsedTime(ms[k], st->ev[from[k]], st->ev[to[k]]));
  roadmap_counts(h, &nv, &ne);
  o.n_vertices = nv; o.n_edges = ne;
  o.host_syncs = h->traffic.syncs - t0.syncs;
  o.bytes_h2d = h->traffic.h2d - t0.h2d;
  o.bytes_d2h = h->traffic.d2h - t0.d2h;
  if (info) *info = o;
  if (rc != ARTP_OK) return rc;
  if (n_path) *n_path = n_out;
  return ARTP_OK;
}

}  // extern "C"
