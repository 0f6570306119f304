// art_planner_b200/csrc/artp_cost.cu -- the cost half of the C ABI (include/artp.h): PathLengthObjective::motionCost, the
// MotionCostFunc edge matrix, and the learned motion cost of edge rows, of states and of whole edges split the way
// MotionCostObjective::motionCost splits them (artp_cnn.cu runs the network).
// Compiled without FMA contraction like artp_capi.cu, so that the rows and costs built here equal the host's bit for bit.
#include <cmath>
#include <vector>

#include "artp_internal.h"

using namespace artp_api;

namespace {

// PathLengthObjective::motionCost (art_planner/src/objectives/path_length_objective.cpp:26-70), double.
__global__ void path_length_kernel(const double* __restrict__ s1, const double* __restrict__ s2, size_t n,
                                   double* __restrict__ cost, int directional, double v_lon, double v_lat,
                                   double v_ang) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const double* a = s1 + 7 * i;
    const double* b = s2 + 7 * i;
    const double x_dif = b[0] - a[0], y_dif = b[1] - a[1], z_dif = b[2] - a[2];
    if (!directional) {
      cost[i] = sqrt(x_dif * x_dif + y_dif * y_dif + z_dif * z_dif) / v_lon;
      continue;
    }
    const double yaw1 = (double)artp::so3_yaw(a);
    const double yaw2 = (double)artp::so3_yaw(b);
    const double d = fabs(yaw1 - yaw2);
    const double yaw_dif = (d > 3.14159265358979323846) ? 2.0 * 3.14159265358979323846 - d : d;
    const double lon_dif = cos(yaw1) * x_dif + sin(yaw1) * y_dif;
    const double lat_dif = -sin(yaw1) * x_dif + cos(yaw1) * y_dif;
    const double t_yaw = fabs(yaw_dif) / v_ang, t_lon = fabs(lon_dif) / v_lon, t_lat = fabs(lat_dif) / v_lat;
    const double m = t_lon > t_lat ? t_lon : t_lat;
    cost[i] = m > t_yaw ? m : t_yaw;
  }
}

// Row [x y yaw] of knot s of the MotionCostFunc edge matrix as PRMMotionCostMaintainer::updateEdges /
// computeCostForVertexEdges fill it (prm_motion_cost.cpp:27-128): x, y cast double -> float by the assignment into the
// float matrix, yaw = getYawFromSO3.
__host__ __device__ __forceinline__ void knot_row(const double* s, float* o) {
  o[0] = (float)s[0]; o[1] = (float)s[1];
  o[2] = artp::so3_yaw(s);
}
// The 6-float row o of the edge from start to target: knot_row(target) ++ knot_row(start).
__host__ __device__ __forceinline__ void edge_row(const double* start, const double* target, float* o) {
  knot_row(target, o);
  knot_row(start, o + 3);
}

// isFeasible and getCost of an (energy, time, risk) triple c (motion_cost_objective.h:54-66) under the weights and the
// risk threshold of artp_params. getEnergy/getTime/getRisk return double (:30-46), so the risk is compared in double and
// the weighted sum is evaluated in double on exact float products.
struct CostRule {
  float we, wt, wr, thr;
  __host__ __device__ bool feasible(const float* c) const { return (double)c[2] <= (double)thr; }
  __host__ __device__ double cost(const float* c) const {
    return (double)c[0] * (double)we + (double)c[1] * (double)wt + (double)c[2] * (double)wr;
  }
  // The edge weight updateEdges gives (prm_motion_cost.cpp:54-60): getCost, +inf when infeasible.
  __device__ double weight(const float* c) const { return feasible(c) ? cost(c) : CUDART_INF; }
};

__global__ void edge_matrix_kernel(const double* __restrict__ s_start, const double* __restrict__ s_target, size_t n,
                                   float* __restrict__ edges) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    edge_row(s_start + 7 * i, s_target + 7 * i, edges + 6 * i);
}
__global__ void combine_cost_kernel(const float* __restrict__ cost3, size_t n, float we, float wt, float wr, float thr,
                                    double* __restrict__ cost, uint8_t* __restrict__ feasible) {
  const CostRule rule{we, wt, wr, thr};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    feasible[i] = rule.feasible(cost3 + 3 * i) ? 1 : 0;
    cost[i] = rule.weight(cost3 + 3 * i);
  }
}

// Rows of roadmap edges straight from the store (updateEdges :35-48, computeCostForVertexEdges :85-118). Without a list,
// row i is edge i from its stored source u to its target v. With one, row i < *count is edge (list[i] & 0x7FFFFFFF),
// reversed (from v to u) when bit 31 is set; rows from *count on are zero (the head prices them, nothing reads the result).
__global__ void store_rows_kernel(const double* __restrict__ states, const uint32_t* __restrict__ edges,
                                  const uint32_t* __restrict__ list, const uint32_t* __restrict__ count, size_t n,
                                  float* __restrict__ rows) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (list && i >= *count) {
      for (int k = 0; k < 6; ++k) rows[6 * i + k] = 0.0f;
      continue;
    }
    const uint32_t e = list ? list[i] & 0x7FFFFFFFu : (uint32_t)i;
    const bool flip = list && (list[i] >> 31);
    const uint32_t u = edges[2 * (size_t)e], v = edges[2 * (size_t)e + 1];
    edge_row(states + 7 * (size_t)(flip ? v : u), states + 7 * (size_t)(flip ? u : v), rows + 6 * i);
  }
}
// The weights of those edges: getCost, or +inf above the risk threshold. updateEdges (no list) also marks the feasible
// edges valid (:51-55); computeCostForVertexEdges (a list) leaves validity alone (:121-125).
__global__ void store_cost_kernel(const float* __restrict__ cost3, const uint32_t* __restrict__ list,
                                  const uint32_t* __restrict__ count, size_t n, float we, float wt, float wr, float thr,
                                  double* __restrict__ ecost, uint8_t* __restrict__ eflag) {
  const CostRule rule{we, wt, wr, thr};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (list && i >= *count) continue;
    const uint32_t e = list ? list[i] & 0x7FFFFFFFu : (uint32_t)i;
    ecost[e] = rule.weight(cost3 + 3 * i);
    if (!list && rule.feasible(cost3 + 3 * i)) eflag[e] |= ARTP_ROADMAP_EDGE_VALID;
  }
}

// MotionCostObjective::motionCost (motion_cost_objective.cpp:36-95) splits edge e into the pieces piece_off[e] ..
// piece_off[e+1] - 1 (n_interp + 1 of them). Knot j of the edge is s1 for j = 0, s2 for j = n_interp + 1 (copied, not
// interpolated) and interior state j in between (:49, :67); piece i's row is knot_row(knot i+1) ++ knot_row(knot i).
__device__ __forceinline__ void split_knot_row(const double* a, const double* b, uint32_t j, uint32_t n_pieces, float* o) {
  if (j == 0) {
    knot_row(a, o);
  } else if (j == n_pieces) {
    knot_row(b, o);
  } else {   // no pointer select between a, b and k: that would put all three in local memory
    double k[7];
    artp::interior_state(a, b, j, n_pieces - 1, k);
    knot_row(k, o);
  }
}
__global__ void split_rows_kernel(const double* __restrict__ s1, const double* __restrict__ s2, uint32_t n_edges,
                                  const uint32_t* __restrict__ piece_off, size_t total, float* __restrict__ rows) {
  for (size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x; p < total; p += (size_t)gridDim.x * blockDim.x) {
    const uint32_t lo = artp::edge_of_item<true>(piece_off, n_edges, (uint32_t)p);
    const uint32_t o0 = __ldg(piece_off + lo), n_pieces = __ldg(piece_off + lo + 1) - o0, i = (uint32_t)p - o0;
    double a[7], b[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) { a[k] = s1[(size_t)lo * 7 + k]; b[k] = s2[(size_t)lo * 7 + k]; }
    split_knot_row(a, b, i + 1, n_pieces, rows + 6 * p);
    split_knot_row(a, b, i, n_pieces, rows + 6 * p + 3);
  }
}
// The rest of motionCost per edge, one thread walking its pieces in order: +inf at the first piece whose risk is above
// the threshold, else the left-to-right double sum of getCost from 0.0.
__global__ void split_reduce_kernel(const float* __restrict__ cost3, const uint32_t* __restrict__ piece_off, size_t n,
                                    float we, float wt, float wr, float thr, double* __restrict__ cost) {
  const CostRule rule{we, wt, wr, thr};
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
    const uint32_t o0 = piece_off[e], o1 = piece_off[e + 1];
    double c = 0.0;
    for (uint32_t k = o0; k < o1; ++k) {
      const float* piece = cost3 + 3 * (size_t)k;
      // motionCost's own test (motion_cost_objective.cpp:87), not !isFeasible: the two differ on a NaN risk
      if ((double)piece[2] > (double)thr) { c = CUDART_INF; break; }
      c += rule.cost(piece);
    }
    cost[e] = c;
  }
}

// MotionCostObjective::motionCost's split of the n - 1 edges of a path (artp::cost_pieces); off = their exclusive prefix
// sums (n entries, the last = total).
// res[0] = the total (64 bits), res[1] = 1 when an edge has 2^32 pieces or more. One CTA.
constexpr int kOffThreads = 1024;
__global__ void __launch_bounds__(kOffThreads)
piece_offsets_kernel(const double* __restrict__ st, size_t n, double mql, uint32_t* __restrict__ off,
                     unsigned long long* __restrict__ res) {
  __shared__ unsigned long long part[kOffThreads];
  __shared__ int bad;
  const size_t ne = n - 1, per = (ne + kOffThreads - 1) / kOffThreads;
  const size_t e0 = threadIdx.x * per, e1 = min(ne, e0 + per);
  if (threadIdx.x == 0) bad = 0;
  __syncthreads();
  auto pieces = [&](size_t e) -> unsigned long long {
    const uint64_t p = artp::cost_pieces(st + 7 * e, st + 7 * (e + 1), mql);
    if (!p) bad = 1;
    return p;
  };
  unsigned long long sum = 0;
  for (size_t e = e0; e < e1; ++e) sum += pieces(e);
  part[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {   // exclusive scan of the 1024 chunk sums
    unsigned long long run = 0;
    for (int t = 0; t < kOffThreads; ++t) { const unsigned long long v = part[t]; part[t] = run; run += v; }
    res[0] = run;
    off[ne] = (uint32_t)run;
  }
  __syncthreads();
  unsigned long long run = part[threadIdx.x];
  for (size_t e = e0; e < e1; ++e) { off[e] = (uint32_t)run; run += pieces(e); }
  __syncthreads();
  if (threadIdx.x == 0) res[1] = bad;
}

}  // namespace

int artp_api::path_length_cost(Handle* h, const double* d_s1, const double* d_s2, size_t n, double* d_cost, cudaStream_t s) {
  return launch(h, path_length_kernel, grid_for(h, n, 256, 8), 256, 0, s, d_s1, d_s2, n, d_cost, h->p.use_directional_cost,
                h->p.max_lon_vel, h->p.max_lat_vel, h->p.max_ang_vel);
}

int artp_api::motion_cost_split(Handle* h, const double* d_s1, const double* d_s2, size_t n, const uint32_t* d_piece_off, size_t total_pieces,
                                 float* d_rows, float* d_cost3, double* d_cost, cudaStream_t s) {
  TRY(launch(h, split_rows_kernel, grid_for(h, total_pieces, 256, 8), 256, 0, s, d_s1, d_s2, (uint32_t)n, d_piece_off,
             total_pieces, d_rows));
  TRY(cost_head(h, d_rows, total_pieces, d_cost3, s));
  return launch(h, split_reduce_kernel, grid_for(h, n, 256, 8), 256, 0, s, d_cost3, d_piece_off, n, h->p.cost_w_energy,
                h->p.cost_w_time, h->p.cost_w_risk, h->p.risk_threshold, d_cost);
}

int artp_api::cost_piece_offsets(Handle* h, const double* s1, const double* s2, size_t n, double max_query_edge_length,
                                 std::vector<uint32_t>& off, size_t* total) {
  off.resize(n + 1);
  size_t t = 0;
  for (size_t e = 0; e < n; ++e) {
    off[e] = (uint32_t)t;
    const uint64_t pieces = artp::cost_pieces(s1 + 7 * e, s2 + 7 * e, max_query_edge_length);
    if (!pieces) { h->err = "edge too long or not finite (n_interp must fit 32 bits)"; return ARTP_E_INVALID; }
    t += pieces;
    if (t > 0xFFFFFFFFull) { h->err = "too many pieces (>= 2^32)"; return ARTP_E_INVALID; }
  }
  off[n] = (uint32_t)t;
  *total = t;
  return ARTP_OK;
}

int artp_api::piece_offsets(Handle* h, const double* d_states, size_t n, double max_query_edge_length, uint32_t* d_off,
                            size_t* total, cudaStream_t s) {
  char* r[1];
  TRY(carve(h, h->d_stage, h->stage_cap, {2 * sizeof(unsigned long long)}, r));
  TRY(launch(h, piece_offsets_kernel, 1, kOffThreads, 0, s, d_states, n, max_query_edge_length, d_off, (unsigned long long*)r[0]));
  unsigned long long res[2];
  TRY(copy_async(h, res, r[0], sizeof(res), cudaMemcpyDeviceToHost, s));
  TRY(sync_stream(h, s));
  if (res[1]) { h->err = "path edge too long for the learned cost"; return ARTP_E_INVALID; }
  if (res[0] > 0xFFFFFFFFull) { h->err = "too many cost pieces (>= 2^32)"; return ARTP_E_INVALID; }
  *total = (size_t)res[0];
  return ARTP_OK;
}

int artp_api::price_store_edges(Handle* h, const double* d_states, const uint32_t* d_edges, const uint32_t* d_list,
                                const uint32_t* d_count, size_t n, float* d_rows, float* d_cost3, double* d_ecost,
                                uint8_t* d_eflag, cudaStream_t s) {
  TRY(check_cost_net(h));
  if (n == 0) return ARTP_OK;
  const unsigned grid = grid_for(h, n, 256, 8);
  TRY(launch(h, store_rows_kernel, grid, 256, 0, s, d_states, d_edges, d_list, d_count, n, d_rows));
  TRY(cost_head(h, d_rows, n, d_cost3, s));
  return launch(h, store_cost_kernel, grid, 256, 0, s, (const float*)d_cost3, d_list, d_count, n, h->p.cost_w_energy,
                h->p.cost_w_time, h->p.cost_w_risk, h->p.risk_threshold, d_ecost, d_eflag);
}

extern "C" {

int artp_edge_matrix_from_states(const double* s_start, const double* s_target, size_t n, float* edges) {
  if (n && (!s_start || !s_target || !edges)) return ARTP_E_INVALID;
  for (size_t i = 0; i < n; ++i) edge_row(s_start + 7 * i, s_target + 7 * i, edges + 6 * i);
  return ARTP_OK;
}

int artp_motion_cost_states(artp_handle* hh, const double* s_start, const double* s_target, size_t n, double* cost,
                            uint8_t* feasible, float* cost3) {
  LOCK_CALL(h, hh);
  if (n == 0) return ARTP_OK;
  if (!s_start || !s_target || !cost || !feasible) return null_buffer(h);
  const size_t sb = n * 7 * sizeof(double);
  char* r[6];   // s_start | s_target | edge matrix | cost3 | cost | feasible
  TRY(host_call_begin(h, {sb, sb, n * 6 * sizeof(float), n * 3 * sizeof(float), n * sizeof(double), n}, r));
  float* d_edges = (float*)r[2];
  float* d_c3 = (float*)r[3];
  CU_TRY(h, cudaMemcpyAsync(r[0], s_start, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], s_target, sb, cudaMemcpyHostToDevice, h->stream));
  const unsigned grid = grid_for(h, n, 256, 8);
  TRY(launch(h, edge_matrix_kernel, grid, 256, 0, h->stream, (const double*)r[0], (const double*)r[1], n, d_edges));
  TRY(check_cost_net(h));
  TRY(cost_head(h, d_edges, n, d_c3, h->stream));
  TRY(launch(h, combine_cost_kernel, grid, 256, 0, h->stream, d_c3, n, h->p.cost_w_energy, h->p.cost_w_time, h->p.cost_w_risk,
      h->p.risk_threshold, (double*)r[4], (uint8_t*)r[5]));
  CU_TRY(h, cudaMemcpyAsync(cost, r[4], n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(h, cudaMemcpyAsync(feasible, r[5], n, cudaMemcpyDeviceToHost, h->stream));
  if (cost3) CU_TRY(h, cudaMemcpyAsync(cost3, d_c3, n * 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

int artp_path_length_cost_device(artp_handle* hh, const double* d_s1, const double* d_s2, size_t n, double* d_cost,
                                 void* stream) {
  LOCK_CALL(h, hh);
  if (n == 0) return ARTP_OK;
  if (!d_s1 || !d_s2 || !d_cost) return null_buffer(h);
  CU_TRY(h, cudaSetDevice(h->device));
  return path_length_cost(h, d_s1, d_s2, n, d_cost, (cudaStream_t)stream);
}

int artp_path_length_cost(artp_handle* hh, const double* s1, const double* s2, size_t n, double* cost) {
  LOCK_CALL(h, hh);
  if (n == 0) return ARTP_OK;
  if (!s1 || !s2 || !cost) return null_buffer(h);
  const size_t sb = n * 7 * sizeof(double);
  char* r[3];
  TRY(host_call_begin(h, {sb, sb, n * sizeof(double)}, r));
  CU_TRY(h, cudaMemcpyAsync(r[0], s1, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], s2, sb, cudaMemcpyHostToDevice, h->stream));
  TRY(path_length_cost(h, (const double*)r[0], (const double*)r[1], n, (double*)r[2], h->stream));
  CU_TRY(h, cudaMemcpyAsync(cost, r[2], n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

int artp_motion_cost_device(artp_handle* hh, const float* d_edges, size_t n, float* d_cost3, void* stream) {
  LOCK_CALL(h, hh);
  if (n && (!d_edges || !d_cost3)) return null_buffer(h);
  TRY(check_cost_net(h));
  return cost_head(h, d_edges, n, d_cost3, (cudaStream_t)stream);
}

int artp_motion_cost(artp_handle* hh, const float* edges, size_t n, float* cost3) {
  LOCK_CALL(h, hh);
  if (n == 0) return ARTP_OK;
  if (!edges || !cost3) return null_buffer(h);
  char* r[2];   // edges | cost3
  TRY(host_call_begin(h, {n * 6 * sizeof(float), n * 3 * sizeof(float)}, r));
  CU_TRY(h, cudaMemcpyAsync(r[0], edges, n * 6 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  TRY(check_cost_net(h));
  TRY(cost_head(h, (const float*)r[0], n, (float*)r[1], h->stream));
  CU_TRY(h, cudaMemcpyAsync(cost3, r[1], n * 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

// Reads only the parameters fixed at artp_create, so it takes no lock.
int artp_combine_cost(artp_handle* hh, const float* cost3, size_t n, double* cost, uint8_t* feasible) {
  if (!hh || (n && (!cost3 || !cost || !feasible))) return ARTP_E_INVALID;
  const artp_params& p = reinterpret_cast<Handle*>(hh)->p;
  const CostRule rule{p.cost_w_energy, p.cost_w_time, p.cost_w_risk, p.risk_threshold};
  for (size_t i = 0; i < n; ++i) {
    cost[i] = rule.cost(cost3 + 3 * i);
    feasible[i] = rule.feasible(cost3 + 3 * i) ? 1 : 0;
  }
  return ARTP_OK;
}

// Touches no per-handle scratch (the head reads the feature map and weights only), so, like artp_motion_cost_device, it
// joins no scratch group.
int artp_motion_cost_split_device(artp_handle* hh, const double* d_s1, const double* d_s2, size_t n,
                                  const uint32_t* d_piece_off, size_t total_pieces, float* d_rows, float* d_cost3,
                                  double* d_cost, void* stream) {
  LOCK_CALL(h, hh);
  if (n == 0) return ARTP_OK;
  if (!d_s1 || !d_s2 || !d_piece_off || !d_rows || !d_cost3 || !d_cost) return null_buffer(h);
  if (total_pieces < n || total_pieces > 0xFFFFFFFFull) {
    h->err = "total_pieces must lie in [n, 2^32) (every edge has at least one piece)";
    return ARTP_E_INVALID;
  }
  TRY(check_cost_net(h));
  CU_TRY(h, cudaSetDevice(h->device));
  return motion_cost_split(h, d_s1, d_s2, n, d_piece_off, total_pieces, d_rows, d_cost3, d_cost, (cudaStream_t)stream);
}

int artp_motion_cost_split(artp_handle* hh, const double* s1, const double* s2, size_t n, double max_query_edge_length,
                           double* cost) {
  LOCK_CALL(h, hh);
  if (n == 0) return ARTP_OK;
  if (!s1 || !s2 || !cost) return null_buffer(h);
  if (!(max_query_edge_length > 0.0)) { h->err = "max_query_edge_length must be > 0"; return ARTP_E_INVALID; }
  TRY(check_cost_net(h));
  std::vector<uint32_t> off;
  size_t total;
  TRY(cost_piece_offsets(h, s1, s2, n, max_query_edge_length, off, &total));
  const size_t sb = n * 7 * sizeof(double);
  char* r[6];   // s1 | s2 | piece offsets | rows | cost3 | cost
  TRY(host_call_begin(h, {sb, sb, (n + 1) * sizeof(uint32_t), total * 6 * sizeof(float), total * 3 * sizeof(float),
                          n * sizeof(double)}, r));
  CU_TRY(h, cudaMemcpyAsync(r[0], s1, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], s2, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[2], off.data(), (n + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  TRY(motion_cost_split(h, (const double*)r[0], (const double*)r[1], n, (const uint32_t*)r[2], total, (float*)r[3],
      (float*)r[4], (double*)r[5], h->stream));
  CU_TRY(h, cudaMemcpyAsync(cost, r[5], n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);   // `off` outlives its H2D copy: the call synchronises before it returns
}

}  // extern "C"
