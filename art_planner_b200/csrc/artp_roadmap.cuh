// art_planner_b200/csrc/artp_roadmap.cuh -- the per-milestone kernels of the device PRM roadmap (artp_roadmap.cu):
// PRMMotionCost::addValidMilestone (art_planner/src/planners/prm_motion_cost.cpp:325-390) as
//   roadmap_neighbours_kernel  KStarStrategy's exact k nearest and the interior states of every connection (one CTA)
//   pose_states_kernel         (artp_kernels.cuh) the interior states' verdicts, one CTA each
//   roadmap_commit_kernel      :335-387 -- the valid prefixes, the edges, the milestone -- and the stop rules (one CTA)
// Each reads the roadmap's control block first and does nothing once a stop bit is set, so a host can queue any number
// of milestones without waiting for one to finish.
#pragma once

#include <math_constants.h>

#include "artp_device.cuh"

namespace artp {

constexpr int kRoadmapThreads = 512;     // the neighbours kernel's CTA
constexpr int kCommitThreads = 256;      // the commit kernel's CTA
constexpr double kMaxLateral = 0.5;      // kMaxDist, prm_motion_cost.cpp:342

enum : uint32_t {
  RM_STOP_CAPS = 1u,        // V >= max_n_vertices or E >= max_n_edges after a milestone (:171-172)
  RM_STOP_RECOMPUTE = 2u,   // V / recompute_density_after_n_samples > n_proc after a milestone (:190-193)
  RM_STOP_FULL = 4u,        // the milestone did not fit the store: not added
  RM_STOP_INTERIOR = 8u,    // the interior states did not fit their buffer: not added
  RM_STOP_QUERY = 16u,      // artp_roadmap_solve found its start or goal invalid: neither is added
};

// The roadmap's device control block: counters, the current milestone's connections and the stop rules.
struct RoadmapCtl {
  uint32_t V, E;            // vertices and edges in the store
  uint32_t stop;            // RM_STOP_* bits; every kernel exits while any is set
  uint32_t done;            // milestones committed since the host last reset it
  uint32_t n_interior;      // interior states of the current milestone
  uint32_t k;               // neighbours of the current milestone
  uint32_t n_proc;          // recomputes so far (sampleGraph's n_proc)
  uint32_t max_v, max_e;    // stop rules, 0 = off
  uint32_t recompute_n;     // 0 = off
  uint32_t n_removed;       // edges a query removed (artp_roadmap_query.cuh): E - n_removed are live
};

struct RoadmapDev {
  RoadmapCtl* ctl;
  double* states;           // vcap x 7
  uint8_t* kind;            // vcap
  uint32_t* edges;          // ecap x 2
  uint8_t* dens;            // vcap: the vertex is one getPlannerData returns (QUERY milestone or edge endpoint)
  const uint32_t* k_of_v;   // vcap + 1: ceil(kc * log(V)), computed by the host
  uint32_t vcap, ecap;
  double* dist;             // vcap: SE(3) distances of the current milestone
  uint32_t* nbr;            // kcap: neighbours in ascending (distance, index)
  uint32_t* n_interp;       // kcap
  uint32_t* off;            // kcap + 1: first interior state of each connection
  uint32_t kcap;
  double* interior;         // icap x 7
  uint8_t* valid;           // icap
  uint32_t icap;
  double* milestone;        // 7: the current milestone
  double* ecost;            // ecap: edge weights (updateEdges / computeCostForVertexEdges); 0.0 until priced
  uint8_t* eflag;           // ecap: ARTP_ROADMAP_EDGE_* bits
};

// (d, j) orders before (e, k): ascending distance, exact ties by vertex index.
__device__ __forceinline__ bool nn_before(double d, uint32_t j, double e, uint32_t k) { return d < e || (d == e && j < k); }

// The current milestone (candidate `i` of `cand`) against the vertices 0 .. V-1: its k nearest, their n_interp and the
// interior states of every connection.
__global__ void __launch_bounds__(kRoadmapThreads)
roadmap_neighbours_kernel(RoadmapDev r, const double* __restrict__ cand, uint32_t i) {
  __shared__ double s_m[7];
  __shared__ double s_bd[kRoadmapThreads / 32];
  __shared__ uint32_t s_bj[kRoadmapThreads / 32];
  __shared__ uint32_t s_total;
  RoadmapCtl* ctl = r.ctl;
  if (ctl->stop) return;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const uint32_t V = ctl->V;
  if (tid < 7) {
    s_m[tid] = cand[(size_t)i * 7 + tid];
    r.milestone[tid] = s_m[tid];
  }
  __syncthreads();
  double m[7];
#pragma unroll
  for (int c = 0; c < 7; ++c) m[c] = s_m[c];
  // num_vertices(g_) counts the milestone (add_vertex comes first, :326); nn_ holds the V others (nn_->add(m), :387)
  const uint32_t k = V < r.vcap ? min(r.k_of_v[V + 1], V) : 0u;
  for (uint32_t j = tid; j < V; j += blockDim.x) r.dist[j] = se3_distance(m, r.states + (size_t)j * 7);
  __syncthreads();
  // k rounds: the least (distance, index) after the previous round's
  double pd = -1.0;
  uint32_t pj = 0xFFFFFFFFu;
  for (uint32_t t = 0; t < k; ++t) {
    double bd = CUDART_INF;
    uint32_t bj = 0xFFFFFFFFu;
    for (uint32_t j = tid; j < V; j += blockDim.x) {
      const double d = r.dist[j];
      if ((pj == 0xFFFFFFFFu || nn_before(pd, pj, d, j)) && nn_before(d, j, bd, bj)) { bd = d; bj = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double od = __shfl_xor_sync(0xffffffffu, bd, o);
      const uint32_t oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (nn_before(od, oj, bd, bj)) { bd = od; bj = oj; }
    }
    if (lane == 0) { s_bd[wid] = bd; s_bj[wid] = bj; }
    __syncthreads();
    bd = s_bd[0]; bj = s_bj[0];
    for (int w = 1; w < kRoadmapThreads / 32; ++w)
      if (nn_before(s_bd[w], s_bj[w], bd, bj)) { bd = s_bd[w]; bj = s_bj[w]; }
    __syncthreads();
    if (tid == 0) r.nbr[t] = bj;
    pd = bd; pj = bj;
  }
  __syncthreads();
  if (tid < (int)k) r.n_interp[tid] = lateral_count(m, r.states + (size_t)r.nbr[tid] * 7, kMaxLateral);   // :340-343
  __syncthreads();
  if (tid == 0) {
    uint32_t total = 0;
    for (uint32_t t = 0; t < k; ++t) {
      r.off[t] = total;
      total += r.n_interp[t];
    }
    r.off[k] = total;
    s_total = total;
    ctl->k = k;
    ctl->n_interior = total <= r.icap ? total : 0u;
    if (total > r.icap) ctl->stop |= RM_STOP_INTERIOR;
  }
  __syncthreads();
  if (s_total > r.icap) return;
  // the interior states of every connection (:348-353); off was written in this launch: plain loads
  for (uint32_t q = tid; q < s_total; q += blockDim.x) {
    const uint32_t t = edge_of_item<false>(r.off, k, q);
    double s[7];
    interior_state(m, r.states + (size_t)r.nbr[t] * 7, q - r.off[t] + 1, r.n_interp[t], s);
#pragma unroll
    for (int c = 0; c < 7; ++c) r.interior[(size_t)q * 7 + c] = s[c];
  }
}

// :335-387 for the current milestone, then the stop rules for the next one. `kind`: the milestone's kind byte.
__global__ void __launch_bounds__(kCommitThreads) roadmap_commit_kernel(RoadmapDev r, uint8_t kind) {
  __shared__ uint32_t s_keep[1024], s_base[1024];
  __shared__ int s_ok;
  RoadmapCtl* ctl = r.ctl;
  if (ctl->stop) return;
  const int tid = threadIdx.x;
  const uint32_t V = ctl->V, E = ctl->E, k = ctl->k;
  // the valid prefix of each connection (interior states are checked in order until the first invalid one, :350-371)
  for (uint32_t t = tid; t < k; t += blockDim.x) s_keep[t] = leading_valid(r.valid + r.off[t], r.n_interp[t]);
  __syncthreads();
  if (tid == 0) {
    uint32_t nv = 1, ne = 0;
    for (uint32_t t = 0; t < k; ++t) {
      s_base[t] = V + nv;
      const uint32_t n = r.n_interp[t], p = s_keep[t];
      nv += p;
      ne += n == 0 ? 1u : p + (p == n ? 1u : 0u);
    }
    s_ok = (uint64_t)V + nv <= r.vcap && (uint64_t)E + ne <= r.ecap;
    if (!s_ok) {
      ctl->stop |= RM_STOP_FULL;
    } else {
      uint32_t e = E;
      auto edge = [&](uint32_t a, uint32_t b) {
        r.edges[2 * (size_t)e] = a; r.edges[2 * (size_t)e + 1] = b; ++e;
        r.dens[a] = 1; r.dens[b] = 1;
      };
      for (uint32_t t = 0; t < k; ++t) {
        const uint32_t n = r.n_interp[t], p = s_keep[t], nb = r.nbr[t];
        if (n == 0) { edge(V, nb); continue; }          // :378-383
        uint32_t prev = V;
        for (uint32_t q = 0; q < p; ++q) { edge(prev, s_base[t] + q); prev = s_base[t] + q; }
        if (p == n) edge(prev, nb);                     // :372-377
      }
      if (kind & 4u) r.dens[V] = 1;                     // startM_ / goalM_ (LazyPRM::getPlannerData)
      const uint32_t V1 = V + nv, E1 = e;
      ctl->V = V1;
      ctl->E = E1;
      ctl->done += 1;
      uint32_t stop = 0;
      if (ctl->recompute_n && V1 / ctl->recompute_n > ctl->n_proc) {   // :190-193
        ctl->n_proc += 1;
        stop |= RM_STOP_RECOMPUTE;
      }
      if (ctl->max_v && !(V1 < ctl->max_v && E1 - ctl->n_removed < ctl->max_e)) stop |= RM_STOP_CAPS;   // num_edges(g_): live edges
      ctl->stop = stop;
    }
  }
  __syncthreads();
  if (!s_ok) return;
  // the milestone (vertex V, :326-328) and the kept interior states (:358-365)
  if (tid < 7) r.states[(size_t)V * 7 + tid] = r.milestone[tid];
  if (tid == 0) r.kind[V] = kind;
  for (uint32_t t = 0; t < k; ++t) {
    const uint32_t p = s_keep[t], o = r.off[t], b = s_base[t];
    for (uint32_t q = tid; q < p * 7; q += blockDim.x) r.states[(size_t)b * 7 + q] = r.interior[(size_t)o * 7 + q];
    for (uint32_t q = tid; q < p; q += blockDim.x) r.kind[b + q] = 2;
  }
}

// The vertices getPlannerData returns, in place, the others as NaN (not counted by the density's histogram).
__global__ void roadmap_density_states_kernel(const double* __restrict__ states, const uint8_t* __restrict__ dens, size_t n,
                                              double* __restrict__ out) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n * 7; i += (size_t)gridDim.x * blockDim.x)
    out[i] = dens[i / 7] ? states[i] : __longlong_as_double(0x7ff8000000000000LL);
}

}  // namespace artp
