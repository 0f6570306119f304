// art_planner_b200/csrc/artp_roadmap.cu -- the PRM roadmap of the C ABI (include/artp.h): PRMMotionCost's graph
// construction (art_planner/src/planners/prm_motion_cost.cpp) on the device. The store and the per-milestone kernels are
// in artp_roadmap.cuh; the interior states go through the latency path's per-pose routine (check_states_cta) and the
// sampler and the distribution through artp_sampling.cu (artp_internal.h). Queries (artp_roadmap_query.cuh) price the
// edges through artp_cost.cu and search and validate paths without leaving the device.
#include <cmath>
#include <vector>

#include "artp_internal.h"
#include "artp_roadmap.cuh"
#include "artp_roadmap_query.cuh"

using namespace artp_api;

namespace artp_api {

struct Roadmap {
  artp::RoadmapDev dev{};
  artp::RoadmapCtl* h_ctl = nullptr;   // pinned: the control block as the last call left it
  uint32_t* h_count = nullptr;         // pinned: valid candidates of a sampled chunk
  uint64_t* h_draws = nullptr;         // pinned: their draw indices (kMaxRound)
  double* d_cand = nullptr;            // kMaxRound candidate milestones
  uint64_t* d_draws = nullptr;
  uint32_t* d_count = nullptr;
  double* d_dens_states = nullptr;     // vcap x 7: the density's vertices (roadmap_density_states_kernel)
  size_t icap = 0;                     // interior-state buffer, in states
  double lo[2] = {0, 0}, hi[2] = {0, 0};   // (x, y) box of every milestone so far: bounds n_interp
  bool has_box = false;
  artp::QueryDev q{};                  // adjacency, path and validation round of artp_roadmap_solve
  artp::QueryCtl* h_q = nullptr;       // pinned: the query's control block as the last solve left it
  uint32_t* d_path_idx = nullptr;      // vcap: the solution's vertex indices from start to goal
  bool search_smem = false;            // roadmap_search_kernel may use its dynamic shared memory
};

}  // namespace artp_api

namespace {

constexpr size_t kMaxRound = 1024;   // candidate milestones queued per round of artp_roadmap_sample_graph

// KStarStrategy (OMPL 1.4.2 ConnectionStrategy.h): kPRMConstant_ = e + e / d, d = SE3StateSpace's dimension 6, and
// k = static_cast<unsigned int>(ceil(kPRMConstant_ * log((double)milestoneCount()))). Computed here with the host's libm,
// for every V the store can reach, so that the device never evaluates log.
uint32_t k_star(size_t V) {
  const double e = 2.718281828459045235360287;   // boost::math::constants::e<double>()
  const double kc = e + e / (double)6u;
  return V == 0 ? 0u : static_cast<unsigned int>(std::ceil(kc * std::log((double)V)));
}

void free_store(Roadmap* r) {
  artp::RoadmapDev& d = r->dev;
  for (void* p : {(void*)d.ctl, (void*)d.states, (void*)d.kind, (void*)d.edges, (void*)d.dens, (void*)d.k_of_v, (void*)d.dist,
                  (void*)d.nbr, (void*)d.n_interp, (void*)d.off, (void*)d.interior, (void*)d.valid, (void*)d.milestone,
                  (void*)r->d_cand, (void*)r->d_draws, (void*)r->d_count, (void*)r->d_dens_states, (void*)d.ecost, (void*)d.eflag,
                  (void*)r->q.ctl, (void*)r->q.csr_off, (void*)r->q.csr_len, (void*)r->q.csr_nbr, (void*)r->q.csr_eid,
                  (void*)r->q.path, (void*)r->q.path_e, (void*)r->q.plist, (void*)r->q.chk_e, (void*)r->q.chk_s1,
                  (void*)r->q.chk_s2, (void*)r->q.chk_off, (void*)r->d_path_idx})
    cudaFree(p);
  if (r->h_q) cudaFreeHost(r->h_q);
  if (r->h_ctl) cudaFreeHost(r->h_ctl);
  if (r->h_count) cudaFreeHost(r->h_count);
  if (r->h_draws) cudaFreeHost(r->h_draws);
  *r = Roadmap{};
}

template <typename T>
int dev_alloc(Handle* h, T*& p, size_t count) {
  CU_TRY(h, cudaMalloc((void**)&p, count * sizeof(T)));
  return ARTP_OK;
}

int require_roadmap(Handle* h) {
  if (!h->roadmap || !h->roadmap->dev.ctl) { h->err = "no roadmap (artp_roadmap_clear first)"; return ARTP_E_INVALID; }
  return ARTP_OK;
}

// Grows the interior-state buffer to what a milestone inside the box can need: k connections of at most
// (box diagonal / kMaxDist) interior states each. Only between calls (grow synchronises the device).
int fit_interior(Handle* h, Roadmap* r) {
  const double dx = r->hi[0] - r->lo[0], dy = r->hi[1] - r->lo[1];
  const double per = std::floor(std::sqrt(dx * dx + dy * dy) / artp::kMaxLateral) + 1.0;
  if (!(per < 1e7)) { h->err = "roadmap states too far apart"; return ARTP_E_LIMIT; }
  const size_t need = (size_t)r->dev.kcap * (size_t)per;
  if (need >= 0x7FFFFFFFull) { h->err = "roadmap states too far apart"; return ARTP_E_LIMIT; }
  if (r->icap >= need) return ARTP_OK;
  CU_TRY(h, cudaDeviceSynchronize());
  cudaFree(r->dev.interior); cudaFree(r->dev.valid);
  r->dev.interior = nullptr; r->dev.valid = nullptr; r->icap = 0; r->dev.icap = 0;
  TRY(dev_alloc(h, r->dev.interior, need * 7));
  TRY(dev_alloc(h, r->dev.valid, need));
  r->icap = need;
  r->dev.icap = (uint32_t)need;
  return ARTP_OK;
}

void grow_box(Roadmap* r, double x0, double y0, double x1, double y1) {
  if (!r->has_box) { r->lo[0] = x0; r->lo[1] = y0; r->hi[0] = x1; r->hi[1] = y1; r->has_box = true; return; }
  r->lo[0] = std::min(r->lo[0], x0); r->lo[1] = std::min(r->lo[1], y0);
  r->hi[0] = std::max(r->hi[0], x1); r->hi[1] = std::max(r->hi[1], y1);
}

// addValidMilestone for candidate i of d_cand: three launches on s, no synchronisation.
int queue_milestone(Handle* h, Roadmap* r, const double* d_cand, uint32_t i, uint8_t kind, cudaStream_t s) {
  TRY(launch(h, artp::roadmap_neighbours_kernel, 1, artp::kRoadmapThreads, 0, s, r->dev, d_cand, i));
  TRY(check_states_cta(h, r->dev.interior, &r->dev.ctl->n_interior, &r->dev.ctl->stop, r->icap, r->dev.valid, s));
  return launch(h, artp::roadmap_commit_kernel, 1, artp::kCommitThreads, 0, s, r->dev, kind);
}

// The host's control block to the device (h_ctl is current: every roadmap call ends with it copied back).
int put_ctl(Handle* h, Roadmap* r, cudaStream_t s) {
  return copy_async(h, r->dev.ctl, r->h_ctl, sizeof(artp::RoadmapCtl), cudaMemcpyHostToDevice, s);
}
int get_ctl(Handle* h, Roadmap* r, cudaStream_t s) {
  return copy_async(h, r->h_ctl, r->dev.ctl, sizeof(artp::RoadmapCtl), cudaMemcpyDeviceToHost, s);
}

int stopped_full(Handle* h, const Roadmap* r) {
  if (r->h_ctl->stop & artp::RM_STOP_FULL) { h->err = "roadmap store full (artp_roadmap_clear capacities)"; return ARTP_E_LIMIT; }
  if (r->h_ctl->stop & artp::RM_STOP_INTERIOR) { h->err = "interior-state buffer overflow"; return ARTP_E_LIMIT; }
  return ARTP_OK;
}

// artp_roadmap_solve's checks of its endpoints, on the device: any non-finite state (-1), then start, then goal outside
// the bounds (no slack: the position inside the RealVectorBounds); then both (x, y).
__global__ void endpoint_check_kernel(const double* __restrict__ sg, artp_se3_space sp, double* __restrict__ out) {
  double verdict = 0.0;
  for (int k = 0; k < 14; ++k)
    if (!isfinite(sg[k])) verdict = -1.0;
  if (verdict == 0.0)
    for (int w = 0; w < 2 && verdict == 0.0; ++w)
      for (int i = 0; i < 3; ++i)
        if (sg[7 * w + i] < sp.low[i] || sg[7 * w + i] > sp.high[i]) { verdict = w ? ARTP_SOLVE_INVALID_GOAL : ARTP_SOLVE_INVALID_START; break; }
  out[0] = verdict;
  out[1] = sg[0]; out[2] = sg[1]; out[3] = sg[7]; out[4] = sg[8];
}

// The call's end: the control block back to the host with the stop rules off, then host_call_end.
int finish(Handle* h, Roadmap* r, int rc) {
  const int rc_end = host_call_end(h, true);
  if (rc_end == ARTP_E_CUDA) return rc_end;
  if (rc == ARTP_OK) rc = stopped_full(h, r);
  artp::RoadmapCtl& c = *r->h_ctl;
  c.stop = 0; c.done = 0; c.max_v = 0; c.max_e = 0; c.recompute_n = 0;
  return rc != ARTP_OK ? rc : rc_end;
}

}  // namespace

void artp_api::roadmap_free(Handle* h) {
  if (!h->roadmap) return;
  free_store(h->roadmap);
  delete h->roadmap;
  h->roadmap = nullptr;
}

int artp_api::roadmap_clear(Handle* h, size_t vertex_capacity, size_t edge_capacity) {
  if (vertex_capacity == 0 || edge_capacity == 0 || vertex_capacity >= 0x7FFFFFFFull || edge_capacity >= 0x7FFFFFFFull) {
    h->err = "roadmap capacities must be > 0 and < 2^31"; return ARTP_E_INVALID;
  }
  TRY(host_call_begin(h));
  if (!h->roadmap) h->roadmap = new Roadmap();
  Roadmap* r = h->roadmap;
  artp::RoadmapDev& d = r->dev;
  if (d.vcap != vertex_capacity || d.ecap != edge_capacity || !d.ctl) {
    CU_TRY(h, cudaStreamSynchronize(h->stream));
    free_store(r);
    const uint32_t kcap = std::max<uint32_t>(k_star(vertex_capacity), 1u);
    TRY(dev_alloc(h, d.ctl, 1));
    TRY(dev_alloc(h, d.states, vertex_capacity * 7));
    TRY(dev_alloc(h, d.kind, vertex_capacity));
    TRY(dev_alloc(h, d.edges, edge_capacity * 2));
    TRY(dev_alloc(h, d.dens, vertex_capacity));
    uint32_t* k_of_v;
    TRY(dev_alloc(h, k_of_v, vertex_capacity + 1));
    d.k_of_v = k_of_v;
    TRY(dev_alloc(h, d.dist, vertex_capacity));
    TRY(dev_alloc(h, d.nbr, kcap));
    TRY(dev_alloc(h, d.n_interp, kcap));
    TRY(dev_alloc(h, d.off, kcap + 1));
    TRY(dev_alloc(h, d.milestone, 7));
    TRY(dev_alloc(h, r->d_cand, kMaxRound * 7));
    TRY(dev_alloc(h, r->d_draws, kMaxRound));
    TRY(dev_alloc(h, r->d_count, 1));
    TRY(dev_alloc(h, r->d_dens_states, vertex_capacity * 7));
    TRY(dev_alloc(h, d.ecost, edge_capacity));
    TRY(dev_alloc(h, d.eflag, edge_capacity));
    artp::QueryDev& q = r->q;
    TRY(dev_alloc(h, q.ctl, 1));
    TRY(dev_alloc(h, q.csr_off, vertex_capacity + 1));
    TRY(dev_alloc(h, q.csr_len, vertex_capacity));
    TRY(dev_alloc(h, q.csr_nbr, edge_capacity * 2));
    TRY(dev_alloc(h, q.csr_eid, edge_capacity * 2));
    TRY(dev_alloc(h, q.path, vertex_capacity));
    TRY(dev_alloc(h, q.path_e, vertex_capacity));
    TRY(dev_alloc(h, q.plist, (size_t)kcap + 2));
    TRY(dev_alloc(h, q.chk_e, (size_t)artp::kQueryBatch));
    TRY(dev_alloc(h, q.chk_s1, (size_t)artp::kQueryBatch));
    TRY(dev_alloc(h, q.chk_s2, (size_t)artp::kQueryBatch));
    TRY(dev_alloc(h, q.chk_off, (size_t)artp::kQueryBatch + 1));
    TRY(dev_alloc(h, r->d_path_idx, vertex_capacity));
    CU_TRY(h, cudaHostAlloc((void**)&r->h_q, sizeof(artp::QueryCtl), cudaHostAllocDefault));
    CU_TRY(h, cudaHostAlloc((void**)&r->h_ctl, sizeof(artp::RoadmapCtl), cudaHostAllocDefault));
    CU_TRY(h, cudaHostAlloc((void**)&r->h_count, sizeof(uint32_t), cudaHostAllocDefault));
    CU_TRY(h, cudaHostAlloc((void**)&r->h_draws, kMaxRound * sizeof(uint64_t), cudaHostAllocDefault));
    d.vcap = (uint32_t)vertex_capacity;
    d.ecap = (uint32_t)edge_capacity;
    d.kcap = kcap;
    std::vector<uint32_t> kt(vertex_capacity + 1);
    for (size_t v = 0; v <= vertex_capacity; ++v) kt[v] = std::min(k_star(v), kcap);
    CU_TRY(h, cudaMemcpy(k_of_v, kt.data(), kt.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  }
  *r->h_ctl = artp::RoadmapCtl{};
  r->has_box = false;
  TRY(put_ctl(h, r, h->stream));
  CU_TRY(h, cudaMemsetAsync(d.dens, 0, vertex_capacity, h->stream));
  // a new edge weighs ob::Cost() = 0.0 with validity unknown until it is priced
  CU_TRY(h, cudaMemsetAsync(d.ecost, 0, edge_capacity * sizeof(double), h->stream));
  CU_TRY(h, cudaMemsetAsync(d.eflag, 0, edge_capacity, h->stream));
  return host_call_end(h);
}

int artp_api::roadmap_sample_graph(Handle* h, const artp_roadmap_params* rp, const artp_sample_distribution_params* dp,
                                   uint64_t seed, uint64_t first_sample, uint64_t* draws_used) {
  if (!rp) { h->err = "null roadmap params"; return ARTP_E_INVALID; }
  TRY(sampler_armed(h));
  TRY(require_whole_map(h));
  TRY(require_roadmap(h));
  if (dp) TRY(check_distribution_args(h, dp));
  if (rp->max_n_vertices >= 0xFFFFFFFFull || rp->max_n_edges >= 0xFFFFFFFFull || rp->recompute_density_after_n_samples >= 0xFFFFFFFFull) {
    h->err = "roadmap caps must be < 2^32"; return ARTP_E_INVALID;
  }
  Roadmap* r = h->roadmap;
  // every sampled milestone lies on the map (the sampler's map_cell test)
  const double Lx = h->map.rows * h->map.res, Ly = h->map.cols * h->map.res;
  grow_box(r, h->chk.cx - 0.5 * Lx, h->chk.cy - 0.5 * Ly, h->chk.cx + 0.5 * Lx, h->chk.cy + 0.5 * Ly);
  TRY(fit_interior(h, r));
  TRY(host_call_begin(h));
  cudaStream_t s = h->stream;
  artp::RoadmapCtl& c = *r->h_ctl;
  const uint32_t max_v = (uint32_t)rp->max_n_vertices, max_e = (uint32_t)rp->max_n_edges;
  const uint32_t recompute_n = dp ? (uint32_t)rp->recompute_density_after_n_samples : 0u;
  c.max_v = max_v; c.max_e = max_e; c.recompute_n = recompute_n; c.n_proc = 0;
  const uint64_t end = first_sample + std::min<uint64_t>(rp->max_draws, ~0ull - first_sample);
  uint64_t draw = first_sample;
  double accept = 0.5, v_per = 1.0, e_per = 1.0;   // running estimates: they size a round, never change its result
  int rc = ARTP_OK;
  while (rc == ARTP_OK && c.V < max_v && c.E - c.n_removed < max_e && draw < end) {   // num_edges(g_): live edges
    // at most this many milestones before a stop rule fires: each adds >= 1 vertex
    uint64_t room = max_v - c.V;
    if (recompute_n) room = std::min<uint64_t>(room, (uint64_t)recompute_n * (c.n_proc + 1) > c.V
                                                         ? (uint64_t)recompute_n * (c.n_proc + 1) - c.V : 1);
    const double guess = std::min((double)room / v_per, (double)(max_e - (c.E - c.n_removed)) / e_per);
    const size_t B = (size_t)std::max<double>(1.0, std::min<double>({std::ceil(guess) + 4.0, (double)room, (double)kMaxRound}));
    const uint64_t n_draw = std::min<uint64_t>(end - draw, (uint64_t)std::max(4096.0, 1.25 * (double)B / accept));
    if ((rc = sample_valid_draws(h, seed, draw, (size_t)n_draw, r->d_cand, r->d_draws, B, r->d_count, s))) break;
    TRY(copy_async(h, r->h_count, r->d_count, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    TRY(sync_stream(h, s));
    const uint32_t count = *r->h_count;
    accept = std::max(1e-4, (double)count / (double)n_draw);
    const size_t C = std::min<size_t>(count, B);
    if (C == 0) { draw += n_draw; continue; }
    const uint32_t V0 = c.V, E0 = c.E;
    c.stop = 0; c.done = 0;
    if ((rc = put_ctl(h, r, s))) break;
    for (size_t i = 0; i < C && rc == ARTP_OK; ++i) rc = queue_milestone(h, r, r->d_cand, (uint32_t)i, ARTP_ROADMAP_MILESTONE, s);
    if (rc) break;
    if ((rc = get_ctl(h, r, s))) break;
    TRY(copy_async(h, r->h_draws, r->d_draws, C * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    TRY(sync_stream(h, s));
    if (c.stop & (artp::RM_STOP_FULL | artp::RM_STOP_INTERIOR)) {
      if (c.done) draw = r->h_draws[c.done - 1] + 1;
      break;
    }
    const bool stop = c.stop != 0;
    if (!stop && c.done == C) draw = count > C ? r->h_draws[C - 1] + 1 : draw + n_draw;
    else draw = r->h_draws[c.done - 1] + 1;   // a stop rule fired after milestone done - 1
    v_per = std::max(1.0, (double)(c.V - V0) / c.done);
    e_per = std::max(1e-3, (double)(c.E - E0) / c.done);
    if (c.stop & artp::RM_STOP_RECOMPUTE) {   // map_->reApplyPreprocessing() (:191) over getPlannerData's vertices
      if ((rc = launch(h, artp::roadmap_density_states_kernel, grid_for(h, (size_t)c.V * 7, 256), 256, 0, s, r->dev.states,
                       r->dev.dens, (size_t)c.V, r->d_dens_states)))
        break;
      if ((rc = update_distribution_rearm(h, dp, r->d_dens_states, c.V, s))) break;
    }
    if (c.stop & artp::RM_STOP_CAPS) break;
  }
  if (draws_used) *draws_used = draw - first_sample;
  return finish(h, r, rc);
}

int artp_api::roadmap_update_edges(Handle* h) {
  TRY(require_roadmap(h));
  Roadmap* r = h->roadmap;
  const size_t E = r->h_ctl->E;
  char* reg[2];   // edge rows | cost3
  TRY(host_call_begin(h, {E * 6 * sizeof(float), E * 3 * sizeof(float)}, reg));
  TRY(price_store_edges(h, r->dev.states, r->dev.edges, nullptr, nullptr, E, (float*)reg[0], (float*)reg[1], r->dev.ecost,
                        r->dev.eflag, h->stream));
  return host_call_end(h);
}

int artp_api::roadmap_solve(Handle* h, const double* start, const double* goal, const double* d_sg, const artp_se3_space* space,
                            double* path_states, double* d_path_out, size_t path_capacity, size_t* n_path, double* cost,
                            artp_roadmap_solve_info* info) {
  TRY(require_roadmap(h));
  TRY(require_whole_map(h));
  if (!space) return null_buffer(h);
  Roadmap* r = h->roadmap;
  artp::QueryDev& q = r->q;
  if (!d_sg)
    for (int i = 0; i < 7; ++i)
      if (!std::isfinite(start[i]) || !std::isfinite(goal[i])) { h->err = "non-finite start or goal"; return ARTP_E_INVALID; }
  if (!artp::segment_lengths(*space, q.seg)) { h->err = "bad SE3 space parameters"; return ARTP_E_INVALID; }
  if (r->dev.vcap > artp::kSearchCtas * artp::kSearchSliceMax) {
    h->err = "roadmap too large for the on-chip search (vertex capacity above 77440)"; return ARTP_E_LIMIT;
  }
  // A cost query without weights fails before the roadmap changes (the check artp_roadmap_update_edges makes).
  TRY(price_store_edges(h, nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr, h->stream));
  if (n_path) *n_path = 0;
  artp_roadmap_solve_info out{};
  out.path_vertices = info ? info->path_vertices : nullptr;
  double xy[4];   // (x, y) of start and goal
  if (d_sg) {      // the device's verdict (endpoint_check_kernel) and the (x, y) that size the interior-state buffer
    double* d_chk;
    double chk[5];
    TRY(host_call_begin(h, {sizeof(chk)}, (char**)&d_chk));
    TRY(launch(h, endpoint_check_kernel, 1, 1, 0, h->stream, d_sg, *space, d_chk));
    TRY(copy_async(h, chk, d_chk, sizeof(chk), cudaMemcpyDeviceToHost, h->stream));
    TRY(host_call_end(h));
    if (chk[0] == -1.0) { h->err = "non-finite start or goal"; return ARTP_E_INVALID; }
    if (chk[0] != 0.0) {
      out.status = (int32_t)chk[0];
      if (info) *info = out;
      return ARTP_OK;
    }
    std::copy_n(chk + 1, 4, xy);
  } else {
    // SE3StateSpace::satisfiesBounds: the position inside the RealVectorBounds
    for (int w = 0; w < 2; ++w)
      for (int i = 0; i < 3; ++i) {
        const double x = (w ? goal : start)[i];
        if (x < space->low[i] || x > space->high[i]) {
          out.status = w ? ARTP_SOLVE_INVALID_GOAL : ARTP_SOLVE_INVALID_START;
          if (info) *info = out;
          return ARTP_OK;
        }
      }
    xy[0] = start[0]; xy[1] = start[1]; xy[2] = goal[0]; xy[3] = goal[1];
  }
  grow_box(r, xy[0], xy[1], xy[0], xy[1]);
  grow_box(r, xy[2], xy[3], xy[2], xy[3]);
  TRY(fit_interior(h, r));
  q.qcap = (uint32_t)std::min<size_t>(r->icap, artp::kQueryBatch);
  const uint32_t slice_cap = (r->dev.vcap + artp::kSearchCtas - 1) / artp::kSearchCtas;
  const size_t search_smem = ((size_t)slice_cap * artp::kSearchVertexBytes + 7) & ~(size_t)7;
  if (!r->search_smem) {
    CU_TRY(h, cudaFuncSetAttribute(artp::roadmap_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)(artp::kSearchSliceMax * artp::kSearchVertexBytes)));
    r->search_smem = true;
  }
  const size_t n_price = (size_t)r->dev.kcap + 2, out_cap = std::min<size_t>(path_capacity, r->dev.vcap);
  char* reg[4];   // start, goal | edge rows | cost3 | path states
  TRY(host_call_begin(h, {14 * sizeof(double), n_price * 6 * sizeof(float), n_price * 3 * sizeof(float),
                          out_cap * 7 * sizeof(double)}, reg));
  cudaStream_t s = h->stream;
  if (!d_sg) {
    TRY(copy_async(h, reg[0], start, 7 * sizeof(double), cudaMemcpyHostToDevice, s));
    TRY(copy_async(h, reg[0] + 7 * sizeof(double), goal, 7 * sizeof(double), cudaMemcpyHostToDevice, s));
    d_sg = (const double*)reg[0];
  }
  double* d_path = d_path_out ? d_path_out : (double*)reg[3];
  TRY(put_ctl(h, r, s));
  *r->h_q = artp::QueryCtl{};
  r->h_q->two = 2;
  TRY(copy_async(h, q.ctl, r->h_q, sizeof(artp::QueryCtl), cudaMemcpyHostToDevice, s));
  CU_TRY(h, cudaMemsetAsync(q.csr_len, 0, (size_t)r->dev.vcap * sizeof(uint32_t), s));
  const unsigned vgrid = grid_for(h, r->dev.vcap, 256, 4), egrid = grid_for(h, r->dev.ecap, 256, 4);
  int rc = ARTP_OK;
  auto step = [&](int x) { if (rc == ARTP_OK) rc = x; };
  // the pose check of both ends, clearQuery, the two milestones
  step(check_states_cta(h, d_sg, &q.ctl->two, &r->dev.ctl->stop, 2, q.ctl->pose_ok, s));
  step(launch(h, artp::query_begin_kernel, vgrid, 256, 0, s, r->dev, q));
  for (int w = 0; w < 2 && rc == ARTP_OK; ++w) {
    step(launch(h, artp::query_mark_kernel, 1, 1, 0, s, r->dev, q, w));
    step(queue_milestone(h, r, d_sg, (uint32_t)w, ARTP_ROADMAP_MILESTONE | ARTP_ROADMAP_QUERY, s));
  }
  // the adjacency, then the edges at the start and at the goal, in that order (:484-485)
  step(launch(h, artp::csr_count_kernel, egrid, 256, 0, s, r->dev, q));
  step(launch(h, artp::csr_scan_kernel, 1, 1024, 0, s, r->dev, q));
  step(launch(h, artp::csr_fill_kernel, egrid, 256, 0, s, r->dev, q));
  step(launch(h, artp::csr_sort_kernel, vgrid, 256, 0, s, r->dev, q));
  for (int w = 0; w < 2 && rc == ARTP_OK; ++w) {
    step(launch(h, artp::query_price_list_kernel, 1, 256, 0, s, r->dev, q, w));
    step(price_store_edges(h, r->dev.states, r->dev.edges, q.plist, &q.ctl->n_price, n_price, (float*)reg[1], (float*)reg[2],
                           r->dev.ecost, r->dev.eflag, s));
  }
  // do constructSolution while (!solution && sameComponent(start, goal)) (:508-512): rounds of search and validation,
  // queued four at a time; the kernels of a round that is not due return at once.
  const uint64_t max_rounds = (uint64_t)r->dev.ecap + r->dev.vcap + 8;   // a round removes an edge, validates one or ends
  for (uint64_t round = 0; rc == ARTP_OK;) {
    for (int k = 0; k < 4 && rc == ARTP_OK; ++k, ++round) {
      step(launch(h, artp::roadmap_search_kernel, artp::kSearchCtas, artp::kSearchThreads, search_smem, s, r->dev, q, slice_cap));
      step(launch(h, artp::query_gather_kernel, 1, 256, 0, s, r->dev, q));
      step(check_states_cta(h, r->dev.interior, &q.ctl->n_check, &q.ctl->idle, q.qcap, r->dev.valid, s));
      step(launch(h, artp::query_apply_kernel, 1, 256, 0, s, r->dev, q));
    }
    if (rc != ARTP_OK) break;
    step(get_ctl(h, r, s));
    TRY(copy_async(h, r->h_q, q.ctl, sizeof(artp::QueryCtl), cudaMemcpyDeviceToHost, s));
    TRY(sync_stream(h, s));
    if (r->h_q->status != artp::Q_RUNNING || r->h_ctl->stop) break;
    if (round > max_rounds) { h->err = "query did not end"; rc = ARTP_E_LIMIT; }
  }
  const artp::QueryCtl& c = *r->h_q;
  if (rc == ARTP_OK && c.status == ARTP_SOLVE_SOLVED) {
    step(launch(h, artp::query_finish_kernel, 1, 256, 0, s, r->dev, q, r->d_path_idx, d_path, (uint32_t)out_cap));
    if (rc == ARTP_OK) {
      TRY(copy_async(h, r->h_q, q.ctl, sizeof(artp::QueryCtl), cudaMemcpyDeviceToHost, s));
      const size_t n = c.path_n;   // read by the rounds' copy: the finish kernel does not change it
      if (n <= path_capacity) {
        if (path_states && !d_path_out) TRY(copy_async(h, path_states, d_path, n * 7 * sizeof(double), cudaMemcpyDeviceToHost, s));
        if (out.path_vertices)
          TRY(copy_async(h, out.path_vertices, r->d_path_idx, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
      }
    }
  }
  rc = finish(h, r, rc);
  if (rc != ARTP_OK) return rc;
  if (c.status == artp::Q_LIMIT) { h->err = "query exceeded a search or validation bound"; return ARTP_E_LIMIT; }
  out.status = c.status; out.searches = c.searches; out.sweeps = c.sweeps; out.edges_checked = c.checked;
  out.edges_removed = c.removed; out.start_vertex = c.start; out.goal_vertex = c.goal;
  if (info) *info = out;
  if (c.status != ARTP_SOLVE_SOLVED) return ARTP_OK;
  if (n_path) *n_path = c.path_n;
  if (cost) *cost = c.cost;
  if (c.path_n > path_capacity) { h->err = "path_capacity too small"; return ARTP_E_LIMIT; }
  return ARTP_OK;
}

bool artp_api::has_roadmap(const Handle* h) { return h->roadmap && h->roadmap->dev.ctl; }

void artp_api::roadmap_counts(const Handle* h, size_t* nv, size_t* ne) {
  *nv = h->roadmap->h_ctl->V;
  *ne = h->roadmap->h_ctl->E;
}

extern "C" {

int artp_roadmap_clear(artp_handle* hh, size_t vertex_capacity, size_t edge_capacity) {
  LOCK_CALL(h, hh);
  return roadmap_clear(h, vertex_capacity, edge_capacity);
}

int artp_roadmap_add_milestones(artp_handle* hh, const double* states, size_t n) {
  LOCK_CALL(h, hh);
  TRY(require_roadmap(h));
  TRY(require_whole_map(h));
  if (n == 0) return ARTP_OK;
  if (!states) return null_buffer(h);
  Roadmap* r = h->roadmap;
  for (size_t i = 0; i < n * 7; ++i)
    if (!std::isfinite(states[i])) { h->err = "non-finite milestone state"; return ARTP_E_INVALID; }
  for (size_t i = 0; i < n; ++i) grow_box(r, states[i * 7], states[i * 7 + 1], states[i * 7], states[i * 7 + 1]);
  TRY(fit_interior(h, r));
  char* d_states;
  TRY(host_call_begin(h, {n * 7 * sizeof(double)}, &d_states));
  cudaStream_t s = h->stream;
  CU_TRY(h, cudaMemcpyAsync(d_states, states, n * 7 * sizeof(double), cudaMemcpyHostToDevice, s));
  TRY(put_ctl(h, r, s));
  int rc = ARTP_OK;
  for (size_t i = 0; i < n && rc == ARTP_OK; ++i)
    rc = queue_milestone(h, r, (const double*)d_states, (uint32_t)i, ARTP_ROADMAP_MILESTONE | ARTP_ROADMAP_QUERY, s);
  if (rc == ARTP_OK) rc = get_ctl(h, r, s);
  return finish(h, r, rc);
}

int artp_roadmap_sample_graph(artp_handle* hh, const artp_roadmap_params* rp, const artp_sample_distribution_params* dp,
                              uint64_t seed, uint64_t first_sample, uint64_t* draws_used) {
  LOCK_CALL(h, hh);
  return roadmap_sample_graph(h, rp, dp, seed, first_sample, draws_used);
}

int artp_roadmap_get(artp_handle* hh, size_t first_vertex, double* states, uint8_t* kinds, size_t first_edge, uint32_t* edges,
                     size_t* nv, size_t* ne) {
  LOCK_CALL(h, hh);
  TRY(require_roadmap(h));
  Roadmap* r = h->roadmap;
  const size_t V = r->h_ctl->V, E = r->h_ctl->E;
  if (first_vertex > V || first_edge > E) { h->err = "roadmap cursor past the end"; return ARTP_E_INVALID; }
  TRY(host_call_begin(h));
  cudaStream_t s = h->stream;
  const size_t tv = V - first_vertex, te = E - first_edge;
  if (states && tv)
    CU_TRY(h, cudaMemcpyAsync(states, r->dev.states + first_vertex * 7, tv * 7 * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (kinds && tv) CU_TRY(h, cudaMemcpyAsync(kinds, r->dev.kind + first_vertex, tv, cudaMemcpyDeviceToHost, s));
  if (edges && te)
    CU_TRY(h, cudaMemcpyAsync(edges, r->dev.edges + first_edge * 2, te * 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  if (nv) *nv = V;
  if (ne) *ne = E;
  return host_call_end(h);
}

int artp_roadmap_update_edges(artp_handle* hh) {
  LOCK_CALL(h, hh);
  return roadmap_update_edges(h);
}

int artp_roadmap_solve(artp_handle* hh, const double* start, const double* goal, const artp_se3_space* space,
                       double* path_states, size_t path_capacity, size_t* n_path, double* cost,
                       artp_roadmap_solve_info* info) {
  LOCK_CALL(h, hh);
  if (!start || !goal) return null_buffer(h);
  return roadmap_solve(h, start, goal, nullptr, space, path_states, nullptr, path_capacity, n_path, cost, info);
}

int artp_roadmap_get_edge_costs(artp_handle* hh, size_t first_edge, double* cost, uint8_t* flags, size_t* n_live) {
  LOCK_CALL(h, hh);
  TRY(require_roadmap(h));
  Roadmap* r = h->roadmap;
  const size_t E = r->h_ctl->E;
  if (first_edge > E) { h->err = "roadmap cursor past the end"; return ARTP_E_INVALID; }
  TRY(host_call_begin(h));
  const size_t te = E - first_edge;
  if (cost && te)
    CU_TRY(h, cudaMemcpyAsync(cost, r->dev.ecost + first_edge, te * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (flags && te) CU_TRY(h, cudaMemcpyAsync(flags, r->dev.eflag + first_edge, te, cudaMemcpyDeviceToHost, h->stream));
  if (n_live) *n_live = E - r->h_ctl->n_removed;
  return host_call_end(h);
}

}  // extern "C"
