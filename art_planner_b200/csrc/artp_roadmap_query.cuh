// art_planner_b200/csrc/artp_roadmap_query.cuh -- queries on the device PRM roadmap (artp_roadmap.cu): PRMMotionCost's
// baseSolve (art_planner/src/planners/prm_motion_cost.cpp:440-532) and constructSolution (:536-673) as
//   query_begin / query_mark          clearQuery (planner.cpp:240) and the vertex indices of the start and the goal
//   csr_count / scan / fill / sort    the adjacency of the live edges, neighbours in ascending edge index
//   query_price_list                  the edges at a query vertex, each from that vertex (computeCostForVertexEdges, :77-128)
//   roadmap_search_kernel             distances, connectivity, the tie rule and the path: one thread-block cluster
//   query_gather / apply              the motion checks of the path's edges of unknown validity (:632-668)
//   query_finish                      the path from start to goal and its cost
// A query is a fixed sequence of these launches. Each reads the control blocks first and returns when the query has
// ended or its step is not due, so the host queues search / validate rounds without looking at a result in between.
#pragma once

#include <cooperative_groups.h>

#include "../../include/artp.h"
#include "artp_roadmap.cuh"

namespace artp {

namespace cg = cooperative_groups;

constexpr int kSearchCtas = 8;                // one cluster of the portable maximum size
constexpr int kSearchThreads = 512;
// Per vertex in the cluster's shared memory: distance 8 B, level 4 B, predecessor 4 B, its edge 4 B, and one word of marks
// (the two frontiers and reachability) that other CTAs set with 32-bit atomics.
constexpr uint32_t kSearchVertexBytes = 24;
constexpr uint32_t kSearchSliceMax = 9680;    // vertices per CTA: 9680 * 24 B = 232 320 B of the 227 KB a CTA can have
constexpr uint32_t kMarkReach = 4u;           // marks: bit 0 / 1 = in the frontier of even / odd sweeps, bit 2 = reachable
constexpr uint32_t kQueryBatch = 2048;        // states of one validation round, at most
constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr unsigned long long kInfBits = 0x7FF0000000000000ull;   // +inf: non-negative doubles order like their bits

enum : int32_t { Q_RUNNING = 0, Q_LIMIT = -4 };   // QueryCtl::status; the others are ARTP_SOLVE_*

struct QueryCtl {
  int32_t status;
  uint32_t phase;            // 0: a search is due, 1: the path's validation is due
  uint32_t start, goal;
  uint32_t searches, sweeps, checked, removed;
  uint32_t path_n;           // vertices of the current path
  uint32_t n_check;          // states of the current validation round
  uint32_t n_chk;            // its edges
  uint32_t more;             // unknown edges of the path that did not fit the round
  uint32_t idle;             // the round has no state to check
  uint32_t n_price;          // edges in the pricing list
  uint32_t two;              // 2: the start and the goal go through the pose check together
  uint8_t pose_ok[4];        // their verdicts
  double cost;
};

struct QueryDev {
  QueryCtl* ctl;
  uint32_t* csr_off;         // vcap + 1
  uint32_t* csr_len;         // vcap: live degree
  uint32_t* csr_nbr;         // 2 ecap
  uint32_t* csr_eid;         // 2 ecap
  uint32_t* path;            // vcap: the path from the goal back to the start
  uint32_t* path_e;          // vcap: the edge between path[i] and path[i + 1]
  uint32_t* plist;           // kcap + 2: edge index, bit 31 = priced from its stored target
  uint32_t* chk_e;           // kQueryBatch: the round's edges from the goal's side, ...
  uint32_t* chk_s1;          // ... their start-side vertex (after the check: 1 if the motion is valid), ...
  uint32_t* chk_s2;          // ... their goal-side vertex ...
  uint32_t* chk_off;         // kQueryBatch + 1: ... and their first state
  uint32_t qcap;             // states a round may hold (the interior-state buffer, at most kQueryBatch)
  SegLen seg;                // the space's segment lengths (segment_count)
};

__device__ __forceinline__ bool query_off(const RoadmapDev& r, const QueryDev& q) {
  return r.ctl->stop != 0 || q.ctl->status != Q_RUNNING;
}

// Dijkstra relaxes an edge of finite weight only (:558-566: the goal is not reached over +inf).
__device__ __forceinline__ bool relaxable(double w) { return w >= 0.0 && w < CUDART_INF; }

// *p = min(*p, x) on a distance in another CTA's shared memory; true if it lowered *p. A compare-and-swap loop: a 64-bit
// atomicMin on shared memory is not one hardware operation, and it lost updates between CTAs racing for one neighbour.
__device__ __forceinline__ bool lower_to(unsigned long long* p, unsigned long long x) {
  unsigned long long old = *(volatile unsigned long long*)p;
  while (x < old) {
    const unsigned long long seen = atomicCAS(p, old, x);
    if (seen == old) return true;
    old = seen;
  }
  return false;
}

// clearQuery: the earlier start / goal milestones stay in the graph but stop being startM_ / goalM_. An invalid start or
// goal ends the query before anything changes.
__global__ void __launch_bounds__(256) query_begin_kernel(RoadmapDev r, QueryDev q) {
  if (r.ctl->stop) return;
  QueryCtl* qc = q.ctl;
  if (!qc->pose_ok[0] || !qc->pose_ok[1]) {
    if (threadIdx.x == 0) {
      qc->status = !qc->pose_ok[0] ? ARTP_SOLVE_INVALID_START : ARTP_SOLVE_INVALID_GOAL;
      r.ctl->stop |= RM_STOP_QUERY;
    }
    return;
  }
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < r.ctl->V; v += gridDim.x * blockDim.x)
    r.kind[v] &= (uint8_t)~ARTP_ROADMAP_QUERY;
}

// The next milestone's vertex index.
__global__ void query_mark_kernel(RoadmapDev r, QueryDev q, int goal) {
  if (r.ctl->stop) return;
  (goal ? q.ctl->goal : q.ctl->start) = r.ctl->V;
}

// ---- adjacency -------------------------------------------------------------------------------------------------------
__global__ void csr_count_kernel(RoadmapDev r, QueryDev q) {
  if (query_off(r, q)) return;
  const uint32_t E = r.ctl->E;
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < E; e += gridDim.x * blockDim.x) {
    if (r.eflag[e] & ARTP_ROADMAP_EDGE_REMOVED) continue;
    atomicAdd(q.csr_len + r.edges[2 * (size_t)e], 1u);
    atomicAdd(q.csr_len + r.edges[2 * (size_t)e + 1], 1u);
  }
}

// Row offsets from the degrees (one CTA), the degrees zeroed to serve as the fill's cursors, and the density's vertex
// set (LazyPRM::getPlannerData: startM_ / goalM_ and the endpoints of edges) over the live edges.
__global__ void __launch_bounds__(1024) csr_scan_kernel(RoadmapDev r, QueryDev q) {
  __shared__ uint32_t s_sum[1024];
  if (query_off(r, q)) return;
  const uint32_t V = r.ctl->V, tid = threadIdx.x, per = (V + 1023u) / 1024u;
  const uint32_t v0 = min(tid * per, V), v1 = min(v0 + per, V);
  uint32_t sum = 0;
  for (uint32_t v = v0; v < v1; ++v) sum += q.csr_len[v];
  s_sum[tid] = sum;
  __syncthreads();
  for (uint32_t o = 1; o < 1024u; o <<= 1) {
    const uint32_t add = tid >= o ? s_sum[tid - o] : 0u;
    __syncthreads();
    s_sum[tid] += add;
    __syncthreads();
  }
  uint32_t run = s_sum[tid] - sum;
  for (uint32_t v = v0; v < v1; ++v) {
    const uint32_t len = q.csr_len[v];
    q.csr_off[v] = run;
    run += len;
    q.csr_len[v] = 0;
    r.dens[v] = (r.kind[v] & ARTP_ROADMAP_QUERY) || len ? 1 : 0;
  }
  if (tid == 1023u) q.csr_off[V] = s_sum[1023];
}

__global__ void csr_fill_kernel(RoadmapDev r, QueryDev q) {
  if (query_off(r, q)) return;
  const uint32_t E = r.ctl->E;
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < E; e += gridDim.x * blockDim.x) {
    if (r.eflag[e] & ARTP_ROADMAP_EDGE_REMOVED) continue;
    const uint32_t u = r.edges[2 * (size_t)e], v = r.edges[2 * (size_t)e + 1];
    const uint32_t su = q.csr_off[u] + atomicAdd(q.csr_len + u, 1u), sv = q.csr_off[v] + atomicAdd(q.csr_len + v, 1u);
    q.csr_nbr[su] = v; q.csr_eid[su] = e;
    q.csr_nbr[sv] = u; q.csr_eid[sv] = e;
  }
}

// Each row into ascending edge index (the fill's order depends on the atomics; rows are a few tens of entries).
__global__ void csr_sort_kernel(RoadmapDev r, QueryDev q) {
  if (query_off(r, q)) return;
  const uint32_t V = r.ctl->V;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) {
    const uint32_t o = q.csr_off[v], len = q.csr_len[v];
    for (uint32_t i = 1; i < len; ++i) {
      const uint32_t e = q.csr_eid[o + i], n = q.csr_nbr[o + i];
      uint32_t j = i;
      for (; j > 0 && q.csr_eid[o + j - 1] > e; --j) { q.csr_eid[o + j] = q.csr_eid[o + j - 1]; q.csr_nbr[o + j] = q.csr_nbr[o + j - 1]; }
      q.csr_eid[o + j] = e; q.csr_nbr[o + j] = n;
    }
  }
}

// computeCostForVertexEdges(v): in_edges, then out_edges; on the undirected graph both hold every incident edge and the
// second pass, with v as the source, writes last. So each incident edge is priced once, from v.
__global__ void query_price_list_kernel(RoadmapDev r, QueryDev q, int goal) {
  QueryCtl* qc = q.ctl;
  if (threadIdx.x == 0) qc->n_price = 0;
  if (query_off(r, q)) return;
  const uint32_t v = goal ? qc->goal : qc->start, o = q.csr_off[v], len = q.csr_len[v];
  if (len > r.kcap + 2u) {
    if (threadIdx.x == 0) qc->status = Q_LIMIT;
    return;
  }
  for (uint32_t j = threadIdx.x; j < len; j += blockDim.x) {
    const uint32_t e = q.csr_eid[o + j];
    q.plist[j] = e | (r.edges[2 * (size_t)e] == v ? 0u : 0x80000000u);
  }
  if (threadIdx.x == 0) qc->n_price = len;
}

// ---- the search ------------------------------------------------------------------------------------------------------
// One cluster. CTA c keeps the vertices c * slice .. (c + 1) * slice - 1 in its shared memory and sweeps over its own
// frontier; the relaxations reach the neighbours' entries, wherever they live, through distributed shared memory.
//   distances     d[v] = least fixpoint of min fl(d[u] + w) over live edges of finite weight, by frontier sweeps with a
//                 64-bit compare-and-swap minimum on the bit pattern. Any relaxation order reaches it (w >= 0, fl(+)
//                 monotone).
//   connectivity  a reachability byte over live edges of any weight, in the same sweeps.
//   the path      edge (u, v) is tight if fl(d[u] + w) == d[v]; level[v] = hops from the start over tight edges;
//                 pred[v] = the tight neighbour one level down with the lowest index (then the lowest edge index).
// Both sweep loops stop after V + 2 sweeps at the latest (status Q_LIMIT): no input can keep the kernel running.
__global__ void __cluster_dims__(kSearchCtas, 1, 1) __launch_bounds__(kSearchThreads, 1)
roadmap_search_kernel(RoadmapDev r, QueryDev q, uint32_t cap) {
  extern __shared__ __align__(8) unsigned char s_mem[];
  __shared__ uint32_t s_flag[3];   // CTA 0's: sweep t changed something (slot t % 3; slot t + 1 is cleared during sweep t)
  QueryCtl* qc = q.ctl;
  if (query_off(r, q) || qc->phase != 0) return;   // the same for every CTA: qc changes after the first cluster.sync only
  cg::cluster_group cluster = cg::this_cluster();
  const uint32_t rank = cluster.block_rank(), tid = threadIdx.x;
  const uint32_t V = r.ctl->V, slice = (V + kSearchCtas - 1) / kSearchCtas;
  const uint32_t start = qc->start, goal = qc->goal;
  unsigned long long* d = reinterpret_cast<unsigned long long*>(s_mem);
  uint32_t* level = reinterpret_cast<uint32_t*>(d + cap);
  uint32_t* pred = level + cap;
  uint32_t* pred_e = pred + cap;
  uint32_t* mark = pred_e + cap;
  // vertex v's entry of a per-vertex array, in the CTA that keeps it
  auto at = [&](auto* base, uint32_t v) {
    const uint32_t c = v / slice;
    return cluster.map_shared_rank(base, c) + (v - c * slice);
  };
  uint32_t* flag = cluster.map_shared_rank(s_flag, 0);
  const uint32_t v0 = rank * slice, nloc = v0 < V ? min(slice, V - v0) : 0u;

  for (uint32_t i = tid; i < slice; i += blockDim.x) {
    d[i] = kInfBits; level[i] = kNone; pred[i] = kNone; pred_e[i] = kNone; mark[i] = 0;
  }
  if (rank == 0 && tid < 3) s_flag[tid] = 0;
  cluster.sync();
  if (rank == start / slice && tid == 0) {
    const uint32_t l = start - v0;
    d[l] = 0ull; level[l] = 0; mark[l] = kMarkReach | 1u;
  }
  cluster.sync();

  bool converged = false;
  uint32_t sweeps = 0;
  for (uint32_t t = 0; t <= V + 1u; ++t) {
    const uint32_t cur = 1u << (t & 1u), nxt = cur ^ 3u;
    if (rank == 0 && tid == 0) s_flag[(t + 1u) % 3u] = 0;
    bool changed = false;
    for (uint32_t l = tid; l < nloc; l += blockDim.x) {
      if (!(*(volatile uint32_t*)(mark + l) & cur)) continue;
      atomicAnd(mark + l, ~cur);
      const unsigned long long dv = *(volatile unsigned long long*)(d + l);
      const uint32_t o = q.csr_off[v0 + l], len = q.csr_len[v0 + l];
      for (uint32_t j = 0; j < len; ++j) {
        const uint32_t u = q.csr_nbr[o + j];
        const double w = r.ecost[q.csr_eid[o + j]];
        uint32_t* mu = at(mark, u);
        uint32_t set = *(volatile uint32_t*)mu & kMarkReach ? 0u : kMarkReach | nxt;
        if (dv != kInfBits && relaxable(w)) {
          const unsigned long long nd = (unsigned long long)__double_as_longlong(__longlong_as_double((long long)dv) + w);
          unsigned long long* du = at(d, u);
          if (lower_to(du, nd)) set |= nxt;
        }
        if (set) { atomicOr(mu, set); changed = true; }
      }
    }
    if (changed) *(volatile uint32_t*)(flag + t % 3u) = 1;
    cluster.sync();
    ++sweeps;
    if (!*(volatile uint32_t*)(flag + t % 3u)) { converged = true; break; }
  }
  if (!converged) {
    if (rank == 0 && tid == 0) qc->status = Q_LIMIT;
    cluster.sync();
    return;
  }

  // levels: a breadth-first search from the start over tight edges (the frontier bits are all zero again)
  if (rank == 0 && tid < 3) s_flag[tid] = 0;
  if (rank == start / slice && tid == 0) mark[start - v0] |= 1u;
  cluster.sync();
  converged = false;
  for (uint32_t t = 0; t <= V + 1u; ++t) {
    const uint32_t cur = 1u << (t & 1u), nxt = cur ^ 3u;
    if (rank == 0 && tid == 0) s_flag[(t + 1u) % 3u] = 0;
    bool changed = false;
    for (uint32_t l = tid; l < nloc; l += blockDim.x) {
      if (!(*(volatile uint32_t*)(mark + l) & cur)) continue;
      atomicAnd(mark + l, ~cur);
      const double dv = __longlong_as_double((long long)d[l]);
      const uint32_t o = q.csr_off[v0 + l], len = q.csr_len[v0 + l];
      for (uint32_t j = 0; j < len; ++j) {
        const uint32_t u = q.csr_nbr[o + j];
        const double w = r.ecost[q.csr_eid[o + j]];
        if (!relaxable(w)) continue;
        const unsigned long long nd = (unsigned long long)__double_as_longlong(dv + w);
        uint32_t* lu = at(level, u);
        if (nd == *at(d, u) && *(volatile uint32_t*)lu == kNone) {   // every writer of this sweep writes t + 1
          *(volatile uint32_t*)lu = t + 1u;
          atomicOr(at(mark, u), nxt);
          changed = true;
        }
      }
    }
    if (changed) *(volatile uint32_t*)(flag + t % 3u) = 1;
    cluster.sync();
    ++sweeps;
    if (!*(volatile uint32_t*)(flag + t % 3u)) { converged = true; break; }
  }
  if (!converged) {
    if (rank == 0 && tid == 0) qc->status = Q_LIMIT;
    cluster.sync();
    return;
  }

  // predecessors: every vertex looks for its own
  for (uint32_t l = tid; l < nloc; l += blockDim.x) {
    const uint32_t L = level[l];
    if (L == kNone || L == 0u) continue;
    const unsigned long long dv = d[l];
    const uint32_t o = q.csr_off[v0 + l], len = q.csr_len[v0 + l];
    uint32_t bu = kNone, be = kNone;
    for (uint32_t j = 0; j < len; ++j) {
      const uint32_t u = q.csr_nbr[o + j], e = q.csr_eid[o + j];
      const double w = r.ecost[e];
      const unsigned long long du = *at(d, u);
      if (!relaxable(w) || du == kInfBits || *at(level, u) != L - 1u) continue;
      if ((unsigned long long)__double_as_longlong(__longlong_as_double((long long)du) + w) != dv) continue;
      if (u < bu || (u == bu && e < be)) { bu = u; be = e; }
    }
    pred[l] = bu; pred_e[l] = be;
  }
  cluster.sync();

  if (rank == 0 && tid == 0) {
    qc->sweeps += sweeps;
    if (!(*at(mark, goal) & kMarkReach)) {
      qc->status = ARTP_SOLVE_NOT_CONNECTED;
    } else {
      qc->searches += 1;
      if (*at(d, goal) == kInfBits) {
        qc->status = ARTP_SOLVE_NO_FEASIBLE_PATH;
      } else {
        uint32_t n = 0, v = goal;
        for (;;) {
          if (n >= V || v == kNone) { qc->status = Q_LIMIT; break; }
          q.path[n] = v;
          if (v == start) { ++n; break; }
          q.path_e[n] = *at(pred_e, v);
          v = *at(pred, v);
          ++n;
        }
        qc->path_n = n;
        qc->phase = 1;
      }
    }
  }
  cluster.sync();   // no CTA leaves while its shared memory is being read
}

// ---- validation ------------------------------------------------------------------------------------------------------
// The path's edges without the VALID flag, from the goal's side, as many as fit a round, and the states
// DiscreteMotionValidator::checkMotion(start-side vertex, goal-side vertex) visits: interpolate(j / nd), j = 1 .. nd - 1,
// then the goal-side vertex itself.
__global__ void __launch_bounds__(256) query_gather_kernel(RoadmapDev r, QueryDev q) {
  __shared__ uint32_t s_n, s_total;
  QueryCtl* qc = q.ctl;
  if (query_off(r, q) || qc->phase != 1) {
    if (threadIdx.x == 0) { qc->idle = 1; qc->n_check = 0; }
    return;
  }
  if (threadIdx.x == 0) {
    uint32_t n = 0, total = 0, more = 0;
    for (uint32_t i = 0; i + 1 < qc->path_n; ++i) {
      const uint32_t e = q.path_e[i];
      if (r.eflag[e] & ARTP_ROADMAP_EDGE_VALID) continue;
      const uint32_t prev = q.path[i], pos = q.path[i + 1];
      const uint32_t nd = segment_count(r.states + (size_t)pos * 7, r.states + (size_t)prev * 7, q.seg);
      if (n == kQueryBatch || total + nd > q.qcap) { more = 1; break; }
      q.chk_e[n] = e; q.chk_s1[n] = pos; q.chk_s2[n] = prev; q.chk_off[n] = total;
      total += nd;
      ++n;
    }
    q.chk_off[n] = total;
    if (n == 0 && more) qc->status = Q_LIMIT;   // one motion alone exceeds the round
    qc->n_chk = n; qc->more = more; qc->n_check = total; qc->idle = total == 0;
    s_n = n; s_total = total;
  }
  __syncthreads();
  const uint32_t n = s_n, total = s_total;
  for (uint32_t item = threadIdx.x; item < total; item += blockDim.x) {
    const uint32_t lo = edge_of_item<false>(q.chk_off, n, item);   // chk_off was written in this launch: plain loads
    const uint32_t o0 = q.chk_off[lo], nd = q.chk_off[lo + 1] - o0, j = item - o0 + 1;
    double a[7], b[7], s[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) { a[k] = r.states[(size_t)q.chk_s1[lo] * 7 + k]; b[k] = r.states[(size_t)q.chk_s2[lo] * 7 + k]; }
    segment_state(a, b, j, nd, s);
#pragma unroll
    for (int k = 0; k < 7; ++k) r.interior[(size_t)item * 7 + k] = s[k];
  }
}

// Edge e leaves vertex v's row (the order of the rest is kept).
__device__ __forceinline__ void csr_remove(const RoadmapDev& r, const QueryDev& q, uint32_t v, uint32_t e) {
  const uint32_t o = q.csr_off[v], len = q.csr_len[v];
  uint32_t j = 0;
  while (j < len && q.csr_eid[o + j] != e) ++j;
  for (; j + 1 < len; ++j) { q.csr_eid[o + j] = q.csr_eid[o + j + 1]; q.csr_nbr[o + j] = q.csr_nbr[o + j + 1]; }
  q.csr_len[v] = len - 1;
  if (len == 1 && !(r.kind[v] & ARTP_ROADMAP_QUERY)) r.dens[v] = 0;
}

// :651-668 over the round: a valid motion makes its edge VALID for good; the first invalid one from the goal's side is
// removed and a new search is due. With every edge valid and none left over, the path is the solution.
__global__ void __launch_bounds__(256) query_apply_kernel(RoadmapDev r, QueryDev q) {
  QueryCtl* qc = q.ctl;
  if (query_off(r, q) || qc->phase != 1) return;
  const uint32_t n = qc->n_chk;
  for (uint32_t c = threadIdx.x; c < n; c += blockDim.x) {
    const uint32_t o0 = q.chk_off[c], nd = q.chk_off[c + 1] - o0;
    const uint32_t ok = leading_valid(r.valid + o0, nd) == nd;
    if (ok) r.eflag[q.chk_e[c]] |= ARTP_ROADMAP_EDGE_VALID;
    q.chk_s1[c] = ok;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  qc->checked += n;
  uint32_t bad = 0;
  while (bad < n && q.chk_s1[bad]) ++bad;
  if (bad < n) {
    const uint32_t e = q.chk_e[bad];
    r.eflag[e] |= ARTP_ROADMAP_EDGE_REMOVED;
    csr_remove(r, q, r.edges[2 * (size_t)e], e);
    csr_remove(r, q, r.edges[2 * (size_t)e + 1], e);
    r.ctl->n_removed += 1;
    qc->removed += 1;
    qc->phase = 0;
  } else if (!qc->more) {
    qc->status = ARTP_SOLVE_SOLVED;
  }
}

// The solution from start to goal: vertex indices, states, and the weights summed from the start (what Dijkstra's
// combineCosts accumulated along it). Nothing is written when the path is longer than `cap`.
__global__ void __launch_bounds__(256) query_finish_kernel(RoadmapDev r, QueryDev q, uint32_t* __restrict__ out_idx,
                                                           double* __restrict__ out_states, uint32_t cap) {
  QueryCtl* qc = q.ctl;
  if (r.ctl->stop || qc->status != ARTP_SOLVE_SOLVED) return;
  const uint32_t n = qc->path_n;
  if (threadIdx.x == 0) {
    double c = 0.0;
    for (uint32_t i = n - 1; i-- > 0;) c += r.ecost[q.path_e[i]];
    qc->cost = c;
  }
  if (n > cap) return;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const uint32_t v = q.path[n - 1 - i];
    out_idx[i] = v;
#pragma unroll
    for (int k = 0; k < 7; ++k) out_states[(size_t)i * 7 + k] = r.states[(size_t)v * 7 + k];
  }
}

}  // namespace artp
