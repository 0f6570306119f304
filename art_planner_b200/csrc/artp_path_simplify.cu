// art_planner_b200/csrc/artp_path_simplify.cu -- artp_simplify_path (include/artp.h): Planner::getSolutionPath(true)
// (art_planner/src/planner.cpp:266-298) on the device -- OMPL 1.4.2's PathSimplifier::simplifyMax as restated in
// oracle/path_simplify_oracle.py, then the check and the cost comparison.
//
// The path is a list of state ids into a state pool; erasures move ids, never states, and every new or replaced state
// takes a new pool slot, so collapseCloseVertices' pair distances (and their +inf marks) can belong to states. The schedule is a state machine in a
// device control block (SimpCtl) that three launches advance, one round at a time:
//   simplify_gather_kernel  the entry work of the calls that start now, then the round's candidate motions -- the next
//                           attempts of reduceVertices / shortcutPath / collapseCloseVertices mapped onto the current
//                           path, one smoothBSpline step's batch, or the final check -- and the states each motion visits
//                           (query_gather_kernel's layout)
//   pose_states_kernel      (artp_kernels.cuh, through check_states_cta) their verdicts, one CTA per state
//   simplify_apply_kernel   walks the round's attempts in order: skips and failures advance the attempt count, the first
//                           attempt that passes (and, in shortcutPath, passes the cost test) is applied and the next round
//                           starts at the attempt after it. The variates depend on (call, attempt) only, so the result is
//                           the sequential loop's whatever the round size.
// The host queues kRoundsPerSync rounds at a time and reads the control block once per batch.
#include <cmath>
#include <vector>

#include "artp_internal.h"

namespace artp_api {

struct Simplify {
  char* d_scratch = nullptr;   // the control block, state pool, path and round buffers of a call (carve)
  size_t cap = 0;
};

}  // namespace artp_api

using namespace artp_api;

namespace {

constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr uint32_t kBatch = 1024;          // states of one round at most: the largest grid of its check launch
constexpr uint32_t kAttempts = 32;         // attempts of one reduceVertices / shortcutPath round at most
constexpr uint32_t kCollapseAttempts = 8;  // closest pairs of one collapseCloseVertices round at most
constexpr uint32_t kRoundsPerSync = 8;
constexpr int kThreads = 256;
constexpr double kRangeRatio = 0.33;       // PathSimplifier's rangeRatio
constexpr double kSnapToVertex = 0.005;    // shortcutPath's snapToVertex
constexpr uint32_t kRepeat = 5;            // simplify: reduceVertices again / shortcutPath, at most
constexpr uint32_t kBsplineSteps = 3;      // simplify: smoothBSpline(path, 3, length / 100)
constexpr uint32_t kTag = 0x41525453u;     // "ARTS"

enum : uint32_t { ST_REDUCE, ST_COLLAPSE, ST_REDUCE_AGAIN, ST_SHORTCUT, ST_BSPLINE, ST_CHECK, ST_DONE };
enum : int32_t { S_RUNNING = 0, S_DONE = 1, S_LIMIT = -4 };

struct SimpCtl {
  int32_t status;            // S_*
  uint32_t stage;            // ST_*: the current call of the schedule
  uint32_t call;             // its index in the schedule (Philox counter word 1)
  uint32_t fresh;            // 1: its entry work is due
  uint32_t repair;           // the schedule ran: the final check includes checkAndRepair's
  uint32_t n, np;            // path states, pool states used
  uint32_t n0;               // collapseCloseVertices: states at entry
  uint32_t i, nochange, max_steps, max_empty;
  uint32_t result;           // the current call changed the path
  uint32_t try_more, repeat;
  uint32_t front_back;       // reduceVertices: its checkMotion(front, back) is due
  uint32_t bs_step, bs_sub, bs_next, bs_u;   // smoothBSpline: step, subdivide due, next even i, replacements
  uint32_t v0, vl, bad_motion;               // final check: first / last state valid, first failing motion
  double threshold, rd, min_change;
  uint32_t n_att, n_mot, n_check;   // the round: attempts (skipped ones included), motions, states
  uint32_t idle;             // the round has no state to check (its check launch returns at once)
  uint32_t want;             // states the round would have liked: sizes the next batch's check grid
  uint32_t n_in, n_simplified;
  uint32_t edits[4], motions, valids, rounds, discarded, check_passed;
};

struct Att {                 // one attempt of a round
  int32_t a, b;              // reduce / collapse: the two path positions; shortcut: pos0, pos1 as drawn
  int32_t ia, ib;            // shortcut: index0, index1 (-1: the point is interpolated)
  uint32_t mot;              // its motion; kNone: no attempt (skipped, or collapse found no pair)
  double s0[7], s1[7];       // shortcut: the two points
};

struct SimpDev {
  SimpCtl* ctl;
  double* pool;              // pcap x 7: pool[0 .. n_in) is the input path
  uint32_t pcap;
  uint32_t* path;            // ncap state ids
  uint32_t* tmp;             // ncap: subdivide's copy
  uint32_t* cid;             // ncap: collapse entry position of each path slot
  uint32_t ncap;
  double* pair;              // collapse: distance of entry positions a < b at pair_index(a, b, n0); +inf = marked
  double* dists;             // ncap: shortcutPath's cumulative distances
  Att* att;                  // kAttempts
  double* mot;               // kBatch x 14: the round's motions, s1 then s2 (a state check: s1 = s2, one state)
  uint32_t* mot_off;         // kBatch + 1: their first state
  uint8_t* mot_ok;           // kBatch
  double* chk;               // kBatch x 7: the states to check
  uint8_t* valid;            // kBatch
  artp::SegLen seg;
  uint64_t seed;
};

__device__ __forceinline__ const double* pst(const SimpDev& d, uint32_t k) { return d.pool + 7 * (size_t)d.path[k]; }

// Row-major upper triangle without the diagonal: pair (a, b), a < b, of n entry positions.
__device__ __forceinline__ size_t pair_index(uint32_t a, uint32_t b, uint32_t n) {
  return (size_t)a * n - (size_t)a * (a + 1) / 2 + (b - a - 1);
}

__device__ __forceinline__ void copy7(double* o, const double* s) {
#pragma unroll
  for (int k = 0; k < 7; ++k) o[k] = s[k];
}

__device__ __forceinline__ void variates(uint64_t seed, uint32_t call, uint32_t i, double& u0, double& u1) {
  uint32_t c[4] = {i, call, 0u, kTag};
  artp::philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  u0 = (double)((((uint64_t)c[1] << 32) | c[0]) >> 11) * (1.0 / 9007199254740992.0);
  u1 = (double)((((uint64_t)c[3] << 32) | c[2]) >> 11) * (1.0 / 9007199254740992.0);
}
__device__ __forceinline__ int uniform_int(double u, int a, int b) {
  return a + min((int)floor(u * (double)(b - a + 1)), b - a);
}
__device__ __forceinline__ double uniform_real(double u, double a, double b) { return a + u * (b - a); }

// shortcutPath's lower_bound over the cumulative distances, then the snap to the next or the previous waypoint.
__device__ void locate(const double* dists, uint32_t n, double p, double thr, int& pos, int& index) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (dists[mid] < p) lo = mid + 1; else hi = mid;
  }
  pos = lo == n ? (int)n - 1 : (int)lo;
  if (pos == 0 || dists[pos] - p < thr) { index = pos; return; }
  while (pos > 0 && p < dists[pos]) --pos;
  index = p - dists[pos] < thr ? pos : -1;
}

// The end of the current call: the schedule's next one (simplify, OMPL 1.4.2).
__device__ void end_call(SimpCtl& s, bool result) {
  switch (s.stage) {
    case ST_REDUCE: s.try_more = result; s.stage = ST_COLLAPSE; break;
    case ST_COLLAPSE: s.repeat = 0; s.stage = s.try_more ? ST_REDUCE_AGAIN : ST_SHORTCUT; break;
    case ST_REDUCE_AGAIN:
      s.repeat += 1; s.try_more = result;
      if (!result || s.repeat >= kRepeat) { s.repeat = 0; s.stage = ST_SHORTCUT; }
      break;
    case ST_SHORTCUT:
      s.repeat += 1;
      if (!result || s.repeat >= kRepeat) s.stage = ST_BSPLINE;
      break;
    case ST_BSPLINE: s.stage = ST_CHECK; s.n_simplified = s.n; break;
    default: break;
  }
  s.call += 1;
  s.fresh = 1;
}

// Erase path slots [from, to) (and their collapse entry positions).
__device__ void erase(const SimpDev& d, SimpCtl& s, uint32_t from, uint32_t to, bool with_cid) {
  const uint32_t k = to - from;
  for (uint32_t j = to; j < s.n; ++j) {
    d.path[j - k] = d.path[j];
    if (with_cid) d.cid[j - k] = d.cid[j];
  }
  s.n -= k;
}

__device__ __forceinline__ uint32_t put_state(const SimpDev& d, SimpCtl& s, const double* st) {
  const uint32_t id = s.np++;
  copy7(d.pool + 7 * (size_t)id, st);
  return id;
}

__device__ void recompute_dists(const SimpDev& d, SimpCtl& s, uint32_t from) {
  if (from == 0) { d.dists[0] = 0.0; from = 1; }
  for (uint32_t j = from; j < s.n; ++j) d.dists[j] = d.dists[j - 1] + artp::se3_distance(pst(d, j - 1), pst(d, j));
  s.threshold = d.dists[s.n - 1] * kSnapToVertex;
  s.rd = kRangeRatio * d.dists[s.n - 1];
}

// Appends motion s1 -> s2 (nd states) to the round unless the cap is reached; false then.
__device__ bool add_motion(const SimpDev& d, SimpCtl& s, const double* s1, const double* s2, uint32_t nd, uint32_t& total,
                           uint32_t cap) {
  if (total + nd > cap) {
    if (s.n_mot == 0) s.want = nd;   // the next grid must hold this motion
    else s.want = min(2u * cap, kBatch);
    return false;
  }
  copy7(d.mot + 14 * (size_t)s.n_mot, s1);
  copy7(d.mot + 14 * (size_t)s.n_mot + 7, s2);
  d.mot_off[s.n_mot] = total;
  total += nd;
  s.n_mot += 1;
  return true;
}

__device__ __forceinline__ uint32_t nd_of(const SimpDev& d, const double* a, const double* b) {
  return artp::segment_count(a, b, d.seg);
}

// The entry work of the call that starts now (the whole CTA; s in shared memory, thread 0 writes it).
__device__ void begin_call(const SimpDev& d, SimpCtl& s) {
  const uint32_t tid = threadIdx.x;
  const bool call_stage = s.stage < ST_CHECK;
  if (call_stage && s.n < 3) {                    // every simplifier function returns at once below 3 states
    __syncthreads();
    if (tid == 0) end_call(s, false);
    __syncthreads();
    return;
  }
  if (s.stage == ST_COLLAPSE) {                   // every pair's distance once, keyed by the states' entry positions
    const uint32_t n = s.n;
    for (uint32_t k = tid; k < n; k += blockDim.x) d.cid[k] = k;
    for (uint64_t lin = tid; lin < (uint64_t)n * n; lin += blockDim.x) {
      const uint32_t a = (uint32_t)(lin / n), b = (uint32_t)(lin % n);
      if (b > a) d.pair[pair_index(a, b, n)] = artp::se3_distance(pst(d, a), pst(d, b));
    }
  }
  __syncthreads();
  if (tid == 0) {
    s.i = 0; s.nochange = 0; s.result = 0;
    s.max_steps = s.max_empty = s.n;
    switch (s.stage) {
      case ST_REDUCE: case ST_REDUCE_AGAIN: s.front_back = 1; break;
      case ST_COLLAPSE: s.n0 = s.n; break;
      case ST_SHORTCUT: recompute_dists(d, s, 0); break;
      case ST_BSPLINE: {
        double L = 0.0;                           // PathGeometric::length
        for (uint32_t k = 1; k < s.n; ++k) L += artp::se3_distance(pst(d, k - 1), pst(d, k));
        s.min_change = L / 100.0;
        s.bs_step = 0; s.bs_sub = 1; s.bs_u = 0;
        break;
      }
      case ST_CHECK: s.v0 = 1; s.vl = 1; s.bad_motion = kNone; s.bs_next = 0; break;
      default: break;
    }
    s.fresh = 0;
  }
  __syncthreads();
}

// The k-th closest unmarked pair after (pd, plin) in (distance, scan position) order, over the whole CTA.
__device__ void collapse_next(const SimpDev& d, const SimpCtl& s, double pd, uint64_t plin, double& bd, uint64_t& blin) {
  __shared__ double s_d[kThreads / 32];
  __shared__ unsigned long long s_l[kThreads / 32];
  const uint32_t n = s.n, n0 = s.n0;
  bd = CUDART_INF; blin = ~0ull;
  for (uint64_t lin = threadIdx.x; lin < (uint64_t)n * n; lin += blockDim.x) {
    const uint32_t a = (uint32_t)(lin / n), b = (uint32_t)(lin % n);
    if (b < a + 2) continue;
    const double dist = d.pair[pair_index(d.cid[a], d.cid[b], n0)];
    if (!(dist < CUDART_INF)) continue;           // d < minDist from minDist = +inf: marked pairs never win
    const bool after = plin == ~0ull || pd < dist || (pd == dist && plin < lin);
    if (after && (dist < bd || (dist == bd && lin < blin))) { bd = dist; blin = lin; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double od = __shfl_xor_sync(0xffffffffu, bd, o);
    const unsigned long long ol = __shfl_xor_sync(0xffffffffu, (unsigned long long)blin, o);
    if (od < bd || (od == bd && ol < blin)) { bd = od; blin = ol; }
  }
  if ((threadIdx.x & 31) == 0) { s_d[threadIdx.x >> 5] = bd; s_l[threadIdx.x >> 5] = blin; }
  __syncthreads();
  bd = s_d[0]; blin = s_l[0];
  for (int w = 1; w < kThreads / 32; ++w)
    if (s_d[w] < bd || (s_d[w] == bd && s_l[w] < blin)) { bd = s_d[w]; blin = s_l[w]; }
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads) simplify_gather_kernel(SimpDev d, uint32_t cap) {
  __shared__ SimpCtl s;
  __shared__ uint32_t s_total;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s = *d.ctl;
  __syncthreads();
  if (s.status != S_RUNNING) {
    if (tid == 0) { d.ctl->idle = 1; d.ctl->n_check = 0; }
    return;
  }
  while (s.fresh && s.stage != ST_DONE) begin_call(d, s);
  if (tid == 0) { s.n_att = 0; s.n_mot = 0; s.want = 0; s_total = 0; }
  __syncthreads();

  if (s.stage == ST_COLLAPSE) {                   // the closest pairs, in the order the steps would take them
    double pd = 0.0;
    uint64_t plin = ~0ull;
    for (uint32_t k = 0; k < kCollapseAttempts; ++k) {
      if (s.i + k >= s.max_steps || s.nochange + k >= s.max_empty) break;
      double bd; uint64_t blin;
      collapse_next(d, s, pd, plin, bd, blin);
      bool stop = false;
      if (tid == 0) {
        Att& at = d.att[s.n_att];
        if (blin == ~0ull) {
          at.mot = kNone;                         // no pair left: the call ends at this step
          s.n_att += 1;
          stop = true;
        } else {
          at.a = (int32_t)(blin / s.n); at.b = (int32_t)(blin % s.n);
          const double* pa = pst(d, at.a);
          const double* pb = pst(d, at.b);
          at.mot = s.n_mot;
          uint32_t total = s_total;
          if (add_motion(d, s, pa, pb, nd_of(d, pa, pb), total, cap)) { s.n_att += 1; s_total = total; }
          else stop = true;
        }
        s.idle = stop;                            // reused as the loop's exit flag
      }
      __syncthreads();
      if (s.idle) break;
      pd = bd; plin = blin;
    }
  } else if (s.stage == ST_BSPLINE) {
    if (s.bs_sub) {                               // PathGeometric::subdivide
      const uint32_t n = s.n, n2 = 2 * n - 1;
      if (n2 > d.ncap || s.np + n - 1 > d.pcap) {
        if (tid == 0) { d.ctl->status = S_LIMIT; d.ctl->idle = 1; d.ctl->n_check = 0; }
        return;
      }
      for (uint32_t k = tid; k < n; k += blockDim.x) d.tmp[k] = d.path[k];
      __syncthreads();
      for (uint32_t k = tid; k < n; k += blockDim.x) {
        d.path[2 * k] = d.tmp[k];
        if (k + 1 < n) {
          double m[7];
          artp::se3_interpolate(d.pool + 7 * (size_t)d.tmp[k], d.pool + 7 * (size_t)d.tmp[k + 1], 0.5, m);
          copy7(d.pool + 7 * (size_t)(s.np + k), m);
          d.path[2 * k + 1] = s.np + k;
        }
      }
      __syncthreads();
      if (tid == 0) { s.np += n - 1; s.n = n2; s.bs_sub = 0; s.bs_next = 2; s.bs_u = 0; }
      __syncthreads();
    }
    // items i = bs_next, bs_next + 2, .. < n - 1: isValid(states[i-1]), checkMotion(states[i-1], m), checkMotion(m,
    // states[i+1]); m and the two segment counts in parallel, the prefix by thread 0
    const uint32_t n_items = min((s.n - 1 - s.bs_next + 1) / 2, kBatch / 3);
    for (uint32_t t = tid; t < n_items; t += blockDim.x) {
      const uint32_t i = s.bs_next + 2 * t;
      const double* a = pst(d, i - 1);
      const double* c = pst(d, i);
      const double* b = pst(d, i + 1);
      double t1[7], t2[7], m[7];
      artp::se3_interpolate(a, c, 0.5, t1);
      artp::se3_interpolate(c, b, 0.5, t2);
      artp::se3_interpolate(t1, t2, 0.5, m);
      double* o = d.mot + 14 * (size_t)(3 * t);
      copy7(o, a); copy7(o + 7, a);
      copy7(o + 14, a); copy7(o + 21, m);
      copy7(o + 28, m); copy7(o + 35, b);
      d.mot_off[3 * t] = 1;
      d.mot_off[3 * t + 1] = nd_of(d, a, m);
      d.mot_off[3 * t + 2] = nd_of(d, m, b);
    }
    __syncthreads();
    if (tid == 0) {
      uint32_t total = 0, t = 0;
      for (; t < n_items; ++t) {
        const uint32_t need = d.mot_off[3 * t] + d.mot_off[3 * t + 1] + d.mot_off[3 * t + 2];
        if (total + need > cap) { s.want = t == 0 ? need : min(2u * cap, kBatch); break; }
        for (int k = 0; k < 3; ++k) { const uint32_t nd = d.mot_off[3 * t + k]; d.mot_off[3 * t + k] = total; total += nd; }
      }
      if (t == n_items && n_items) s.want = total;
      s.n_att = t; s.n_mot = 3 * t; s_total = total;
    }
  } else if (s.stage == ST_CHECK) {
    // items 0: isValid(front), 1: isValid(back), 2 + k: checkMotion(states[k], states[k+1])
    const uint32_t n_all = s.n + 1, n_items = min(n_all - s.bs_next, kBatch);
    for (uint32_t t = tid; t < n_items; t += blockDim.x) {
      const uint32_t item = s.bs_next + t;
      double* o = d.mot + 14 * (size_t)t;
      if (item < 2) {
        const double* a = pst(d, item == 0 ? 0 : s.n - 1);
        copy7(o, a); copy7(o + 7, a);
        d.mot_off[t] = 1;
      } else {
        const double* a = pst(d, item - 2);
        const double* b = pst(d, item - 1);
        copy7(o, a); copy7(o + 7, b);
        d.mot_off[t] = nd_of(d, a, b);
      }
    }
    __syncthreads();
    if (tid == 0) {
      uint32_t total = 0, t = 0;
      for (; t < n_items; ++t) {
        const uint32_t nd = d.mot_off[t];
        if (total + nd > cap) { s.want = t == 0 ? nd : min(2u * cap, kBatch); break; }
        d.mot_off[t] = total;
        total += nd;
      }
      if (t == n_items) s.want = total;
      s.n_att = t; s.n_mot = t; s_total = total;
    }
  } else if (tid == 0 && (s.stage == ST_REDUCE || s.stage == ST_REDUCE_AGAIN)) {
    uint32_t total = 0;
    if (s.front_back) {
      Att& at = d.att[0];
      at.a = 0; at.b = (int32_t)s.n - 1; at.mot = 0;
      if (add_motion(d, s, pst(d, 0), pst(d, s.n - 1), nd_of(d, pst(d, 0), pst(d, s.n - 1)), total, cap)) s.n_att = 1;
    } else {
      const int count = (int)s.n, max_n = count - 1;
      const int range = 1 + (int)floor(0.5 + (double)count * kRangeRatio);
      for (uint32_t k = 0; k < kAttempts; ++k) {
        if (s.i + k >= s.max_steps || s.nochange + k >= s.max_empty) break;
        double u0, u1;
        variates(d.seed, s.call, s.i + k, u0, u1);
        int p1 = uniform_int(u0, 0, max_n);
        int p2 = uniform_int(u1, max(p1 - range, 0), min(max_n, p1 + range));
        Att& at = d.att[s.n_att];
        at.mot = kNone;
        if (abs(p1 - p2) < 2) {
          if (p1 < max_n - 1) p2 = p1 + 2;
          else if (p1 > 1) p2 = p1 - 2;
          else { s.n_att += 1; continue; }
        }
        if (p1 > p2) { const int t = p1; p1 = p2; p2 = t; }
        at.a = p1; at.b = p2; at.mot = s.n_mot;
        if (!add_motion(d, s, pst(d, p1), pst(d, p2), nd_of(d, pst(d, p1), pst(d, p2)), total, cap)) break;
        s.n_att += 1;
      }
      if (s.want == 0) s.want = total;
    }
    s_total = total;
  } else if (tid == 0 && s.stage == ST_SHORTCUT) {
    uint32_t total = 0;
    const uint32_t n = s.n;
    for (uint32_t k = 0; k < kAttempts; ++k) {
      if (s.i + k >= s.max_steps || s.nochange + k >= s.max_empty) break;
      double u0, u1;
      variates(d.seed, s.call, s.i + k, u0, u1);
      const double L = d.dists[n - 1];
      int pos0, index0, pos1, index1;
      const double p0 = uniform_real(u0, 0.0, L);
      locate(d.dists, n, p0, s.threshold, pos0, index0);
      const double p1 = uniform_real(u1, fmax(0.0, p0 - s.rd), fmin(p0 + s.rd, L));
      locate(d.dists, n, p1, s.threshold, pos1, index1);
      Att& at = d.att[s.n_att];
      at.mot = kNone;
      // same or adjacent segments or waypoints (the restatement's rule: OMPL 1.4.2's first three tests, then the three
      // of later releases that keep the edits below off reversed and empty ranges)
      if (pos0 == pos1 || index0 == pos1 || index1 == pos0 || pos0 + 1 == index1 || pos1 + 1 == index0 ||
          (index0 >= 0 && index1 >= 0 && abs(index0 - index1) < 2)) {
        s.n_att += 1;
        continue;
      }
      at.a = pos0; at.b = pos1; at.ia = index0; at.ib = index1;
      if (index0 >= 0) {
        copy7(at.s0, pst(d, index0));
      } else {
        const double t0 = (p0 - d.dists[pos0]) / (d.dists[pos0 + 1] - d.dists[pos0]);
        artp::se3_interpolate(pst(d, pos0), pst(d, pos0 + 1), t0, at.s0);
      }
      if (index1 >= 0) {
        copy7(at.s1, pst(d, index1));
      } else {
        const double t1 = (p1 - d.dists[pos1]) / (d.dists[pos1 + 1] - d.dists[pos1]);
        artp::se3_interpolate(pst(d, pos1), pst(d, pos1 + 1), t1, at.s1);
      }
      at.mot = s.n_mot;
      if (!add_motion(d, s, at.s0, at.s1, nd_of(d, at.s0, at.s1), total, cap)) break;
      s.n_att += 1;
    }
    if (s.want == 0) s.want = total;
    s_total = total;
  }
  __syncthreads();

  const uint32_t total = s_total, n_mot = s.n_mot;
  if (tid == 0) {
    d.mot_off[n_mot] = total;
    if (n_mot == 0 && s.want > kBatch) s.status = S_LIMIT;   // one motion alone exceeds the largest round
    s.n_check = total;
    s.idle = total == 0;
  }
  __syncthreads();
  // the states of every motion (mot_off was written in this launch: plain loads)
  for (uint32_t item = tid; item < total; item += blockDim.x) {
    const uint32_t lo = artp::edge_of_item<false>(d.mot_off, n_mot, item);
    const uint32_t o0 = d.mot_off[lo], nd = d.mot_off[lo + 1] - o0, j = item - o0 + 1;
    double a[7], b[7], st[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) { a[k] = d.mot[14 * (size_t)lo + k]; b[k] = d.mot[14 * (size_t)lo + 7 + k]; }
    artp::segment_state(a, b, j, nd, st);
    copy7(d.chk + 7 * (size_t)item, st);
  }
  if (tid == 0) *d.ctl = s;
}

// The round's attempts in the order the sequential loop takes them.
__global__ void __launch_bounds__(kThreads) simplify_apply_kernel(SimpDev d) {
  __shared__ SimpCtl s;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) s = *d.ctl;
  __syncthreads();
  if (s.status != S_RUNNING || s.n_att == 0) return;   // a round cut before its first attempt does nothing
  for (uint32_t m = tid; m < s.n_mot; m += blockDim.x) {
    const uint32_t o0 = d.mot_off[m], nd = d.mot_off[m + 1] - o0;
    d.mot_ok[m] = artp::leading_valid(d.valid + o0, nd) == nd;
  }
  __syncthreads();
  if (tid != 0) return;
  s.rounds += s.n_check > 0;
  auto later_motions = [&](uint32_t from) {
    uint32_t c = 0;
    for (uint32_t t = from; t < s.n_att; ++t) c += d.att[t].mot != kNone;
    return c;
  };
  switch (s.stage) {
    case ST_REDUCE: case ST_REDUCE_AGAIN:
      if (s.front_back) {
        s.motions += 1;
        s.front_back = 0;
        if (d.mot_ok[0]) {
          d.path[1] = d.path[s.n - 1];
          s.n = 2;
          s.edits[0] += 1;
          end_call(s, true);
        }
        break;
      }
      for (uint32_t t = 0; t < s.n_att; ++t) {
        const Att& at = d.att[t];
        bool applied = false;
        if (at.mot != kNone) {
          s.motions += 1;
          if (d.mot_ok[at.mot]) {
            erase(d, s, at.a + 1, at.b, false);
            s.edits[0] += 1; s.result = 1; s.nochange = 0;
            applied = true;
          }
        }
        s.i += 1; s.nochange += 1;
        if (applied) { s.discarded += later_motions(t + 1); break; }
      }
      // at two states every later attempt is skipped (no motion): the loop's end changes nothing
      if (s.i >= s.max_steps || s.nochange >= s.max_empty || s.n == 2) end_call(s, s.result);
      break;
    case ST_COLLAPSE:
      for (uint32_t t = 0; t < s.n_att; ++t) {
        const Att& at = d.att[t];
        if (at.mot == kNone) { s.max_steps = 0; break; }   // no pair: the loop breaks
        s.motions += 1;
        if (d.mot_ok[at.mot]) {
          erase(d, s, at.a + 1, at.b, true);
          s.edits[1] += 1; s.result = 1; s.nochange = 0;
          s.i += 1; s.nochange += 1;
          s.discarded += later_motions(t + 1);
          break;
        }
        d.pair[pair_index(d.cid[at.a], d.cid[at.b], s.n0)] = CUDART_INF;
        s.i += 1; s.nochange += 1;
      }
      if (s.i >= s.max_steps || s.nochange >= s.max_empty) end_call(s, s.result);
      break;
    case ST_SHORTCUT:
      for (uint32_t t = 0; t < s.n_att; ++t) {
        const Att& at = d.att[t];
        s.i += 1; s.nochange += 1;
        if (at.mot == kNone) continue;
        s.motions += 1;
        if (!d.mot_ok[at.mot]) continue;
        int a = at.a, b = at.b, ia = at.ia, ib = at.ib;
        const double* s0 = at.s0;
        const double* s1 = at.s1;
        if (a > b) { int x = a; a = b; b = x; x = ia; ia = ib; ib = x; const double* y = s0; s0 = s1; s1 = y; }
        double along = ia >= 0 ? 0.0 : artp::se3_distance(s0, pst(d, a + 1));
        for (int k = a + 1; k < b; ++k) along += artp::se3_distance(pst(d, k), pst(d, k + 1));
        along += ib >= 0 ? 0.0 : artp::se3_distance(pst(d, b), s1);
        if (along < artp::se3_distance(s0, s1)) continue;
        if (s.np + 2 > d.pcap || s.n + 1 > d.ncap) { s.status = S_LIMIT; break; }
        if (ia < 0 && ib < 0) {
          if (a + 1 == b) {
            d.path[b] = put_state(d, s, s0);
            for (uint32_t j = s.n; j > (uint32_t)a + 2; --j) d.path[j] = d.path[j - 1];
            d.path[a + 2] = put_state(d, s, s1);
            s.n += 1;
          } else {
            d.path[a + 1] = put_state(d, s, s0);
            d.path[b] = put_state(d, s, s1);
            erase(d, s, a + 2, b, false);
          }
        } else if (ia >= 0 && ib >= 0) {
          erase(d, s, ia + 1, ib, false);
        } else if (ia < 0) {
          d.path[a + 1] = put_state(d, s, s0);
          erase(d, s, a + 2, ib, false);
        } else {
          d.path[b] = put_state(d, s, s1);
          erase(d, s, ia + 1, b, false);
        }
        recompute_dists(d, s, a + 1);
        s.edits[2] += 1; s.result = 1; s.nochange = 1;
        s.discarded += later_motions(t + 1);
        break;
      }
      if (s.status == S_RUNNING && (s.i >= s.max_steps || s.nochange >= s.max_empty)) end_call(s, s.result);
      break;
    case ST_BSPLINE:
      if (s.np + s.n_att > d.pcap) { s.status = S_LIMIT; break; }
      for (uint32_t t = 0; t < s.n_att; ++t) {
        const uint32_t i = s.bs_next + 2 * t;
        s.valids += 1;
        if (!d.mot_ok[3 * t]) continue;
        s.motions += 1;
        if (!d.mot_ok[3 * t + 1]) continue;
        s.motions += 1;
        if (!d.mot_ok[3 * t + 2]) continue;
        const double* m = d.mot + 14 * (size_t)(3 * t + 1) + 7;
        if (artp::se3_distance(pst(d, i), m) > s.min_change) {
          d.path[i] = put_state(d, s, m);
          s.bs_u += 1;
        }
      }
      s.bs_next += 2 * s.n_att;
      if (s.bs_next >= s.n - 1) {                 // the step is complete
        s.edits[3] += s.bs_u;
        s.bs_step += 1;
        if (s.bs_u == 0 || s.bs_step >= kBsplineSteps) end_call(s, false);
        else s.bs_sub = 1;
      }
      break;
    case ST_CHECK: {
      for (uint32_t t = 0; t < s.n_att; ++t) {
        const uint32_t item = s.bs_next + t;
        const bool ok = d.mot_ok[t];
        if (item == 0) s.v0 = ok;
        else if (item == 1) s.vl = ok;
        else if (!ok && s.bad_motion == kNone) s.bad_motion = item - 2;
      }
      s.bs_next += s.n_att;
      if (s.bad_motion == kNone && s.bs_next < s.n + 1) break;
      // checkAndRepair's check, then PathGeometric::check, each stopping at its first failure
      const uint32_t through = s.bad_motion == kNone ? s.n - 1 : s.bad_motion + 1;   // motions checked up to the failure
      bool pass = true;
      if (s.repair) {
        s.valids += 1;
        if (!s.v0) {
          pass = false;
        } else {
          s.valids += 1;
          if (!s.vl) pass = false;
          else if (s.n >= 3) { s.motions += through; pass = s.bad_motion == kNone; }
        }
      }
      if (pass) {
        s.valids += 1;
        if (!s.v0) pass = false;
        else { s.motions += through; pass = s.bad_motion == kNone; }
      }
      s.check_passed = pass;
      s.stage = ST_DONE;
      s.status = S_DONE;
      break;
    }
    default: break;
  }
  *d.ctl = s;
}

// The path's states, in order, to out.
__global__ void simplify_out_kernel(SimpDev d, double* __restrict__ out) {
  const uint32_t n = d.ctl->n;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n * 7; k += gridDim.x * blockDim.x)
    out[k] = d.pool[7 * (size_t)d.path[k / 7] + k % 7];
}

// SE3StateSpace::distance(a[i], b[i]) and interpolate(a[i], b[i], t[i]) with the simplifier's arithmetic (the test hook
// artp_debug_se3_ops).
__global__ void se3_ops_kernel(const double* __restrict__ a, const double* __restrict__ b, const double* __restrict__ t,
                               size_t n, double* __restrict__ dist, double* __restrict__ interp) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    dist[i] = artp::se3_distance(a + 7 * i, b + 7 * i);
    artp::se3_interpolate(a + 7 * i, b + 7 * i, t[i], interp + 7 * i);
  }
}

// PathGeometric::cost under the objective: the per-edge costs on the device, summed left to right from 0.0. states: the
// HOST copy of the path, or NULL: the learned cost's piece offsets are then computed on the device into d_off (n entries).
int path_cost(Handle* h, const double* d_states, const double* states, size_t n, int objective, double max_query_edge_length,
              uint32_t* d_off, double* cost) {
  *cost = 0.0;
  if (n < 2) return ARTP_OK;
  const size_t ne = n - 1;
  std::vector<uint32_t> off;
  size_t total = 0;
  if (objective == ARTP_OBJ_LEARNED && !states) {
    TRY(piece_offsets(h, d_states, n, max_query_edge_length, d_off, &total, h->stream));
  } else if (objective == ARTP_OBJ_LEARNED) {
    TRY(cost_piece_offsets(h, states, states + 7, ne, max_query_edge_length, off, &total));
  }
  char* r[4];   // costs | piece offsets | rows | cost3
  TRY(carve(h, h->d_stage, h->stage_cap, {ne * sizeof(double), (ne + 1) * sizeof(uint32_t), total * 6 * sizeof(float),
                                          total * 3 * sizeof(float)}, r));
  cudaStream_t s = h->stream;
  if (objective == ARTP_OBJ_LEARNED) {
    if (states) TRY(copy_async(h, r[1], off.data(), (ne + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    TRY(motion_cost_split(h, d_states, d_states + 7, ne, states ? (const uint32_t*)r[1] : d_off, total, (float*)r[2],
                          (float*)r[3], (double*)r[0], s));
  } else {
    TRY(path_length_cost(h, d_states, d_states + 7, ne, (double*)r[0], s));
  }
  std::vector<double> c(ne);
  TRY(copy_async(h, c.data(), r[0], ne * sizeof(double), cudaMemcpyDeviceToHost, s));
  TRY(sync_stream(h, s));   // `off` outlives its copy
  double sum = 0.0;
  for (double v : c) sum += v;
  *cost = sum;
  return ARTP_OK;
}

}  // namespace

extern "C" {

int artp_simplify_path(artp_handle* hh, const double* path, size_t n, const artp_se3_space* space, int objective,
                       double max_query_edge_length, uint64_t seed, double* out, size_t capacity, size_t* n_out,
                       artp_simplify_info* info) {
  LOCK_CALL(h, hh);
  if (n && !path) return null_buffer(h);
  return simplify_path(h, path, nullptr, n, space, objective, max_query_edge_length, seed, out, capacity, n_out, info);
}

}  // extern "C"

void artp_api::simplify_free(Handle* h) {
  if (!h->simplify) return;
  cudaFree(h->simplify->d_scratch);
  delete h->simplify;
  h->simplify = nullptr;
}

int artp_api::simplify_path(Handle* h, const double* path, const double* d_path, size_t n, const artp_se3_space* space,
                            int objective, double max_query_edge_length, uint64_t seed, double* out, size_t capacity,
                            size_t* n_out, artp_simplify_info* info) {
  if (!space) return null_buffer(h);
  if (n == 0) { h->err = "empty path"; return ARTP_E_INVALID; }
  if (objective != ARTP_OBJ_LEARNED && objective != ARTP_OBJ_PATH_LENGTH && objective != ARTP_OBJ_NONE) {
    h->err = "objective must be ARTP_OBJ_LEARNED, ARTP_OBJ_PATH_LENGTH or ARTP_OBJ_NONE"; return ARTP_E_INVALID;
  }
  TRY(require_whole_map(h));
  if (!d_path)
    for (size_t i = 0; i < n * 7; ++i)
      if (!std::isfinite(path[i])) { h->err = "non-finite path state"; return ARTP_E_INVALID; }
  if (n > ARTP_SIMPLIFY_MAX_STATES) { h->err = "path longer than ARTP_SIMPLIFY_MAX_STATES"; return ARTP_E_LIMIT; }
  if (objective == ARTP_OBJ_LEARNED) {
    if (!(max_query_edge_length > 0.0)) { h->err = "max_query_edge_length must be > 0"; return ARTP_E_INVALID; }
    TRY(check_cost_net(h));
  }
  SimpDev d{};
  if (!artp::segment_lengths(*space, d.seg)) { h->err = "bad SE3 space parameters"; return ARTP_E_INVALID; }
  d.seed = seed;
  // Worst case: a shortcutPath call adds at most one state per attempt and makes at most its entry length of attempts,
  // so five calls leave <= 32 n states, with <= 62 n new pool states; subdivide thrice -> <= 256 n states, and
  // smoothBSpline adds <= 7 midpoints and <= 7 replacements per state it starts from (<= 448 n).
  d.ncap = (uint32_t)(256 * n + 64);
  d.pcap = (uint32_t)(512 * n + 64);
  const size_t pairs = n * (n - 1) / 2 + 1;
  char* r[14];
  if (!h->simplify) h->simplify = new Simplify();
  TRY(carve(h, h->simplify->d_scratch, h->simplify->cap,
            {sizeof(SimpCtl), (size_t)d.pcap * 7 * sizeof(double), (size_t)d.ncap * sizeof(uint32_t),
             (size_t)d.ncap * sizeof(uint32_t), (size_t)d.ncap * sizeof(uint32_t), pairs * sizeof(double),
             (size_t)d.ncap * sizeof(double), kAttempts * sizeof(Att), kBatch * 14 * sizeof(double),
             (kBatch + 1) * sizeof(uint32_t), kBatch * 2, kBatch * 7 * sizeof(double), (size_t)d.ncap * 7 * sizeof(double),
             d_path ? (size_t)d.ncap * sizeof(uint32_t) : 0},
            r));
  d.ctl = (SimpCtl*)r[0]; d.pool = (double*)r[1]; d.path = (uint32_t*)r[2]; d.tmp = (uint32_t*)r[3]; d.cid = (uint32_t*)r[4];
  d.pair = (double*)r[5]; d.dists = (double*)r[6]; d.att = (Att*)r[7]; d.mot = (double*)r[8]; d.mot_off = (uint32_t*)r[9];
  d.mot_ok = (uint8_t*)r[10]; d.valid = (uint8_t*)r[10] + kBatch; d.chk = (double*)r[11];
  double* d_simp = (double*)r[12];   // the simplified path, in order
  uint32_t* d_off = (uint32_t*)r[13];  // device piece offsets of the learned cost (device path only)
  TRY(host_call_begin(h));
  cudaStream_t s = h->stream;
  // the input path is pool states 0 .. n-1
  std::vector<uint32_t> ids(n);
  for (size_t k = 0; k < n; ++k) ids[k] = (uint32_t)k;
  SimpCtl c{};
  c.status = S_RUNNING;
  c.stage = n >= 3 ? ST_REDUCE : ST_CHECK;
  c.repair = n >= 3;
  c.fresh = 1;
  c.n = c.np = c.n_in = (uint32_t)n;
  c.n_simplified = (uint32_t)n;
  if (d_path) CU_TRY(h, cudaMemcpyAsync(d.pool, d_path, n * 7 * sizeof(double), cudaMemcpyDeviceToDevice, s));
  else TRY(copy_async(h, d.pool, path, n * 7 * sizeof(double), cudaMemcpyHostToDevice, s));
  TRY(copy_async(h, d.path, ids.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
  TRY(copy_async(h, d.ctl, &c, sizeof(SimpCtl), cudaMemcpyHostToDevice, s));
  // rounds, kRoundsPerSync at a time; the check grid follows what the rounds asked for
  uint32_t cap = 256;
  const uint64_t max_batches = 64 * (uint64_t)n + 1024;   // far above any schedule: every round advances an attempt
  int rc = ARTP_OK;
  for (uint64_t b = 0; rc == ARTP_OK; ++b) {
    for (uint32_t k = 0; k < kRoundsPerSync && rc == ARTP_OK; ++k) {
      rc = launch(h, simplify_gather_kernel, 1, kThreads, 0, s, d, cap);
      if (rc == ARTP_OK) rc = check_states_cta(h, d.chk, &d.ctl->n_check, &d.ctl->idle, cap, d.valid, s);
      if (rc == ARTP_OK) rc = launch(h, simplify_apply_kernel, 1, kThreads, 0, s, d);
    }
    if (rc != ARTP_OK) break;
    TRY(copy_async(h, &c, d.ctl, sizeof(SimpCtl), cudaMemcpyDeviceToHost, s));
    TRY(sync_stream(h, s));
    if (c.status != S_RUNNING) break;
    cap = std::min<uint32_t>(kBatch, std::max<uint32_t>(64, (c.want + 63) & ~63u));
    if (b > max_batches) { h->err = "path simplification did not end"; rc = ARTP_E_LIMIT; }
  }
  if (rc == ARTP_OK && c.status == S_LIMIT) {
    h->err = "a motion of more than 1024 states (or the state pool overflowed)";
    rc = ARTP_E_LIMIT;
  }
  // the simplified path, and the comparison
  std::vector<double> simp(d_path ? 0 : (size_t)c.n * 7);   // a device path: the costs' piece offsets come from the device
  if (rc == ARTP_OK) rc = launch(h, simplify_out_kernel, grid_for(h, (size_t)c.n * 7, 256, 4), 256, 0, s, d, d_simp);
  if (rc == ARTP_OK && !d_path) {
    TRY(copy_async(h, simp.data(), d_simp, simp.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    TRY(sync_stream(h, s));
  }
  double cost_o = std::nan(""), cost_s = std::nan("");
  if (rc == ARTP_OK && c.check_passed && objective != ARTP_OBJ_NONE) {
    rc = path_cost(h, d_simp, d_path ? nullptr : simp.data(), c.n, objective, max_query_edge_length, d_off, &cost_s);
    if (rc == ARTP_OK) rc = path_cost(h, d.pool, path, n, objective, max_query_edge_length, d_off, &cost_o);
  }
  const int rc_end = host_call_end(h, true);
  if (rc != ARTP_OK) return rc;
  if (rc_end != ARTP_OK) return rc_end;
  const bool simplified = c.check_passed && !(cost_o < cost_s);
  const size_t nr = simplified ? c.n : n;
  if (info) {
    artp_simplify_info o{};
    o.n_in = (uint32_t)n; o.n_simplified = c.n_simplified; o.n_out = (uint32_t)nr;
    o.reduce_edits = c.edits[0]; o.collapse_edits = c.edits[1]; o.shortcut_edits = c.edits[2]; o.bspline_edits = c.edits[3];
    o.motion_checks = c.motions; o.state_checks = c.valids; o.rounds = c.rounds; o.discarded = c.discarded;
    o.check_passed = (int32_t)c.check_passed; o.returned_simplified = simplified;
    o.cost_original = cost_o; o.cost_simplified = cost_s;
    *info = o;
  }
  if (n_out) *n_out = nr;
  if (nr > capacity) { h->err = "capacity too small"; return ARTP_E_LIMIT; }
  if (out && d_path) {   // the returned path's one trip to the host
    TRY(copy_async(h, out, simplified ? d_simp : d.pool, nr * 7 * sizeof(double), cudaMemcpyDeviceToHost, s));
    TRY(sync_stream(h, s));
  } else if (out) {
    std::copy_n(simplified ? simp.data() : path, nr * 7, out);
  }
  return ARTP_OK;
}

extern "C" {

int artp_debug_se3_ops(artp_handle* hh, const double* a, const double* b, const double* t, size_t n, double* dist,
                       double* interp) {
  LOCK_CALL(h, hh);
  if (n == 0) return ARTP_OK;
  if (!a || !b || !t || !dist || !interp) return null_buffer(h);
  const size_t sb = n * 7 * sizeof(double);
  char* r[5];   // a | b | t | dist | interp
  TRY(host_call_begin(h, {sb, sb, n * sizeof(double), n * sizeof(double), sb}, r));
  cudaStream_t s = h->stream;
  CU_TRY(h, cudaMemcpyAsync(r[0], a, sb, cudaMemcpyHostToDevice, s));
  CU_TRY(h, cudaMemcpyAsync(r[1], b, sb, cudaMemcpyHostToDevice, s));
  CU_TRY(h, cudaMemcpyAsync(r[2], t, n * sizeof(double), cudaMemcpyHostToDevice, s));
  TRY(launch(h, se3_ops_kernel, grid_for(h, n, 256, 4), 256, 0, s, (const double*)r[0], (const double*)r[1], (const double*)r[2],
             n, (double*)r[3], (double*)r[4]));
  CU_TRY(h, cudaMemcpyAsync(dist, r[3], n * sizeof(double), cudaMemcpyDeviceToHost, s));
  CU_TRY(h, cudaMemcpyAsync(interp, r[4], sb, cudaMemcpyDeviceToHost, s));
  return host_call_end(h);
}

}  // extern "C"
