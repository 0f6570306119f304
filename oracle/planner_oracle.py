"""CPU restatement of the rules artp_planner_set_map / artp_plan add to the stages they compose (TEST INFRASTRUCTURE ONLY).

The stages themselves are restated elsewhere: Basic (basic_oracle.py), the sample distribution
(sample_distribution_oracle.py), the roadmap (roadmap_oracle.py), its queries (roadmap_query_oracle.py), the start / goal
search (tests/start_goal_oracle.py) and the simplifier (path_simplify_oracle.py). What is new here, with its reference lines:
  observed        addKnownCells (art_planner/src/map/processors/basic.cpp:25-38) over Map::setMap's basic layers
                  {elevation, traversability} (map.cpp:16); grid_map's isValid (all basic layers finite) is not in the
                  reference tree: restated, unpinned. checkTraversability (basic.cpp:13-21) supplies 1.0 when the map has
                  no traversability layer.
  se3_bounds      Planner::setMap (planner.cpp:146-156): x, y = position -+ the FULL length; z = (double)minCoeffOfFinites
                  - reach.z / 2 .. (double)maxCoeffOfFinites + reach.z / 2 of the RAW elevation. -0 counts as +0. No finite
                  cell: an error (grid_map's result is not pinned).
  satisfies_bounds / enforce_bounds
                  Planner::plan (planner.cpp:207-221) on the goal, OMPL 1.4.2's SE3StateSpace (not in the tree: restated,
                  unpinned): RealVectorStateSpace::satisfiesBounds with the DBL_EPSILON slack and the clamp of
                  enforceBounds; SO3StateSpace::satisfiesBounds |norm - 1| < MAX_QUATERNION_NORM_ERROR (1e-9), and its
                  enforceBounds: when |x^2 + y^2 + z^2 + w^2 - 1| > DBL_EPSILON, the identity below a norm of
                  DBL_EPSILON, else the components divided by the norm.
  status          Planner::plan's switch (planner.cpp:254-261) and planner_status.h.
  sample_rule     PRMMotionCostMaintainer::sampleGraph (prm_motion_cost.cpp:146-153): sample (and updateEdges) only when the
                  map's timestamp differs from the one the last sampleGraph saw; the map generation stands in for it.
  streams         the positions artp_plan keeps: sampler draws advance by the draws used, each search by k (candidate k
                  returned) or n_iter (none valid), the simplifier's key by one per simplify.
"""
from __future__ import annotations

import math
import sys

import numpy as np

DBL_EPSILON = sys.float_info.epsilon
QUAT_NORM_ERROR = 1e-9

UNKNOWN, INVALID_START, INVALID_GOAL, NO_MAP, NOT_SOLVED, SOLVED = range(6)          # planner_status.h
SOLVE_SOLVED, SOLVE_NOT_CONNECTED, SOLVE_NO_FEASIBLE_PATH, SOLVE_INVALID_START, SOLVE_INVALID_GOAL = 1, 2, 3, 4, 5


def observed(elevation, traversability=None) -> np.ndarray:
    """addKnownCells: float32 1 where elevation (and traversability, when given) is finite, else 0."""
    ok = np.isfinite(np.asarray(elevation, np.float32))
    if traversability is not None:
        ok &= np.isfinite(np.asarray(traversability, np.float32))
    return np.asfortranarray(ok.astype(np.float32))


def se3_bounds(elevation, res: float, cx: float, cy: float, reach_z: float):
    """(low[3], high[3]) of Planner::setMap from the raw elevation; ValueError without a finite cell."""
    e = np.asarray(elevation, np.float32)
    f = e[np.isfinite(e)]
    if f.size == 0:
        raise ValueError("no finite cell")
    lo, hi = float(f.min() + np.float32(0)), float(f.max() + np.float32(0))   # -0 as +0
    lx, ly = e.shape[0] * res, e.shape[1] * res
    return [cx - lx, cy - ly, lo - reach_z / 2], [cx + lx, cy + ly, hi + reach_z / 2]


def quat_norm(s) -> float:
    return math.sqrt(s[3] * s[3] + s[4] * s[4] + s[5] * s[5] + s[6] * s[6])


def satisfies_bounds(s, low, high) -> bool:
    for i in range(3):
        if s[i] - DBL_EPSILON > high[i] or s[i] + DBL_EPSILON < low[i]:
            return False
    return abs(quat_norm(s) - 1.0) < QUAT_NORM_ERROR


def enforce_bounds(s, low, high) -> np.ndarray:
    out = np.array(s, dtype=np.float64).reshape(7)
    for i in range(3):
        if out[i] > high[i]:
            out[i] = high[i]
        elif out[i] < low[i]:
            out[i] = low[i]
    nrm_sq = out[3] * out[3] + out[4] * out[4] + out[5] * out[5] + out[6] * out[6]
    if abs(nrm_sq - 1.0) > DBL_EPSILON:
        n = math.sqrt(nrm_sq)
        if n < DBL_EPSILON:
            out[3:] = (0.0, 0.0, 0.0, 1.0)
        else:
            for k in range(3, 7):
                out[k] = out[k] / n
    return out


def clip_goal(goal, low, high):
    """(state, clipped): planner.cpp:207-221."""
    g = np.array(goal, dtype=np.float64).reshape(7)
    if satisfies_bounds(g, low, high):
        return g, False
    return enforce_bounds(g, low, high), True


def status(solve_status: int) -> int:
    return {SOLVE_SOLVED: SOLVED, SOLVE_NOT_CONNECTED: NOT_SOLVED, SOLVE_NO_FEASIBLE_PATH: NOT_SOLVED,
            SOLVE_INVALID_START: INVALID_START, SOLVE_INVALID_GOAL: INVALID_GOAL}.get(solve_status, UNKNOWN)


class GenerationRule:
    """The map-generation rule of PRMMotionCostMaintainer::sampleGraph, with clear_roadmap (PRMMotionCost::clear)."""

    def __init__(self):
        self.generation = 0
        self.sampled = 0

    def new_map(self) -> None:
        self.generation += 1

    def plan(self, clear_roadmap: bool):
        """(clear the roadmap, sample + updateEdges) for one plan."""
        sample = self.sampled != self.generation
        self.sampled = self.generation
        return bool(clear_roadmap), sample


def advance(draw: int, index: int, n_iter: int) -> int:
    """A search's stream position after it returned candidate `index` (-1: none valid)."""
    return draw + (index if index >= 0 else n_iter)


class Replan:
    """The whole replan of Planner::setMap + plan + getSolutionPath(simplify) for prm_motion_cost (planner.cpp:135-298),
    composed from the restatements of its stages and the rules above. Each stage cites its own restatement:
      set_map  observed, se3_bounds; processors::Basic (basic_oracle.masked_elevation, basic.cpp:42-106); estimateNormals
               (orc.estimate_normals, utils.cpp:213-324); with sample_from_distribution, setTraversabilityFilter
               (sample_distribution_oracle.sample_filter, basic.cpp:110-125) and the distribution without vertices
               (sample_distribution_oracle.distribution, planner.cpp:39-58); the sampler's bounds (planner.cpp:148-160).
      plan     NO_MAP (:197-200); PRMMotionCost::clear when asked; sampleGraph + updateEdges under the generation rule
               (roadmap_oracle.sample_graph, prm_motion_cost.cpp:145-219; roadmap_query_oracle.update_edges, :27-73);
               clip_goal (:207-221); the projection (start_goal_oracle.pose_from_2d, :223-237); the start and goal searches
               (start_goal_oracle.find_valid_near, start.cpp:7-41, goal.cpp:11-41, called at :167-189); baseSolve
               (roadmap_query_oracle.base_solve, prm_motion_cost.cpp:440-673); the status table (:254-261); when solved and
               simplifying, getSolutionPath (path_simplify_oracle.get_solution_path, :266-298).
    What the restatements take from outside, exactly as their own tests do: isValid from `oracle` (orc.Oracle), the
    learned cost of edges and paths (`edge_cost(src, tgt)`, `path_cost(states)`), SE(3) distance / interpolate for the
    simplifier (`ops`), the searches' offsets (`ball_offsets(seed, first_draw, n_iter, radius)` -> [n_iter, 2]) and the
    sampler's variates (roadmap_oracle.sdo_uniforms). Streams follow artp_plan's: the sampler key is the seed, the start
    search's key the seed and the goal search's ~seed, the simplifier's seed + the number of simplifies so far."""

    def __init__(self, rp, params, oracle, edge_cost, path_cost, ops, ball_offsets, sample_distribution_params):
        self.rp, self.pp, self.o = rp, params, oracle
        self.edge_cost, self.path_cost, self.ops, self.ball_offsets = edge_cost, path_cost, ops, ball_offsets
        self.dp = sample_distribution_params
        self.rule = GenerationRule()
        self.rm = None
        self.m = None
        self.seed = None

    def set_map(self, e, t, ei, ti, res, cx, cy):
        import copy
        from art_planner_b200 import synth
        from oracle import basic_oracle as bo
        from oracle import orc
        from oracle import sample_distribution_oracle as sdo
        pp, rp = self.pp, self.rp
        obs = observed(e, t)
        self.low, self.high = se3_bounds(e, res, cx, cy, rp.reach_z)
        if ti is None:
            ti = np.ones(np.shape(e), np.float32, order="F")
        masked, thr = bo.masked_elevation(ei, ti, obs, res, pp.basic)
        m = synth.SynthMap(np.asfortranarray(ei, dtype=np.float32), masked, res, cx, cy, "planner")
        nx, ny, nz, sd = orc.estimate_normals(m, (rp.torso_length + rp.torso_width) * 0.25)
        self.filter = self.obs = None
        cum = np.zeros((m.rows, m.cols), np.float32, order="F")
        row = np.zeros(m.rows, np.float32)
        if pp.sample_from_distribution:
            self.filter, self.obs = sdo.sample_filter(thr, rp, res), obs
            d = sdo.distribution(np.zeros((0, 7)), m, self.dp, self.filter, self.obs)
            cum, row = d["cum_prob"], d["cum_prob_rowwise"]
        self.layers = synth.SamplerLayers(nx, ny, nz, sd, None, cum, row)
        self.sp = synth.SamplerParams(float(pp.max_roll_pert), float(pp.max_pitch_pert), bool(pp.sample_from_distribution),
                                      (self.low[0], self.low[1]), (self.high[0], self.high[1]))
        self.o.set_map(m)
        self.m = m
        self.layers0 = copy.copy(self.layers)
        self.rule.new_map()

    def plan(self, start, goal):
        """(status, path [n, 7], record): the record holds what artp_plan_info reports (the roadmap as self.rm)."""
        from oracle import path_simplify_oracle as pso
        from oracle import roadmap_oracle as ro
        from oracle import roadmap_query_oracle as rqo
        import start_goal_oracle as sgo   # tests/ is on sys.path under pytest
        pp = self.pp
        if self.m is None:
            return NO_MAP, np.zeros((0, 7)), {"status": NO_MAP}
        if self.seed != pp.seed:
            self.seed = pp.seed
            self.next_sample = self.start_draw = self.goal_draw = self.simplify_calls = 0
        rec = {"first_sample": self.next_sample, "start_draw": self.start_draw, "goal_draw": self.goal_draw, "sampled": 0,
               "draws_used": 0}
        clear, sample = self.rule.plan(bool(pp.clear_roadmap))
        if self.rm is None or clear:
            self.rm = rqo.QueryRoadmap(int(pp.vertex_capacity))
        is_valid = ro.validity(self.o)
        if sample:
            used, _, _ = ro.sample_graph(self.rm, self.o, self.m, self.layers0, self.sp, self.rp.reach_z, pp.seed, self.next_sample,
                                         pp.max_n_vertices, pp.max_n_edges,
                                         pp.recompute_density_after_n_samples if pp.sample_from_distribution else 0,
                                         pp.max_draws, self.dp if pp.sample_from_distribution else None, self.filter, self.obs,
                                         is_valid=is_valid)
            rqo.update_edges(self.rm, self.edge_cost)
            self.next_sample += used
            rec.update(sampled=1, draws_used=used)
        clipped, was_clipped = clip_goal(goal, self.low, self.high)
        proj, inside = sgo.pose_from_2d(self.m, self.layers0, clipped.reshape(1, 7))
        s_rep, s_idx = sgo.find_valid_near(self.o, np.asarray(start, np.float64).reshape(1, 7), pp.n_iter,
                                           self.ball_offsets(pp.seed, self.start_draw, pp.n_iter, pp.start_radius))
        g_rep, g_idx = sgo.find_valid_near(self.o, proj, pp.n_iter,
                                           self.ball_offsets(~pp.seed & ((1 << 64) - 1), self.goal_draw, pp.n_iter, pp.goal_radius))
        self.start_draw = advance(self.start_draw, int(s_idx[0]), pp.n_iter)
        self.goal_draw = advance(self.goal_draw, int(g_idx[0]), pp.n_iter)
        rec.update(goal_clipped=int(was_clipped), goal_inside=int(inside[0]), start_index=int(s_idx[0]), goal_index=int(g_idx[0]),
                   goal_clipped_state=clipped, goal_projected=proj[0], start_repaired=s_rep[0], goal_repaired=g_rep[0])
        space = (self.low, self.high, 0.01)
        check_motion = rqo.discrete_motion(is_valid, space)
        in_bounds = lambda s: all(self.low[i] <= s[i] <= self.high[i] for i in range(3))
        ref = rqo.base_solve(self.rm, s_rep[0], g_rep[0], is_valid, self.edge_cost, check_motion, in_bounds)
        rec["solve"] = ref
        st = status(ref["status"])
        path = np.zeros((0, 7))
        if st == SOLVED:
            path = self.rm.states[ref["path"]].copy()
            rec["path_cost"] = ref["cost"]
            if pp.simplify:
                rec["simplify_seed"] = pp.seed + self.simplify_calls
                self.simplify_calls += 1
                path, rec["simplify"], _ = pso.get_solution_path(path, is_valid, space, rec["simplify_seed"], self.path_cost,
                                                                 ops=self.ops)
        rec["status"] = st
        return st, path, rec
