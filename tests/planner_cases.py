"""The replan through the chained public calls, step for step what artp_planner_set_map + artp_plan do in one call each, and
the raw / inpainted layers both routes take. Used by tests/test_planner_gpu.py and profiles/replan_time.py."""
from __future__ import annotations

import ctypes as C
import numpy as np

from art_planner_b200 import capi, synth
from oracle import planner_oracle as po

MASK64 = (1 << 64) - 1


def raw_layers(m: synth.SynthMap, seed: int = 13, holes: float = 0.01, traversability: bool = True):
    """(raw elevation, raw traversability, inpainted elevation, inpainted traversability): NaN holes punched into the map's
    layers stand for unknown cells; the map's own layers stand for what inpaintMatrix returns (finite everywhere)."""
    trav, _ = synth.make_traversability(m, seed=seed)
    k = np.arange(m.rows * m.cols).reshape(m.rows, m.cols)
    hole = synth.hash_uniform(seed, 51, (np.arange(m.rows)[:, None] // 9) * 4096 + (np.arange(m.cols)[None, :] // 7)) < holes * 8
    hole |= synth.hash_uniform(seed, 52, k) < holes
    raw_e = np.asfortranarray(np.where(hole, np.nan, m.elevation).astype(np.float32))
    if not traversability:
        return raw_e, None, np.asfortranarray(m.elevation), None
    raw_t = np.asfortranarray(np.where(synth.hash_uniform(seed, 53, k) < holes, np.nan, trav).astype(np.float32))
    return raw_e, raw_t, np.asfortranarray(m.elevation), trav


class Chained:
    """The replan of artp_plan through the public entry points (the route a caller had before the planner calls)."""

    def __init__(self, chk, params):
        self.chk, self.pp = chk, params
        self.h = chk.handle
        self.generation = self.sampled = 0
        self.rm = None
        self.seed = None

    def setMap(self, e, t, ei, ti, res, cx, cy):
        pp, h, rp = self.pp, self.h, self.h.params
        obs = po.observed(e, t)
        low, high = po.se3_bounds(e, res, cx, cy, rp.reach_z)
        self.space = capi.ArtpSe3Space((C.c_double * 3)(*low), (C.c_double * 3)(*high), 0.01)
        if ti is None:
            ti = np.ones(e.shape, np.float32, order="F")
        masked, thr = self.chk.processBasic(ei, ti, obs, res, pp.basic)
        self.chk.setMap(synth.SynthMap(np.asfortranarray(ei, dtype=np.float32), masked, res, cx, cy, "planner"))
        # the layers the public calls take and return: Basic's three in and two out, the map upload's two in
        lb = 4 * ei.size
        self.map_bytes = {"bytes_h2d": 3 * lb + 2 * lb, "bytes_d2h": masked.nbytes + thr.nbytes}
        self.chk.updateHeightField()
        self.chk.estimateNormals((rp.torso_length + rp.torso_width) * 0.25, want_host=False)
        if pp.sample_from_distribution:
            self.chk.setSampleFilter(None, None, want_host=False)
            self.chk.updateSampleDistribution(np.zeros((0, 7)), self.dp(), want_host=False)
        sp = capi.ArtpSamplerParams(pp.max_roll_pert, pp.max_pitch_pert, pp.sample_from_distribution, (C.c_double * 2)(low[0], low[1]),
                                    (C.c_double * 2)(high[0], high[1]))
        h.check(h.lib.artp_set_sampler(h.h, C.byref(sp), None, None, None, None, None, None))
        net = C.c_int()
        if h.lib.artp_get_cost_network(h.h, C.byref(net)) == 0:
            h.check(h.lib.artp_update_features(h.h))
        self.generation += 1

    def dp(self):
        rp, pp = self.h.params, self.pp
        return capi.ArtpSampleDistributionParams(pp.use_inverse_vertex_density, (rp.torso_length + rp.torso_width) * 0.25,
                                                 pp.use_max_prob_unknown_samples, pp.max_prob_unknown_samples)

    def plan(self, start, goal):
        """(status, path, record): record holds what artp_plan_info reports."""
        import art_planner_b200 as ap
        pp, h = self.pp, self.h
        if self.seed != pp.seed:
            self.seed = pp.seed
            self.next_sample = self.start_draw = self.goal_draw = self.simplify_calls = 0
        rec = dict(sampled=0, draws_used=0, first_sample=self.next_sample, start_draw=self.start_draw, goal_draw=self.goal_draw)
        if self.rm is None:
            self.rm = ap.PRMRoadmap(self.chk, pp.vertex_capacity, pp.edge_capacity)
        elif pp.clear_roadmap:
            self.rm.clear()
        if self.sampled != self.generation:
            rp = capi.ArtpRoadmapParams(pp.max_n_vertices, pp.max_n_edges, pp.recompute_density_after_n_samples, pp.max_draws)
            dp = self.dp()
            used = C.c_uint64(0)
            h.check(h.lib.artp_roadmap_sample_graph(h.h, C.byref(rp), C.byref(dp) if pp.sample_from_distribution else None,
                                                    pp.seed, self.next_sample, C.byref(used)))
            self.rm.updateEdges()
            self.sampled = self.generation
            self.next_sample += used.value
            rec.update(sampled=1, draws_used=used.value)
        low, high = list(self.space.low), list(self.space.high)
        clipped, was_clipped = po.clip_goal(goal, low, high)
        proj, inside = self.chk.poseFrom2D(clipped.reshape(1, 7))
        s_rep, s_idx = self.chk.findValidNear(np.asarray(start, np.float64).reshape(1, 7), pp.start_radius, pp.n_iter,
                                              seed=pp.seed, first_draw=self.start_draw)
        g_rep, g_idx = self.chk.findValidNear(proj, pp.goal_radius, pp.n_iter, seed=~pp.seed & MASK64, first_draw=self.goal_draw)
        self.start_draw = po.advance(self.start_draw, int(s_idx[0]), pp.n_iter)
        self.goal_draw = po.advance(self.goal_draw, int(g_idx[0]), pp.n_iter)
        rec.update(goal_clipped=int(was_clipped), goal_inside=int(inside[0]), start_index=int(s_idx[0]), goal_index=int(g_idx[0]),
                   goal_clipped_state=clipped, goal_projected=proj[0], start_repaired=s_rep[0], goal_repaired=g_rep[0])
        solve_status, states, _, cost, sinfo = self.rm.solve(s_rep[0], g_rep[0], self.space, path_capacity=pp.vertex_capacity)
        rec.update(solve=dict(status=solve_status, **sinfo), path_cost=cost if solve_status == po.SOLVE_SOLVED else 0.0)
        status = po.status(solve_status)
        path = np.zeros((0, 7))
        if status == po.SOLVED:
            path = states
            if pp.simplify:
                rec["simplify_seed"] = pp.seed + self.simplify_calls
                self.simplify_calls += 1
                path, rec["simplify"] = ap.PathSimplifier(self.chk, self.space, "learned", rec["simplify_seed"],
                                                          pp.max_query_edge_length).getSolutionPath(states)
        nv, ne = self.rm.counts()
        rec.update(n_vertices=nv, n_edges=ne)
        return status, path, rec


def queries(chk, n, seed, dist):
    """n (start, goal) pairs of valid states about `dist` apart in (x, y), drawn from the sampler chk holds (its own
    stream, `seed`: a planner's draws are untouched); the goals keep their (x, y) and yaw at z = 0, as a 2-D goal arrives
    (Planner::plan projects it onto the map)."""
    h = chk.handle
    out = np.empty((4096, 7))
    nv = C.c_size_t(0)
    h.check(h.lib.artp_sample_valid(h.h, 1000 + seed, 0, 1 << 16, out.ctypes.data, 4096, C.byref(nv)))
    v = out[:min(nv.value, 4096)]
    q = []
    for k in range(n):
        d = np.hypot(v[:, 0] - v[k, 0], v[:, 1] - v[k, 1])
        b = v[int(np.argmin(np.abs(d - dist)))].copy()
        yaw = np.arctan2(2.0 * (b[6] * b[5] + b[3] * b[4]), 1.0 - 2.0 * (b[4] * b[4] + b[5] * b[5]))
        b[2:] = (0.0, 0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2))
        q.append((v[k], b))
    return q


def small_params(**kw):
    """Planner parameters at the roadmap_cases caps."""
    import art_planner_b200 as ap
    d = dict(max_n_vertices=1500, max_n_edges=6000, recompute_density_after_n_samples=300, max_draws=1 << 22,
             vertex_capacity=8000, edge_capacity=20000, n_iter=200)
    d.update(kw)
    return ap.Planner.params(**d)
