"""GPU parity (-m gpu) of artp_simplify_path against oracle/path_simplify_oracle.py. The restatement takes isValid from
the port oracle, the same Philox stream, SE(3) distance / interpolate from artp_debug_se3_ops and the device's own cost
calls for the final comparison (artp_motion_cost_split / artp_path_length_cost: the same kernels, so costs are compared
exactly). Compared: every counter of the info, which
path was returned, its length exactly and its states within 1e-9. Inputs: paths solved on the device roadmap over the
roadmap_cases maps (both robot presets, the off-origin map), both objectives, 2- and 3-state paths, a straight path,
paths whose simplified form fails the check, and one query at the shipped caps."""
import numpy as np
import pytest

import roadmap_cases as rc
from art_planner_b200 import capi, costnet, synth
from oracle import orc
from oracle import path_simplify_oracle as pso
from oracle import roadmap_oracle as ro
from oracle import roadmap_query_oracle as rqo

pytestmark = pytest.mark.gpu
STATE_TOL = 1e-9
COUNTERS = ("n_in", "n_simplified", "n_out", "reduce_edits", "collapse_edits", "shortcut_edits", "bspline_edits",
            "motion_checks", "state_checks", "check_passed", "returned_simplified")


class DeviceOps:
    """SE3StateSpace::distance / ::interpolate from artp_debug_se3_ops: the device's own arithmetic."""

    def __init__(self, handle):
        self.h = handle

    def _run(self, A, B, T):
        A = np.ascontiguousarray(A, np.float64).reshape(-1, 7)
        B = np.ascontiguousarray(B, np.float64).reshape(-1, 7)
        T = np.ascontiguousarray(np.broadcast_to(np.asarray(T, np.float64), (len(A),)))
        dist, interp = np.empty(len(A)), np.empty((len(A), 7))
        self.h.check(self.h.lib.artp_debug_se3_ops(self.h.h, A.ctypes.data, B.ctypes.data, T.ctypes.data, len(A),
                                                   dist.ctypes.data, interp.ctypes.data))
        return dist, interp

    def distance(self, A, B):
        return self._run(A, B, 0.0)[0]

    def interpolate(self, A, B, T):
        return self._run(A, B, T)[1]


class Env:
    def __init__(self, c, thr=0.6, weights=True):
        import art_planner_b200 as ap
        from art_planner_b200.checker import _Handle
        self.c = c
        self.chk = ap.StateValidityChecker(c.rp, handle=_Handle(c.rp, 0, risk_threshold=thr))
        self.chk.setMap(c.m)
        self.chk.updateHeightField()
        self.obj = ap.MotionCostObjective(self.chk)
        if weights:
            self.obj.setWeights(costnet.make_state_dict(seed=5))
            self.obj.updateFeatures()
        self.plo = ap.PathLengthObjective(self.chk)
        self.o = orc.Oracle(c.rp, "port")
        self.o.set_map(c.m)
        self.is_valid = ro.validity(self.o)
        self.space = ap.MotionValidator.se3Space(c.m, c.rp.reach_z)
        self.bounds = (list(self.space.low), list(self.space.high), 0.01)
        self.check_motion = rqo.discrete_motion(self.is_valid, self.bounds)
        self.ops = DeviceOps(self.chk.handle)

    def path_cost(self, objective):
        def cost(states):
            if len(states) < 2:
                return 0.0
            if objective == "learned":
                return self.obj.pathCost(states)
            total = 0.0
            for v in self.plo.motionCostBatch(states[:-1], states[1:]).tolist():
                total += v
            return total
        return cost

    def both(self, path, objective="learned", seed=7):
        import art_planner_b200 as ap
        ps = ap.PathSimplifier(self.chk, self.space, objective, seed)
        got, info = ps.getSolutionPath(path)
        ref, rinfo, _ = pso.get_solution_path(path, self.is_valid, self.bounds, seed, self.path_cost(objective), ops=self.ops)
        assert {k: info[k] for k in COUNTERS} == {k: rinfo[k] for k in COUNTERS}, f"\ndevice {info}\nrestated {rinfo}"
        assert got.shape == ref.shape and np.abs(got - ref).max(initial=0.0) <= STATE_TOL
        if info["check_passed"]:
            assert info["cost_original"] == rinfo["cost_original"]
            assert info["cost_simplified"] == rinfo["cost_simplified"]
        else:
            assert np.isnan(info["cost_original"]) and np.isnan(info["cost_simplified"])
        # the returned path: the input's endpoints, every motion valid under the port oracle, no dearer than the input
        assert np.array_equal(got[0], np.asarray(path)[0]) and np.array_equal(got[-1], np.asarray(path)[-1])
        if info["returned_simplified"] and len(got) > 1:
            assert all(self.check_motion(a, b) for a, b in zip(got[:-1], got[1:]))
            assert info["cost_simplified"] <= info["cost_original"]
        return got, info


def solved_paths(c, n_queries, seed, caps=rc.CAPS, vcap=8000, ecap=20000, thr=0.6):
    """Paths of artp_roadmap_solve between valid states near far-apart milestones."""
    import art_planner_b200 as ap
    env = Env(c, thr)
    smp = ap.SE3FromSE2Sampler(env.chk, c.layers, c.sp, seed=rc.SEED)
    rm = ap.PRMRoadmap(env.chk, vcap, ecap)
    rm.sampleGraph(smp, *caps, max_draws=rc.MAX_DRAWS, distribution=False)
    rm.updateEdges()
    st, kinds = rm.vertices()
    ms = st[kinds == ro.MILESTONE]
    k = (synth.hash_uniform(seed, 1, np.arange(8 * n_queries)) * len(ms)).astype(int)
    cand = ms[k] + np.array([0.011, -0.017, 0, 0, 0, 0, 0])
    cand = cand[env.is_valid(cand)]
    paths = []
    for a, b in zip(cand[0::2], cand[1::2]):
        status, states, _, _, _ = rm.solve(a, b, env.space)
        if status == rqo.SOLVED:
            paths.append(states)
        if len(paths) == n_queries:
            break
    return env, paths


@pytest.mark.parametrize("name", list(rc.CASES))
@pytest.mark.parametrize("objective", ["learned", "path_length"])
def test_solved_paths_match_restatement(name, objective):
    env, paths = solved_paths(rc.make_case(name), 4, seed=101)
    assert paths
    edited = 0
    for i, p in enumerate(paths):
        _, info = env.both(p, objective, seed=11 + i)
        edited += info["reduce_edits"] + info["collapse_edits"] + info["shortcut_edits"] + info["bspline_edits"]
        assert info["rounds"] >= 1
    assert edited > 0


def test_short_and_straight_paths():
    env, paths = solved_paths(rc.make_case("rough_fbm"), 2, seed=102)
    p = max(paths, key=len)
    # 2 and 3 states: the schedule does not run (2) or runs on the smallest path it edits (3)
    got, info = env.both(p[[0, -1]], "path_length")
    assert info["n_simplified"] == 2 and info["motion_checks"] == 1
    env.both(p[[0, len(p) // 2, -1]], "learned")
    env.both(p[:1], "learned")
    # a straight, valid path of many states: reduceVertices' first check connects the ends
    # a straight path of 9 states along the solved path's first edge (a motion the query validated): its ends connect
    straight = np.array([ro.interpolate(p[0], p[1], t) for t in np.linspace(0.0, 1.0, 9)])
    assert env.check_motion(straight[0], straight[-1])
    _, info = env.both(straight, "path_length")
    assert info["reduce_edits"] >= 1 and info["n_simplified"] == 2 and info["collapse_edits"] == 0


def test_failing_check_returns_the_original():
    env, paths = solved_paths(rc.make_case("gentle_inf"), 2, seed=103)
    p = max(paths, key=len).copy()
    p[-1, 2] += 3.0                      # the goal in the air: invalid
    assert not env.is_valid(p[-1:])[0]
    got, info = env.both(p, "learned")
    assert info["check_passed"] == 0 and info["returned_simplified"] == 0 and np.array_equal(got, p)
    q = p[[0, -1]].copy()                # two states: only PathGeometric::check runs
    got, info = env.both(q, "path_length")
    assert info["check_passed"] == 0 and np.array_equal(got, q)


def test_seed_changes_draws_not_rules():
    env, paths = solved_paths(rc.make_case("offgrid_r1"), 1, seed=104)
    for seed in (0, 1, 2 ** 40 + 3):
        env.both(paths[0], "learned", seed)


def test_error_codes():
    import ctypes as C
    import art_planner_b200 as ap
    env = Env(rc.make_case("rough_fbm"), weights=False)
    h, lib = env.chk.handle, env.chk.handle.lib
    p = synth.make_terrain_poses(env.c.m, 1000, seed=5)
    p = np.ascontiguousarray(p[env.is_valid(p)][:5])
    assert p.shape == (5, 7)   # every call below reads 5 states from p
    out = np.empty((400, 7))

    def call(path, n, objective=capi.ARTP_OBJ_PATH_LENGTH, cap=400, handle=h.h):
        return lib.artp_simplify_path(handle, path.ctypes.data, n, C.byref(env.space), objective, 0.5, 1, out.ctypes.data,
                                      cap, None, None)
    assert call(p, 0) == capi.ARTP_E_INVALID
    bad = p.copy(); bad[1, 0] = np.nan
    assert call(bad, 5) == capi.ARTP_E_INVALID
    assert call(p, 5, objective=7) == capi.ARTP_E_INVALID
    big = np.repeat(p[:1], capi.ARTP_SIMPLIFY_MAX_STATES + 1, axis=0)
    assert call(big, len(big)) == capi.ARTP_E_LIMIT
    assert call(p, 5, cap=1) == capi.ARTP_E_LIMIT and b"capacity" in lib.artp_last_error(h.h), lib.artp_last_error(h.h)
    assert call(p, 5, objective=capi.ARTP_OBJ_LEARNED) == capi.ARTP_E_NOWEIGHTS
    assert call(p, 5) == capi.ARTP_OK, lib.artp_last_error(h.h)
    c2 = ap.StateValidityChecker(env.c.rp, device=0)
    assert call(p, 5, handle=c2.handle.h) == capi.ARTP_E_NOMAP
    m = env.c.m
    c2.setMap(m)
    c2.updateHeightField(window=(0, 64))
    assert call(p, 5, handle=c2.handle.h) == capi.ARTP_E_INVALID


def test_shipped_caps_config1():
    """One query at the shipped caps (10 000 vertices / 50 000 edges) on the configs[1] map."""
    import dataclasses
    from oracle import basic_oracle as bo
    from oracle import sample_distribution_oracle as sdo
    m = synth.make_fbm_map(1000, 1000)
    rp = synth.PARAMS_YAML
    trav, obs = synth.make_traversability(m, seed=13)
    _, thr = bo.masked_elevation(m.elevation, trav, obs, m.res, bo.BasicParams())
    sp = dataclasses.replace(synth.sampler_params_for(m), use_inverse_vertex_density=True, use_max_prob_unknown_samples=True)
    c = rc.Case(m, rp, synth.make_sampler_layers(m, seed=7), sp, None, thr, sdo.sample_filter(thr, rp, m.res), obs)
    env, paths = solved_paths(c, 1, seed=105, caps=(10000, 50000, 1000), vcap=20000, ecap=60000)
    assert paths
    env.both(paths[0], "learned")


@pytest.mark.parametrize("name", ["gentle_inf", "rough_fbm"])
def test_golden_paths(name):
    """The golden's input paths (tests/golden/path_simplify.npz, the restatement over the reference's compiled ODE): the
    device's simplifyMax (no cost comparison) against the golden's simplified path and counters."""
    import os
    from oracle import make_golden_path_simplify as mg
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "path_simplify.npz"))
    import art_planner_b200 as ap
    env = Env(rc.make_case(name))
    col = {k: i for i, k in enumerate(mg.INFO_KEYS)}
    for k in range(len(mg.SEEDS)):
        key = f"{name}/{k}"
        path, seed, ginfo = g[f"{key}/path"], int(g[f"{key}/seed"][0]), g[f"{key}/info"]
        got, info = ap.PathSimplifier(env.chk, env.space, "path_length", seed).simplifyMax(path)
        for c in ("n_in", "n_simplified", "reduce_edits", "collapse_edits", "shortcut_edits", "bspline_edits",
                  "motion_checks", "state_checks", "check_passed"):
            assert info[c] == ginfo[col[c]], (key, c, info[c], int(ginfo[col[c]]))
        want = g[f"{key}/simplified"] if info["check_passed"] else path
        assert got.shape == want.shape and np.abs(got - want).max() <= STATE_TOL


@pytest.mark.parametrize("name", list(rc.CASES))
def test_solved_paths_match_libm_restatement(name):
    """The same comparison with the restatement's own libm distance / interpolate: on these paths no tie is broken
    differently, so the device also matches a restatement that shares none of its arithmetic."""
    env, paths = solved_paths(rc.make_case(name), 4, seed=101)
    import art_planner_b200 as ap
    for i, p in enumerate(paths):
        got, info = ap.PathSimplifier(env.chk, env.space, "path_length", 11 + i).getSolutionPath(p)
        ref, rinfo, _ = pso.get_solution_path(p, env.is_valid, env.bounds, 11 + i, env.path_cost("path_length"))
        assert {k: info[k] for k in COUNTERS} == {k: rinfo[k] for k in COUNTERS}, f"\ndevice {info}\nrestated {rinfo}"
        assert got.shape == ref.shape and np.abs(got - ref).max(initial=0.0) <= STATE_TOL
