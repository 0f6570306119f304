"""GPU (-m gpu): artp_planner_set_map + artp_plan against the same replan through the chained public calls
(tests/planner_cases.py), bit for bit: the SE(3) bounds, the roadmap (states, kinds, edges, weights, flags), the repaired
endpoints, the returned path, every info counter and both costs; every status, repeated plans, the error paths, the host
synchronisations and copies, and the Python mirror."""
import ctypes as C

import numpy as np
import pytest

import planner_cases as pc
import roadmap_cases as rc
from art_planner_b200 import capi, costnet, synth
from oracle import planner_oracle as po

pytestmark = pytest.mark.gpu


def make_pair(rp, network="light", thr=0.6, weights=True):
    import art_planner_b200 as ap
    from art_planner_b200.checker import _Handle
    out = []
    for _ in range(2):
        chk = ap.StateValidityChecker(rp, handle=_Handle(rp, 0, risk_threshold=thr))
        if weights:
            ap.MotionCostObjective(chk).setWeights(costnet.make_state_dict(seed=5, network=network))
        out.append(chk)
    return out


def roadmap_dump(h):
    nv, ne = C.c_size_t(0), C.c_size_t(0)
    h.check(h.lib.artp_roadmap_get(h.h, 0, None, None, 0, None, C.byref(nv), C.byref(ne)))
    st, kinds = np.empty((nv.value, 7)), np.empty(nv.value, np.uint8)
    edges = np.empty((ne.value, 2), np.uint32)
    cost, flags = np.empty(ne.value), np.empty(ne.value, np.uint8)
    h.check(h.lib.artp_roadmap_get(h.h, 0, st.ctypes.data, kinds.ctypes.data, 0, edges.ctypes.data, None, None))
    h.check(h.lib.artp_roadmap_get_edge_costs(h.h, 0, cost.ctypes.data, flags.ctypes.data, None))
    return st, kinds, edges, cost, flags


def same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


class Pair:
    def __init__(self, rp, pp, **kw):
        import art_planner_b200 as ap
        c1, c2 = make_pair(rp, **kw)
        self.one = ap.Planner(c1, pp)
        self.chain = pc.Chained(c2, pp)
        self.pp = pp

    def set_map(self, layers, m):
        mi = self.one.setMap(*layers, m.res, m.cx, m.cy)
        self.chain.setMap(*layers, m.res, m.cx, m.cy)
        a, b = self.one.space(), self.chain.space
        assert list(a.low) == list(b.low) and list(a.high) == list(b.high)
        return mi

    def plan(self, start, goal):
        status = self.one.plan(start, goal)
        info = self.one.info()
        s2, path2, rec = self.chain.plan(start, goal)
        assert status == s2 == info["status"]
        for k in ("sampled", "draws_used", "first_sample", "start_draw", "goal_draw", "goal_clipped", "goal_inside",
                  "start_index", "goal_index", "n_vertices", "n_edges", "path_cost"):
            assert info[k] == rec[k], (k, info[k], rec[k])
        for k in ("goal_clipped_state", "goal_projected", "start_repaired", "goal_repaired"):
            assert same(info[k], rec[k]), k
        for k, v in rec["solve"].items():
            assert info["solve"][k] == v, ("solve", k)
        if "simplify" in rec:
            assert info["simplify_seed"] == rec["simplify_seed"]
            for k, v in rec["simplify"].items():
                assert same(info["simplify"][k], v), ("simplify", k)
        path = self.one.getSolutionPath() if status == po.SOLVED else np.zeros((0, 7))
        assert same(path, path2)
        for x, y in zip(roadmap_dump(self.one._c.handle), roadmap_dump(self.chain.h)):
            assert same(x, y)
        return status, info


def far_queries(m, n, seed, chk):
    """n (start, goal) pairs of valid states 0.4 map lengths apart (planner_cases.queries), at most 4 m."""
    return pc.queries(chk, n, seed, min(4.0, 0.4 * min(m.length)))


@pytest.mark.parametrize("name", list(rc.CASES))
@pytest.mark.parametrize("network", ["light", "full"])
def test_one_call_equals_chained_calls(name, network):
    c = rc.make_case(name)
    pp = pc.small_params(seed=77)
    pair = Pair(c.rp, pp, network=network)
    layers = pc.raw_layers(c.m)
    pair.set_map(layers, c.m)
    statuses = [pair.plan(s, g)[0] for s, g in far_queries(c.m, 3, seed=5, chk=pair.chain.chk)]
    assert set(statuses) <= {po.SOLVED, po.NOT_SOLVED, po.INVALID_START, po.INVALID_GOAL}


def test_missing_traversability_and_off_map_goal():
    c = rc.make_case("gentle_inf")
    pair = Pair(c.rp, pc.small_params(seed=3))
    pair.set_map(pc.raw_layers(c.m, traversability=False), c.m)
    lx, ly = c.m.length
    s, _ = far_queries(c.m, 1, seed=9, chk=pair.chain.chk)[0]
    # outside the bounds: clipped to the bound, which is off the map: not projected
    status, info = pair.plan(s, np.array([c.m.cx + 3 * lx, c.m.cy, 5.0, 0, 0, 0, 2.0]))
    assert info["goal_clipped"] == 1 and info["goal_inside"] == 0
    # inside the bounds, off the map: neither clipped nor projected
    status, info = pair.plan(s, np.array([c.m.cx + 0.8 * lx, c.m.cy, 0.3, 0, 0, 0, 1.0]))
    assert info["goal_clipped"] == 0 and info["goal_inside"] == 0


def test_repeated_plans_and_the_generation_rule():
    c = rc.make_case("rough_fbm")
    pp = pc.small_params(seed=11)
    pair = Pair(c.rp, pp)
    layers = pc.raw_layers(c.m)
    pair.set_map(layers, c.m)
    q = far_queries(c.m, 3, seed=21, chk=pair.chain.chk)
    _, i1 = pair.plan(*q[0])
    assert i1["sampled"] == 1 and i1["draws_used"] > 0
    _, i2 = pair.plan(*q[1])                      # same map: no resampling, no draws
    assert i2["sampled"] == 0 and i2["draws_used"] == 0 and i2["first_sample"] == i1["first_sample"] + i1["draws_used"]
    assert i2["n_vertices"] - i1["n_vertices"] <= 2 * 64
    pp.clear_roadmap = 1                          # same map, cleared: only start and goal (the reference's quirk)
    _, i3 = pair.plan(*q[2])
    assert i3["sampled"] == 0 and i3["n_vertices"] <= 2 + 2 * 64
    pair.set_map(layers, c.m)                     # a new map rebuilds it
    _, i4 = pair.plan(*q[2])
    assert i4["sampled"] == 1 and i4["n_vertices"] > 100


def test_every_status():
    import art_planner_b200 as ap
    c = rc.make_case("gentle_inf")
    pp = pc.small_params(seed=5, n_iter=0)
    pair = Pair(c.rp, pp)
    # NO_MAP
    assert pair.one.plan(np.array([0, 0, 0, 0, 0, 0, 1.0]), np.array([0, 0, 0, 0, 0, 0, 1.0])) == po.NO_MAP
    pair.set_map(pc.raw_layers(c.m), c.m)
    s, g = far_queries(c.m, 1, seed=31, chk=pair.chain.chk)[0]
    # a cell inside an untraversable (-inf) blob of the masked layer, on the ground with the terrain's attitude
    bad = np.argwhere(~np.isfinite(c.m.elevation_masked))
    x, y = c.m.cell_xy()
    wall = pair.chain.chk.poseFrom2D(np.array([[x[bad[0][0]], y[bad[0][1]], 0, 0, 0, 0, 1.0]]))[0][0]
    assert not pair.chain.chk.isValid(wall)
    # INVALID_START: a start in a wall with no search
    status, info = pair.plan(wall, g)
    assert status == po.INVALID_START and info["start_index"] == -1
    # INVALID_GOAL: a valid start, a goal whose projection lands in the wall, no search
    status, info = pair.plan(s, np.array([wall[0], wall[1], 0, 0, 0, 0, 1.0]))
    assert status == po.INVALID_GOAL and info["goal_index"] == -1
    # NOT_SOLVED, no feasible path: every edge infeasible
    pair2 = Pair(c.rp, pc.small_params(seed=5, n_iter=200), thr=-1.0)
    pair2.set_map(pc.raw_layers(c.m), c.m)
    sts = [pair2.plan(a, b) for a, b in far_queries(c.m, 2, seed=33, chk=pair2.chain.chk)]
    assert any(st == po.NOT_SOLVED and i["solve"]["status"] == po.SOLVE_NO_FEASIBLE_PATH for st, i in sts)
    # NOT_SOLVED, disconnected: a roadmap of three milestones between far-apart ends
    pair4 = Pair(c.rp, pc.small_params(seed=5, n_iter=200, max_n_vertices=3))
    pair4.set_map(pc.raw_layers(c.m), c.m)
    sts = [pair4.plan(a, b) for a, b in pc.queries(pair4.chain.chk, 4, 37, 0.8 * min(c.m.length))]
    assert any(st == po.NOT_SOLVED and i["solve"]["status"] == po.SOLVE_NOT_CONNECTED for st, i in sts)
    # SOLVED
    pair3 = Pair(c.rp, pc.small_params(seed=5))
    pair3.set_map(pc.raw_layers(c.m), c.m)
    assert po.SOLVED in [pair3.plan(a, b)[0] for a, b in far_queries(c.m, 4, seed=35, chk=pair3.chain.chk)]


def test_errors_leave_the_handle_usable():
    import art_planner_b200 as ap
    c = rc.make_case("gentle_inf")
    pp = pc.small_params(seed=2)
    (chk,) = make_pair(c.rp, weights=False)[:1]
    pl = ap.Planner(chk, pp)
    layers = pc.raw_layers(c.m)
    pl.setMap(*layers, c.m.res, c.m.cx, c.m.cy)
    s, g = far_queries(c.m, 1, seed=41, chk=chk)[0]
    with pytest.raises(capi.ArtpError) as e:
        pl.plan(s, g)
    assert e.value.code == capi.ARTP_E_NOWEIGHTS
    ap.MotionCostObjective(chk).setWeights(costnet.make_state_dict(seed=5))
    pl.setMap(*layers, c.m.res, c.m.cx, c.m.cy)
    with pytest.raises(capi.ArtpError) as e:       # no finite cell
        pl.setMap(np.full_like(layers[0], np.nan), *layers[1:], c.m.res, c.m.cx, c.m.cy)
    assert e.value.code == capi.ARTP_E_INVALID
    bad = s.copy(); bad[0] = np.nan
    with pytest.raises(capi.ArtpError) as e:
        pl.plan(bad, g)
    assert e.value.code == capi.ARTP_E_INVALID
    pp.start_radius = -1.0
    with pytest.raises(capi.ArtpError) as e:
        pl.plan(s, g)
    assert e.value.code == capi.ARTP_E_INVALID
    pp.start_radius = 0.2
    statuses = []
    for a, b in far_queries(c.m, 4, seed=43, chk=chk):
        statuses.append(pl.plan(a, b))
        if statuses[-1] == po.SOLVED:
            n = len(pl.getSolutionPath())
            if n > 1:
                with pytest.raises(capi.ArtpError) as e:
                    pl.plan(a, b, capacity=1)
                assert e.value.code == capi.ARTP_E_LIMIT
            break
    assert po.SOLVED in statuses
    assert pl.plan(*far_queries(c.m, 1, seed=45, chk=chk)[0]) in (po.SOLVED, po.NOT_SOLVED, po.INVALID_START, po.INVALID_GOAL)
    with pytest.raises(RuntimeError):
        pl._solved = False
        pl.getSolutionPath()


def test_host_syncs_and_copies():
    c = rc.make_case("offgrid_r1")
    pair = Pair(c.rp, pc.small_params(seed=8))
    m = c.m
    layers = pc.raw_layers(m)
    mi = pair.set_map(layers, m)
    # the map call: four layers up; back only the finite ranges (bounds, and the compact codes of the two uploaded layers)
    assert mi["bytes_h2d"] == 4 * 4 * m.rows * m.cols and mi["bytes_d2h"] <= 64, mi
    assert mi["host_syncs"] <= 8, mi
    for s, g in far_queries(m, 3, seed=51, chk=pair.chain.chk):
        status, info = pair.plan(s, g)
        sol = info["solve"]
        loops = (sol["searches"] * 64 + 64) // 4 + 4               # the solve loop reads its control block every 4 rounds
        simp = info["simplify"]["rounds"] // 8 + 8 if status == po.SOLVED else 0
        # sampleGraph's loop: two reads per round, a round adds a milestone or uses at least 4096 draws
        sample = 2 * (info["n_vertices"] + info["draws_used"] // 4096 + 2) if info["sampled"] else 0
        assert info["host_syncs"] <= sample + loops + simp + 8
        # no layer comes back: what the call copies to the host is control words, the info and the path
        nv = info["n_vertices"]
        assert info["bytes_d2h"] < 64 * 1024 + (nv * 8 if info["sampled"] else 0) + 7 * 8 * 4096
        if not info["sampled"]:
            assert info["bytes_d2h"] < 64 * 1024


def test_shipped_caps_config1():
    """The one-call replan equals the chained one at the shipped caps on the configs[1] map, gentle and rough."""
    for m in (synth.make_fbm_map(1000, 1000), synth.make_fbm_map(1000, 1000, seed=12, amp=1.2, wavelength=3.0, persistence=0.7)):
        import art_planner_b200 as ap
        pair = Pair(synth.PARAMS_YAML, ap.Planner.params(seed=1))
        pair.set_map(pc.raw_layers(m), m)
        for s, g in far_queries(m, 2, seed=61, chk=pair.chain.chk):
            pair.plan(s, g)


def test_one_call_equals_composed_restatement():
    """artp_plan against oracle/planner_oracle.Replan, the replan composed from the restatements of its stages with the
    port oracle's isValid, on a small map at small caps: status, streams, endpoints, the roadmap, weights, path, counters
    and costs. Like the stage tests, the restatement takes the learned cost and the simplifier's SE(3) arithmetic from
    the device."""
    import art_planner_b200 as ap
    import philox_ball_ref as pbr
    import test_path_simplify_gpu as tps
    from oracle import orc
    from oracle import sample_distribution_oracle as sdo
    c = rc.make_case("gentle_inf")
    pp = pc.small_params(seed=29, max_n_vertices=300, max_n_edges=1500, recompute_density_after_n_samples=100, n_iter=100)
    (chk,) = make_pair(c.rp)[:1]
    pl = ap.Planner(chk, pp)
    layers = pc.raw_layers(c.m)
    pl.setMap(*layers, c.m.res, c.m.cx, c.m.cy)
    obj = ap.MotionCostObjective(chk)
    dp = sdo.DistributionParams(True, (c.rp.torso_length + c.rp.torso_width) * 0.25, True, pp.max_prob_unknown_samples)
    ref = po.Replan(c.rp, pp, orc.Oracle(c.rp, "port"), lambda a, b: obj.updateEdgesBatch(a, b)[0],
                    lambda st: obj.pathCost(st, pp.max_query_edge_length), tps.DeviceOps(chk.handle),
                    lambda seed, first, n_iter, r: pbr.ball_offsets(seed, first, 1, n_iter, r), dp)
    ref.set_map(*layers, c.m.res, c.m.cx, c.m.cy)
    sp = pl.space()
    assert list(sp.low) == ref.low and list(sp.high) == ref.high
    reached = set()
    for k, (s, g) in enumerate(pc.queries(chk, 3, 53, 0.4 * min(c.m.length))):
        if k == 2:
            pp.clear_roadmap = 1                       # same map, cleared: start and goal only
        status = pl.plan(s, g)
        info = pl.info()
        rstatus, rpath, rec = ref.plan(s, g)
        assert status == rstatus
        reached.add(status)
        for key in ("sampled", "draws_used", "first_sample", "start_draw", "goal_draw", "goal_clipped", "goal_inside",
                    "start_index", "goal_index"):
            assert info[key] == rec[key], (key, info[key], rec[key])
        for key in ("goal_clipped_state", "goal_projected", "start_repaired", "goal_repaired"):
            assert np.abs(info[key] - rec[key]).max() <= tps.STATE_TOL, key
        sol = rec["solve"]
        assert info["solve"]["status"] == sol["status"] and info["solve"]["searches"] == sol["searches"]
        assert info["solve"]["edges_removed"] == len(sol["removed"])
        # the roadmap: kinds and edges exactly, states to the restatement's tolerance, weights of the live edges
        st, kinds, edges, cost, flags = roadmap_dump(chk.handle)
        rst, rkinds, redges = ref.rm.result()
        assert np.array_equal(kinds, rkinds) and np.array_equal(edges, redges)
        assert np.abs(st - rst).max(initial=0.0) <= tps.STATE_TOL
        rcost = np.array(ref.rm.cost)
        fin = np.isfinite(rcost)
        assert np.array_equal(np.isfinite(cost), fin)
        assert np.allclose(cost[fin], rcost[fin], rtol=1e-12, atol=0.0)
        assert np.array_equal(flags & 2, np.array(ref.rm.flag, np.uint8) & 2)
        if status == po.SOLVED:
            assert info["solve"]["start_vertex"] == sol["start"] and info["solve"]["goal_vertex"] == sol["goal"]
            assert np.isclose(info["path_cost"], rec["path_cost"], rtol=1e-12, atol=0.0)
            got = pl.getSolutionPath()
            assert got.shape == rpath.shape and np.abs(got - rpath).max() <= tps.STATE_TOL
            for key in tps.COUNTERS:
                assert info["simplify"][key] == rec["simplify"][key], key
    assert po.SOLVED in reached
