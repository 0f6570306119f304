"""GPU parity (-m gpu) of the queries on the device roadmap (artp_roadmap_update_edges / _solve / _get_edge_costs) against
oracle/roadmap_query_oracle.py. The restatement starts from the device's own roadmap and edge weights, prices the query
edges with artp_motion_cost_states (the same head kernels: equality, not a tolerance) and takes isValid from the port
oracle. Compared: status, path vertex indices, REMOVED flags, searches run, every weight, the roadmap itself; VALID flags
may exceed the restatement's by edges the oracle's motion check passes too (a validation round checks further along the
path than the reference walks)."""
import numpy as np
import pytest

import roadmap_cases as rc
from art_planner_b200 import synth
from oracle import orc
from oracle import roadmap_oracle as ro
from oracle import roadmap_query_oracle as rqo
from query_parity import Env

pytestmark = pytest.mark.gpu


def query_states(env, n, seed):
    """Valid states near far-apart milestones of the roadmap."""
    st, kinds = env.rm.vertices()
    ms = st[kinds == ro.MILESTONE]
    k = (synth.hash_uniform(seed, 1, np.arange(4 * n)) * len(ms)).astype(int)
    cand = ms[k] + np.array([0.011, -0.017, 0, 0, 0, 0, 0])
    return cand[env.is_valid(cand)][:n]


@pytest.mark.parametrize("network", ["light", "full"])
def test_update_edges_equals_motion_cost_states(network):
    env = Env(rc.make_case("rough_fbm"), network, thr=0.5 if network == "light" else 0.375)
    env.rm.sampleGraph(env.smp, *rc.CAPS, max_draws=rc.MAX_DRAWS)
    cost0, flags0, live = env.rm.edgeCosts()
    assert not cost0.any() and not flags0.any() and live == len(cost0)      # never priced: 0.0, no flag
    env.rm.updateEdges()
    st, _ = env.rm.vertices()
    edges = env.rm.edges()
    ref_cost, feas, _ = env.obj.updateEdgesBatch(st[edges[:, 0]], st[edges[:, 1]])
    cost, flags, _ = env.rm.edgeCosts()
    assert np.array_equal(cost, ref_cost) and np.array_equal(flags, feas)
    assert np.isinf(cost).any() and feas.any()
    assert np.array_equal(env.rm.edgeCosts(first=len(cost) - 5)[0], cost[-5:])


@pytest.mark.parametrize("name", list(rc.CASES))
def test_solve_matches_restatement(name):
    """Queries one after another on one roadmap: both robot presets, the off-origin non-square map; from the second query
    on the first pair's vertices are plain milestones and their zero-weight chain edges are in play."""
    env = Env(rc.make_case(name))
    env.rm.sampleGraph(env.smp, *rc.CAPS, max_draws=rc.MAX_DRAWS, distribution=False)   # the sampler keeps its layers
    env.rm.updateEdges()
    qs = query_states(env, 12, seed=91)
    seen = set()
    for a, b in zip(qs[0::2], qs[1::2]):
        status, idx, info, _ = env.solve_both(a, b)
        seen.add(status)
        _, kinds = env.rm.vertices()
        assert set(np.flatnonzero(kinds & ro.QUERY)) == {info["start_vertex"], info["goal_vertex"]}
    # the -inf patches split the gentle map's roadmap: there, goals in another component; elsewhere, solutions
    assert (rqo.NOT_CONNECTED if name == "gentle_inf" else rqo.SOLVED) in seen
    # the roadmap keeps growing like the restatement's after queries (live-edge cap, density set)
    nv, ne = env.rm.counts()
    q = env.mirror()
    used = env.rm.sampleGraph(env.smp, nv + 100, ne + 1000, 300, max_draws=1 << 22, first_sample=1 << 23, distribution=False)
    r_used, _, _ = ro.sample_graph(q, env.o, env.c.m, env.c.layers, env.c.sp, env.c.rp.reach_z, rc.SEED, 1 << 23, nv + 100,
                                   ne + 1000, 300, 1 << 22)
    assert used == r_used and np.array_equal(env.rm.edges(), q.result()[2])


def test_every_route_infeasible():
    """A risk threshold below every edge's risk: connected, but not over edges of finite weight."""
    env = Env(rc.make_case("rough_fbm"), thr=1e-6)
    env.rm.sampleGraph(env.smp, 400, 2000, 0, max_draws=rc.MAX_DRAWS, distribution=False)
    env.rm.updateEdges()
    assert np.isinf(env.rm.edgeCosts()[0]).all()
    qs = query_states(env, 2, seed=92)
    status, _, info, _ = env.solve_both(qs[0], qs[1])
    assert status in (rqo.NO_FEASIBLE_PATH, rqo.NOT_CONNECTED)


def removal_scene():
    """A start and a goal on the gentle map with -inf patches whose straight connection has valid interior states and a
    motion that fails between two of them, and a third milestone that gives a detour (found offline with the port oracle)."""
    c = rc.make_case("gentle_inf")
    o = orc.Oracle(c.rp, "port")
    o.set_map(c.m)
    poses = synth.make_terrain_poses(c.m, 3000, seed=3)
    poses = poses[o.check_poses(poses).astype(bool)]
    return c, poses[1], poses[12], poses[2]


def test_failed_motion_removes_one_edge_and_searches_again():
    c, a, b, third = removal_scene()
    env = Env(c, thr=10.0)                       # every edge feasible: the route is decided by the motion checks
    # start and goal alone: the only route loses an edge
    status, _, info, ref = env.solve_both(a, b)
    assert status == rqo.NOT_CONNECTED and info["edges_removed"] == 1 and info["searches"] == 1
    assert np.count_nonzero(env.rm.edgeCosts()[1] & rqo.REMOVED) == 1
    # sampleGraph after a removal: the live-edge cap and the density's vertex set follow the restatement
    q = env.mirror()
    nv, ne = env.rm.counts()
    used = env.rm.sampleGraph(env.smp, nv + 200, ne + 1000, 50, max_draws=1 << 22)
    r_used, _, rec = ro.sample_graph(q, env.o, c.m, c.layers, c.sp, c.rp.reach_z, rc.SEED, 0, nv + 200, ne + 1000, 50, 1 << 22,
                                     c.dp, c.sample_filter, c.observed)
    assert used == r_used and len(rec) >= 1
    assert np.array_equal(env.rm.edges(), q.result()[2])
    # with a third milestone there is a detour: every removal is followed by another search
    env.rm.clear()
    env.rm.addValidMilestones(third[None])
    status, idx, info, ref = env.solve_both(a, b)
    assert status == rqo.SOLVED and info["searches"] == info["edges_removed"] + 1


def test_distances_equal_scipy_dijkstra():
    """The path cost to many goals equals scipy's Dijkstra on the same weights exactly (both round every sum the same way)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import dijkstra
    env = Env(rc.make_case("rough_fbm"), thr=0.6)
    env.rm.sampleGraph(env.smp, *rc.CAPS, max_draws=rc.MAX_DRAWS)
    env.rm.updateEdges()
    qs = query_states(env, 21, seed=93)
    solved = 0
    for g in qs[1:]:
        status, _, idx, cost, info = env.rm.solve(qs[0], g, env.space)
        if status != rqo.SOLVED:
            continue
        solved += 1
        w, flags, _ = env.rm.edgeCosts()
        e = env.rm.edges()
        keep = np.isfinite(w) & ((flags & rqo.REMOVED) == 0)
        nv = env.rm.counts()[0]
        g2 = coo_matrix((w[keep], (e[keep, 0], e[keep, 1])), shape=(nv, nv)).tocsr()   # explicit zeros are zero-weight edges
        d = dijkstra(g2, directed=False, indices=info["start_vertex"])
        assert d[info["goal_vertex"]] == cost
    assert solved >= 10


def test_error_codes_leave_the_roadmap_untouched():
    import art_planner_b200 as ap
    import ctypes as C
    env = Env(rc.make_case("rough_fbm"))
    capi, h = env.capi, env.chk.handle
    env.rm.sampleGraph(env.smp, 300, 2000, 0, max_draws=rc.MAX_DRAWS, distribution=False)
    env.rm.updateEdges()
    qs = query_states(env, 2, seed=94)
    before = (env.rm.counts(), env.rm.vertices()[1].copy(), env.rm.edgeCosts()[0].copy())

    def unchanged():
        return env.rm.counts() == before[0] and np.array_equal(env.rm.vertices()[1], before[1]) and \
            np.array_equal(env.rm.edgeCosts()[0], before[2])

    # an invalid start (in the air), a goal outside the bounds
    bad = qs[0].copy(); bad[2] += 3.0
    assert env.solve_both(bad, qs[1])[0] == rqo.INVALID_START and unchanged()
    far = qs[1].copy(); far[0] += 1000.0
    assert env.rm.solve(qs[0], far, env.space)[0] == rqo.INVALID_GOAL and unchanged()
    assert env.rm.solve(qs[0], bad, env.space)[0] == rqo.INVALID_GOAL and unchanged()
    # a path buffer too small: ARTP_E_LIMIT with the length reported
    n, cost = C.c_size_t(0), C.c_double(0)
    buf = np.empty((1, 7))
    rcode = h.lib.artp_roadmap_solve(h.h, qs[0].ctypes.data, qs[1].ctypes.data, C.byref(env.space), buf.ctypes.data, 1,
                                     C.byref(n), C.byref(cost), None)
    assert rcode == capi.ARTP_E_LIMIT and n.value > 1
    assert env.rm.solve(qs[0], qs[1], env.space)[0] == rqo.SOLVED
    # no weights, no roadmap
    c2 = ap.StateValidityChecker(env.c.rp, device=0)
    c2.setMap(env.c.m)
    c2.updateHeightField()
    lib = h.lib
    assert lib.artp_roadmap_update_edges(c2.handle.h) == capi.ARTP_E_INVALID
    assert lib.artp_roadmap_get_edge_costs(c2.handle.h, 0, None, None, None) == capi.ARTP_E_INVALID
    rm2 = ap.PRMRoadmap(c2, 100, 400)
    rm2.addValidMilestones(qs[:1])
    assert lib.artp_roadmap_update_edges(c2.handle.h) == capi.ARTP_E_NOWEIGHTS
    assert lib.artp_roadmap_solve(c2.handle.h, qs[0].ctypes.data, qs[1].ctypes.data, C.byref(env.space), None, 0, None, None,
                                  None) == capi.ARTP_E_NOWEIGHTS
    assert rm2.counts() == (1, 0)
    assert lib.artp_roadmap_get_edge_costs(h.h, 10 ** 7, None, None, None) == capi.ARTP_E_INVALID


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
    env = Env(c, thr=0.6)
    import art_planner_b200 as ap
    env.rm = ap.PRMRoadmap(env.chk, 20000, 60000)
    env.rm.sampleGraph(env.smp, 10000, 50000, 1000)
    env.rm.updateEdges()
    qs = query_states(env, 2, seed=95)
    status, idx, info, _ = env.solve_both(qs[0], qs[1])
    assert status in (rqo.SOLVED, rqo.NO_FEASIBLE_PATH, rqo.NOT_CONNECTED)
