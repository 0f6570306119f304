"""The query restatement (oracle/roadmap_query_oracle.py: updateEdges, computeCostForVertexEdges, baseSolve,
constructSolution) on hand-built graphs of a few vertices, one rule at a time. The device (tests/test_roadmap_query_gpu.py)
is compared with this restatement, so each rule is pinned here without a GPU."""
import math

import numpy as np

from oracle import roadmap_oracle as ro
from oracle import roadmap_query_oracle as rqo

INF = math.inf


def graph(n, edges, cost=None, flag=None):
    """n vertices at x = 0, 1, 2, ... with the identity rotation; edges as (u, v) in insertion order."""
    g = rqo.QueryRoadmap(64)
    for i in range(n):
        g._vertex([float(i), 0, 0, 0, 0, 0, 1], ro.MILESTONE)
    for a, b in edges:
        g._edge(a, b)
    if cost is not None:
        g.cost = [float(c) for c in cost]
    if flag is not None:
        g.flag = list(flag)
    return g


def directed_cost(src, tgt):
    """A cost that tells the direction: 10 + x(source) - 0.1 x(target)."""
    return 10.0 + src[:, 0] - 0.1 * tgt[:, 0]


def all_valid(states):
    return np.ones(len(states), bool)


def solve_on(g, start, goal, check_motion):
    """baseSolve's loop on a graph that already holds its start and goal."""
    out = {"searches": 0, "checked": 0, "removed": []}
    if not rqo.connected(g, start, goal):
        return rqo.NOT_CONNECTED, None, out
    while True:
        try:
            sol = rqo.construct_solution(g, start, goal, check_motion, out)
        except rqo.NoPath:
            return rqo.NO_FEASIBLE_PATH, None, out
        if sol is not None:
            return rqo.SOLVED, sol, out
        if not rqo.connected(g, start, goal):
            return rqo.NOT_CONNECTED, None, out


def test_update_edges_prices_from_source_and_marks_feasible_valid():
    g = graph(3, [(0, 1), (2, 1)])
    rqo.update_edges(g, lambda s, t: np.where(s[:, 0] == 2, INF, directed_cost(s, t)))
    assert g.cost == [10.0 + 0 - 0.1, INF]
    assert g.flag == [rqo.VALID, 0]              # infeasible: +inf, validity untouched


def test_query_vertex_edges_are_priced_from_the_query_vertex():
    # vertex 2 is the query vertex: once as an edge's target, once as its source
    g = graph(4, [(0, 2), (2, 3), (0, 1)], cost=[7, 7, 7], flag=[1, 0, 1])
    rqo.cost_for_vertex_edges(g, 2, directed_cost)
    assert g.cost[0] == 10.0 + 2 - 0.0           # stored (0, 2), priced from 2 towards 0: the out_edges pass wins
    assert g.cost[1] == 10.0 + 2 - 0.3
    assert g.cost[2] == 7.0                      # not incident: untouched
    assert g.flag == [1, 0, 1]                   # validity untouched


def test_start_goal_edge_keeps_the_goal_direction_and_chain_edges_stay_zero():
    # an empty roadmap, start at x = 0, goal at x = 1.2: the goal connects through two interpolated vertices
    g = rqo.QueryRoadmap(64)
    a = np.array([0.0, 0, 0, 0, 0, 0, 1])
    b = np.array([1.2, 0, 0, 0, 0, 0, 1])
    r = rqo.base_solve(g, a, b, all_valid, directed_cost, lambda s1, s2: True)
    assert r["status"] == rqo.SOLVED and r["start"] == 0 and r["goal"] == 1
    assert g.edges == [(1, 2), (2, 3), (3, 0)] and r["path"] == [0, 3, 2, 1]
    x = g.states[:, 0]
    assert g.cost[0] == 10.0 + x[1] - 0.1 * x[2]     # at the goal: from the goal
    assert g.cost[1] == 0.0                          # between two interpolated vertices: never priced
    assert g.cost[2] == 10.0 + x[0] - 0.1 * x[3]     # at the start: from the start
    assert r["cost"] == (g.cost[2] + g.cost[1]) + g.cost[0] and r["checked"] == 3
    assert g.flag == [rqo.VALID] * 3
    # a direct edge joins start and goal: the goal is priced last
    g = rqo.QueryRoadmap(64)
    r = rqo.base_solve(g, a, np.array([0.3, 0, 0, 0, 0, 0, 1]), all_valid, directed_cost, lambda s1, s2: True)
    assert g.edges == [(1, 0)] and g.cost[0] == 10.0 + 0.3 - 0.0 and r["path"] == [0, 1]
    # the second query: the first pair stays as plain milestones
    r2 = rqo.base_solve(g, np.array([0.1, 0, 0, 0, 0, 0, 1]), np.array([0.2, 0, 0, 0, 0, 0, 1]), all_valid, directed_cost,
                        lambda s1, s2: True)
    assert list(g.kinds[:4]) == [ro.MILESTONE, ro.MILESTONE, ro.MILESTONE | ro.QUERY, ro.MILESTONE | ro.QUERY]
    assert r2["status"] == rqo.SOLVED and (r2["start"], r2["goal"]) == (2, 3)


def test_infinite_edges_never_relax():
    g = graph(3, [(0, 1), (1, 2), (0, 2)], cost=[1, 1, INF], flag=[1, 1, 1])
    assert rqo.dijkstra(g, 0) == [0.0, 1.0, 2.0]
    status, sol, _ = solve_on(g, 0, 2, lambda a, b: True)
    assert status == rqo.SOLVED and sol[0] == [0, 1, 2]


def test_not_connected_and_no_feasible_path():
    g = graph(4, [(0, 1), (2, 3)], cost=[1, 1], flag=[1, 1])
    assert solve_on(g, 0, 3, lambda a, b: True)[0] == rqo.NOT_CONNECTED
    g = graph(3, [(0, 1), (1, 2)], cost=[1, INF], flag=[1, 0])
    status, _, out = solve_on(g, 0, 2, lambda a, b: True)
    assert status == rqo.NO_FEASIBLE_PATH and out["searches"] == 1


def test_tie_rule_on_a_diamond_and_fewest_hops():
    # 0 -> {1, 2} -> 3 at equal cost: the lower predecessor index wins
    g = graph(4, [(0, 2), (0, 1), (2, 3), (1, 3)], cost=[1, 1, 1, 1], flag=[1] * 4)
    assert solve_on(g, 0, 3, lambda a, b: True)[1][0] == [0, 1, 3]
    # equal cost over two and over three edges: the fewest edges win, whatever the indices
    g = graph(5, [(0, 1), (1, 2), (2, 4), (0, 3), (3, 4)], cost=[1, 1, 1, 1.5, 1.5], flag=[1] * 5)
    assert solve_on(g, 0, 4, lambda a, b: True)[1][0] == [0, 3, 4]


def test_zero_cost_cycle_gives_no_predecessor_loop():
    # 1, 2, 3 form a cycle of zero-weight edges (a query's chain edges): all at distance 1
    g = graph(5, [(0, 1), (1, 2), (2, 3), (3, 1), (3, 4)], cost=[1, 0, 0, 0, 1], flag=[1] * 5)
    d = rqo.dijkstra(g, 0)
    assert d == [0.0, 1.0, 1.0, 1.0, 2.0]
    verts, edges = rqo.shortest_path(g, d, 0, 4)
    assert verts == [4, 3, 1, 0] and edges == [4, 3, 0]
    for goal in (1, 2, 3, 4):
        assert len(rqo.shortest_path(g, d, 0, goal)[0]) <= 4


def test_first_invalid_edge_from_the_goal_is_removed_and_the_search_runs_again():
    # path 0-1-2-3 with two unknown edges failing; the detour 0-4-3 costs more
    g = graph(5, [(0, 1), (1, 2), (2, 3), (0, 4), (4, 3)], cost=[1, 1, 1, 5, 5], flag=[0, 1, 0, 1, 1])
    checked = []

    def check(s1, s2):
        checked.append((s1[0], s2[0]))
        return False

    status, sol, out = solve_on(g, 0, 3, check)
    assert status == rqo.SOLVED and sol[0] == [0, 4, 3]
    assert out["removed"] == [2] and out["searches"] == 2      # the goal-side edge only; (0, 1) was never reached
    assert checked == [(2.0, 3.0)]                              # from the start-side vertex to the goal-side one
    assert g.flag == [0, 1, rqo.REMOVED, 1, 1] and g.E == 4
    assert not g.dens[2] or any(g.live(e) and 2 in g.edges[e] for e in range(5))
    # removing the only route: the loop ends on connectivity
    g = graph(3, [(0, 1), (1, 2)], cost=[1, 1], flag=[1, 0])
    status, _, out = solve_on(g, 0, 2, lambda a, b: False)
    assert status == rqo.NOT_CONNECTED and out["removed"] == [1] and out["searches"] == 1
    assert list(g.dens[:3]) == [True, True, False]              # vertex 2 lost its last edge


def test_invalid_start_and_goal_leave_the_roadmap_alone():
    g = graph(2, [(0, 1)], cost=[1], flag=[1])
    a = np.array([0.5, 0, 0, 0, 0, 0, 1])
    r = rqo.base_solve(g, a, a, lambda s: np.zeros(len(s), bool), directed_cost, lambda s1, s2: True)
    assert r["status"] == rqo.INVALID_START and g.V == 2
    r = rqo.base_solve(g, a, a + 5, all_valid, directed_cost, lambda s1, s2: True, in_bounds=lambda s: s[0] < 3)
    assert r["status"] == rqo.INVALID_GOAL and g.V == 2 and g.E == 1


def test_discrete_motion_visits_the_interior_states_then_s2():
    space = ([0, 0, 0], [30, 40, 0], 0.01)          # extent 50: segments of 0.5
    seen = []

    def is_valid(states):
        seen.extend(states[:, 0].tolist())
        return np.ones(len(states), bool)

    a = np.array([0.0, 0, 0, 0, 0, 0, 1])
    b = np.array([1.2, 0, 0, 0, 0, 0, 1])
    assert rqo.segment_count(space, a, b) == 3
    assert rqo.discrete_motion(is_valid, space)(a, b)
    assert np.allclose(seen, [0.4, 0.8, 1.2]) and seen[-1] == 1.2
