"""roadmap_search_kernel (artp_roadmap_query.cuh) where it is hard to get right, against the query restatement
(tests/query_parity.py, oracle/roadmap_query_oracle.py): the on-chip vertex capacity (77 440, all eight slices full) and one
past it, roadmaps so small that whole CTAs hold no vertex, corridor paths of over a thousand edges and thousands of sweeps, paths whose
unknown edges take several validation rounds, edges removed deep inside a long path, and exact ties of learned weights on
a lattice. Each query's status, path, cost, REMOVED flags and searches equal the restatement's."""
import ctypes as C
import time

import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import dijkstra, shortest_path

import search_cases as sc
from oracle import roadmap_oracle as ro
from oracle import roadmap_query_oracle as rqo
from query_parity import Env

pytestmark = pytest.mark.gpu
ALL_FEASIBLE = 10.0      # a risk threshold above every edge's risk: every weight finite
N_QUERIES = 4            # queries on the full-capacity lattice; the last one brings V to the capacity


def report(**kw):
    print(" ".join(f"{k}={v}" for k, v in kw.items()))


def scipy_distance(env, start, goal):
    w, flags, _ = env.rm.edgeCosts()
    e = env.rm.edges()
    keep = np.isfinite(w) & ((flags & rqo.REMOVED) == 0)
    nv = env.rm.counts()[0]
    g = coo_matrix((w[keep], (e[keep, 0], e[keep, 1])), shape=(nv, nv)).tocsr()   # explicit zeros are zero-weight edges
    return dijkstra(g, directed=False, indices=start)[goal]


def tie_vertices(env, start):
    """Vertices with two or more distinct tight neighbours one level down from `start` (the tie rule decides between
    them)."""
    w, flags, _ = env.rm.edgeCosts()
    e = env.rm.edges().astype(np.int64)
    nv = env.rm.counts()[0]
    keep = np.isfinite(w) & ((flags & rqo.REMOVED) == 0)
    g = coo_matrix((w[keep], (e[keep, 0], e[keep, 1])), shape=(nv, nv)).tocsr()
    d = dijkstra(g, directed=False, indices=start)
    src = np.concatenate([e[keep, 0], e[keep, 1]])
    dst = np.concatenate([e[keep, 1], e[keep, 0]])
    ww = np.concatenate([w[keep], w[keep]])
    tight = np.isfinite(d[src]) & (d[src] + ww == d[dst])
    t = coo_matrix((np.ones(int(tight.sum())), (src[tight], dst[tight])), shape=(nv, nv)).tocsr()
    lev = shortest_path(t, directed=True, unweighted=True, indices=start)
    down = tight & (lev[src] == lev[dst] - 1)
    pairs = np.unique(np.stack([dst[down], src[down]], 1), axis=0)
    return np.flatnonzero(np.bincount(pairs[:, 0], minlength=nv) >= 2)


# ---- capacity and slice layout -----------------------------------------------------------------------------------------
def test_lattice_edges_equal_restatement():
    """k nearest with exact distance ties everywhere, milestones in shuffled order: the edge list of the device equals
    roadmap_oracle's (ties to the lower vertex index)."""
    env = Env(sc.flat_case(), thr=ALL_FEASIBLE, vertex_capacity=4096, edge_capacity=sc.edges_added(0, 3000) + 1)
    st, _ = sc.lattice_states(3000, seed=1)
    env.rm.addValidMilestones(st)
    rm = ro.Roadmap(4096)
    for s in st:
        rm.add_milestone(s, env.is_valid)
    dst, dk = env.rm.vertices()
    rst, rk, redges = rm.result()
    assert env.rm.counts() == (3000, sc.edges_added(0, 3000))
    assert np.array_equal(dst, rst) and np.array_equal(env.rm.edges(), redges)


@pytest.fixture(scope="module")
def full():
    """A lattice of 77 440 - 2 N_QUERIES milestones in a store of exactly 77 440 vertices."""
    n = sc.SEARCH_VERTEX_LIMIT - 2 * N_QUERIES
    ne = sc.edges_added(0, n + 2 * N_QUERIES)
    env = Env(sc.flat_case(), thr=ALL_FEASIBLE, vertex_capacity=sc.SEARCH_VERTEX_LIMIT, edge_capacity=ne)
    st, _ = sc.lattice_states(n)
    t = time.perf_counter()
    env.rm.addValidMilestones(st)
    report(lattice_milestones=n, insert_s=round(time.perf_counter() - t, 1), counts=env.rm.counts())
    assert env.rm.counts() == (n, sc.edges_added(0, n))
    return env, n


def test_full_capacity_queries(full):
    """Queries until V is the capacity: the first on weights never priced (all 0.0: every distance ties), the others after
    updateEdges. The third starts where the second did and ends exactly on a vertex that had several tight predecessors
    from there, so the tie rule decides its path on learned weights. The last one's start and goal are the last two
    vertices of CTA 7's slice."""
    env, n = full
    rows = n // sc.LATTICE_SIDE
    a1, b1 = sc.lattice_query(rows, (2, 3), (rows - 3, sc.LATTICE_SIDE - 5))
    queries = [sc.lattice_query(rows), (a1, b1), None,
               sc.lattice_query(rows, (rows // 2, 0), (rows // 2 + 1, sc.LATTICE_SIDE - 2))]
    assert len(queries) == N_QUERIES
    for q, ab in enumerate(queries):
        if q == 1:
            env.rm.updateEdges()
        if ab is None:
            ties = tie_vertices(env, info["start_vertex"])
            ties = ties[ties < n]                        # lattice milestones
            assert len(ties) >= 10
            ab = a1, env.rm.vertices()[0][ties[-1]]
        t = time.perf_counter()
        status, idx, info, ref = env.solve_both(*ab)
        nv, ne = env.rm.counts()
        assert status == rqo.SOLVED
        assert ref["cost"] == scipy_distance(env, info["start_vertex"], info["goal_vertex"])
        on_path = len(np.intersect1d(idx[1:], tie_vertices(env, info["start_vertex"]))) if q else 0
        report(query=q, V=nv, E=ne, hops=len(idx) - 1, sweeps=info["sweeps"], searches=info["searches"],
               path_tie_vertices=on_path, s=round(time.perf_counter() - t, 1))
        if q == 2:
            assert on_path >= 1
    assert nv == sc.SEARCH_VERTEX_LIMIT
    assert (info["start_vertex"], info["goal_vertex"]) == (nv - 2, nv - 1)


def test_lattice_weights_tie(full):
    """Translated copies of an edge weigh the same bit for bit: many vertices have several tight neighbours one level down,
    and the tie rule picks the path."""
    env, _ = full
    env.rm.updateEdges()                                 # prices every edge (again, after the queries)
    w = env.rm.edgeCosts()[0]
    assert np.isfinite(w).all() and w.any()              # learned weights, not the 0.0 of an edge never priced
    fan = len(tie_vertices(env, env.rm.counts()[0] - 2))
    report(distinct_weights=len(np.unique(w)), edges=len(w), tight_fan_in=fan)
    assert len(np.unique(w)) < len(w) // 100 and fan >= 100


def test_capacity_above_the_limit_is_refused():
    """A store of 77 441 vertices: artp_roadmap_solve returns ARTP_E_LIMIT and the roadmap does not change."""
    from art_planner_b200 import capi
    env = Env(sc.flat_case(), thr=ALL_FEASIBLE, vertex_capacity=sc.SEARCH_VERTEX_LIMIT + 1, edge_capacity=4000)
    st, _ = sc.lattice_states(60)
    env.rm.addValidMilestones(st)
    env.rm.updateEdges()
    before = (env.rm.counts(), env.rm.vertices()[1].copy(), env.rm.edgeCosts()[0].copy(), env.rm.edgeCosts()[1].copy())
    a, b = sc.lattice_query(1, (0, 1), (0, 40))
    h = env.chk.handle
    n, cost = C.c_size_t(0), C.c_double(0)
    buf = np.empty((64, 7))
    rcode = h.lib.artp_roadmap_solve(h.h, a.ctypes.data, b.ctypes.data, C.byref(env.space), buf.ctypes.data, 64, C.byref(n),
                                     C.byref(cost), None)
    assert rcode == capi.ARTP_E_LIMIT
    assert env.rm.counts() == before[0] and np.array_equal(env.rm.vertices()[1], before[1])
    assert np.array_equal(env.rm.edgeCosts()[0], before[2]) and np.array_equal(env.rm.edgeCosts()[1], before[3])


def test_small_roadmaps_every_slice_layout():
    """0 .. 15 milestones plus the query: V = 2 .. 17, so slices of 1 and 2 vertices, CTAs without vertices, and start and
    goal in one CTA or in two."""
    env = Env(sc.flat_case(), thr=ALL_FEASIBLE, vertex_capacity=64, edge_capacity=512)
    for m in range(16):
        env.rm.clear()
        st, _ = sc.lattice_states(m, seed=m)
        if m:
            env.rm.addValidMilestones(st)
        if m % 2:
            env.rm.updateEdges()
        a, b = sc.lattice_query(1, (0, 0), (0, 3 + m))
        status, idx, info, _ = env.solve_both(a, b)
        assert status == rqo.SOLVED and env.rm.counts()[0] == m + 2
        assert (info["start_vertex"], info["goal_vertex"]) == (m, m + 1)


# ---- corridors ---------------------------------------------------------------------------------------------------------
def query_round_cap(env, states):
    """The states one validation round may hold, as artp_roadmap_solve sizes it: min(interior-state buffer, 2048), the
    buffer being k*(vertex capacity) connections of floor(box diagonal / 0.5 m) + 1 states over the (x, y) box of every
    milestone and query end (restated from artp_roadmap.cu; the device does not report it)."""
    diag = np.hypot(np.ptp(states[:, 0]), np.ptp(states[:, 1]))
    return min(max(ro.k_star(env.rm.vertex_capacity), 1) * (int(np.floor(diag / ro.MAX_LATERAL)) + 1), 2048)


def validation_rounds(env, idx, qcap):
    """The rounds query_gather_kernel packs the path's unknown edges into, from the goal's side, and their states
    (restated: the device counts neither)."""
    st = env.rm.vertices()[0]
    nd = [rqo.segment_count(env.bounds, st[idx[i]], st[idx[i + 1]]) for i in range(len(idx) - 1)][::-1]
    rounds, total, n = 1, 0, 0
    for x in nd:
        if n == 2048 or total + x > qcap:
            rounds, total, n = rounds + 1, 0, 0
        total, n = total + x, n + 1
    return rounds, int(sum(nd))


def corridor_path_checks(env, idx, info):
    st = env.rm.vertices()[0][idx]
    step = np.hypot(*np.diff(st[:, :2], axis=0).T)
    assert abs(step.sum() - sc.corridor_length()) < 0.01 * sc.corridor_length()   # the path follows the corridor
    assert env.is_valid(st).all()
    assert info["sweeps"] >= len(idx) - 1


def test_corridor_at_capacity():
    """77 436 centreline milestones and two queries between the corridor's ends: V reaches 77 440. First on weights never
    priced: every weight 0.0, every distance ties, the path is the fewest-edges, lowest-index one and none of its edges is
    VALID, so its validation takes several rounds (query_gather_kernel's `more`). Then after updateEdges."""
    n = sc.CORRIDOR_N
    env = Env(sc.corridor_case(), thr=ALL_FEASIBLE, vertex_capacity=sc.SEARCH_VERTEX_LIMIT,
              edge_capacity=sc.edges_added(0, sc.SEARCH_VERTEX_LIMIT))
    p, st, a, b = sc.corridor_states(n)
    t = time.perf_counter()
    env.rm.addValidMilestones(st)
    report(corridor_milestones=n, insert_s=round(time.perf_counter() - t, 1), counts=env.rm.counts())
    assert env.rm.counts()[0] == n                       # no interpolated vertex
    qcap = query_round_cap(env, np.concatenate([st, [a, b]]))
    assert not env.rm.edgeCosts()[0].any()
    status, idx, info, ref = env.solve_both(a, b, path_capacity=n + 4)
    assert status == rqo.SOLVED
    corridor_path_checks(env, idx, info)
    rounds, states = validation_rounds(env, idx, qcap)
    report(never_priced_hops=len(idx) - 1, sweeps=info["sweeps"], states=states, round_cap=qcap, rounds=rounds,
           checked=info["edges_checked"])
    assert states > qcap and rounds >= 2
    env.rm.updateEdges()
    status, idx, info, ref = env.solve_both(a, b, path_capacity=n + 4)
    report(priced_hops=len(idx) - 1, sweeps=info["sweeps"], cost=ref["cost"], V=env.rm.counts()[0])
    assert status == rqo.SOLVED and env.rm.counts()[0] == sc.SEARCH_VERTEX_LIMIT
    corridor_path_checks(env, idx, info)
    assert ref["cost"] == scipy_distance(env, info["start_vertex"], info["goal_vertex"])


def test_removal_deep_in_a_corridor_path():
    """A sparse corridor (chains of interpolated vertices, dead ends across the walls) built on the open map and never
    priced; then a second map with a ridge across the middle lane. Every path runs through the ridge, so each search's
    first invalid motion from the goal's side lies mid-corridor: edges are removed one search at a time until start and
    goal fall apart (NOT_CONNECTED), as in the restatement."""
    env = Env(sc.corridor_case(), thr=ALL_FEASIBLE, vertex_capacity=8192, edge_capacity=32768)
    p, st, a, b = sc.corridor_states(sc.REMOVAL_N)
    env.rm.addValidMilestones(st)
    kinds = env.rm.vertices()[1]
    assert (kinds & ro.INTERPOLATED).any()
    blocked = sc.corridor_case(sc.OBSTACLE_LANE)
    env.chk.setMap(blocked.m)
    env.chk.updateHeightField()
    env.obj.updateFeatures()
    env.o.set_map(blocked.m)
    status, idx, info, ref = env.solve_both(a, b)
    report(removal_V=env.rm.counts()[0], E=env.rm.counts()[1], searches=info["searches"], removed=info["edges_removed"],
           sweeps=info["sweeps"])
    assert status == rqo.NOT_CONNECTED
    assert info["searches"] == info["edges_removed"] >= 10
    vs = env.rm.vertices()[0]
    ends = vs[env.rm.edges()[ref["removed"]].reshape(-1)]
    # edges are removed at the ridge, mid-corridor (and where a never-checked edge cuts a U-turn's corner)
    at_ridge = (np.abs(ends[:, 1] - sc.lane_y(sc.OBSTACLE_LANE)) <= sc.HALF_WIDTH) & (np.abs(ends[:, 0]) < 1.5)
    report(removed_at_ridge=int(at_ridge.reshape(-1, 2).any(1).sum()))
    assert at_ridge.reshape(-1, 2).any(1).sum() >= 10
