"""The query restatement's search (oracle/roadmap_query_oracle.py: dijkstra, shortest_path, connected) against a formulation
it does not share, on graphs built to tie: scipy's Dijkstra in float64 for the distances, a breadth-first search over the
tight-edge subgraph for the levels, and the predecessor as a numpy minimum over the tight neighbours one level down. Then
the roadmaps of tests/search_cases.py: what the GPU search tests rely on, checked with the port oracle."""
import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components, dijkstra, shortest_path

import search_cases as sc
from oracle import orc
from oracle import roadmap_oracle as ro
from oracle import roadmap_query_oracle as rqo

INF = float("inf")
WEIGHTS = {
    "zero": lambda rng, n: np.zeros(n),
    "few": lambda rng, n: rng.choice([0.25, 0.5, 1.0], n),
    "mix": lambda rng, n: np.select([rng.random(n) < p for p in (0.25, 0.5, 0.85)],
                                    [np.zeros(n), np.full(n, 0.5), rng.random(n)], np.full(n, INF)),
}


def tie_graph(seed, kind):
    """A random graph of 2-4 components (vertex blocks), some of them joined only by +inf edges, with weights from `kind`.
    Parallel edges and removed edges included."""
    rng = np.random.default_rng(seed)
    blocks = np.cumsum(rng.integers(1, 25, rng.integers(2, 5)))
    V = int(blocks[-1])
    g = rqo.QueryRoadmap(V)
    g.V = V
    lo = 0
    for hi in blocks:
        n = hi - lo
        for _ in range(int(rng.integers(n - 1, 3 * n + 1))):
            if n > 1:
                g._edge(int(lo + rng.integers(n)), int(lo + rng.integers(n)))
        lo = hi
    g.cost = list(WEIGHTS[kind](rng, len(g.edges)))
    for b in range(len(blocks) - 1):                     # blocks joined by +inf edges (or not at all)
        if rng.random() < 0.5:
            g._edge(int(rng.integers(blocks[b])), int(blocks[b] + rng.integers(blocks[b + 1] - blocks[b])))
            g.cost[-1] = INF
    for e in rng.choice(len(g.edges), len(g.edges) // 10, replace=False):
        g.remove_edge(int(e))
    return g


def independent_search(g, start):
    """(distances, levels, pred, pred_e) without the restatement's code."""
    e = np.array(g.edges, np.int64).reshape(-1, 2)
    w = np.array(g.cost)
    live = np.array([g.live(i) for i in range(len(g.edges))], bool)
    fin = live & np.isfinite(w)
    # parallel edges: scipy would sum them; keep the least weight of each pair instead
    m = coo_matrix((w[fin], (e[fin, 0], e[fin, 1])), shape=(g.V, g.V))
    pairs = {}
    for a, b, x in zip(m.row, m.col, m.data):
        k = (min(a, b), max(a, b))
        pairs[k] = min(pairs.get(k, INF), x)
    r = np.array([k[0] for k in pairs], np.int64).reshape(-1)
    c = np.array([k[1] for k in pairs], np.int64).reshape(-1)
    d = dijkstra(coo_matrix((np.array(list(pairs.values())), (r, c)), shape=(g.V, g.V)).tocsr(), directed=False,
                 indices=start)
    # tight directed edges u -> v: d[u] + w == d[v]
    src = np.concatenate([e[fin, 0], e[fin, 1]])
    dst = np.concatenate([e[fin, 1], e[fin, 0]])
    ww = np.concatenate([w[fin], w[fin]])
    eid = np.concatenate([np.flatnonzero(fin), np.flatnonzero(fin)])
    tight = np.isfinite(d[src]) & (d[src] + ww == d[dst])
    t = coo_matrix((np.ones(int(tight.sum())), (src[tight], dst[tight])), shape=(g.V, g.V)).tocsr()
    lev = shortest_path(t, directed=True, unweighted=True, indices=start)
    pred = np.full(g.V, -1)
    pred_e = np.full(g.V, -1)
    for v in range(g.V):
        if not np.isfinite(lev[v]) or lev[v] == 0:
            continue
        cand = tight & (dst == v) & (lev[src] == lev[v] - 1)
        k = np.lexsort((eid[cand], src[cand]))[0]
        pred[v], pred_e[v] = src[cand][k], eid[cand][k]
    comp = connected_components(coo_matrix((np.ones(int(live.sum())), (e[live, 0], e[live, 1])), shape=(g.V, g.V)),
                                directed=False)[1]
    return d, lev, pred, pred_e, comp


@pytest.mark.parametrize("kind", list(WEIGHTS))
@pytest.mark.parametrize("seed", range(12))
def test_search_equals_independent_formulation(kind, seed):
    g = tie_graph(seed, kind)
    d_ref, lev, pred, pred_e, comp = independent_search(g, 0)
    d = np.array(rqo.dijkstra(g, 0))
    assert np.array_equal(d, d_ref)
    reached = 0
    for goal in range(g.V):
        assert rqo.connected(g, 0, goal) == (comp[goal] == comp[0])
        if not np.isfinite(d[goal]):
            continue
        verts, edges = rqo.shortest_path(g, d.tolist(), 0, goal)
        assert len(verts) == lev[goal] + 1
        v, walk, walk_e = goal, [goal], []
        while v != 0:
            walk_e.append(int(pred_e[v]))
            v = int(pred[v])
            walk.append(v)
        assert verts == walk and edges == walk_e
        reached += 1
    assert reached >= 1


def test_tie_graphs_cover_the_regimes():
    """The generator's graphs hold what the test above is for: vertices with several tight predecessors one level down,
    goals reachable only over +inf edges (NO_FEASIBLE_PATH), goals in another component (NOT_CONNECTED)."""
    multi = infeasible = apart = 0
    for kind in WEIGHTS:
        for seed in range(12):
            g = tie_graph(seed, kind)
            d, lev, pred, _, comp = independent_search(g, 0)
            e = np.array(g.edges).reshape(-1, 2)
            w = np.array(g.cost)
            for v in range(g.V):
                if np.isfinite(lev[v]) and lev[v] > 0:
                    ups = {int(u) for (a, b), x, i in zip(e, w, range(len(w))) if g.live(i) and np.isfinite(x)
                           for u, t in ((a, b), (b, a)) if t == v and lev[u] == lev[v] - 1 and d[u] + x == d[v]}
                    multi += len(ups) >= 2
                infeasible += comp[v] == comp[0] and not np.isfinite(d[v])
                apart += comp[v] != comp[0]
    assert multi >= 30 and infeasible >= 10 and apart >= 10, (multi, infeasible, apart)


# ---- the roadmaps of the GPU tests -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def oracle():
    return orc.Oracle(sc.RP, "port")


def test_lattice_poses_valid_and_every_connection_direct(oracle):
    c = sc.flat_case()
    oracle.set_map(c.m)
    n = sc.SEARCH_VERTEX_LIMIT - 2
    st, perm = sc.lattice_states(n)
    a, b = sc.lattice_query(n // sc.LATTICE_SIDE)
    allst = np.concatenate([st, [a, b]])
    assert oracle.check_poses(allst).all()
    assert len(np.unique(perm)) == n
    # the whole lattice and the query inside a square whose diagonal is below the 0.5 m lateral step
    assert np.hypot(np.ptp(allst[:, 0]), np.ptp(allst[:, 1])) < ro.MAX_LATERAL
    # and so the restatement adds exactly one vertex and min(k*, V) edges per milestone (a prefix of the shuffled lattice)
    rm = ro.Roadmap(2048)
    valid = ro.validity(oracle)
    for s in st[:1200]:
        rm.add_milestone(s, valid)
    assert rm.V == 1200 and rm.E == sc.edges_added(0, 1200)


def test_corridor_poses(oracle):
    c = sc.corridor_case()
    oracle.set_map(c.m)
    p, st, a, b = sc.corridor_states(sc.CORRIDOR_N)
    assert oracle.check_poses(np.concatenate([st, [a, b]])).all()
    assert not oracle.check_poses(sc.wall_states()).any()           # the torso collides with every wall ridge
    # the second map's ridge blocks the corridor in the middle of its lane only
    oracle.set_map(sc.corridor_case(sc.OBSTACLE_LANE).m)
    bad = ~oracle.check_poses(st).astype(bool)
    assert bad.any()
    x, y = sc.centreline(p[bad])
    assert np.allclose(y, sc.lane_y(sc.OBSTACLE_LANE)) and np.abs(x).max() < 1.0


def test_corridor_connections_stay_direct(oracle):
    """The first milestones of the corridor's insertion order: no connection needs an interpolated state."""
    oracle.set_map(sc.corridor_case().m)
    _, st, _, _ = sc.corridor_states(sc.CORRIDOR_N)
    rm = ro.Roadmap(4096)
    valid = ro.validity(oracle)
    for s in st[:1500]:
        rm.add_milestone(s, valid)
    assert rm.V == 1500 and not (rm.kinds[:rm.V] & ro.INTERPOLATED).any()
