"""Restatement of PRMMotionCost's query side (TEST INFRASTRUCTURE ONLY), plain Python over roadmap_oracle.Roadmap:

  updateEdges                 art_planner/src/planners/prm_motion_cost.cpp:27-73
  computeCostForVertexEdges   :77-128
  baseSolve                   :440-532, after Planner::plan's clearQuery (planner.cpp:240)
  constructSolution           :536-673

The Boost graph and OMPL are not in the tree; restated from their documented behaviour (unpinned):
  boost::edges / in_edges / out_edges   insertion order; on an undirected graph both incident lists hold every incident
                                        edge, in_edges with the vertex as target, out_edges with it as source
  boost::astar_search                   with motionCostHeuristic == 0 (motion_cost_objective.cpp:99-103): Dijkstra; an edge
                                        of infinite weight never relaxes; ties are left to its heap -- here the optimal
                                        path with the fewest edges, the lowest predecessor index on ties
  DiscreteMotionValidator::checkMotion  interpolate(s1, s2, j / nd) for j = 1 .. nd - 1, then s2; nd = validSegmentCount

The per-edge cost function and the validity function are arguments, so the same code runs over the port oracle, the
compiled reference, or costs read back from the device.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import roadmap_oracle as ro

INF = float("inf")
VALID, REMOVED = 1, 2
SOLVED, NOT_CONNECTED, NO_FEASIBLE_PATH, INVALID_START, INVALID_GOAL = 1, 2, 3, 4, 5


class QueryRoadmap(ro.Roadmap):
    """g_ with its edge weights and validity: cost[e] (ob::Cost() = 0.0 until priced), flag[e] (VALID, REMOVED). The store is
    append-only like the device's: a removed edge keeps its index."""

    def __init__(self, capacity: int = 1 << 16):
        super().__init__(capacity)
        self.cost, self.flag = [], []
        self.n_removed = 0

    @property
    def E(self) -> int:                     # num_edges(g_)
        return len(self.edges) - self.n_removed

    def _edge(self, a: int, b: int) -> None:
        super()._edge(a, b)
        self.cost.append(0.0)
        self.flag.append(0)

    def live(self, e: int) -> bool:
        return not self.flag[e] & REMOVED

    def _live_edges(self):
        """(edge indices, [n, 2] endpoints) of the live edges in ascending edge index. The int64 copy of the edge list and
        the rows of csr() are cached under (id(edges), len(edges), n_removed), which assumes two things: an edge becomes
        REMOVED only through remove_edge, and `edges` is only appended to or replaced together with a fresh roadmap
        (a new list of the same length under a reused id would be missed). Code that breaks either calls
        invalidate()."""
        key = (id(self.edges), len(self.edges), self.n_removed)
        if getattr(self, "_live_key", None) != key:
            ea = getattr(self, "_ea", None)
            if ea is None or getattr(self, "_ea_of", None) != id(self.edges) or ea.shape[0] > len(self.edges):
                ea = np.zeros((0, 2), np.int64)
            if ea.shape[0] < len(self.edges):
                ea = np.concatenate([ea, np.asarray(self.edges[ea.shape[0]:], np.int64).reshape(-1, 2)])
            self._ea, self._ea_of = ea, id(self.edges)
            ids = np.flatnonzero((np.asarray(self.flag, np.uint8).reshape(-1) & REMOVED) == 0)
            self._live, self._live_key, self._csr = (ids, ea[ids]), key, None
        return self._live

    def invalidate(self) -> None:
        """Drops the cached edge array and rows (after changing `edges` or REMOVED flags other than by appending or
        remove_edge)."""
        self._live_key, self._ea = None, None

    def incident(self, v: int):
        """(edge index, other endpoint) of v's live edges in ascending edge index."""
        ids, ea = self._live_edges()
        at = (ea[:, 0] == v) | (ea[:, 1] == v)
        return [(int(e), int(b if a == v else a)) for e, (a, b) in zip(ids[at], ea[at])]

    def csr(self):
        """The live edges as rows per vertex, neighbours in ascending edge index: (offsets [V + 1], neighbour, edge index).
        An edge appears in both endpoints' rows (twice in one row for a loop)."""
        ids, ea = self._live_edges()
        if self._csr is None or self._csr[0].shape[0] != self.V + 1:
            row = np.concatenate([ea[:, 0], ea[:, 1]])
            nbr = np.concatenate([ea[:, 1], ea[:, 0]])
            eid = np.concatenate([ids, ids])
            order = np.lexsort((eid, row))
            self._csr = np.searchsorted(row[order], np.arange(self.V + 1)), nbr[order], eid[order]
        return self._csr

    def adjacency(self):
        off, nbr, eid = self.csr()
        return [list(zip(eid[off[v]:off[v + 1]].tolist(), nbr[off[v]:off[v + 1]].tolist())) for v in range(self.V)]

    def refresh_density(self) -> None:
        """LazyPRM::getPlannerData's vertices: startM_ / goalM_ and the endpoints of (live) edges."""
        self.dens[:] = False
        self.dens[self._live_edges()[1].reshape(-1)] = True
        self.dens[:self.V] |= (self.kinds[:self.V] & ro.QUERY) != 0

    def clear_query(self) -> None:
        self.kinds[:self.V] &= np.uint8(~ro.QUERY & 0xFF)
        self.refresh_density()

    def remove_edge(self, e: int) -> None:
        self.flag[e] |= REMOVED
        self.n_removed += 1
        self.refresh_density()


def update_edges(rm: QueryRoadmap, edge_cost) -> None:
    """updateEdges: every edge from its source u to its target v; feasible -> weight and VALIDITY_TRUE, else +inf.
    edge_cost(source states [n, 7], target states [n, 7]) -> weights [n], +inf where infeasible."""
    ids = [e for e in range(len(rm.edges)) if rm.live(e)]
    if not ids:
        return
    src = rm.states[[rm.edges[e][0] for e in ids]]
    tgt = rm.states[[rm.edges[e][1] for e in ids]]
    for e, c in zip(ids, edge_cost(src, tgt)):
        rm.cost[e] = float(c)
        if c < INF:
            rm.flag[e] |= VALID


def cost_for_vertex_edges(rm: QueryRoadmap, v: int, edge_cost) -> None:
    """computeCostForVertexEdges(v): the in_edges rows, then the out_edges rows, one cost call, then the weights written in
    that order -- so the out_edges pass, with v as the source, is the one that stays. Validity is not touched."""
    inc = rm.incident(v)
    if not inc:
        return
    rows = [(e, n, v) for e, n in inc]          # in_edges(v): source = the neighbour, target = v
    rows += [(e, v, n) for e, n in inc]         # out_edges(v): source = v, target = the neighbour
    cost = edge_cost(rm.states[[s for _, s, _ in rows]], rm.states[[t for _, _, t in rows]])
    for (e, _, _), c in zip(rows, cost):
        rm.cost[e] = float(c)


def _rows(off, vs):
    """The CSR positions of the rows of vertices vs, and the row vertex of each."""
    lo, n = off[vs], off[vs + 1] - off[vs]
    pos = np.repeat(lo - np.cumsum(n) + n, n) + np.arange(int(n.sum()))
    return pos, np.repeat(vs, n)


def connected(rm: QueryRoadmap, a: int, b: int) -> bool:
    """sameComponent: over live edges of any weight."""
    off, nbr, _ = rm.csr()
    seen = np.zeros(rm.V, bool)
    seen[a] = True
    frontier = np.array([a])
    while frontier.size and not seen[b]:
        n = nbr[_rows(off, frontier)[0]]
        frontier = np.unique(n[~seen[n]])
        seen[frontier] = True
    return bool(seen[b])


def dijkstra(rm: QueryRoadmap, start: int):
    """d[v] over live edges of finite weight, each sum rounded as Dijkstra's combineCosts rounds it: the least fixpoint of
    d[v] = min fl(d[u] + w), reached by relaxing the rows of the vertices whose distance fell until none falls (w >= 0 and
    fl(+) monotone: any relaxation order ends there)."""
    off, nbr, eid = rm.csr()
    w = np.asarray(rm.cost, np.float64).reshape(-1)[eid]
    d = np.full(rm.V, INF)
    d[start] = 0.0
    frontier = np.array([start])
    while frontier.size:
        pos, src = _rows(off, frontier)
        ok = w[pos] < INF
        pos, src = pos[ok], src[ok]
        nd = d[src] + w[pos]
        lower = d.copy()
        np.minimum.at(lower, nbr[pos], nd)
        frontier = np.flatnonzero(lower < d)
        d = lower
    return d.tolist()


def shortest_path(rm: QueryRoadmap, d, start: int, goal: int):
    """The tie rule: edge (u, v) is tight if fl(d[u] + w) == d[v]; level = hops from the start over tight edges (a BFS);
    pred[v] = the tight neighbour one level down with the lowest index, then the lowest edge index. Returns the path's
    (vertices, edges) from the goal back to the start."""
    off, nbr, eid = rm.csr()
    w = np.asarray(rm.cost, np.float64).reshape(-1)[eid]
    d = np.asarray(d, np.float64)
    level = np.full(rm.V, -1, np.int64)
    level[start] = 0
    frontier, t = np.array([start]), 0
    while frontier.size:
        pos, src = _rows(off, frontier)
        n = nbr[pos]
        tight = (w[pos] < INF) & (d[src] + w[pos] == d[n]) & (level[n] < 0)
        frontier = np.unique(n[tight])
        t += 1
        level[frontier] = t
    verts, edges, v = [goal], [], goal
    while v != start:
        sl = slice(off[v], off[v + 1])
        n, e, we = nbr[sl], eid[sl], w[sl]
        ok = (we < INF) & (d[n] < INF) & (level[n] == level[v] - 1) & (d[n] + we == d[v])
        k = np.lexsort((e[ok], n[ok]))[0]
        v = int(n[ok][k])
        edges.append(int(e[ok][k]))
        verts.append(v)
    return verts, edges


class NoPath(Exception):
    """ompl::Exception("Could not find solution path"): Planner::plan reports NOT_SOLVED."""


def construct_solution(rm: QueryRoadmap, start: int, goal: int, check_motion, stats):
    """One constructSolution: the path from start to goal, or None after removing its first invalid edge from the goal's
    side. The vertex pass (:580-630) is dead: addValidMilestone marks every vertex valid."""
    stats["searches"] += 1
    d = dijkstra(rm, start)
    if not d[goal] < INF:
        raise NoPath()
    verts, edges = shortest_path(rm, d, start, goal)
    for i, e in enumerate(edges):               # prevVertex = verts[i] (goal side), pos = verts[i + 1]
        if rm.flag[e] & VALID:
            continue
        stats["checked"] += 1
        if check_motion(rm.states[verts[i + 1]], rm.states[verts[i]]):
            rm.flag[e] |= VALID
        else:
            rm.remove_edge(e)
            stats["removed"].append(e)
            return None
    return verts[::-1], edges[::-1]


def base_solve(rm: QueryRoadmap, start_state, goal_state, is_valid, edge_cost, check_motion, in_bounds=None):
    """clearQuery + baseSolve. Returns a dict: status, path (vertex indices from the start), cost (left-to-right sum of the
    path's weights), searches, checked, removed (edge indices), start, goal."""
    out = {"status": 0, "path": [], "cost": 0.0, "searches": 0, "checked": 0, "removed": [], "start": -1, "goal": -1}
    for s, bad in ((start_state, INVALID_START), (goal_state, INVALID_GOAL)):
        s = np.asarray(s, np.float64)
        if (in_bounds is not None and not in_bounds(s)) or not bool(np.asarray(is_valid(s.reshape(1, 7)))[0]):
            out["status"] = bad
            return out
    rm.clear_query()
    start = out["start"] = rm.add_milestone(start_state, is_valid, ro.MILESTONE | ro.QUERY)
    goal = out["goal"] = rm.add_milestone(goal_state, is_valid, ro.MILESTONE | ro.QUERY)
    cost_for_vertex_edges(rm, start, edge_cost)
    cost_for_vertex_edges(rm, goal, edge_cost)
    if not connected(rm, start, goal):
        out["status"] = NOT_CONNECTED
        return out
    while True:
        try:
            sol = construct_solution(rm, start, goal, check_motion, out)
        except NoPath:
            out["status"] = NO_FEASIBLE_PATH
            return out
        if sol is not None:
            out["status"] = SOLVED
            out["path"] = sol[0]
            c = 0.0
            for e in sol[1]:
                c += rm.cost[e]
            out["cost"] = c
            return out
        if not connected(rm, start, goal):
            out["status"] = NOT_CONNECTED
            return out


def segment_count(space, a, b) -> int:
    """SE3StateSpace::validSegmentCount. space: (low[3], high[3], fraction)."""
    low, high, frac = space
    frac = frac if frac > 0 else 0.01
    ext = math.sqrt(sum((high[i] - low[i]) ** 2 for i in range(3)))
    d3 = math.sqrt(sum((a[i] - b[i]) ** 2 for i in range(3)))
    dq = abs(a[3] * b[3] + a[4] * b[4] + a[5] * b[5] + a[6] * b[6])
    ds = 0.0 if dq > 1.0 - 1e-9 else math.acos(dq)
    return max(int(math.ceil(d3 / (ext * frac))), int(math.ceil(ds / (0.5 * math.pi * frac))))


def discrete_motion(is_valid, space):
    """DiscreteMotionValidator::checkMotion(s1, s2) over is_valid(states [n, 7]) -> bool [n]."""
    def check(s1, s2) -> bool:
        nd = max(segment_count(space, s1, s2), 1)
        states = [ro.interpolate(s1, s2, j / nd) for j in range(1, nd)] + [np.asarray(s2, np.float64)]
        return bool(np.all(np.asarray(is_valid(np.array(states).reshape(-1, 7)), bool)))
    return check
