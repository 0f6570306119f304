"""The parity harness of the queries on the device roadmap (artp_roadmap_update_edges / _solve / _get_edge_costs) against
oracle/roadmap_query_oracle.py: Env.solve_both runs one query on the device and on the restatement of the device's own
roadmap and edge weights, pricing the query edges with artp_motion_cost_states (the same head kernels: equality, not a
tolerance) and taking isValid from the port oracle. Compared: status, path vertex indices, REMOVED flags, searches run,
every weight, the roadmap itself; VALID flags may exceed the restatement's by edges the oracle's motion check passes too
(a validation round checks further along the path than the reference walks)."""
import numpy as np

import roadmap_cases as rc
from art_planner_b200 import costnet
from oracle import orc
from oracle import roadmap_oracle as ro
from oracle import roadmap_query_oracle as rqo

STATE_TOL = 1e-9
THR = 0.5          # seeded light-network risks lie around 0.5: feasible and infeasible edges


class Env:
    def __init__(self, c, network="light", thr=THR, vertex_capacity=8000, edge_capacity=20000):
        import art_planner_b200 as ap
        from art_planner_b200 import capi
        from art_planner_b200.checker import _Handle
        self.c, self.capi = c, capi
        self.chk = ap.StateValidityChecker(c.rp, handle=_Handle(c.rp, 0, risk_threshold=thr))
        self.chk.setMap(c.m)
        self.chk.updateHeightField()
        self.chk.setSampleFilter(c.thr, c.observed)
        self.smp = ap.SE3FromSE2Sampler(self.chk, c.layers, c.sp, seed=rc.SEED)
        self.obj = ap.MotionCostObjective(self.chk)
        self.obj.setWeights(costnet.make_state_dict(seed=5, network=network))
        self.obj.updateFeatures()
        self.o = orc.Oracle(c.rp, "port")
        self.o.set_map(c.m)
        self.is_valid = ro.validity(self.o)
        self.space = ap.MotionValidator.se3Space(c.m, c.rp.reach_z)
        self.bounds = (list(self.space.low), list(self.space.high), 0.01)
        self.check_motion = rqo.discrete_motion(self.is_valid, self.bounds)
        self.rm = ap.PRMRoadmap(self.chk, vertex_capacity, edge_capacity)

    def edge_cost(self, src, tgt):
        return self.obj.updateEdgesBatch(src, tgt)[0]

    def in_bounds(self, s):
        return all(self.bounds[0][i] <= s[i] <= self.bounds[1][i] for i in range(3))

    def mirror(self):
        """The device roadmap as the restatement's graph."""
        st, kinds = self.rm.vertices()
        cost, flags, live = self.rm.edgeCosts()
        q = rqo.QueryRoadmap(max(2 * len(st), 1024))
        q.V = len(st)
        q.states[:q.V], q.kinds[:q.V] = st, kinds
        q.edges = self.rm.edges().astype(np.int64).tolist()
        q.cost, q.flag = cost.tolist(), flags.astype(int).tolist()
        q.n_removed = int(np.count_nonzero(flags & rqo.REMOVED))
        assert live == q.E
        q.refresh_density()
        return q

    def solve_both(self, start, goal, path_capacity=4096):
        """One query on the device and on the restatement of the roadmap as it stood; everything compared."""
        q = self.mirror()
        ref = rqo.base_solve(q, start, goal, self.is_valid, self.edge_cost, self.check_motion, self.in_bounds)
        status, states, idx, cost, info = self.rm.solve(start, goal, self.space, path_capacity)
        assert status == ref["status"]
        assert list(idx) == ref["path"], (info, {k: ref[k] for k in ("searches", "checked", "removed", "cost")}, cost)
        assert info["searches"] == ref["searches"] and info["edges_removed"] == len(ref["removed"])
        st, kinds = self.rm.vertices()
        rst, rkinds, redges = q.result()
        assert np.array_equal(kinds, rkinds) and np.array_equal(self.rm.edges(), redges)
        assert np.abs(st - rst).max(initial=0.0) <= STATE_TOL
        dcost, dflags, live = self.rm.edgeCosts()
        assert np.array_equal(dcost, np.array(q.cost)) and live == q.E
        rflags = np.array(q.flag, np.uint8)
        assert np.array_equal(dflags & rqo.REMOVED, rflags & rqo.REMOVED)
        assert not ((rflags & rqo.VALID) & ~dflags).any()
        for e in np.flatnonzero((dflags & rqo.VALID) & ~rflags):
            a, b = q.edges[e]
            assert self.check_motion(st[a], st[b]) or self.check_motion(st[b], st[a])
        if status >= rqo.INVALID_START:
            return status, idx, info, ref
        assert (info["start_vertex"], info["goal_vertex"]) == (ref["start"], ref["goal"])
        assert list(idx) == ref["path"]
        if status == rqo.SOLVED:
            off, nbr, eid = q.csr()
            fold = 0.0
            for a, b in zip(idx[:-1], idx[1:]):
                row = slice(off[a], off[a + 1])
                fold += dcost[eid[row][nbr[row] == b][0]]
            assert cost == fold == ref["cost"]
            assert np.abs(states - st[idx]).max() <= STATE_TOL
            assert info["edges_checked"] >= ref["checked"]
        return status, idx, info, ref
