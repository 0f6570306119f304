"""Time one planning query on the roadmap of the shipped caps (10 000 vertices / 50 000 edges) on the configs[1] map
(1000 x 1000 fBm) at both roughness levels, two ways, and check that both return the same path:
  device   artp_roadmap_update_edges once, then artp_roadmap_solve: start / goal milestones, their edges priced, search and
           motion checks without leaving the device
  host     the route without these calls: artp_roadmap_add_milestones, artp_roadmap_get, artp_motion_cost_states on the
           copied-out edges (all of them once, then the ones at the start and at the goal), scipy.sparse.csgraph.dijkstra,
           artp_check_motions_segments on the path's edges of unknown validity, repeated while an edge fails
Every repeat builds both roadmaps afresh (a query changes its roadmap), so each timed call does the same work; times are
host clocks around calls that end in a stream synchronise, medians over the warm repeats. The stages inside
artp_roadmap_solve are not timed separately. Prints one JSON line with the card's name and power limit."""
import dataclasses
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
from scipy.sparse import coo_matrix  # noqa: E402
from scipy.sparse.csgraph import connected_components, dijkstra  # noqa: E402

import art_planner_b200 as ap  # noqa: E402
from art_planner_b200 import costnet, synth  # noqa: E402
from art_planner_b200.checker import _Handle  # noqa: E402
from oracle import basic_oracle as bo  # noqa: E402

CAPS = (10000, 50000, 1000)
REPEATS = 6
THR = 10.0         # every edge feasible: the query is decided by the graph and the motion checks


class Side:
    def __init__(self, m, rp, thr_layer, obs, L, sp):
        self.chk = ap.StateValidityChecker(rp, handle=_Handle(rp, 0, risk_threshold=THR))
        self.chk.setMap(m)
        self.chk.updateHeightField()
        self.chk.setSampleFilter(thr_layer, obs)
        self.obj = ap.MotionCostObjective(self.chk)
        self.obj.setWeights(costnet.make_state_dict(seed=5))
        self.obj.updateFeatures()
        self.mv = ap.MotionValidator(self.chk)
        self.L, self.sp = L, sp

    def build(self):
        smp = ap.SE3FromSE2Sampler(self.chk, self.L, self.sp, seed=1234)
        self.rm = ap.PRMRoadmap(self.chk, 20000, 60000)
        self.rm.sampleGraph(smp, *CAPS)


def clock(f):
    t0 = time.perf_counter()
    r = f()
    return r, (time.perf_counter() - t0) * 1e3


def host_query(s, start, goal, space, t):
    """Today's route. Appends its stage times to t; returns (status, path)."""
    rm, obj = s.rm, s.obj
    (st, edges), ms = clock(lambda: (rm.vertices()[0], rm.edges()))
    t["host_copy_out"].append(ms)
    (w, feas, _), ms = clock(lambda: obj.updateEdgesBatch(st[edges[:, 0]], st[edges[:, 1]]))
    t["host_update_edges"].append(ms)
    valid = feas.astype(bool)
    nv0, ne0 = len(st), len(edges)
    _, ms = clock(lambda: rm.addValidMilestones(np.stack([start, goal])))
    (st2, e2), ms2 = clock(lambda: (rm.vertices(first=nv0)[0], rm.edges(first=ne0)))
    t["host_add"].append(ms + ms2)
    st, edges = np.concatenate([st, st2]), np.concatenate([edges, e2])
    w, valid = np.concatenate([w, np.zeros(len(e2))]), np.concatenate([valid, np.zeros(len(e2), bool)])
    live = np.ones(len(edges), bool)
    sv = nv0
    gv = int(np.flatnonzero(rm.vertices()[1] & 4)[1])

    def price():
        for v in (sv, gv):
            inc = np.flatnonzero((edges[:, 0] == v) | (edges[:, 1] == v))
            other = np.where(edges[inc, 0] == v, edges[inc, 1], edges[inc, 0])
            w[inc] = obj.updateEdgesBatch(np.repeat(st[v][None], len(inc), 0), st[other])[0]
    _, ms = clock(price)
    t["host_price"].append(ms)
    search_ms = check_ms = 0.0
    searches = 0
    while True:
        keep = live & np.isfinite(w)

        def search():
            g = coo_matrix((w[keep], (edges[keep, 0], edges[keep, 1])), shape=(len(st), len(st))).tocsr()
            return dijkstra(g, directed=False, indices=sv, return_predecessors=True)
        (d, pred), ms = clock(search)
        search_ms += ms
        searches += 1
        if not np.isfinite(d[gv]):
            path = None
            break
        path = [gv]
        while path[-1] != sv:
            path.append(int(pred[path[-1]]))
        eid = {frozenset((int(a), int(b))): i for i, (a, b) in enumerate(edges) if live[i]}
        pe = [eid[frozenset((path[i], path[i + 1]))] for i in range(len(path) - 1)]
        unknown = [i for i, e in enumerate(pe) if not valid[e]]
        if not unknown:
            break
        s1, s2 = st[[path[i + 1] for i in unknown]], st[[path[i] for i in unknown]]
        (ok, _), ms = clock(lambda: s.mv.checkMotionSegments(s1, s2, space=space))
        check_ms += ms
        bad = np.flatnonzero(ok == 0)
        for i, o in zip(unknown, ok):
            if o:
                valid[pe[i]] = True
        if not bad.size:
            break
        live[pe[unknown[int(bad[0])]]] = False
    t["host_search"].append(search_ms)
    t["host_validate"].append(check_ms)
    t["host_searches"] = searches
    return (1 if path else 3), (path[::-1] if path else [])


def run(kind):
    m = synth.make_fbm_map(1000, 1000) if kind == "gentle" else \
        synth.make_fbm_map(1000, 1000, seed=12, amp=1.2, wavelength=3.0, persistence=0.7)
    rp = synth.PARAMS_YAML
    trav, obs = synth.make_traversability(m, seed=13)
    _, thr = bo.masked_elevation(m.elevation, trav, obs, m.res, bo.BasicParams())
    L = synth.make_sampler_layers(m, seed=7)
    sp = dataclasses.replace(synth.sampler_params_for(m), use_inverse_vertex_density=True, use_max_prob_unknown_samples=True)
    dev, host = Side(m, rp, thr, obs, L, sp), Side(m, rp, thr, obs, L, sp)
    space = ap.MotionValidator.se3Space(m, rp.reach_z)
    t = {k: [] for k in ("update_edges", "solve", "host_copy_out", "host_update_edges", "host_add", "host_price", "host_search",
                         "host_validate", "host_total")}
    info = None
    for rep in range(REPEATS):
        dev.build()
        host.build()
        st, kinds = dev.rm.vertices()
        if rep == 0:                                     # two far-apart milestones of the largest component, nudged
            e = dev.rm.edges()
            lab = connected_components(coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(len(st), len(st))),
                                       directed=False)[1]
            ms_ = st[(kinds == 1) & (lab == np.bincount(lab).argmax())]
            a = ms_[np.argmin(ms_[:, 0] + ms_[:, 1])] + np.array([0.011, -0.017, 0, 0, 0, 0, 0])
            b = ms_[np.argmax(ms_[:, 0] + ms_[:, 1])] + np.array([-0.013, 0.019, 0, 0, 0, 0, 0])
            assert dev.chk.isValidBatch(np.stack([a, b])).all(), "the query's ends are not valid poses"
        _, ms = clock(dev.rm.updateEdges)
        t["update_edges"].append(ms)
        (status, _, idx, cost, info), ms = clock(lambda: dev.rm.solve(a, b, space))
        t["solve"].append(ms)
        (h_status, h_path), ms = clock(lambda: host_query(host, a, b, space, t))
        t["host_total"].append(ms)
        assert status == 1 and status == h_status and list(idx) == h_path, \
            f"the two routes disagree: {status} {h_status} {list(idx)[:8]} {h_path[:8]} {len(idx)} {len(h_path)} {cost} {info}"
    out = {k: float(np.median(v[1:])) for k, v in t.items() if isinstance(v, list)}
    out = {k + "_ms": v for k, v in out.items()}
    out.update({"vertices": int(len(kinds)), "status": int(status), "path_vertices": int(len(idx)), "cost": cost,
                "searches": info["searches"], "sweeps": info["sweeps"], "edges_checked": info["edges_checked"],
                "edges_removed": info["edges_removed"], "host_searches": t["host_searches"]})
    return out


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"gpu": gpu, "caps": CAPS, "gentle": run("gentle"), "rough": run("rough")}))


if __name__ == "__main__":
    main()
