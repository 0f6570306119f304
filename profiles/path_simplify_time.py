"""Time Planner::getSolutionPath(true) on one far-corner query of the roadmap at the shipped caps (10 000 vertices /
50 000 edges) on the configs[1] map (1000 x 1000 fBm) at both roughness levels, two ways, and check that both return
the same path:
  device   artp_simplify_path: the whole schedule, the check and both costs, the path on the device throughout
  host     what an OMPL simplifier over this library's adapters does: oracle/path_simplify_oracle.py driving one
           artp_check_motions_segments call per checkMotion and one artp_check_poses call per isValid, the costs through
           artp_motion_cost_split, SE(3) distance / interpolate through artp_debug_se3_ops (batched where the restatement
           batches them). host_check_calls_ms is the time inside the checkMotion / isValid calls -- the route's own cost;
           host_se3_calls_ms the SE(3) helper round trips (arithmetic an OMPL simplifier does in-process, so not part of
           that route) and host_cost_calls_ms the final pricing; the rest of host_total_ms (host_python_ms) is the
           restatement's Python bookkeeping, which a C++ simplifier would largely not pay.
Times are host clocks around calls that end in a stream synchronise, medians over the warm repeats. Prints one JSON line
with the card's name and power limit."""
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
from scipy.sparse.csgraph import connected_components  # noqa: E402

import art_planner_b200 as ap  # noqa: E402
from art_planner_b200 import costnet, synth  # noqa: E402
from art_planner_b200.checker import _Handle  # noqa: E402
from oracle import basic_oracle as bo  # noqa: E402
from oracle import path_simplify_oracle as pso  # noqa: E402

CAPS = (10000, 50000, 1000)
REPEATS = 6
THR = 10.0
SEED = 17


class TimedOps:
    """SE(3) distance / interpolate through artp_debug_se3_ops (the device's arithmetic, so both routes take the same
    decisions), timed as library calls."""

    def __init__(self, chk, owner):
        import test_path_simplify_gpu as tg
        self.ops, self.owner = tg.DeviceOps(chk.handle), owner

    def distance(self, A, B):
        t0 = time.perf_counter()
        r = self.ops.distance(A, B)
        self.owner.se3 += time.perf_counter() - t0
        return r

    def interpolate(self, A, B, T):
        t0 = time.perf_counter()
        r = self.ops.interpolate(A, B, T)
        self.owner.se3 += time.perf_counter() - t0
        return r


class HostSimplifier(pso.Simplifier):
    """The restatement with one library call per checkMotion / isValid; `spent` is the time inside library calls."""

    def __init__(self, chk, space, seed):
        super().__init__(None, space, seed, ops=TimedOps(chk, self))
        self.chk, self.mv, self.sp = chk, ap.MotionValidator(chk), space
        self.spent, self.se3, self.cost = 0.0, 0.0, 0.0   # checkMotion + isValid calls, SE(3) helper calls, pricing

    def is_valid(self, s):
        self.stats["valids"] += 1
        t0 = time.perf_counter()
        ok = bool(self.chk.isValidBatch(np.asarray(s, np.float64).reshape(1, 7))[0])
        self.spent += time.perf_counter() - t0
        return ok

    def check_motion(self, a, b):
        self.stats["motions"] += 1
        t0 = time.perf_counter()
        ok, _ = self.mv.checkMotionSegments(np.asarray(a).reshape(1, 7), np.asarray(b).reshape(1, 7), space=self.sp)
        self.spent += time.perf_counter() - t0
        return bool(ok[0])


def host_route(chk, obj, space, path):
    sim = HostSimplifier(chk, space, SEED)
    simp = [np.array(s) for s in path]
    t0 = time.perf_counter()
    passed = sim.simplify_max(simp) and sim.check(simp)
    out = path
    if passed:
        t1 = time.perf_counter()
        cs, co = obj.pathCost(np.array(simp)), obj.pathCost(path)
        sim.cost += time.perf_counter() - t1
        out = path if co < cs else np.array(simp)
    total = (time.perf_counter() - t0) * 1e3
    return out, sim.stats, total, (sim.spent * 1e3, sim.se3 * 1e3, sim.cost * 1e3)


def run(kind):
    m = synth.make_fbm_map(1000, 1000) if kind == "gentle" else \
        synth.make_fbm_map(1000, 1000, seed=12, amp=1.2, wavelength=3.0, persistence=0.7)
    rp = synth.PARAMS_YAML
    trav, obs = synth.make_traversability(m, seed=13)
    _, thr = bo.masked_elevation(m.elevation, trav, obs, m.res, bo.BasicParams())
    L = synth.make_sampler_layers(m, seed=7)
    sp = dataclasses.replace(synth.sampler_params_for(m), use_inverse_vertex_density=True, use_max_prob_unknown_samples=True)
    chk = ap.StateValidityChecker(rp, handle=_Handle(rp, 0, risk_threshold=THR))
    chk.setMap(m)
    chk.updateHeightField()
    chk.setSampleFilter(thr, obs)
    obj = ap.MotionCostObjective(chk)
    obj.setWeights(costnet.make_state_dict(seed=5))
    obj.updateFeatures()
    space = ap.MotionValidator.se3Space(m, rp.reach_z)
    rm = ap.PRMRoadmap(chk, 20000, 60000)
    rm.sampleGraph(ap.SE3FromSE2Sampler(chk, L, sp, seed=1234), *CAPS)
    rm.updateEdges()
    st, kinds = rm.vertices()
    e = rm.edges()
    lab = connected_components(coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(len(st), len(st))), directed=False)[1]
    ms_ = st[(kinds == 1) & (lab == np.bincount(lab).argmax())]
    a = ms_[np.argmin(ms_[:, 0] + ms_[:, 1])] + np.array([0.011, -0.017, 0, 0, 0, 0, 0])
    b = ms_[np.argmax(ms_[:, 0] + ms_[:, 1])] + np.array([-0.013, 0.019, 0, 0, 0, 0, 0])
    status, path, _, _, _ = rm.solve(a, b, space)
    assert status == 1, f"the query was not solved ({status})"
    ps = ap.PathSimplifier(chk, space, "learned", SEED)
    t = {"device": [], "host_total": [], "host_check_calls": [], "host_se3_calls": [], "host_cost_calls": []}
    for _ in range(REPEATS):
        t0 = time.perf_counter()
        got, info = ps.getSolutionPath(path)
        t["device"].append((time.perf_counter() - t0) * 1e3)
        ref, stats, total, calls = host_route(chk, obj, space, path)
        t["host_total"].append(total)
        for k, v in zip(("host_check_calls", "host_se3_calls", "host_cost_calls"), calls):
            t[k].append(v)
        assert got.shape == ref.shape and np.abs(got - ref).max() <= 1e-9, "the two routes disagree"
        assert (stats["motions"], stats["valids"]) == (info["motion_checks"], info["state_checks"])
    out = {k + "_ms": float(np.median(v[1:])) for k, v in t.items()}
    out["host_python_ms"] = out["host_total_ms"] - out["host_check_calls_ms"] - out["host_se3_calls_ms"] - out["host_cost_calls_ms"]
    out.update({"path_in": info["n_in"], "path_simplified": info["n_simplified"], "path_out": info["n_out"],
                "motion_checks": info["motion_checks"], "state_checks": info["state_checks"], "rounds": info["rounds"],
                "discarded": info["discarded"], "returned_simplified": info["returned_simplified"],
                "edits": [info["reduce_edits"], info["collapse_edits"], info["shortcut_edits"], info["bspline_edits"]]})
    return out


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"gpu": gpu, "caps": CAPS, "gentle": run("gentle"), "rough": run("rough")}))


if __name__ == "__main__":
    main()
