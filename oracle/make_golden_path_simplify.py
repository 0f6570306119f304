"""Golden results of Planner::getSolutionPath(true) as restated in oracle/path_simplify_oracle.py, with every isValid
answered by the reference's own compiled ODE (oracle/_ref/liborc_ref.so) and SE(3) distance / interpolate in libm. The
inputs are fixed paths over the golden roadmaps of the two maps of tests/roadmap_cases.py (tests/golden/roadmap.npz):
per map, breadth-first paths along roadmap edges from a milestone to the milestone the most hops away in its component.
The comparison cost is the path's SE(3) length (PathGeometric::length). Run where the reference tree is available:
    python oracle/make_golden_path_simplify.py  -> tests/golden/path_simplify.npz"""
import os
import sys
from collections import deque

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import orc  # noqa: E402
from oracle import path_simplify_oracle as pso  # noqa: E402
from oracle import roadmap_oracle as ro  # noqa: E402
import roadmap_cases as rc  # noqa: E402

SEEDS = (3, 4, 5)
INFO_KEYS = ("n_in", "n_simplified", "n_out", "reduce_edits", "collapse_edits", "shortcut_edits", "bspline_edits",
             "motion_checks", "state_checks", "check_passed", "returned_simplified", "calls")


def bfs_paths(states, kinds, edges, count):
    """`count` paths: from the milestones at 0, 1/3, 2/3 of the milestone list, each to its farthest vertex in hops."""
    adj = [[] for _ in range(len(states))]
    for a, b in edges:
        adj[a].append(b)
        adj[b].append(a)
    ms = np.flatnonzero(kinds == ro.MILESTONE)
    out = []
    for k in range(count):
        src = int(ms[k * len(ms) // count])
        pred, order, q = {src: -1}, [src], deque([src])
        while q:
            v = q.popleft()
            for w in sorted(adj[v]):
                if w not in pred:
                    pred[w] = v
                    order.append(w)
                    q.append(w)
        v, path = order[-1], []
        while v != -1:
            path.append(v)
            v = pred[v]
        out.append(states[path[::-1]])
    return out


def cases():
    """(name, case, [paths]) per golden map, from the committed roadmap golden."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "roadmap.npz"))
    for name in rc.GOLDEN_CASES:
        yield name, rc.make_case(name), bfs_paths(g[f"{name}/states"], g[f"{name}/kinds"], g[f"{name}/edges"], len(SEEDS))


def space_of(c):
    """MotionValidator.se3Space's bounds: centre +- the full map length in x / y, the finite elevation range -+ reach.z / 2."""
    m = c.m
    lx, ly = m.length
    e = m.elevation[np.isfinite(m.elevation)]
    return ([m.cx - lx, m.cy - ly, float(e.min()) - c.rp.reach_z / 2], [m.cx + lx, m.cy + ly, float(e.max()) + c.rp.reach_z / 2],
            0.01)


def simplify_all(kind):
    """{key: array} of every golden case with isValid from the oracle `kind` ("reference" or "port")."""
    res = {}
    for name, c, paths in cases():
        o = orc.Oracle(c.rp, kind)
        o.set_map(c.m)
        is_valid = ro.validity(o)
        for k, (p, seed) in enumerate(zip(paths, SEEDS)):
            out, info, simp = pso.get_solution_path(p, is_valid, space_of(c), seed, pso.path_length)
            key = f"{name}/{k}"
            res.update({f"{key}/path": p, f"{key}/seed": np.array([seed], np.int64), f"{key}/out": out,
                        f"{key}/simplified": simp, f"{key}/info": np.array([info[i] for i in INFO_KEYS], np.int64),
                        f"{key}/costs": np.array([info["cost_original"], info["cost_simplified"]])})
    return res


def main():
    res = simplify_all("reference")
    for k in sorted(res):
        if k.endswith("/info"):
            print(k, dict(zip(INFO_KEYS, res[k].tolist())))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "path_simplify.npz"), **res)


if __name__ == "__main__":
    main()
