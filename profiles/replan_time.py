"""Whole-replan timing: artp_planner_set_map + artp_plan (one call each) against the same replan through the chained public
calls (tests/planner_cases.py), on the configs[1] map (1000 x 1000 at 0.04 m, gentle and rough fBm) at the shipped caps,
with the same seeds; both routes must return the same path and counters. Also the map-update stage alone on a
4000 x 4000 map. Prints one JSON object: per route the median wall ms of set_map and plan, the one-call route's stage
split (device ms from its events), host synchronisations and host <-> device bytes. The one-call route's bytes are the
counts the library reports for its copies (artp_planner_map_info, artp_plan_info); the chained route's are the layers
its public calls take and return (Basic: three in, two out; the map upload: two in)."""
from __future__ import annotations

import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import planner_cases as pc  # noqa: E402
import art_planner_b200 as ap  # noqa: E402
from art_planner_b200 import costnet, synth  # noqa: E402
from art_planner_b200.checker import _Handle  # noqa: E402


def handle(rp):
    chk = ap.StateValidityChecker(rp, handle=_Handle(rp, 0, risk_threshold=0.6))
    ap.MotionCostObjective(chk).setWeights(costnet.make_state_dict(seed=5))
    return chk


def ms(f):
    t = time.perf_counter()
    r = f()
    return (time.perf_counter() - t) * 1e3, r


def replan(m, reps=3):
    rp = synth.PARAMS_YAML
    layers = pc.raw_layers(m)
    one_set, one_plan, ch_set, ch_plan, infos, map_info = [], [], [], [], [], []
    for r in range(reps):
        pp = ap.Planner.params(seed=1 + r)
        pl, ch = ap.Planner(handle(rp), pp), pc.Chained(handle(rp), pp)
        t, mi = ms(lambda: pl.setMap(*layers, m.res, m.cx, m.cy)); one_set.append(t); map_info.append(mi)
        t, _ = ms(lambda: ch.setMap(*layers, m.res, m.cx, m.cy)); ch_set.append(t)
        for k, (s, g) in enumerate(pc.queries(ch.chk, 2, 7 + r, 4.0)):
            t, st = ms(lambda: pl.plan(s, g)); one_plan.append((k, t))
            t, (st2, path2, _) = ms(lambda: ch.plan(s, g)); ch_plan.append((k, t))
            assert st == st2 and (st != pl.SOLVED or np.array_equal(pl.getSolutionPath(), path2))
            i = pl.info()
            infos.append({k2: i[k2] for k2 in ("status", "sampled", "ms_sample_graph", "ms_update_edges", "ms_endpoints", "ms_solve",
                                              "ms_simplify", "host_syncs", "bytes_h2d", "bytes_d2h")})
    med = lambda xs: float(np.median(xs))
    first = lambda xs: [t for k, t in xs if k == 0]
    later = lambda xs: [t for k, t in xs if k > 0]
    return {
        "map": m.desc, "one_call": {"set_map_ms": med(one_set), "plan_with_sampling_ms": med(first(one_plan)),
                                    "plan_on_same_map_ms": med(later(one_plan)), "map": map_info[-1]},
        "chained": {"set_map_ms": med(ch_set), "plan_with_sampling_ms": med(first(ch_plan)), "plan_on_same_map_ms": med(later(ch_plan)),
                    "map": ch.map_bytes},
        "plans": infos}


def map_update(rows=4000, reps=3):
    m = synth.make_fbm_map(rows, rows, seed=3)
    layers = pc.raw_layers(m)
    rp = synth.PARAMS_YAML
    pp = ap.Planner.params(seed=1)
    pl, ch = ap.Planner(handle(rp), pp), pc.Chained(handle(rp), pp)
    one = [ms(lambda: pl.setMap(*layers, m.res, m.cx, m.cy))[0] for _ in range(reps)]
    chained = [ms(lambda: ch.setMap(*layers, m.res, m.cx, m.cy))[0] for _ in range(reps)]
    return {"map": f"{rows}x{rows}", "one_call_set_map_ms": float(np.median(one)), "chained_set_map_ms": float(np.median(chained)),
            "layer_mb": 4 * rows * rows / 2 ** 20}


def main():
    import torch
    out = {"gpu": torch.cuda.get_device_name(0),
           "configs1": [replan(synth.make_fbm_map(1000, 1000)),
                        replan(synth.make_fbm_map(1000, 1000, seed=12, amp=1.2, wavelength=3.0, persistence=0.7))],
           "map_update": map_update()}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
