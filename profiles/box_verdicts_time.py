"""Time the box verdicts (artp_box_verdicts_device) against a check of the same states (artp_check_poses_device) on the
benchmark's configs[1] maps (1000 x 1000 at 0.04 m, gentle and rough), and the box-verdict layer
(artp_box_verdict_layer_device) at 1000 x 1000 and 4000 x 4000. The explain form decides all five boxes of every pose,
where a check drops a pose at its first failing box, so it is expected to be slower, most of all where many poses fail.
Both give the same valid set. Prints one JSON line with the card's name and power limit, read in the same run.

    python profiles/box_verdicts_time.py [--reps 5] [--n 1048576]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.dirname(os.path.abspath(__file__))]

import heading_layer_cases as hlc  # noqa: E402
from art_planner_b200 import synth  # noqa: E402
from heading_layer_time import card  # noqa: E402


def timed_ms(fn, reps):
    import torch
    fn()                                                           # warm-up: scratch, queues, modules
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def checker(ap, m):
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    chk.estimateNormals(hlc.normal_radius(synth.PARAMS_YAML), want_host=False)
    return chk


def main() -> None:
    import torch
    import art_planner_b200 as ap
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--reps", type=int, default=5)
    ap_.add_argument("--n", type=int, default=1 << 20)
    a = ap_.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    res = {"card": card(), "maps": "configs[1]: fBm 1000x1000@0.04m seed 2 (gentle amp 0.6 m; rough amp 1.2 m, wavelength 3, "
           "persistence 0.7), yaml robot; 4000x4000 gentle fBm", "reps": a.reps, "n": a.n, "runs": []}
    for kind in ("gentle", "rough"):
        m = hlc.large_map(kind)
        chk = checker(ap, m)
        states = torch.from_numpy(synth.make_terrain_poses(m, a.n, seed=3, normal_cells=12)).cuda()
        valid = torch.empty(a.n, dtype=torch.uint8, device="cuda")
        why = torch.empty(a.n, dtype=torch.int16, device="cuda")
        check_ms = timed_ms(lambda: chk.isValidBatch(states, out=valid), a.reps)
        why_ms = timed_ms(lambda: chk.boxVerdicts(states, out=why), a.reps)
        assert torch.equal((why & 0x1F) == 0, valid != 0), kind
        d_layer = torch.empty((m.cols, m.rows), dtype=torch.int16, device="cuda").t()
        layer_ms = timed_ms(lambda: chk.boxVerdictLayer(0.7, out=d_layer), a.reps)
        res["runs"].append({"map": kind, "valid_share": round(float((valid != 0).float().mean()), 4),
                            "check_ms": round(check_ms, 3), "check_poses_per_s": float(f"{a.n / check_ms * 1e3:.3g}"),
                            "verdicts_ms": round(why_ms, 3), "verdicts_poses_per_s": float(f"{a.n / why_ms * 1e3:.3g}"),
                            "layer_1000_ms": round(layer_ms, 3)})
    m = synth.make_fbm_map(4000, 4000, 0.04, seed=2, amp=0.6)
    chk = checker(ap, m)
    d_layer = torch.empty((m.cols, m.rows), dtype=torch.int16, device="cuda").t()
    res["layer_4000_gentle_ms"] = round(timed_ms(lambda: chk.boxVerdictLayer(0.7, out=d_layer), a.reps), 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
