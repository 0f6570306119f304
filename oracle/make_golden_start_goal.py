"""Generate tests/golden/start_goal.npz with the reference's own compiled ODE (oracle/_ref/liborc_ref.so): the start / goal
disc search (StartState / GoalStateRegion::sampleGoal, start.cpp:7-41, goal.cpp:11-41) walked in candidate order through
the reference's isValid (tests/start_goal_oracle.py), on the queries of tests/start_goal_cases.py with explicit offsets.

Run where the reference sources are (oracle/Makefile builds the library):  python oracle/make_golden_start_goal.py
Inputs are regenerated from seeds; the fixture holds the expected index and state of every query plus a checksum of the
inputs (so generator drift is detected).
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import cases  # noqa: E402
import start_goal_cases as sgc  # noqa: E402
import start_goal_oracle  # noqa: E402
from oracle.make_golden import digest  # noqa: E402
from oracle.orc import Oracle, build  # noqa: E402


def main() -> None:
    build("ref")
    out = {}
    for name, mk, pk, n, n_iter, seed in sgc.GOLDEN_CASES:
        m = cases.MAPS[mk]()
        o = Oracle(cases.PARAMS[pk], "reference")
        o.set_map(m)
        centres, radius, off = sgc.golden_inputs(m, n, n_iter, seed)
        states, idx = start_goal_oracle.find_valid_near(o, centres, n_iter, off)
        out[name + "/index"] = idx.astype(np.int32)
        out[name + "/states"] = states
        out[name + "/sha"] = np.array(digest(m.elevation, m.elevation_masked, centres, radius, off))
        hist = {"centre": int((idx == 0).sum()), "k<=10": int(((idx > 0) & (idx <= 10)).sum()),
                "k>10": int((idx > 10).sum()), "none": int((idx < 0).sum())}
        print(f"{name}: {hist}")
    path = os.path.join(ROOT, "tests", "golden", "start_goal.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
