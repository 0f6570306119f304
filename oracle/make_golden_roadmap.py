"""Golden roadmaps of PRMMotionCost's sampleGraph loop (prm_motion_cost.cpp:171-194, addValidMilestone :325-390), restated
in oracle/roadmap_oracle.py with every isValid answered by the reference's own compiled ODE (oracle/_ref/liborc_ref.so)
on the two maps of tests/roadmap_cases.py at scaled caps. Run where the reference tree is available:
    python oracle/make_golden_roadmap.py  -> tests/golden/roadmap.npz"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import orc  # noqa: E402
from oracle import roadmap_oracle as ro  # noqa: E402
import roadmap_cases as rc  # noqa: E402


def main():
    out = {}
    for name in rc.GOLDEN_CASES:
        c = rc.make_case(name)
        o = orc.Oracle(c.rp, "reference")
        o.set_map(c.m)
        rm = ro.Roadmap()
        used, draws, rec = ro.sample_graph(rm, o, c.m, c.layers, c.sp, c.rp.reach_z, rc.SEED, 0, *rc.CAPS, rc.MAX_DRAWS, c.dp,
                                           c.sample_filter, c.observed)
        st, kinds, edges = rm.result()
        out.update({f"{name}/states": st, f"{name}/kinds": kinds, f"{name}/edges": edges, f"{name}/draws": draws,
                    f"{name}/recompute_v": rec, f"{name}/draws_used": np.array([used], np.int64)})
        print(name, "V", rm.V, "E", rm.E, "milestones", len(draws), "draws", used, "recomputes", list(rec))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "roadmap.npz"), **out)


if __name__ == "__main__":
    main()
