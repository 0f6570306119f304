"""Generate tests/golden/reference_offgrid.npz with the reference's own compiled ODE (oracle/_ref/liborc_ref.so): the
verdicts of the off-grid geometries of tests/offgrid_cases.py (rows = 1, 2, 3 mod 4, non-square and off-origin maps,
0.025 to 0.2 m cells, maps smaller than the robot and two vertices wide).

Run where the reference tree is present:  python oracle/make_golden_offgrid.py
Like make_golden.py, the file holds the packed result masks plus a checksum of the inputs (generator drift is detected).
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import cases  # noqa: E402
import offgrid_cases as oc  # noqa: E402
from art_planner_b200 import synth  # noqa: E402
from oracle.make_golden import digest  # noqa: E402
from oracle.orc import Oracle, build  # noqa: E402


def main() -> None:
    build("ref")
    out = {}
    maps = {k: f() for k, f in oc.MAPS.items()}
    for name, mk, pk, seed in oc.POSE_CASES:
        m = maps[mk]
        o = Oracle(oc.PARAMS[pk], "reference")
        o.set_map(m)
        poses = oc.case_poses(m, mk, seed)
        v = o.check_poses(poses)
        out[name + "/mask"] = np.packbits(v)
        out[name + "/sha"] = np.array(digest(m.elevation, m.elevation_masked, poses))
        print(f"{name}: valid={int(v.sum())}/{len(v)}")
    for mk, seed, tilt, zr in oc.BOX_CASES:
        m = maps[mk]
        o = Oracle(oc.PARAMS["yaml"], "reference")
        o.set_map(m)
        for which in (0, 1):
            org, rot = cases.box_samples(m, oc.BOX_N, seed, which, tilt, zr)
            hit = o.box_collide(which, org, rot)
            out[f"box_{mk}/{which}/mask"] = np.packbits(hit)
            out[f"box_{mk}/{which}/sha"] = np.array(digest(m.elevation, m.elevation_masked, org, rot))
            print(f"box_{mk}/{which}: hit={int(hit.sum())}/{len(hit)}")
    for mk in oc.EDGE_MAPS:
        m = maps[mk]
        o = Oracle(oc.PARAMS["yaml"], "reference")
        o.set_map(m)
        n, steps, seed = oc.EDGES
        s1, s2 = synth.make_edges(m, n, seed)
        v = o.check_motions(s1, s2, steps)
        out[f"edges_{mk}/mask"] = np.packbits(v)
        out[f"edges_{mk}/sha"] = np.array(digest(m.elevation, m.elevation_masked, s1, s2))
        n, seed, dmin, dmax = oc.INTERIORS
        s1, s2 = synth.make_edges(m, n, seed, dmin=dmin, dmax=dmax)
        k = o.check_edge_interiors(s1, s2, None, 0.5)
        out[f"interior_{mk}/prefix"] = k.astype(np.int8)
        out[f"interior_{mk}/sha"] = np.array(digest(m.elevation, m.elevation_masked, s1, s2))
        n, seed, dmin, dmax = oc.SEGMENTS
        s1, s2 = synth.make_edges(m, n, seed, dmin=dmin, dmax=dmax)
        low, high = oc.se3_bounds(m, oc.PARAMS["yaml"].reach_z)
        nd = o.valid_segment_count(low, high, s1, s2)
        sv, t = o.check_motions_segments(s1, s2, nd)
        out[f"segments_{mk}/mask"] = np.packbits(sv)
        out[f"segments_{mk}/nd"] = nd.astype(np.int32)
        out[f"segments_{mk}/last_t"] = t
        out[f"segments_{mk}/sha"] = np.array(digest(m.elevation, m.elevation_masked, s1, s2))
        print(f"{mk}: edges valid={int(v.sum())}, interior prefix histogram {np.bincount(k).tolist()}, "
              f"segments valid={int(sv.sum())} nd {nd.min()}..{nd.max()}")
    path = os.path.join(ROOT, "tests", "golden", "reference_offgrid.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
