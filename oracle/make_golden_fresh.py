"""Generate tests/golden/reference_fresh.npz with the reference's own compiled ODE (oracle/_ref/liborc_ref.so):
the pose and box verdicts of the fresh-seed and adversarial-map cases of tests/test_oracle.py.

Run where the reference tree is present:  python oracle/make_golden_fresh.py
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
from art_planner_b200 import synth  # noqa: E402
from oracle.make_golden import digest  # noqa: E402
from oracle.orc import Oracle, build  # noqa: E402

#: (name, map factory, poses, pose seed, boxes per kind, box seed, tilt, z range) -- the inputs test_oracle.py rebuilds
FRESH_CASES = [(mk, cases.MAPS[mk], 5000, 1234, 5000, 4321, 0.8, 0.4) for mk in ("fixture", "ramp", "fbm_rough")]
ADVERSARIAL_CASES = [(f.__name__, f, 20000, 31, 20000, 99, 0.9, 0.35) for f in (cases.terraces, cases.spikes, cases.terraces_tilted)]


def main() -> None:
    build("ref")
    out = {}
    for name, mk, n_poses, pseed, n_boxes, bseed, tilt, zr in FRESH_CASES + ADVERSARIAL_CASES:
        m = mk()
        o = Oracle(cases.PARAMS["yaml"], "reference")
        o.set_map(m)
        poses = synth.make_terrain_poses(m, n_poses, seed=pseed)
        v = o.check_poses(poses)
        out[f"{name}/poses/mask"] = np.packbits(v)
        out[f"{name}/poses/sha"] = np.array(digest(m.elevation, m.elevation_masked, poses))
        for which in (0, 1):
            org, rot = cases.box_samples(m, n_boxes, bseed, which, tilt, zr)
            hit = o.box_collide(which, org, rot)
            out[f"{name}/{which}/mask"] = np.packbits(hit)
            out[f"{name}/{which}/sha"] = np.array(digest(m.elevation, m.elevation_masked, org, rot))
        print(f"{name}: valid={int(v.sum())}/{len(v)}")
    path = os.path.join(ROOT, "tests", "golden", "reference_fresh.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
