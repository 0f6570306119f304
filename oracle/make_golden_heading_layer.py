"""Generate tests/golden/heading_layer.npz with the reference's own compiled ODE (oracle/_ref/liborc_ref.so): the
valid-heading layer (artp_valid_heading_layer) of the cases in tests/heading_layer_cases.py. Each cell centre at each
heading is projected with tests/start_goal_oracle.pose_from_2d (Planner::plan's goal projection) on the normals of
oracle.orc.estimate_normals, and the reference's isValid decides the bit.

Run where the reference sources are (oracle/Makefile builds the library):  python oracle/make_golden_heading_layer.py
Inputs are regenerated from seeds; the fixture holds each case's masks, the projected poses of POSE_CELLS of its cells
and a checksum of the inputs (so generator drift is detected).
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import heading_layer_cases as hlc  # noqa: E402
import start_goal_oracle  # noqa: E402
from oracle import orc  # noqa: E402
from oracle.make_golden import digest  # noqa: E402


class Normals:
    def __init__(self, m, radius):
        self.normal_x, self.normal_y, self.normal_z, _ = orc.estimate_normals(m, radius)


def layer(oracle, m, normals, yaws):
    """(masks uint32 [rows, cols], poses [rows * cols * n, 7]) of one case."""
    poses, inside = start_goal_oracle.pose_from_2d(m, normals, hlc.yaw_states(m, yaws))
    assert inside.all()
    return hlc.pack(oracle.check_poses(poses), len(yaws), (m.rows, m.cols)), poses


def main() -> None:
    orc.build("ref")
    out = {}
    for name, mk, pk, hk in hlc.GOLDEN_CASES:
        m, p, yaws = hlc.MAPS[mk](), hlc.PARAMS[pk], hlc.HEADINGS[hk]
        assert m.rows * m.cols <= 40000 and len(yaws) <= 8
        o = orc.Oracle(p, "reference")
        o.set_map(m)
        masks, poses = layer(o, m, Normals(m, hlc.normal_radius(p)), yaws)
        cells = hlc.pose_cells(m)
        n = len(yaws)
        out[name + "/masks"] = masks
        out[name + "/pose_cells"] = cells
        out[name + "/poses"] = poses.reshape(-1, n, 7)[cells].reshape(-1, 7)
        out[name + "/sha"] = np.array(digest(m.elevation, m.elevation_masked, yaws))
        counts = np.bitwise_count(masks) if hasattr(np, "bitwise_count") else None
        print(f"{name}: {m.rows}x{m.cols} x {n} headings, valid share {float(counts.mean()) / n if counts is not None else 0:.3f}")
    path = os.path.join(ROOT, "tests", "golden", "heading_layer.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
