"""Maps, heading sets and the composition route of the valid-heading layer (artp_valid_heading_layer), shared by
oracle/make_golden_heading_layer.py (generation with the compiled reference) and the tests.

The layer's definition, restated: bit k of cell (r, c) is isValid of the goal projection (start_goal_oracle.pose_from_2d,
Planner::plan's planner.cpp:223-237) of the state at the cell's centre whose getYawFromSO3 is (float)yaw[k]. Poses are
numbered cell-major (cells in the layers' column-major order), heading-minor.
"""
from __future__ import annotations

import numpy as np

import cases
import offgrid_cases
from art_planner_b200 import synth

MAPS = {
    "fixture": cases.MAPS["fixture"],
    "terraces": cases.MAPS["terraces"],
    "spikes": cases.MAPS["spikes"],
    "fbm_rough": cases.MAPS["fbm_rough"],
    "r1": offgrid_cases.MAPS["r1"],                                      # 201 x 199, centred at (137.37, -52.81)
    "fbm_rough_200": lambda: synth.make_fbm_map(200, 200, amp=0.6),     # fbm_rough's recipe at the golden's size
}
PARAMS = cases.PARAMS

_F0 = float(np.float32(0.7))                 # a float; its neighbours one double ulp and one float ulp away
HEADINGS = {
    "one": np.array([0.0]),
    "even8": np.linspace(-np.pi, np.pi, 8, endpoint=False),
    "even32": np.linspace(-np.pi, np.pi, 32, endpoint=False),
    "irregular_pi": np.array([np.pi, -np.pi, 0.3, -2.1, 1e-3, 2.9, -0.77]),
    # yaws 1 and 2 are one double ulp either side of yaw 0 and round to the same float: their bits must equal yaw 0's.
    # yaw 3 is the next float up.
    "ulp": np.array([_F0, np.nextafter(_F0, 4.0), np.nextafter(_F0, -4.0),
                     float(np.nextafter(np.float32(_F0), np.float32(4.0))), -1.3, 2.4]),
}
#: indices of yaws in HEADINGS["ulp"] whose bits must equal those of yaw 0
ULP_SAME = (1, 2)

# (name, map, params, headings): at most 200^2 cells x 8 headings each, so the reference writes the golden in minutes
GOLDEN_CASES = [
    ("hl_fixture_yaml", "fixture", "yaml", "even8"),
    ("hl_fixture_header", "fixture", "header", "irregular_pi"),
    ("hl_terraces_yaml", "terraces", "yaml", "ulp"),
    ("hl_terraces_header", "terraces", "header", "even8"),
    ("hl_spikes_yaml", "spikes", "yaml", "irregular_pi"),
    ("hl_spikes_header", "spikes", "header", "one"),
    ("hl_fbm_rough_yaml", "fbm_rough_200", "yaml", "even8"),
    ("hl_fbm_rough_header", "fbm_rough_200", "header", "ulp"),
    ("hl_r1_yaml", "r1", "yaml", "even8"),
    ("hl_r1_yaml_pi", "r1", "yaml", "irregular_pi"),
]
POSE_CELLS = 128   # cells per golden case whose projected poses the golden stores


def normal_radius(p) -> float:
    """The estimation radius Planner passes to estimateNormals (processors::Basic, basic.cpp:47)."""
    return (p.torso_length + p.torso_width) * 0.25


def cell_centres(m):
    """(x, y) of every cell centre, column-major: grid_map::getPositionFromIndex as sample_state computes it."""
    r, c = np.indices((m.rows, m.cols))
    r, c = r.ravel(order="F").astype(np.float64), c.ravel(order="F").astype(np.float64)
    Lx, Ly = m.rows * m.res, m.cols * m.res
    return (m.cx + (0.5 * Lx - 0.5 * m.res)) + m.res * (-r), (m.cy + (0.5 * Ly - 0.5 * m.res)) + m.res * (-c)


def so3_yaw(s):
    """getYawFromSO3 (utils.h:80-88): double atan2, returned as float."""
    return np.arctan2(2 * (s[..., 6] * s[..., 5] + s[..., 3] * s[..., 4]),
                      1 - 2 * (s[..., 4] * s[..., 4] + s[..., 5] * s[..., 5])).astype(np.float32)


def yaw_states(m, yaws, cells=None):
    """The layer's input states [len(cells) * n, 7], cell-major: the centre of each cell (all cells by default, in
    column-major order), z = 0, and a quaternion about z whose getYawFromSO3 is (float)yaw[k]."""
    x, y = cell_centres(m)
    if cells is not None:
        x, y = x[cells], y[cells]
    q = heading_quaternions(yaws)
    n = len(q)
    s = np.zeros((len(x) * n, 7))
    s[:, 0], s[:, 1] = np.repeat(x, n), np.repeat(y, n)
    s[:, 3:] = np.tile(q, (len(x), 1))
    return s


def heading_quaternions(yaws):
    """[n, 4] quaternions (qx, qy, qz, qw) about z whose getYawFromSO3 is (float)yaw[k]: the rotation by yaw[k] itself, or,
    where that rounds to another float, by (float)yaw[k] (its float can lie past +-pi, where atan2 wraps)."""
    q = np.zeros((len(yaws), 4))
    for k, yaw in enumerate(np.asarray(yaws, np.float64)):
        for a in (yaw, float(np.float32(yaw))):
            q[k] = (0.0, 0.0, np.sin(0.5 * a), np.cos(0.5 * a))
            if so3_yaw(np.concatenate([[0.0, 0.0, 0.0], q[k]])) == np.float32(yaw):
                break
        else:
            raise AssertionError(f"no quaternion about z has getYawFromSO3 == (float){yaw!r}")
    return q


def pack(valid, n: int, shape):
    """Verdict bytes of cell-major poses -> uint32 masks [rows, cols] (column-major), bit k = heading k."""
    v = (np.asarray(valid).reshape(-1, n) != 0).astype(np.uint32)
    bits = (v << np.arange(n, dtype=np.uint32)).sum(axis=1, dtype=np.uint32)
    return bits.reshape(shape, order="F")


def pose_cells(m, seed: int = 0):
    """POSE_CELLS seeded cells (flat column-major indices), the four corners among them."""
    n = m.rows * m.cols
    corners = np.array([0, m.rows - 1, n - m.rows, n - 1])
    rest = np.random.default_rng(seed).choice(n, POSE_CELLS - 4, replace=False)
    return np.concatenate([corners, rest]).astype(np.int64)


def large_map(kind: str):
    """The benchmark's configs[1] map (1000 x 1000 at 0.04 m, seed 2): "gentle" is the metric's fBm (amp 0.6 m), "rough"
    its second roughness level."""
    rough = dict(amp=1.2, wavelength=3.0, persistence=0.7) if kind == "rough" else dict(amp=0.6)
    return synth.make_fbm_map(1000, 1000, 0.04, seed=2, **rough)
