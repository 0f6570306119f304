"""Seeded map geometries off the usual grid (oracle/make_golden_offgrid.py, tests/test_offgrid_*.py).

Every other parity case uses rows that are a multiple of 4, 0.04 / 0.05 m cells, a square map and a map centred at the
origin. The device code depends on exactly those properties in several places: the padded pitch (rows + 3) & ~3 of the
layers and range tables, the table levels kmax and the classify stage's window paths, the tile configuration, the map
position in the float box frame and in the sampler / normals / goal projection, and the rows-vs-cols order of every
layer walk. These cases vary each of them: rows = 1, 2, 3 mod 4, non-square maps, 0.025 to 0.2 m cells, centres far
from the origin, negative heights, maps smaller than a robot and maps two vertices wide.

The inputs are a pure function of the seeds below: cases.py is not touched (its inputs are hashed into the older goldens).
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

from art_planner_b200 import synth

PARAMS = {"yaml": synth.PARAMS_YAML, "header": synth.PARAMS_HEADER,
          # a long, narrow torso: zones of up to ~67 x 7 vertices at 0.04 m, whose window count along the long side
          # (cx * cz > 32) sends them to the exact reduction (REC_NEEDS_REDUCE) -- no robot preset has such zones
          "rail": dataclasses.replace(synth.PARAMS_YAML, torso_length=2.6, torso_width=0.12, torso_height=0.2)}


def _shift(m, dz):
    e = np.asfortranarray(m.elevation + np.float32(dz))
    k = np.asfortranarray(m.elevation_masked + np.float32(dz))          # -inf stays -inf
    return dataclasses.replace(m, elevation=e, elevation_masked=k, desc=m.desc + f" shifted by {dz} m")


def terraces(rows, cols, res=0.04):
    """The cases.terraces recipe (piecewise-constant steps: mergeable planes everywhere) at any size."""
    m = synth.make_flat_map(rows, cols, res)
    r, c = np.indices((rows, cols))
    e = np.asfortranarray((0.07 * ((r // 9) % 4) + 0.05 * ((c // 13) % 3)).astype(np.float32))
    return dataclasses.replace(m, elevation=e, elevation_masked=e.copy(order="F"), desc=f"terraces {rows}x{cols}@{res}")


MAPS = {
    "r3": lambda: synth.make_fbm_map(203, 157, 0.04, seed=41),
    "r1": lambda: synth.make_fbm_map(201, 199, 0.04, seed=42, cx=137.37, cy=-52.81),
    "far": lambda: _shift(synth.make_fbm_map(202, 206, 0.04, seed=43, cx=1024.51, cy=-2047.77), -40.0),
    "coarse": lambda: synth.make_fbm_map(150, 97, 0.1, seed=44),
    "coarser": lambda: synth.make_fbm_map(61, 43, 0.2, seed=45, cx=3.3, cy=-1.7),
    "fine": lambda: synth.make_fbm_map(330, 290, 0.025, seed=46),
    "terr": lambda: terraces(203, 157),
    "tiny_h": lambda: synth.make_fbm_map(27, 23, 0.04, seed=47),
    "tiny_y": lambda: synth.make_fbm_map(41, 38, 0.04, seed=48),
    "thin_r": lambda: synth.make_fbm_map(2, 300, 0.04, seed=49),
    "thin_c": lambda: synth.make_fbm_map(300, 2, 0.04, seed=50),
}

#: maps whose poses must be a healthy mix of valid and invalid (the tiny and thin maps are exempt)
MIXED = ("r3", "r1", "far", "coarse", "coarser", "fine", "terr")

N_TERRAIN, N_FLAT = 7000, 2000


def poses(m, seed, tiny=False):
    """make_terrain_poses (inside the map) + a make_flat_poses share reaching 0.3 m past the border (outside-map rules),
    its z around the map's median height. On maps smaller than the robot the terrain poses stay within 0.12 m of the
    centre, so that the feet land on the map and some poses are valid."""
    xy = None
    if tiny:
        k = np.arange(N_TERRAIN)
        xy = (m.cx + (synth.hash_uniform(seed, 7, k) - 0.5) * 0.24, m.cy + (synth.hash_uniform(seed, 8, k) - 0.5) * 0.24)
    t = synth.make_terrain_poses(m, N_TERRAIN, seed=seed, xy=xy)
    f = synth.make_flat_poses(m, N_FLAT, seed=seed + 1, margin=0.3)
    f[:, 2] += float(np.median(m.elevation))
    return np.concatenate([t, f])


def case_poses(m, mk, seed):
    return poses(m, seed, tiny=mk.startswith("tiny"))


def _pose_cases():
    out = []
    for i, mk in enumerate(MAPS):
        pks = {"tiny_h": ("header",), "tiny_y": ("yaml",)}.get(mk, ("yaml", "header"))
        for pk in pks:
            out.append((f"{mk}_{pk}", mk, pk, 100 + 2 * i))
    out.append(("r3_rail", "r3", "rail", 130))
    return out


#: (name, map, preset, pose seed)
POSE_CASES = _pose_cases()

#: box-level hits, both kinds of the yaml boxes: (map, seed, tilt, z range)
BOX_CASES = [(mk, 200 + i, 0.6, 0.35) for i, mk in enumerate(MAPS)]
BOX_N = 4000

#: edge cases on r3, coarse and far (yaml): check_motions (n, n_steps, seed), edge interiors (n, seed, dmin, dmax),
#: segment counts / lastValid (n, seed, dmin, dmax)
EDGE_MAPS = ("r3", "coarse", "far")
EDGES = (2000, 9, 301)
INTERIORS = (2000, 302, 0.05, 3.0)
SEGMENTS = (1500, 303, 0.05, 2.0)


def se3_bounds(m, reach_z):
    """RealVectorBounds of the SE3 space as Planner::setMap sets them (planner.cpp:146-156)."""
    lx, ly = m.length
    e = m.elevation[np.isfinite(m.elevation)]
    return ([m.cx - lx, m.cy - ly, float(e.min()) - reach_z / 2], [m.cx + lx, m.cy + ly, float(e.max()) + reach_z / 2])


# ---------------------------------------------------------------------------------------------------------------------
# The classify stage's path choice, restated (artp_kernels.cuh zone_classify, artp_map.cu artp_set_map_window)
# ---------------------------------------------------------------------------------------------------------------------
K_MAX_LEVEL = 6


def table_kmax(m, p):
    """kmax of the torso (0) and reach (1) tables as artp_set_map_window derives them from the box half-diagonal."""
    out = []
    iW = 1.0 / (np.float32(m.rows * m.res) / np.float32(m.rows - 1.0))
    iD = 1.0 / (np.float32(m.cols * m.res) / np.float32(m.cols - 1.0))
    for sd in ((p.torso_length, p.torso_width, p.torso_height), (p.reach_x, p.reach_y, p.reach_z)):
        r = 0.5 * math.sqrt(sum(float(np.float32(s)) ** 2 for s in sd))
        nxm = min(m.rows, math.ceil(2.0 * r * iW) + 4)
        nzm = min(m.cols, math.ceil(2.0 * r * iD) + 4)
        kk = 0
        while (2 << kk) <= min(nxm, nzm) and kk < K_MAX_LEVEL:
            kk += 1
        out.append(kk)
    return out


def zone_paths(m, p, states):
    """Per (pose, box) the path zone_classify takes, for every box whose centre lies on the map and whose AABB meets it:
    'words8' (one 8-word request), 'loop' (cx * cz > 8 windows), 'kk<1', 'kk>kmax', 'cxcz>32' (the three causes of
    REC_NEEDS_REDUCE); the zone restated in float64 (near a cell border it may be one vertex off, which only moves a
    count). Returns a dict name -> number of boxes."""
    s = np.asarray(states, np.float64)
    t = s[:, :3]
    x, y, z, w = (s[:, i] for i in range(3, 7))
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                  2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                  2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    lx, ly = m.length
    sW, sD = lx / (m.rows - 1), ly / (m.cols - 1)
    kmax = table_kmax(m, p)
    counts = dict.fromkeys(("words8", "loop", "kk<1", "kk>kmax", "cxcz>32"), 0)
    for k in range(5):
        if k == 0:
            off, side = (p.torso_off_x, p.torso_off_y, p.torso_off_z), (p.torso_length, p.torso_width, p.torso_height)
        else:
            fk = k - 1
            off = (-p.feet_off_x if fk & 2 else p.feet_off_x, -p.feet_off_y if fk & 1 else p.feet_off_y, 0.0)
            side = (p.reach_x, p.reach_y, p.reach_z)
        c = np.einsum("nij,j->ni", R, np.array(off)) + t
        sd = np.array(side)
        xr = 0.5 * (np.abs(R[:, 0, :]) * sd).sum(1)
        wr = 0.5 * (np.abs(R[:, 1, :]) * sd).sum(1)
        P0 = -(c[:, 0] - m.cx) + 0.5 * lx
        P2 = (c[:, 1] - m.cy) + 0.5 * ly
        on = (P0 >= 0) & (P0 <= lx) & (P2 >= 0) & (P2 <= ly)          # grid_map isInside of the box centre
        x0 = np.maximum(np.floor((P0 - xr) / sW), 0)
        x1 = np.minimum(np.ceil((P0 + xr) / sW), m.rows - 1)
        z0 = np.maximum(np.floor((P2 - wr) / sD), 0)
        z1 = np.minimum(np.ceil((P2 + wr) / sD), m.cols - 1)
        nX, nZ = (x1 - x0 + 1)[on].astype(np.int64), (z1 - z0 + 1)[on].astype(np.int64)
        mn = np.maximum(np.minimum(nX, nZ), 1)
        kk = np.floor(np.log2(mn)).astype(np.int64)
        cx = (nX + (1 << kk) - 1) >> kk
        cz = (nZ + (1 << kk) - 1) >> kk
        km = kmax[0 if k == 0 else 1]
        counts["kk<1"] += int((kk < 1).sum())
        counts["kk>kmax"] += int((kk > km).sum())
        counts["cxcz>32"] += int(((kk >= 1) & (kk <= km) & (cx * cz > 32)).sum())
        ok = (kk >= 1) & (kk <= km) & (cx * cz <= 32)
        counts["words8"] += int((ok & (cx * cz <= 8)).sum())
        counts["loop"] += int((ok & (cx * cz > 8)).sum())
    return counts
