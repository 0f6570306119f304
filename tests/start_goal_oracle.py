"""Test-only CPU restatements for the start / goal search and the goal projection, on top of the pose oracle
(oracle/orc.py: the C port or the reference's own compiled ODE).

find_valid_near  StartState / GoalStateRegion::sampleGoal (start.cpp:7-41, goal.cpp:11-41): isValid on the centre, then
                 on the centre moved in x / y by each offset, in order, stopping at the first valid candidate. isValid is
                 a pure function of the state, so the candidates are handed to the oracle's isValid in short ordered
                 runs and the walk stops at the run that holds the first valid one: the answer is the serial loop's.
pose_from_2d     Planner::plan's goal projection (planner.cpp:223-237): grid_map isInside / getIndexFromPosition,
                 Map::get3DPoseFrom2D (map.cpp:77-90) with Eigen's quaternion rotation order, setSO3FromRPY
                 (utils.h:101-115), in numpy doubles.
"""
from __future__ import annotations

import numpy as np

RUN = 32   # candidates per isValid call after the centre


def find_valid_near(oracle, centres, n_iter: int, offsets):
    """centres [n, 7], offsets [n, n_iter, 2] -> (states [n, 7], index int32 [n]); -1 and the last candidate when no
    candidate is valid."""
    c = np.ascontiguousarray(centres, dtype=np.float64).reshape(-1, 7)
    n = c.shape[0]
    off = np.asarray(offsets, dtype=np.float64).reshape(n, int(n_iter), 2)
    out = c.copy()
    idx = np.full(n, -1, np.int32)
    for q in range(n):
        if oracle.check_poses(c[q:q + 1])[0]:
            idx[q] = 0
            continue
        for k0 in range(0, n_iter, RUN):
            k1 = min(n_iter, k0 + RUN)
            cand = np.repeat(c[q:q + 1], k1 - k0, axis=0)
            cand[:, 0] = c[q, 0] + off[q, k0:k1, 0]
            cand[:, 1] = c[q, 1] + off[q, k0:k1, 1]
            v = np.nonzero(oracle.check_poses(cand))[0]
            if len(v):
                idx[q] = k0 + v[0] + 1
                out[q] = cand[v[0]]
                break
        else:
            if n_iter:
                out[q, 0] = c[q, 0] + off[q, n_iter - 1, 0]
                out[q, 1] = c[q, 1] + off[q, n_iter - 1, 1]
    return out, idx


def _cross(a, b):
    return np.stack([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def pose_from_2d(m, layers, states):
    """states [n, 7] -> (states [n, 7], inside uint8 [n]); layers carries normal_x / normal_y / normal_z (grid_map
    matrices). States off the map are copied unchanged."""
    s = np.ascontiguousarray(states, dtype=np.float64).reshape(-1, 7)
    out = s.copy()
    Lx, Ly = m.rows * m.res, m.cols * m.res
    x, y = s[:, 0], s[:, 1]
    # grid_map getIndexFromPosition + checkIfPositionWithinMap
    with np.errstate(invalid="ignore"):
        row = np.trunc(-(((x - 0.5 * Lx) - m.cx) / m.res))
        col = np.trunc(-(((y - 0.5 * Ly) - m.cy) / m.res))
    tx, ty = -((x - m.cx) - 0.5 * Lx), -((y - m.cy) - 0.5 * Ly)
    inside = (tx >= 0.0) & (ty >= 0.0) & (tx < Lx) & (ty < Ly) & (row >= 0) & (col >= 0) & (row < m.rows) & (col < m.cols)
    i, j = row[inside].astype(np.int64), col[inside].astype(np.int64)
    si = s[inside]
    nw = np.stack([np.asarray(layers.normal_x, np.float32)[i, j], np.asarray(layers.normal_y, np.float32)[i, j],
                   np.asarray(layers.normal_z, np.float32)[i, j]]).astype(np.float64)
    qx, qy, qz, qw = si[:, 3], si[:, 4], si[:, 5], si[:, 6]
    yaw = np.arctan2(2 * (qw * qz + qx * qy), 1 - 2 * (qy * qy + qz * qz)).astype(np.float32).astype(np.float64)
    # Quaterniond(AngleAxisd(yaw, UnitZ)).inverse() * normal_w, Eigen's order
    sn, cs = np.sin(0.5 * yaw), np.cos(0.5 * yaw)
    q = np.stack([sn * 0.0, sn * 0.0, sn * 1.0, cs])
    n2 = (q[0] * q[0] + q[2] * q[2]) + (q[1] * q[1] + q[3] * q[3])
    qi, qwi = np.stack([-q[0] / n2, -q[1] / n2, -q[2] / n2]), q[3] / n2
    uv = _cross(qi, nw)
    uv = uv + uv
    nb = (nw + qwi * uv) + _cross(qi, uv)
    roll, pitch = -np.arctan2(nb[1], nb[2]), np.arctan2(nb[0], nb[2])
    cr, sr = np.cos(roll * 0.5), np.sin(roll * 0.5)
    cp, sp = np.cos(pitch * 0.5), np.sin(pitch * 0.5)
    cy, sy = np.cos(yaw * 0.5), np.sin(yaw * 0.5)
    o = out[inside]
    o[:, 2] = np.asarray(m.elevation, np.float32)[i, j].astype(np.float64)
    o[:, 6] = cy * cp * cr + sy * sp * sr
    o[:, 3] = cy * cp * sr - sy * sp * cr
    o[:, 4] = sy * cp * sr + cy * sp * cr
    o[:, 5] = sy * cp * cr - cy * sp * sr
    out[inside] = o
    return out, inside.astype(np.uint8)
