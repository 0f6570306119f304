"""Roadmaps for the search tests (tests/test_roadmap_search_*.py): milestone sets whose vertex count, geometry and ties
are known in advance.

  lattice   a square grid of milestones 2^-10 m apart, all facing +x, on a flat map. Every coordinate difference is exact,
            so distances and (away from the map border) learned weights tie between translated copies of an edge. The
            whole grid fits in a 0.28 m square: no connection reaches the 0.5 m lateral step, every connection is one edge
            and V is the number of milestones exactly.
  corridor  one serpentine corridor between 0.5 m wall ridges on a flat map, milestones along its centreline. The yaw
            turns 3 rad per metre of corridor, so that a motion between neighbours spans several validation states.
            The milestones go in in shuffled blocks of CORRIDOR_BLOCK along the corridor: vertex index and position
            disagree, while every milestone's nearest neighbours at insertion lie close behind it along the corridor.
            A fully shuffled order would connect the first milestones over metres, through interpolated chains that
            fill the store; in block order an edge spans at most about k + CORRIDOR_BLOCK spacings (k = 46 at the
            capacity), and the fewest-edges path of CORRIDOR_N milestones measures 2 205 hops, about n / 35.
The port oracle decides validity; tests/test_roadmap_search_cpu.py checks these claims without a GPU."""
from __future__ import annotations

import math

import numpy as np

import roadmap_cases as rc
from art_planner_b200 import synth
from oracle import roadmap_oracle as ro

LATTICE_H = 2.0 ** -10           # lattice spacing (m)
LATTICE_SIDE = 279               # columns: 279^2 >= 77 438
SEARCH_VERTEX_LIMIT = 77440      # the search's on-chip vertex capacity (include/artp.h)
RP = synth.PARAMS_YAML

# corridor: lanes along x, joined by U-turns at alternating ends
LANES, LANE_X, LANE_PITCH, HALF_WIDTH = 6, 4.0, 2.1, 0.9
WALL_HEIGHT = 0.5
YAW_RATE = 3.0                   # rad per metre of centreline
CORRIDOR_BLOCK = 8
CORRIDOR_N = SEARCH_VERTEX_LIMIT - 4   # centreline milestones: two queries bring V to the search's capacity
REMOVAL_N = 600                  # the sparse corridor of the removal test (interpolated chains, dead ends across walls)
OBSTACLE_LANE = 2                # the lane the second map blocks


def pose(x, y, yaw=0.0, z=0.0):
    """[n, 7] states at body height z (valid on a flat map at height 0)."""
    x, y, yaw = np.broadcast_arrays(np.asarray(x, np.float64), np.asarray(y, np.float64), np.asarray(yaw, np.float64))
    qx, qy, qz, qw = synth.quat_from_rpy(np.zeros(x.shape), np.zeros(x.shape), yaw)
    return np.ascontiguousarray(np.stack([x, y, np.full(x.shape, z), qx, qy, qz, qw], axis=-1).reshape(-1, 7))


# ---- lattice -----------------------------------------------------------------------------------------------------------
def flat_case():
    """A flat 4 m map: the lattice sits in its middle, far from the border."""
    return rc._build(synth.make_flat_map(100, 100, res=0.04), RP)


def lattice_cells(n: int):
    """(i, j) grid indices of the first n lattice points, row by row."""
    k = np.arange(n)
    return k // LATTICE_SIDE, k % LATTICE_SIDE


def lattice_states(n: int, seed: int = 0):
    """n lattice milestones in a shuffled order (seeded), and the permutation: row r is lattice point perm[r]."""
    perm = np.random.default_rng(seed).permutation(n)
    i, j = lattice_cells(n)
    return pose(i[perm] * LATTICE_H, j[perm] * LATTICE_H), perm


def lattice_query(rows: int, a=(0, 0), b=None):
    """Start and goal between lattice points (half a spacing off in x and y, exact), at cells a and b of the first
    `rows` full rows."""
    b = b if b is not None else (rows - 2, LATTICE_SIDE - 2)
    st = pose([(a[0] + 0.5) * LATTICE_H, (b[0] + 0.5) * LATTICE_H], [(a[1] + 0.5) * LATTICE_H, (b[1] + 0.5) * LATTICE_H])
    return st[0], st[1]


def edges_added(n_before: int, n_new: int) -> int:
    """Edges that n_new milestones add to a roadmap of n_before vertices when no connection is interpolated."""
    return sum(min(ro.k_star(v + 1), v) for v in range(n_before, n_before + n_new))


# ---- corridor ----------------------------------------------------------------------------------------------------------
def lane_y(k):
    return -0.5 * (LANES - 1) * LANE_PITCH + k * LANE_PITCH


def corridor_length() -> float:
    return LANES * 2 * LANE_X + (LANES - 1) * LANE_PITCH


def centreline(p):
    """(x, y) of the centreline at arc length p: lane 0 from x = -LANE_X to +LANE_X, up the U-turn, lane 1 back, ..."""
    p = np.asarray(p, np.float64)
    seg = 2 * LANE_X + LANE_PITCH
    k = np.minimum((p // seg).astype(np.int64), LANES - 1)
    q = p - k * seg
    sign = np.where(k % 2 == 0, 1.0, -1.0)
    in_lane = q <= 2 * LANE_X
    x = np.where(in_lane, sign * (q - LANE_X), sign * LANE_X)
    y = np.where(in_lane, lane_y(k), lane_y(k) + (q - 2 * LANE_X))
    return x, y


def corridor_map(obstacle_lane=None):
    """A flat 14 m map at height 0 with everything outside the corridor raised by WALL_HEIGHT; with obstacle_lane, a
    0.3 m ridge across that lane's middle as well."""
    m = synth.make_flat_map(350, 350, res=0.04)
    x, y = m.cell_xy()
    X, Y = x[:, None], y[None, :]
    free = np.zeros(m.elevation.shape, bool)
    for k in range(LANES):
        free |= (np.abs(Y - lane_y(k)) <= HALF_WIDTH) & (np.abs(X) <= LANE_X + HALF_WIDTH)
        if k + 1 < LANES:
            xe = LANE_X if k % 2 == 0 else -LANE_X
            free |= (np.abs(X - xe) <= HALF_WIDTH) & (Y >= lane_y(k)) & (Y <= lane_y(k + 1))
    if obstacle_lane is not None:
        free &= ~((np.abs(Y - lane_y(obstacle_lane)) <= HALF_WIDTH + 0.05) & (np.abs(X) <= 0.15))
    e = np.asfortranarray(np.where(free, 0.0, WALL_HEIGHT).astype(np.float32))
    return synth.SynthMap(e, e.copy(order="F"), m.res, m.cx, m.cy, f"serpentine corridor, obstacle lane {obstacle_lane}")


def corridor_case(obstacle_lane=None):
    return rc._build(corridor_map(obstacle_lane), RP)


def corridor_states(n: int, seed: int = 0):
    """n centreline milestones strictly inside the corridor's ends (arc length, then the states in insertion order: shuffled
    within blocks of CORRIDOR_BLOCK), and the start and goal at the two ends. At CORRIDOR_N the spacing is 0.76 mm and
    every connection direct; at REMOVAL_N it is 9.7 cm and the longer connections become chains of interpolated
    vertices, cut short where they enter a wall."""
    L = corridor_length()
    p = (np.arange(n) + 1.0) * (L / (n + 1))
    rng = np.random.default_rng(seed)
    order = np.concatenate([b0 + rng.permutation(min(CORRIDOR_BLOCK, n - b0)) for b0 in range(0, n, CORRIDOR_BLOCK)])
    p = p[order]
    st = pose(*centreline(p), YAW_RATE * p)
    ends = pose(*centreline(np.array([0.0, L])), YAW_RATE * np.array([0.0, L]))
    return p, st, ends[0], ends[1]


def wall_states():
    """Poses centred on the walls between lanes, at several yaws."""
    x = np.linspace(-LANE_X + 1.0, LANE_X - 1.0, 5)
    out = []
    for k in range(LANES - 1):
        yw = 0.5 * (lane_y(k) + lane_y(k + 1))
        for yaw in (0.0, 0.7, math.pi / 2):
            out.append(pose(x, np.full(x.shape, yw), yaw))
    return np.concatenate(out)
