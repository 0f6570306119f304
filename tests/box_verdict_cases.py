"""Seeded cases of the box verdicts (artp_box_verdicts), shared by oracle/make_golden_box_verdicts.py and the tests: every
map of tests/cases.py under both robot geometries and both values of unknown_space_untraversable, each with samples on
the terrain, samples past the map edge and samples built so that the torso and several reach boxes fail together."""
from __future__ import annotations

import dataclasses

import numpy as np

import cases
from art_planner_b200 import synth

N_TERRAIN, N_EDGE, N_COMBO = 600, 300, 600

# (name, map, params, unknown_space_untraversable)
CASES = [(f"bv_{mk}_{pk}_u{u}", mk, pk, u) for mk in sorted(cases.MAPS) for pk in ("yaml", "header") for u in (1, 0)]


def params(pk: str, unknown: int):
    return dataclasses.replace(cases.PARAMS[pk], unknown_space_untraversable=bool(unknown))


def samples(m, seed: int = 5) -> np.ndarray:
    """[N_TERRAIN + N_EDGE + N_COMBO, 7] states of map m."""
    terrain = synth.make_terrain_poses(m, N_TERRAIN, seed=seed, z_range=0.08)   # mostly valid: the queues' paths
    # centres up to 1 m past every edge: single reach boxes, then the torso, leave the map
    k = np.arange(N_EDGE)
    lx, ly = m.length
    x = m.cx + (synth.hash_uniform(seed, 21, k) - 0.5) * (lx + 2.0)
    y = m.cy + (synth.hash_uniform(seed, 22, k) - 0.5) * (ly + 2.0)
    edge = synth.make_terrain_poses(m, N_EDGE, seed=seed + 1, z_range=0.08, xy=(x, y))
    # several boxes at once: the body from 0.5 m below to 0.6 m above the terrain (torso in the ground, feet in the air),
    # and rolls / pitches up to 0.6 / 0.4 rad that lift single feet off the ground
    combo = synth.make_terrain_poses(m, N_COMBO, seed=seed + 2, z_range=0.0, roll_pert=0.6, pitch_pert=0.4)
    combo[:, 2] += -0.5 + 1.1 * synth.hash_uniform(seed, 23, np.arange(N_COMBO))
    return np.ascontiguousarray(np.concatenate([terrain, edge, combo]))


def lowest_fail(why: np.ndarray) -> np.ndarray:
    """The box at which isValid's && chain stops (torso, then the reach boxes in order), -1 for a valid state."""
    fails = (why[:, None] >> np.arange(5, dtype=np.uint16)) & 1
    return np.where(fails.any(axis=1), np.argmax(fails, axis=1), -1)
