"""Seeded start / goal search queries (StartState / GoalStateRegion::sampleGoal, start.cpp:7-41, goal.cpp:11-41), shared
by oracle/make_golden_start_goal.py (generation with the compiled reference) and the tests. Centres are mixed so that
every outcome occurs: a valid centre, a first valid draw at small and large k, no valid draw, a centre outside the map
and boxes at the map border."""
from __future__ import annotations

import numpy as np

import philox_ball_ref
from art_planner_b200 import synth

RADII = np.array([0.2, 0.5, 1.0])


def make_queries(m, n: int, seed: int):
    """(centres [n, 7], radius [n]): terrain poses, most of them moved up or down by up to 12 cm (the search often has to
    move them), some 1 m into the ground (nothing near is valid), some moved off the map or onto its border."""
    k = np.arange(n)
    c = synth.make_terrain_poses(m, n, seed=seed)
    kind = synth.hash_uniform(seed, 20, k)
    lx, ly = m.length
    u = synth.hash_uniform(seed, 21, k)
    side = np.where(synth.hash_uniform(seed, 22, k) < 0.5, -1.0, 1.0)
    shift = kind < 0.7
    c[shift, 2] += 0.24 * u[shift] - 0.12
    deep = (kind >= 0.7) & (kind < 0.8)
    c[deep, 2] -= 1.0
    out = (kind >= 0.8) & (kind < 0.9)
    c[out, 0] = m.cx + side[out] * (0.5 * lx + 0.05 + 0.6 * u[out])
    edge = kind >= 0.9
    c[edge, 1] = m.cy + side[edge] * (0.5 * ly - 0.3 * u[edge])
    radius = RADII[(synth.hash_uniform(seed, 23, k) * len(RADII)).astype(np.int64)]
    return np.ascontiguousarray(c), radius


# (name, map, params, n queries, n_iter, seed); the offsets are draws 0 .. n_iter-1 of the "ARTB" stream under `seed`
GOLDEN_CASES = [
    ("sg_fixture_yaml", "fixture", "yaml", 60, 300, 101),
    ("sg_fixture_header", "fixture", "header", 60, 300, 102),
    ("sg_terraces_yaml", "terraces", "yaml", 60, 300, 103),
    ("sg_terraces_header", "terraces", "header", 60, 300, 104),
    ("sg_spikes_yaml", "spikes", "yaml", 60, 300, 105),
    ("sg_spikes_header", "spikes", "header", 60, 300, 106),
    ("sg_fbm_rough_yaml", "fbm_rough", "yaml", 60, 300, 107),
    ("sg_fbm_rough_header", "fbm_rough", "header", 60, 300, 108),
]


def golden_inputs(m, n: int, n_iter: int, seed: int):
    centres, radius = make_queries(m, n, seed)
    return centres, radius, philox_ball_ref.ball_offsets(seed, 0, n, n_iter, radius)
