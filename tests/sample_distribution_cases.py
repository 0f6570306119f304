"""Inputs of the sampling-distribution tests: maps, the processors::Basic layers the chain starts from, and roadmap vertex
states (clustered, some off the map, some NaN, some on cell and map edges). Shared by the CPU and GPU tests and by
oracle/make_golden_sample_distribution.py."""
from __future__ import annotations

import dataclasses

import numpy as np

from art_planner_b200 import synth
from oracle import basic_oracle as bo
from oracle import sample_distribution_oracle as sdo


@dataclasses.dataclass
class Case:
    m: synth.SynthMap
    rp: synth.RobotParams
    dp: sdo.DistributionParams
    bp: bo.BasicParams
    traversability: np.ndarray
    observed: np.ndarray
    thr: np.ndarray            # traversability_thresholded (basic_oracle, = the device's processBasic output)
    vertices: np.ndarray       # [n, 7]


def make_vertices(m, n: int, seed: int) -> np.ndarray:
    """Half uniform over the map's extent grown by 10 % (some fall off the map), half in three Gaussian clusters; then
    NaN states, positions on cell edges and on the four map edges (the +x / +y edges are inside, the others outside)."""
    rng = np.random.default_rng(seed)
    lx, ly = m.length
    nu = n // 2
    xy = np.empty((n, 2))
    xy[:nu, 0] = m.cx + rng.uniform(-0.55, 0.55, nu) * lx
    xy[:nu, 1] = m.cy + rng.uniform(-0.55, 0.55, nu) * ly
    centres = np.stack([m.cx + rng.uniform(-0.4, 0.4, 3) * lx, m.cy + rng.uniform(-0.4, 0.4, 3) * ly], 1)
    k = rng.integers(0, 3, n - nu)
    xy[nu:] = centres[k] + rng.normal(0, 0.08, (n - nu, 2)) * np.array([lx, ly])
    s = np.zeros((n, 7))
    s[:, :2] = xy
    s[:, 2] = rng.normal(0, 0.3, n)
    s[:, 6] = 1.0
    s[0:5, 0] = np.nan
    s[5:10, 1] = np.nan
    x0, y0 = m.cx + 0.5 * lx, m.cy + 0.5 * ly
    e = 10
    for r in range(0, min(m.rows, 12)):                      # cell edges along x
        s[e, 0], s[e, 1] = x0 - r * m.res, m.cy
        e += 1
    for x, y in ((x0, m.cy), (m.cx - 0.5 * lx, m.cy), (m.cx, y0), (m.cx, m.cy - 0.5 * ly), (x0, y0)):
        s[e, 0], s[e, 1] = x, y
        e += 1
    return s


def _build(mk, rp, n, seed, bp=bo.BasicParams(), unknown_frac=None) -> Case:
    m = mk()
    trav, obs = synth.make_traversability(m, seed=seed)
    if unknown_frac is not None:                             # larger unobserved patches than make_traversability's
        blk = (np.arange(m.rows)[:, None] // 9) * 4096 + (np.arange(m.cols)[None, :] // 13)
        obs = np.asfortranarray((synth.hash_uniform(seed, 44, blk) > unknown_frac).astype(np.float32))
    _, thr = bo.masked_elevation(m.elevation, trav, obs, m.res, bp)
    dp = sdo.DistributionParams(density_blur_radius=sdo.blur_radius(rp))
    return Case(m, rp, dp, bp, trav, obs, thr, make_vertices(m, n, seed + 1))


CASES = {
    # yaml robot, ksize 73; unknown space traversable with 30 % unobserved: the cap applies
    "fbm_yaml": lambda: _build(lambda: synth.make_fbm_map(120, 100, res=0.04, seed=5), synth.PARAMS_YAML, 3000, 21,
                               bo.BasicParams(unknown_space_untraversable=False), unknown_frac=0.3),
    # header robot, off-origin, non-square, 0.05 m cells: ksize 49
    "offorigin_header": lambda: _build(lambda: synth.make_fbm_map(97, 131, res=0.05, seed=6, cx=3.3, cy=-1.7),
                                       synth.PARAMS_HEADER, 2000, 22),
    # a map smaller than the kernel (41 x 38 against 73 taps): repeated reflection at the border
    "small_yaml": lambda: _build(lambda: synth.make_fbm_map(41, 38, res=0.04, seed=7, cx=-2.0, cy=0.5), synth.PARAMS_YAML,
                                 400, 23, bo.BasicParams(unknown_space_untraversable=False), unknown_frac=0.5),
}
GOLDEN_CASES = ("fbm_yaml", "offorigin_header", "small_yaml")

_cache = {}


def make_case(name: str) -> Case:
    if name not in _cache:
        _cache[name] = CASES[name]()
    return _cache[name]
