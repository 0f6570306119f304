"""Inputs of the roadmap golden (oracle/make_golden_roadmap.py) and the CPU test that reads it: two small maps -- gentle
fBm with untraversable (-inf) patches, and rough fBm -- with the processors::Basic layers, the sampler's layers and
parameters, and scaled sampleGraph caps; plus an off-origin, non-square map of tests/offgrid_cases.py (the shipped 10 000 / 50 000 / 1000 cut by about 7)."""
from __future__ import annotations

import dataclasses

import offgrid_cases as og
from art_planner_b200 import synth
from oracle import basic_oracle as bo
from oracle import sample_distribution_oracle as sdo

SEED = 4321
CAPS = (1500, 6000, 300)         # max_n_vertices, max_n_edges, recompute_density_after_n_samples
MAX_DRAWS = 1 << 22


@dataclasses.dataclass
class Case:
    m: synth.SynthMap
    rp: synth.RobotParams
    layers: synth.SamplerLayers
    sp: synth.SamplerParams
    dp: sdo.DistributionParams
    thr: object                # traversability_thresholded (basic_oracle)
    sample_filter: object
    observed: object


def _build(m, rp) -> Case:
    trav, obs = synth.make_traversability(m, seed=13)
    _, thr = bo.masked_elevation(m.elevation, trav, obs, m.res, bo.BasicParams())
    sp = dataclasses.replace(synth.sampler_params_for(m), use_inverse_vertex_density=True, use_max_prob_unknown_samples=True)
    dp = sdo.DistributionParams(True, (rp.torso_length + rp.torso_width) * 0.25, True, sp.max_prob_unknown_samples)
    return Case(m, rp, synth.make_sampler_layers(m, seed=7), sp, dp, thr, sdo.sample_filter(thr, rp, m.res), obs)


CASES = {
    # offgrid_cases' r1 map: 201 x 199, centred at (137.37, -52.81); not in the golden
    "offgrid_r1": lambda: _build(og.MAPS["r1"](), synth.PARAMS_HEADER),
    "gentle_inf": lambda: _build(synth.make_fbm_map(150, 140, res=0.04, seed=11, blob_frac=0.05), synth.PARAMS_YAML),
    "rough_fbm": lambda: _build(synth.make_fbm_map(140, 150, res=0.04, seed=12, amp=1.2, wavelength=3.0, persistence=0.7),
                                synth.PARAMS_YAML),
}

GOLDEN_CASES = ("gentle_inf", "rough_fbm")

_cache = {}


def make_case(name: str) -> Case:
    if name not in _cache:
        _cache[name] = CASES[name]()
    return _cache[name]
