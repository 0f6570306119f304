"""GPU parity (-m gpu) of the device PRM roadmap (artp_roadmap_*: PRMMotionCost's sampleGraph / addValidMilestone) against
the restatement oracle/roadmap_oracle.py over the port oracle: structure (kinds, edges, their order, counts, draws used)
exactly, vertex states within 1e-9."""
import dataclasses

import numpy as np
import pytest

import os

import roadmap_cases as rc
import sample_distribution_cases as sdc
from art_planner_b200 import synth
from oracle import orc
from oracle import roadmap_oracle as ro
from oracle import sample_distribution_oracle as sdo

pytestmark = pytest.mark.gpu
STATE_TOL = 1e-9
SEED = 1234


def sampler_params(m):
    """params.yaml:45-51: distribution sampling with the inverse vertex density and the unknown-space cap."""
    return dataclasses.replace(synth.sampler_params_for(m), use_inverse_vertex_density=True, use_max_prob_unknown_samples=True)


def dist_params(rp, sp):
    return sdo.DistributionParams(sp.use_inverse_vertex_density, (rp.torso_length + rp.torso_width) * 0.25,
                                  sp.use_max_prob_unknown_samples, sp.max_prob_unknown_samples)


class Setup:
    def __init__(self, m, rp, thr, observed, layers_seed=7):
        import art_planner_b200 as ap
        self.m, self.rp, self.thr, self.observed = m, rp, thr, observed
        self.chk = ap.StateValidityChecker(rp, device=0)
        self.chk.setMap(m)
        self.chk.updateHeightField()
        self.chk.setSampleFilter(thr, observed)
        self.L = synth.make_sampler_layers(m, seed=layers_seed)
        self.sp = sampler_params(m)
        self.smp = ap.SE3FromSE2Sampler(self.chk, self.L, self.sp, seed=SEED)
        self.o = orc.Oracle(rp, "port")
        self.o.set_map(m)

    def restate(self, rm, caps, first=0, max_draws=1 << 22, layers=None):
        return ro.sample_graph(rm, self.o, self.m, layers or self.L, self.sp, self.rp.reach_z, SEED, first, caps[0], caps[1], caps[2],
                               max_draws, dist_params(self.rp, self.sp), sdo.sample_filter(self.thr, self.rp, self.m.res),
                               self.observed)


def case_setup(name):
    c = sdc.make_case(name)
    return Setup(c.m, c.rp, c.thr, c.observed)


def assert_same(rm_dev, rm_ref):
    st, kinds = rm_dev.vertices()
    edges = rm_dev.edges()
    rst, rkinds, redges = rm_ref.result()
    assert len(kinds) == len(rkinds) and np.array_equal(kinds, rkinds)
    assert np.array_equal(edges, redges)
    assert np.abs(st - rst).max(initial=0.0) <= STATE_TOL


@pytest.mark.parametrize("name", ["fbm_yaml", "offorigin_header"])
def test_sample_graph_matches_restatement(name):
    import art_planner_b200 as ap
    s = case_setup(name)
    caps = (600, 2400, 150)
    rm = ap.PRMRoadmap(s.chk, 8000, 20000)
    used = rm.sampleGraph(s.smp, *caps, max_draws=1 << 22)
    ref = ro.Roadmap()
    r_used, draws, recomputes = s.restate(ref, caps)
    assert used == r_used == draws[-1] + 1
    assert len(recomputes) >= 3
    assert_same(rm, ref)
    nv, ne = rm.counts()
    assert (nv >= caps[0] or ne >= caps[1]) and ref.V == nv and ref.E == ne
    st, kinds = rm.vertices()
    assert (kinds == ro.INTERPOLATED).any() and (kinds == ro.MILESTONE).sum() == len(draws)
    # incremental copy-out: the tails since a cursor
    st2, k2 = rm.vertices(first=nv // 2)
    assert np.array_equal(st2, st[nv // 2:]) and np.array_equal(k2, kinds[nv // 2:])
    assert np.array_equal(rm.edges(first=ne - 7), rm.edges()[ne - 7:])
    assert rm.vertices(first=nv)[0].shape == (0, 7)
    # start / goal milestones on the existing roadmap (baseSolve, :451-479), then more sampling on top: the sampler goes on
    # with the distribution of the last recompute, and the first milestone recomputes it (V / 150 > 0 recomputes so far)
    q = st[kinds == ro.MILESTONE][[3, 11]] + np.array([0.013, -0.021, 0, 0, 0, 0, 0])
    rm.addValidMilestones(q)
    for x in q:
        ref.add_milestone(x, ro.validity(s.o), ro.MILESTONE | ro.QUERY)
    assert_same(rm, ref)
    caps2 = (nv + 150, ne + 2000, 150)
    used2 = rm.sampleGraph(s.smp, *caps2, max_draws=1 << 22, first_sample=used)
    r_used2, _, _ = s.restate(ref, caps2, first=used, layers=ref.layers)
    assert used2 == r_used2
    assert_same(rm, ref)


def test_draw_budget_and_no_distribution():
    import art_planner_b200 as ap
    s = case_setup("fbm_yaml")
    rm = ap.PRMRoadmap(s.chk, 8000, 20000)
    used = rm.sampleGraph(s.smp, 5000, 50000, 100, max_draws=900)
    assert used == 900                                        # the budget ends the loop
    ref = ro.Roadmap()
    r_used, _, rec = ro.sample_graph(ref, s.o, s.m, s.L, s.sp, s.rp.reach_z, SEED, 0, 5000, 50000, 100, 900,
                                     dist_params(s.rp, s.sp), sdo.sample_filter(s.thr, s.rp, s.m.res), s.observed)
    assert r_used == 900 and len(rec) >= 1
    assert_same(rm, ref)
    # no distribution parameters: the sampler's layers stay as they are
    s2 = case_setup("offorigin_header")
    rm2 = ap.PRMRoadmap(s2.chk, 8000, 20000)
    used2 = rm2.sampleGraph(s2.smp, 300, 5000, 100, distribution=False)
    ref2 = ro.Roadmap()
    r_used2, _, _ = ro.sample_graph(ref2, s2.o, s2.m, s2.L, s2.sp, s2.rp.reach_z, SEED, 0, 300, 5000, 100, 1 << 26)
    assert used2 == r_used2
    assert_same(rm2, ref2)


def test_errors_and_launch_accounting():
    import art_planner_b200 as ap
    from art_planner_b200 import capi
    s = case_setup("fbm_yaml")
    h = s.chk.handle
    st = h.stats()
    rm = ap.PRMRoadmap(s.chk, 200, 400)
    # the store fills: ARTP_E_LIMIT, and the roadmap keeps the milestones that fitted
    with pytest.raises(capi.ArtpError) as e:
        rm.sampleGraph(s.smp, 10000, 50000, 1000)
    assert e.value.code == capi.ARTP_E_LIMIT
    nv, ne = rm.counts()
    assert 0 < nv <= 200 and ne <= 400
    ref = ro.Roadmap()
    _, kinds = rm.vertices()
    for x in rm.vertices()[0][kinds == ro.MILESTONE]:
        ref.add_milestone(x, ro.validity(s.o))
    assert_same(rm, ref)
    # launch accounting: last_launches = the kernels of the call
    rm.clear()
    before = h.stats()["kernel_launches"]
    rm.sampleGraph(s.smp, 50, 5000, 20)
    after = h.stats()
    assert after["last_launches"] == after["kernel_launches"] - before > 0
    before = after["kernel_launches"]
    rm.addValidMilestones(rm.vertices()[0][:2])
    after = h.stats()
    assert after["last_launches"] == after["kernel_launches"] - before == 6
    rm.vertices()
    assert h.stats()["last_launches"] == 0
    # cursors past the end, bad capacities
    lib = h.lib
    assert lib.artp_roadmap_get(h.h, 10 ** 6, None, None, 0, None, None, None) == capi.ARTP_E_INVALID
    assert lib.artp_roadmap_clear(h.h, 0, 10) == capi.ARTP_E_INVALID
    # no roadmap yet, no sampler, no map, a map window
    c2 = ap.StateValidityChecker(s.rp, device=0)
    p = capi.ArtpRoadmapParams(100, 100, 10, 1000)
    x = np.zeros((1, 7)); x[0, 6] = 1.0
    assert lib.artp_roadmap_add_milestones(c2.handle.h, x.ctypes.data, 1) == capi.ARTP_E_INVALID
    assert lib.artp_roadmap_clear(c2.handle.h, 100, 100) == 0
    assert lib.artp_roadmap_add_milestones(c2.handle.h, x.ctypes.data, 1) == capi.ARTP_E_NOMAP
    assert lib.artp_roadmap_sample_graph(c2.handle.h, p, None, 0, 0, None) == capi.ARTP_E_NOMAP
    c2.setMap(s.m)
    c2.updateHeightField()
    assert lib.artp_roadmap_sample_graph(c2.handle.h, p, None, 0, 0, None) == capi.ARTP_E_NOMAP     # no sampler
    c2.updateHeightField(window=(0, 48))
    assert lib.artp_roadmap_add_milestones(c2.handle.h, x.ctypes.data, 1) == capi.ARTP_E_INVALID
    assert lib.artp_roadmap_sample_graph(h.h, None, None, 0, 0, None) == capi.ARTP_E_INVALID
    bad = x.copy(); bad[0, 0] = np.nan
    assert lib.artp_roadmap_add_milestones(h.h, bad.ctypes.data, 1) == capi.ARTP_E_INVALID
    del st


def test_shipped_caps_config1():
    """The shipped caps (10 000 vertices / 50 000 edges, recompute every 1000) on the configs[1] map."""
    import art_planner_b200 as ap
    from oracle import basic_oracle as bo
    m = synth.make_fbm_map(1000, 1000)
    rp = synth.PARAMS_YAML
    trav, obs = synth.make_traversability(m, seed=13)
    _, thr = bo.masked_elevation(m.elevation, trav, obs, m.res, bo.BasicParams())
    s = Setup(m, rp, thr, obs)
    rm = ap.PRMRoadmap(s.chk, 20000, 60000)
    used = rm.sampleGraph(s.smp, 10000, 50000, 1000)
    ref = ro.Roadmap()
    r_used, draws, rec = s.restate(ref, (10000, 50000, 1000), max_draws=1 << 26)
    assert used == r_used and len(rec) >= 9
    assert_same(rm, ref)


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "roadmap.npz"))


@pytest.mark.parametrize("name", list(rc.CASES))
def test_sample_graph_matches_golden_and_offgrid(name, golden):
    """The device against the compiled reference's golden (gentle map with -inf patches, rough fBm), and against the
    restatement on offgrid_cases' off-origin, non-square r1 map."""
    import art_planner_b200 as ap
    c = rc.make_case(name)
    chk = ap.StateValidityChecker(c.rp, device=0)
    chk.setMap(c.m)
    chk.updateHeightField()
    chk.setSampleFilter(c.thr, c.observed)
    smp = ap.SE3FromSE2Sampler(chk, c.layers, c.sp, seed=rc.SEED)
    rm = ap.PRMRoadmap(chk, 8000, 20000)
    used = rm.sampleGraph(smp, *rc.CAPS, max_draws=rc.MAX_DRAWS)
    st, kinds = rm.vertices()
    edges = rm.edges()
    if name in rc.GOLDEN_CASES:
        assert used == golden[name + "/draws_used"][0]
        assert np.array_equal(kinds, golden[name + "/kinds"]) and np.array_equal(edges, golden[name + "/edges"])
        assert np.abs(st - golden[name + "/states"]).max() <= STATE_TOL
    else:
        o = orc.Oracle(c.rp, "port")
        o.set_map(c.m)
        ref = ro.Roadmap()
        r_used, _, rec = ro.sample_graph(ref, o, c.m, c.layers, c.sp, c.rp.reach_z, rc.SEED, 0, *rc.CAPS, rc.MAX_DRAWS, c.dp,
                                         c.sample_filter, c.observed)
        assert used == r_used and len(rec) >= 2
        assert_same(rm, ref)
