"""GPU parity (-m gpu) of the sampler's distribution chain (artp_set_sample_filter, artp_update_sample_distribution[_device])
against the restatement oracle/sample_distribution_oracle.py, bit for bit, and against the cv2-made golden layers."""
import copy
import dataclasses
import os

import numpy as np
import pytest

import philox_ref
import sample_distribution_cases as sdc
from art_planner_b200 import synth
from oracle import sample_distribution_oracle as sdo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLUR_TOL = 2e-6


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def same(a, b):
    """Bit-equal float32 layers (NaN where the other is NaN)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(b)
    return a.shape == b.shape and np.array_equal(np.isnan(a), nan) and np.array_equal(bits(a[~nan]), bits(b[~nan]))


def checker(m, rp):
    import art_planner_b200 as ap
    chk = ap.StateValidityChecker(rp, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    return chk


def yaml_sampler_params(m):
    """params.yaml:45-51: distribution sampling with the inverse vertex density and the unknown-space cap."""
    return dataclasses.replace(synth.sampler_params_for(m), use_inverse_vertex_density=True, use_max_prob_unknown_samples=True)


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "sample_distribution.npz"))


@pytest.mark.parametrize("name", list(sdc.CASES))
def test_layers_match_restatement_and_golden(name, golden, port_lib):
    c = sdc.make_case(name)
    chk = checker(c.m, c.rp)
    filt = chk.setSampleFilter(c.thr, c.observed)
    rfilt = sdo.sample_filter(c.thr, c.rp, c.m.res)
    assert same(filt, rfilt)
    prob, cum, row = chk.updateSampleDistribution(c.vertices, c.dp)
    ref = sdo.distribution(c.vertices, c.m, c.dp, rfilt, c.observed)
    assert same(prob, ref["sample_probability"])
    assert same(cum, ref["cum_prob"]) and same(row, ref["cum_prob_rowwise"])
    # the CDF is artp_compute_sample_cdf's of the same probability layer
    cum2, row2 = chk.computeSampleCdf(ref["sample_probability"])
    assert same(cum, cum2) and same(row, row2)
    if name in sdc.GOLDEN_CASES:
        assert np.array_equal(np.packbits((filt > 0.5).ravel(order="F")), golden[name + "/filter"])
        gp = golden[name + "/sample_probability"]
        assert np.abs(prob - gp).max() <= 4 * BLUR_TOL * gp.max()
        assert np.abs(row - golden[name + "/cum_prob_rowwise"]).max() <= 1e-5


def test_density_and_cap_switches(port_lib):
    c = sdc.make_case("fbm_yaml")
    chk = checker(c.m, c.rp)
    filt = chk.setSampleFilter(c.thr, c.observed)
    for dens in (False, True):
        for cap in (False, True):
            dp = sdo.DistributionParams(dens, c.dp.density_blur_radius, cap, 0.1)
            prob, cum, row = chk.updateSampleDistribution(c.vertices, dp)
            ref = sdo.distribution(c.vertices, c.m, dp, filt, c.observed)
            assert same(prob, ref["sample_probability"]) and same(cum, ref["cum_prob"]) and same(row, ref["cum_prob_rowwise"])
    # zero vertices and vertices all off the map: the uniform density (times filter and cap)
    for v in (np.zeros((0, 7)), c.vertices[10:50] + np.array([1e4, 0, 0, 0, 0, 0, 0])):
        prob, _, _ = chk.updateSampleDistribution(v, c.dp)
        assert same(prob, sdo.apply_cap(filt, c.observed, 0.1))


@pytest.fixture(scope="module")
def config1():
    """configs[1]: the 1000 x 1000 fBm map, processBasic on the device, ~10 k roadmap vertices drawn by the device sampler."""
    from oracle import basic_oracle as bo
    m = synth.make_fbm_map(1000, 1000)
    rp = synth.PARAMS_YAML
    chk = checker(m, rp)
    trav, obs = synth.make_traversability(m, seed=13)
    _, thr = chk.processBasic(m.elevation, trav, obs, m.res, bo.BasicParams())
    L = synth.make_sampler_layers(m, seed=7)
    import art_planner_b200 as ap
    smp = ap.SE3FromSE2Sampler(chk, L, yaml_sampler_params(m), seed=99)
    v, nv = smp.sampleValidBatch(40000, first=0, capacity=10000)
    assert nv >= 10000
    return m, rp, chk, smp, L, thr, obs, v


def test_config1_null_layers_and_device_form(config1):
    import torch
    m, rp, chk, smp, L, thr, obs, v = config1
    dp = sdo.DistributionParams(density_blur_radius=sdo.blur_radius(rp))
    filt = chk.setSampleFilter()                              # the layers processBasic kept on the device
    assert same(filt, chk.setSampleFilter(thr, obs))          # == the host-layer path
    rfilt = sdo.sample_filter(thr, rp, m.res)
    assert same(filt, rfilt)
    prob, cum, row = chk.updateSampleDistribution(v, dp)
    ref = sdo.distribution(v, m, dp, rfilt, obs)
    assert same(prob, ref["sample_probability"]) and same(cum, ref["cum_prob"]) and same(row, ref["cum_prob_rowwise"])
    # the device form, then the sampler re-armed on the resident CDF: fixed variates land where the oracle puts them
    chk.updateSampleDistribution(v[:10], dp)                  # something else resident first
    assert chk.updateSampleDistribution(torch.from_numpy(v).cuda(), dp) is None
    torch.cuda.synchronize()
    smp.updateDistribution(torch.from_numpy(v).cuda())
    u = philox_ref.sampler_uniforms(5, 0, 20000)
    got, rc = smp.sampleUniformBatch(20000, u=u, want_cells=True)
    from oracle import orc
    L2 = copy.copy(L)
    L2.cum_prob, L2.cum_prob_rowwise = ref["cum_prob"], ref["cum_prob_rowwise"]
    _, ref_rc = orc.sample_states(m, L2, yaml_sampler_params(m), rp.reach_z, u)
    assert np.array_equal(rc, ref_rc)
    assert (rc[:, 0] >= 0).all()
    assert (ref["sample_probability"][rc[:, 0], rc[:, 1]] > 0).all()     # no draw in a zero-probability cell


def test_map_change_invalidates_and_errors():
    from art_planner_b200 import capi
    import art_planner_b200 as ap
    c = sdc.make_case("offorigin_header")
    chk = checker(c.m, c.rp)
    with pytest.raises(capi.ArtpError) as e:                  # no processBasic layers on this handle
        chk.setSampleFilter()
    assert e.value.code == capi.ARTP_E_INVALID
    with pytest.raises(capi.ArtpError) as e:                  # the cap without an observed layer
        chk.updateSampleDistribution(c.vertices, c.dp)
    assert e.value.code == capi.ARTP_E_INVALID
    filt = chk.setSampleFilter(c.thr, c.observed)
    chk.updateSampleDistribution(c.vertices, c.dp)
    for bad, code in ((sdo.DistributionParams(density_blur_radius=0.0), capi.ARTP_E_INVALID),
                      (sdo.DistributionParams(density_blur_radius=float("nan")), capi.ARTP_E_INVALID),
                      (sdo.DistributionParams(density_blur_radius=0.4, max_prob_unknown_samples=1.5), capi.ARTP_E_INVALID),
                      (sdo.DistributionParams(density_blur_radius=9.0), capi.ARTP_E_LIMIT)):        # ksize 1081 > 1023
        with pytest.raises(capi.ArtpError) as e:
            chk.updateSampleDistribution(c.vertices, bad)
        assert e.value.code == code
    with pytest.raises(capi.ArtpError) as e:                  # size mismatch against the map
        chk.setSampleFilter(c.thr[:-1], c.observed[:-1])
    assert e.value.code == capi.ARTP_E_INVALID
    # a new map drops the filter and observed layers: the cap is refused, the density runs without the filter
    chk.updateHeightField()
    with pytest.raises(capi.ArtpError) as e:
        chk.updateSampleDistribution(c.vertices, c.dp)
    assert e.value.code == capi.ARTP_E_INVALID
    dp = sdo.DistributionParams(density_blur_radius=c.dp.density_blur_radius, use_max_prob_unknown_samples=False)
    prob, _, _ = chk.updateSampleDistribution(c.vertices, dp)
    assert same(prob, sdo.distribution(c.vertices, c.m, dp)["sample_probability"])
    assert not same(prob, sdo.distribution(c.vertices, c.m, dp, filt)["sample_probability"])
    # processBasic layers of another map size are not taken for NULL
    from oracle import basic_oracle as bo
    small = sdc.make_case("small_yaml")
    chk.processBasic(small.m.elevation, small.traversability, small.observed, small.m.res, bo.BasicParams())
    with pytest.raises(capi.ArtpError) as e:
        chk.setSampleFilter()
    assert e.value.code == capi.ARTP_E_INVALID
    # map windows are refused
    w = ap.StateValidityChecker(c.rp, device=0)
    w.setMap(c.m)
    w.updateHeightField(window=(0, 48))
    for f in (lambda: w.setSampleFilter(c.thr, c.observed), lambda: w.updateSampleDistribution(c.vertices, dp)):
        with pytest.raises(capi.ArtpError) as e:
            f()
        assert e.value.code == capi.ARTP_E_INVALID
