"""GPU parity (-m gpu) for the device sampler (SE3FromSE2Sampler::sampleUniform, sampler.cpp:40-131) and the fused
sample -> isValid -> compact path, against the CPU oracle fed with the same uniform variates."""
import numpy as np
import pytest

import cases
import philox_ref
from art_planner_b200 import synth

pytestmark = pytest.mark.gpu

STATE_TOL = 1e-12      # double states: CUDA vs libm sin/cos/acos/atan2 differ in the last ulps; cells are exact


@pytest.fixture(scope="module")
def rig(maps):
    import art_planner_b200 as ap
    from art_planner_b200 import build
    build.build()
    m = maps("fbm_rough")
    chk = ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)
    chk.setMap(m)
    chk.updateHeightField()
    L = synth.make_sampler_layers(m, seed=7)
    return ap, m, chk, L


def test_uniform_stream_matches_philox_restatement(rig):
    ap, m, chk, L = rig
    smp = ap.SE3FromSE2Sampler(chk, L, synth.sampler_params_for(m), seed=0x1234567890ABCDEF)
    for first, n in ((0, 1000), (2 ** 32 - 100, 300), (2 ** 40 + 17, 64)):      # crosses the 32-bit counter word
        assert np.array_equal(smp.uniforms(first, n), philox_ref.sampler_uniforms(0x1234567890ABCDEF, first, n))


@pytest.mark.parametrize("from_dist", [True, False], ids=["distribution", "uniform"])
def test_states_match_oracle(rig, port_lib, from_dist):
    ap, m, chk, L = rig
    sp = synth.sampler_params_for(m, from_dist)
    smp = ap.SE3FromSE2Sampler(chk, L, sp, seed=11)
    n = 50000
    u = philox_ref.sampler_uniforms(11, 0, n)
    u[:8, 1] = np.nextafter(1.0, 0.0)            # last-row fallback (a NaN CDF row)
    u[8:16, 0] = 0.0
    u[16:24, 4] = 0.0                            # acos(1) branch of eulerRPY
    ref, ref_rc = port_lib.sample_states(m, L, sp, cases.PARAMS["yaml"].reach_z, u)
    got, rc = smp.sampleUniformBatch(n, u=u, want_cells=True)
    assert np.array_equal(rc, ref_rc)
    nan = np.isnan(ref[:, 0])
    assert np.array_equal(np.isnan(got[:, 0]), nan)
    assert np.abs(got[~nan] - ref[~nan]).max() < STATE_TOL
    # the same call driven by the internal Philox stream
    got2 = smp.sampleUniformBatch(1000, first=0)
    ref2, _ = port_lib.sample_states(m, L, sp, cases.PARAMS["yaml"].reach_z, philox_ref.sampler_uniforms(11, 0, 1000))
    ok = ~np.isnan(ref2[:, 0])
    assert np.abs(got2[ok] - ref2[ok]).max() < STATE_TOL and np.isnan(got2[~ok]).all()


@pytest.mark.parametrize("from_dist", [True, False], ids=["distribution", "uniform"])
def test_fused_sample_check_compact(rig, port_lib, from_dist):
    """sample_valid == candidates filtered by the validity oracle, in draw order (rejection loop semantics)."""
    ap, m, chk, L = rig
    sp = synth.sampler_params_for(m, from_dist)
    smp = ap.SE3FromSE2Sampler(chk, L, sp, seed=21)
    n = 60000
    cand = smp.sampleUniformBatch(n, first=1000)
    o = port_lib.Oracle(cases.PARAMS["yaml"], "port")
    o.set_map(m)
    ok = ~np.isnan(cand[:, 0])
    flags = np.zeros(n, np.uint8)
    flags[ok] = o.check_poses(cand[ok])
    assert 0.02 < flags.mean() < 0.98
    got, nv = smp.sampleValidBatch(n, first=1000)
    assert nv == int(flags.sum())
    assert np.array_equal(got, cand[flags != 0])
    # truncated output: first `capacity` valid states, n_valid still the total
    got_c, nv_c = smp.sampleValidBatch(n, first=1000, capacity=100)
    assert nv_c == nv and np.array_equal(got_c, got[:100])


def test_fused_path_across_chunks_and_device_buffers(rig):
    import torch
    ap, m, chk, L = rig
    smp = ap.SE3FromSE2Sampler(chk, L, synth.sampler_params_for(m), seed=5)
    n = (1 << 21) + 12345                        # two chunks of the fused path
    got, nv = smp.sampleValidBatch(n, first=0)
    a, na = smp.sampleValidBatch(1 << 21, first=0)
    b, nb = smp.sampleValidBatch(12345, first=1 << 21)
    assert nv == na + nb and np.array_equal(got, np.concatenate([a, b]))
    out = torch.empty((nv, 7), dtype=torch.float64, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    smp.sampleValidDevice(n, 0, out, cnt)
    torch.cuda.synchronize()
    assert int(cnt.item()) == nv and np.array_equal(out.cpu().numpy(), got)
    # every returned state is valid according to the checker itself
    assert chk.isValidBatch(got[:200000]).all()


def test_sampler_errors(rig):
    ap, m, chk, L = rig
    import copy
    chk2 = ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)
    chk2.setMap(m)
    chk2.updateHeightField()
    bad = copy.copy(L)
    cp = L.cum_prob.copy(order="F")
    cp[5, 10] = cp[5, 9] - 0.25                  # not a CDF any more
    bad.cum_prob = cp
    with pytest.raises(RuntimeError):
        ap.SE3FromSE2Sampler(chk2, bad, synth.sampler_params_for(m))
    smp = ap.SE3FromSE2Sampler(chk2, L, synth.sampler_params_for(m))
    assert smp.sampleUniformBatch(0).shape == (0, 7)
    chk2.updateHeightField()                     # a new map invalidates the sampler layers
    with pytest.raises(RuntimeError):
        smp.sampleUniformBatch(4)


def test_refused_arming_keeps_the_armed_sampler(rig):
    """artp_set_sampler refusing CDF layers that are not cumulative leaves an armed sampler as it was: still uniform, in
    its own bounds, drawing what it drew before."""
    ap, m, chk, L = rig
    import copy
    import dataclasses
    chk2 = ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)
    chk2.setMap(m)
    chk2.updateHeightField()
    full = synth.sampler_params_for(m)
    narrow = dataclasses.replace(synth.sampler_params_for(m, from_distribution=False),
                                 low=tuple(0.75 * a + 0.25 * b for a, b in zip(full.low, full.high)),
                                 high=tuple(0.25 * a + 0.75 * b for a, b in zip(full.low, full.high)))
    smp = ap.SE3FromSE2Sampler(chk2, L, narrow, seed=9)
    want = smp.sampleUniformBatch(512, first=0)
    bad = copy.copy(L)
    cp = L.cum_prob.copy(order="F")
    cp[5, 10] = cp[5, 9] - 0.25                  # not a CDF any more
    bad.cum_prob = cp
    with pytest.raises(RuntimeError):
        smp.setLayers(bad, full)
    assert np.array_equal(smp.sampleUniformBatch(512, first=0), want, equal_nan=True)


@pytest.mark.parametrize("mk", ["fbm_rough", "ramp", "fixture", "flat_holes_terrace"])
def test_estimate_normals_bit_exact(maps, port_lib, mk):
    """artp_estimate_normals == the CPU restatement of utils.cpp:213-324, bit for bit (float32 layers)."""
    import art_planner_b200 as ap
    m = maps(mk)
    chk = ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)
    chk.setMap(m)
    chk.updateHeightField()
    p = cases.PARAMS["yaml"]
    radius = (p.torso_length + p.torso_width) * 0.25            # basic.cpp:47
    got = chk.estimateNormals(radius)
    ref = port_lib.estimate_normals(m, radius)
    for g, r, name in zip(got, ref, ("normal_x", "normal_y", "normal_z", "plane_fit_std_dev")):
        fin = np.isfinite(r)
        assert np.array_equal(np.isfinite(g), fin), name
        assert np.array_equal(g[fin].view(np.uint32), r[fin].view(np.uint32)), name


def test_sampler_on_device_normals(rig, port_lib):
    """set_map -> estimate_normals (device) -> sampler without host normal layers == oracle fed the oracle's normals."""
    ap, m, chk0, L = rig
    chk = ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)
    chk.setMap(m)
    chk.updateHeightField()
    sp = synth.sampler_params_for(m)

    class OnlyCdf:
        cum_prob, cum_prob_rowwise = L.cum_prob, L.cum_prob_rowwise
    with pytest.raises(RuntimeError):                      # no normals yet
        ap.SE3FromSE2Sampler(chk, OnlyCdf, sp, seed=3)
    chk.estimateNormals(0.49, want_host=False)
    smp = ap.SE3FromSE2Sampler(chk, OnlyCdf, sp, seed=3)
    nx, ny, nz, sd = port_lib.estimate_normals(m, 0.49)
    import copy
    L2 = copy.copy(L)
    L2.normal_x, L2.normal_y, L2.normal_z, L2.plane_fit_std_dev = nx, ny, nz, sd
    u = philox_ref.sampler_uniforms(3, 0, 20000)
    ref, ref_rc = port_lib.sample_states(m, L2, sp, cases.PARAMS["yaml"].reach_z, u)
    got, rc = smp.sampleUniformBatch(20000, first=0, want_cells=True)
    assert np.array_equal(rc, ref_rc)
    ok = ~np.isnan(ref).any(axis=1)
    assert np.array_equal(np.isnan(got).any(axis=1), ~ok)
    assert np.abs(got[ok] - ref[ok]).max() < STATE_TOL


def test_sample_cdf_on_device_and_full_device_chain(rig, port_lib):
    """artp_compute_sample_cdf == the CPU restatement of probability_distribution.cpp:20-46 bit for bit, and the chain
    set_map -> estimate_normals -> compute_sample_cdf -> sampler (no host layers at all) samples like the oracle."""
    ap, m, chk0, L = rig
    chk = ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)
    chk.setMap(m)
    chk.updateHeightField()
    cum, row = chk.computeSampleCdf(L.sample_probability)
    rcum, rrow = port_lib.compute_cdf(L.sample_probability)
    nan = np.isnan(rcum)
    assert nan.any() and np.array_equal(np.isnan(cum), nan)
    assert np.array_equal(cum[~nan].view(np.uint32), rcum[~nan].view(np.uint32))
    assert np.array_equal(row.view(np.uint32), rrow.view(np.uint32))
    chk.estimateNormals(0.49, want_host=False)
    sp = synth.sampler_params_for(m)

    class Nothing:
        pass
    smp = ap.SE3FromSE2Sampler(chk, Nothing, sp, seed=8)
    import copy
    L2 = copy.copy(L)
    L2.normal_x, L2.normal_y, L2.normal_z, L2.plane_fit_std_dev = port_lib.estimate_normals(m, 0.49)
    L2.cum_prob, L2.cum_prob_rowwise = rcum, rrow
    u = philox_ref.sampler_uniforms(8, 0, 20000)
    ref, ref_rc = port_lib.sample_states(m, L2, sp, cases.PARAMS["yaml"].reach_z, u)
    got, rc = smp.sampleUniformBatch(20000, first=0, want_cells=True)
    assert np.array_equal(rc, ref_rc)
    ok = ~np.isnan(ref).any(axis=1)
    assert np.abs(got[ok] - ref[ok]).max() < STATE_TOL
