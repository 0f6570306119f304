"""GPU parity (-m gpu) of the start / goal search (StartState / GoalStateRegion::sampleGoal, start.cpp:7-41,
goal.cpp:11-41) and of the goal projection (planner.cpp:223-237, map.cpp:77-90) against the compiled reference's fixture
and the CPU oracle."""
import os

import numpy as np
import pytest

import cases
import philox_ball_ref
import start_goal_cases as sgc
import start_goal_oracle as sgo
from art_planner_b200 import capi, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATE_TOL = 1e-12      # CUDA vs numpy atan2 / sin / cos in the projected quaternion (the sampler's tolerance)


@pytest.fixture(scope="module")
def ap():
    import art_planner_b200
    from art_planner_b200 import build
    build.build()
    return art_planner_b200


def _checker(ap, m, pk="yaml", params=None):
    chk = ap.StateValidityChecker(params or cases.PARAMS[pk], device=0)
    chk.setMap(m)
    chk.updateHeightField()
    return chk


def _oracle(port_lib, m, pk="yaml", params=None):
    o = port_lib.Oracle(params or cases.PARAMS[pk], "port")
    o.set_map(m)
    return o


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name,mk,pk,n,n_iter,seed", sgc.GOLDEN_CASES, ids=[c[0] for c in sgc.GOLDEN_CASES])
def test_golden_cases(ap, maps, port_lib, name, mk, pk, n, n_iter, seed, mode):
    g = np.load(os.path.join(ROOT, "tests", "golden", "start_goal.npz"))
    m = maps(mk)
    centres, radius, off = sgc.golden_inputs(m, n, n_iter, seed)
    chk = _checker(ap, m, pk)
    chk.setMode(mode)
    states, idx = chk.findValidNear(centres, radius, n_iter, offsets=off)
    assert np.array_equal(idx, g[name + "/index"]) and _same(states, g[name + "/states"])
    rs, ri = sgo.find_valid_near(_oracle(port_lib, m, pk), centres, n_iter, off)
    assert np.array_equal(idx, ri) and _same(states, rs)


@pytest.mark.parametrize("pk", ["yaml", "header"])
def test_random_queries_match_oracle(ap, maps, port_lib, pk):
    """10 k queries on each of fbm_rough and terraces, explicit offsets, both grouping routes."""
    for mk, seed in (("fbm_rough", 201), ("terraces", 202)):
        m = maps(mk)
        n, n_iter = 10000, 24
        centres, radius = sgc.make_queries(m, n, seed)
        off = philox_ball_ref.ball_offsets(seed, 0, n, n_iter, radius)
        rs, ri = sgo.find_valid_near(_oracle(port_lib, m, pk), centres, n_iter, off)
        assert (ri == 0).any() and (ri > 0).any() and (ri < 0).any()
        chk = _checker(ap, m, pk)
        for mode in (0, 1):
            chk.setMode(mode)
            s, i = chk.findValidNear(centres, radius, n_iter, offsets=off)
            assert np.array_equal(i, ri) and _same(s, rs), (mk, mode)


def test_outcomes(ap, maps, port_lib):
    m = maps("fbm_rough")
    chk = _checker(ap, m)
    o = _oracle(port_lib, m)
    centres, radius = sgc.make_queries(m, 2000, 301)
    flags = o.check_poses(centres)
    n_iter = 30
    off = philox_ball_ref.ball_offsets(301, 0, 2000, n_iter, radius)
    s, i = chk.findValidNear(centres, radius, n_iter, offsets=off)
    ok = flags == 1
    assert ok.any() and (i[ok] == 0).all() and _same(s[ok], centres[ok])          # centre valid -> index 0, the centre
    none = i < 0
    assert none.any()
    last = centres[none].copy()
    last[:, 0] = centres[none, 0] + off[none, n_iter - 1, 0]
    last[:, 1] = centres[none, 1] + off[none, n_iter - 1, 1]
    assert _same(s[none], last)                                                  # none valid -> candidate n_iter
    s0, i0 = chk.findValidNear(centres, radius, 0)                               # n_iter = 0: the centre alone
    assert np.array_equal(i0, np.where(ok, 0, -1)) and _same(s0, centres)
    sr, ir = chk.findValidNear(centres, 0.0, 50, seed=4)                         # radius 0: every candidate is the centre
    assert np.array_equal(ir, np.where(ok, 0, -1)) and _same(sr, centres)


@pytest.mark.parametrize("unknown", [True, False])
def test_centres_outside_the_map(ap, maps, port_lib, unknown):
    import dataclasses
    m = maps("fixture")
    params = dataclasses.replace(cases.PARAMS["yaml"], unknown_space_untraversable=unknown)
    lx, _ = m.length
    c = synth.make_terrain_poses(m, 300, seed=41)
    c[:, 0] = m.cx + np.where(np.arange(300) % 2 == 0, 1.0, -1.0) * (0.5 * lx + np.linspace(0.01, 1.5, 300))
    off = philox_ball_ref.ball_offsets(41, 0, 300, 40, 0.5)
    s, i = _checker(ap, m, params=params).findValidNear(c, 0.5, 40, offsets=off)
    rs, ri = sgo.find_valid_near(_oracle(port_lib, m, params=params), c, 40, off)
    assert np.array_equal(i, ri) and _same(s, rs)
    # far off the map no box of any candidate is on it: only the feet's unknown-space rule decides
    far = np.abs(c[:, 0] - m.cx) > 0.5 * lx + 1.3
    assert far.any() and (i[far] == (-1 if unknown else 0)).all()


@pytest.mark.parametrize("n,n_iter", [(3, 12), (2, 1000), (64, 40000)], ids=["tiny", "start+goal", "chunks"])
def test_batch_equals_single_queries(ap, maps, n, n_iter):
    """n queries with different radii in one call == n one-query calls, also across candidate chunks and rounds."""
    m = maps("fbm_rough")
    chk = _checker(ap, m)
    centres, _ = sgc.make_queries(m, n, 401)
    radius = np.linspace(0.05, 1.2, n)
    off = philox_ball_ref.ball_offsets(401, 0, n, n_iter, radius)
    s, i = chk.findValidNear(centres, radius, n_iter, offsets=off)
    for q in range(n):
        sq, iq = chk.findValidNear(centres[q:q + 1], radius[q], n_iter, offsets=off[q:q + 1])
        assert iq[0] == i[q] and _same(sq[0], s[q]), q
    if n == 64:
        assert (i > 0).any() or (i < 0).any()


def test_stream_mode(ap, maps):
    m = maps("terraces")
    chk = _checker(ap, m)
    n, n_iter = 50, 400
    centres, radius = sgc.make_queries(m, n, 501)
    for seed, first in ((9, 0), (0xFEDCBA9876543210, 2 ** 32 - 150)):      # the second crosses the counter's 32-bit word
        got = chk.ballOffsets(seed, first, n, n_iter, radius)
        want = philox_ball_ref.ball_offsets(seed, first, n, n_iter, radius)
        assert np.abs(got - want).max() <= 1e-15 * radius.max()
        assert (np.hypot(got[..., 0], got[..., 1]) <= radius[:, None] * (1 + 1e-15)).all()
        s, i = chk.findValidNear(centres, radius, n_iter, seed=seed, first_draw=first)
        s2, i2 = chk.findValidNear(centres, radius, n_iter, offsets=got)
        assert np.array_equal(i, i2) and _same(s, s2)


def test_device_form_on_a_side_stream(ap, maps):
    import torch
    m = maps("fbm_rough")
    chk = _checker(ap, m)
    centres, radius = sgc.make_queries(m, 300, 601)
    n_iter = 200
    off = philox_ball_ref.ball_offsets(601, 0, 300, n_iter, radius)
    s, i = chk.findValidNear(centres, radius, n_iter, offsets=off)
    ss, si = chk.findValidNear(centres, radius, n_iter, seed=3, first_draw=77)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        dc = torch.from_numpy(centres).cuda()
        dr = torch.from_numpy(radius).cuda()
        do = torch.from_numpy(off).cuda()
        ds, di = chk.findValidNear(dc, dr, n_iter, offsets=do)
        ds2, di2 = chk.findValidNear(dc, dr, n_iter, seed=3, first_draw=77)
    side.synchronize()
    assert np.array_equal(di.cpu().numpy(), i) and _same(ds.cpu().numpy(), s)
    assert np.array_equal(di2.cpu().numpy(), si) and _same(ds2.cpu().numpy(), ss)


def test_argument_errors(ap, maps):
    m = maps("fixture")
    chk = _checker(ap, m)
    c = synth.make_terrain_poses(m, 4, seed=1)
    for r in (-0.1, np.nan, np.inf):
        with pytest.raises(capi.ArtpError) as e:
            chk.findValidNear(c, r, 10)
        assert e.value.code == capi.ARTP_E_INVALID
    with pytest.raises(capi.ArtpError) as e:
        chk.findValidNear(c, 0.5, 2 ** 30)                       # 4 * (2^30 + 1) >= 2^32 candidates
    assert e.value.code == capi.ARTP_E_INVALID
    bare = ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)
    with pytest.raises(capi.ArtpError) as e:
        bare.findValidNear(c, 0.5, 10)
    assert e.value.code == capi.ARTP_E_NOMAP


def test_pose_from_2d(ap, maps, port_lib):
    m = maps("fbm_rough")
    chk = _checker(ap, m)
    g = synth.make_terrain_poses(m, 5000, seed=701)
    lx, ly = m.length
    g[::7, 0] = m.cx + 0.5 * lx + 0.3                     # off the map in x
    g[3::11, 1] = m.cy - 0.5 * ly - 0.01                  # off the map in y
    with pytest.raises(capi.ArtpError) as e:              # no normals yet
        chk.poseFrom2D(g)
    assert e.value.code == capi.ARTP_E_INVALID
    nx, ny, nz, sd = chk.estimateNormals(0.49)
    got, inside = chk.poseFrom2D(g)

    class Layers:
        normal_x, normal_y, normal_z = nx, ny, nz
    want, want_in = sgo.pose_from_2d(m, Layers, g)
    assert np.array_equal(inside, want_in) and (inside == 0).any() and (inside == 1).mean() > 0.7
    out = inside == 0
    assert _same(got[out], g[out])                         # off the map: untouched
    assert _same(got[:, :2], g[:, :2]) and _same(got[:, 2], want[:, 2])
    assert np.abs(got[:, 3:] - want[:, 3:]).max() < STATE_TOL
    chk.updateHeightField()                                # a new map invalidates the normal layers
    with pytest.raises(capi.ArtpError) as e:
        chk.poseFrom2D(g)
    assert e.value.code == capi.ARTP_E_INVALID


def test_mirror_draw_positions(ap, maps):
    """StartState / GoalStateRegion advance their stream by what the reference consumes: k draws for candidate k, n_iter
    when none is valid, none for a valid centre; every call equals the batch call at the same stream position."""
    m = maps("fbm_rough")
    chk = _checker(ap, m)
    centres, _ = sgc.make_queries(m, 60, 801)
    for cls, r in ((ap.StartState, 0.2), (ap.GoalStateRegion, 0.5)):
        obj = cls(chk, seed=17)
        obj.setThreshold(r)
        obj.setMaxNumSamples(1000)
        seen = set()
        for q in range(60):
            before = obj.draw
            obj.setState(centres[q])
            st, k = obj.sampleGoal()
            ws, wi = chk.findValidNear(centres[q:q + 1], r, 1000, seed=17, first_draw=before)
            assert k == wi[0] and _same(st, ws[0])
            assert obj.draw - before == (k if k >= 0 else 1000)
            seen.add(0 if k == 0 else (1 if k > 0 else -1))
        assert seen == {0, 1, -1}
