"""GPU (-m gpu): artp_planner_set_map refuses, before any work, exactly the maps whose chain would hit a size limit, and
with the code and message of the call that would hit it. Each case makes one limit the binding one -- Basic's largest
structuring element, the sample filter's reach, its wall element, the density blur's 1023 taps -- and tries resolutions
just either side of it: setMap / setMapRaw, the component call at that resolution, the previous map after a refusal,
and the parameters that switch the filter and the blur off."""
import dataclasses
import math
import types

import numpy as np
import pytest

import planner_cases as pc
from art_planner_b200 import capi, costnet, synth

pytestmark = pytest.mark.gpu

BASIC = dict(traversability_thres=0.15, unknown_space_untraversable=1, foothold_margin=0.3, foothold_margin_max_hole_size=0.3,
             foothold_margin_max_drop=0.3, foothold_margin_max_drop_search_radius=0.16, foothold_margin_min_step=0.3,
             foothold_size=0.1)
MORPH, TAPS = "structuring element larger than 64 cells", "Gaussian kernel larger than 1023 cells"


def binding(rp, bp, res):
    """The limits the map chain hits at resolution res, restated (basic.cpp:65-74, :116-122, sample_density.cpp:33-35 with
    planner.cpp:48's radius): Basic's largest element, the filter's reach and wall elements, the blur's kernel size."""
    basic = max(math.ceil(bp.foothold_size / res), math.ceil(2 * bp.foothold_margin / res),
                math.floor(bp.foothold_margin_max_hole_size / res), math.ceil(2 * bp.foothold_margin_max_drop_search_radius / res))
    reach = int(math.hypot(rp.reach_x, rp.reach_y) / res)
    wall = int(min((rp.torso_length - rp.reach_x) * 0.5, (rp.torso_width - rp.reach_y) * 0.5) / res)
    cells = 6 * ((rp.torso_length + rp.torso_width) * 0.25) / res
    blur = not cells < 1024 or (int(cells) | 1) > 1023
    return {k for k, hit in (("basic", basic > 64), ("reach", reach > 64), ("wall", wall > 64), ("blur", blur)) if hit}


BLUR_6R = 6 * (22.0 + 5.3) * 0.25
# (name, robot, Basic, the resolution at the limit, map cells per side, message, extra resolutions); a small map keeps the
# box kernels' tiles within their shared memory whatever the robot's size in cells (the motion-cost network needs 64 x 64).
CASES = [
    ("basic", synth.PARAMS_YAML, dict(BASIC, foothold_margin_max_hole_size=2.6), 0.04, 120, MORPH, ()),
    ("reach", dataclasses.replace(synth.PARAMS_YAML, torso_length=6.0, torso_width=5.0, reach_x=2.0, reach_y=2.0), BASIC,
     math.hypot(2.0, 2.0) / 65, 64, MORPH, ()),
    ("wall", dataclasses.replace(synth.PARAMS_YAML, torso_length=6.0, torso_width=6.0, reach_x=0.5, reach_y=0.5), BASIC,
     2.75 / 65, 64, MORPH, ()),
    # and the blur's kernel at 1023 taps from cells in [1023, 1024), then just past 1024 cells
    ("blur", dataclasses.replace(synth.PARAMS_YAML, torso_length=22.0, torso_width=5.3, reach_x=1.0, reach_y=1.0), BASIC,
     BLUR_6R / 1024, 64, TAPS, (BLUR_6R / 1023.5, BLUR_6R / 1024.2)),
]
IDS = [c[0] for c in CASES]


def probes(case):
    """(accepted resolutions, refused resolutions): 0.5 % either side of the limit and the case's extra ones, with the
    case's limit the only one hit."""
    name, rp, basic, res, _, _, extra = case
    bp = types.SimpleNamespace(**basic)
    ok, bad = [], []
    for r in (res * 1.005, res * 0.995) + extra:
        hit = binding(rp, bp, r)
        assert hit in (set(), {name}), (name, r, hit)
        (bad if hit else ok).append(r)
    assert ok and bad
    return ok, bad


def layers(res, n):
    return pc.raw_layers(synth.make_fbm_map(n, n, res=res, seed=3, amp=0.2), seed=9)


def checker(rp):
    import art_planner_b200 as ap
    chk = ap.StateValidityChecker(rp)
    ap.MotionCostObjective(chk).setWeights(costnet.make_state_dict(seed=5))
    return chk


def planner(rp, basic, **kw):
    import art_planner_b200 as ap
    return ap.Planner(checker(rp), pc.small_params(seed=4, max_draws=1 << 18, basic=types.SimpleNamespace(**basic), **kw))


def raises(msg, fn, *args):
    with pytest.raises(capi.ArtpError) as e:
        fn(*args)
    assert e.value.code == capi.ARTP_E_LIMIT and str(e.value) == f"artp error {capi.ARTP_E_LIMIT}: {msg}"


def space(pl):
    s = pl.space()
    return tuple(s.low) + tuple(s.high) + (s.longest_valid_segment_fraction,)


def plan(pl, n, res):
    a = np.array([n * res * 0.3, 0.0, 0.3, 0.0, 0.0, 0.0, 1.0])
    b = np.array([-n * res * 0.3, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
    status = pl.plan(a, b)
    return status, (pl.getSolutionPath().copy() if status == pl.SOLVED else None)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_set_map_refuses_exactly_past_the_limit(case):
    name, rp, basic, _, n, msg, _ = case
    oks, bads = probes(case)
    pl = planner(rp, basic)
    for r in oks:
        e, t, ei, ti = layers(r, n)
        pl.setMap(e, t, ei, ti, r, 0.0, 0.0)
        pl.setMapRaw(e, t, r, 0.0, 0.0)
    last = oks[-1]
    before = space(pl)
    for r in bads:
        e2, t2, ei2, ti2 = layers(r, n)
        raises(msg, pl.setMap, e2, t2, ei2, ti2, r, 0.0, 0.0)
        raises(msg, pl.setMapRaw, e2, t2, r, 0.0, 0.0)
    # the refused maps left the last accepted one installed: its space, and a plan equal to a fresh planner's on it
    assert space(pl) == before
    fresh = planner(rp, basic)
    fresh.setMapRaw(e, t, last, 0.0, 0.0)
    got, want = plan(pl, n, last), plan(fresh, n, last)
    assert got[0] == want[0] and (got[1] is None) == (want[1] is None)
    assert got[1] is None or np.array_equal(got[1], want[1])


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_component_call_refuses_the_same_way(case):
    import art_planner_b200 as ap
    name, rp, basic, _, n, msg, _ = case
    oks, bads = probes(case)
    bp = types.SimpleNamespace(**basic)
    for r, refused in [(r, False) for r in oks] + [(r, True) for r in bads]:
        e, t, ei, ti = layers(r, n)
        chk = checker(rp)
        if name == "basic":
            call = lambda: chk.processBasic(ei, ti, np.isfinite(e).astype(np.float32), r, bp)
        else:
            m = synth.make_fbm_map(n, n, res=r, seed=3, amp=0.2)
            chk.setMap(m)
            chk.updateHeightField()
            thr = (ti > 0.5).astype(np.float32)
            if name != "blur":
                call = lambda: chk.setSampleFilter(thr, None)
            else:
                chk.setSampleFilter(thr, None)
                sp = types.SimpleNamespace(use_inverse_vertex_density=1, use_max_prob_unknown_samples=0,
                                           max_prob_unknown_samples=0.1)
                dp = ap.checker._distribution_params(sp, rp)
                assert dp.density_blur_radius == (rp.torso_length + rp.torso_width) * 0.25
                call = lambda: chk.updateSampleDistribution(np.zeros((0, 7)), dp)
        if refused:
            raises(msg, call)
        else:
            call()


@pytest.mark.parametrize("case", CASES[1:], ids=IDS[1:])
def test_limits_of_switched_off_stages_do_not_apply(case):
    name, rp, basic, _, n, msg, _ = case
    for bad in probes(case)[1]:
        e, t, ei, ti = layers(bad, n)
        no_dist = planner(rp, basic, sample_from_distribution=0)
        no_dist.setMap(e, t, ei, ti, bad, 0.0, 0.0)
        no_dist.setMapRaw(e, t, bad, 0.0, 0.0)
        no_density = planner(rp, basic, use_inverse_vertex_density=0)
        if name == "blur":
            no_density.setMap(e, t, ei, ti, bad, 0.0, 0.0)
            no_density.setMapRaw(e, t, bad, 0.0, 0.0)
        else:
            raises(msg, no_density.setMap, e, t, ei, ti, bad, 0.0, 0.0)
            raises(msg, no_density.setMapRaw, e, t, bad, 0.0, 0.0)
