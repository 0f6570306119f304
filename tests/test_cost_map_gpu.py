"""GPU (-m gpu): the cost server's map preparation on the device (artp_cost_map_layer[_device]) against the golden maps
made through cv2 and the restatement (oracle/cost_map_oracle.py) bit for bit; the refusals; the features of
artp_update_features_raw against the torch restatement of both networks on the prepared map, and bit for bit against
artp_set_map + artp_update_features where the trunk's input is the same; the planner's cost_map_from_raw against the
chained calls (set_map_raw with 0, artp_update_features_raw, plan), also beside another handle planning on the device;
and refused calls that leave the installed map and the features in place."""
import os
import threading

import numpy as np
import pytest

import cost_map_cases as cc
import planner_cases as pc
import roadmap_cases as rc
from art_planner_b200 import capi, costnet, synth
from oracle import cost_map_oracle as cm
from oracle import inpaint_oracle as io

pytestmark = pytest.mark.gpu
GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cost_map.npz"))
RTOL, ATOL = 1e-4, 1e-5


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def chk():
    import art_planner_b200 as ap
    return ap.StateValidityChecker(rc.make_case("gentle_inf").rp)


def on_device(fn, layer, *args):
    """fn on a column-major CUDA copy of `layer`, on a side stream."""
    import torch
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d = torch.from_numpy(np.ascontiguousarray(np.asarray(layer, np.float32).T)).cuda().t()
        out = fn(d, *args)
        if out is not None:
            out = out.cpu().numpy()
    s.synchronize()
    return out


def case(name):
    """(layer, geometry, golden map, restated map)."""
    a, geom, want = cc.golden_case(GOLDEN, name)
    labels = io.interaction_components(~np.isfinite(cm.server_image(a)))[0]
    restated = cm.cost_map_layer(a, lambda u, m: io.telea_by_components(u, m, labels=labels)[0])
    return a, geom, want, restated


@pytest.mark.parametrize("name", list(cc.CASES) + list(cc.LARGE_CASES))
def test_cost_map_equals_golden_and_restatement(chk, name):
    import art_planner_b200 as ap
    a, _, want, restated = case(name)
    obj = ap.MotionCostObjective(chk)
    host = obj.costMap(a)
    dev = on_device(obj.costMap, a)
    assert not GOLDEN[name + "/diverging"].size       # cv2 and the restatement agree on every case
    for got, what in ((host, "artp_cost_map_layer"), (dev, "artp_cost_map_layer_device")):
        assert np.array_equal(bits(got), bits(want)), f"{what}: {int((bits(got) != bits(want)).sum())} cells differ from cv2"
        assert np.array_equal(bits(got), bits(restated)), what


def test_refusals_and_edges(chk):
    import art_planner_b200 as ap
    obj = ap.MotionCostObjective(chk)
    for name, (a, _) in cc.refused_layers().items():
        for fn in (obj.costMap, lambda x: on_device(obj.costMap, x)):
            with pytest.raises(ap.ArtpError) as e:
                fn(a)
            assert e.value.code == capi.ARTP_E_INVALID, name
    for name, a in cc.accepted_edges().items():
        want = cm.cost_map_layer(a)
        assert np.array_equal(bits(obj.costMap(a)), bits(want)), name
        assert np.array_equal(bits(on_device(obj.costMap, a)), bits(want)), name


def synth_map(a, geom):
    res, cx, cy = geom
    return synth.SynthMap(np.asfortranarray(a, dtype=np.float32), np.asfortranarray(a, dtype=np.float32), res, cx, cy, "")


@pytest.mark.parametrize("network", ["light", "full"])
@pytest.mark.parametrize("name", ["fbm_blobs", "border_holes", "off_origin"])
def test_features_raw_match_restatement(network, name):
    import art_planner_b200 as ap
    from oracle.cnn_oracle import CostNetOracle
    a, geom = cc.CASES[name]()
    c = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    obj = ap.MotionCostObjective(c)
    sd = costnet.make_state_dict(seed=5, network=network)
    obj.setWeights(sd)
    obj.updateFeaturesRaw(a, *geom)
    got = obj.features()
    orc = CostNetOracle(sd)
    feat = orc.features(cm.prepare(cm.server_image(a)))
    ref = feat.permute(1, 2, 0).numpy()
    assert got.shape == ref.shape
    assert float(np.abs(got - ref).max()) / float(np.abs(ref).max()) < 1e-4
    m = synth_map(a, geom)
    q = costnet.make_queries(m, 2048, seed=6)
    lx, ly = m.length
    cost = obj.costQuery(q)
    assert np.allclose(cost, orc.query(feat, q, m.res, lx, ly, m.cx, m.cy), rtol=RTOL, atol=ATOL)
    on_device(obj.updateFeaturesRaw, a, *geom)
    assert np.array_equal(obj.features(), got)
    assert np.array_equal(obj.costQuery(q), cost)


def test_hole_free_layer_equals_set_map_features():
    """Without holes the trunk's input is the raw layer itself: the features equal artp_set_map + artp_update_features."""
    import art_planner_b200 as ap
    a, geom = cc.hole_free()
    c = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    obj = ap.MotionCostObjective(c)
    obj.setWeights(costnet.make_state_dict(seed=5))
    for mode in (0, 1):
        obj.setMode(mode)
        c.setMap(synth_map(a, geom))
        c.updateHeightField()
        obj.updateFeatures()
        want = obj.features()
        obj.updateFeaturesRaw(a, *geom)
        assert np.array_equal(obj.features(), want), mode
    obj.setMode(0)


def dump(planner):
    import ctypes as C
    h = planner._c.handle
    nv, ne = C.c_size_t(0), C.c_size_t(0)
    h.check(h.lib.artp_roadmap_get(h.h, 0, None, None, 0, None, C.byref(nv), C.byref(ne)))
    cost, flags = np.empty(ne.value), np.empty(ne.value, np.uint8)
    h.check(h.lib.artp_roadmap_get_edge_costs(h.h, 0, cost.ctypes.data, flags.ctypes.data, None))
    return cost, flags


def run_plans(planner, qs):
    out = []
    for s, g in qs:
        status = planner.plan(s, g)
        info = planner.info()
        for k in [k for k in info if k.startswith("ms_")]:
            info.pop(k)
        path = planner.getSolutionPath() if status == planner.SOLVED else np.zeros((0, 7))
        out.append((status, info, path, dump(planner)))
    return out


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def planners(network, n=2, **kw):
    import art_planner_b200 as ap
    from art_planner_b200.checker import _Handle
    c = rc.make_case("gentle_inf")
    out = []
    for _ in range(n):
        chk = ap.StateValidityChecker(c.rp, handle=_Handle(c.rp, 0, risk_threshold=0.6))
        ap.MotionCostObjective(chk).setWeights(costnet.make_state_dict(seed=5, network=network))
        out.append((chk, ap.Planner(chk, pc.small_params(seed=41, **kw))))
    return c, out


@pytest.mark.parametrize("busy", [False, True], ids=["alone", "beside-another-handle"])
@pytest.mark.parametrize("network", ["light", "full"])
def test_planner_cost_map_from_raw_equals_chained_calls(network, busy):
    """set_map_raw with cost_map_from_raw = 1, then plan, equals set_map_raw with 0, artp_update_features_raw of the
    raw elevation, then plan: statuses, paths, info records and every roadmap edge cost, bit for bit."""
    import art_planner_b200 as ap
    c, [(c1, p1), (c2, p2)] = planners(network)
    p1.parameters.cost_map_from_raw = 1
    m = c.m
    e, t, _, _ = pc.raw_layers(m, holes=0.02)
    stop, errors = threading.Event(), []
    if busy:                                           # a third handle planning on the same device meanwhile
        _, [(c3, p3)] = planners(network, n=1)
        p3.setMapRaw(e, t, m.res, m.cx, m.cy)
        qs3 = pc.queries(c3, 2, 9, 0.4 * min(m.length))

        def work():
            try:
                k = 0
                while not stop.is_set() and k < 50:
                    p3.parameters.clear_roadmap = k % 2
                    p3.plan(*qs3[k % 2])
                    k += 1
            except Exception as ex:                   # surfaced below
                errors.append(ex)
        th = threading.Thread(target=work)
        th.start()
    try:
        p1.setMapRaw(e, t, m.res, m.cx, m.cy)
        p2.setMapRaw(e, t, m.res, m.cx, m.cy)
        ap.MotionCostObjective(c2).updateFeaturesRaw(e, m.res, m.cx, m.cy)
        f1, f2 = ap.MotionCostObjective(c1).features(), ap.MotionCostObjective(c2).features()
        assert np.array_equal(f1, f2)
        qs = pc.queries(c1, 3, 5, min(4.0, 0.4 * min(m.length)))
        r1, r2 = run_plans(p1, qs), run_plans(p2, qs)
    finally:
        stop.set()
        if busy:
            th.join()
    assert not errors, errors
    assert same(r1, r2)
    assert {r[0] for r in r1} <= {p1.SOLVED, p1.NOT_SOLVED, p1.INVALID_START, p1.INVALID_GOAL}
    assert len(r1[0][3][0]) > 0                        # the first plan priced a roadmap with the learned cost


def test_refused_calls_keep_map_and_features():
    import art_planner_b200 as ap
    c, [(c1, p1)] = planners("light", n=1)
    p1.parameters.cost_map_from_raw = 1
    m = c.m
    e, t, _, _ = pc.raw_layers(m, holes=0.02)
    p1.setMapRaw(e, t, m.res, m.cx, m.cy)
    obj = ap.MotionCostObjective(c1)
    feat, space = obj.features(), p1.space()
    qs = pc.queries(c1, 1, 5, min(4.0, 0.4 * min(m.length)))
    bad = e.copy(order="F")
    bad[10, 10] = np.inf
    for call in (lambda: p1.setMapRaw(bad, t, m.res, m.cx, m.cy),
                 lambda: p1.setMap(bad, t, np.nan_to_num(bad, posinf=0.0), np.nan_to_num(t), m.res, m.cx, m.cy),
                 lambda: obj.updateFeaturesRaw(bad, m.res, m.cx, m.cy),
                 lambda: on_device(obj.updateFeaturesRaw, bad, m.res, m.cx, m.cy),
                 lambda: obj.updateFeaturesRaw(np.full(e.shape, np.nan, np.float32), m.res, m.cx, m.cy)):
        with pytest.raises(ap.ArtpError) as ex:
            call()
        assert ex.value.code == capi.ARTP_E_INVALID
        assert np.array_equal(obj.features(), feat)
        sp = p1.space()
        assert list(sp.low) == list(space.low) and list(sp.high) == list(space.high)
    assert p1.plan(*qs[0]) in (p1.SOLVED, p1.NOT_SOLVED, p1.INVALID_START, p1.INVALID_GOAL)
    p1.parameters.cost_map_from_raw = 2
    with pytest.raises(ap.ArtpError):
        p1.setMapRaw(e, t, m.res, m.cx, m.cy)
    assert ap.Planner.params().cost_map_from_raw == 0
    nw = ap.MotionCostObjective(ap.StateValidityChecker(synth.PARAMS_YAML, device=0))
    with pytest.raises(ap.ArtpError) as ex:
        nw.updateFeaturesRaw(e, m.res, m.cx, m.cy)
    assert ex.value.code == capi.ARTP_E_NOWEIGHTS
