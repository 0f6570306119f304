"""GPU (-m gpu): the box verdicts (artp_box_verdicts[_device]) and the box-verdict layer (artp_box_verdict_layer[_device])
bit for bit against the fixture the compiled reference wrote and the port oracle, on the case maps in both pipeline modes
and on the benchmark's 1000 x 1000 maps; the words against artp_check_poses; host against device form; the layer against
artp_pose_from_2d -> artp_box_verdicts and against the valid-heading layer, up to 4000 x 4000; the refusals; the
plane-store overflow; and calls between plans and checks that leave those calls' results and counters as they were."""
import os

import numpy as np
import pytest

import box_verdict_cases as bvc
import cases
import heading_layer_cases as hlc
import planner_cases as pc
import roadmap_cases as rc
from art_planner_b200 import capi, synth
from oracle import box_verdict_oracle as bvo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ap():
    import art_planner_b200
    from art_planner_b200 import build
    build.build()
    return art_planner_b200


@pytest.fixture(scope="module")
def bv_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "box_verdicts.npz"))


def _checker(ap, m, p, normals=False):
    chk = ap.StateValidityChecker(p, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    if normals:
        chk.estimateNormals(hlc.normal_radius(p), want_host=False)
    return chk


@pytest.mark.parametrize("mode", [0, 1], ids=["warp+group", "group-only"])
@pytest.mark.parametrize("mk", sorted(cases.MAPS))
def test_words_equal_reference_fixture_and_port(ap, bv_golden, port_lib, mk, mode):
    m = cases.MAPS[mk]()
    states = bvc.samples(m)
    for name, mk2, pk, u in bvc.CASES:
        if mk2 != mk:
            continue
        p = bvc.params(pk, u)
        chk = _checker(ap, m, p)
        chk.setMode(mode)
        got = chk.boxVerdicts(states)
        valid = chk.isValidBatch(states)
        o = port_lib.Oracle(p, "port")
        o.set_map(m)
        assert got.dtype == np.uint16 and np.array_equal(got, bv_golden[name + "/why"]), (name, mode)
        assert np.array_equal(got, bvo.box_verdicts(o, p, m, states)), (name, mode)
        assert np.array_equal((got & 0x1F) == 0, valid != 0), (name, mode)
        if mode == 1:
            st = chk.stats()
            assert st["last_deferred"] == st["last_queued_boxes"] > 0


@pytest.mark.parametrize("kind", ["gentle", "rough"])
def test_words_on_the_benchmark_maps(ap, port_lib, kind):
    """2^20 states, one chunk of the pipeline, all five boxes queued where undecided; a strided subset against the port."""
    m = hlc.large_map(kind)
    chk = _checker(ap, m, synth.PARAMS_YAML)
    n = 1 << 20
    states = synth.make_terrain_poses(m, n, seed=17, z_range=0.25, roll_pert=0.4, pitch_pert=0.4, normal_cells=12)
    got = chk.boxVerdicts(states)
    assert np.array_equal((got & 0x1F) == 0, chk.isValidBatch(states) != 0)
    sub = np.arange(0, n, 41)
    o = port_lib.Oracle(synth.PARAMS_YAML, "port")
    o.set_map(m)
    assert np.array_equal(got[sub], bvo.box_verdicts(o, synth.PARAMS_YAML, m, states[sub]))
    assert 0.05 < float(((got & 0x1F) == 0).mean()) < 0.95 and (np.bitwise_count(got & 0x1F) >= 2).any()


def test_words_agree_with_check_on_non_finite_and_off_map_states(ap, port_lib):
    m = cases.MAPS["fixture"]()
    for u in (1, 0):
        p = bvc.params("yaml", u)
        chk = _checker(ap, m, p)
        s = bvc.samples(m, seed=9)
        bad = s[:64].copy()
        bad[0::4, 0] = np.nan
        bad[1::4, 3:] = np.nan
        bad[2::4, 2] = np.inf
        bad[3::4, 1] = -np.inf
        far = s[64:128].copy()
        far[:, 0] += 50.0                                              # every box off the map
        states = np.concatenate([bad, far, s])
        got = chk.boxVerdicts(states)
        assert np.array_equal((got & 0x1F) == 0, chk.isValidBatch(states) != 0), u
        o = port_lib.Oracle(p, "port")
        o.set_map(m)
        assert np.array_equal(got, bvo.box_verdicts(o, p, m, states)), u
        assert np.all(got[64:128] >> 8 == 0x1F)
        assert np.all((got[64:128] & 0x1F) == (0x1E if u else 0))
        one = chk.boxVerdicts(states[:1])                              # n = 1: the pipeline, not the latency path
        assert np.array_equal(one, got[:1])


def test_host_and_device_forms_agree(ap):
    import torch
    m = cases.MAPS["spikes"]()
    chk = _checker(ap, m, synth.PARAMS_YAML)
    states = bvc.samples(m)
    want = chk.boxVerdicts(states)
    d_states = torch.from_numpy(states).cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out16 = torch.full((len(states),), -1, dtype=torch.int16, device="cuda")
        assert chk.boxVerdicts(d_states, out=out16) is out16
        outu = chk.boxVerdicts(d_states)
    side.synchronize()
    assert outu.dtype == torch.uint16
    assert np.array_equal(out16.cpu().numpy().view(np.uint16), want)
    assert np.array_equal(outu.view(torch.int16).cpu().numpy().view(np.uint16), want)


def test_counters_move_as_for_a_check_of_the_same_size(ap):
    import torch
    m = cases.MAPS["terraces"]()
    chk = _checker(ap, m, synth.PARAMS_YAML)
    d = torch.from_numpy(bvc.samples(m)).cuda()
    chk.isValidBatch(d)
    torch.cuda.synchronize()
    st0 = chk.stats()
    chk.boxVerdicts(d)
    torch.cuda.synchronize()
    st1 = chk.stats()
    assert st1["last_launches"] == st0["last_launches"] > 0
    assert st1["kernel_launches"] - st0["kernel_launches"] == st0["last_launches"]
    assert st1["poses_checked"] - st0["poses_checked"] == d.shape[0]
    assert st1["last_queued_boxes"] >= st0["last_queued_boxes"] > 0     # every undecided box is queued, not only those of valid poses


def _layer_composed(chk, m, yaw, cells=None):
    proj, inside = chk.poseFrom2D(hlc.yaw_states(m, [yaw], cells))
    assert inside.all()
    return chk.boxVerdicts(proj)


@pytest.mark.parametrize("pk", ["yaml", "header"])
@pytest.mark.parametrize("mk", ["fixture", "terraces", "spikes", "fbm_rough", "r1"])
def test_layer_equals_composition_and_heading_layer(ap, mk, pk):
    m = hlc.MAPS[mk]()
    chk = _checker(ap, m, hlc.PARAMS[pk], normals=True)
    for yaw in (0.0, 0.9, -2.6, np.pi):
        got = chk.boxVerdictLayer(yaw)
        assert got.dtype == np.uint16 and got.shape == (m.rows, m.cols) and got.flags.f_contiguous
        assert np.array_equal(got.ravel(order="F"), _layer_composed(chk, m, yaw)), (mk, pk, yaw)
        assert np.array_equal((got & 0x1F) == 0, (chk.validHeadingLayer([yaw]) & 1) != 0), (mk, pk, yaw)


@pytest.mark.parametrize("kind", ["gentle", "rough"])
def test_layer_on_the_benchmark_maps(ap, kind):
    m = hlc.large_map(kind)
    chk = _checker(ap, m, synth.PARAMS_YAML, normals=True)
    got = chk.boxVerdictLayer(1.1)
    cells = np.arange(0, m.rows * m.cols, 37)
    assert np.array_equal(got.ravel(order="F")[cells], _layer_composed(chk, m, 1.1, cells))
    assert np.array_equal((got & 0x1F) == 0, (chk.validHeadingLayer([1.1]) & 1) != 0)


def test_layer_at_4000(ap):
    """16 M cells: eight chunks of 2^21 poses."""
    m = synth.make_fbm_map(4000, 4000, 0.04, seed=2, amp=0.6)
    chk = _checker(ap, m, synth.PARAMS_YAML, normals=True)
    got = chk.boxVerdictLayer(-0.7)
    n = m.rows * m.cols
    rng = np.random.default_rng(4)
    r, c = np.arange(m.rows), np.arange(m.cols)
    border = np.concatenate([r, r + (m.cols - 1) * m.rows, c * m.rows, (m.rows - 1) + c * m.rows])
    cells = np.unique(np.concatenate([border, rng.integers(0, n, 30000), [0, m.rows - 1, n - m.rows, n - 1]]))
    assert np.array_equal(got.ravel(order="F")[cells], _layer_composed(chk, m, -0.7, cells))
    assert ((got & 0x1F) == 0).any() and ((got & 0x1F) != 0).any()


def test_refusals(ap):
    import torch
    m = hlc.MAPS["fixture"]()
    bare = ap.StateValidityChecker(hlc.PARAMS["yaml"], device=0)
    lib, h = bare.handle.lib, bare.handle.h
    states = bvc.samples(m)[:100]
    why = np.zeros(100, np.uint16)
    layer = np.zeros(m.rows * m.cols, np.uint16)
    d_states = torch.from_numpy(states).cuda()
    d_why = torch.zeros(100, dtype=torch.int16, device="cuda")
    d_layer = torch.zeros(m.rows * m.cols, dtype=torch.int16, device="cuda")
    assert lib.artp_box_verdicts(h, states.ctypes.data, 100, why.ctypes.data) == capi.ARTP_E_NOMAP
    assert lib.artp_box_verdicts_device(h, d_states.data_ptr(), 100, d_why.data_ptr(), None) == capi.ARTP_E_NOMAP
    assert lib.artp_box_verdict_layer(h, 0.0, layer.ctypes.data) == capi.ARTP_E_NOMAP
    assert lib.artp_box_verdict_layer_device(h, 0.0, d_layer.data_ptr(), None) == capi.ARTP_E_NOMAP
    bare.setMap(m)
    bare.updateHeightField()
    assert lib.artp_box_verdict_layer(h, 0.0, layer.ctypes.data) == capi.ARTP_E_INVALID          # no normals yet
    assert lib.artp_box_verdict_layer_device(h, 0.0, d_layer.data_ptr(), None) == capi.ARTP_E_INVALID
    bare.estimateNormals(hlc.normal_radius(hlc.PARAMS["yaml"]), want_host=False)
    assert lib.artp_box_verdicts(h, None, 100, why.ctypes.data) == capi.ARTP_E_INVALID
    assert lib.artp_box_verdicts(h, states.ctypes.data, 100, None) == capi.ARTP_E_INVALID
    assert lib.artp_box_verdicts_device(h, None, 100, d_why.data_ptr(), None) == capi.ARTP_E_INVALID
    assert lib.artp_box_verdicts_device(h, d_states.data_ptr(), 100, None, None) == capi.ARTP_E_INVALID
    assert lib.artp_box_verdict_layer(h, 0.0, None) == capi.ARTP_E_INVALID
    assert lib.artp_box_verdict_layer_device(h, 0.0, None, None) == capi.ARTP_E_INVALID
    for yaw in (np.nan, np.inf, -np.inf):
        assert lib.artp_box_verdict_layer(h, yaw, layer.ctypes.data) == capi.ARTP_E_INVALID
        assert lib.artp_box_verdict_layer_device(h, yaw, d_layer.data_ptr(), None) == capi.ARTP_E_INVALID
    torch.cuda.synchronize()
    assert not why.any() and not layer.any() and not d_why.any() and not d_layer.any()   # before any device work
    assert lib.artp_box_verdicts(h, states.ctypes.data, 0, None) == capi.ARTP_OK           # n = 0, as artp_check_poses
    bare.updateHeightField(window=(0, 100))                                                 # a map window
    assert lib.artp_box_verdicts(h, states.ctypes.data, 100, why.ctypes.data) == capi.ARTP_E_INVALID
    assert lib.artp_box_verdicts_device(h, d_states.data_ptr(), 100, d_why.data_ptr(), None) == capi.ARTP_E_INVALID
    assert lib.artp_box_verdict_layer(h, 0.0, layer.ctypes.data) == capi.ARTP_E_INVALID
    torch.cuda.synchronize()
    assert not why.any() and not d_why.any() and not layer.any()


def test_plane_store_overflow_fails_the_deferred_box(ap, bv_golden):
    """A zone that does not fit the plane store: the call returns ARTP_E_LIMIT and the deferred box counts as failing,
    as artp_check_poses treats it; no other bit moves."""
    import torch
    m = cases.MAPS["terraces"]()
    states = bvc.samples(m)
    truth = bv_golden["bv_terraces_yaml_u1/why"]
    chk = ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)
    chk.debugSetGroupCapacity(64)
    chk.setMap(m)
    chk.updateHeightField()
    chk.setMode(1)
    with pytest.raises(ap.ArtpError) as ei:
        chk.isValidBatch(states)
    assert ei.value.code == capi.ARTP_E_LIMIT
    valid = chk.isValidBatch(torch.from_numpy(states).cuda()).cpu().numpy()
    torch.cuda.synchronize()
    with pytest.raises(ap.ArtpError):
        chk.pollError()
    why = np.zeros(len(states), np.uint16)
    lib, h = chk.handle.lib, chk.handle.h
    assert lib.artp_box_verdicts(h, states.ctypes.data, len(states), why.ctypes.data) == capi.ARTP_E_LIMIT
    chk.pollError()
    assert np.array_equal((why & 0x1F) == 0, valid != 0)
    assert np.array_equal(why & truth, truth)                          # every true failure is still there
    assert np.array_equal(why >> 8, truth >> 8)
    extra = why & ~truth
    assert extra.any() and (extra & 1).any()                           # torso zones overflowed: their bit set
    d = chk.boxVerdicts(torch.from_numpy(states).cuda())
    torch.cuda.synchronize()
    with pytest.raises(ap.ArtpError) as ei:
        chk.pollError()
    assert ei.value.code == capi.ARTP_E_LIMIT
    assert np.array_equal(d.view(torch.int16).cpu().numpy().view(np.uint16), why)
    chk.debugSetGroupCapacity(0)
    chk.setMap(m)
    chk.updateHeightField()
    assert np.array_equal(chk.boxVerdicts(states), truth)
    chk.setMode(0)


def test_calls_between_checks_leave_them_unchanged(ap):
    """Check calls with verdict and layer calls between them -- on the same handle, and on a second handle on the same
    device -- give the verdicts and per-call counters of the same checks made without them."""
    import torch
    m = cases.MAPS["fbm_rough"]()
    m2 = cases.MAPS["terraces"]()
    batches = [synth.make_terrain_poses(m, 3000 + 500 * i, seed=40 + i) for i in range(3)]
    keys = ("last_launches", "last_queued_boxes", "last_queued_warp_stage", "last_queued_reach_stage", "last_deferred")
    runs = []
    for between in (False, True):
        chk = _checker(ap, m, synth.PARAMS_YAML, normals=True)
        other = _checker(ap, m2, synth.PARAMS_YAML, normals=True)
        out = []
        for b in batches:
            if between:
                chk.boxVerdicts(b)
                chk.boxVerdictLayer(0.3)
                other.boxVerdicts(torch.from_numpy(bvc.samples(m2)).cuda())
                other.boxVerdictLayer(-1.0)
            v = chk.isValidBatch(b)
            d = chk.isValidBatch(torch.from_numpy(b).cuda()).cpu().numpy()
            st = chk.stats()
            out.append((v, d, {k: st[k] for k in keys}))
        torch.cuda.synchronize()
        runs.append(out)
    for (v0, d0, s0), (v1, d1, s1) in zip(*runs):
        assert np.array_equal(v0, v1) and np.array_equal(d0, d1) and s0 == s1


def test_calls_between_plans_leave_the_planner_unchanged(ap):
    from art_planner_b200 import costnet
    from art_planner_b200.checker import _Handle
    c = rc.make_case("gentle_inf")
    m = c.m
    e, t, _, _ = pc.raw_layers(m, holes=0.02)
    runs = []
    for between in (False, True):
        chk = ap.StateValidityChecker(c.rp, handle=_Handle(c.rp, 0, risk_threshold=0.6))
        other = _checker(ap, cases.MAPS["spikes"](), c.rp, normals=True)
        ap.MotionCostObjective(chk).setWeights(costnet.make_state_dict(seed=5, network="light"))
        p = ap.Planner(chk, pc.small_params(seed=41))
        p.setMapRaw(e, t, m.res, m.cx, m.cy)
        qs = pc.queries(chk, 3, 5, min(4.0, 0.4 * min(m.length)))
        out = []
        for s, g in qs:
            if between:
                why = chk.boxVerdicts(np.stack([s, g]))
                assert why.shape == (2,)
                chk.boxVerdictLayer(0.5)
                other.boxVerdictLayer(0.5)
            status = p.plan(s, g)
            info = p.info()
            for k in [k for k in info if k.startswith("ms_")]:
                info.pop(k)
            out.append((status, info, p.getSolutionPath() if status == p.SOLVED else np.zeros((0, 7))))
        runs.append(out)
    assert _same(runs[0], runs[1])
    assert runs[0][0][1]["n_vertices"] > 0


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)
