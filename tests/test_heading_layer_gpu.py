"""GPU (-m gpu): the valid-heading layer (artp_valid_heading_layer[_device]) bit for bit against its definition, the
composition artp_pose_from_2d -> artp_check_poses on the same states, on the case maps and the benchmark's 1000 x 1000 maps
(several chunks); against the fixture the compiled reference wrote; host against device form; its refusals; and a layer
call between two plans that leaves the planner's results as they were."""
import os

import numpy as np
import pytest

import heading_layer_cases as hlc
import planner_cases as pc
import roadmap_cases as rc
from art_planner_b200 import capi

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATE_TOL = 1e-12      # CUDA vs numpy atan2 / sin / cos in the projected quaternion (test_start_goal_gpu.py's tolerance)


@pytest.fixture(scope="module")
def ap():
    import art_planner_b200
    from art_planner_b200 import build
    build.build()
    return art_planner_b200


def _checker(ap, m, pk):
    chk = ap.StateValidityChecker(hlc.PARAMS[pk], device=0)
    chk.setMap(m)
    chk.updateHeightField()
    chk.estimateNormals(hlc.normal_radius(hlc.PARAMS[pk]), want_host=False)
    return chk


def _composed(chk, m, yaws, cells=None):
    """The definition through the public calls: artp_pose_from_2d, then artp_check_poses, packed per cell."""
    proj, inside = chk.poseFrom2D(hlc.yaw_states(m, yaws, cells))
    assert inside.all()
    return hlc.pack(chk.isValidBatch(proj), len(yaws), (-1,) if cells is not None else (m.rows, m.cols))


@pytest.mark.parametrize("pk", ["yaml", "header"])
@pytest.mark.parametrize("mk", ["fixture", "terraces", "spikes", "fbm_rough", "r1"])
def test_layer_equals_composition_on_case_maps(ap, mk, pk):
    m = hlc.MAPS[mk]()
    chk = _checker(ap, m, pk)
    for hk, yaws in hlc.HEADINGS.items():
        got = chk.validHeadingLayer(yaws)
        assert got.dtype == np.uint32 and got.shape == (m.rows, m.cols) and got.flags.f_contiguous
        assert np.array_equal(got, _composed(chk, m, yaws)), (mk, pk, hk)
        assert (got >> np.uint32(len(yaws)) == 0).all() if len(yaws) < 32 else True
        if hk == "ulp":
            bits = (got[..., None] >> np.arange(len(yaws), dtype=np.uint32)) & 1
            for k in hlc.ULP_SAME:
                assert np.array_equal(bits[..., k], bits[..., 0])


@pytest.mark.parametrize("kind", ["gentle", "rough"])
def test_layer_equals_composition_on_the_benchmark_maps(ap, kind):
    """1000 x 1000 cells x 7 headings = 7 M poses: four chunks of whole cells, none a power-of-two size."""
    m = hlc.large_map(kind)
    chk = _checker(ap, m, "yaml")
    yaws = np.array([0.0, 0.9, -1.7, 2.6, np.pi, -0.2, 1.4])
    got = chk.validHeadingLayer(yaws)
    cells = np.arange(0, m.rows * m.cols, 37)                   # 27 028 cells, every row and column met
    assert len(cells) >= 20000
    want = _composed(chk, m, yaws, cells)
    assert np.array_equal(got.ravel(order="F")[cells], want)
    share = np.bitwise_count(want).mean() / len(yaws)
    assert 0.05 < share < 0.95


@pytest.mark.parametrize("name,mk,pk,hk", hlc.GOLDEN_CASES, ids=[c[0] for c in hlc.GOLDEN_CASES])
def test_layer_equals_reference_fixture(ap, name, mk, pk, hk):
    g = np.load(os.path.join(ROOT, "tests", "golden", "heading_layer.npz"))
    m, yaws = hlc.MAPS[mk](), hlc.HEADINGS[hk]
    chk = _checker(ap, m, pk)
    assert np.array_equal(chk.validHeadingLayer(yaws), g[name + "/masks"])
    cells = g[name + "/pose_cells"]
    got, inside = chk.poseFrom2D(hlc.yaw_states(m, yaws, cells))
    want = g[name + "/poses"]
    assert inside.all() and np.array_equal(got[:, :3], want[:, :3])
    assert np.abs(got[:, 3:] - want[:, 3:]).max() < STATE_TOL


def test_host_and_device_forms_agree(ap):
    import torch
    m = hlc.MAPS["r1"]()
    chk = _checker(ap, m, "yaml")
    yaws = hlc.HEADINGS["even32"]
    want = chk.validHeadingLayer(yaws)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        out = torch.full((m.cols, m.rows), -1, dtype=torch.int32, device="cuda").t()
        assert chk.validHeadingLayer(yaws, out=out) is out
    side.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want)
    assert (want == 0xFFFFFFFF).any() or (want != 0).any()


def test_errors_leave_the_checker_as_it_was(ap):
    import torch
    m = hlc.MAPS["fixture"]()
    bare = ap.StateValidityChecker(hlc.PARAMS["yaml"], device=0)
    lib, h = bare.handle.lib, bare.handle.h
    mask = np.zeros(m.rows * m.cols, np.uint32)
    d_mask = torch.zeros(m.rows * m.cols, dtype=torch.int32, device="cuda")
    y = np.zeros(4)

    def rc_of(yaws, n, out):
        return lib.artp_valid_heading_layer(h, None if yaws is None else yaws.ctypes.data, n,
                                            None if out is None else out.ctypes.data)

    assert rc_of(y, 4, mask) == capi.ARTP_E_NOMAP
    assert lib.artp_valid_heading_layer_device(h, y.ctypes.data, 4, d_mask.data_ptr(), None) == capi.ARTP_E_NOMAP
    bare.setMap(m)
    bare.updateHeightField()
    states = hlc.yaw_states(m, [0.4, -2.0])
    before = bare.isValidBatch(states)
    assert rc_of(y, 4, mask) == capi.ARTP_E_INVALID                       # no normals yet
    bare.estimateNormals(hlc.normal_radius(hlc.PARAMS["yaml"]), want_host=False)
    proj_before = bare.poseFrom2D(states)[0]
    for yaws, n, out in ((y, 0, mask), (np.zeros(33), 33, mask), (y, -1, mask), (None, 4, mask), (y, 4, None),
                         (np.array([0.0, np.nan]), 2, mask), (np.array([np.inf]), 1, mask), (np.array([-np.inf]), 1, mask)):
        assert rc_of(yaws, n, out) == capi.ARTP_E_INVALID, (n, yaws)
        assert lib.artp_valid_heading_layer_device(h, None if yaws is None else yaws.ctypes.data, n,
                                                   None if out is None else d_mask.data_ptr(), None) == capi.ARTP_E_INVALID
    torch.cuda.synchronize()
    assert not mask.any() and not d_mask.any()                            # refused before any device work
    assert np.array_equal(bare.isValidBatch(states), before)
    assert np.array_equal(bare.poseFrom2D(states)[0], proj_before)
    full = bare.validHeadingLayer(np.zeros(32))                           # both ends of 1..32 are accepted
    assert np.array_equal(full, bare.validHeadingLayer([0.0]) * np.uint32(0xFFFFFFFF))
    bare.updateHeightField(window=(0, 100))                               # a map window
    assert rc_of(y, 4, mask) == capi.ARTP_E_INVALID


def test_layer_between_plans_leaves_the_planner_unchanged(ap):
    """set_map_raw leaves normals on the device: the layer works right after it, and a layer call between two plans
    changes no path, counter or cost against a planner that made none."""
    from art_planner_b200 import costnet
    from art_planner_b200.checker import _Handle
    c = rc.make_case("gentle_inf")
    m = c.m
    e, t, _, _ = pc.raw_layers(m, holes=0.02)
    runs = []
    for layer_calls in (False, True):
        chk = ap.StateValidityChecker(c.rp, handle=_Handle(c.rp, 0, risk_threshold=0.6))
        ap.MotionCostObjective(chk).setWeights(costnet.make_state_dict(seed=5, network="light"))
        p = ap.Planner(chk, pc.small_params(seed=41))
        p.setMapRaw(e, t, m.res, m.cx, m.cy)
        qs = pc.queries(chk, 3, 5, min(4.0, 0.4 * min(m.length)))
        out, layers = [], []
        for s, g in qs:
            if layer_calls:
                layers.append(chk.validHeadingLayer(hlc.HEADINGS["even8"]))
            status = p.plan(s, g)
            info = p.info()
            for k in [k for k in info if k.startswith("ms_")]:
                info.pop(k)
            out.append((status, info, p.getSolutionPath() if status == p.SOLVED else np.zeros((0, 7))))
        runs.append(out)
        if layer_calls:
            assert all(np.array_equal(x, layers[0]) for x in layers)        # the map did not change between plans
            assert (layers[0] != 0).any() and (layers[0] != 0xFF).any()
    assert _same(runs[0], runs[1])
    assert runs[0][0][1]["n_vertices"] > 0                                # the first plan grew a roadmap


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)
