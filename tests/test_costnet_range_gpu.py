"""GPU (-m gpu): the motion-cost network across its input range, against the float64 restatement (oracle/cnn_oracle.py).

Trunk: both networks, both kernel paths (setMode(0) wgmma with the fp16 hi/lo split, setMode(1) fp32 CUDA cores), on
trained-like (calibrated) weights over elevations from 1 mm noise to +4000 m, and on weight variants from 1e-3 to 10x
scales, near-dead, tiny and all-zero channels. Every feature must lie within the per-element bound of
oracle.cnn_oracle.trunk_error_bound (its docstring derives it: 2^-22 of |a| (*) |w|, of the bias and of the
accumulator chain's partial sums per layer, earlier layers' errors carried in quadrature), which the fp32 torch module
must meet too. A case whose activations leave the fp16 range of the split must instead make updateFeatures raise
ARTP_E_LIMIT on the wgmma path, and leave no features behind. Head: the queries' edges (clamped start cells, the yaw
wrap, zero-length edges, far off-origin maps, the truncated row bias, the block-size switch) against the float64 head.
"""
import math

import numpy as np
import pytest
import torch

from art_planner_b200 import costnet, synth
from oracle import cnn_oracle as co

pytestmark = pytest.mark.gpu
NETS = ["light", "full"]

# elevation cases (calibrated weights): name -> map
ELEVATIONS = {
    "c4-range": lambda: synth.make_fbm_map(256, 256, 0.04, seed=2, amp=0.6),
    "offset-50": lambda: _offset(synth.make_fbm_map(256, 256, 0.04, seed=2, amp=0.6), -50.0),
    "offset+300": lambda: _offset(synth.make_fbm_map(256, 256, 0.04, seed=2, amp=0.6), 300.0),
    "offset+1000": lambda: _offset(synth.make_fbm_map(256, 256, 0.04, seed=2, amp=0.6), 1000.0),
    "offset+4000": lambda: _offset(synth.make_fbm_map(256, 256, 0.04, seed=2, amp=0.6), 4000.0),
    "flat": lambda: synth.make_flat_map(256, 256, 0.04, height=0.37),
    "noise-1mm": lambda: synth.make_fbm_map(256, 256, 0.04, seed=3, amp=0.001, n_walls=0),
    "steep-5m": lambda: synth.make_fbm_map(256, 256, 0.04, seed=4, amp=5.0),
    "300x260+1000": lambda: _offset(synth.make_fbm_map(300, 260, 0.04, seed=2, amp=0.6), 1000.0),
}
# weight cases (c4-range map): name -> (calibrated_state_dict variant, value, trunk layers it applies to)
WEIGHTS = {
    "calibrated": (None, 1.0, range(6)),
    "wscale-1e-3": ("wscale", 1e-3, range(6)), "wscale-10": ("wscale", 10.0, range(6)),
    "gamma-1e-3": ("gamma", 1e-3, range(6)), "gamma-10": ("gamma", 10.0, range(6)),
    "dead-flatten-300": ("dead", 300.0, (5,)), "dead-all-300": ("dead", 300.0, range(6)),
    "tiny-1e-6": ("tiny", 1e-6, range(6)), "zero": ("zero", 0.0, range(6)),
}


def _offset(m, dz):
    import dataclasses
    return dataclasses.replace(m, elevation=np.asfortranarray(m.elevation + np.float32(dz)),
                               elevation_masked=np.asfortranarray(m.elevation_masked + np.float32(dz)))


def _objective(m, sd):
    import art_planner_b200 as ap
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    obj = ap.MotionCostObjective(chk)
    obj.setWeights(sd)
    return obj


@pytest.fixture(scope="module", autouse=True)
def built():
    from art_planner_b200 import build
    build.build()


def _check_case(net, map_name, weight_name):
    import art_planner_b200 as ap
    from art_planner_b200 import capi
    variant, value, layers = WEIGHTS[weight_name]
    sd = co.calibrated_state_dict(5, net, variant, value, layers=layers)
    m = ELEVATIONS[map_name]()
    E = co.cnn_input_from_layer(m.elevation)
    ref, bound, site_max = co.trunk_error_bound(sd, E, device="cuda")
    ref, bound = ref.permute(1, 2, 0).cpu(), bound.permute(1, 2, 0).cpu()
    overflow = max(site_max) >= co.FP16_OVERFLOW
    f32 = co.CostNetOracle(sd).features(E).permute(1, 2, 0).double()
    r32 = float(((f32 - ref).abs() / bound).max())
    assert r32 < 1.0, f"fp32 torch module outside the bound ({r32:.3g}): the case is not well-conditioned"
    obj = _objective(m, sd)
    q = costnet.make_queries(m, 4096, seed=6)
    lx, ly = m.length
    head64 = co.CostNetOracle(sd, dtype=torch.float64)
    for mode in (0, 1):
        obj.setMode(mode)
        if mode == 0 and overflow:
            with pytest.raises(ap.ArtpError) as ei:
                obj.updateFeatures()
            assert ei.value.code == capi.ARTP_E_LIMIT and "init_conv" in str(ei.value)
            with pytest.raises(ap.ArtpError):
                obj.costQuery(q)                              # no features survive the failed update
            print(f"{net:5s} {map_name:13s} {weight_name:17s} mode 0: ARTP_E_LIMIT (split-site max |a| "
                  f"{max(site_max):.3g})")
            continue
        obj.updateFeatures()
        got = torch.from_numpy(obj.features()).double()
        assert got.shape == ref.shape
        assert torch.isfinite(got).all()
        err = (got - ref).abs()
        ratio = float((err / bound).max())
        per_channel = float((err.amax(dim=(0, 1)) / ref.abs().amax(dim=(0, 1)).clamp_min(1e-30)).max())
        print(f"{net:5s} {map_name:13s} {weight_name:17s} mode {mode}: worst channel max|err|/max|ref_c| "
              f"{per_channel:.2e}, max err/bound {ratio:.3f}, fp32 module {r32:.3f}, bound/max|ref| "
              f"{float(bound.max() / ref.abs().max()):.2e}")
        assert ratio <= 1.0, (mode, ratio)
        cost = obj.costQuery(q)
        want = head64.query(got.permute(2, 0, 1), q, m.res, lx, ly, m.cx, m.cy)
        assert np.allclose(cost, want, rtol=1e-4, atol=1e-5), float(np.abs(cost - want).max())


@pytest.mark.parametrize("map_name", list(ELEVATIONS))
@pytest.mark.parametrize("net", NETS)
def test_trunk_across_elevations(net, map_name):
    _check_case(net, map_name, "calibrated")


@pytest.mark.parametrize("weight_name", [w for w in WEIGHTS if w != "calibrated"])
@pytest.mark.parametrize("net", NETS)
def test_trunk_across_weight_ranges(net, weight_name):
    _check_case(net, "c4-range", weight_name)


# ---------------------------------------------------------------------------------------------------------------------
# Head at its input edges: the device's costs against the float64 head over the device's own features, so that every
# difference is the head's (index arithmetic, yaw wrap, fp32 math).
def _head_env(net, m):
    sd = co.calibrated_state_dict(5, net)
    obj = _objective(m, sd)
    obj.updateFeatures()
    feats = torch.from_numpy(obj.features()).permute(2, 0, 1).double()
    return obj, feats, co.CostNetOracle(sd, dtype=torch.float64)


def _compare(obj, feats, head64, m, q):
    q = np.ascontiguousarray(q, dtype=np.float32)
    lx, ly = m.length
    got = obj.costQuery(q)
    want = head64.query(feats, q, m.res, lx, ly, m.cx, m.cy)
    assert np.allclose(got, want, rtol=1e-4, atol=1e-5), float(np.abs(got - want).max())


def _start_for_index(m, rr, axis):
    """The map-frame start coordinate whose feature index (rr in the head's formula) is `rr`, before float32."""
    lx, ly = m.length
    bias = int(((lx if axis == 0 else ly) / m.res - 48) / 2 * 0.5)
    return (rr - bias) * 2 * m.res + (m.cx if axis == 0 else m.cy)


@pytest.mark.parametrize("net", NETS)
def test_head_start_cells_at_and_beyond_the_clamp(net):
    m = synth.make_fbm_map(256, 256, 0.04, seed=2, amp=0.6)
    obj, feats, head64 = _head_env(net, m)
    hf, wf = feats.shape[1], feats.shape[2]
    rows = []
    for axis, n in ((0, hf), (1, wf)):
        for rr in (1.0, n - 2.0, -5.0, n + 5.0, 0.0, n - 1.0, 1.5, n - 2.5):
            c = np.float32(_start_for_index(m, rr, axis))
            for s in (np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf))):
                xy = [m.cx, m.cy]
                xy[axis] = float(s)
                rows.append([xy[0] + 0.2, xy[1] - 0.1, 0.3, xy[0], xy[1], -0.4])
    for sx in (m.cx - 50.0, m.cx + 50.0):                    # far outside on both sides of both axes
        for sy in (m.cy - 50.0, m.cy + 50.0):
            rows.append([sx, sy, 1.0, sx, sy, 2.0])
    _compare(obj, feats, head64, m, np.array(rows))


@pytest.mark.parametrize("net", NETS)
def test_head_yaw_wrap_and_zero_length_edges(net):
    m = synth.make_fbm_map(256, 256, 0.04, seed=2, amp=0.6)
    obj, feats, head64 = _head_env(net, m)
    pi32 = np.float32(math.pi)
    dyaws = [pi32, np.nextafter(pi32, np.float32(0)), np.nextafter(pi32, np.float32(4)), np.float32(2 * math.pi),
             np.float32(math.pi) * 2, np.nextafter(np.float32(2 * math.pi), np.float32(0))]
    dyaws += [-d for d in dyaws] + [np.float32(0.0)]
    rows = []
    for syaw in (np.float32(0.0), np.float32(-math.pi), np.float32(1.0)):
        for d in dyaws:
            for length in (0.0, 0.3):
                rows.append([m.cx + length, m.cy, np.float32(syaw + d), m.cx, m.cy, syaw])
    q = np.array(rows, dtype=np.float32)
    assert (q[:, 0] == q[:, 3]).any() and (q[:, 1] == q[:, 4]).all()   # zero-length edges: atan2f(0, 0)
    _compare(obj, feats, head64, m, q)


@pytest.mark.parametrize("net", NETS)
def test_head_far_off_origin_map(net):
    """cx, cy ~ 1e4 m: the float32 request rows carry ~1 mm steps; the float64 head gets the same float32 rows."""
    m = synth.make_fbm_map(256, 256, 0.04, seed=2, amp=0.6, cx=10000.3, cy=-9999.7)
    obj, feats, head64 = _head_env(net, m)
    _compare(obj, feats, head64, m, costnet.make_queries(m, 4096, seed=11))


@pytest.mark.parametrize("rows,cols,res", [(116, 256, 0.04), (464, 128, 0.04), (256, 172, 0.05), (128, 88, 0.06)])
def test_head_truncated_row_bias(rows, cols, res):
    """rows * res / res < rows in float64 for these sizes, so the (int) of the head's row / column bias drops by one.
    The library restates that truncating formula; this pins agreement with the float64 restatement on such maps.
    Whether grid_map's stored length is exactly size * res is not pinned here (grid_map is not in this tree)."""
    assert int((rows * res / res - 48) / 2 * 0.5) != int((rows - 48) / 2 * 0.5) or \
        int((cols * res / res - 48) / 2 * 0.5) != int((cols - 48) / 2 * 0.5)
    m = synth.make_fbm_map(rows, cols, res, seed=2, amp=0.6)
    obj, feats, head64 = _head_env("light", m)
    _compare(obj, feats, head64, m, costnet.make_queries(m, 2048, seed=12))


@pytest.mark.parametrize("net", NETS)
def test_head_batch_sizes_around_the_block_switch(net):
    """n <= sm_count * 128 runs 32-thread blocks, larger batches 128-thread blocks."""
    m = synth.make_fbm_map(256, 256, 0.04, seed=2, amp=0.6)
    obj, feats, head64 = _head_env(net, m)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    for n in (1, 31, 33, sm * 128 - 1, sm * 128, sm * 128 + 1):
        _compare(obj, feats, head64, m, costnet.make_queries(m, n, seed=13))
