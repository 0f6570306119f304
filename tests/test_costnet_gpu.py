"""GPU parity (-m gpu) of the learned motion cost (BASELINE configs[3]): feature map and costs against the fp32
evaluation of the reference module (golden file produced from the reference's own network_light.py) and against the
torch restatement in oracle/cnn_oracle.py. Tolerance from BASELINE.json: 1e-4 relative (plus 1e-5 absolute, because
two of the three outputs pass through a ReLU and are exactly 0 for part of the batch)."""
import os

import numpy as np
import pytest

import cases
from art_planner_b200 import costnet

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL, ATOL = 1e-4, 1e-5


@pytest.fixture(scope="module")
def setup():
    import art_planner_b200 as ap
    from art_planner_b200 import build, synth
    from oracle.cnn_oracle import CostNetOracle, cnn_input_from_layer
    build.build()
    m = cases.c4_map()
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    obj = ap.MotionCostObjective(chk)
    sd = costnet.make_state_dict(seed=5)
    obj.setWeights(sd)
    orc = CostNetOracle(sd)
    feat = orc.features(cnn_input_from_layer(m.elevation))
    golden = np.load(os.path.join(ROOT, "tests", "golden", "cnn_c4.npz"))
    assert abs(float(costnet.pack_blob(sd).astype(np.float64).sum()) - float(golden["blob_sum"])) < 1e-9, "weight generator drift"
    return m, obj, orc, feat, golden


@pytest.mark.parametrize("mode", [1, 0], ids=["cuda-core", "wgmma"])
def test_feature_map(setup, mode):
    m, obj, orc, feat, golden = setup
    obj.setMode(mode)
    obj.updateFeatures()
    got = obj.features()                      # [Hf, Wf, 48]
    ref = feat.permute(1, 2, 0).numpy()
    assert got.shape == ref.shape == (104, 104, 48)
    scale = float(np.abs(ref).max())
    err = float(np.abs(got - ref).max()) / scale
    # 10 800-term fp32 accumulations in different orders (and the tensor core's fp32 accumulator): 1e-4 of the max
    tol = 1e-5 if mode == 1 else 1e-4
    assert err < tol, f"feature map max error {err:.3e} of max |f| = {scale:.3f}"
    assert np.allclose(got[::13, ::13].transpose(2, 0, 1), golden["feat_sample"], rtol=1e-4, atol=tol * scale)
    obj.setMode(0)


def test_costs_match_reference_module(setup):
    import torch
    m, obj, orc, feat, golden = setup
    obj.setMode(0)
    obj.updateFeatures()
    q = costnet.make_queries(m, 4096, seed=6)
    got = obj.costQuery(q)
    ref = golden["cost"]
    assert np.allclose(got, ref, rtol=RTOL, atol=ATOL), float(np.abs(got - ref).max())
    lx, ly = m.length
    assert np.allclose(got, orc.query(feat, q, m.res, lx, ly, m.cx, m.cy), rtol=RTOL, atol=ATOL)
    dev = obj.costQuery(torch.from_numpy(q).cuda())
    torch.cuda.synchronize()
    assert np.array_equal(dev.cpu().numpy(), got)
    cost, feas = obj.getCost(got)
    assert np.allclose(cost, got[:, 1] * 1.0 + got[:, 2] * 5.0, rtol=1e-6)
    assert np.array_equal(feas, (got[:, 2] <= 0.5).astype(np.uint8))
    assert obj.costQuery(np.zeros((0, 6), np.float32)).shape == (0, 3)


def test_errors_without_weights_or_features():
    import art_planner_b200 as ap
    from art_planner_b200 import synth
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    obj = ap.MotionCostObjective(chk)
    with pytest.raises(ap.ArtpError):
        obj.updateFeatures()            # no map
    chk.setMap(cases.c4_map()); chk.updateHeightField()
    with pytest.raises(ap.ArtpError):
        obj.updateFeatures()            # no weights
    obj.setWeights(costnet.make_state_dict(seed=5))
    with pytest.raises(ap.ArtpError):
        obj.costQuery(np.zeros((4, 6), np.float32))   # features not computed
    for mode in (2, 4, 8, 12):
        with pytest.raises(ap.ArtpError):
            obj.setMode(mode)           # bit 0 is the only mode bit


@pytest.mark.parametrize("shape", [(300, 260), (1000, 1000), (121, 97)], ids=["300x260-partial-tiles", "1000x1000-metric-map", "121x97-odd"])
def test_feature_map_other_sizes(shape):
    """The trunk away from the 256x256 patch: partial output tiles in both axes, odd extents, and the metric's full
    1000x1000 map (feature map 476 x 476), against the fp32 torch restatement of network_light.py:78-110."""
    import art_planner_b200 as ap
    from art_planner_b200 import synth
    from oracle.cnn_oracle import CostNetOracle, cnn_input_from_layer
    rows, cols = shape
    m = synth.make_fbm_map(rows, cols, 0.04, seed=2, amp=0.6)
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m); chk.updateHeightField()
    obj = ap.MotionCostObjective(chk)
    sd = costnet.make_state_dict(seed=5)
    obj.setWeights(sd)
    obj.updateFeatures()
    got = obj.features()
    ref = CostNetOracle(sd).features(cnn_input_from_layer(m.elevation)).permute(1, 2, 0).numpy()
    assert got.shape == ref.shape == ((cols - 48) // 2, (rows - 48) // 2, 48) or got.shape == ref.shape
    scale = float(np.abs(ref).max())
    assert float(np.abs(got - ref).max()) / scale < 1e-4
    q = costnet.make_queries(m, 2048, seed=6)
    lx, ly = m.length
    feat = CostNetOracle(sd).features(cnn_input_from_layer(m.elevation))
    assert np.allclose(obj.costQuery(q), CostNetOracle(sd).query(feat, q, m.res, lx, ly, m.cx, m.cy), rtol=RTOL, atol=ATOL)


def test_error_against_the_fp16_module_as_shipped(setup):
    """BASELINE.md section 3: the reference runs its module in fp16 (predictor.py:22). Report how far that evaluation is
    from the fp32 one and check that this implementation is closer to fp32 than fp16 is (it must be: 1e-4 vs ~1e-3)."""
    import torch
    m, obj, orc, feat, golden = setup
    from oracle.cnn_oracle import CostNetOracle, cnn_input_from_layer
    sd = costnet.make_state_dict(seed=5)
    h = CostNetOracle(sd)
    h.p = {k: v.cuda().half() for k, v in h.p.items()}
    E = torch.as_tensor(cnn_input_from_layer(m.elevation)).cuda().half()
    import torch.nn.functional as F
    with torch.no_grad():
        t = E[None, None]
        t = h._conv_bn(t, "init_conv1", "init_conv1_bn")
        t = F.leaky_relu(h._conv_bn(t, "init_conv2", "init_conv2_bn"), 0.3); t = F.max_pool2d(t, (2, 2), stride=2)
        t = F.leaky_relu(h._conv_bn(t, "init_conv3", "init_conv3_bn"), 0.3)
        t = F.leaky_relu(h._conv_bn(t, "init_conv4", "init_conv4_bn"), 0.3); t = F.max_pool2d(t, (3, 3), stride=1)
        t = F.leaky_relu(h._conv_bn(t, "init_conv5", "init_conv5_bn"), 0.3)
        t = F.leaky_relu(h._conv_bn(t, "init_flatten", "init_flatten_bn"), 0.3)
    f16 = t[0].float().cpu().permute(1, 2, 0).numpy()
    ref = feat.permute(1, 2, 0).numpy()
    obj.setMode(0); obj.updateFeatures()
    got = obj.features()
    scale = float(np.abs(ref).max())
    e16, e_us = float(np.abs(f16 - ref).max()) / scale, float(np.abs(got - ref).max()) / scale
    print(f"feature-map max error / max|f|: fp16 module as shipped {e16:.2e}, this implementation {e_us:.2e}")
    assert e_us < 1e-4 and e_us < e16
