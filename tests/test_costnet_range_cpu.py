"""CPU-only: the float64 restatement of the motion-cost network, trained-like (calibrated) weights, and the per-element
error bound the GPU range tests hold the library to (oracle/cnn_oracle.py), checked on an emulation of the library's
fp16 operand split: the bound accepts the split as built and rejects each of a set of small implementation errors."""
import os

import numpy as np
import pytest
import torch

import cases
from art_planner_b200 import costnet, synth
from oracle import cnn_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NETS = ["light", "full"]


@pytest.mark.parametrize("net", NETS)
def test_float64_oracle_agrees_with_fp32_on_the_golden_case(net):
    golden = np.load(os.path.join(ROOT, "tests", "golden", "cnn_c4.npz" if net == "light" else "cnn_full_c4.npz"))
    m = cases.c4_map()
    sd = costnet.make_state_dict(seed=5, network=net)
    E = co.cnn_input_from_layer(m.elevation)
    f32, f64 = co.CostNetOracle(sd).features(E), co.CostNetOracle(sd, dtype=torch.float64).features(E)
    assert f32.dtype == torch.float32 and f64.dtype == torch.float64
    scale = float(f64.abs().max())
    ref, bound, _ = co.trunk_error_bound(sd, E)
    assert float((ref - f64).abs().max()) < 1e-12 * scale
    assert _ratio(f32, f64, bound) < 0.5                                   # fp32 rounding, element by element
    assert np.allclose(f64[:, ::13, ::13].numpy(), golden["feat_sample"], rtol=0, atol=1e-5 * scale)
    q = costnet.make_queries(m, 4096, seed=6)
    lx, ly = m.length
    c32 = co.CostNetOracle(sd).query(f32, q, m.res, lx, ly, m.cx, m.cy)
    c64 = co.CostNetOracle(sd, dtype=torch.float64).query(f64, q, m.res, lx, ly, m.cx, m.cy)
    assert c64.dtype == np.float64 and np.abs(c32 - c64).max() < 1e-5
    assert np.abs(c64 - golden["cost"]).max() < 1e-5


def test_fp32_oracle_is_unchanged_by_the_dtype_argument():
    m = cases.c4_map()
    sd = costnet.make_state_dict(seed=5)
    E = co.cnn_input_from_layer(m.elevation)
    assert torch.equal(co.CostNetOracle(sd).features(E), co.CostNetOracle(sd, dtype=torch.float32).features(E))


@pytest.mark.parametrize("net", NETS)
def test_calibrated_weights_keep_activations_order_one(net):
    sd = co.calibrated_state_dict(5, net)
    assert costnet.pack_blob(sd).size == costnet.blob_size(net)
    assert np.array_equal(costnet.pack_blob(sd), costnet.pack_blob(co.calibrated_state_dict(5, net)))   # deterministic
    E = co.cnn_input_from_layer(synth.make_fbm_map(112, 112, 0.04, seed=9, amp=0.6).elevation)
    _, _, site_max = co.trunk_error_bound(sd, E)
    assert all(0.5 < s < 50 for s in site_max), site_max


def _case_input(offset, rows=112, cols=112):
    return co.cnn_input_from_layer(synth.make_fbm_map(rows, cols, 0.04, seed=9, amp=0.6).elevation) + np.float32(offset)


def _ratio(f, ref, bound):
    return float(((f.double() - ref).abs() / bound).max())


@pytest.mark.parametrize("net", NETS)
def test_split_predictions_for_the_weight_range(net):
    """What the emulated split predicts for the range cases, with the former constant weight scale (1024) and with the
    per-channel power of two the library now chooses. A near-dead channel of init_flatten (folded weights up to 300)
    overflows w_hi = fp16(w * 1024) -- silently, as inf / NaN features -- and stays finite and within the bound with
    the channel scale. A near-dead channel in every layer amplifies its input by ~300 per layer, and the activations
    leave the fp16 range (the library reports that). The other variants are within the bound either way."""
    E = _case_input(0.0)
    dead = co.calibrated_state_dict(5, net, "dead", 300.0, layers=(5,))
    ref, bound, site_max = co.trunk_error_bound(dead, E)
    assert max(site_max) < 100
    assert not torch.isfinite(co.trunk_features_split(dead, E, weight_scale=1024.0)).all()
    assert _ratio(co.trunk_features_split(dead, E), ref, bound) < 0.1
    _, _, site_max = co.trunk_error_bound(co.calibrated_state_dict(5, net, "dead", 300.0), E)
    assert max(site_max) > co.FP16_OVERFLOW
    for variant, value in (("tiny", 1e-6), ("zero", 0.0), ("gamma", 10.0), ("gamma", 1e-3), ("wscale", 1e-3),
                           ("wscale", 10.0)):
        sd = co.calibrated_state_dict(5, net, variant, value)
        ref, bound, _ = co.trunk_error_bound(sd, E)
        for scale in ("channel", 1024.0):
            r = _ratio(co.trunk_features_split(sd, E, weight_scale=scale), ref, bound)
            assert r < 0.1, (variant, value, scale, r)


def test_channel_scale_is_a_power_of_two_below_2_15():
    wf = torch.tensor([300.0, 1e-6, 0.0, 1.0, 32767.0, 2.0 ** 14], dtype=torch.float64)[:, None, None, None]
    sc = co.channel_weight_scale(wf)
    m, e = torch.frexp(sc)
    assert torch.all(m == 0.5)
    prod = (wf[:, 0, 0, 0] * sc)[[0, 1, 3, 4, 5]]
    assert torch.all(prod < 2 ** 15) and torch.all(prod >= 2 ** 14)


@pytest.mark.parametrize("offset", [0.0, 300.0], ids=["0m", "300m"])
@pytest.mark.parametrize("net", NETS)
def test_bound_rejects_injected_defects(net, offset):
    """The bound is sharp enough: the emulated split as built stays far inside it, and each defect exceeds it --
    dropping the a_lo * w_hi product, dropping w_lo, storing light init_conv2's 24 channels at the pixel stride of its
    N = 32 instantiation, and shifting one tap of the 15x15 layer by one pixel. The fp32 torch module meets it."""
    sd = co.calibrated_state_dict(5, net)
    E = _case_input(offset)
    ref, bound, _ = co.trunk_error_bound(sd, E)
    ok = _ratio(co.trunk_features_split(sd, E), ref, bound)
    f32 = _ratio(co.CostNetOracle(sd).features(E), ref, bound)
    print(f"{net} +{offset} m: split as built {ok:.3f} of the bound, fp32 module {f32:.3f}")
    assert ok < 0.1 and f32 < 0.5
    for defect in ("drop_alo_whi", "drop_wlo", "pad_stride", "tap_shift"):
        if defect == "pad_stride" and net == "full":
            continue                                          # init_conv2 has Cout = N = 32: no pad channels
        r = _ratio(co.trunk_features_split(sd, E, defect=defect), ref, bound)
        print(f"  {defect}: {r:.3g} x the bound")
        assert r > 1.0, (defect, r)
