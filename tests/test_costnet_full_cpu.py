"""CPU-only: the full-width motion-cost network (network.py) beside the light one -- the blob layout of both, the
oracle against the golden file made from the reference's own network.py, and the C ABI's blob sizes."""
import ctypes
import os
import shutil

import numpy as np
import pytest

import cases
from art_planner_b200 import costnet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIGHT_FLOATS, FULL_FLOATS = 584_543, 1_036_771


def test_layer_tables_and_blob_sizes():
    light, full = costnet.LAYERS, costnet.LAYERS_FULL
    assert [l[:2] for l in light] == [l[:2] for l in full]            # same layers, same order, same BatchNorms
    widths = {name: (co, ci, k) for name, _, co, ci, k in full}
    assert widths["init_conv1"] == (32, 1, 3) and widths["init_conv2"] == (32, 32, 3)
    assert widths["init_conv3"] == (64, 32, 3) and widths["init_conv4"] == widths["init_conv5"] == (64, 64, 3)
    assert widths["init_flatten"] == (64, 64, 15) and widths["tar0_conv1"] == (16, 10, 1)
    assert widths["out0_conv1"] == (80 - 16, 80, 1)                      # 64 features ++ 16 target features
    assert all(widths[f"out1_conv{i}"] == (32, 64, 1) and widths[f"out2_conv{i}"] == (1, 32, 1) for i in (1, 2, 3))
    assert costnet.blob_size() == costnet.blob_size("light") == LIGHT_FLOATS
    assert costnet.blob_size("full") == FULL_FLOATS
    sd = costnet.make_state_dict(seed=5, network="full")
    params = sum(v.size for k, v in sd.items() if "running_" not in k)
    assert params == 1_035_779                                           # network.py's parameter count
    assert costnet.network_of(sd) == "full" and costnet.network_of(costnet.make_state_dict(seed=5)) == "light"
    blob = costnet.pack_blob(sd)
    assert blob.size == FULL_FLOATS and blob.dtype == np.float32
    assert np.array_equal(blob[:32 * 9], sd["init_conv1.weight"].reshape(-1))
    assert np.array_equal(blob[-2:], np.concatenate([sd["out2_conv3.weight"].reshape(-1)[-1:], sd["out2_conv3.bias"]]))


def test_pack_blob_rejects_an_unknown_width():
    sd = costnet.make_state_dict(seed=5)
    sd["init_conv1.weight"] = np.zeros((40, 1, 3, 3), np.float32)
    with pytest.raises(ValueError):
        costnet.pack_blob(sd)


def test_light_generator_stream_is_unchanged():
    golden = np.load(os.path.join(ROOT, "tests", "golden", "cnn_c4.npz"))
    sd = costnet.make_state_dict(seed=5, network="light")
    assert abs(float(costnet.pack_blob(sd).astype(np.float64).sum()) - float(golden["blob_sum"])) < 1e-9


def test_oracle_reproduces_the_full_golden_file():
    from oracle.cnn_oracle import CostNetOracle, cnn_input_from_layer
    golden = np.load(os.path.join(ROOT, "tests", "golden", "cnn_full_c4.npz"))
    m = cases.c4_map()
    sd = costnet.make_state_dict(seed=5, network="full")
    assert abs(float(costnet.pack_blob(sd).astype(np.float64).sum()) - float(golden["blob_sum"])) < 1e-9
    orc = CostNetOracle(sd)
    feat = orc.features(cnn_input_from_layer(m.elevation))
    assert tuple(feat.shape) == (64, 104, 104)
    scale = float(golden["feat_abs_max"])
    assert abs(float(feat.abs().max()) - scale) <= 1e-6 * scale
    assert np.allclose(feat[:, ::13, ::13].numpy(), golden["feat_sample"], rtol=0, atol=1e-6 * scale)
    q = costnet.make_queries(m, 4096, seed=6)
    lx, ly = m.length
    cost = orc.query(feat, q, m.res, lx, ly, m.cx, m.cy)
    assert np.abs(cost - golden["cost"]).max() < 1e-5


@pytest.fixture(scope="module")
def lib():
    from art_planner_b200 import build, capi
    if not os.path.exists(capi.LIB_PATH):
        if shutil.which("nvcc") is None:
            pytest.skip("libartp.so not built and nvcc absent")
        build.build()
    return capi.load()


def test_abi_blob_sizes_match_costnet(lib):
    from art_planner_b200 import capi
    for name, (_, net) in costnet.NETWORKS.items():
        assert lib.artp_cost_weights_size_for(net) == costnet.blob_size(name)
    assert lib.artp_cost_weights_size() == costnet.blob_size("light")
    assert lib.artp_cost_weights_size_for(2) == 0 and lib.artp_cost_weights_size_for(-1) == 0
    net = ctypes.c_int(7)
    assert lib.artp_get_cost_network(None, ctypes.byref(net)) == capi.ARTP_E_INVALID
