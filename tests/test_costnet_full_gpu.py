"""GPU parity (-m gpu) of the full-width motion-cost network (network.py, 32/64 channels) on the device beside the
light one: feature map and costs against the fp32 evaluation of the reference module (golden file made from the
reference's own network.py) and against the torch restatement in oracle/cnn_oracle.py, switching networks on one
handle, and the edge / path cost entry points running the full network."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

import cases
from art_planner_b200 import costnet, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL, ATOL = 1e-4, 1e-5
THR = 0.375   # the seeded full-network risks lie in ~0.16-0.46: both feasible and infeasible edges


def make_obj(m, sd, **kw):
    import art_planner_b200 as ap
    from art_planner_b200.checker import _Handle
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, handle=_Handle(synth.PARAMS_YAML, 0, **kw))
    chk.setMap(m)
    chk.updateHeightField()
    obj = ap.MotionCostObjective(chk)
    obj.setWeights(sd)
    return obj


@pytest.fixture(scope="module")
def setup():
    from art_planner_b200 import build
    from oracle.cnn_oracle import CostNetOracle, cnn_input_from_layer
    build.build()
    m = cases.c4_map()
    sd = costnet.make_state_dict(seed=5, network="full")
    obj = make_obj(m, sd)
    orc = CostNetOracle(sd)
    feat = orc.features(cnn_input_from_layer(m.elevation))
    golden = np.load(os.path.join(ROOT, "tests", "golden", "cnn_full_c4.npz"))
    assert abs(float(costnet.pack_blob(sd).astype(np.float64).sum()) - float(golden["blob_sum"])) < 1e-9, "weight generator drift"
    return m, obj, orc, feat, golden


@pytest.mark.parametrize("mode", [1, 0], ids=["cuda-core", "wgmma"])
def test_feature_map(setup, mode):
    m, obj, orc, feat, golden = setup
    assert obj.network() == "full"
    obj.setMode(mode)
    obj.updateFeatures()
    got = obj.features()                      # [Hf, Wf, 64]
    ref = feat.permute(1, 2, 0).numpy()
    assert got.shape == ref.shape == (104, 104, 64)
    scale = float(np.abs(ref).max())
    err = float(np.abs(got - ref).max()) / scale
    tol = 1e-5 if mode == 1 else 1e-4
    print(f"full network, mode {mode}: feature map max error {err:.3e} of max |f| = {scale:.3f}")
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
    # more queries than 128 per SM: the 128-thread head configuration
    q2 = costnet.make_queries(m, 40_000, seed=8)
    assert np.allclose(obj.costQuery(q2), orc.query(feat, q2, m.res, lx, ly, m.cx, m.cy), rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("shape", [(300, 260), (1000, 1000), (121, 97)], ids=["300x260-partial-tiles", "1000x1000-metric-map", "121x97-odd"])
def test_feature_map_other_sizes(shape):
    """The full trunk away from the 256x256 patch against the fp32 torch restatement of network.py:78-110."""
    from oracle.cnn_oracle import CostNetOracle, cnn_input_from_layer
    rows, cols = shape
    m = synth.make_fbm_map(rows, cols, 0.04, seed=2, amp=0.6)
    sd = costnet.make_state_dict(seed=5, network="full")
    obj = make_obj(m, sd)
    obj.updateFeatures()
    got = obj.features()
    orc = CostNetOracle(sd)
    feat = orc.features(cnn_input_from_layer(m.elevation))
    ref = feat.permute(1, 2, 0).numpy()
    assert got.shape == ref.shape and got.shape[2] == 64
    scale = float(np.abs(ref).max())
    assert float(np.abs(got - ref).max()) / scale < 1e-4
    q = costnet.make_queries(m, 2048, seed=6)
    lx, ly = m.length
    assert np.allclose(obj.costQuery(q), orc.query(feat, q, m.res, lx, ly, m.cx, m.cy), rtol=RTOL, atol=ATOL)


def fp16_features(sd, E):
    """The module as the reference runs it (predictor.py:22: .half() on the GPU), through the oracle's layer calls."""
    import torch
    import torch.nn.functional as F
    from oracle.cnn_oracle import CostNetOracle
    h = CostNetOracle(sd)
    h.p = {k: v.cuda().half() for k, v in h.p.items()}
    with torch.no_grad():
        t = torch.as_tensor(E).cuda().half()[None, None]
        t = h._conv_bn(t, "init_conv1", "init_conv1_bn")
        t = F.leaky_relu(h._conv_bn(t, "init_conv2", "init_conv2_bn"), 0.3); t = F.max_pool2d(t, (2, 2), stride=2)
        t = F.leaky_relu(h._conv_bn(t, "init_conv3", "init_conv3_bn"), 0.3)
        t = F.leaky_relu(h._conv_bn(t, "init_conv4", "init_conv4_bn"), 0.3); t = F.max_pool2d(t, (3, 3), stride=1)
        t = F.leaky_relu(h._conv_bn(t, "init_conv5", "init_conv5_bn"), 0.3)
        t = F.leaky_relu(h._conv_bn(t, "init_flatten", "init_flatten_bn"), 0.3)
    return t[0].float().cpu().permute(1, 2, 0).numpy()


def test_error_against_the_fp16_module_as_shipped(setup):
    from oracle.cnn_oracle import cnn_input_from_layer
    m, obj, orc, feat, golden = setup
    f16 = fp16_features(costnet.make_state_dict(seed=5, network="full"), cnn_input_from_layer(m.elevation))
    ref = feat.permute(1, 2, 0).numpy()
    obj.setMode(0); obj.updateFeatures()
    got = obj.features()
    scale = float(np.abs(ref).max())
    e16, e_us = float(np.abs(f16 - ref).max()) / scale, float(np.abs(got - ref).max()) / scale
    print(f"full network feature-map max error / max|f|: fp16 module as shipped {e16:.2e}, this implementation {e_us:.2e}")
    assert e_us < 1e-4 and e_us < e16


def _run(obj, q, mode):
    obj.setMode(mode)
    obj.updateFeatures()
    return obj.features(), obj.costQuery(q)


@pytest.mark.parametrize("mode", [0, 1], ids=["wgmma", "cuda-core"])
def test_switching_networks_on_one_handle_equals_fresh_handles(mode):
    """light -> full -> light on one handle: buffers, tensor maps and kernel attributes follow the loaded network."""
    import art_planner_b200 as ap
    m = cases.c4_map()
    light, full = costnet.make_state_dict(seed=5), costnet.make_state_dict(seed=5, network="full")
    q = costnet.make_queries(m, 4096, seed=6)
    want_l = _run(make_obj(m, light), q, mode)
    want_f = _run(make_obj(m, full), q, mode)
    assert want_l[0].shape == (104, 104, 48) and want_f[0].shape == (104, 104, 64)
    obj = make_obj(m, light)
    for sd, name, want in ((light, "light", want_l), (full, "full", want_f), (light, "light", want_l)):
        obj.setWeights(sd)
        assert obj.network() == name
        with pytest.raises(ap.ArtpError):
            obj.costQuery(q)                  # new weights: the features of the old ones are gone
        got = _run(obj, q, mode)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), name


def test_blob_sizes_and_network_query():
    import art_planner_b200 as ap
    from art_planner_b200 import capi
    m = cases.c4_map()
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m); chk.updateHeightField()
    obj = ap.MotionCostObjective(chk)
    h = chk.handle
    net = ctypes.c_int(7)
    assert h.lib.artp_get_cost_network(h.h, ctypes.byref(net)) == capi.ARTP_E_NOWEIGHTS
    blob = costnet.pack_blob(costnet.make_state_dict(seed=5, network="full"))
    for n in (blob.size - 1, blob.size + 1, costnet.blob_size("light") + 1, 0):
        assert h.lib.artp_set_cost_weights(h.h, blob.ctypes.data, n) == capi.ARTP_E_INVALID
    assert h.lib.artp_get_cost_network(h.h, ctypes.byref(net)) == capi.ARTP_E_NOWEIGHTS
    assert h.lib.artp_set_cost_weights(h.h, blob.ctypes.data, blob.size) == capi.ARTP_OK
    assert h.lib.artp_get_cost_network(h.h, ctypes.byref(net)) == capi.ARTP_OK and net.value == 1
    assert obj.network() == "full"
    # a rejected blob leaves the loaded network in place
    assert h.lib.artp_set_cost_weights(h.h, blob.ctypes.data, 12345) == capi.ARTP_E_INVALID
    obj.updateFeatures()
    hf, wf = ctypes.c_int(), ctypes.c_int()
    out = np.empty((104, 104, 48), np.float32)      # the light network's size: wrong for the full one
    assert h.lib.artp_get_features(h.h, out.ctypes.data, out.size, ctypes.byref(hf), ctypes.byref(wf)) == capi.ARTP_E_INVALID
    assert obj.features().shape == (104, 104, 64)


@pytest.fixture(scope="module")
def edges_env():
    from test_motion_cost_split_gpu import edge_set
    m = cases.c4_map()
    sd = costnet.make_state_dict(seed=5, network="full")
    obj = make_obj(m, sd, risk_threshold=THR)
    obj.updateFeatures()
    s1, s2 = edge_set(m)
    return dict(m=m, sd=sd, obj=obj, s1=s1, s2=s2, cost=obj.motionCostBatch(s1, s2))


def test_motion_cost_batch_equals_per_edge(edges_env):
    import torch
    from test_motion_cost_split_gpu import reduce_costs, split_rows
    obj, s1, s2, cost = edges_env["obj"], edges_env["s1"], edges_env["s2"], edges_env["cost"]
    fin = np.isfinite(cost)
    assert 0 < fin.sum() < len(cost)
    sel = np.arange(0, len(s1), 11)
    assert np.array_equal(np.array([obj.motionCost(s1[i], s2[i]) for i in sel]), cost[sel])
    rows, off = split_rows(s1, s2)
    assert np.array_equal(cost, reduce_costs(obj.costQuery(rows), off, THR))
    dev = obj.motionCostBatch(torch.from_numpy(s1).cuda(), torch.from_numpy(s2).cuda())
    torch.cuda.synchronize()
    assert np.array_equal(dev.cpu().numpy(), cost)


def test_cpp_mirror_batch_equals_per_edge(edges_env, tmp_path):
    """The unchanged tests/host_cpp/motion_cost_batch.cpp driver reads the blob's length from its input file."""
    from art_planner_b200 import capi
    from test_motion_cost_split_gpu import _walk
    libdir = os.path.dirname(capi.LIB_PATH)
    exe = str(tmp_path / "motion_cost_batch")
    subprocess.run(["g++", "-std=c++14", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_cpp", "motion_cost_batch.cpp"), "-o", exe,
                    "-L", libdir, "-l:libartp.so", f"-Wl,-rpath,{libdir}"], check=True)
    m, s1, s2 = edges_env["m"], edges_env["s1"], edges_env["s2"]
    path = _walk(m, 200, 82)
    blob = costnet.pack_blob(edges_env["sd"]).astype(np.float32)
    assert blob.size == costnet.blob_size("full")
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("5i", m.rows, m.cols, len(s1), len(path), blob.size))
        f.write(struct.pack("4d", m.res, m.cx, m.cy, THR))
        f.write(np.asfortranarray(m.elevation).tobytes(order="F"))
        f.write(np.asfortranarray(m.elevation_masked).tobytes(order="F"))
        f.write(s1.tobytes()); f.write(s2.tobytes()); f.write(path.tobytes()); f.write(blob.tobytes())
    r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = np.fromfile(fout, np.uint8)
    n, ns = len(s1), len(path) - 1
    v = np.frombuffer(raw.tobytes(), np.float64, 3 * n + ns + 3)
    single, batch = v[:n], v[n:2 * n]
    assert np.array_equal(batch, single)
    assert np.array_equal(batch, edges_env["cost"])
