"""The C++ host mirror (include/artp_host.hpp) over the C ABI: compiles with plain g++ (CPU suite), fails loudly
without a GPU, and -- on the GPU box -- gives the oracle's answers when driven the way the reference's facade drives
its plugins (tests/host_cpp/host_check.cpp)."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import cases
from art_planner_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    """The driver, compiled into a temporary directory: the source tree may be read-only."""
    from art_planner_b200 import build, capi
    if not os.path.exists(capi.LIB_PATH):
        if shutil.which("nvcc") is None:
            pytest.skip("libartp.so not built and nvcc absent")
        build.build()
    libdir = os.path.dirname(capi.LIB_PATH)
    exe_path = str(tmp_path_factory.mktemp("host_cpp") / "host_check")
    subprocess.run(["g++", "-std=c++14", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_cpp", "host_check.cpp"), "-o", exe_path,
                    "-L", libdir, "-l:libartp.so", f"-Wl,-rpath,{libdir}"], check=True)
    return exe_path


def test_host_mirror_compiles_and_fails_loudly_without_gpu(exe):
    import torch
    r = subprocess.run([exe, "--expect-no-gpu"], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert r.returncode == 3
    else:
        assert r.returncode == 0 and "failed loudly" in r.stdout and "CUDA" in r.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("preset,mk", [(0, "fixture"), (1, "fbm_rough")], ids=["yaml-fixture", "header-fbm"])
def test_host_mirror_matches_oracle(exe, preset, mk, maps, port_lib, tmp_path):
    m = maps(mk)
    params = synth.PARAMS_YAML if preset == 0 else synth.PARAMS_HEADER
    poses = synth.make_terrain_poses(m, 5000, seed=61)
    s1, s2 = synth.make_edges(m, 800, seed=62)
    nseg = 6
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("6i", m.rows, m.cols, len(poses), len(s1), nseg, preset))
        f.write(struct.pack("3d", m.res, m.cx, m.cy))
        f.write(np.asfortranarray(m.elevation).tobytes(order="F"))
        f.write(np.asfortranarray(m.elevation_masked).tobytes(order="F"))
        f.write(poses.tobytes()); f.write(s1.tobytes()); f.write(s2.tobytes())
        L = synth.make_sampler_layers(m, seed=7)
        for a in (L.normal_x, L.normal_y, L.normal_z, L.plane_fit_std_dev, L.cum_prob):
            f.write(np.asfortranarray(a, dtype=np.float32).tobytes(order="F"))
        f.write(np.ascontiguousarray(L.cum_prob_rowwise, dtype=np.float32).tobytes())
        low, high = cases.se3_bounds(m, params.reach_z)
        f.write(struct.pack("6d", *low, *high))
        n_cost = 0
        if preset == 1:      # the learned edge cost: network weights + how many edges go through motionCost
            from art_planner_b200 import costnet
            sd = costnet.make_state_dict(seed=5)
            blob = costnet.pack_blob(sd)
            n_cost = 60
            f.write(struct.pack("i", blob.size)); f.write(blob.astype(np.float32).tobytes()); f.write(struct.pack("i", n_cost))
        else:
            f.write(struct.pack("i", 0))
    r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(fout, "rb").read()
    o = 0
    valid = np.frombuffer(raw, np.uint8, len(poses), o); o += len(poses)
    single = np.frombuffer(raw, np.uint8, 16, o); o += 16
    motion = np.frombuffer(raw, np.uint8, len(s1), o); o += len(s1)
    motion1 = np.frombuffer(raw, np.uint8, 8, o); o += 8
    cost = np.frombuffer(raw, np.float64, len(s1), o); o += 8 * len(s1)
    n_interp = np.frombuffer(raw, np.int32, len(s1), o); o += 4 * len(s1)
    prefix = np.frombuffer(raw, np.int32, len(s1), o); o += 4 * len(s1)
    drawn, n_sampled = np.frombuffer(raw, np.uint64, 2, o); o += 16
    sampled = np.frombuffer(raw, np.float64, 7 * int(n_sampled), o).reshape(-1, 7); o += 56 * int(n_sampled)
    drawn64 = np.frombuffer(raw, np.float64, 7 * 64, o).reshape(-1, 7); o += 56 * 64
    n_accepted, next_index = np.frombuffer(raw, np.uint64, 2, o); o += 16
    accepted = np.frombuffer(raw, np.float64, 7 * int(n_accepted), o).reshape(-1, 7); o += 56 * int(n_accepted)
    seg_nd = np.frombuffer(raw, np.int32, len(s1), o); o += 4 * len(s1)
    seg_valid = np.frombuffer(raw, np.uint8, len(s1), o); o += len(s1)
    seg_t = np.frombuffer(raw, np.float64, len(s1), o); o += 8 * len(s1)
    one = raw[o]; o += 1
    one_t = np.frombuffer(raw, np.float64, 1, o)[0]; o += 8
    one_state = np.frombuffer(raw, np.float64, 7, o); o += 56
    if n_cost:
        mcost = np.frombuffer(raw, np.float64, n_cost, o); o += 8 * n_cost
        batch_ok = raw[o]; o += 1
        ecost = np.frombuffer(raw, np.float64, len(s1), o); o += 8 * len(s1)
        efeas = np.frombuffer(raw, np.uint8, len(s1), o); o += len(s1)
    orc = port_lib.Oracle(params, "port")
    orc.set_map(m)
    ref = orc.check_poses(poses)
    assert np.array_equal(valid, ref) and np.array_equal(single, ref[:16])
    refm = orc.check_motions(s1, s2, nseg - 1)
    assert np.array_equal(motion, refm) and np.array_equal(motion1, refm[:8])
    refc = orc.path_length_cost(s1, s2)
    assert np.allclose(cost, refc, rtol=1e-12, atol=0)
    # addValidMilestone connection loop and the batched rejection-sampling helper
    d = np.sqrt((s2[:, 0] - s1[:, 0]) ** 2 + (s2[:, 1] - s1[:, 1]) ** 2)
    assert np.array_equal(n_interp, (d / 0.5).astype(np.int32))
    assert np.array_equal(prefix, orc.check_edge_interiors(s1, s2, None, 0.5))
    want = poses[ref != 0][:100]
    assert int(n_sampled) == len(want) and np.array_equal(sampled, want)
    if len(want) == 100:
        last = np.nonzero(ref)[0][99]
        assert int(drawn) == min(len(poses), (last // 64 + 1) * 64)
    # SE3FromSE2Sampler mirror: stream positions 0..63, then the fused batch over 64..2063
    import philox_ref
    sp = synth.sampler_params_for(m)
    ref64, _ = port_lib.sample_states(m, L, sp, params.reach_z, philox_ref.sampler_uniforms(99, 0, 64))
    assert np.abs(drawn64 - ref64).max() < 1e-12
    cand, _ = port_lib.sample_states(m, L, sp, params.reach_z, philox_ref.sampler_uniforms(99, 64, 2000))
    assert int(next_index) == 2064
    # validity is decided on the device's own candidates (ulp-level differences to `cand`): compare with a tolerance
    # on the states and exactly on the count unless a candidate sits on a decision boundary
    flags = orc.check_poses(cand)
    if int(n_accepted) == int(flags.sum()):
        assert np.abs(accepted - cand[flags != 0]).max() < 1e-12
    else:
        assert abs(int(n_accepted) - int(flags.sum())) <= 2
    # per-edge OMPL segment rule + lastValid (DiscreteMotionValidator with validSegmentCount, restated in oracle/)
    ref_nd = orc.valid_segment_count(low, high, s1, s2)
    ref_sv, ref_st = orc.check_motions_segments(s1, s2, ref_nd)
    assert np.array_equal(seg_nd, ref_nd) and np.array_equal(seg_valid, ref_sv) and np.array_equal(seg_t, ref_st)
    v1, t1 = orc.check_motions_segments(s1[:1], s2[:1], np.array([nseg], np.int32))
    assert bool(one) == bool(v1[0])
    if not v1[0]:
        assert one_t == t1[0] and np.abs(one_state - _interpolate(s1[0], s2[0], t1[0])).max() < 1e-12
    if n_cost:
        _check_learned_cost(m, params, s1, s2, n_cost, mcost, batch_ok, ecost, efeas, orc)


def _interpolate(a, b, t):
    """OMPL 1.4.2 SE3StateSpace::interpolate (lerp + slerp), numpy doubles."""
    o = np.empty(7)
    o[:3] = a[:3] + (b[:3] - a[:3]) * t
    dq = float(np.dot(a[3:], b[3:]))
    theta = 0.0 if abs(dq) > 1.0 - 1e-9 else float(np.arccos(abs(dq)))
    if theta > np.finfo(np.float64).eps:
        d = 1.0 / np.sin(theta); s0 = np.sin((1.0 - t) * theta); s1 = np.sin(t * theta)
        if dq < 0:
            s1 = -s1
        o[3:] = (a[3:] * s0 + b[3:] * s1) * d
    else:
        o[3:] = a[3:]
    return o


def _check_learned_cost(m, params, s1, s2, n_cost, mcost, batch_ok, ecost, efeas, orc):
    """MotionCostObjective::motionCost with its edge splitting (motion_cost_objective.cpp:36-95) and the updateEdges batch
    (prm_motion_cost.cpp:27-73), restated on top of the CNN oracle; 1e-4 relative (BASELINE.json)."""
    from art_planner_b200 import costnet
    from oracle.cnn_oracle import CostNetOracle, cnn_input_from_layer
    net = CostNetOracle(costnet.make_state_dict(seed=5))
    feat = net.features(cnn_input_from_layer(m.elevation))
    lx, ly = m.length
    w_e, w_t, w_r, thr, max_len = np.float32(0.0), np.float32(1.0), np.float32(5.0), np.float32(0.55), np.float32(0.5)   # params.h defaults, threshold as host_check sets it
    yaw = lambda s: np.float32(np.arctan2(2 * (s[6] * s[5] + s[3] * s[4]), 1 - 2 * (s[4] ** 2 + s[5] ** 2)))
    for i in range(n_cost):
        a, b = s1[i], s2[i]
        n_interp = int(np.sqrt((b[0] - a[0]) ** 2 + (b[1] - a[1]) ** 2) / float(max_len))
        div = 1.0 / (n_interp + 1)
        em = np.zeros((n_interp + 1, 6), np.float32)
        em[0, 3:] = (a[0], a[1], yaw(a)); em[n_interp, :3] = (b[0], b[1], yaw(b))
        for step in range(1, n_interp + 1):
            cur = _interpolate(a, b, step * div)
            em[step - 1, :3] = (cur[0], cur[1], yaw(cur)); em[step, 3:] = (cur[0], cur[1], yaw(cur))
        c3 = net.query(feat, em, m.res, lx, ly, m.cx, m.cy)
        want = np.inf if (c3[:, 2].astype(np.float64) > float(thr)).any() else float(
            (c3[:, 0].astype(np.float64) * float(w_e) + c3[:, 1].astype(np.float64) * float(w_t) + c3[:, 2].astype(np.float64) * float(w_r)).sum())
        if np.isinf(want) or np.isinf(mcost[i]):
            # a risk within 1e-4 of the threshold may fall either way
            assert np.isinf(want) == np.isinf(mcost[i]) or np.abs(c3[:, 2] - float(thr)).min() < 1e-4 * float(thr) + 1e-5, i
        else:
            assert abs(mcost[i] - want) <= 1e-4 * abs(want) + 1e-5, (i, mcost[i], want)
    assert batch_ok == 1
    em = orc.edge_matrix(s1, s2)
    c3 = net.query(feat, em, m.res, lx, ly, m.cx, m.cy).astype(np.float64)
    feas = c3[:, 2] <= float(thr)
    near = np.abs(c3[:, 2] - float(thr)) < 1e-4 * float(thr) + 1e-5
    assert np.array_equal(efeas.astype(bool)[~near], feas[~near])
    want = c3[:, 0] * float(w_e) + c3[:, 1] * float(w_t) + c3[:, 2] * float(w_r)
    sel = feas & efeas.astype(bool)
    assert np.allclose(ecost[sel], want[sel], rtol=1e-4, atol=1e-5) and np.isinf(ecost[~efeas.astype(bool)]).all()
    assert 0 < sel.sum() < len(sel)
