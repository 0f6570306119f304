"""GPU (-m gpu): artp_stats.last_launches is what artp.h says it is, the number of kernels the most recent call launched,
i.e. the change of kernel_launches across that call, for calls that launch the validity pipeline directly, inside a
larger call, or not at all; and the motion-cost network's kernels (17 to fold the weights, 8 per trunk run) count in
both, and the trunk's synchronisation and read-back in artp_planner_map_info."""
import ctypes

import numpy as np
import pytest

import cases
import planner_cases as pc
import roadmap_cases as rc
from art_planner_b200 import costnet, synth

pytestmark = pytest.mark.gpu


def _launches(chk, call):
    """(kernels the call added to kernel_launches, last_launches after it)"""
    before = chk.stats()["kernel_launches"]
    out = call()
    s = chk.stats()
    return s["kernel_launches"] - before, s["last_launches"], out


def test_last_launches_counts_the_kernels_of_the_call(maps):
    import torch
    import art_planner_b200 as ap
    m = maps("fbm_rough")
    chk = ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)
    chk.setMap(m)

    added, last, _ = _launches(chk, chk.updateHeightField)              # artp_set_map
    assert last == added > 0

    poses = synth.make_terrain_poses(m, 20000, seed=3)
    added, last, host = _launches(chk, lambda: chk.isValidBatch(poses))  # artp_check_poses, pipeline
    assert last == added > 0
    added, last, _ = _launches(chk, lambda: chk.isValid(poses[0]))       # artp_check_poses, latency path
    assert last == added == 1

    d_poses = torch.from_numpy(poses).cuda()
    added, last, dev = _launches(chk, lambda: chk.isValidBatch(d_poses))  # artp_check_poses_device
    torch.cuda.synchronize()
    assert last == added > 0
    assert np.array_equal(dev.cpu().numpy(), host)
    pipeline = added

    valid = torch.empty(len(poses), dtype=torch.uint8, device="cuda")
    bits = torch.empty((len(poses) + 31) // 32, dtype=torch.int32, device="cuda")
    added, last, _ = _launches(chk, lambda: chk.isValidBatchBits(d_poses, valid, bits))   # artp_check_poses_bits_device
    torch.cuda.synchronize()
    assert last == added == pipeline + 1

    idx = torch.empty(1, dtype=torch.int32, device="cuda")
    cnt = torch.empty(1, dtype=torch.int32, device="cuda")
    h = chk.handle                                                        # artp_compact_valid_u32_device, n == 0: no kernel
    added, last, _ = _launches(chk, lambda: h.check(h.lib.artp_compact_valid_u32_device(
        h.h, ctypes.c_void_p(valid.data_ptr()), 0, 0, ctypes.c_void_p(idx.data_ptr()), ctypes.c_void_p(cnt.data_ptr()), None)))
    torch.cuda.synchronize()
    assert int(cnt.item()) == 0
    assert last == added == 0

    smp = ap.SE3FromSE2Sampler(chk, synth.make_sampler_layers(m, seed=7), synth.sampler_params_for(m), seed=13)
    added, last, (_, n_valid) = _launches(chk, lambda: smp.sampleValidBatch(20000))   # artp_sample_valid
    assert last == added > 0 and n_valid > 0

    centres = poses[:64].copy()
    added, last, _ = _launches(chk, lambda: chk.findValidNear(centres, 0.3, 16, seed=5))   # artp_find_valid_near
    assert last == added > 0


@pytest.mark.parametrize("network", ["light", "full"])
def test_cost_network_calls_count_their_kernels(network):
    import art_planner_b200 as ap
    c = rc.make_case("gentle_inf")
    chk = ap.StateValidityChecker(c.rp, device=0)
    chk.setMap(c.m)
    chk.updateHeightField()
    obj = ap.MotionCostObjective(chk)
    added, last, _ = _launches(chk, lambda: obj.setWeights(costnet.make_state_dict(seed=5, network=network)))
    assert last == added == 17                                            # artp_set_cost_weights: the folding kernels
    for mode in (0, 1):                                                   # tensor-core path, CUDA-core path
        obj.setMode(mode)
        added, last, _ = _launches(chk, obj.updateFeatures)              # artp_update_features: the trunk
        assert last == added == 8, mode


def test_calls_that_run_the_trunk_count_it():
    """artp_update_features_raw launches the trunk's 8 kernels beyond the preparation artp_cost_map_layer launches, and
    artp_planner_set_map[_raw] 8 more with a network than without; set_map's host_syncs and bytes_d2h count the trunk's
    synchronisation and its 4-byte overflow read-back."""
    import art_planner_b200 as ap
    c = rc.make_case("gentle_inf")
    m = c.m
    e, t, ei, ti = pc.raw_layers(m, holes=0.02)
    got = {}
    for with_net in (False, True):
        chk = ap.StateValidityChecker(c.rp, device=0)
        obj = ap.MotionCostObjective(chk)
        if with_net:
            obj.setWeights(costnet.make_state_dict(seed=5))
            added, last, _ = _launches(chk, lambda: obj.costMap(e))                                 # artp_cost_map_layer
            assert last == added > 0
            prep = added
            added, last, _ = _launches(chk, lambda: obj.updateFeaturesRaw(e, m.res, m.cx, m.cy))  # artp_update_features_raw
            assert last == added == prep + 8
        p = ap.Planner(chk, pc.small_params(seed=41))
        for name, call in (("set_map", lambda: p.setMap(e, t, ei, ti, m.res, m.cx, m.cy)),
                           ("set_map_raw", lambda: p.setMapRaw(e, t, m.res, m.cx, m.cy))):
            added, last, info = _launches(chk, call)
            assert last == added > 0, name
            got[with_net, name] = added, info
    for name in ("set_map", "set_map_raw"):
        (n0, i0), (n1, i1) = got[False, name], got[True, name]
        assert n1 == n0 + 8, name
        assert i1["host_syncs"] == i0["host_syncs"] + 1, name
        assert i1["bytes_d2h"] == i0["bytes_d2h"] + 4, name
        assert i1["bytes_h2d"] == i0["bytes_h2d"], name
