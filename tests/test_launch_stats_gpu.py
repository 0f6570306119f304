"""GPU (-m gpu): artp_stats.last_launches is what artp.h says it is, the number of kernels the most recent call launched,
i.e. the change of kernel_launches across that call, for calls that launch the validity pipeline directly, inside a
larger call, or not at all."""
import ctypes

import numpy as np
import pytest

import cases
from art_planner_b200 import synth

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
