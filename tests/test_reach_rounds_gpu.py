"""GPU parity (-m gpu) of the reach-box kernels at queue lengths that end their claims and rounds unevenly.

reach_groups_kernel decides four boxes per warp round, with the next round's tiles in flight, over guided claims of one
to eight rounds; box_tiles_warp_kernel takes the reach boxes that need the merge screen or -inf handling. Batches of the bench map's poses are put together so that the 8-lane kernel's
queue holds exactly 1, 3, 4, 5, 33 and 4 * 8 * k +- 1 boxes (partial last rounds, one-round claims, and a queue long
enough for claims of several rounds), and every mask must equal the oracle's, with stage timing off (the box kernels
side by side) and on (one after the other), and with every reach box sent to the one-warp-per-box kernel
(ARTP_NO_GROUPS, read at artp_set_map)."""
import os

import numpy as np
import pytest

import bench
from art_planner_b200 import synth

pytestmark = pytest.mark.gpu

TARGETS = [1, 3, 4, 5, 33, 4 * 8 * 1 - 1, 4 * 8 * 2 - 1, 4 * 8 * 2 + 1, 4 * 8 * 3000 - 1, 4 * 8 * 3000 + 1]
N_POOL = 400_000     # bench poses: the long batches are a prefix of them
N_SINGLES = 2_000    # bench poses after the pool: each one's queue contribution is measured alone


@pytest.fixture(scope="module")
def setup(port_lib):
    import torch
    m = synth.make_fbm_map(bench.MAP_N, bench.MAP_N, bench.MAP_RES, seed=bench.MAP_SEED, amp=0.6)
    poses = synth.make_terrain_poses(m, N_POOL + N_SINGLES, seed=bench.POSE_SEED)
    o = port_lib.Oracle(synth.PARAMS_YAML, "port")
    o.set_map(m)
    ref = o.check_poses(poses)
    return m, poses, torch.from_numpy(poses).cuda(), ref


def checker(m):
    import art_planner_b200 as ap
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    return chk


def group_queue(chk, d):
    chk.isValidBatch(d)
    return chk.stats()["last_reach_plane_stage"]


@pytest.fixture(scope="module")
def batches(setup):
    """Pose indices per target: the longest prefix of the pool that queues at most `target` boxes for the 8-lane kernel,
    topped up with single poses that queue one box each (a pose's boxes are classified on their own, so the counts add;
    the tests check the sum)."""
    m, poses, d, _ = setup
    chk = checker(m)
    ones = [N_POOL + i for i in range(N_SINGLES) if group_queue(chk, d[N_POOL + i:N_POOL + i + 1]) == 1]
    out = {}
    for t in TARGETS:
        lo, hi = 0, N_POOL          # count(lo) <= t < count(hi) (the pool queues far more than any target)
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if group_queue(chk, d[:mid]) <= t:
                lo = mid
            else:
                hi = mid
        short = t - (group_queue(chk, d[:lo]) if lo else 0)
        assert short <= len(ones), (t, short, len(ones))
        out[t] = np.concatenate([np.arange(lo), np.array(ones[:short], dtype=np.int64)]).astype(np.int64)
    return out


@pytest.mark.parametrize("timing", [False, True], ids=["side-by-side", "serial"])
@pytest.mark.parametrize("target", TARGETS)
def test_reach_queues_at_uneven_lengths_equal_the_oracle(setup, batches, target, timing):
    import torch
    m, poses, d, ref = setup
    idx = batches[target]
    x = d[torch.from_numpy(idx).cuda()].contiguous()
    chk = checker(m)
    chk.setTiming(timing)
    got = chk.isValidBatch(x).cpu().numpy()
    st = chk.stats()
    assert st["last_reach_plane_stage"] == target, st
    bad = np.nonzero(got != ref[idx])[0]
    assert bad.size == 0, f"{bad.size} mismatches of {len(idx)}, first {bad[:8]}, stats {st}"
    # the same batch again on the same handle: the claim counters and queues of the previous call are reset
    again = chk.isValidBatch(x).cpu().numpy()
    assert np.array_equal(again, got)


@pytest.mark.parametrize("target", [5, 33, 4 * 8 * 3000 + 1])
def test_reach_boxes_all_on_the_warp_kernel_equal_the_oracle(setup, batches, target):
    """ARTP_NO_GROUPS: every reach box of the same batches takes box_tiles_warp_kernel."""
    import torch
    m, poses, d, ref = setup
    idx = batches[target]
    os.environ["ARTP_NO_GROUPS"] = "1"
    try:
        chk = checker(m)
    finally:
        os.environ.pop("ARTP_NO_GROUPS", None)
    got = chk.isValidBatch(d[torch.from_numpy(idx).cuda()].contiguous()).cpu().numpy()
    st = chk.stats()
    assert st["last_reach_plane_stage"] == 0 and st["last_queued_reach_stage"] >= target, st
    bad = np.nonzero(got != ref[idx])[0]
    assert bad.size == 0, f"{bad.size} mismatches of {len(idx)}, first {bad[:8]}, stats {st}"
