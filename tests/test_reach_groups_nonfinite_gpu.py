"""GPU parity (-m gpu) of reach_groups_kernel on reach boxes whose zones hold -inf heights.

The classify stage sends every merge-free reach box that the range tables reduced to the 8-lane-group kernel, whether
or not its zone cuts a -inf blob of `elevation_masked`; only zones with mergeable planes (and zones the tables did not
reduce) stay on the one-warp-per-box kernel. Single poses of the bench map and of two off-grid maps of offgrid_cases.py
(flat poses there reach past the map border, so some zones are clipped at it) are picked whose one queued reach box has a
-inf height in its zone (read back from the one-warp queue with ARTP_NO_GROUPS), and batches of them are put together
so that the 8-lane queue holds exactly 1, 3, 4, 5 and 33 such boxes. Every mask must equal the oracle's with the box
kernels side by side and one after the other, and with ARTP_NO_GROUPS (read at artp_set_map)."""
import os

import numpy as np
import pytest

import bench
import offgrid_cases as oc
from art_planner_b200 import synth

pytestmark = pytest.mark.gpu

REC_ALLFINITE, REC_NEEDS_REDUCE, REC_MERGEFREE = 8, 16, 32
TARGETS = [1, 3, 4, 5, 33]
MAPS = ["bench", "coarse", "fine"]   # the off-grid maps with the most -inf blobs under reach boxes
N_PROBE = 6000       # candidate single poses per map


def make_map(mk):
    if mk == "bench":
        return synth.make_fbm_map(bench.MAP_N, bench.MAP_N, bench.MAP_RES, seed=bench.MAP_SEED, amp=0.6)
    return oc.MAPS[mk]()


def make_poses(m, mk):
    if mk == "bench":
        return synth.make_terrain_poses(m, N_PROBE, seed=bench.POSE_SEED)
    p = oc.poses(m, 300 + MAPS.index(mk))
    # the flat poses past the border first: they hold the zones clipped at it
    return np.concatenate([p[oc.N_TERRAIN:], p[:oc.N_TERRAIN]])[:N_PROBE]


def checker(m, no_groups=False):
    import art_planner_b200 as ap
    if no_groups:
        os.environ["ARTP_NO_GROUPS"] = "1"
    try:
        chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
        chk.setMap(m)
        chk.updateHeightField()
    finally:
        os.environ.pop("ARTP_NO_GROUPS", None)
    return chk


@pytest.fixture(scope="module", params=MAPS)
def case(request, port_lib):
    """(map, poses, oracle mask, the poses whose only queued box is a non-finite reach box of the 8-lane queue, and
    which of those have a zone clipped at the map border)."""
    mk = request.param
    m = make_map(mk)
    poses = make_poses(m, mk)
    o = port_lib.Oracle(synth.PARAMS_YAML, "port")
    o.set_map(m)
    ref = o.check_poses(poses)
    import torch
    d = torch.from_numpy(poses).cuda()
    chk, chk_ng = checker(m), checker(m, no_groups=True)
    picks, clipped = [], []
    for i in range(len(poses)):
        one = d[i:i + 1]   # device buffers: the queue path even for one pose
        chk.isValidBatch(one)
        st = chk.stats()
        if st["last_reach_plane_stage"] != 1 or st["last_queued_reach_stage"] or st["last_queued_warp_stage"]:
            continue
        chk_ng.isValidBatch(one)
        zone, fl = chk_ng.debugReachQueue()
        if len(fl) == 1 and (fl[0] & (REC_ALLFINITE | REC_NEEDS_REDUCE | REC_MERGEFREE)) == REC_MERGEFREE:
            picks.append(i)
            x0, x1, z0, z1 = zone[0]
            if x0 == 0 or z0 == 0 or x1 == m.rows - 1 or z1 == m.cols - 1:
                clipped.append(i)
        if len(picks) >= max(TARGETS) and (mk == "bench" or clipped):
            break
    return m, poses, ref, np.array(picks, np.int64), np.array(clipped, np.int64), mk


def batch(case, target):
    m, poses, ref, picks, clipped, mk = case
    if len(picks) < target:
        pytest.skip(f"{mk}: {len(picks)} poses with one non-finite reach box")
    import torch
    # the border-clipped ones first, so that short queues hold them too
    idx = np.concatenate([clipped, np.setdiff1d(picks, clipped)])[:target]
    return torch.from_numpy(poses[idx]).cuda(), ref[idx]


def test_non_finite_zones_are_found(case):
    m, poses, ref, picks, clipped, mk = case
    print(f"{mk}: {len(picks)} poses with one non-finite reach box, {len(clipped)} of them clipped at the border")
    assert len(picks) >= max(TARGETS), (mk, len(picks))
    if mk == "fine":
        assert len(clipped) > 0


@pytest.mark.parametrize("timing", [False, True], ids=["side-by-side", "serial"])
@pytest.mark.parametrize("target", TARGETS)
def test_non_finite_group_queue_equals_the_oracle(case, target, timing):
    x, want = batch(case, target)
    chk = checker(case[0])
    chk.setTiming(timing)
    got = chk.isValidBatch(x).cpu().numpy()
    st = chk.stats()
    assert st["last_reach_plane_stage"] == target and st["last_queued_reach_stage"] == 0, st
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{bad.size} mismatches of {len(x)}, first {bad[:8]}, stats {st}"


@pytest.mark.parametrize("target", TARGETS)
def test_non_finite_on_the_warp_kernel_equals_the_oracle(case, target):
    x, want = batch(case, target)
    chk = checker(case[0], no_groups=True)
    got = chk.isValidBatch(x).cpu().numpy()
    st = chk.stats()
    assert st["last_reach_plane_stage"] == 0 and st["last_queued_reach_stage"] == target, st
    assert np.array_equal(got, want)


def test_only_mergeable_zones_stay_on_the_warp_kernel(case):
    """A whole probe batch: every record left in the one-warp reach queue is there for its mergeable planes."""
    m, poses = case[0], case[1]
    import torch
    chk = checker(m)
    got = chk.isValidBatch(torch.from_numpy(poses).cuda()).cpu().numpy()
    assert np.array_equal(got, case[2])
    zone, fl = chk.debugReachQueue()
    assert np.all(((fl & REC_MERGEFREE) == 0) | ((fl & REC_NEEDS_REDUCE) != 0)), fl
