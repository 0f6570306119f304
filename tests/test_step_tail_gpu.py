"""The step after the box kernels: the one-pass ordered compaction (compact_kernel) against numpy.nonzero, and the forked
device round, whose grouping stage no longer waits for the 8-lane reach kernel, against the serial round and the oracle."""
import numpy as np
import pytest

import cases
from art_planner_b200 import synth

pytestmark = pytest.mark.gpu

TILE = 4096   # items per compaction tile
SIZES = [1, 31, 32, 33, TILE - 1, TILE, TILE + 1, (1 << 20) + 7]
PATTERNS = ["all", "none", "alternating", "last", "random"]


@pytest.fixture(scope="module")
def chk():
    import art_planner_b200 as ap
    from art_planner_b200 import build
    build.build()
    return ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)


def mask(n, pattern, seed=0):
    if pattern == "all":
        return np.ones(n, np.uint8)
    if pattern == "none":
        return np.zeros(n, np.uint8)
    if pattern == "alternating":
        return (np.arange(n) % 2).astype(np.uint8)
    if pattern == "last":
        v = np.zeros(n, np.uint8)
        v[-1] = 1
        return v
    rng = np.random.default_rng(seed + n)
    return (rng.random(n) < 0.43).astype(np.uint8) * rng.integers(1, 256, n, dtype=np.uint8)   # any non-zero byte is valid


def bits_of(v, tail_ones=False):
    """Bit-packed words of v (item i = bit i&31 of word i>>5); with tail_ones the bits past n are set (not items)."""
    import torch
    n = len(v)
    w = (n + 31) // 32
    pad = np.zeros(w * 32, np.uint64)
    pad[:n] = v != 0
    if tail_ones:
        pad[n:] = 1
    words = (pad.reshape(w, 32) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)
    return torch.from_numpy(words.view(np.int32).copy()).cuda()


def run_all_forms(chk, v, base64, base32, outs):
    """Queue the three forms of one mask on the current stream; outs receives (form, base, want-mask, idx, cnt)."""
    import torch
    d = torch.from_numpy(v).cuda()
    idx, cnt = chk.compactValid(d, base=base64)
    outs.append(("i64", base64, v, idx, cnt))
    idx, cnt = chk.compactValidU32(d, base=base32)
    outs.append(("u32", base32, v, idx, cnt))
    idx, cnt = chk.compactBits(bits_of(v, tail_ones=True), len(v), base=base64)
    outs.append(("bits", base64, v, idx, cnt))


def check_outs(outs):
    import torch
    torch.cuda.synchronize()
    for form, base, v, idx, cnt in outs:
        want = np.nonzero(v)[0].astype(np.int64) + base
        got_n = int(cnt.item())
        got = idx[:got_n].cpu().numpy().astype(np.int64)
        if form == "u32":
            got &= 0xFFFFFFFF
        assert got_n == len(want), (form, len(v), got_n, len(want))
        assert np.array_equal(got, want), (form, len(v), np.nonzero(got != want)[0][:8])


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("pattern", PATTERNS)
def test_compaction_matches_nonzero(chk, n, pattern):
    outs = []
    run_all_forms(chk, mask(n, pattern), 1000, (1 << 31) - 5, outs)
    check_outs(outs)


def test_compaction_back_to_back_and_on_a_side_stream(chk):
    """Many calls queued on one handle without a synchronise: the tile statuses of one call are reused by the next (large
    calls before small ones leave statuses of later tiles behind), on the default stream and on a side stream."""
    import torch
    outs = []
    order = [(1 << 20) + 7, 33, TILE + 1, 1, (1 << 20) + 7, TILE, 31, 3 * TILE + 5]
    for k, n in enumerate(order):
        run_all_forms(chk, mask(n, PATTERNS[k % len(PATTERNS)], seed=k), 7 * k, (1 << 31) + k, outs)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for k, n in enumerate(order[:4]):
            run_all_forms(chk, mask(n, "random", seed=100 + k), 0, 0, outs)
    torch.cuda.current_stream().wait_stream(side)
    run_all_forms(chk, mask(TILE + 1, "random", seed=200), 3, 3, outs)
    check_outs(outs)


@pytest.mark.parametrize("mode", [0, 1], ids=["warp+group", "group-only"])
@pytest.mark.parametrize("name", ["terraces_low_yaml", "terraces_tilted_yaml"])
def test_forked_rounds_match_the_serial_rounds_and_the_oracle(maps, port_lib, name, mode):
    """Two rounds (2^20 + 20000 poses): every round forks the reach kernels, and its grouping stage runs beside the 8-lane
    kernel. The last round is the case's own poses, so its deferrals are counted. The host-fed (sliced) path too."""
    import torch
    import art_planner_b200 as ap
    _, mk, pk, gen = [c for c in cases.POSE_CASES if c[0] == name][0]
    m = maps(mk)
    p = gen(m)
    o = port_lib.Oracle(cases.PARAMS[pk], "port")
    o.set_map(m)
    r = o.check_poses(p)
    reps = -(-(1 << 20) // len(p))
    poses = np.concatenate([np.tile(p, (reps, 1))[: 1 << 20], p])
    ref = np.concatenate([np.tile(r, reps)[: 1 << 20], r])
    c = ap.StateValidityChecker(cases.PARAMS[pk], device=0)
    c.setMap(m)
    c.updateHeightField()
    c.setMode(mode)
    d = torch.from_numpy(poses).cuda()
    c.setTiming(False)
    fork = c.isValidBatch(d).cpu().numpy()
    st = c.stats()
    host = c.isValidBatch(poses)
    c.setTiming(True)
    serial = c.isValidBatch(d).cpu().numpy()
    assert st["last_deferred"] > 0, st
    assert np.array_equal(serial, ref), np.nonzero(serial != ref)[0][:8]
    assert np.array_equal(fork, serial), np.nonzero(fork != serial)[0][:8]
    assert np.array_equal(host, serial), np.nonzero(host != serial)[0][:8]
