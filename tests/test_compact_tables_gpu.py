"""GPU (-m gpu): the classify stage decides most boxes from the compact range tables (a 15-bit code interval around the
exact zone max / min) and falls back to the exact tables when an interval leaves a test open. These poses put box
bottoms and tops within about one code step of their zone's max or min, on a map whose codes are coarse (heights
around +300 m, -inf patches in the masked layer), so both outcomes of every interval test occur. Masks must equal the
oracle's."""
import numpy as np
import pytest

import cases
from art_planner_b200 import synth

pytestmark = pytest.mark.gpu


def offset_map():
    m = synth.make_fbm_map(400, 400, amp=0.6, seed=5)
    m.elevation += np.float32(300.0)
    masked = m.elevation_masked + np.float32(300.0)
    masked[40:60, 100:130] = -np.inf
    masked[200:203, 50:300] = -np.inf
    m.elevation_masked = np.asfortranarray(masked)
    return m


def code_step(layer):
    """The compact tables' step: the smallest power of two with base + 32765 * step >= the largest finite height
    (kCodeMax, artp_device.cuh)."""
    h = layer[np.isfinite(layer)]
    base, top = np.float32(h.min()), np.float32(h.max())
    e = -126
    while base + np.float32(32765) * np.float32(2.0 ** e) < top:
        e += 1
    return 2.0 ** e


def boundary_poses(m, n, seed, p=synth.PARAMS_YAML):
    """Terrain poses whose z is shifted so that one box (torso or a reach box, drawn per pose) has its bottom or top
    within ~1.5 code steps of its zone's max or min (the zone restated in float64; near cell borders it may be one
    vertex off, which only moves the target)."""
    poses = synth.make_terrain_poses(m, n, seed=seed)
    rng = np.random.default_rng(seed)
    t = poses[:, :3]
    x, y, z, w = (poses[:, i] for i in range(3, 7))
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                  2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                  2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    lx, ly = m.length
    sW, sD = np.float32(lx) / (m.rows - 1), np.float32(ly) / (m.cols - 1)
    box = rng.integers(0, 5, n)            # 0 torso, 1..4 reach boxes
    kind = rng.integers(0, 4, n)           # bottom vs max, top vs min, bottom vs min, top vs max
    frac = rng.uniform(-1.5, 1.5, n)
    out = poses.copy()
    for k in range(5):
        sel = np.nonzero(box == k)[0]
        if k == 0:
            off, side, layer = (p.torso_off_x, p.torso_off_y, p.torso_off_z - p.feet_off_z), \
                (p.torso_length, p.torso_width, p.torso_height), m.elevation
        else:
            fk = k - 1
            off = (-p.feet_off_x if fk & 2 else p.feet_off_x, -p.feet_off_y if fk & 1 else p.feet_off_y, 0.0)
            side, layer = (p.reach_x, p.reach_y, p.reach_z), m.elevation_masked
        step = code_step(layer)
        Rs = R[sel]
        c = np.einsum("nij,j->ni", Rs, np.array(off)) + t[sel]
        s = np.array(side)
        xr = 0.5 * (np.abs(Rs[:, 0, :]) * s).sum(1)
        yr = 0.5 * (np.abs(Rs[:, 2, :]) * s).sum(1)
        zr = 0.5 * (np.abs(Rs[:, 1, :]) * s).sum(1)
        P0 = -(c[:, 0] - m.cx) + 0.5 * lx
        P2 = (c[:, 1] - m.cy) + 0.5 * ly
        x0 = np.clip(np.floor((P0 - xr) / sW), 0, m.rows - 1).astype(int)
        x1 = np.clip(np.ceil((P0 + xr) / sW), 0, m.rows - 1).astype(int)
        z0 = np.clip(np.floor((P2 - zr) / sD), 0, m.cols - 1).astype(int)
        z1 = np.clip(np.ceil((P2 + zr) / sD), 0, m.cols - 1).astype(int)
        for a, i in enumerate(sel):
            # field vertex (x, z) holds layer[x, cols - 1 - z]
            zone = layer[x0[a]:x1[a] + 1, m.cols - 1 - z1[a]:m.cols - z0[a]]
            fin = zone[np.isfinite(zone)]
            if fin.size == 0:
                continue
            ref = fin.max() if kind[i] in (0, 3) else fin.min()
            edge = c[a, 2] - yr[a] if kind[i] in (0, 2) else c[a, 2] + yr[a]
            out[i, 2] += (float(ref) + frac[i] * step) - edge
    return out


@pytest.mark.parametrize("mode", [0, 1], ids=["default", "group-only"])
def test_compact_table_intervals_agree_with_the_oracle(port_lib, mode):
    import art_planner_b200 as ap
    m = offset_map()
    assert code_step(m.elevation_masked) >= 2.0 ** -15        # coarse: ~ the float spacing of the heights themselves
    poses = boundary_poses(m, 20000, seed=91)
    o = port_lib.Oracle(cases.PARAMS["yaml"], "port")
    o.set_map(m)
    ref = o.check_poses(poses)
    assert 0.05 < ref.mean() < 0.95, ref.mean()
    chk = ap.StateValidityChecker(cases.PARAMS["yaml"], device=0)
    chk.setMap(m)
    chk.updateHeightField()
    chk.setMode(mode)
    got = chk.isValidBatch(poses)
    bad = np.nonzero(got != ref)[0]
    assert bad.size == 0, f"{bad.size} mismatches, first {bad[:8]}"
    one = np.array([chk.isValid(s) for s in poses[:64]], dtype=np.uint8)   # the single-state latency path
    assert np.array_equal(one, ref[:64])
