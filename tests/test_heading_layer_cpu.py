"""CPU checks of the valid-heading layer's definition (artp_valid_heading_layer): the port oracle against the fixture the
compiled reference wrote, the cell centres the layer projects, and the headings' float cast."""
import os

import numpy as np
import pytest

import heading_layer_cases as hlc
import start_goal_oracle as sgo
from oracle.make_golden import digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def hl_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "heading_layer.npz"))


class _Normals:
    def __init__(self, port_lib, m, radius):
        self.normal_x, self.normal_y, self.normal_z, _ = port_lib.estimate_normals(m, radius)


@pytest.mark.parametrize("name,mk,pk,hk", hlc.GOLDEN_CASES, ids=[c[0] for c in hlc.GOLDEN_CASES])
def test_port_oracle_matches_reference_fixture(hl_golden, port_lib, name, mk, pk, hk):
    m, p, yaws = hlc.MAPS[mk](), hlc.PARAMS[pk], hlc.HEADINGS[hk]
    assert str(hl_golden[name + "/sha"]) == digest(m.elevation, m.elevation_masked, yaws), "generator drift"
    o = port_lib.Oracle(p, "port")
    o.set_map(m)
    poses, inside = sgo.pose_from_2d(m, _Normals(port_lib, m, hlc.normal_radius(p)), hlc.yaw_states(m, yaws))
    assert inside.all()
    masks = hlc.pack(o.check_poses(poses), len(yaws), (m.rows, m.cols))
    want = hl_golden[name + "/masks"]
    assert masks.dtype == want.dtype == np.uint32 and np.array_equal(masks, want)
    cells = hl_golden[name + "/pose_cells"]
    assert np.array_equal(cells, hlc.pose_cells(m))
    got = poses.reshape(-1, len(yaws), 7)[cells].reshape(-1, 7)
    assert np.array_equal(got.view(np.uint64), hl_golden[name + "/poses"].view(np.uint64))


def test_fixture_covers_mixed_verdicts_and_the_ulp_rule(hl_golden):
    for name, mk, pk, hk in hlc.GOLDEN_CASES:
        masks = hl_golden[name + "/masks"]
        n = len(hlc.HEADINGS[hk])
        assert (masks >> np.uint32(n) == 0).all(), name                    # no bit past the last heading
        bits = (masks[..., None] >> np.arange(n, dtype=np.uint32)) & 1
        assert bits.any() and not bits.all(), name
        if hk == "ulp":                                                    # yaws that round to yaw 0's float
            for k in hlc.ULP_SAME:
                assert np.array_equal(bits[..., k], bits[..., 0]), name
    # some cells accept only some of their headings: the layer is not a per-cell verdict
    m8 = hl_golden["hl_fbm_rough_yaml/masks"]
    assert ((m8 != 0) & (m8 != 0xFF)).mean() > 0.05


@pytest.mark.parametrize("mk", sorted(hlc.MAPS))
def test_every_cell_centre_maps_back_to_its_cell(mk):
    """grid_map::getIndexFromPosition + isInside restated (start_goal_oracle.pose_from_2d's rule) sends each cell centre the
    layer projects to the cell it came from."""
    m = hlc.MAPS[mk]()
    x, y = hlc.cell_centres(m)
    Lx, Ly = m.rows * m.res, m.cols * m.res
    row = np.trunc(-(((x - 0.5 * Lx) - m.cx) / m.res))
    col = np.trunc(-(((y - 0.5 * Ly) - m.cy) / m.res))
    tx, ty = -((x - m.cx) - 0.5 * Lx), -((y - m.cy) - 0.5 * Ly)
    assert ((tx >= 0.0) & (ty >= 0.0) & (tx < Lx) & (ty < Ly)).all()
    r, c = np.indices((m.rows, m.cols))
    assert np.array_equal(row, r.ravel(order="F")) and np.array_equal(col, c.ravel(order="F"))


def test_heading_states_carry_the_float_yaw():
    """Every heading set gives states whose getYawFromSO3 is (float)yaw, +-pi included (their float lies past +-pi)."""
    for hk, yaws in hlc.HEADINGS.items():
        q = hlc.heading_quaternions(yaws)
        s = np.concatenate([np.zeros((len(q), 3)), q], axis=1)
        assert np.array_equal(hlc.so3_yaw(s), np.asarray(yaws).astype(np.float32)), hk
    y = hlc.HEADINGS["ulp"]
    assert y[1] != y[0] and y[2] != y[0] and np.float32(y[1]) == np.float32(y[0]) == np.float32(y[2])
    assert np.float32(y[3]) == np.nextafter(np.float32(y[0]), np.float32(4.0))


def test_pack_layout():
    """Bit k of a cell is heading k of that cell; cells are column-major."""
    valid = np.zeros(2 * 3 * 5, np.uint8)
    valid[(1 + 2 * 2) * 5 + 3] = 1                                         # cell (1, 2), heading 3
    masks = hlc.pack(valid, 5, (2, 3))
    assert masks[1, 2] == 8 and masks.sum() == 8 and masks.flags.f_contiguous
