"""Box verdicts (artp_box_verdicts) restated over the oracle libraries' single-box collider (TEST INFRASTRUCTURE ONLY).

StateValidityChecker::isValid (validity_checker.cpp:39-45) stops at its first failing box. The box verdicts decide each of
its five boxes on their own: box k = 0 is the torso (ValidityCheckerBody::isValid, validity_checker_body.cpp:27-42),
k = 1..4 the reach boxes (+,+), (+,-), (-,+), (-,-) (boxIsValidAtPose, validity_checker_feet.cpp:32-70). The word has
bit k when box k fails and bit 8 + k when box k's centre is off the map (grid_map isInside).

The boxes are placed exactly as orc_state_valid places them (oracle/artp_wrappers.h): Pose3FromSE3's float32 rotation
(utils.h:25-38, no normalisation), Eigen's R * o + t reduced as a0 + (a1 + a2), isInside in double. numpy's float32
products and sums are single IEEE operations (no FMA contraction), so the centres equal the C ones bit for bit. Each box
is then decided by Oracle.box_collide, i.e. orc_box_collide of the port library or of the reference's compiled ODE.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def pose3_from_se3(states):
    """(t [n, 3], R [n, 9] row-major) in float32, as orc_pose3_from_se3."""
    s = np.ascontiguousarray(states, dtype=np.float64)
    t = s[:, :3].astype(F32)
    x, y, z, w = (s[:, 3 + i].astype(F32) for i in range(4))
    two = F32(2.0)
    one = F32(1.0)
    tx, ty, tz = two * x, two * y, two * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    R = np.stack([one - (tyy + tzz), txy - twz, txz + twy,
                  txy + twz, one - (txx + tzz), tyz - twx,
                  txz - twy, tyz + twx, one - (txx + tyy)], axis=1)
    return t, R


def box_offsets(p):
    """The five box offsets in the body frame, float32 as the C casts make them: the torso, then the feet."""
    fx, fy = F32(p.feet_off_x), F32(p.feet_off_y)
    torso = (F32(p.torso_off_x), F32(p.torso_off_y), F32(p.torso_off_z - p.feet_off_z))
    return [torso] + [((-fx if (k & 2) else fx), (-fy if (k & 1) else fy), F32(0.0)) for k in range(4)]


def box_centre(R, t, o):
    """Translation of pose * Pose3FromXYZ(o): R o + t with the dot product reduced as a0 + (a1 + a2)."""
    return np.stack([(R[:, 3 * i] * o[0] + (R[:, 3 * i + 1] * o[1] + R[:, 3 * i + 2] * o[2])) + t[:, i]
                     for i in range(3)], axis=1)


def is_inside(m, px, py):
    """grid_map checkIfPositionWithinMap in double, on the float centre (orc_is_inside)."""
    lx, ly = m.rows * m.res, m.cols * m.res
    tx = -((px.astype(np.float64) - m.cx) - 0.5 * lx)
    ty = -((py.astype(np.float64) - m.cy) - 0.5 * ly)
    return (tx >= 0.0) & (ty >= 0.0) & (tx < lx) & (ty < ly)


def box_verdicts(oracle, p, m, states) -> np.ndarray:
    """uint16 [n] words of the states on map m (installed in `oracle`, an orc.Oracle) under robot parameters p."""
    t, R = pose3_from_se3(states)
    n = t.shape[0]
    rot12 = np.zeros((n, 12), F32)
    for r in range(3):
        rot12[:, 4 * r:4 * r + 3] = R[:, 3 * r:3 * r + 3]
    why = np.zeros(n, np.uint16)
    for k, o in enumerate(box_offsets(p)):
        foot = k > 0
        c = box_centre(R, t, o)
        inside = is_inside(m, c[:, 0], c[:, 1])
        fails = np.zeros(n, bool)
        if foot and p.unknown_space_untraversable:
            fails[~inside] = True                                   # validity_checker_feet.cpp:34-37
        idx = np.nonzero(inside)[0]
        if idx.size:
            hit = oracle.box_collide(1 if foot else 0, c[idx], rot12[idx]) != 0
            fails[idx] = ~hit if foot else hit                      # the torso must be free, a reach box must touch
        why |= (fails.astype(np.uint16) << np.uint16(k)) | ((~inside).astype(np.uint16) << np.uint16(8 + k))
    return why
