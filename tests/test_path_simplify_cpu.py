"""The path-simplifier restatement (oracle/path_simplify_oracle.py) pinned rule by rule on hand-built paths in a synthetic
free space -- discs of invalid (x, y) -- with explicit variates. The device (tests/test_path_simplify_gpu.py) is compared
with this restatement, so each rule is pinned here without a GPU."""
import numpy as np
import pytest

import philox_ref
from oracle import path_simplify_oracle as pso

SPACE = ([-20.0, -20.0, -1.0], [20.0, 20.0, 1.0], 0.01)    # segments of about 0.57 m


def discs(*d):
    """isValid: (x, y) outside every disc (cx, cy, r)."""
    def valid(states):
        s = np.asarray(states, np.float64).reshape(-1, 7)
        ok = np.ones(len(s), bool)
        for cx, cy, r in d:
            ok &= (s[:, 0] - cx) ** 2 + (s[:, 1] - cy) ** 2 > r * r
        return ok
    return valid


def st(x, y):
    return np.array([x, y, 0.0, 0.0, 0.0, 0.0, 1.0])


def path_xy(pts):
    return [st(x, y) for x, y in pts]


def fixed(u):
    """variates(call, attempt) -> u[attempt] (then the last one)."""
    return lambda c, i: u[min(i, len(u) - 1)]


class Recorder(pso.Simplifier):
    """A simplifier whose checkMotion answers from `verdict(a, b)` and records the (x, y) of both ends."""

    def __init__(self, verdict, variates=None):
        super().__init__(discs(), SPACE, 0, variates)
        self.verdict, self.seen = verdict, []

    def check_motion(self, a, b):
        self.stats["motions"] += 1
        self.seen.append(((float(a[0]), float(a[1])), (float(b[0]), float(b[1]))))
        return self.verdict(a, b)


def u_int(k, a, b):
    """A variate that uniformInt(a, b) maps to k."""
    return (k - a + 0.5) / (b - a + 1)


def test_philox_draws_match_reference():
    for seed, call, i in ((0, 0, 0), (7, 3, 11), (2 ** 40 + 5, 17, 2 ** 20)):
        u0, u1 = pso.philox_variates(seed, call, i)
        ctr = np.array([[i, call, 0, 0x41525453]], np.uint32)
        w = philox_ref.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32)).astype(np.uint64)[0]
        assert u0 == int((w[1] << np.uint64(32) | w[0]) >> np.uint64(11)) * 2.0 ** -53
        assert u1 == int((w[3] << np.uint64(32) | w[2]) >> np.uint64(11)) * 2.0 ** -53
        assert 0.0 <= u0 < 1.0 and 0.0 <= u1 < 1.0
    assert pso.philox_variates(1, 0, 0) != pso.philox_variates(1, 1, 0) != pso.philox_variates(1, 0, 1)
    assert pso.uniform_int(0.0, 2, 5) == 2 and pso.uniform_int(1.0 - 2 ** -53, 2, 5) == 5 and pso.uniform_int(0.5, 0, 0) == 0


def test_reduce_front_back_success():
    p = path_xy([(0, 0), (1, 1), (2, 0), (3, 1), (4, 0)])
    sim = pso.Simplifier(discs(), SPACE, 1)
    assert sim.reduce_vertices(p) and len(p) == 2 and sim.stats["motions"] == 1 and sim.stats["reduce"] == 1


def test_reduce_plus_minus_two_rule_and_skips():
    p = path_xy([(k, 0) for k in range(6)])          # maxN = 5, range = 1 + floor(0.5 + 6 * 0.33) = 3
    # p1 = 4, p2 = 4: p1 < maxN - 1 fails, p1 > 1 -> p2 = 2 (swapped: 2, 4); p1 = 0, p2 = 1 -> p2 = 2
    u = [(u_int(4, 0, 5), u_int(4, 1, 5)), (u_int(0, 0, 5), u_int(1, 0, 3))]
    sim = Recorder(lambda a, b: False, fixed(u))
    sim.call = 0
    p0 = list(p)
    sim.reduce_vertices(p)
    assert sim.seen[1] == ((2.0, 0.0), (4.0, 0.0)) and sim.seen[2] == ((0.0, 0.0), (2.0, 0.0))
    # nochange: every motion fails -> exactly maxSteps = 6 attempts after the front-back check
    assert len(sim.seen) == 1 + 6 and p == p0
    # three states: p1 = 1 has no partner (skip), p1 = 0 -> (0, 2), p1 = 2 -> (0, 2)
    q = path_xy([(0, 0), (1, 0), (2, 0)])
    sim = Recorder(lambda a, b: False, fixed([(u_int(1, 0, 2), 0.5)]))
    sim.reduce_vertices(q)
    assert len(sim.seen) == 1                          # the front-back check only: all 3 attempts skipped
    sim = Recorder(lambda a, b: False, fixed([(u_int(2, 0, 2), 0.5)]))
    sim.reduce_vertices(q)
    assert sim.seen[1:] == [((0.0, 0.0), (2.0, 0.0))] * 3


def test_reduce_success_resets_nochange():
    p = path_xy([(k, 0) for k in range(8)])
    # attempt 0 erases between 1 and 3 (front-back fails); the call then runs until 8 attempts (maxSteps)
    u = [(u_int(1, 0, 7), u_int(3, 0, 5))]            # range = 4: p2 in [0, 5]
    sim = Recorder(lambda a, b: not (a[0] == 0 and b[0] == 7) and (a[0], b[0]) == (1, 3), fixed(u))
    assert sim.reduce_vertices(p) and [s[0] for s in p] == [0, 1, 3, 4, 5, 6, 7]
    assert sim.stats["reduce"] == 1 and len(sim.seen) == 1 + 8


def test_collapse_mark_survives_erasure():
    pts = [(0.25, 1.0), (5, 0), (0, 1), (-5, 0), (0, 1.1), (5, 5)]
    p = path_xy(pts)
    bad = ((0.0, 1.0), (0.0, 1.1))
    sim = Recorder(lambda a, b: ((a[0], a[1]), (b[0], b[1])) == ((0.25, 1.0), (0.0, 1.0)))
    assert sim.collapse_close_vertices(p)
    assert sim.seen[0] == bad and sim.seen[1] == ((0.25, 1.0), (0.0, 1.0))
    assert sim.seen.count(bad) == 1                    # after state (5, 0) is erased the pair keeps its mark
    assert [(s[0], s[1]) for s in p] == [(0.25, 1.0), (0, 1), (-5, 0), (0, 1.1), (5, 5)]


ZIG = path_xy([(k, 3.0 * (k % 2)) for k in range(9)])    # 8 segments of sqrt(10): L = 25.3, rd = 8.35, snap 0.126


def shortcut_once(p0, p1, verdict=lambda a, b: True):
    """One shortcutPath attempt on ZIG with its points at arc lengths p0, p1."""
    path = [s.copy() for s in ZIG]
    dists = [0.0]
    for a, b in zip(path[:-1], path[1:]):
        dists.append(dists[-1] + pso.distance(a, b))
    L = dists[-1]
    sc = {"dists": dists, "threshold": L * pso.SNAP_TO_VERTEX, "rd": pso.RANGE_RATIO * L}
    lo, hi = max(0.0, p0 - sc["rd"]), min(p0 + sc["rd"], L)
    sim = Recorder(verdict, fixed([(p0 / L, (p1 - lo) / (hi - lo))]))
    changed = sim._shortcut_attempt(path, sc, 0, 0)
    return changed, path, sim, dists


def xy(path):
    return [(round(s[0], 9), round(s[1], 9)) for s in path]


def test_shortcut_edit_cases():
    d = 10.0 ** 0.5
    # both snapped (vertices 2 and 4): the states between are erased
    ok, p, _, _ = shortcut_once(2 * d, 4 * d)
    assert ok and xy(p) == xy(ZIG[:3] + ZIG[4:])
    # both interpolated, not adjacent (segments 1 and 3): states 2 and 3 become s0 and s1
    ok, p, _, _ = shortcut_once(1.5 * d, 3.5 * d)
    assert ok and len(p) == 9 and xy(p)[2:4] == [(1.5, 1.5), (3.5, 1.5)] and xy(p)[4:] == xy(ZIG[4:])
    # both interpolated, adjacent segments (1 and 2): state 2 becomes s0 and s1 is inserted after it
    ok, p, _, _ = shortcut_once(1.5 * d, 2.5 * d)
    assert ok and len(p) == 10 and xy(p)[2:4] == [(1.5, 1.5), (2.5, 1.5)] and xy(p)[4:] == xy(ZIG[3:])
    # snapped then interpolated (vertex 2, segment 4): state 4 becomes s1, state 3 is erased
    ok, p, _, _ = shortcut_once(2 * d, 4.5 * d)
    assert ok and xy(p) == xy(ZIG[:3]) + [(4.5, 1.5)] + xy(ZIG[5:])
    # interpolated then snapped (segment 1, vertex 4): state 2 becomes s0, state 3 is erased
    ok, p, _, _ = shortcut_once(1.5 * d, 4 * d)
    assert ok and xy(p) == xy(ZIG[:2]) + [(1.5, 1.5)] + xy(ZIG[4:])
    # drawn in the other order: the same edit, checkMotion from the first-drawn point
    ok, p, sim, _ = shortcut_once(4 * d, 1.5 * d)
    assert ok and xy(p) == xy(ZIG[:2]) + [(1.5, 1.5)] + xy(ZIG[4:]) and sim.seen[0][0] == (4.0, 0.0)


def test_shortcut_skips_and_rejections():
    d = 10.0 ** 0.5
    # same segment, and a vertex next to the other point's segment: no motion is checked
    for p0, p1 in ((1.2 * d, 1.7 * d), (2 * d, 2.5 * d), (2.5 * d, 2 * d)):
        ok, p, sim, _ = shortcut_once(p0, p1)
        assert not ok and sim.seen == [] and xy(p) == xy(ZIG)
    # a point snapped to the waypoint that ends the other point's segment, and two snapped neighbours
    for p0, p1 in ((1.5 * d, 2 * d - 0.01), (2 * d - 0.01, 1.5 * d), (2 * d, 3 * d), (3 * d + 0.01, 2 * d)):
        ok, p, sim, _ = shortcut_once(p0, p1)
        assert not ok and sim.seen == [] and xy(p) == xy(ZIG)
    # a failing motion, and a shortcut no cheaper than the path (vertex 2 to segment 3: along 1.58 < direct 2.12)
    ok, _, sim, _ = shortcut_once(1.5 * d, 3.5 * d, lambda a, b: False)
    assert not ok and len(sim.seen) == 1
    ok, p, sim, _ = shortcut_once(2 * d, 3.5 * d)
    assert not ok and len(sim.seen) == 1 and xy(p) == xy(ZIG)


def test_shortcut_snapping_at_threshold():
    d = 10.0 ** 0.5
    _, _, _, dists = shortcut_once(0.0, 0.0)
    thr = dists[-1] * pso.SNAP_TO_VERTEX
    assert pso.Simplifier._locate(dists, 2 * d - 0.9 * thr, thr) == (2, 2)     # snapped to the next waypoint
    assert pso.Simplifier._locate(dists, 2 * d + 0.9 * thr, thr) == (2, 2)     # snapped to the previous one
    assert pso.Simplifier._locate(dists, 2 * d - 1.1 * thr, thr) == (1, -1)
    assert pso.Simplifier._locate(dists, 2 * d + 1.1 * thr, thr) == (2, -1)
    assert pso.Simplifier._locate(dists, 0.0, thr) == (0, 0)
    assert pso.Simplifier._locate(dists, dists[-1], thr) == (8, 8)


def test_bspline_subdivide_min_change_and_early_stop():
    p = path_xy([(0, 0), (1, 1), (2, 0)])
    s = pso.subdivide(p)
    assert xy(s) == [(0, 0), (0.5, 0.5), (1, 1), (1.5, 0.5), (2, 0)]
    # min_change above every change: nothing replaced, the first step ends it (1 isValid, 2 checkMotion)
    sim = pso.Simplifier(discs(), SPACE)
    q = list(p)
    sim.smooth_bspline(q, 3, 10.0)
    assert len(q) == 5 and sim.stats["bspline"] == 0 and sim.stats["valids"] == 1 and sim.stats["motions"] == 2
    # a small min_change: the corner moves to mid(mid(a, c), mid(c, b)) = (1, 0.75), then two more steps
    sim = pso.Simplifier(discs(), SPACE)
    q = list(p)
    sim.smooth_bspline(q, 3, 1e-3)
    assert len(q) == 17 and sim.stats["bspline"] >= 3
    # minChange at the first replacement's distance: strictly greater is required. The corner (1, 1) moves to
    # mid(mid(a, c), mid(c, b)) = (1, 0.75), a distance of 0.25
    first = pso.distance(st(1, 1), st(1, 0.75))
    for mc, replaced in ((np.nextafter(first, 0.0), 1), (first, 0), (np.nextafter(first, 1.0), 0)):
        sim = pso.Simplifier(discs(), SPACE)
        q = list(p)
        sim.smooth_bspline(q, 1, mc)
        assert sim.stats["bspline"] == replaced and len(q) == 5
        assert xy(q)[2] == ((1.0, 0.75) if replaced else (1.0, 1.0))
    # an invalid state before i: no motion is checked for that i
    sim = pso.Simplifier(discs((0.5, 0.5, 0.1)), SPACE)
    q = list(p)
    sim.smooth_bspline(q, 1, 1e-3)
    assert sim.stats["valids"] == 1 and sim.stats["motions"] == 0 and sim.stats["bspline"] == 0


def path_cost_const(c):
    return lambda states: c


def test_get_solution_path_returns():
    p = path_xy([(0, 0), (1, 1), (2, 0), (3, 1), (4, 0)])
    # equal cost: the simplified path
    out, info, simp = pso.get_solution_path(p, discs(), SPACE, 3, path_cost_const(1.0))
    assert info["returned_simplified"] == 1 and len(out) == len(simp) == 2 and info["check_passed"] == 1
    # the original strictly cheaper: the original
    out, info, _ = pso.get_solution_path(p, discs(), SPACE, 3, lambda s: 1.0 / len(s))
    assert info["returned_simplified"] == 0 and len(out) == 5 and info["cost_original"] < info["cost_simplified"]
    # the end state invalid: the check fails, the original comes back, nothing is priced
    out, info, _ = pso.get_solution_path(p, discs((4, 0, 0.2)), SPACE, 3, path_cost_const(1.0))
    assert info["check_passed"] == 0 and info["returned_simplified"] == 0 and np.array_equal(out, np.array(p))
    assert np.isnan(info["cost_original"])
    # fewer than 3 states: only PathGeometric::check (isValid(front), then the motion)
    out, info, _ = pso.get_solution_path(p[:2], discs(), SPACE, 3, path_cost_const(1.0))
    assert (info["motion_checks"], info["state_checks"], info["calls"]) == (1, 1, 0)


def test_schedule_calls_and_seed():
    """A path around a disc: every stage runs and the schedule is deterministic in the seed. With seed 8 a shortcut
    passes the discrete motion check while its chord cuts the disc between two checked states; subdivide's midpoints
    then fall inside, so the final check fails and the original comes back (what checkAndRepair would repair)."""
    pts = [(np.cos(t) * 3, np.sin(t) * 3) for t in np.linspace(0, np.pi, 25)]
    p = path_xy(pts)
    runs = [pso.get_solution_path(p, discs((0, 0, 2.5)), SPACE, s, path_cost_const(0.0)) for s in (8, 8, 9)]

    def counters(info):
        return {k: v for k, v in info.items() if not k.startswith("cost")}
    assert counters(runs[0][1]) == counters(runs[1][1]) and np.array_equal(runs[0][2], runs[1][2])
    info = runs[0][1]
    assert info["calls"] == 9 and info["reduce_edits"] and info["shortcut_edits"] and info["bspline_edits"]
    assert info["check_passed"] == 0 and np.array_equal(runs[0][0], np.array(p))
    assert not discs((0, 0, 2.5))(runs[0][2]).all()
    assert counters(runs[2][1]) != counters(info)


def test_golden_rebuilt_over_the_port():
    """tests/golden/path_simplify.npz (isValid from the reference's compiled ODE) rebuilt with the port oracle: equal."""
    import os
    from oracle import make_golden_path_simplify as mg
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "path_simplify.npz"))
    res = mg.simplify_all("port")
    assert sorted(res) == sorted(g.files)
    for k in g.files:
        assert np.array_equal(res[k], g[k], equal_nan=k.endswith("/costs")), k
    info = np.array([g[k] for k in g.files if k.endswith("/info")])
    col = {name: i for i, name in enumerate(mg.INFO_KEYS)}
    assert info[:, col["check_passed"]].any() and not info[:, col["check_passed"]].all()
    assert info[:, col["shortcut_edits"]].any() and info[:, col["bspline_edits"]].any() and info[:, col["collapse_edits"]].any()
