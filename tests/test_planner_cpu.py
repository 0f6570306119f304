"""CPU: the rules oracle/planner_oracle.py restates for artp_planner_set_map / artp_plan -- observed, the SE(3) bounds,
satisfiesBounds / enforceBounds at their edges, the status table, the map-generation rule and the stream positions -- and
the C ABI's planner declarations."""
import math
import sys

import numpy as np
import pytest

from oracle import planner_oracle as po

EPS = sys.float_info.epsilon


def test_bounds_from_raw_layers_with_nan_inf_and_negative_zero():
    e = np.array([[np.nan, -np.inf, 2.5], [-0.0, np.inf, np.nan]], np.float32, order="F")
    low, high = po.se3_bounds(e, 0.5, 1.0, -2.0, 0.2)
    assert low[:2] == [1.0 - 1.0, -2.0 - 1.5] and high[:2] == [1.0 + 1.0, -2.0 + 1.5]   # +- the FULL length
    assert low[2] == 0.0 - 0.1 and high[2] == 2.5 + 0.1
    z = np.array([[-0.0, np.nan]], np.float32)
    low, high = po.se3_bounds(z, 1.0, 0.0, 0.0, 0.0)
    assert math.copysign(1.0, low[2]) == 1.0 and math.copysign(1.0, high[2]) == 1.0     # -0 counts as +0
    with pytest.raises(ValueError):
        po.se3_bounds(np.array([[np.nan, np.inf], [-np.inf, np.nan]], np.float32), 1.0, 0.0, 0.0, 0.2)


def test_observed_with_missing_or_holed_traversability():
    e = np.array([[0.0, np.nan], [np.inf, 1.0]], np.float32)
    t = np.array([[np.nan, 1.0], [1.0, 0.5]], np.float32)
    assert po.observed(e).tolist() == [[1.0, 0.0], [0.0, 1.0]]          # no traversability: checkTraversability's 1.0
    assert po.observed(e, t).tolist() == [[0.0, 0.0], [0.0, 1.0]]
    assert po.observed(e, t).dtype == np.float32


def test_satisfies_bounds_at_the_epsilon_slack():
    low, high = [-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]
    q = [0.0, 0.0, 0.0, 1.0]
    at = [1.0 + EPS, 0.0, 0.0] + q
    assert po.satisfies_bounds(at, low, high)                            # exactly high + DBL_EPSILON: inside
    beyond = [np.nextafter(1.0 + EPS, 2.0), 0.0, 0.0] + q
    assert not po.satisfies_bounds(beyond, low, high)                    # one ulp beyond
    g, clipped = po.clip_goal(at, low, high)
    assert not clipped and g[0] == 1.0 + EPS                             # satisfied: not clamped
    g, clipped = po.clip_goal(beyond, low, high)
    assert clipped and g[0] == 1.0
    below = [-1.0 - 2 * EPS, 0.0, 0.0] + q
    assert not po.satisfies_bounds(below, low, high)
    assert po.clip_goal(below, low, high)[0][0] == -1.0


def test_enforce_bounds_quaternions():
    """SO3StateSpace: satisfiesBounds at |norm - 1| < 1e-9, enforceBounds on the SQUARED norm against DBL_EPSILON."""
    low, high = [-1.0] * 3, [1.0] * 3
    w = 1.0 + 2 * EPS                                                     # norm 1 + 2 eps: the SO3 test alone passes
    assert po.satisfies_bounds([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, w], low, high)
    g, clipped = po.clip_goal([2.0, 0.0, 0.0, 0.0, 0.0, 0.0, w], low, high)
    assert clipped and g[0] == 1.0                                        # position clamped ...
    assert g[6] == w / math.sqrt(w * w) == 1.0                            # ... and |norm^2 - 1| = 4 eps > eps: normalised
    w = 1.0 + EPS / 2                                                     # rounds to 1: norm^2 - 1 = 0, untouched
    g, _ = po.clip_goal([2.0, 0.0, 0.0, 0.0, 0.0, 0.0, w], low, high)
    assert g[6] == w
    for s in (1.0 + 2e-9, 1.0 - 2e-9):                                    # outside the 1e-9 tolerance: normalised
        g, clipped = po.clip_goal([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, s], low, high)
        assert clipped and g[6] == s / math.sqrt(s * s)
    g, clipped = po.clip_goal([0.5, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0], low, high)
    assert clipped and g.tolist() == [0.5, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]   # zero quaternion: identity
    g, _ = po.clip_goal([0.5, 0.0, 0.0, 0.0, 0.0, 0.0, EPS / 2], low, high)
    assert g.tolist() == [0.5, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]               # norm below DBL_EPSILON: identity
    g, _ = po.clip_goal([3.0, -4.0, 0.0, 0.0, 0.0, 0.0, 2.0], low, high)
    assert g.tolist() == [1.0, -1.0, 0.0, 0.0, 0.0, 0.0, 1.0]             # both components enforced


def test_status_table():
    assert po.status(po.SOLVE_SOLVED) == po.SOLVED == 5
    assert po.status(po.SOLVE_NOT_CONNECTED) == po.status(po.SOLVE_NO_FEASIBLE_PATH) == po.NOT_SOLVED == 4
    assert po.status(po.SOLVE_INVALID_START) == po.INVALID_START == 1
    assert po.status(po.SOLVE_INVALID_GOAL) == po.INVALID_GOAL == 2
    assert po.NO_MAP == 3 and po.UNKNOWN == 0 and po.status(0) == po.UNKNOWN


def test_map_generation_rule():
    r = po.GenerationRule()
    r.new_map()
    assert r.plan(False) == (False, True)         # first plan on a map: sample
    assert r.plan(False) == (False, False)        # same map: no sampling
    assert r.plan(True) == (True, False)          # same map, cleared: start and goal only (the reference's quirk)
    r.new_map()
    assert r.plan(True) == (True, True)           # a new map: sample again
    assert r.plan(False) == (False, False)


def test_stream_positions():
    assert po.advance(10, 3, 100) == 13 and po.advance(10, -1, 100) == 110 and po.advance(10, 0, 100) == 10


def test_header_declares_the_planner():
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    txt = open(os.path.join(root, "include", "artp.h")).read()
    for name in ("artp_planner_set_map", "artp_planner_get_space", "artp_plan"):
        assert re.search(r"\b%s\s*\(" % name, txt)
    for k, v in (("UNKNOWN", 0), ("INVALID_START", 1), ("INVALID_GOAL", 2), ("NO_MAP", 3), ("NOT_SOLVED", 4), ("SOLVED", 5)):
        assert re.search(r"#define ARTP_PLANNER_%s\s+%d\b" % (k, v), txt)


def test_ctypes_structs_match_the_header_layout():
    """The Python mirror's structs have the C layout: compiled with the host compiler against include/artp.h."""
    import ctypes as C
    import os
    import shutil
    import subprocess
    import tempfile
    from art_planner_b200 import capi
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("g++ absent")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = ('#include <cstdio>\n#include <cstddef>\n#include "artp.h"\nint main() { std::printf("%zu %zu %zu %zu\\n", '
           'sizeof(artp_planner_params), sizeof(artp_plan_info), offsetof(artp_plan_info, simplify), '
           'offsetof(artp_plan_info, host_syncs)); }\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.cpp"), "w").write(src)
        subprocess.run([cxx, "-I", os.path.join(root, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.cpp")], check=True)
        out = subprocess.run([os.path.join(d, "t")], capture_output=True, text=True, check=True).stdout.split()
    assert [int(x) for x in out] == [C.sizeof(capi.ArtpPlannerParams), C.sizeof(capi.ArtpPlanInfo),
                                      capi.ArtpPlanInfo.simplify.offset, capi.ArtpPlanInfo.host_syncs.offset]
