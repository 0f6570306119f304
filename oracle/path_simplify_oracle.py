"""Restatement of OMPL 1.4.2's path simplifier as Planner::getSolutionPath uses it (TEST INFRASTRUCTURE ONLY): the
definition artp_simplify_path follows. OMPL is not in the reference tree; every rule below is restated from OMPL 1.4.2
(unpinned) and cites the function it restates:

  PathSimplifier::simplifyMax / simplify        the schedule (simplify_max)
  PathSimplifier::reduceVertices                random vertex-to-vertex shortcuts (reduce_vertices)
  PathSimplifier::collapseCloseVertices         closest-pair shortcuts (collapse_close_vertices)
  PathSimplifier::shortcutPath                  random point-to-point shortcuts with a cost test (shortcut_path)
  PathSimplifier::smoothBSpline                 subdivide + corner smoothing (smooth_bspline)
  PathGeometric::subdivide / length / check     (subdivide, path_length, check)
  PathGeometric::checkAndRepair                 the check only: no repair sampling (check_and_repair)

The simplifier is built from the space information alone, so its objective is PathLengthOptimizationObjective: motion
cost = SE3StateSpace::distance, costs combine by +, a < b is "better"; it has no goal region, so findBetterGoal never
runs. The in-tree part, Planner::getSolutionPath (art_planner/src/planner.cpp:266-298), is get_solution_path.

Randomness: OMPL's RNG is a serial mt19937 whose stream cannot be reproduced here. Attempt i of the c-th simplifier call
of the schedule (every call of the five functions above takes the next c, from 0, whether or not it does anything)
draws two doubles from Philox4x32-10(key = seed, counter = (i, c, 0, "ARTS")), formed as artp_sampler_uniforms forms
them (u0 from words 0-1, u1 from words 2-3); uniformInt(a, b) = a + min(floor(u * (b - a + 1)), b - a) and
uniformReal(a, b) = a + u * (b - a).

isValid is an argument (states [n, 7] -> bool [n]), so the same code runs over the port oracle and the compiled
reference. checkMotion is DiscreteMotionValidator with validSegmentCount from the SE(3) space, as
oracle/roadmap_query_oracle.discrete_motion states it. SE3StateSpace::distance and ::interpolate are an argument too
(Se3Ops, libm by default): the schedule decides on exact ties -- evenly spaced states give equal distances -- that CUDA's
acos / sin and libm's can break differently, so a comparison with the device takes both from artp_debug_se3_ops.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import roadmap_oracle as ro
from oracle import roadmap_query_oracle as rqo

RANGE_RATIO = 0.33        # PathSimplifier's default rangeRatio
SNAP_TO_VERTEX = 0.005    # shortcutPath's default snapToVertex
REPEAT = 5                # simplify: reduceVertices again / shortcutPath at most this many times
BSPLINE_STEPS = 3         # simplify: smoothBSpline(path, 3, length / 100)
TAG = 0x41525453          # "ARTS"
INF = float("inf")


def philox_variates(seed: int, call: int, attempt: int):
    """(u0, u1) of attempt `attempt` of schedule call `call`."""
    import philox_ref   # tests/ is on sys.path under pytest and in the golden script
    ctr = np.array([[attempt & 0xFFFFFFFF, call & 0xFFFFFFFF, 0, TAG]], np.uint32)
    w = philox_ref.philox4x32_10(ctr, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)).astype(np.uint64)[0]
    u0 = float(int((w[1] << np.uint64(32) | w[0]) >> np.uint64(11))) / 9007199254740992.0
    u1 = float(int((w[3] << np.uint64(32) | w[2]) >> np.uint64(11))) / 9007199254740992.0
    return u0, u1


def uniform_int(u: float, a: int, b: int) -> int:
    return a + min(int(math.floor(u * float(b - a + 1))), b - a)


def uniform_real(u: float, a: float, b: float) -> float:
    return a + u * (b - a)


def distance(a, b) -> float:
    """SE3StateSpace::distance (R^3 Euclidean + acos(|q1.q2|), 0 above 1 - 1e-9), in the device's operation order."""
    r = 0.0
    for i in range(3):
        d = float(a[i]) - float(b[i])
        r += d * d
    dq = abs(float(a[3]) * float(b[3]) + float(a[4]) * float(b[4]) + float(a[5]) * float(b[5]) + float(a[6]) * float(b[6]))
    return math.sqrt(r) + (0.0 if dq > 1.0 - 1e-9 else math.acos(dq))


class Se3Ops:
    """SE3StateSpace::distance and ::interpolate over rows: distance(A, B) -> [n], interpolate(A, B, T) -> [n, 7].
    This one restates them with libm (distance above, roadmap_oracle.interpolate)."""

    @staticmethod
    def distance(A, B):
        return np.array([distance(a, b) for a, b in zip(A, B)], np.float64)

    @staticmethod
    def interpolate(A, B, T):
        return np.array([ro.interpolate(a, b, float(t)) for a, b, t in zip(A, B, T)], np.float64).reshape(-1, 7)


def path_length(path, ops=Se3Ops) -> float:
    """PathGeometric::length: the left-to-right sum of distance over consecutive states from 0.0."""
    L = 0.0
    if len(path) > 1:
        for d in ops.distance(np.array(path[:-1]), np.array(path[1:])).tolist():
            L += d
    return L


def subdivide(path, ops=Se3Ops) -> list:
    """PathGeometric::subdivide: interpolate(a, b, 0.5) after every state but the last."""
    if len(path) < 2:
        return list(path)
    mid = ops.interpolate(np.array(path[:-1]), np.array(path[1:]), np.full(len(path) - 1, 0.5))
    out = [path[0]]
    for m, s in zip(mid, path[1:]):
        out.append(m)
        out.append(s)
    return out


class Simplifier:
    """PathSimplifier(si) over is_valid and the SE(3) space (low[3], high[3], fraction). `variates(call, attempt)` ->
    (u0, u1) replaces the Philox stream (tests pin rules with explicit variates). The path is a list of [7] arrays;
    the functions edit it in place. `stats` counts edits per stage, checkMotion and isValid calls."""

    def __init__(self, is_valid, space, seed: int = 0, variates=None, ops=Se3Ops):
        self._valid = is_valid
        self._space = space
        self.ops = ops
        self.seed = int(seed)
        self.variates = variates or (lambda c, i: philox_variates(self.seed, c, i))
        self.call = 0
        self.stats = {"reduce": 0, "collapse": 0, "shortcut": 0, "bspline": 0, "motions": 0, "valids": 0}

    def _next_call(self) -> int:
        c = self.call
        self.call += 1
        return c

    def is_valid(self, s) -> bool:
        self.stats["valids"] += 1
        return bool(np.asarray(self._valid(np.asarray(s, np.float64).reshape(1, 7)))[0])

    def check_motion(self, a, b) -> bool:
        """DiscreteMotionValidator::checkMotion: interpolate(a, b, j / nd), j = 1 .. nd - 1, then b."""
        self.stats["motions"] += 1
        a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
        nd = max(rqo.segment_count(self._space, a, b), 1)
        states = b.reshape(1, 7)
        if nd > 1:
            t = np.array([j / nd for j in range(1, nd)])
            states = np.concatenate([self.ops.interpolate(np.repeat(a[None], nd - 1, 0), np.repeat(b[None], nd - 1, 0), t),
                                     states])
        return bool(np.all(np.asarray(self._valid(states), bool)))

    def _d(self, a, b) -> float:
        return float(self.ops.distance(np.asarray(a).reshape(1, 7), np.asarray(b).reshape(1, 7))[0])

    def _i(self, a, b, t: float):
        return self.ops.interpolate(np.asarray(a).reshape(1, 7), np.asarray(b).reshape(1, 7), [t])[0]

    # -- PathSimplifier::reduceVertices(path, 0, 0, 0.33) -----------------------------------------------------------
    def reduce_vertices(self, path) -> bool:
        call = self._next_call()
        if len(path) < 3:
            return False
        max_steps = max_empty = len(path)
        if self.check_motion(path[0], path[-1]):
            path[:] = [path[0], path[-1]]
            self.stats["reduce"] += 1
            return True
        result, nochange, i = False, 0, 0
        while i < max_steps and nochange < max_empty:
            count = len(path)
            max_n = count - 1
            rng = 1 + int(math.floor(0.5 + float(count) * RANGE_RATIO))
            u0, u1 = self.variates(call, i)
            p1 = uniform_int(u0, 0, max_n)
            p2 = uniform_int(u1, max(p1 - rng, 0), min(max_n, p1 + rng))
            skip = False
            if abs(p1 - p2) < 2:
                if p1 < max_n - 1:
                    p2 = p1 + 2
                elif p1 > 1:
                    p2 = p1 - 2
                else:
                    skip = True
            if not skip:
                if p1 > p2:
                    p1, p2 = p2, p1
                if self.check_motion(path[p1], path[p2]):
                    del path[p1 + 1:p2]
                    nochange = 0
                    result = True
                    self.stats["reduce"] += 1
            i += 1
            nochange += 1
        return result

    # -- PathSimplifier::collapseCloseVertices(path, 0, 0) ---------------------------------------------------------
    def collapse_close_vertices(self, path) -> bool:
        self._next_call()
        if len(path) < 3:
            return False
        max_steps = max_empty = len(path)
        pairs = [(i, j) for i in range(len(path)) for j in range(i + 2, len(path))]
        d = self.ops.distance(np.array([path[i] for i, _ in pairs]), np.array([path[j] for _, j in pairs]))
        dist = {(id(path[i]), id(path[j])): float(x) for (i, j), x in zip(pairs, d)}   # keyed by state identity:
        # a +inf mark survives erasures
        result, nochange, s = False, 0, 0
        while s < max_steps and nochange < max_empty:
            best, p1, p2 = INF, -1, -1
            for i in range(len(path)):
                for j in range(i + 2, len(path)):
                    d = dist[(id(path[i]), id(path[j]))]
                    if d < best:
                        best, p1, p2 = d, i, j
            if p1 < 0:
                break
            if self.check_motion(path[p1], path[p2]):
                del path[p1 + 1:p2]
                result = True
                nochange = 0
                self.stats["collapse"] += 1
            else:
                dist[(id(path[p1]), id(path[p2]))] = INF
            s += 1
            nochange += 1
        return result

    # -- PathSimplifier::shortcutPath(path, 0, 0, 0.33, 0.005) -----------------------------------------------------
    @staticmethod
    def _locate(dists, p, threshold):
        """lower_bound, then the snap to the next or the previous waypoint: (pos, index), index = -1 when interpolated."""
        n = len(dists)
        pos = next((k for k in range(n) if not dists[k] < p), n - 1)
        if pos == 0 or dists[pos] - p < threshold:
            return pos, pos
        while pos > 0 and p < dists[pos]:
            pos -= 1
        return pos, (pos if p - dists[pos] < threshold else -1)

    def shortcut_path(self, path) -> bool:
        call = self._next_call()
        if len(path) < 3:
            return False
        max_steps = max_empty = len(path)
        dists = [0.0]
        for x in self.ops.distance(np.array(path[:-1]), np.array(path[1:])).tolist():
            dists.append(dists[-1] + x)
        threshold = dists[-1] * SNAP_TO_VERTEX
        rd = RANGE_RATIO * dists[-1]
        sc = {"dists": dists, "threshold": threshold, "rd": rd}
        result, nochange, i = False, 0, 0
        while i < max_steps and nochange < max_empty:
            if self._shortcut_attempt(path, sc, call, i):
                result = True
                nochange = 0
            i += 1
            nochange += 1
        return result

    def _shortcut_attempt(self, path, sc, call: int, i: int) -> bool:
        """Attempt i of shortcutPath's loop; True when it changed the path (sc: dists, threshold, rd, updated)."""
        dists, threshold, rd = sc["dists"], sc["threshold"], sc["rd"]
        u0, u1 = self.variates(call, i)
        L = dists[-1]
        p0 = uniform_real(u0, 0.0, L)
        pos0, index0 = self._locate(dists, p0, threshold)
        p1 = uniform_real(u1, max(0.0, p0 - rd), min(p0 + rd, L))
        pos1, index1 = self._locate(dists, p1, threshold)
        # same or adjacent segments or waypoints. OMPL 1.4.2 tests only the first three; a point snapped to the waypoint
        # that ends the other point's segment then reaches an erase over a reversed range (undefined behaviour), and two
        # snapped neighbours an empty edit. The last three are the rule of later OMPL releases.
        if pos0 == pos1 or index0 == pos1 or index1 == pos0 or pos0 + 1 == index1 or pos1 + 1 == index0 or \
                (index0 >= 0 and index1 >= 0 and abs(index0 - index1) < 2):
            return False
        t0 = t1 = 0.0
        if index0 >= 0:
            s0 = path[index0]
        else:
            t0 = (p0 - dists[pos0]) / (dists[pos0 + 1] - dists[pos0])
            s0 = self._i(path[pos0], path[pos0 + 1], t0)
        if index1 >= 0:
            s1 = path[index1]
        else:
            t1 = (p1 - dists[pos1]) / (dists[pos1 + 1] - dists[pos1])
            s1 = self._i(path[pos1], path[pos1 + 1], t1)
        if not self.check_motion(s0, s1):
            return False
        if pos0 > pos1:
            pos0, pos1, index0, index1, s0, s1 = pos1, pos0, index1, index0, s1, s0
        along = 0.0 if index0 >= 0 else self._d(s0, path[pos0 + 1])
        if pos1 > pos0 + 1:
            for x in self.ops.distance(np.array(path[pos0 + 1:pos1]), np.array(path[pos0 + 2:pos1 + 1])).tolist():
                along += x
        along += 0.0 if index1 >= 0 else self._d(path[pos1], s1)
        if along < self._d(s0, s1):
            return False
        if index0 < 0 and index1 < 0:
            if pos0 + 1 == pos1:
                path[pos1] = np.array(s0)
                path.insert(pos0 + 2, np.array(s1))
            else:
                path[pos0 + 1] = np.array(s0)
                path[pos1] = np.array(s1)
                del path[pos0 + 2:pos1]
        elif index0 >= 0 and index1 >= 0:
            del path[index0 + 1:index1]
        elif index0 < 0:
            path[pos0 + 1] = np.array(s0)
            del path[pos0 + 2:index1]
        else:
            path[pos1] = np.array(s1)
            del path[index0 + 1:pos1]
        del dists[len(path):]
        while len(dists) < len(path):
            dists.append(0.0)
        tail = self.ops.distance(np.array(path[pos0:-1]), np.array(path[pos0 + 1:])).tolist()
        for j, x in zip(range(pos0 + 1, len(path)), tail):
            dists[j] = dists[j - 1] + x
        sc["threshold"] = dists[-1] * SNAP_TO_VERTEX
        sc["rd"] = RANGE_RATIO * dists[-1]
        self.stats["shortcut"] += 1
        return True

    # -- PathSimplifier::smoothBSpline(path, max_steps, min_change) ------------------------------------------------
    def smooth_bspline(self, path, max_steps: int, min_change: float) -> None:
        self._next_call()
        if len(path) < 3:
            return
        for _ in range(max_steps):
            path[:] = subdivide(path, self.ops)
            u, n1 = 0, len(path) - 1
            ev = list(range(2, n1, 2))    # every even i reads only odd states: m and its distance up front
            P = np.array(path)
            half = np.full(len(ev), 0.5)
            t1 = self.ops.interpolate(P[[i - 1 for i in ev]], P[ev], half)
            t2 = self.ops.interpolate(P[ev], P[[i + 1 for i in ev]], half)
            ms = self.ops.interpolate(t1, t2, half)
            moved = self.ops.distance(P[ev], ms)
            for i, m, dm in zip(ev, ms, moved.tolist()):
                if not self.is_valid(path[i - 1]):
                    continue
                if self.check_motion(path[i - 1], m) and self.check_motion(m, path[i + 1]):
                    if dm > min_change:
                        path[i] = m
                        u += 1
            self.stats["bspline"] += u
            if u == 0:
                break

    # -- PathGeometric::checkAndRepair, without the repair ---------------------------------------------------------
    def check_and_repair(self, path) -> bool:
        if len(path) < 2:
            return len(path) == 0 or self.is_valid(path[0])
        n1 = len(path) - 1
        if not self.is_valid(path[0]) or not self.is_valid(path[n1]):
            return False
        for i in range(1, n1):
            if not self.check_motion(path[i - 1], path[i]) or (i == n1 - 1 and not self.check_motion(path[i], path[i + 1])):
                return False
        return True

    # -- PathGeometric::check --------------------------------------------------------------------------------------
    def check(self, path) -> bool:
        if not path:
            return True
        if not self.is_valid(path[0]):
            return False
        for a, b in zip(path[:-1], path[1:]):
            if not self.check_motion(a, b):
                return False
        return True

    # -- PathSimplifier::simplifyMax -> simplify --------------------------------------------------------------------
    def simplify_max(self, path) -> bool:
        """The schedule on `path` in place; False when checkAndRepair's check fails (OMPL would then repair)."""
        if len(path) < 3:
            return True
        try_more = self.reduce_vertices(path)
        self.collapse_close_vertices(path)
        times = 0
        while try_more and times < REPEAT:
            times += 1
            try_more = self.reduce_vertices(path)
        times = 0
        while True:
            times += 1
            if not self.shortcut_path(path) or times >= REPEAT:
                break
        self.smooth_bspline(path, BSPLINE_STEPS, path_length(path, self.ops) / 100.0)
        return self.check_and_repair(path)


def get_solution_path(path, is_valid, space, seed: int, path_cost, variates=None, ops=Se3Ops):
    """Planner::getSolutionPath(true) (planner.cpp:266-298): simplifySolution, then path_simple.check(), then the strict
    cost comparison under path_cost(states [n, 7]) -> float (PathGeometric::cost of the planner's objective). A failing
    checkAndRepair returns the original (no repair). Returns (states [n, 7], info keyed like artp_simplify_info plus
    the number of schedule calls, the simplified path [m, 7])."""
    orig = [np.array(s, np.float64) for s in np.asarray(path, np.float64).reshape(-1, 7)]
    simp = list(orig)
    sim = Simplifier(is_valid, space, seed, variates, ops)
    repaired = sim.simplify_max(simp)
    n_simplified = len(simp)
    passed = repaired and sim.check(simp)
    cost_o = cost_s = float("nan")
    keep_orig = True
    if passed:
        cost_s = float(path_cost(np.array(simp).reshape(-1, 7)))
        cost_o = float(path_cost(np.array(orig).reshape(-1, 7)))
        keep_orig = cost_o < cost_s
    out = orig if keep_orig else simp
    st = sim.stats
    info = {"n_in": len(orig), "n_simplified": n_simplified, "n_out": len(out), "reduce_edits": st["reduce"],
            "collapse_edits": st["collapse"], "shortcut_edits": st["shortcut"], "bspline_edits": st["bspline"],
            "motion_checks": st["motions"], "state_checks": st["valids"], "check_passed": int(passed),
            "returned_simplified": int(not keep_orig), "cost_original": cost_o, "cost_simplified": cost_s,
            "calls": sim.call}
    return np.array(out).reshape(-1, 7), info, np.array(simp).reshape(-1, 7)
