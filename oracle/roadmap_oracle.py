"""Restatement of PRMMotionCost's roadmap construction (TEST INFRASTRUCTURE ONLY), brute force, on the CPU:

  addValidMilestone   art_planner/src/planners/prm_motion_cost.cpp:325-390
  sampleGraph's loop  prm_motion_cost.cpp:171-194, with a draw budget in place of max_sample_time (:177-184)

and of the OMPL 1.4.2 pieces they call, which are not in the tree (restated, unpinned):
  KStarStrategy              ConnectionStrategy.h: k = ceil((e + e / d) * log(milestoneCount())), d = 6 for SE(3)
  LazyPRM::milestoneCount    num_vertices(g_), which counts the new milestone (add_vertex comes first, :326)
  GNAT nearestK              exact, ascending distance; exact ties (left unspecified by GNAT) go to the lower vertex index
  SE3StateSpace::distance    R^3 Euclidean + acos(|q1.q2|) (0 above 1 - 1e-9)
  SE3StateSpace::interpolate R^3 lerp + SO3 slerp
  LazyPRM::getPlannerData    start / goal milestones plus the endpoints of edges: the density's vertices

Validity comes from an orc.Oracle (port restatement or the compiled reference), candidates from orc.sample_states over
tests/philox_ref.py's stream, the distribution recompute from oracle/sample_distribution_oracle.py.
"""
from __future__ import annotations

import copy
import math

import numpy as np

from oracle import orc
from oracle import sample_distribution_oracle as sdo

E = 2.718281828459045            # boost::math::constants::e<double>()
K_STAR = E + E / 6.0             # kPRMConstant_ for SE3StateSpace::getDimension() == 6
MAX_LATERAL = 0.5                # kMaxDist, prm_motion_cost.cpp:342
MILESTONE, INTERPOLATED, QUERY = 1, 2, 4


def k_star(V: int) -> int:
    return 0 if V == 0 else int(math.ceil(K_STAR * math.log(V)))


def se3_distance(a, S):
    """SE3StateSpace::distance from state a to every row of S."""
    r = np.zeros(S.shape[0])
    for i in range(3):
        d = a[i] - S[:, i]
        r = r + d * d
    dq = np.abs(a[3] * S[:, 3] + a[4] * S[:, 4] + a[5] * S[:, 5] + a[6] * S[:, 6])
    with np.errstate(invalid="ignore"):
        so3 = np.where(dq > 1.0 - 1e-9, 0.0, np.arccos(np.minimum(dq, 1.0)))
    return np.sqrt(r) + so3


def nearest(a, S, k: int):
    """The k nearest rows of S in ascending (distance, index)."""
    if k == 0 or S.shape[0] == 0:
        return np.zeros(0, np.int64)
    d = se3_distance(a, S)
    return np.lexsort((np.arange(S.shape[0]), d))[:k]


def interpolate(a, b, t: float):
    """SE3StateSpace::interpolate(a, b, t) (libm, scalar)."""
    out = np.empty(7)
    for i in range(3):
        out[i] = a[i] + (b[i] - a[i]) * t
    dq = a[3] * b[3] + a[4] * b[4] + a[5] * b[5] + a[6] * b[6]
    dqa = abs(dq)
    theta = 0.0 if dqa > 1.0 - 1e-9 else math.acos(dqa)
    if theta > 2.220446049250313e-16:
        d = 1.0 / math.sin(theta)
        s0 = math.sin((1.0 - t) * theta)
        s1 = math.sin(t * theta)
        if dq < 0:
            s1 = -s1
        for i in range(3, 7):
            out[i] = (a[i] * s0 + b[i] * s1) * d
    else:
        out[3:] = a[3:]
    return out


class Roadmap:
    """The Boost graph g_ as arrays in insertion order: states, kinds, edges (u, v), and the density flags."""

    def __init__(self, capacity: int = 1 << 16):
        self.states = np.zeros((capacity, 7))
        self.kinds = np.zeros(capacity, np.uint8)
        self.dens = np.zeros(capacity, bool)
        self.V = 0
        self.edges = []

    @property
    def E(self) -> int:
        return len(self.edges)

    def _vertex(self, s, kind: int) -> int:
        if self.V == self.states.shape[0]:
            grow = self.states.shape[0]
            self.states = np.concatenate([self.states, np.zeros((grow, 7))])
            self.kinds = np.concatenate([self.kinds, np.zeros(grow, np.uint8)])
            self.dens = np.concatenate([self.dens, np.zeros(grow, bool)])
        v = self.V
        self.states[v] = s
        self.kinds[v] = kind
        self.V += 1
        return v

    def _edge(self, a: int, b: int) -> None:
        self.edges.append((a, b))
        self.dens[a] = self.dens[b] = True

    def add_milestone(self, s, is_valid, kind: int = MILESTONE) -> int:
        """addValidMilestone (:325-390); is_valid(states [n, 7]) -> bool [n]."""
        s = np.asarray(s, np.float64)
        V = self.V
        nbrs = nearest(s, self.states[:V], min(k_star(V + 1), V))
        S = self.states[:V].copy()
        m = self._vertex(s, kind)
        if kind & QUERY:
            self.dens[m] = True
        plan, interior = [], []
        for n in nbrs:
            dx, dy = S[n, 0] - s[0], S[n, 1] - s[1]
            ni = int(math.sqrt(dx * dx + dy * dy) / MAX_LATERAL)
            div = 1.0 / (ni + 1)
            states = [interpolate(s, S[n], step * div) for step in range(1, ni + 1)]
            plan.append((int(n), ni, len(interior)))
            interior.extend(states)
        valid = np.asarray(is_valid(np.array(interior).reshape(-1, 7)), bool) if interior else np.zeros(0, bool)
        for n, ni, o in plan:
            if ni == 0:
                self._edge(m, n)
                continue
            prev = m
            p = 0
            while p < ni and valid[o + p]:
                v = self._vertex(interior[o + p], INTERPOLATED)
                self._edge(prev, v)
                prev = v
                p += 1
            if p == ni:
                self._edge(prev, n)
        return m

    def density_states(self):
        """The vertices LazyPRM::getPlannerData returns (order irrelevant for the histogram)."""
        return self.states[:self.V][self.dens[:self.V]]

    def result(self):
        return self.states[:self.V].copy(), self.kinds[:self.V].copy(), np.array(self.edges, np.uint32).reshape(-1, 2)


def validity(oracle: orc.Oracle):
    return lambda states: oracle.check_poses(states).astype(bool)


def sample_graph(rm: Roadmap, oracle: orc.Oracle, m, layers, sp, reach_z: float, seed: int, first_sample: int,
                 max_n_vertices: int, max_n_edges: int, recompute_n: int, max_draws: int, dp=None, sample_filter=None,
                 observed=None, chunk: int = 4096, is_valid=None, max_milestones=None):
    """sampleGraph's loop (:171-194), or its first max_milestones milestones. Returns (draws used, draw index of every milestone, V at every recompute); the
    sampler's layers as the loop leaves them (after its last recompute) go to rm.layers."""
    is_valid = is_valid or validity(oracle)
    layers = copy.copy(layers)
    end = first_sample + max_draws
    draw, n_proc = first_sample, 0
    milestones, recomputes = [], []
    cache = (None, None, None)                         # first draw, states, verdicts of the current chunk
    while rm.V < max_n_vertices and rm.E < max_n_edges and (max_milestones is None or len(milestones) < max_milestones):
        found = None
        while draw < end:
            c0, cs, cv = cache
            if c0 is None or not (c0 <= draw < c0 + len(cs)):
                n = min(chunk, end - draw)
                u = sdo_uniforms(seed, draw, n)
                cs, _ = orc.sample_states(m, layers, sp, reach_z, u)
                cv = np.zeros(n, bool)
                ok = ~np.isnan(cs[:, 0])
                if ok.any():
                    cv[ok] = is_valid(cs[ok])
                cache = c0, cs, cv = draw, cs, cv
            hit = np.flatnonzero(cv[draw - c0:])
            if hit.size:
                found = draw + int(hit[0])
                break
            draw = c0 + len(cs)
        if found is None:
            draw = end
            break
        rm.add_milestone(cache[1][found - cache[0]], is_valid)
        milestones.append(found)
        draw = found + 1
        if dp is not None and recompute_n and rm.V // recompute_n > n_proc:   # :190-193
            ref = sdo.distribution(rm.density_states(), m, dp, sample_filter, observed)
            layers = copy.copy(layers)
            layers.cum_prob, layers.cum_prob_rowwise = ref["cum_prob"], ref["cum_prob_rowwise"]
            cache = (None, None, None)
            recomputes.append(rm.V)
            n_proc += 1
    rm.layers = layers
    return draw - first_sample, np.array(milestones, np.int64), np.array(recomputes, np.int64)


def sdo_uniforms(seed: int, first: int, n: int):
    import philox_ref   # tests/ is on sys.path under pytest and in the golden script
    return philox_ref.sampler_uniforms(seed, first, n)
