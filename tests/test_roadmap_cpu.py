"""CPU checks of the roadmap restatement (oracle/roadmap_oracle.py) and of the roadmap's C ABI symbols."""
import math
import os
import re

import numpy as np
import pytest

import roadmap_cases as rc
from oracle import roadmap_oracle as ro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_k_star_table():
    assert ro.K_STAR == math.e + math.e / 6
    assert [ro.k_star(v) for v in (0, 1, 2, 3, 10, 1000, 10000)] == [0, 0, 3, 4, 8, 22, 30]
    # past V = 2, k grows by at most 1 from one V to the next and never shrinks
    k = np.array([ro.k_star(v) for v in range(2, 60001)])
    assert (np.diff(k) >= 0).all() and (np.diff(k) <= 1).all()


def test_distance_formula():
    rng = np.random.default_rng(3)
    a = np.r_[rng.normal(size=3), rng.normal(size=4)]
    a[3:] /= np.linalg.norm(a[3:])
    S = np.c_[rng.normal(size=(50, 3)), rng.normal(size=(50, 4))]
    S[:, 3:] /= np.linalg.norm(S[:, 3:], axis=1, keepdims=True)
    d = ro.se3_distance(a, S)
    want = np.linalg.norm(S[:, :3] - a[:3], axis=1) + np.arccos(np.minimum(np.abs(S[:, 3:] @ a[3:]), 1.0))
    assert np.allclose(d, want, rtol=0, atol=1e-12)
    # |q1.q2| above 1 - 1e-9 counts as no rotation; q and -q are the same rotation
    b = a.copy(); b[3:] = -a[3:]
    assert ro.se3_distance(a, b[None])[0] == 0.0


def test_ties_go_to_the_lower_index():
    a = np.array([0, 0, 0, 0, 0, 0, 1.0])
    S = np.zeros((6, 7)); S[:, 6] = 1.0
    S[:, 0] = [2.0, 1.0, -1.0, 1.0, 0.5, -0.5]
    assert list(ro.nearest(a, S, 5)) == [4, 5, 1, 2, 3]


def test_isolated_milestones_are_not_in_the_density():
    rm = ro.Roadmap()
    far = np.array([0, 0, 0, 0, 0, 0, 1.0])
    rm.add_milestone(far, lambda s: np.ones(len(s), bool))                       # V = 1: k = 0, no edge
    assert rm.density_states().shape == (0, 7)
    rm.add_milestone(far + [0.3, 0, 0, 0, 0, 0, 0], lambda s: np.ones(len(s), bool))   # k = 3 > V: connects to vertex 0
    assert rm.E == 1 and rm.density_states().shape == (2, 7)
    q = far + [50.0, 0, 0, 0, 0, 0, 0]
    rm.add_milestone(q, lambda s: np.zeros(len(s), bool), ro.MILESTONE | ro.QUERY)   # every connection blocked
    assert rm.E == 1
    assert rm.dens[2]                                                               # a query milestone always counts


def test_connection_prefix_and_final_edge():
    rm = ro.Roadmap()
    ok = lambda s: np.ones(len(s), bool)
    rm.add_milestone(np.array([0, 0, 0, 0, 0, 0, 1.0]), ok)
    # 1.2 m away: n_interp = 2 interior states; the second is invalid -> one interpolated vertex, no final edge
    calls = []
    def second_bad(s):
        calls.append(len(s))
        v = np.ones(len(s), bool); v[1] = False
        return v
    rm.add_milestone(np.array([1.2, 0, 0, 0, 0, 0, 1.0]), second_bad)
    st, kinds, edges = rm.result()
    assert calls == [2] and list(kinds) == [1, 1, 2] and edges.tolist() == [[1, 2]]
    assert np.allclose(st[2, :3], [0.8, 0, 0])
    # all valid: chain m -> i1 -> i2 -> n
    rm2 = ro.Roadmap()
    rm2.add_milestone(np.array([0, 0, 0, 0, 0, 0, 1.0]), ok)
    rm2.add_milestone(np.array([1.2, 0, 0, 0, 0, 0, 1.0]), ok)
    assert rm2.result()[2].tolist() == [[1, 2], [2, 3], [3, 0]]


def test_recompute_counter_and_caps_before_each_milestone(monkeypatch):
    """n_proc grows by one per milestone even when V jumps over two multiples (:190-193); the caps are checked before
    each milestone (:171-172), so the last milestone may overshoot them."""
    calls = []
    monkeypatch.setattr(ro.sdo, "distribution", lambda v, *a, **k: calls.append(len(v)) or
                        {"cum_prob": None, "cum_prob_rowwise": None})
    states = [np.array([x, 0, 0, 0, 0, 0, 1.0]) for x in (0.0, 2.6, 5.2, 7.8)]

    class Fake:
        pass
    monkeypatch.setattr(ro.orc, "sample_states", lambda m, L, sp, rz, u: (np.array(states * (len(u) // 4 + 1))[:len(u)], None))
    rm = ro.Roadmap()
    used, draws, rec = ro.sample_graph(rm, Fake(), None, Fake(), None, 0.0, 0, 0, 9, 10 ** 6, 2, 100,
                                       dp=object(), is_valid=lambda s: np.ones(len(s), bool))
    # V after each milestone: 1, 7 and 23 (interior states towards the earlier milestones): 7 // 2 = 3 and 23 // 2 = 11 jump
    # over several multiples, yet each milestone recomputes once; then V >= 9 ends the loop
    assert len(draws) == 3 and list(rec) == [7, 23] and len(calls) == 2
    assert rm.V == 23 and used == draws[-1] + 1


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "roadmap.npz"))


@pytest.mark.parametrize("name", rc.GOLDEN_CASES)
def test_restatement_matches_reference_golden(name, golden):
    """The restatement over the port oracle rebuilds the golden the compiled reference's ODE answered."""
    from oracle import orc
    c = rc.make_case(name)
    o = orc.Oracle(c.rp, "port")
    o.set_map(c.m)
    rm = ro.Roadmap()
    used, draws, rec = ro.sample_graph(rm, o, c.m, c.layers, c.sp, c.rp.reach_z, rc.SEED, 0, *rc.CAPS, rc.MAX_DRAWS, c.dp,
                                       c.sample_filter, c.observed)
    st, kinds, edges = rm.result()
    assert np.array_equal(kinds, golden[name + "/kinds"]) and np.array_equal(edges, golden[name + "/edges"])
    assert np.array_equal(draws, golden[name + "/draws"]) and np.array_equal(rec, golden[name + "/recompute_v"])
    assert used == golden[name + "/draws_used"][0]
    assert np.abs(st - golden[name + "/states"]).max() <= 1e-12
    assert (kinds == ro.INTERPOLATED).any() and len(rec) >= 3


def test_abi_symbols():
    hdr = open(os.path.join(ROOT, "include", "artp.h")).read()
    names = ("artp_roadmap_clear", "artp_roadmap_add_milestones", "artp_roadmap_sample_graph", "artp_roadmap_get")
    for name in names:
        assert re.search(r"\bint " + name + r"\(", hdr)
    from art_planner_b200 import capi
    if os.path.exists(capi.LIB_PATH):                        # the library exports them (no device needed to load it)
        lib = capi.load()
        assert all(hasattr(lib, n) for n in names)
    for n in ("ARTP_ROADMAP_MILESTONE     1", "ARTP_ROADMAP_INTERPOLATED  2", "ARTP_ROADMAP_QUERY         4"):
        assert n in hdr
