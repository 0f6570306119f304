"""CPU checks of the start / goal search (StartState / GoalStateRegion::sampleGoal, start.cpp:7-41, goal.cpp:11-41): the
port oracle against the fixture the compiled reference wrote, and the numpy restatement of the offset stream."""
import os

import numpy as np
import pytest

import cases
import philox_ball_ref
import philox_ref
import start_goal_cases as sgc
import start_goal_oracle as sgo
from oracle.make_golden import digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sg_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "start_goal.npz"))


@pytest.mark.parametrize("name,mk,pk,n,n_iter,seed", sgc.GOLDEN_CASES, ids=[c[0] for c in sgc.GOLDEN_CASES])
def test_port_oracle_matches_reference_fixture(sg_golden, maps, port_lib, name, mk, pk, n, n_iter, seed):
    m = maps(mk)
    centres, radius, off = sgc.golden_inputs(m, n, n_iter, seed)
    assert str(sg_golden[name + "/sha"]) == digest(m.elevation, m.elevation_masked, centres, radius, off), "generator drift"
    o = port_lib.Oracle(cases.PARAMS[pk], "port")
    o.set_map(m)
    states, idx = sgo.find_valid_near(o, centres, n_iter, off)
    assert np.array_equal(idx, sg_golden[name + "/index"])
    assert np.array_equal(states.view(np.uint64), sg_golden[name + "/states"].view(np.uint64))


def test_fixture_covers_every_outcome(sg_golden, maps):
    idx = np.concatenate([sg_golden[c[0] + "/index"] for c in sgc.GOLDEN_CASES])
    assert (idx == 0).any() and ((idx > 0) & (idx <= 10)).any() and (idx > 100).any() and (idx < 0).any()
    # centres off the map and on its border are among the queries
    m = maps("fixture")
    centres, _ = sgc.make_queries(m, 60, 101)
    lx, ly = m.length
    assert (np.abs(centres[:, 0] - m.cx) > 0.5 * lx).any() and (np.abs(np.abs(centres[:, 1] - m.cy) - 0.5 * ly) < 0.3).any()


def test_oracle_loop_semantics(maps, port_lib):
    """Candidate k moves only x, y by offset k; none valid leaves candidate n_iter; n_iter = 0 leaves the centre."""
    m = maps("fbm_rough")
    o = port_lib.Oracle(cases.PARAMS["yaml"], "port")
    o.set_map(m)
    centres, radius, off = sgc.golden_inputs(m, 200, 50, 7)
    states, idx = sgo.find_valid_near(o, centres, 50, off)
    k = np.where(idx < 0, 50, idx)
    want = centres.copy()
    sel = k > 0
    want[sel, 0] = centres[sel, 0] + off[sel, k[sel] - 1, 0]
    want[sel, 1] = centres[sel, 1] + off[sel, k[sel] - 1, 1]
    assert np.array_equal(states, want)
    flags = o.check_poses(centres)
    assert np.array_equal(idx == 0, flags == 1)
    s0, i0 = sgo.find_valid_near(o, centres, 0, np.zeros((200, 0, 2)))
    assert np.array_equal(s0, centres) and np.array_equal(i0, np.where(flags == 1, 0, -1))


def test_ball_stream_restatement():
    """The words are Philox4x32-10 of (draw lo, draw hi, query, "ARTB") under the seed; offsets lie in the disc and are
    uniform over it (mean squared radius r^2 / 2, mean direction 0)."""
    seed = 0x0123456789ABCDEF
    w = philox_ball_ref.ball_words(seed, 2 ** 32 - 3, 3, 6)          # crosses the 32-bit word of the draw counter
    d = np.uint64(2 ** 32 - 3) + np.arange(6, dtype=np.uint64)
    for q in range(3):
        ctr = np.stack([(d & np.uint64(0xFFFFFFFF)).astype(np.uint32), (d >> np.uint64(32)).astype(np.uint32),
                        np.full(6, q, np.uint32), np.full(6, 0x41525442, np.uint32)], axis=1)
        assert np.array_equal(w[q], philox_ref.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32)))
    r = np.array([0.2, 0.5, 0.0, 3.0])
    off = philox_ball_ref.ball_offsets(5, 0, 4, 20000, r)
    rad = np.hypot(off[..., 0], off[..., 1])
    assert (rad <= r[:, None] * (1 + 1e-15)).all() and (off[2] == 0).all()
    assert np.allclose((rad[[0, 1, 3]] ** 2).mean(1), r[[0, 1, 3]] ** 2 / 2, rtol=0.03)
    assert np.abs(off[[0, 1, 3]].mean(1)).max() < 0.02 * r.max()
    # a different tag from the sampler's stream: the same key and counter words give other numbers
    assert not np.array_equal(philox_ball_ref.ball_words(5, 0, 1, 4)[0],
                              philox_ref.philox4x32_10(np.array([[k, 0, 0, philox_ref.TAG] for k in range(4)], np.uint32), (5, 0)))
