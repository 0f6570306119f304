"""CPU checks of the box verdicts' definition (artp_box_verdicts): the per-box composition of oracle/box_verdict_oracle.py
over the port library's collider against the fixture the compiled reference wrote, the words against isValid and its
short-circuit (finite and non-finite states), and the ctypes mirror against include/artp.h."""
import os
import re

import numpy as np
import pytest

import box_verdict_cases as bvc
import cases
from oracle import box_verdict_oracle as bvo
from oracle.make_golden import digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def bv_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "box_verdicts.npz"))


@pytest.mark.parametrize("mk", sorted(cases.MAPS))
def test_port_oracle_matches_reference_fixture(bv_golden, port_lib, mk):
    m = cases.MAPS[mk]()
    states = bvc.samples(m)
    for name, mk2, pk, u in bvc.CASES:
        if mk2 != mk:
            continue
        assert str(bv_golden[name + "/sha"]) == digest(m.elevation, m.elevation_masked), "generator drift"
        p = bvc.params(pk, u)
        o = port_lib.Oracle(p, "port")
        o.set_map(m)
        why = bvo.box_verdicts(o, p, m, states)
        want = bv_golden[name + "/why"]
        assert why.dtype == want.dtype == np.uint16 and np.array_equal(why, want), name


@pytest.mark.parametrize("mk", sorted(cases.MAPS))
def test_words_agree_with_is_valid_and_its_short_circuit(bv_golden, port_lib, mk):
    """(word & 0x1F) == 0 exactly where isValid holds; the lowest fail bit is the box where isValid's && chain stops: the
    torso, else the first reach box in order -- which is the one box whose verdict alone decides the state, so making
    every box before it pass leaves the state invalid (checked by the port's single-box collider)."""
    m = cases.MAPS[mk]()
    states = bvc.samples(m)
    for name, mk2, pk, u in bvc.CASES:
        if mk2 != mk:
            continue
        why = bv_golden[name + "/why"]
        o = port_lib.Oracle(bvc.params(pk, u), "port")
        o.set_map(m)
        valid = o.check_poses(states)
        assert np.array_equal((why & 0x1F) == 0, valid != 0), name
        assert not (why & 0xE0E0).any(), name                             # no bit outside 0-4 and 8-12
        torso_out = (why >> 8) & 1
        assert not (torso_out & why & 1).any(), name                       # an off-map torso never fails
        feet_out = (why >> 9) & 0xF
        feet_fail = (why >> 1) & 0xF
        if u:
            assert np.array_equal(feet_out & feet_fail, feet_out), name    # off the map fails a reach box
        else:
            assert not (feet_out & feet_fail).any(), name                  # ... and only then
        # isValid's verdict from the words in its own order: the torso first, the reach boxes after it
        stop = bvc.lowest_fail(why)
        assert np.array_equal(stop == -1, valid != 0)


@pytest.mark.parametrize("u", [1, 0])
def test_non_finite_and_off_map_states(port_lib, u):
    """The composition places and decides boxes of non-finite states as orc_state_valid does: its words agree with
    check_poses there too. A state far off the map has every box off it."""
    m = cases.MAPS["fixture"]()
    s = bvc.samples(m, seed=9)[:128].copy()
    s[0:64:4, 0] = np.nan
    s[1:64:4, 3:] = np.nan
    s[2:64:4, 2] = np.inf
    s[3:64:4, 1] = -np.inf
    s[64:, 0] += 50.0
    p = bvc.params("yaml", u)
    o = port_lib.Oracle(p, "port")
    o.set_map(m)
    why = bvo.box_verdicts(o, p, m, s)
    assert np.array_equal((why & 0x1F) == 0, o.check_poses(s) != 0)
    assert np.all(why[64:] >> 8 == 0x1F) and np.all((why[64:] & 0x1F) == (0x1E if u else 0))


def test_fixture_covers_the_no_short_circuit_bits(bv_golden):
    """Every case has states where the torso and reach boxes fail together, states where several reach boxes fail,
    off-map boxes of each kind and valid states, so that the bits past the first failing box are pinned."""
    for name, _, _, u in bvc.CASES:
        why = bv_golden[name + "/why"]
        fails = (why & 0x1F)
        assert ((fails & 1) & (fails >> 1 != 0)).any(), name              # torso and a reach box
        assert (np.bitwise_count(fails >> 1) >= 2).any(), name             # two or more reach boxes
        assert (why & 0x100).any() and (why & 0x1E00).any(), name         # the torso off the map; a reach box off it
        assert (fails == 0).any() and (fails != 0).any(), name
        for k in range(1, 5):
            assert (fails == (1 << k)).any(), (name, k)                    # each reach box failing alone
    for name in [c[0] for c in bvc.CASES if c[1] in ("fbm_hard", "spikes")]:
        assert ((bv_golden[name + "/why"] & 0x1F) == 1).any(), name         # the torso failing alone


def test_ctypes_mirror_matches_the_header():
    from art_planner_b200 import capi
    h = open(os.path.join(ROOT, "include", "artp.h")).read()
    defs = dict(re.findall(r"#define (ARTP_BOX_\w+)\s+(0x[0-9A-Fa-f]+|\d+)u?\b", h))
    for name in ("ARTP_BOX_TORSO", "ARTP_BOX_FOOT_PP", "ARTP_BOX_FOOT_PM", "ARTP_BOX_FOOT_MP", "ARTP_BOX_FOOT_MM",
                 "ARTP_BOX_FAIL_MASK", "ARTP_BOX_OUTSIDE_MASK"):
        assert getattr(capi, name) == int(defs[name], 0), name
    assert "#define ARTP_BOX_FAILS(k)     (1u << (k))" in h and "#define ARTP_BOX_OUTSIDE(k)   (1u << (8 + (k)))" in h
    for k in range(5):
        assert capi.ARTP_BOX_FAILS(k) == 1 << k and capi.ARTP_BOX_OUTSIDE(k) == 1 << (8 + k)
        assert capi.ARTP_BOX_FAIL_MASK & capi.ARTP_BOX_FAILS(k) and capi.ARTP_BOX_OUTSIDE_MASK & capi.ARTP_BOX_OUTSIDE(k)
    protos = {
        "artp_box_verdicts": "artp_handle* h, const double* states, size_t n, uint16_t* why",
        "artp_box_verdicts_device": "artp_handle* h, const double* d_states, size_t n, uint16_t* d_why, void* stream",
        "artp_box_verdict_layer": "artp_handle* h, double yaw, uint16_t* out",
        "artp_box_verdict_layer_device": "artp_handle* h, double yaw, uint16_t* d_out, void* stream",
    }
    for fn, args in protos.items():
        assert f"int {fn}({args});" in h, fn
    src = open(os.path.join(ROOT, "art_planner_b200", "capi.py")).read()
    assert "lib.artp_box_verdicts.argtypes = [vp, vp, sz, vp]" in src
    assert "lib.artp_box_verdicts_device.argtypes = [vp, vp, sz, vp, vp]" in src
    assert "lib.artp_box_verdict_layer.argtypes = [vp, C.c_double, vp]" in src
    assert "lib.artp_box_verdict_layer_device.argtypes = [vp, C.c_double, vp, vp]" in src
