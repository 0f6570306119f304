"""GPU (-m gpu): artp_inpaint_layer[_device] against the golden layers made through cv2 and the restatement
(oracle/inpaint_oracle.py) bit for bit, including one interaction component far larger than any on-chip front; and
artp_planner_set_map_raw + artp_plan against artp_planner_set_map with artp_inpaint_layer's outputs + artp_plan, bit for
bit, with both networks and on a device another handle is planning on."""
import os
import threading

import numpy as np
import pytest

import inpaint_cases as ic
import planner_cases as pc
import roadmap_cases as rc
from art_planner_b200 import capi, costnet
from oracle import inpaint_oracle as io
from oracle import planner_oracle as po
from test_planner_gpu import make_pair, roadmap_dump, same, far_queries

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "inpaint.npz"))


@pytest.fixture(scope="module")
def chk():
    import art_planner_b200 as ap
    return ap.StateValidityChecker(rc.make_case("gentle_inf").rp)


@pytest.mark.parametrize("name", list(ic.CASES) + list(ic.LARGE_CASES))
def test_inpaint_layer_equals_golden(name, gold, chk):
    import torch
    a = gold[name + "/in"]
    want = bits(gold[name + "/out"])
    assert np.array_equal(bits(chk.inpaint(a)), want)
    d = torch.from_numpy(np.ascontiguousarray(a.T)).cuda().t()
    out = chk.inpaint(d)
    torch.cuda.synchronize()
    assert np.array_equal(bits(out.cpu().numpy()), want)


def test_inpaint_layer_equals_oracle_on_planner_maps(chk):
    for name in ("gentle_inf", "rough_fbm"):
        m = rc.make_case(name).m
        raw_e, raw_t, _, _ = pc.raw_layers(m, holes=0.02)
        for layer in (raw_e, raw_t):
            assert np.array_equal(bits(chk.inpaint(layer)), bits(io.inpaint_matrix(layer))), name


def test_inpaint_refusals(chk):
    with pytest.raises(capi.ArtpError):
        chk.inpaint(np.full((6, 5), np.nan, np.float32))
    with pytest.raises(capi.ArtpError):
        chk.inpaint(np.zeros((1, 5), np.float32))


def installed_state(chk, network):
    """What the installed map determines, read back directly: the cost network's feature map, 2048 draws of the armed
    sampler (its distribution, normals and bounds) and the validity of those states and of copies lifted by 5 cm (the
    uploaded map and its masked layer)."""
    import ctypes as C
    h = chk.handle
    hf, wf = C.c_int(), C.c_int()
    h.check(h.lib.artp_get_features(h.h, None, 0, C.byref(hf), C.byref(wf)))
    feat = np.empty((hf.value, wf.value, costnet.NETWORKS[network][0][5][2]), np.float32)
    h.check(h.lib.artp_get_features(h.h, feat.ctypes.data, feat.size, C.byref(hf), C.byref(wf)))
    n = 2048
    st = np.empty((n, 7))
    rowcol = np.empty((n, 2), np.int32)
    h.check(h.lib.artp_sample_states(h.h, None, 123, 0, n, st.ctypes.data, rowcol.ctypes.data))
    poses = np.concatenate([st, st + np.array([0, 0, 0.05, 0, 0, 0, 0])])
    valid = np.empty(2 * n, np.uint8)
    h.check(h.lib.artp_check_poses(h.h, np.ascontiguousarray(poses).ctypes.data, 2 * n, valid.ctypes.data))
    return feat, st, rowcol, valid


class RawPair:
    """Planner.setMapRaw on one handle; Planner.setMap with the device inpaint's layers on another."""

    def __init__(self, rp, pp, network="light", **kw):
        import art_planner_b200 as ap
        c1, c2 = make_pair(rp, network=network, **kw)
        self.raw, self.ref = ap.Planner(c1, pp), ap.Planner(c2, pp)
        self.c1, self.c2, self.network = c1, c2, network

    def set_map(self, raw_e, raw_t, m):
        ei = self.c2.inpaint(raw_e)
        ti = None if raw_t is None else self.c2.inpaint(raw_t)
        mi = self.raw.setMapRaw(raw_e, raw_t, m.res, m.cx, m.cy)
        self.ref.setMap(raw_e, raw_t, ei, ti, m.res, m.cx, m.cy)
        a, b = self.raw.space(), self.ref.space()
        assert list(a.low) == list(b.low) and list(a.high) == list(b.high)
        for x, y in zip(installed_state(self.c1, self.network), installed_state(self.c2, self.network)):
            assert np.array_equal(x, y)
        return mi

    def plan(self, s, g):
        st1, st2 = self.raw.plan(s, g), self.ref.plan(s, g)
        i1, i2 = self.raw.info(), self.ref.info()
        assert st1 == st2
        for k in i1:
            if not k.startswith("ms_"):
                assert same(i1[k], i2[k]) if not isinstance(i1[k], dict) else \
                    all(same(i1[k][q], i2[k][q]) for q in i1[k] if not q.startswith("ms_")), k
        if st1 == po.SOLVED:
            assert same(self.raw.getSolutionPath(), self.ref.getSolutionPath())
        for x, y in zip(roadmap_dump(self.raw._c.handle), roadmap_dump(self.ref._c.handle)):
            assert same(x, y)
        return st1


@pytest.mark.parametrize("network", ["light", "full"])
@pytest.mark.parametrize("name", ["gentle_inf", "rough_fbm"])
def test_set_map_raw_equals_set_map_with_inpainted_layers(name, network):
    c = rc.make_case(name)
    pair = RawPair(c.rp, pc.small_params(seed=77), network=network)
    raw_e, raw_t, _, _ = pc.raw_layers(c.m, holes=0.02)
    mi = pair.set_map(raw_e, raw_t, c.m)
    n = raw_e.size * 4
    assert mi["bytes_h2d"] >= 2 * n and mi["bytes_h2d"] < 3 * n   # two layers go up
    for s, g in far_queries(c.m, 3, seed=5, chk=pair.c2):
        pair.plan(s, g)


def test_set_map_raw_without_traversability():
    c = rc.make_case("gentle_inf")
    pair = RawPair(c.rp, pc.small_params(seed=3))
    raw_e, _, _, _ = pc.raw_layers(c.m, traversability=False, holes=0.02)
    mi = pair.set_map(raw_e, None, c.m)
    assert mi["bytes_h2d"] < 2 * raw_e.size * 4
    for s, g in far_queries(c.m, 2, seed=9, chk=pair.c2):
        pair.plan(s, g)


def test_set_map_raw_refuses_a_traversability_without_finite_cells():
    c = rc.make_case("gentle_inf")
    pair = RawPair(c.rp, pc.small_params(seed=3))
    raw_e, raw_t, _, _ = pc.raw_layers(c.m)
    with pytest.raises(capi.ArtpError):
        pair.raw.setMapRaw(raw_e, np.full_like(raw_t, np.nan), c.m.res, c.m.cx, c.m.cy)


def test_two_handles_one_inpainting_while_the_other_plans(gold):
    c = rc.make_case("gentle_inf")
    pp = pc.small_params(seed=77)
    import art_planner_b200 as ap
    c1, c2 = make_pair(c.rp)
    c3, _ = make_pair(c.rp)
    raw_e, raw_t, _, _ = pc.raw_layers(c.m, holes=0.02)
    ref = ap.Planner(c2, pp)
    ref.setMap(raw_e, raw_t, c2.inpaint(raw_e), c2.inpaint(raw_t), c.m.res, c.m.cx, c.m.cy)
    q = far_queries(c.m, 2, seed=5, chk=c2)
    alone = ap.Planner(c3, pp)
    alone.setMapRaw(raw_e, raw_t, c.m.res, c.m.cx, c.m.cy)
    want = [(alone.plan(*x), alone.info()["n_vertices"]) for x in q]
    a, w = gold["giant/in"], bits(gold["giant/out"])
    errs = []

    def inpaint_loop():
        try:
            for _ in range(3):
                assert np.array_equal(bits(c2.inpaint(a)), w)
        except Exception as e:   # noqa: BLE001
            errs.append(e)
    planner = ap.Planner(c1, pp)
    th = threading.Thread(target=inpaint_loop)
    th.start()
    planner.setMapRaw(raw_e, raw_t, c.m.res, c.m.cx, c.m.cy)
    got = [(planner.plan(*x), planner.info()["n_vertices"]) for x in q]
    th.join()
    assert not errs, errs
    assert got == want
