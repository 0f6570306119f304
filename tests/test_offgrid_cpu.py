"""CPU-only: the oracle restatement (oracle/artp_oracle.c) on the off-grid geometries of offgrid_cases.py against the
golden verdicts of the reference's own compiled ODE (oracle/make_golden_offgrid.py), the library's host segment count
against the same golden, and the classify-path coverage of that matrix restated in numpy."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import cases
import offgrid_cases as oc
from art_planner_b200 import capi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def unpack(g, key, n):
    return np.unpackbits(g[key])[:n]


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "reference_offgrid.npz"))


@pytest.fixture(scope="module")
def omaps():
    cache = {}

    def get(mk):
        if mk not in cache:
            cache[mk] = oc.MAPS[mk]()
        return cache[mk]
    return get


def test_geometry_matrix_reaches_the_intended_shapes(omaps):
    """The shapes the matrix exists for: every rows mod 4, non-square, off-origin, the resolutions and the pitch-4 maps."""
    shapes = {mk: (omaps(mk).rows, omaps(mk).cols, omaps(mk).res, omaps(mk).cx, omaps(mk).cy) for mk in oc.MAPS}
    assert {r % 4 for r, *_ in shapes.values()} == {0, 1, 2, 3}
    assert all(r != c for r, c, *_ in shapes.values())
    assert {res for _, _, res, *_ in shapes.values()} >= {0.025, 0.04, 0.1, 0.2}
    assert sum(1 for *_, cx, cy in shapes.values() if cx != 0 and cy != 0) >= 3
    assert (omaps("thin_r").rows + 3) & ~3 == 4 and omaps("thin_c").cols == 2
    assert float(omaps("far").elevation.max()) < -38.0


@pytest.mark.parametrize("case", oc.POSE_CASES, ids=[c[0] for c in oc.POSE_CASES])
def test_port_pose_masks_match_reference_golden(case, gold, omaps, port_lib):
    name, mk, pk, seed = case
    m = omaps(mk)
    poses = oc.case_poses(m, mk, seed)
    assert digest(m.elevation, m.elevation_masked, poses) == str(gold[name + "/sha"]), "generator drift"
    o = port_lib.Oracle(oc.PARAMS[pk], "port")
    o.set_map(m)
    v = o.check_poses(poses)
    assert np.array_equal(v, unpack(gold, name + "/mask", len(v)))
    if mk in oc.MIXED:
        assert 0.05 < v.mean() < 0.95, v.mean()
    elif mk.startswith("tiny"):
        assert v.any()


@pytest.mark.parametrize("case", oc.BOX_CASES, ids=[c[0] for c in oc.BOX_CASES])
def test_port_box_hits_match_reference_golden(case, gold, omaps, port_lib):
    mk, seed, tilt, zr = case
    m = omaps(mk)
    o = port_lib.Oracle(oc.PARAMS["yaml"], "port")
    o.set_map(m)
    for which in (0, 1):
        org, rot = cases.box_samples(m, oc.BOX_N, seed, which, tilt, zr)
        assert digest(m.elevation, m.elevation_masked, org, rot) == str(gold[f"box_{mk}/{which}/sha"])
        hit = o.box_collide(which, org, rot)
        assert np.array_equal(hit, unpack(gold, f"box_{mk}/{which}/mask", len(hit)))
        assert 0 < hit.sum() < len(hit)


@pytest.mark.parametrize("mk", oc.EDGE_MAPS)
def test_port_edges_match_reference_golden(mk, gold, omaps, port_lib):
    m = omaps(mk)
    o = port_lib.Oracle(oc.PARAMS["yaml"], "port")
    o.set_map(m)
    n, steps, seed = oc.EDGES
    s1, s2 = synth.make_edges(m, n, seed)
    assert digest(m.elevation, m.elevation_masked, s1, s2) == str(gold[f"edges_{mk}/sha"])
    v = o.check_motions(s1, s2, steps)
    assert np.array_equal(v, unpack(gold, f"edges_{mk}/mask", n)) and v.any()
    n, seed, dmin, dmax = oc.INTERIORS
    s1, s2 = synth.make_edges(m, n, seed, dmin=dmin, dmax=dmax)
    assert digest(m.elevation, m.elevation_masked, s1, s2) == str(gold[f"interior_{mk}/sha"])
    k = o.check_edge_interiors(s1, s2, None, 0.5)
    assert np.array_equal(k, gold[f"interior_{mk}/prefix"].astype(np.int32)) and (k > 0).any()
    n, seed, dmin, dmax = oc.SEGMENTS
    s1, s2 = synth.make_edges(m, n, seed, dmin=dmin, dmax=dmax)
    assert digest(m.elevation, m.elevation_masked, s1, s2) == str(gold[f"segments_{mk}/sha"])
    low, high = oc.se3_bounds(m, oc.PARAMS["yaml"].reach_z)
    nd = o.valid_segment_count(low, high, s1, s2)
    assert np.array_equal(nd, gold[f"segments_{mk}/nd"])
    # the library's host count (no handle, no device) gives the same nd
    space = capi.ArtpSe3Space((C.c_double * 3)(*low), (C.c_double * 3)(*high), 0.01)
    a, b = np.ascontiguousarray(s1, np.float64), np.ascontiguousarray(s2, np.float64)
    lib_nd = np.empty(n, np.int32)
    assert capi.load().artp_valid_segment_count(C.byref(space), a.ctypes.data, b.ctypes.data, n, lib_nd.ctypes.data) == capi.ARTP_OK
    assert np.array_equal(lib_nd, gold[f"segments_{mk}/nd"])
    sv, t = o.check_motions_segments(s1, s2, nd)
    assert np.array_equal(sv, unpack(gold, f"segments_{mk}/mask", n)) and np.array_equal(t, gold[f"segments_{mk}/last_t"])


def test_classify_paths_are_all_reached(omaps):
    """Across the matrix, the classify stage's zone reduction takes the one-request 8-word path, the window loop
    (cx * cz > 8) and the exact reduction for cx * cz > 32 (the long 'rail' torso) at least 100 times each.

    The other two causes of REC_NEEDS_REDUCE cannot occur for a map the handle accepts, and the matrix confirms it:
    kk < 1 needs a zone one vertex wide, but floor / ceil of the AABB's two faces always span two vertices (and a zone
    clipped to one vertex needs a face exactly on the map's last vertex); kk > kmax needs a zone wider than the
    half-diagonal bound kmax is derived from, or kmax capped at level 6, which needs 128 x 128-vertex zones that the
    plane store (200 KB) rejects long before. They stay as guards."""
    tot = dict.fromkeys(("words8", "loop", "kk<1", "kk>kmax", "cxcz>32"), 0)
    for name, mk, pk, seed in oc.POSE_CASES:
        m = omaps(mk)
        for k, v in oc.zone_paths(m, oc.PARAMS[pk], oc.case_poses(m, mk, seed)).items():
            tot[k] += v
    assert tot["words8"] >= 100 and tot["loop"] >= 100 and tot["cxcz>32"] >= 100, tot
    assert tot["kk<1"] == 0 and tot["kk>kmax"] == 0, tot


def test_table_levels_span_the_range(omaps):
    """kmax as artp_set_map_window derives it: from 1 (two-vertex maps) to the cap of 6 (yaml torso at 0.025 m)."""
    km = {(mk, pk): tuple(oc.table_kmax(omaps(mk), oc.PARAMS[pk])) for _, mk, pk, _ in oc.POSE_CASES}
    assert km[("thin_r", "yaml")] == (1, 1) and km[("fine", "yaml")][0] == oc.K_MAX_LEVEL
    assert len({k[0] for k in km.values()}) >= 5
