"""GPU parity (-m gpu) on the off-grid geometries of offgrid_cases.py: rows = 1, 2, 3 mod 4 (pad columns in every layer,
range table and TMA tile), non-square maps, 0.025 to 0.2 m cells (other table levels, classify paths and tile
configurations), centres far from the origin (the map position in the float box frame, the sampler, the normals and the
goal projection) and maps smaller than the robot or two vertices wide. Every verdict must equal the compiled reference's
golden (oracle/make_golden_offgrid.py) and the port oracle, bit for bit."""
import os

import numpy as np
import pytest

import offgrid_cases as oc
import philox_ball_ref
import philox_ref
import start_goal_cases as sgc
import start_goal_oracle as sgo
from art_planner_b200 import capi, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATE_TOL = 1e-12      # CUDA vs libm / numpy sin, cos, acos, atan2 in double states; cells and verdicts are exact
LAYER_MAPS = ("r3", "r1", "far", "coarse")
FBM = ("r3", "r1", "far", "coarse", "coarser", "fine")


def unpack(g, key, n):
    return np.unpackbits(g[key])[:n]


def same_bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


@pytest.fixture(scope="module")
def ap():
    import art_planner_b200
    from art_planner_b200 import build
    build.build()
    return art_planner_b200


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


def checker(ap, m, pk="yaml", window=None):
    chk = ap.StateValidityChecker(oc.PARAMS[pk], device=0)
    chk.setMap(m)
    chk.updateHeightField(window=window)
    return chk


def oracle(port_lib, m, pk="yaml"):
    o = port_lib.Oracle(oc.PARAMS[pk], "port")
    o.set_map(m)
    return o


@pytest.mark.parametrize("case", oc.POSE_CASES, ids=[c[0] for c in oc.POSE_CASES])
def test_pose_masks_bit_exact(ap, case, gold, omaps, port_lib):
    """Both routes (mode 0, mode 1 = every in-map box through the grouping stage), double and float states, host and
    device buffers, and the single-state latency path; the default route's queues must have run."""
    import torch
    name, mk, pk, seed = case
    m = omaps(mk)
    poses = oc.case_poses(m, mk, seed)
    ref = unpack(gold, name + "/mask", len(poses))
    assert np.array_equal(oracle(port_lib, m, pk).check_poses(poses), ref)
    chk = checker(ap, m, pk)
    got = chk.isValidBatch(poses)
    st = chk.stats()
    bad = np.nonzero(got != ref)[0]
    assert bad.size == 0, f"{bad.size} mismatches, first {bad[:8]}, stats {st}"
    if mk in FBM:
        assert st["last_queued_warp_stage"] > 0 and st["last_reach_plane_stage"] > 0, st
    if mk == "terr":
        assert st["last_deferred"] > 0, st
    assert np.array_equal(chk.isValidBatch(poses.astype(np.float32)), ref)
    d = torch.from_numpy(poses).cuda()
    dv, dv32 = chk.isValidBatch(d), chk.isValidBatch(d.float().contiguous())
    torch.cuda.synchronize()
    assert np.array_equal(dv.cpu().numpy(), ref) and np.array_equal(dv32.cpu().numpy(), ref)
    sl = np.arange(0, len(poses), len(poses) // 24)[:24]
    assert np.array_equal(np.array([chk.isValid(poses[i]) for i in sl], np.uint8), ref[sl])
    chk.setMode(1)
    got1 = chk.isValidBatch(poses)
    st1 = chk.stats()
    bad = np.nonzero(got1 != ref)[0]
    assert bad.size == 0, f"group-only: {bad.size} mismatches, first {bad[:8]}"
    assert st1["last_deferred"] == st1["last_queued_boxes"]


@pytest.mark.parametrize("pk", ["yaml", "header"])
def test_one_warp_per_box_route(ap, pk, gold, omaps):
    """ARTP_NO_GROUPS (read at artp_set_map) sends every reach box to the one-warp-per-box kernel: same masks."""
    os.environ["ARTP_NO_GROUPS"] = "1"
    try:
        chk = ap.StateValidityChecker(oc.PARAMS[pk], device=0)
        for name, mk, cpk, seed in oc.POSE_CASES:
            if cpk != pk:
                continue
            m = omaps(mk)
            chk.setMap(m)
            chk.updateHeightField()
            poses = oc.case_poses(m, mk, seed)
            got = chk.isValidBatch(poses)
            assert chk.stats()["last_reach_plane_stage"] == 0
            bad = np.nonzero(got != unpack(gold, name + "/mask", len(poses)))[0]
            assert bad.size == 0, f"{name}: {bad.size} mismatches, first {bad[:8]}"
    finally:
        os.environ.pop("ARTP_NO_GROUPS", None)


def test_host_batch_over_2_pow_20_off_origin(ap, omaps, port_lib):
    """A host batch of more than 2^20 states (several rounds, sliced copies) on the off-origin rows = 1 mod 4 map."""
    import torch
    m = omaps("r1")
    chk = checker(ap, m)
    n = (1 << 20) + 4099
    poses = synth.make_terrain_poses(m, n, seed=77)
    host = chk.isValidBatch(poses)
    dev = chk.isValidBatch(torch.from_numpy(poses).cuda()).cpu().numpy()
    assert np.array_equal(host, dev)
    assert np.array_equal(host, oracle(port_lib, m).check_poses_mt(poses, 8))
    assert 0.05 < host.mean() < 0.95


@pytest.mark.parametrize("mk", oc.EDGE_MAPS)
def test_edges_bit_exact(ap, mk, gold, omaps):
    """checkMotionBatch, checkEdgeInteriors and checkMotionSegments (counts given and from the space) on r3, coarse, far."""
    m = omaps(mk)
    chk = checker(ap, m)
    n, steps, seed = oc.EDGES
    s1, s2 = synth.make_edges(m, n, seed)
    assert np.array_equal(ap.MotionValidator(chk, steps).checkMotionBatch(s1, s2), unpack(gold, f"edges_{mk}/mask", n))
    n, seed, dmin, dmax = oc.INTERIORS
    s1, s2 = synth.make_edges(m, n, seed, dmin=dmin, dmax=dmax)
    k, _ = ap.MotionValidator(chk).checkEdgeInteriors(s1, s2, None, 0.5)
    assert np.array_equal(k, gold[f"interior_{mk}/prefix"].astype(np.int32))
    n, seed, dmin, dmax = oc.SEGMENTS
    s1, s2 = synth.make_edges(m, n, seed, dmin=dmin, dmax=dmax)
    mv = ap.MotionValidator(chk)
    sp = mv.se3Space(m, oc.PARAMS["yaml"].reach_z)
    nd = mv.validSegmentCount(sp, s1, s2)
    assert np.array_equal(nd, gold[f"segments_{mk}/nd"])
    for kw in (dict(nd=nd), dict(space=sp)):
        v, t = mv.checkMotionSegments(s1, s2, **kw)
        assert np.array_equal(v, unpack(gold, f"segments_{mk}/mask", n))
        assert same_bits(t, gold[f"segments_{mk}/last_t"])


#: row slabs and windows (row0 a multiple of 4, nrows not): the last window ends at the map's last row
WINDOWS = {"r3": [((0, 68), (0, 111)), ((68, 136), (24, 155)), ((136, 203), (92, 111))],
           "r1": [((0, 68), (0, 111)), ((68, 136), (24, 155)), ((136, 201), (92, 109))]}


@pytest.mark.parametrize("mk", list(WINDOWS))
def test_map_windows_with_unaligned_rows(ap, mk, gold, omaps):
    m = omaps(mk)
    name = f"{mk}_yaml"
    poses = oc.case_poses(m, mk, [c[3] for c in oc.POSE_CASES if c[0] == name][0])
    poses = poses[:oc.N_TERRAIN]                                   # inside the map: every one is routed to a slab
    ref = unpack(gold, name + "/mask", oc.N_TERRAIN)
    lx, _ = m.length
    row = np.floor((m.cx + 0.5 * lx - poses[:, 0]) / m.res).astype(int)
    got = np.full(len(poses), 255, np.uint8)
    for (s0, s1), (lo, nrows) in WINDOWS[mk]:
        assert lo % 4 == 0 and nrows % 4 != 0 and (lo == 0 or lo <= s0 - 40) and (lo + nrows >= s1 + 40 or lo + nrows == m.rows)
        shard = checker(ap, m, window=(lo, nrows))
        sel = np.nonzero((row >= s0) & (row < s1))[0]
        got[sel] = shard.isValidBatch(poses[sel])
        shard.pollError()
        if lo == 24:                 # samples far from this window: loud failure, never a wrong 'valid'
            far = np.nonzero(row < 8)[0][:300]
            assert far.size
            with pytest.raises(ap.ArtpError) as ei:
                shard.isValidBatch(poses[far])
            assert ei.value.code == capi.ARTP_E_WINDOW
    assert WINDOWS[mk][-1][1][0] + WINDOWS[mk][-1][1][1] == m.rows
    bad = np.nonzero(got != ref)[0]
    assert bad.size == 0, f"{bad.size} mismatches, first {bad[:8]}"


def check_pose_from_2d(chk, m, layers):
    """poseFrom2D over the normals the handle holds (layers: the same normals on the host) == the numpy restatement."""
    g = synth.make_terrain_poses(m, 3000, seed=701)
    lx, ly = m.length
    g[::7, 0] = m.cx + 0.5 * lx + 0.3                     # off the map in x
    g[3::11, 1] = m.cy - 0.5 * ly - 0.01                  # off the map in y
    pg, inside = chk.poseFrom2D(g)
    want, want_in = sgo.pose_from_2d(m, layers, g)
    assert np.array_equal(inside, want_in) and (inside == 0).any() and (inside == 1).mean() > 0.7
    assert same_bits(pg[:, :3], want[:, :3])
    assert np.abs(pg[:, 3:] - want[:, 3:]).max() < STATE_TOL


@pytest.mark.parametrize("mk", LAYER_MAPS)
def test_map_derived_layers(ap, mk, omaps, port_lib):
    """estimateNormals, poseFrom2D, computeSampleCdf, sampleUniformBatch (both modes) and findValidNear on non-square,
    off-origin maps against the CPU restatements."""
    m = omaps(mk)
    chk = checker(ap, m)
    p = oc.PARAMS["yaml"]
    radius = (p.torso_length + p.torso_width) * 0.25            # basic.cpp:47
    got = chk.estimateNormals(radius)
    ref = port_lib.estimate_normals(m, radius)
    for g, r, what in zip(got, ref, ("normal_x", "normal_y", "normal_z", "plane_fit_std_dev")):
        fin = np.isfinite(r)
        assert np.array_equal(np.isfinite(g), fin) and fin.mean() > 0.5, what
        assert np.array_equal(g[fin].view(np.uint32), r[fin].view(np.uint32)), what

    class Normals:
        normal_x, normal_y, normal_z = got[:3]
    check_pose_from_2d(chk, m, Normals)
    L = synth.make_sampler_layers(m, seed=7)
    cum, row = chk.computeSampleCdf(L.sample_probability)
    rcum, rrow = port_lib.compute_cdf(L.sample_probability)
    nan = np.isnan(rcum)
    assert nan.any() and np.array_equal(np.isnan(cum), nan)
    assert np.array_equal(cum[~nan].view(np.uint32), rcum[~nan].view(np.uint32))
    assert np.array_equal(row.view(np.uint32), rrow.view(np.uint32))
    for from_dist in (True, False):
        sp = synth.sampler_params_for(m, from_dist)
        smp = ap.SE3FromSE2Sampler(chk, L, sp, seed=11)
        u = philox_ref.sampler_uniforms(11, 0, 20000)
        want, want_rc = port_lib.sample_states(m, L, sp, p.reach_z, u)
        st, rc = smp.sampleUniformBatch(20000, u=u, want_cells=True)
        assert np.array_equal(rc, want_rc), from_dist
        ok = ~np.isnan(want[:, 0])
        assert ok.mean() > 0.2 and np.array_equal(np.isnan(st[:, 0]), ~ok)
        assert np.abs(st[ok] - want[ok]).max() < STATE_TOL, from_dist
    check_pose_from_2d(chk, m, L)                              # the sampler's host normal layers replaced the estimate
    centres, rad = sgc.make_queries(m, 240, 401)
    n_iter = 24
    off = philox_ball_ref.ball_offsets(401, 0, 240, n_iter, rad)
    rs, ri = sgo.find_valid_near(oracle(port_lib, m), centres, n_iter, off)
    assert (ri == 0).any() and (ri > 0).any() and (ri < 0).any()
    for mode in (0, 1):
        chk.setMode(mode)
        s, i = chk.findValidNear(centres, rad, n_iter, offsets=off)
        assert np.array_equal(i, ri) and same_bits(s, rs), mode


@pytest.mark.parametrize("shape", [(203, 157), (157, 203)], ids=["203x157", "157x203"])
def test_process_basic_non_square(ap, shape):
    """processors::Basic on a non-square map and its transpose: a rows <-> cols swap shows up on one of the two."""
    from oracle import basic_oracle as bo
    m = synth.make_fbm_map(*shape, 0.04, seed=41)
    trav, obs = synth.make_traversability(m, seed=13)
    chk = ap.StateValidityChecker(oc.PARAMS["yaml"], device=0)
    p = bo.BasicParams()
    masked, thr = chk.processBasic(m.elevation, trav, obs, m.res, p)
    ref_m, ref_t = bo.masked_elevation(m.elevation, trav, obs, m.res, p)
    assert masked.shape == shape and np.isinf(ref_m).any() and np.isfinite(ref_m).any()
    assert np.array_equal(masked.view(np.uint32), ref_m.view(np.uint32))
    assert np.array_equal(thr, ref_t)


def test_resolution_limit_of_the_plane_store(ap, gold, omaps):
    """At 0.02 m the yaml torso's zone bound needs 2 * 78 * 78 * 21 B ~ 255 KB of plane store (cap 200 KB): the map is
    refused with ARTP_E_LIMIT; the smaller header torso needs ~172 KB and is accepted. The refused handle then takes the
    0.025 m map and checks it like a fresh one."""
    m = synth.make_fbm_map(300, 300, 0.02, seed=51)
    chk = ap.StateValidityChecker(oc.PARAMS["yaml"], device=0)
    chk.setMap(m)
    with pytest.raises(ap.ArtpError) as ei:
        chk.updateHeightField()
    assert ei.value.code == capi.ARTP_E_LIMIT and "shared-memory store" in str(ei.value)
    assert not chk.hasMap()
    hdr = checker(ap, m, "header")
    assert hdr.hasMap()
    fine = omaps("fine")
    chk.setMap(fine)
    chk.updateHeightField()
    poses = oc.case_poses(fine, "fine", [c[3] for c in oc.POSE_CASES if c[0] == "fine_yaml"][0])
    assert np.array_equal(chk.isValidBatch(poses), unpack(gold, "fine_yaml/mask", len(poses)))
