"""GPU (-m gpu): handles and map changes that share one device. Every handle's launch shapes are derived from its map
(upload_map / set_shapes), but a kernel's max-dynamic-shared-memory attribute belongs to the device's context and is
shared by every handle in the process. So these tests install maps of different sizes on several handles and then use
each handle without reinstalling it, change maps under one handle while it keeps working (other sizes, cell sizes, height
offsets, windows, a refused map, a map without a reach-box queue, the ARTP_NO_GROUPS route), and recompute what is derived
from the map after a change. Every answer must equal the port oracle's (and the compiled reference's golden where one
exists for the map) and a fresh handle's, bit for bit."""
from __future__ import annotations

import dataclasses
import math
import os
import threading

import numpy as np
import pytest

import philox_ball_ref
import start_goal_cases as sgc
import start_goal_oracle as sgo
from art_planner_b200 import capi, costnet, synth
from oracle import roadmap_oracle as ro
from test_compact_tables_gpu import boundary_poses

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KB = 1024
STATE_TOL = 1e-9        # roadmap interpolation: CUDA vs numpy sin / cos / acos of the slerp; vertex kinds and edges are exact


# ---- the per-map launch shapes, restated from upload_map (artp_map.cu) and set_shapes (artp_capi.cu) -------------------
@dataclasses.dataclass
class Tile:
    tw: int
    th: int
    stride: int
    slots: int
    wpc: int            # warps per CTA
    smem: int


@dataclasses.dataclass
class Shapes:
    span: list          # [torso, reach] (vertices along x, along z) of a box's zone bound
    kmax: list          # [torso, reach] highest range-table level
    tcap: int           # triangles of the grouping stage's plane store
    store: int          # its bytes: box_items_block_kernel's dynamic shared memory
    tiles: list         # [big-tile queue, reach-box queue] box_tiles_warp_kernel configurations; reach None: no queue
    groups: int | None  # reach_groups_kernel's dynamic shared memory, None: no 8-lane queue
    accepted: bool      # the store fits its 200 KB cap


def launch_shapes(p, res, rows, cols, no_groups=False) -> Shapes:
    f32 = np.float32
    W, D = f32(rows * res), f32(cols * res)
    iW, iD = f32(1) / (W / (f32(rows) - f32(1))), f32(1) / (D / (f32(cols) - f32(1)))
    span, kmax, tcap = [], [], 0
    for sides in ((p.torso_length, p.torso_width, p.torso_height), (p.reach_x, p.reach_y, p.reach_z)):
        s = [float(f32(v)) for v in sides]
        r = 0.5 * math.sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2])
        sx, sz = math.ceil(2.0 * r * float(iW)), math.ceil(2.0 * r * float(iD))
        span.append((sx, sz))
        nxm, nzm = min(rows, sx + 4), min(cols, sz + 4)
        tcap = max(tcap, 2 * (nxm - 1) * (nzm - 1))
        k = 0
        while (2 << k) <= min(nxm, nzm) and k < 6:
            k += 1
        kmax.append(k)
    tcap = (tcap + 3) & ~3
    store = tcap * 21 + 64
    tiles = []
    for q in range(2):
        tw, th = min((span[q][0] + 9) & ~3, 256), min(span[q][1] + 3, 256)
        stride = (tw * th * 4 + 127) & ~127
        slots = 1 if stride > 2048 else 2
        wpc = 8
        while wpc > 1 and wpc * slots * stride + 128 > 72 * KB:
            wpc >>= 1
        if wpc * slots * stride + 128 > 200 * KB:
            if q == 1:
                tiles.append(None)
                continue
            tw, th, stride, slots, wpc = 64, 64, 64 * 64 * 4, 1, 4
        tiles.append(Tile(tw, th, stride, slots, wpc, wpc * slots * stride + 128))
    groups = None
    if tiles[1] is not None and tiles[1].tw <= 127 and tiles[1].th <= 255 and not no_groups:
        gsm = 8 * 8 * tiles[1].stride + 128
        groups = gsm if gsm <= 160 * KB else None
    return Shapes(span, kmax, tcap, store, tiles, groups, store <= 200 * KB)


def tile_smem(s: Shapes) -> int:
    """The largest box_tiles_warp_kernel launch of the map (one kernel runs both tile sizes)."""
    return max(t.smem for t in s.tiles if t is not None)


def test_launch_shapes_restated():
    """The restatement against sizes worked out by hand from set_shapes for the shipped robots (400 x 400 maps)."""
    a = launch_shapes(synth.PARAMS_YAML, 0.04, 400, 400)
    b = launch_shapes(synth.PARAMS_HEADER, 0.04, 400, 400)
    c = launch_shapes(synth.PARAMS_YAML, 0.10, 400, 400)
    assert (a.store, tile_smem(a), a.groups) == (70708, 58496, 49280)
    assert (b.store, tile_smem(b), b.groups) == (45844, 39040, 49280)
    assert (c.store, tile_smem(c), c.groups) == (13672, 28800, 24704)
    assert a.kmax == [5, 3] and c.kmax == [4, 3] and a.tiles[0].wpc == 8
    assert not launch_shapes(synth.PARAMS_YAML, 0.02, 300, 300).accepted
    assert launch_shapes(synth.PARAMS_HEADER, 0.02, 300, 300).accepted


# ---- maps, handles, oracles ----------------------------------------------------------------------------------------------
def fbm(rows=400, cols=400, res=0.04, seed=2, **kw):
    return synth.make_fbm_map(rows, cols, res, seed=seed, amp=0.6, **kw)


def offset(m, dz):
    return dataclasses.replace(m, elevation=np.asfortranarray(m.elevation + np.float32(dz)),
                               elevation_masked=np.asfortranarray(m.elevation_masked + np.float32(dz)))


def strip(res):
    """A map two vertices wide and 50 long: the zones of every box are clamped to two rows."""
    rows, cols = 2, 50
    j = np.arange(cols, dtype=np.float32)
    e = np.asfortranarray(np.stack([0.3 * np.sin(0.3 * j), 0.3 * np.cos(0.2 * j) - 0.1]).astype(np.float32))
    mk = e.copy(order="F")
    mk[1, 20:24] = -np.inf
    return synth.SynthMap(e, mk, res, 0.0, 0.0, f"strip 2x50@{res}")


def strip_poses(m, n, seed, p):
    """Poses with one foot over the strip: a point of the strip, a foot, a yaw, and the pose placed so that this foot's box
    is centred on the point, its bottom within 0.15 m of the strip's height there. The rest of the robot is off the map."""
    k = np.arange(n)
    u = lambda stream: synth.hash_uniform(seed, stream, k)  # noqa: E731
    lx, ly = m.length
    tx, ty = m.cx + (u(1) - 0.5) * lx, m.cy + (u(2) - 0.5) * ly
    i, j = m.index_of(tx, ty)
    h = m.elevation[i, j].astype(np.float64)
    foot = (u(3) * 4).astype(int)
    fx = np.where(foot & 2, -p.feet_off_x, p.feet_off_x)
    fy = np.where(foot & 1, -p.feet_off_y, p.feet_off_y)
    yaw = (u(4) * 2 - 1) * math.pi
    c, s = np.cos(yaw), np.sin(yaw)
    x, y = tx - (c * fx - s * fy), ty - (s * fx + c * fy)
    z = h + 0.5 * p.reach_z + (u(5) * 2 - 1) * 0.15
    q = synth.quat_from_rpy((u(6) * 2 - 1) * 0.1, (u(7) * 2 - 1) * 0.1, yaw)
    return np.ascontiguousarray(np.stack([x, y, z, *q], axis=1))


@pytest.fixture(scope="module")
def ap():
    import art_planner_b200
    from art_planner_b200 import build
    build.build()
    return art_planner_b200


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "reference_masks.npz"))


def unpack(g, key, n):
    return np.unpackbits(g[key])[:n]


def same_bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


def install(chk, m, window=None):
    chk.setMap(m)
    chk.updateHeightField(window=window)


def checker(ap, p, m, window=None):
    chk = ap.StateValidityChecker(p, device=0)
    install(chk, m, window)
    return chk


# ---- (b) handles of different map sizes on one device, each used without reinstalling ------------------------------------
#: the three handles: robot, map, the golden's case names for it (None: port oracle only)
HANDLES = {
    "A": (synth.PARAMS_YAML, lambda: fbm(), ("fbm_rough_yaml", "edges_fbm_rough_yaml", "interior_fbm_rough_yaml",
                                                "segments_fbm_rough_yaml")),
    "B": (synth.PARAMS_HEADER, lambda: fbm(), ("fbm_rough_header", None, None, None)),
    "C": (synth.PARAMS_YAML, lambda: fbm(160, 160, 0.10, seed=8), (None, None, None, None)),
}
N_POSES, N_EDGES, EDGE_STEPS, N_INTERIOR, N_SEGMENTS = 20000, 3000, 20, 4000, 3000


class Expected:
    """Inputs and the port oracle's answers for one handle's map, checked once against the golden where it exists."""

    def __init__(self, port_lib, gold, key):
        p, mk, (gp, ge, gi, gs) = HANDLES[key]
        self.p, self.m = p, mk()
        m = self.m
        o = port_lib.Oracle(p, "port")
        o.set_map(m)
        self.o = o
        self.poses = synth.make_terrain_poses(m, N_POSES, seed=3)
        self.valid = o.check_poses_mt(self.poses, 8)
        if gp:
            assert np.array_equal(self.valid, unpack(gold, gp + "/mask", N_POSES))
        assert 0.05 < self.valid.mean() < 0.95
        self.e1, self.e2 = synth.make_edges(m, N_EDGES, 4)
        self.edges = o.check_motions_mt(self.e1, self.e2, EDGE_STEPS, 8)
        if ge:
            assert np.array_equal(self.edges, unpack(gold, ge + "/mask", N_EDGES))
        self.i1, self.i2 = synth.make_edges(m, N_INTERIOR, 21, dmin=0.05, dmax=3.4)
        self.prefix = o.check_edge_interiors(self.i1, self.i2, None, 0.5)
        if gi:
            assert np.array_equal(self.prefix, gold[gi + "/prefix"].astype(np.int32))
        self.g1, self.g2 = synth.make_edges(m, N_SEGMENTS, 51, dmin=0.05, dmax=2.5)
        lo, hi = ([m.cx - m.length[0], m.cy - m.length[1]], [m.cx + m.length[0], m.cy + m.length[1]])
        e = m.elevation[np.isfinite(m.elevation)]
        lo.append(float(e.min()) - p.reach_z / 2)
        hi.append(float(e.max()) + p.reach_z / 2)
        self.nd = o.valid_segment_count(lo, hi, self.g1, self.g2)
        self.seg_valid, self.seg_t = o.check_motions_segments(self.g1, self.g2, self.nd)
        if gs:
            assert np.array_equal(self.nd, gold[gs + "/nd"])
            assert np.array_equal(self.seg_valid, unpack(gold, gs + "/mask", N_SEGMENTS))
            assert same_bits(self.seg_t, gold[gs + "/last_t"])
        self.centres, self.radius = sgc.make_queries(m, 200, 401)
        self.n_iter = 16
        self.offsets = philox_ball_ref.ball_offsets(401, 0, 200, self.n_iter, self.radius)
        self.near_states, self.near_idx = sgo.find_valid_near(o, self.centres, self.n_iter, self.offsets)
        self.layers = synth.make_sampler_layers(m, seed=7)
        self.sp = synth.sampler_params_for(m)


@pytest.fixture(scope="module")
def expected(port_lib, gold):
    cache = {}

    def get(key):
        if key not in cache:
            cache[key] = Expected(port_lib, gold, key)
        return cache[key]
    return get


def check_everything(ap, chk, x: Expected, what: str):
    """Every entry point that launches the box kernels, on a handle holding x's map."""
    import torch
    st = chk.stats()
    assert np.array_equal(chk.isValidBatch(x.poses), x.valid), f"{what}: host double states"
    assert np.array_equal(chk.isValidBatch(x.poses.astype(np.float32)), x.valid), f"{what}: host float states"
    d = torch.from_numpy(x.poses).cuda()
    dv, dv32 = chk.isValidBatch(d), chk.isValidBatch(d.float().contiguous())
    torch.cuda.synchronize()
    assert np.array_equal(dv.cpu().numpy(), x.valid), f"{what}: device double states"
    assert np.array_equal(dv32.cpu().numpy(), x.valid), f"{what}: device float states"
    sl = np.arange(0, N_POSES, N_POSES // 32)[:32]
    assert np.array_equal(np.array([chk.isValid(x.poses[i]) for i in sl], np.uint8), x.valid[sl]), f"{what}: isValid"
    mv = ap.MotionValidator(chk, EDGE_STEPS)
    assert np.array_equal(mv.checkMotionBatch(x.e1, x.e2), x.edges), f"{what}: checkMotionBatch"
    v, t = mv.checkMotionSegments(x.g1, x.g2, nd=x.nd)
    assert np.array_equal(v, x.seg_valid) and same_bits(t, x.seg_t), f"{what}: checkMotionSegments"
    k, _ = mv.checkEdgeInteriors(x.i1, x.i2, None, 0.5)
    assert np.array_equal(k, x.prefix), f"{what}: checkEdgeInteriors"
    smp = ap.SE3FromSE2Sampler(chk, x.layers, x.sp, seed=13)
    cand = smp.sampleUniformBatch(20000, first=0)
    inside = ~np.isnan(cand[:, 0])
    keep = np.zeros(len(cand), bool)
    keep[inside] = x.o.check_poses(cand[inside]) != 0
    got, n_valid = smp.sampleValidBatch(20000, first=0)
    assert n_valid == keep.sum() > 0 and same_bits(got, cand[keep]), f"{what}: sampleValidBatch"
    s, i = chk.findValidNear(x.centres, x.radius, x.n_iter, offsets=x.offsets)
    assert np.array_equal(i, x.near_idx) and same_bits(s, x.near_states), f"{what}: findValidNear"
    rm = ap.PRMRoadmap(chk, 8000, 20000)
    ms = x.poses[x.valid != 0][:48]
    rm.addValidMilestones(ms)
    ref = ro.Roadmap()
    for s in ms:
        ref.add_milestone(s, ro.validity(x.o), ro.MILESTONE | ro.QUERY)
    vs, kinds = rm.vertices()
    rst, rkinds, redges = ref.result()
    assert np.array_equal(kinds, rkinds) and np.array_equal(rm.edges(), redges), f"{what}: addValidMilestones"
    assert len(redges) > 0 and np.abs(vs - rst).max(initial=0.0) <= STATE_TOL, f"{what}: addValidMilestones"
    assert chk.stats()["poses_checked"] > st["poses_checked"]


@pytest.mark.parametrize("order", ["ABC", "CBA"], ids=["largest-first", "largest-last"])
@pytest.mark.parametrize("mode", [0, 1], ids=["default", "group-only"])
def test_handles_keep_their_maps(ap, expected, order, mode):
    """Install A's, B's and C's maps in `order`, then use A, then B, then C, none of them reinstalled. A's map asks the most
    of the grouping stage and of the tile kernel, C's the least."""
    a, b, c = (launch_shapes(HANDLES[k][0], expected(k).m.res, *expected(k).m.elevation.shape) for k in "ABC")
    assert a.store > 48 * KB and a.store > b.store > c.store and tile_smem(a) > tile_smem(b) > tile_smem(c)
    assert a.groups > c.groups and a.tiles[1] is not None and c.tiles[1] is not None
    chks = {k: ap.StateValidityChecker(HANDLES[k][0], device=0) for k in "ABC"}
    for k in order:
        install(chks[k], expected(k).m)
        chks[k].setMode(mode)
    for k in "ABC":
        check_everything(ap, chks[k], expected(k), f"handle {k} after installing {order}")
        st = chks[k].stats()
        if mode == 1:
            assert st["last_deferred"] == st["last_queued_boxes"] > 0, (k, st)


def test_threads_with_their_own_handles(ap, expected):
    """Two threads, each with its own handle of a differently sized map (A and C), alternate installing their map with
    batch checks: A's map installed last, C's installed last, both installed at once."""
    import torch
    xs = {k: expected(k) for k in "AC"}
    a, c = (launch_shapes(HANDLES[k][0], xs[k].m.res, *xs[k].m.elevation.shape) for k in "AC")
    assert a.store > 48 * KB > c.store and tile_smem(a) > tile_smem(c)
    chks = {k: ap.StateValidityChecker(HANDLES[k][0], device=0) for k in "AC"}
    for k in "AC":
        chks[k].setMap(xs[k].m)
    barrier = threading.Barrier(2)
    errors = []

    def run(k):
        try:
            chk, x = chks[k], xs[k]
            torch.cuda.set_device(0)
            stream = torch.cuda.Stream()
            for r in range(6):
                barrier.wait()
                if r % 3 < 2:          # one thread installs its map right after the other's, then both check
                    first = "AC"[r % 3]
                    if k != first:
                        barrier.wait()
                    chk.updateHeightField()
                    if k == first:
                        barrier.wait()
                else:                  # both at once
                    chk.updateHeightField()
                chk.setMode(r % 2)
                for _ in range(2):
                    assert np.array_equal(chk.isValidBatch(x.poses), x.valid), f"{k} round {r}: host states"
                    with torch.cuda.stream(stream):
                        dv = chk.isValidBatch(torch.from_numpy(x.poses).cuda())
                    stream.synchronize()
                    assert np.array_equal(dv.cpu().numpy(), x.valid), f"{k} round {r}: device states"
                    assert np.array_equal(ap.MotionValidator(chk, EDGE_STEPS).checkMotionBatch(x.e1, x.e2), x.edges), \
                        f"{k} round {r}: motions"
        except BaseException as e:          # noqa: BLE001 -- re-raised on the main thread
            errors.append(e)
            barrier.abort()

    threads = [threading.Thread(target=run, args=(k,)) for k in "AC"]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    real = [e for e in errors if not isinstance(e, threading.BrokenBarrierError)]
    if real or errors:
        raise (real or errors)[0]


# ---- (d) one handle walked through maps -----------------------------------------------------------------------------------
class Walk:
    """One handle of the yaml robot taken through a sequence of maps; at each step its masks must equal the port oracle's and
    those of a fresh handle holding the same map. Unknown space is traversable here: on the strip maps every pose has boxes
    off the map, and only then are the boxes over the strip decided at all."""

    def __init__(self, ap, port_lib):
        self.ap, self.port_lib = ap, port_lib
        self.p = dataclasses.replace(synth.PARAMS_YAML, unknown_space_untraversable=False)
        self.chk = ap.StateValidityChecker(self.p, device=0)
        self.last = None

    def poses(self, m, n, seed, rows=None):
        if m.rows == 2:
            return strip_poses(m, n, seed, self.p)
        t = synth.make_terrain_poses(m, n, seed=seed)
        b = boundary_poses(m, min(n, 3000), seed + 1, self.p)
        s = np.concatenate([t, b])
        if rows is not None:          # a window: only poses whose boxes stay inside the rows it holds
            lx, _ = m.length
            row = np.floor((m.cx + 0.5 * lx - s[:, 0]) / m.res).astype(int)
            s = s[(row >= rows[0]) & (row < rows[1])]
        return s

    def step(self, m, what, n=4000, seed=3, window=None, rows=None, big=False):
        import torch
        install(self.chk, m, window)
        assert self.chk.hasMap()
        s = self.poses(m, n, seed, rows)
        o = self.port_lib.Oracle(self.p, "port")
        o.set_map(m)
        ref = o.check_poses_mt(s, 8)
        assert 0.02 < ref.mean() < 0.98, (what, ref.mean())
        got = self.chk.isValidBatch(s)
        st = self.chk.stats()
        bad = np.nonzero(got != ref)[0]
        assert bad.size == 0, f"{what}: {bad.size} mismatches, first {bad[:8]}, stats {st}"
        fresh = checker(self.ap, self.p, m, window)
        assert np.array_equal(fresh.isValidBatch(s), got), what
        if big:
            dev = self.chk.isValidBatch(torch.from_numpy(s).cuda()).cpu().numpy()
            assert np.array_equal(dev, ref), what
        fresh.handle.close()
        self.last = (s, got)
        return st


def test_one_handle_walks_through_maps(ap, port_lib):
    w = Walk(ap, port_lib)
    P = w.p
    sh = lambda m, **kw: launch_shapes(P, m.res, *m.elevation.shape, **kw)  # noqa: E731

    m400 = fbm()
    st = w.step(m400, "400x400 at 0.04 m")
    assert st["last_reach_plane_stage"] > 0 and st["last_queued_reach_stage"] > 0, st
    # shrink: new dimensions reallocate the layers and every table level; a batch of more than 2^20 poses grows the queues
    small = fbm(203, 157, 0.04, seed=41, cx=3.1, cy=-1.7)
    w.step(small, "203x157 at 0.04 m, > 2^20 poses", n=(1 << 20) + 4099, seed=77, big=True)
    w.step(small, "203x157 again, a small batch on the grown queues", n=3000, seed=78)
    # same dimensions, other cell sizes: kmax rises (levels allocated on the reused layers), then falls (levels above stay)
    s04, s025, s10 = sh(small), sh(dataclasses.replace(small, res=0.025)), sh(dataclasses.replace(small, res=0.10))
    assert s025.kmax[0] > s04.kmax[0] > s10.kmax[0] and s025.kmax[1] > s04.kmax[1], (s025.kmax, s04.kmax, s10.kmax)
    w.step(fbm(203, 157, 0.025, seed=42), "203x157 at 0.025 m")
    w.step(fbm(203, 157, 0.10, seed=43), "203x157 at 0.10 m")
    # grow back; +300 m moves the compact codes' base and step, then the offset goes again
    w.step(offset(m400, 300.0), "400x400 +300 m")
    w.step(m400, "400x400, offset removed")
    # a window, the whole map, a window of the same height at another row0 (the layers are reused, the offsets are not)
    w.step(m400, "window rows 100..249", window=(100, 150), rows=(140, 210))
    w.step(m400, "whole map after a window")
    w.step(m400, "window rows 200..349", window=(200, 150), rows=(240, 310))
    w.chk.pollError()
    st = w.step(m400, "whole map")
    # a refused map between two accepted ones leaves the previous map installed and its verdicts unchanged
    fine = fbm(300, 300, 0.02, seed=51)
    assert not sh(fine).accepted
    s, before = w.last
    w.chk.setMap(fine)
    with pytest.raises(ap.ArtpError) as ei:
        w.chk.updateHeightField()
    assert ei.value.code == capi.ARTP_E_LIMIT
    assert w.chk.hasMap()
    assert np.array_equal(w.chk.isValidBatch(s), before)
    assert np.array_equal(w.chk.isValidBatch(s.astype(np.float32)), before)
    assert np.array_equal(np.array([w.chk.isValid(x) for x in s[:16]], np.uint8), before[:16])
    st2 = w.chk.stats()
    assert st2["last_reach_plane_stage"] == st["last_reach_plane_stage"] > 0, (st, st2)
    # a map whose reach tile would need more than 200 KB has no reach-box queue (and the torso tile takes its 64 x 64 cap);
    # the strip before it has the same dimensions and a reach queue, so nothing but set_shapes can drop that queue
    wide, tight = sh(strip(0.002)), sh(strip(0.0009))
    assert wide.tiles[1] is not None and wide.groups is None and wide.tiles[1].th >= 50 and wide.tiles[1].tw >= 8
    assert tight.tiles[1] is None and tight.tiles[0].tw == tight.tiles[0].th == 64 and tight.accepted
    # a host batch of one round launches classify, the box kernels of the map's queues and the grouping stage
    st = w.step(strip(0.002), "2x50 strip at 2 mm", n=20000, seed=5)
    assert st["last_launches"] == 4 and st["last_reach_plane_stage"] == 0, st
    st = w.step(strip(0.0009), "2x50 strip at 0.9 mm: no reach-box queue", n=20000, seed=5)
    assert st["last_launches"] == 3 and st["last_queued_reach_stage"] == 0 and st["last_reach_plane_stage"] == 0, st
    st = w.step(m400, "400x400 after the strip")
    assert st["last_reach_plane_stage"] > 0 and st["last_queued_reach_stage"] > 0, st
    # ARTP_NO_GROUPS is read at the install: the route follows it both ways, the masks do not
    assert sh(m400).groups is not None and sh(m400, no_groups=True).groups is None
    os.environ["ARTP_NO_GROUPS"] = "1"
    try:
        st = w.step(m400, "ARTP_NO_GROUPS set")
    finally:
        os.environ.pop("ARTP_NO_GROUPS", None)
    assert st["last_reach_plane_stage"] == 0 and st["last_queued_reach_stage"] > 0, st
    st = w.step(m400, "ARTP_NO_GROUPS unset")
    assert st["last_reach_plane_stage"] > 0, st


# ---- (e) what is derived from the map, after a change -----------------------------------------------------------------------
def test_map_derived_state_after_a_change(ap):
    from oracle import sample_distribution_oracle as sdo
    p = synth.PARAMS_YAML
    radius = (p.torso_length + p.torso_width) * 0.25
    m1, m2 = fbm(256, 256, 0.04, seed=2), fbm(200, 232, 0.04, seed=9, cx=1.5, cy=-0.5)

    def derive(chk, m, seed):
        """Normals, CDF, sample filter, distribution and samples of m on chk; returns them."""
        normals = chk.estimateNormals(radius)
        L = synth.make_sampler_layers(m, seed=seed)
        cdf = chk.computeSampleCdf(L.sample_probability)
        trav, obs = synth.make_traversability(m, seed=seed)
        filt = chk.setSampleFilter((trav > 0.3).astype(np.float32), obs)
        verts = synth.make_terrain_poses(m, 300, seed=seed)
        dist = chk.updateSampleDistribution(verts, sdo.DistributionParams())
        Lr = dataclasses.replace(L, normal_x=None, normal_y=None, normal_z=None, plane_fit_std_dev=None,
                                 cum_prob=None, cum_prob_rowwise=None)
        smp = ap.SE3FromSE2Sampler(chk, Lr, synth.sampler_params_for(m), seed=5)     # the device layers just computed
        samples = smp.sampleUniformBatch(5000, first=0)
        return [*normals, *cdf, filt, *dist, samples], smp

    chk = checker(ap, p, m1)
    obj = ap.MotionCostObjective(chk)
    obj.setWeights(costnet.make_state_dict(seed=5))
    obj.updateFeatures()
    _, smp = derive(chk, m1, 7)
    install(chk, m2)
    # the sampler, the normals, the CDF, the sample filter and observed layers belonged to m1: refused until recomputed
    with pytest.raises(ap.ArtpError) as ei:
        smp.sampleUniformBatch(16, first=0)
    assert ei.value.code == capi.ARTP_E_NOMAP
    with pytest.raises(ap.ArtpError) as ei:
        chk.poseFrom2D(synth.make_terrain_poses(m2, 4, seed=1))
    assert ei.value.code == capi.ARTP_E_INVALID
    L2 = synth.make_sampler_layers(m2, seed=8)
    no_normals = dataclasses.replace(L2, normal_x=None, normal_y=None, normal_z=None, plane_fit_std_dev=None)
    with pytest.raises(ap.ArtpError) as ei:
        ap.SE3FromSE2Sampler(chk, no_normals, synth.sampler_params_for(m2))
    assert ei.value.code == capi.ARTP_E_INVALID
    no_cdf = dataclasses.replace(L2, cum_prob=None, cum_prob_rowwise=None)
    with pytest.raises(ap.ArtpError) as ei:
        ap.SE3FromSE2Sampler(chk, no_cdf, synth.sampler_params_for(m2))
    assert ei.value.code == capi.ARTP_E_INVALID
    with pytest.raises(ap.ArtpError) as ei:            # the unknown-space cap needs this map's observed layer
        chk.updateSampleDistribution(synth.make_terrain_poses(m2, 10, seed=1), sdo.DistributionParams())
    assert ei.value.code == capi.ARTP_E_INVALID
    # recomputed, everything equals a fresh handle's bit for bit
    got, _ = derive(chk, m2, 8)
    fresh = checker(ap, p, m2)
    want, _ = derive(fresh, m2, 8)
    for i, (g, r) in enumerate(zip(got, want)):
        assert g.shape == r.shape and g.tobytes() == r.tobytes(), f"derived output {i}"
    assert np.isfinite(got[0]).mean() > 0.5 and (~np.isnan(got[-1][:, 0])).mean() > 0.2
    obj.updateFeatures()
    fobj = ap.MotionCostObjective(fresh)
    fobj.setWeights(costnet.make_state_dict(seed=5))
    fobj.updateFeatures()
    f, ff = obj.features(), fobj.features()
    assert f.shape == ff.shape and f.shape[:2] != (104, 104) and f.tobytes() == ff.tobytes()
