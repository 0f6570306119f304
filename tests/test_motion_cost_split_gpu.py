"""GPU tests (-m gpu) of the learned cost of whole edges and paths: MotionCostObjective::motionCost
(motion_cost_objective.cpp:36-95) split on the device by artp_motion_cost_split[_device], the Python mirror's
motionCost / motionCostBatch / pathCost and the C++ mirror's motionCostBatch / pathCost.

The numpy restatement below builds the pieces' rows as the reference does: n_interp = (unsigned)(lateralDistance / 0.5),
knots s1, interpolate(s1, s2, j * (1.0 / (n_interp + 1))), s2, row i = [x y yaw](knot i+1) ++ [x y yaw](knot i). x and y
are pure lerp and compared exactly. Yaw goes through double acos / sin / atan2, whose CUDA and libm results may differ by
an ulp; the float cast absorbs that except with probability ~2^-29 per value (DESIGN.md section 2), and the committed
seeded cases are exact."""
import os
import struct
import subprocess

import numpy as np
import pytest

import cases
from art_planner_b200 import costnet, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL, ATOL = 1e-4, 1e-5
THR = 0.55                    # seeded random weights give risks around 0.5: both feasible and infeasible pieces
W_E, W_T, W_R = 0.0, 1.0, 5.0   # the handle's default cost weights (params.h:57-61)


def _interpolate(a, b, t):
    """OMPL 1.4.2 SE3StateSpace::interpolate (lerp + slerp) row by row, numpy doubles, the operation order of
    test_host_cpp._interpolate."""
    o = np.empty_like(a)
    o[:, :3] = a[:, :3] + (b[:, :3] - a[:, :3]) * t[:, None]
    dq = a[:, 3] * b[:, 3] + a[:, 4] * b[:, 4] + a[:, 5] * b[:, 5] + a[:, 6] * b[:, 6]
    dqa = np.abs(dq)
    with np.errstate(all="ignore"):
        theta = np.where(dqa > 1.0 - 1e-9, 0.0, np.arccos(np.minimum(dqa, 1.0)))
        d = 1.0 / np.sin(theta)
        s0 = np.sin((1.0 - t) * theta)
        s1 = np.sin(t * theta)
        s1 = np.where(dq < 0, -s1, s1)
        slerp = (a[:, 3:] * s0[:, None] + b[:, 3:] * s1[:, None]) * d[:, None]
    o[:, 3:] = np.where((theta > np.finfo(np.float64).eps)[:, None], slerp, a[:, 3:])
    return o


def _yaw(s):
    """getYawFromSO3 (utils.h:80-88): double atan2, float result."""
    return np.arctan2(2 * (s[:, 6] * s[:, 5] + s[:, 3] * s[:, 4]), 1 - 2 * (s[:, 4] * s[:, 4] + s[:, 5] * s[:, 5])).astype(np.float32)


def split_rows(s1, s2, max_len=0.5):
    """The piece rows of every edge and the n + 1 piece offsets (motion_cost_objective.cpp:36-70)."""
    dx, dy = s2[:, 0] - s1[:, 0], s2[:, 1] - s1[:, 1]
    n_pieces = (np.sqrt(dx * dx + dy * dy) / max_len).astype(np.int64) + 1
    off = np.zeros(len(s1) + 1, np.int64)
    off[1:] = np.cumsum(n_pieces)
    e = np.repeat(np.arange(len(s1)), n_pieces)
    i = np.arange(off[-1]) - off[e]
    a, b, npc = s1[e], s2[e], n_pieces[e]

    def knots(j):
        k = np.where((j == 0)[:, None], a, b)
        inner = (j > 0) & (j < npc)
        t = j.astype(np.float64) * (1.0 / npc.astype(np.float64))
        k[inner] = _interpolate(a[inner], b[inner], t[inner])
        return k

    ka, kb = knots(i), knots(i + 1)
    rows = np.empty((len(e), 6), np.float32)
    rows[:, 0], rows[:, 1], rows[:, 2] = kb[:, 0], kb[:, 1], _yaw(kb)
    rows[:, 3], rows[:, 4], rows[:, 5] = ka[:, 0], ka[:, 1], _yaw(ka)
    return rows, off


def reduce_costs(c3, off, thr):
    """Per edge: +inf if a piece's risk is above the threshold, else the left-to-right double sum of getCost."""
    t = float(np.float32(thr))
    out = np.empty(len(off) - 1)
    for e in range(len(off) - 1):
        c = 0.0
        for k in range(off[e], off[e + 1]):
            ce, ct, cr = (float(v) for v in c3[k])
            if cr > t:
                c = np.inf
                break
            c += ce * W_E + ct * W_T + cr * W_R
        out[e] = c
    return out


def edge_set(m):
    """Edges 0-3 m long, lengths on the n_interp truncation boundary, zero-length and turn-in-place edges, quaternion
    pairs with a negative dot product, and starts outside the feature area (the head clamps them)."""
    s1r, s2r = synth.make_edges(m, 3000, seed=71, dmin=0.0, dmax=3.0)
    base = synth.make_terrain_poses(m, 240, seed=72)
    L = np.tile(np.arange(1, 7) * 0.5, 40)
    b1 = base.copy()
    b1[:, :2] = np.round(b1[:, :2] * 64) / 64               # dyadic: s1 + L and the difference back are exact
    ax = b1.copy()
    ax[:, 0] += L                                            # lateral distance exactly k * 0.5
    ax[:, 3:] = s2r[:240, 3:]
    hd = synth.hash_uniform(73, 1, np.arange(240)) * 2 * np.pi
    dg = b1.copy()
    dg[:, 0] += L * np.cos(hd)                               # k * 0.5 up to rounding: either side of the boundary
    dg[:, 1] += L * np.sin(hd)
    dg[:, 3:] = s2r[240:480, 3:]
    z = base[:40]
    turn = z.copy()
    turn[:, 3:] = np.stack(synth.quat_from_rpy(np.zeros(40), np.zeros(40), np.linspace(-3.0, 3.0, 40)), 1)
    neg = s2r[:200].copy()
    neg[:, 3:] = -neg[:, 3:]                                 # same rotation, negative dot product with s1
    out1 = base[:100].copy()
    k = np.arange(100)
    out1[:, 0] = np.where(k % 2 == 0, 1.0, -1.0) * (4.3 + 1.5 * synth.hash_uniform(74, 1, k))
    out2 = out1.copy()
    out2[:, 0] -= np.sign(out1[:, 0]) * 2.0 * synth.hash_uniform(74, 2, k)
    out2[:, 3:] = s2r[500:600, 3:]
    s1 = np.concatenate([s1r, b1, b1, z, z, s1r[:200], out1])
    s2 = np.concatenate([s2r, ax, dg, z, turn, neg, out2])
    return np.ascontiguousarray(s1), np.ascontiguousarray(s2)


def make_obj(m, sd, thr):
    import art_planner_b200 as ap
    from art_planner_b200.checker import _Handle
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, handle=_Handle(synth.PARAMS_YAML, 0, risk_threshold=thr))
    chk.setMap(m)
    chk.updateHeightField()
    obj = ap.MotionCostObjective(chk)
    obj.setWeights(sd)
    obj.updateFeatures()
    return obj


def device_run(obj, s1, s2, total):
    import torch
    rows = torch.empty((total, 6), dtype=torch.float32, device="cuda")
    c3 = torch.empty((total, 3), dtype=torch.float32, device="cuda")
    cost = obj.motionCostBatch(torch.from_numpy(s1).cuda(), torch.from_numpy(s2).cuda(), rows=rows, cost3=c3)
    torch.cuda.synchronize()
    return cost.cpu().numpy(), rows.cpu().numpy(), c3.cpu().numpy()


@pytest.fixture(scope="module")
def env():
    from art_planner_b200 import build
    build.build()
    m = cases.c4_map()
    sd = costnet.make_state_dict(seed=5)
    s1, s2 = edge_set(m)
    rows, off = split_rows(s1, s2)
    obj = make_obj(m, sd, THR)
    cost, drows, c3 = device_run(obj, s1, s2, int(off[-1]))
    return dict(m=m, sd=sd, s1=s1, s2=s2, rows=rows, off=off, obj=obj, cost=cost, drows=drows, c3=c3)


def test_edge_set_covers_the_cases(env):
    s1, s2, off = env["s1"], env["s2"], env["off"]
    pieces = np.diff(off)
    assert set(range(1, 7)) <= set(pieces.tolist())
    assert (pieces[3000:3240] == np.tile(np.arange(2, 8), 40)).all()       # exact multiples: L / 0.5 + 1 pieces
    dq = (s1[:, 3:] * s2[:, 3:]).sum(1)
    assert (dq < 0).sum() > 100 and (np.abs(s1[:, 0]) > 4.3).sum() >= 100


def test_sum_and_threshold_are_exact(env):
    cost, c3, off, obj = env["cost"], env["c3"], env["off"], env["obj"]
    assert np.array_equal(cost, reduce_costs(c3, off, THR))
    assert np.array_equal(obj.costQuery(env["drows"]), c3)          # the pieces went through the unchanged head
    fin = np.isfinite(cost)
    assert 0 < fin.sum() < len(cost)


def test_rows_match_the_restatement(env):
    assert np.array_equal(env["drows"], env["rows"])


def test_host_and_device_entry_points_agree(env):
    import torch
    obj, s1, s2 = env["obj"], env["s1"], env["s2"]
    host = obj.motionCostBatch(s1, s2)
    assert obj._c.stats()["last_launches"] == 3
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        dev = obj.motionCostBatch(torch.from_numpy(s1).cuda(), torch.from_numpy(s2).cuda())
    st.synchronize()
    assert obj._c.stats()["last_launches"] == 3
    assert np.array_equal(host, dev.cpu().numpy()) and np.array_equal(host, env["cost"])
    for i in (0, 3000, 3500, 3800):
        assert obj.motionCost(s1[i], s2[i]) == host[i]


def test_against_the_fp32_reference_module(env):
    from oracle.cnn_oracle import CostNetOracle, cnn_input_from_layer
    m, off, c3 = env["m"], env["off"], env["c3"]
    net = CostNetOracle(env["sd"])
    lx, ly = m.length
    ref = net.query(net.features(cnn_input_from_layer(m.elevation)), env["rows"], m.res, lx, ly, m.cx, m.cy)
    assert np.allclose(c3, ref, rtol=RTOL, atol=ATOL), float(np.abs(c3 - ref).max())
    want = reduce_costs(ref, off, THR)
    got = env["cost"]
    for e in range(len(got)):
        if np.isinf(want[e]) or np.isinf(got[e]):
            # a risk within 1e-4 of the threshold may fall either way
            r = ref[off[e]:off[e + 1], 2]
            assert np.isinf(want[e]) == np.isinf(got[e]) or np.abs(r - THR).min() < 1e-4 * THR + 1e-5, e
        else:
            assert abs(got[e] - want[e]) <= 1e-4 * abs(want[e]) + 1e-5, (e, got[e], want[e])


def test_threshold_boundary(env):
    off, c3 = env["off"], env["c3"]
    single = np.nonzero(np.diff(off) == 1)[0]
    risks = c3[off[single], 2]
    order = np.argsort(risks, kind="stable")
    mid = single[order[len(order) // 2]]
    thr = float(c3[off[mid], 2])                            # exactly a piece's float risk
    obj = make_obj(env["m"], env["sd"], thr)
    cost, _, c3b = device_run(obj, env["s1"], env["s2"], int(off[-1]))
    assert c3b[off[mid], 2] == np.float32(thr)
    assert np.isfinite(cost[mid])                           # risk == threshold is feasible
    above = single[c3b[off[single], 2] > np.float32(thr)]
    just = above[np.argmin(c3b[off[above], 2])]             # the smallest risk above the threshold
    assert np.isinf(cost[just])
    assert np.array_equal(cost, reduce_costs(c3b, off, thr))
    assert 0 < np.isfinite(cost).sum() < len(cost)


def _walk(m, n, seed):
    k = np.arange(n)
    step = 0.2 + 1.3 * synth.hash_uniform(seed, 1, k)
    hd = synth.hash_uniform(seed, 2, k) * 2 * np.pi
    lim = 0.45 * m.length[0]
    x, y = np.zeros(n), np.zeros(n)
    for i in range(1, n):
        x[i] = np.clip(x[i - 1] + step[i] * np.cos(hd[i]), -lim, lim)
        y[i] = np.clip(y[i - 1] + step[i] * np.sin(hd[i]), -lim, lim)
    return synth.make_terrain_poses(m, n, seed, xy=(x, y))


def test_path_cost(env):
    import torch
    m, sd = env["m"], env["sd"]
    path = _walk(m, 200, 81)
    rows, off = split_rows(path[:-1], path[1:])
    feasible = make_obj(m, sd, 1.0)                          # risk = 1 - p <= 1: every piece feasible
    seg, _, c3 = device_run(feasible, path[:-1], path[1:], int(off[-1]))
    assert np.isfinite(seg).all()
    want = 0.0
    for v in seg.tolist():
        want += v
    assert feasible.pathCost(path) == want
    assert feasible.pathCost(torch.from_numpy(path).cuda()) == want
    assert feasible.pathCost(path[:1]) == 0.0 and feasible.pathCost(np.zeros((0, 7))) == 0.0
    risky = make_obj(m, sd, float(np.median(c3[:, 2])))     # half the pieces too risky
    seg = risky.motionCostBatch(path[:-1], path[1:])
    assert np.isinf(seg).any() and np.isinf(risky.pathCost(path))


def test_errors(env):
    import torch
    import art_planner_b200 as ap
    from art_planner_b200 import capi
    m, s1, s2 = env["m"], env["s1"][:8], env["s2"][:8]
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    obj = ap.MotionCostObjective(chk)
    t1, t2 = torch.from_numpy(s1).cuda(), torch.from_numpy(s2).cuda()
    for a, b in ((s1, s2), (t1, t2)):
        with pytest.raises(ap.ArtpError) as e:
            obj.motionCostBatch(a, b)                       # no weights
        assert e.value.code == capi.ARTP_E_NOWEIGHTS
    obj.setWeights(env["sd"])
    for a, b in ((s1, s2), (t1, t2)):
        with pytest.raises(ap.ArtpError) as e:
            obj.motionCostBatch(a, b)                       # no features
        assert e.value.code == capi.ARTP_E_NOWEIGHTS
    obj.updateFeatures()
    for a, b in ((s1, s2), (t1, t2)):
        for bad in (0.0, -0.5):
            with pytest.raises(ap.ArtpError) as e:
                obj.motionCostBatch(a, b, max_query_edge_length=bad)
            assert e.value.code == capi.ARTP_E_INVALID
    for length, count in ((1.5e9, 2), (3e9, 1)):           # 2 x (3e9 + 1) pieces; one edge with n_interp >= 2^32
        far = s1[:count].copy()
        far[:, 0] += length
        for a, b in ((s1[:count], far), (t1[:count].contiguous(), torch.from_numpy(far).cuda())):
            with pytest.raises(ap.ArtpError) as e:
                obj.motionCostBatch(a, b)
            assert e.value.code == capi.ARTP_E_INVALID
    assert obj.motionCostBatch(s1[:0], s2[:0]).shape == (0,)
    assert obj.motionCostBatch(t1[:0], t2[:0]).shape == (0,)
    assert obj.motionCostBatch(s1, s2).shape == (8,)         # the handle is still usable


def test_scale_on_the_1000_map():
    """200 k edges on the 1000 x 1000 map (feature map 476 x 476): the head's 128-thread configuration, a multi-block
    reduce; rows and costs match the restatement on a strided subset."""
    m = synth.make_fbm_map(1000, 1000, 0.04, seed=2, amp=0.6)
    sd = costnet.make_state_dict(seed=5)
    obj = make_obj(m, sd, THR)
    s1, s2 = synth.make_edges(m, 200_000, seed=91, dmin=0.0, dmax=3.0)
    dx, dy = s2[:, 0] - s1[:, 0], s2[:, 1] - s1[:, 1]
    off = np.zeros(len(s1) + 1, np.int64)
    off[1:] = np.cumsum((np.sqrt(dx * dx + dy * dy) / 0.5).astype(np.int64) + 1)
    total = int(off[-1])
    assert total > 132 * 128
    cost, rows, c3 = device_run(obj, s1, s2, total)
    sel = np.arange(0, len(s1), 97)
    want_rows, sub_off = split_rows(s1[sel], s2[sel])
    idx = np.concatenate([np.arange(off[e], off[e + 1]) for e in sel])
    assert np.array_equal(rows[idx], want_rows)
    assert np.array_equal(cost[sel], reduce_costs(c3[idx], sub_off, THR))
    assert np.array_equal(obj.motionCostBatch(s1, s2), cost)


def test_cpp_mirror_batch_equals_per_edge(env, tmp_path):
    from art_planner_b200 import capi
    libdir = os.path.dirname(capi.LIB_PATH)
    exe = str(tmp_path / "motion_cost_batch")
    subprocess.run(["g++", "-std=c++14", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_cpp", "motion_cost_batch.cpp"), "-o", exe,
                    "-L", libdir, "-l:libartp.so", f"-Wl,-rpath,{libdir}"], check=True)
    m, s1, s2 = env["m"], env["s1"], env["s2"]
    path = _walk(m, 200, 82)
    blob = costnet.pack_blob(env["sd"]).astype(np.float32)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("5i", m.rows, m.cols, len(s1), len(path), blob.size))
        f.write(struct.pack("4d", m.res, m.cx, m.cy, THR))
        f.write(np.asfortranarray(m.elevation).tobytes(order="F"))
        f.write(np.asfortranarray(m.elevation_masked).tobytes(order="F"))
        f.write(s1.tobytes()); f.write(s2.tobytes()); f.write(path.tobytes()); f.write(blob.tobytes())
    r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = np.fromfile(fout, np.uint8)
    n, ns = len(s1), len(path) - 1
    v = np.frombuffer(raw.tobytes(), np.float64, 3 * n + ns + 3)
    single, batch, seg = v[:n], v[n:2 * n], v[2 * n:2 * n + ns]
    path_cost, one_state, empty = v[2 * n + ns:2 * n + ns + 3]
    custom = np.frombuffer(raw.tobytes(), np.float64, n, 8 * (2 * n + ns + 3))
    calls = int(np.frombuffer(raw.tobytes(), np.uint64, 1, 8 * (3 * n + ns + 3))[0])
    assert np.array_equal(batch, single)
    assert np.array_equal(batch, env["cost"])               # the C++ mirror's call is the Python mirror's call
    want = 0.0
    for c in seg.tolist():
        want += c
    assert path_cost == want or (np.isnan(want) and np.isnan(path_cost))
    assert one_state == 0.0 and empty == 0.0
    assert np.array_equal(custom, single) and calls == n
