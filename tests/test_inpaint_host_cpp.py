"""The C++ host mirror's inpaintMatrix and raw-layer Planner::setMap (include/artp_host.hpp): compile with plain g++ (CPU
suite), fail loudly without a GPU, and on the GPU return what the Python mirror returns: the inpainted layers
(StateValidityChecker.inpaint) and, after Planner.setMapRaw, the path and info of one replan (tests/host_cpp/inpaint.cpp)."""
import ctypes
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    """The driver, compiled into a temporary directory: the source tree may be read-only."""
    from art_planner_b200 import build, capi
    if not os.path.exists(capi.LIB_PATH):
        if shutil.which("nvcc") is None:
            pytest.skip("libartp.so not built and nvcc absent")
        build.build()
    libdir = os.path.dirname(capi.LIB_PATH)
    exe_path = str(tmp_path_factory.mktemp("host_cpp") / "inpaint")
    subprocess.run(["g++", "-std=c++14", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_cpp", "inpaint.cpp"), "-o", exe_path,
                    "-L", libdir, "-l:libartp.so", f"-Wl,-rpath,{libdir}"], check=True)
    return exe_path


def test_inpaint_mirror_compiles_and_fails_loudly_without_gpu(exe):
    import torch
    r = subprocess.run([exe, "--expect-no-gpu"], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert r.returncode == 3
    else:
        assert r.returncode == 0 and "failed loudly" in r.stdout and "CUDA" in r.stdout


@pytest.mark.gpu
def test_inpaint_mirror_matches_python_mirror(exe, tmp_path):
    import art_planner_b200 as ap
    import planner_cases as pc
    import roadmap_cases as rc
    import test_planner_gpu as tg
    from art_planner_b200 import capi, costnet
    from art_planner_b200.checker import _Handle
    from oracle import planner_oracle as po
    c = rc.make_case("gentle_inf")
    m, rp = c.m, c.rp
    pp = pc.small_params(seed=19)
    sd = costnet.make_state_dict(seed=5)
    chk = ap.StateValidityChecker(rp, handle=_Handle(rp, 0, risk_threshold=0.6))
    ap.MotionCostObjective(chk).setWeights(sd)
    raw_e, raw_t, _, _ = pc.raw_layers(m, holes=0.02)
    ei, ti = chk.inpaint(raw_e), chk.inpaint(raw_t)
    qchk = ap.StateValidityChecker(rp, handle=_Handle(rp, 0, risk_threshold=0.6))
    ap.Planner(qchk, pp).setMap(raw_e, raw_t, ei, ti, m.res, m.cx, m.cy)   # a map for the query search
    start, goal = tg.far_queries(m, 1, seed=71, chk=qchk)[0]
    pl = ap.Planner(chk, pp)
    ref_map = pl.setMapRaw(raw_e, raw_t, m.res, m.cx, m.cy)
    status = pl.plan(start, goal)
    ref_info = capi.ArtpPlanInfo.from_buffer_copy(bytes(pl._info))
    ref_path = pl._path
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    blob = costnet.pack_blob(sd).astype(np.float32)
    with open(fin, "wb") as f:
        f.write(struct.pack("2i", m.rows, m.cols))
        f.write(struct.pack("3d", m.res, m.cx, m.cy))
        f.write(struct.pack("12d", rp.torso_length, rp.torso_width, rp.torso_height, rp.torso_off_x, rp.torso_off_y,
                            rp.torso_off_z, rp.feet_off_x, rp.feet_off_y, rp.feet_off_z, rp.reach_x, rp.reach_y, rp.reach_z))
        f.write(bytes(pp))
        f.write(np.concatenate([start, goal]).astype(np.float64).tobytes())
        for a in (raw_e, raw_t):
            f.write(np.asfortranarray(a, dtype=np.float32).tobytes(order="F"))
        f.write(struct.pack("Q", blob.size))
        f.write(blob.tobytes())
    r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(fout, "rb").read()
    n = m.rows * m.cols
    got_e = np.frombuffer(raw, np.float32, n, 0).reshape(m.cols, m.rows).T
    got_t = np.frombuffer(raw, np.float32, n, 4 * n).reshape(m.cols, m.rows).T
    assert np.array_equal(got_e.view(np.uint32), ei.view(np.uint32))
    assert np.array_equal(got_t.view(np.uint32), ti.view(np.uint32))
    off = 8 * n
    npath, = struct.unpack_from("Q", raw, off)
    got = np.frombuffer(raw, np.float64, npath * 7, off + 8).reshape(npath, 7)
    info = capi.ArtpPlanInfo.from_buffer_copy(raw, off + 8 + npath * 56)
    mi = capi.ArtpPlannerMapInfo.from_buffer_copy(raw, off + 8 + npath * 56 + ctypes.sizeof(capi.ArtpPlanInfo))
    assert info.status == status
    if status == po.SOLVED:
        assert np.array_equal(got, ref_path)
    else:
        assert npath == 0
    for k in ("status", "sampled", "draws_used", "n_vertices", "n_edges", "path_cost", "start_index", "goal_index"):
        assert getattr(info, k) == getattr(ref_info, k), k
    assert list(info.start_repaired) == list(ref_info.start_repaired)
    assert list(info.goal_repaired) == list(ref_info.goal_repaired)
    assert mi.bytes_h2d == ref_map["bytes_h2d"] and mi.host_syncs == ref_map["host_syncs"]

