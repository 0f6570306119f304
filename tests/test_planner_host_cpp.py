"""The C++ host mirror's Planner (include/artp_host.hpp): compiles with plain g++ (CPU suite), fails loudly without a GPU,
and on the GPU returns for one replan the path and info the Python mirror returns (tests/host_cpp/planner.cpp)."""
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
    exe_path = str(tmp_path_factory.mktemp("host_cpp") / "planner")
    subprocess.run(["g++", "-std=c++14", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_cpp", "planner.cpp"), "-o", exe_path,
                    "-L", libdir, "-l:libartp.so", f"-Wl,-rpath,{libdir}"], check=True)
    return exe_path


def test_planner_mirror_compiles_and_fails_loudly_without_gpu(exe):
    import torch
    r = subprocess.run([exe, "--expect-no-gpu"], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert r.returncode == 3
    else:
        assert r.returncode == 0 and "failed loudly" in r.stdout and "CUDA" in r.stdout


@pytest.mark.gpu
def test_planner_mirror_matches_python_mirror(exe, tmp_path):
    import ctypes as C
    import art_planner_b200 as ap
    import planner_cases as pc
    import roadmap_cases as rc
    import test_planner_gpu as tg
    from art_planner_b200 import capi, costnet
    from art_planner_b200.checker import _Handle
    c = rc.make_case("gentle_inf")
    m, rp = c.m, c.rp
    pp = pc.small_params(seed=19)
    sd = costnet.make_state_dict(seed=5)
    chk = ap.StateValidityChecker(rp, handle=_Handle(rp, 0, risk_threshold=0.6))
    ap.MotionCostObjective(chk).setWeights(sd)
    pl = ap.Planner(chk, pp)
    layers = pc.raw_layers(m)
    pl.setMap(*layers, m.res, m.cx, m.cy)
    start, goal = tg.far_queries(m, 1, seed=71, chk=chk)[0]
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
        for a in layers:
            f.write(np.asfortranarray(a, dtype=np.float32).tobytes(order="F"))
        f.write(struct.pack("Q", blob.size))
        f.write(blob.tobytes())
    r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(fout, "rb").read()
    n, = struct.unpack_from("Q", raw)
    got = np.frombuffer(raw, np.float64, n * 7, 8).reshape(n, 7)
    info = capi.ArtpPlanInfo.from_buffer_copy(raw, 8 + n * 56)
    assert info.status == status
    assert np.array_equal(got, ref_path)
    for k in ("status", "sampled", "first_sample", "draws_used", "start_draw", "goal_draw", "n_vertices", "n_edges",
              "path_cost", "start_index", "goal_index"):
        assert getattr(info, k) == getattr(ref_info, k), k
    for k, _ in capi.ArtpSimplifyInfo._fields_:
        a, b = getattr(info.simplify, k), getattr(ref_info.simplify, k)
        assert a == b or (np.isnan(a) and np.isnan(b)), k
    assert list(info.start_repaired) == list(ref_info.start_repaired)
    assert list(info.goal_repaired) == list(ref_info.goal_repaired)
