"""The C++ host mirror's PathSimplifier (include/artp_host.hpp): compiles with plain g++ (CPU suite), fails loudly without a
GPU, and on the GPU returns for one solved query what the Python mirror's getSolutionPath returns
(tests/host_cpp/path_simplify.cpp)."""
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
    exe_path = str(tmp_path_factory.mktemp("host_cpp") / "path_simplify")
    subprocess.run(["g++", "-std=c++14", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_cpp", "path_simplify.cpp"), "-o", exe_path,
                    "-L", libdir, "-l:libartp.so", f"-Wl,-rpath,{libdir}"], check=True)
    return exe_path


def test_path_simplifier_mirror_compiles_and_fails_loudly_without_gpu(exe):
    import torch
    r = subprocess.run([exe, "--expect-no-gpu"], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert r.returncode == 3
    else:
        assert r.returncode == 0 and "failed loudly" in r.stdout and "CUDA" in r.stdout


@pytest.mark.gpu
def test_path_simplifier_mirror_matches_python_mirror(exe, tmp_path):
    import art_planner_b200 as ap
    import roadmap_cases as rc
    import test_path_simplify_gpu as tg
    from art_planner_b200 import capi
    c = rc.make_case("rough_fbm")
    env, paths = tg.solved_paths(c, 1, seed=106)
    assert paths
    path = paths[0]
    m, rp, space, seed = c.m, c.rp, env.space, 23
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("5i", m.rows, m.cols, len(path), int(rp.unknown_space_untraversable), int(rp.use_directional_cost)))
        f.write(struct.pack("3d", m.res, m.cx, m.cy))
        f.write(struct.pack("15d", rp.torso_length, rp.torso_width, rp.torso_height, rp.torso_off_x, rp.torso_off_y,
                            rp.torso_off_z, rp.feet_off_x, rp.feet_off_y, rp.feet_off_z, rp.reach_x, rp.reach_y, rp.reach_z,
                            rp.max_lon_vel, rp.max_lat_vel, rp.max_ang_vel))
        f.write(struct.pack("7d", *space.low, *space.high, space.longest_valid_segment_fraction))
        f.write(struct.pack("Q", seed))
        f.write(np.asfortranarray(m.elevation, dtype=np.float32).tobytes(order="F"))
        f.write(np.asfortranarray(m.elevation_masked, dtype=np.float32).tobytes(order="F"))
        f.write(np.ascontiguousarray(path, np.float64).tobytes())
    r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(fout, "rb").read()
    n, = struct.unpack_from("Q", raw)
    got = np.frombuffer(raw, np.float64, n * 7, 8).reshape(n, 7)
    info = capi.ArtpSimplifyInfo.from_buffer_copy(raw, 8 + n * 56)
    # the Python mirror on the same handle kind, map, objective and stream
    ref, rinfo = ap.PathSimplifier(env.chk, space, "path_length", seed).getSolutionPath(path)
    assert np.array_equal(got, ref)
    for k, _ in capi.ArtpSimplifyInfo._fields_:
        a, b = getattr(info, k), rinfo[k]
        assert a == b or (np.isnan(a) and np.isnan(b)), k
    assert info.n_in == len(path) and info.reduce_edits + info.collapse_edits + info.shortcut_edits + info.bspline_edits > 0
