"""The start / goal search of the C++ host mirror (include/artp_host.hpp: StartState, GoalStateRegion, findValidNearBatch,
poseFrom2D): compiles with plain g++ (CPU suite), fails loudly without a GPU, and on the GPU gives the Python mirror's
answers (tests/host_cpp/start_goal.cpp)."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import start_goal_cases as sgc
from art_planner_b200 import synth

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
    exe_path = str(tmp_path_factory.mktemp("host_cpp") / "start_goal")
    subprocess.run(["g++", "-std=c++14", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_cpp", "start_goal.cpp"), "-o", exe_path,
                    "-L", libdir, "-l:libartp.so", f"-Wl,-rpath,{libdir}"], check=True)
    return exe_path


def test_start_goal_mirror_compiles_and_fails_loudly_without_gpu(exe):
    import torch
    r = subprocess.run([exe, "--expect-no-gpu"], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert r.returncode == 3
    else:
        assert r.returncode == 0 and "failed loudly" in r.stdout and "CUDA" in r.stdout


@pytest.mark.gpu
def test_start_goal_mirror_matches_python_mirror(exe, maps, tmp_path):
    import art_planner_b200 as ap
    m = maps("fbm_rough")
    n, n_iter, r_start, r_goal, seeds = 40, 300, 0.2, 0.5, (11, 12)
    starts, _ = sgc.make_queries(m, n, 31)
    goals, _ = sgc.make_queries(m, n, 32)
    off = np.random.default_rng(3).uniform(-r_start, r_start, (n, n_iter, 2))
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("4i", m.rows, m.cols, n, n_iter))
        f.write(struct.pack("5d", m.res, m.cx, m.cy, r_start, r_goal))
        f.write(struct.pack("2Q", *seeds))
        f.write(np.asfortranarray(m.elevation).tobytes(order="F"))
        f.write(np.asfortranarray(m.elevation_masked).tobytes(order="F"))
        f.write(starts.tobytes()); f.write(goals.tobytes()); f.write(off.tobytes())
    r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(fout, "rb").read()
    o = 0

    def take(dtype, count, shape=None):
        nonlocal o
        a = np.frombuffer(raw, dtype, count, o)
        o += a.nbytes
        return a.reshape(shape) if shape else a
    projected, inside = take(np.float64, 7 * n, (n, 7)), take(np.uint8, n)
    s_out, s_idx, s_next = take(np.float64, 7 * n, (n, 7)), take(np.int32, n), take(np.uint64, n)
    g_out, g_idx, g_next = take(np.float64, 7 * n, (n, 7)), take(np.int32, n), take(np.uint64, n)
    b_out, b_idx = take(np.float64, 7 * n, (n, 7)), take(np.int32, n)
    assert o == len(raw)
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    p = synth.PARAMS_YAML
    chk.estimateNormals((p.torso_length + p.torso_width) * 0.25, want_host=False)
    want_p, want_in = chk.poseFrom2D(goals)
    assert np.array_equal(projected, want_p) and np.array_equal(inside, want_in)
    start, goal = ap.StartState(chk, seed=seeds[0]), ap.GoalStateRegion(chk, seed=seeds[1])
    start.setThreshold(r_start); start.setMaxNumSamples(n_iter)
    goal.setThreshold(r_goal); goal.setMaxNumSamples(n_iter)
    for q in range(n):
        start.setState(starts[q])
        st, k = start.sampleGoal()
        assert np.array_equal(st, s_out[q]) and k == s_idx[q] and start.draw == s_next[q]
        goal.setState(want_p[q])
        st, k = goal.sampleGoal()
        assert np.array_equal(st, g_out[q]) and k == g_idx[q] and goal.draw == g_next[q]
    bs, bi = chk.findValidNear(starts, r_start, n_iter, offsets=off)
    assert np.array_equal(bs, b_out) and np.array_equal(bi, b_idx)
    assert (s_idx == 0).any() and (s_idx < 0).any()
