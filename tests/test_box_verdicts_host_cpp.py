"""The box verdicts of the C++ host mirror (include/artp_host.hpp: StateValidityChecker::boxVerdicts and boxVerdictLayer):
compiles with plain g++ (CPU suite), fails loudly without a GPU, and on the GPU returns the Python mirror's words
(tests/host_cpp/box_verdicts.cpp)."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import box_verdict_cases as bvc
import heading_layer_cases as hlc
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
    exe_path = str(tmp_path_factory.mktemp("host_cpp") / "box_verdicts")
    subprocess.run(["g++", "-std=c++14", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_cpp", "box_verdicts.cpp"), "-o", exe_path,
                    "-L", libdir, "-l:libartp.so", f"-Wl,-rpath,{libdir}"], check=True)
    return exe_path


def test_box_verdicts_mirror_compiles_and_fails_loudly_without_gpu(exe):
    import torch
    r = subprocess.run([exe, "--expect-no-gpu"], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert r.returncode == 3
    else:
        assert r.returncode == 0 and "failed loudly" in r.stdout and "CUDA" in r.stdout


@pytest.mark.gpu
def test_box_verdicts_mirror_matches_python_mirror(exe, tmp_path):
    import art_planner_b200 as ap
    m = hlc.MAPS["r1"]()
    states = bvc.samples(m)
    yaw = 0.8
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("3i", m.rows, m.cols, len(states)))
        f.write(struct.pack("4d", m.res, m.cx, m.cy, yaw))
        f.write(np.asfortranarray(m.elevation, dtype=np.float32).tobytes(order="F"))
        f.write(np.asfortranarray(m.elevation_masked, dtype=np.float32).tobytes(order="F"))
        f.write(np.ascontiguousarray(states, dtype=np.float64).tobytes())
    r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.fromfile(fout, np.uint16)
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    chk.estimateNormals(hlc.normal_radius(synth.PARAMS_YAML), want_host=False)
    want_why = chk.boxVerdicts(states)
    want_layer = chk.boxVerdictLayer(yaw)
    assert np.array_equal(got[:len(states)], want_why)
    assert np.array_equal(got[len(states):].reshape((m.rows, m.cols), order="F"), want_layer)
    assert ((want_why & 0x1F) == 0).any() and ((want_layer & 0x1F) != 0).any()
