"""The C++ host mirror's PRMRoadmap (include/artp_host.hpp): compiles with plain g++ (CPU suite), fails loudly without a
GPU, and on the GPU builds the roadmap the Python mirror builds (tests/host_cpp/roadmap.cpp)."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

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
    exe_path = str(tmp_path_factory.mktemp("host_cpp") / "roadmap")
    subprocess.run(["g++", "-std=c++14", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_cpp", "roadmap.cpp"), "-o", exe_path,
                    "-L", libdir, "-l:libartp.so", f"-Wl,-rpath,{libdir}"], check=True)
    return exe_path


def test_roadmap_mirror_compiles_and_fails_loudly_without_gpu(exe):
    import torch
    r = subprocess.run([exe, "--expect-no-gpu"], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert r.returncode == 3
    else:
        assert r.returncode == 0 and "failed loudly" in r.stdout and "CUDA" in r.stdout


@pytest.mark.gpu
def test_roadmap_mirror_matches_python_mirror(exe, tmp_path):
    import art_planner_b200 as ap
    m = synth.make_fbm_map(150, 130, res=0.04, seed=9, cx=1.5, cy=-0.5)
    rp = synth.PARAMS_YAML
    lx, ly = m.length
    low, high = (m.cx - 0.5 * lx, m.cy - 0.5 * ly), (m.cx + 0.5 * lx, m.cy + 0.5 * ly)
    caps, seed = (700, 3000, 200), 77
    q = np.zeros((2, 7)); q[:, 6] = 1.0
    q[:, 0], q[:, 1], q[:, 2] = (m.cx + 0.3, m.cx - 0.4), (m.cy, m.cy + 0.2), (0.4, 0.5)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(fin, "wb") as f:
        f.write(struct.pack("5i", m.rows, m.cols, *caps))
        f.write(struct.pack("7d", m.res, m.cx, m.cy, *low, *high))
        f.write(struct.pack("Q", seed))
        f.write(np.asfortranarray(m.elevation).tobytes(order="F"))
        f.write(np.asfortranarray(m.elevation_masked).tobytes(order="F"))
        f.write(q.tobytes())
    r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(fout, "rb").read()
    used, nv, ne = struct.unpack_from("3Q", raw)
    o = 24
    st = np.frombuffer(raw, np.float64, nv * 7, o).reshape(nv, 7); o += nv * 56
    kinds = np.frombuffer(raw, np.uint8, nv, o); o += nv
    edges = np.frombuffer(raw, np.uint32, 2 * ne, o).reshape(ne, 2)
    # the Python mirror on the same map, robot, sampler and stream
    chk = ap.StateValidityChecker(rp, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    nx, ny, nz, sd = chk.estimateNormals((rp.torso_length + rp.torso_width) * 0.25)
    layers = synth.SamplerLayers(nx, ny, nz, sd, None, None, None)
    sp = synth.SamplerParams(sample_from_distribution=False, low=low, high=high)
    smp = ap.SE3FromSE2Sampler(chk, layers, sp, seed=seed)
    rm = ap.PRMRoadmap(chk, 20000, 40000)
    assert rm.sampleGraph(smp, *caps, max_draws=1 << 24, distribution=False) == used
    rm.addValidMilestones(q)
    pst, pk = rm.vertices()
    assert np.array_equal(pst, st) and np.array_equal(pk, kinds) and np.array_equal(rm.edges(), edges)
    assert (kinds == (ap.PRMRoadmap.MILESTONE | ap.PRMRoadmap.QUERY)).sum() == 2
