"""Build libartp.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc."""
from __future__ import annotations

import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libartp.so")
# (source, extra flags): the geometric kernels need bit-exact fp32 (no FMA contraction, SURVEY.md section 7);
# the motion-cost network does not.
# The eight units built with these flags all build heights, rows, costs and states that must equal the host's bit for bit.
GEOMETRY_FLAGS = ["-fmad=false", "-Xcompiler", "-fPIC,-ffp-contract=off"]
SOURCES = [("artp_capi.cu", GEOMETRY_FLAGS), ("artp_map.cu", GEOMETRY_FLAGS), ("artp_sampling.cu", GEOMETRY_FLAGS),
           ("artp_cost.cu", GEOMETRY_FLAGS), ("artp_roadmap.cu", GEOMETRY_FLAGS), ("artp_path_simplify.cu", GEOMETRY_FLAGS),
           ("artp_planner.cu", GEOMETRY_FLAGS), ("artp_inpaint.cu", GEOMETRY_FLAGS),
           ("artp_cnn.cu", ["-Xcompiler", "-fPIC"])]
HEADERS = ["artp_internal.h", "artp_device.cuh", "artp_kernels.cuh", "artp_sampler.cuh", "artp_tiles.cuh", "artp_basic.cuh",
           "artp_distribution.cuh", "artp_roadmap.cuh", "artp_roadmap_query.cuh", "artp_inpaint.cuh", "artp.map", os.path.join("..", "..", "include", "artp.h")]
# The library exports the C ABI (artp_*) and nothing else.
VERSION_SCRIPT = os.path.join(CSRC, "artp.map")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17"]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in [x[0] for x in SOURCES] + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    objs = []
    for src, extra in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, os.path.join(CSRC, src)]
        subprocess.run(cmd, check=True)
        objs.append(obj)
    subprocess.run([nvcc, "-shared"] + NVCC_FLAGS[:2] + ["-Xlinker", "--version-script=" + VERSION_SCRIPT, "-o", LIB] + objs,
                   check=True)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
