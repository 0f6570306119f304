"""CPU-only: the C-ABI library loads and exports every symbol include/artp.h declares (no compute calls)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    txt = open(os.path.join(ROOT, "include", "artp.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(artp_[a-z_0-9]+)\s*\(", txt)))


@pytest.fixture(scope="module")
def lib():
    from art_planner_b200 import build, capi
    if not os.path.exists(capi.LIB_PATH):
        if shutil.which("nvcc") is None:
            pytest.skip("libartp.so not built and nvcc absent")
        build.build()
    return ctypes.CDLL(capi.LIB_PATH)


def test_header_declares_the_expected_entry_points():
    syms = declared_symbols()
    for s in ("artp_create", "artp_destroy", "artp_set_map", "artp_check_poses", "artp_check_motions",
              "artp_path_length_cost", "artp_last_error"):
        assert s in syms


def test_library_exports_every_declared_symbol(lib):
    for s in declared_symbols():
        assert hasattr(lib, s), f"libartp.so does not export {s}"


def test_library_exports_only_the_declared_functions(lib):
    """Kernels, C++ helpers and template instantiations stay inside libartp.so: its dynamic symbol table holds exactly
    the functions include/artp.h declares."""
    from art_planner_b200 import capi
    nm = shutil.which("nm")
    assert nm is not None, "nm (binutils) is needed to read the library's symbol table"
    out = subprocess.run([nm, "-D", "--defined-only", capi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert exported == set(declared_symbols())


def test_product_path_fails_loudly_without_gpu(lib):
    """No CPU fallback: without a CUDA device artp_create must fail with ARTP_E_CUDA (on a GPU box it succeeds)."""
    import torch
    from art_planner_b200 import capi, synth
    capi.load()
    p = capi.make_params(synth.PARAMS_YAML)
    h = ctypes.c_void_p()
    rc = capi.load().artp_create(ctypes.byref(p), ctypes.byref(h))
    if torch.cuda.is_available():
        assert rc == 0
        capi.load().artp_destroy(h)
    else:
        assert rc == capi.ARTP_E_CUDA
        assert b"CUDA" in capi.load().artp_last_error(None) or b"device" in capi.load().artp_last_error(None)


def test_product_package_never_uses_the_oracle():
    """The oracle is test infrastructure: nothing under art_planner_b200/ or include/ may import, link or call it."""
    bad = ("import oracle", "from oracle", "liborc", "orc_", "artp_oracle", "artp_wrappers")
    for top in ("art_planner_b200", "include"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, top)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                    txt = open(os.path.join(dirpath, f)).read()
                    for b in bad:
                        assert b not in txt, f"{f} mentions {b}"
