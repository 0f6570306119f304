"""Time the valid-heading layer (artp_valid_heading_layer[_device]) on the benchmark's configs[1] maps (1000 x 1000 at
0.04 m, gentle and rough) at 8, 16 and 32 headings, against the composition a caller has without it: artp_pose_from_2d
(host buffers) and artp_check_poses_f32_device over the same chunks of whole cells, packed on the host. Both routes must
give the same masks. Prints one JSON line with the card's name and power limit, read in the same run.

    python profiles/heading_layer_time.py [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import heading_layer_cases as hlc  # noqa: E402
from art_planner_b200 import synth  # noqa: E402

CHUNK = 1 << 21          # poses per chunk, as the layer chunks them


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                         # the name from torch alone
        q = f"{torch.cuda.get_device_name(0)}, power limit unread ({e})"
    return q


def composed(chk, m, yaws):
    """artp_pose_from_2d + artp_check_poses_f32_device per chunk of whole cells; masks packed on the host."""
    import torch
    n = len(yaws)
    cells_per = CHUNK // n
    ncell = m.rows * m.cols
    out = np.empty(ncell, np.uint32)
    valid = torch.empty(cells_per * n, dtype=torch.uint8, device="cuda")
    for c0 in range(0, ncell, cells_per):
        cells = np.arange(c0, min(ncell, c0 + cells_per))
        proj, _ = chk.poseFrom2D(hlc.yaw_states(m, yaws, cells))
        d = torch.from_numpy(proj.astype(np.float32)).cuda()
        v = chk.isValidBatch(d, out=valid[:len(proj)])
        out[c0:c0 + len(cells)] = hlc.pack(v.cpu().numpy(), n, (-1,))
    return out.reshape((m.rows, m.cols), order="F")


def main() -> None:
    import torch
    import art_planner_b200 as ap
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--reps", type=int, default=5)
    a = ap_.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    res = {"card": card(), "maps": "configs[1]: fBm 1000x1000@0.04m seed 2 (gentle amp 0.6 m; rough amp 1.2 m, wavelength 3, "
           "persistence 0.7), yaml robot", "reps": a.reps, "runs": []}
    for kind in ("gentle", "rough"):
        m = hlc.large_map(kind)
        chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
        chk.setMap(m)
        chk.updateHeightField()
        chk.estimateNormals(hlc.normal_radius(synth.PARAMS_YAML), want_host=False)
        for n in (8, 16, 32):
            yaws = np.linspace(-np.pi, np.pi, n, endpoint=False)
            poses = m.rows * m.cols * n
            d_out = torch.empty((m.cols, m.rows), dtype=torch.int32, device="cuda").t()
            chk.validHeadingLayer(yaws, out=d_out)                 # warm-up: scratch, modules
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            for _ in range(a.reps):
                chk.validHeadingLayer(yaws, out=d_out)
            ev[1].record()
            torch.cuda.synchronize()
            dev_ms = ev[0].elapsed_time(ev[1]) / a.reps
            host = chk.validHeadingLayer(yaws)
            t0 = time.perf_counter()
            for _ in range(a.reps):
                host = chk.validHeadingLayer(yaws)
            host_ms = (time.perf_counter() - t0) * 1e3 / a.reps
            assert np.array_equal(d_out.cpu().numpy().view(np.uint32), host)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            comp = composed(chk, m, yaws)
            torch.cuda.synchronize()
            comp_ms = (time.perf_counter() - t0) * 1e3
            assert np.array_equal(comp, host), f"{kind} n={n}: the routes differ"
            res["runs"].append({"map": kind, "n_yaw": n, "poses": poses, "device_ms": round(dev_ms, 3),
                                "device_poses_per_s": float(f"{poses / dev_ms * 1e3:.3g}"), "host_call_ms": round(host_ms, 3),
                                "host_poses_per_s": float(f"{poses / host_ms * 1e3:.3g}"), "composition_ms": round(comp_ms, 1),
                                "composition_poses_per_s": float(f"{poses / comp_ms * 1e3:.3g}"),
                                "valid_share": round(float(np.bitwise_count(host).mean()) / n, 4), "masks_equal": True})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
