"""Per-kernel timeline of the bench step (configs[1], N = 1, the calls of bench.py's step_device) in the shipped default:
stage timing off, so the three box kernels of a round run side by side. Warms up, records STEPS steps under torch.profiler
with CUDA activities (an L2 flush before each step, as bench.py does) and prints, per kernel of the step, the median start
and end relative to the end of the classify stage and the median gap before it: its start minus the latest end of any
kernel of the step that started before it (negative: it overlaps one). The two box_tiles_warp_kernel launches are told
apart by launch order (the trace's correlation id): the big-tile queue's launch comes first, the reach queue's second.
Prints one JSON line with the card's name and power limit; with --out DIR it also writes it, and the raw trace, there."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import art_planner_b200 as ap  # noqa: E402
from art_planner_b200 import synth  # noqa: E402
import bench  # noqa: E402

KERNELS = ["classify_items_kernel", "box_tiles_warp_kernel", "reach_groups_kernel", "box_items_block_kernel",
           "pack_bits_kernel", "compact_"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(",")
    return {"name": name.strip(), "power_limit": power.strip()}


def label(ev, big_corr):
    n = ev["name"]
    for k in KERNELS:
        if k in n:
            if k == "box_tiles_warp_kernel":
                return "box_tiles_warp_kernel[big]" if ev["args"].get("correlation") in big_corr else "box_tiles_warp_kernel[reach]"
            if k == "compact_":   # the compaction kernel(s), by name
                return re.search(r"compact_\w+", n).group(0)
            return k
    return None


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--steps", type=int, default=50)
    ap_.add_argument("--warmup", type=int, default=10)
    ap_.add_argument("--out", default=None, help="directory for step_trace.json and the raw chrome trace")
    args = ap_.parse_args()
    assert torch.cuda.is_available(), "step_trace.py needs a CUDA device"

    n = bench.POSES_PER_GPU
    m, poses = bench.make_inputs(0, n)
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    chk.setTiming(False)
    d_poses = torch.from_numpy(poses).cuda()
    d_valid = torch.empty(n, dtype=torch.uint8, device="cuda")
    bits = torch.empty(n // 32, dtype=torch.int32, device="cuda")
    idx = torch.empty(n, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")

    def step():
        chk.isValidBatchBits(d_poses, d_valid, bits)
        chk.compactValidU32(d_valid, base=0, out_idx=idx, out_cnt=cnt)

    for i in range(args.warmup):
        flush.fill_(i % 255 + 1)
        step()
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for i in range(args.steps):
            flush.fill_(i % 255 + 1)   # never 0: a zero fill may become a memset, which would blur the step boundary
            step()
        torch.cuda.synchronize()
    out_dir = args.out or tempfile.mkdtemp()
    os.makedirs(out_dir, exist_ok=True)
    raw = os.path.join(out_dir, "step_trace.pt.trace.json")
    prof.export_chrome_trace(raw)
    with open(raw) as f:
        evs = [e for e in json.load(f)["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset")]
    evs.sort(key=lambda e: e["ts"])
    cls = [e for e in evs if "classify_items_kernel" in e["name"]]
    assert len(cls) == args.steps, f"{len(cls)} classify launches for {args.steps} steps"
    tiles = [e for e in evs if "box_tiles_warp_kernel" in e["name"]]
    cs = set()   # correlation ids of the big-tile launches: the first of each step's two
    for i, c in enumerate(cls):
        nxt = cls[i + 1]["ts"] if i + 1 < len(cls) else float("inf")
        cs.add(min(e["args"]["correlation"] for e in tiles if c["ts"] <= e["ts"] < nxt))
    rows = {}
    spans = []
    for i, c in enumerate(cls):
        t_end_cls = c["ts"] + c["dur"]
        nxt = cls[i + 1]["ts"] if i + 1 < len(cls) else float("inf")
        mset = [e for e in evs if e["cat"] == "gpu_memset" and e["ts"] < c["ts"]]
        step_evs = [e for e in evs if e["cat"] == "kernel" and c["ts"] <= e["ts"] < nxt and label(e, cs)]
        started = []
        for e in step_evs:
            k = label(e, cs)
            s0, s1 = e["ts"] - t_end_cls, e["ts"] + e["dur"] - t_end_cls
            gap = e["ts"] - max((p["ts"] + p["dur"] for p in started), default=e["ts"])
            started.append(e)
            rows.setdefault(k, []).append((s0, s1, e["dur"], gap if k != "classify_items_kernel" else 0.0, e["args"].get("grid")))
        t0 = mset[-1]["ts"] if mset else c["ts"]
        spans.append(max(e["ts"] + e["dur"] for e in step_evs) - t0)
    kern = {}
    for k, v in rows.items():
        a = np.array([r[:4] for r in v], dtype=np.float64)
        med = np.median(a, axis=0)
        kern[k] = {"launches_per_step": len(v) / len(cls), "start_us": round(float(med[0]), 2), "end_us": round(float(med[1]), 2),
                   "dur_us": round(float(med[2]), 2), "gap_before_us": round(float(med[3]), 2), "grid": v[-1][4]}
    res = {"card": card(), "steps": len(cls), "times": "median us relative to the end of classify_items_kernel",
           "step_span_us": round(float(np.median(spans)), 2), "kernels": kern,
           "last_deferred": chk.stats()["last_deferred"]}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(os.path.join(args.out, "step_trace.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
