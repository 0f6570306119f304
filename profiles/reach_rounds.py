"""The two reach-box kernels of the bench step (configs[1]: 1 M poses on the 1000 x 1000 fBm map), one at a time: stage
timing on (artp_set_timing), so every stage of a round runs alone on the call's stream and its CUDA events time it.
Reports the median of reach_queue_warp (box_tiles_warp_kernel over the reach queue, B) and reach_queue_groups
(reach_groups_kernel, B') over STEPS steps (an L2 flush before each, as bench.py does), their queue lengths from stats(),
the rates per SM (B: boxes/s, B': rounds of four boxes/s), each launch's grid from a short torch.profiler pass (CTAs per
SM = grid / SMs), and the card's name, power limit and max SM clock. --rough runs bench.py's secondary rough level
(c2_rough) instead. Prints one JSON line; with --out DIR it also writes it there."""
import argparse
import json
import os
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

STAGES = ("classify", "torso_queue", "reach_queue_warp", "reach_queue_groups", "group")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power, clock = (x.strip() for x in (q.stdout.strip().split(",") + ["", "", ""])[:3])
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--steps", type=int, default=100)
    ap_.add_argument("--warmup", type=int, default=10)
    ap_.add_argument("--rough", action="store_true", help="the rough level (bench.py's c2_rough) instead of configs[1]")
    ap_.add_argument("--out", default=None, help="directory for reach_rounds.json")
    args = ap_.parse_args()
    assert torch.cuda.is_available(), "reach_rounds.py needs a CUDA device"

    n = bench.POSES_PER_GPU
    if args.rough:
        m = synth.make_fbm_map(bench.MAP_N, bench.MAP_N, bench.MAP_RES, seed=bench.MAP_SEED, **bench.ROUGH_MAP)
        poses = synth.make_terrain_poses(m, n, seed=bench.POSE_SEED, **bench.ROUGH_POSES)
    else:
        m, poses = bench.make_inputs(0, n)
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    chk.setTiming(True)
    d_poses = torch.from_numpy(poses).cuda()
    d_valid = torch.empty(n, dtype=torch.uint8, device="cuda")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    for i in range(args.warmup):
        flush.fill_(i % 255 + 1)
        chk.isValidBatch(d_poses, out=d_valid)
    torch.cuda.synchronize()
    times = []
    for i in range(args.steps):
        flush.fill_(i % 255 + 1)
        chk.isValidBatch(d_poses, out=d_valid)
        times.append(chk.lastStageTimesMs())
        torch.cuda.synchronize()
    st = chk.stats()
    t = np.array(times, dtype=np.float64)
    med = dict(zip(STAGES, (round(float(x), 5) for x in np.median(t, 0))))
    spread = dict(zip(STAGES, (round(float(x), 5) for x in np.percentile(t, 90, 0) - np.percentile(t, 10, 0))))
    q_warp, q_groups = st["last_queued_reach_stage"], st["last_reach_plane_stage"]

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for i in range(3):
            chk.isValidBatch(d_poses, out=d_valid)
        torch.cuda.synchronize()
    raw = os.path.join(args.out or tempfile.mkdtemp(), "reach_rounds.pt.trace.json")
    os.makedirs(os.path.dirname(raw), exist_ok=True)
    prof.export_chrome_trace(raw)
    with open(raw) as f:
        evs = [e for e in json.load(f)["traceEvents"] if e.get("ph") == "X" and e.get("cat") == "kernel"]
    evs.sort(key=lambda e: e["ts"])
    tiles = [e for e in evs if "box_tiles_warp_kernel" in e["name"]]
    groups = [e for e in evs if "reach_groups_kernel" in e["name"]]
    # per call the big-tile launch comes first, the reach-queue launch second
    grid_warp = tiles[1]["args"]["grid"][0] if len(tiles) > 1 else None
    grid_groups = groups[0]["args"]["grid"][0] if groups else None

    ms_w, ms_g = med["reach_queue_warp"], med["reach_queue_groups"]
    res = {
        "card": card(), "workload": "c2_rough" if args.rough else "configs[1]", "sms": sms, "steps": args.steps, "stage_ms_median": med, "stage_ms_p90_minus_p10": spread,
        "reach_warp": {"queued_boxes": q_warp, "ms": ms_w, "grid": grid_warp,
                       "ctas_per_sm": grid_warp / sms if grid_warp else None,
                       "boxes_per_s_per_sm": q_warp / (ms_w * 1e-3) / sms if ms_w > 0 else None},
        "reach_groups": {"queued_boxes": q_groups, "rounds": (q_groups + 3) // 4, "ms": ms_g, "grid": grid_groups,
                         "ctas_per_sm": grid_groups / sms if grid_groups else None,
                         "rounds_per_s_per_sm": (q_groups + 3) // 4 / (ms_g * 1e-3) / sms if ms_g > 0 else None},
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(os.path.join(args.out, "reach_rounds.json"), "w") as f:
            f.write(line + "\n")
        os.remove(raw)


if __name__ == "__main__":
    main()
