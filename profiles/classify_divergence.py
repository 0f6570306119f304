"""Is the classify stage bound by divergence inside its warps?

Classify evaluates an item's boxes in order: reach boxes 1..4, stopping at the first reach box that touches nothing, then
the torso; an evaluated reach box that passes the collider's early outs also runs the vertex probe. When one thread walks
an item's boxes, consecutive bench poses take different paths and a warp runs every box as long as its slowest lane.

This probe times the classify stage (library stage events, L2 flushed before every step) on two 1M-pose inputs of the
bench map (BASELINE configs[1]) that alternate step by step: the bench order, and the same poses sorted by their path
key (number of evaluated boxes, whether any evaluated reach box reaches the probe). The sorted input gives warps whose
lanes agree on their path. The poses, the work and the range-table footprint are the same; the bench poses are drawn
by a hash, so the sort costs no locality. The key comes from the port oracle's per-box exit stages
(`pose_box_stats`: the collider's stage of each box without the pose-level short-circuits).

  python profiles/classify_divergence.py [--steps 30]            # GPU: stage times of both inputs, one JSON line
  python profiles/classify_divergence.py --key-only [--n 65536]  # CPU only: the path statistics of the key
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
sys.dont_write_bytecode = True

import numpy as np

import bench
from art_planner_b200 import synth

# ORC_ST_* exit stages of pose_box_stats
ST_AABB, ST_ABOVE, ST_UNDER, ST_SPAN, ST_PLANE1, ST_OUTSIDE = 0, 1, 2, 3, 4, 255


def path_key(m, poses, threads):
    """Per pose: the number of boxes classify evaluates (1..5) and whether any evaluated reach box passes the early outs
    (and so runs the vertex probe). Restated from the oracle's exit stages; the early outs are the collider's own."""
    from oracle import orc
    chunks = np.array_split(np.arange(len(poses)), threads)

    def run(idx):
        o = orc.Oracle(synth.PARAMS_YAML, "port")
        o.set_map(m)
        return o.pose_box_stats(poses[idx])[:2]
    with ThreadPoolExecutor(threads) as ex:
        res = list(ex.map(run, chunks))
    st = np.concatenate([r[0] for r in res])
    hit = np.concatenate([r[1] for r in res])
    reach_st, reach_hit = st[:, 1:], hit[:, 1:]
    fails = np.isin(reach_st, (ST_AABB, ST_ABOVE, ST_UNDER)) | ((reach_st == ST_PLANE1) & (reach_hit == 0))
    if synth.PARAMS_YAML.unknown_space_untraversable:
        fails |= reach_st == ST_OUTSIDE
    probe = ~np.isin(reach_st, (ST_AABB, ST_ABOVE, ST_UNDER, ST_SPAN, ST_PLANE1, ST_OUTSIDE))
    first_fail = np.where(fails.any(1), fails.argmax(1), 4)          # index of the first failing reach box, 4 = none
    n_eval = np.minimum(first_fail + 1, 4) + (first_fail == 4)       # reach boxes evaluated (+ the torso if none failed)
    evaluated = np.arange(4)[None, :] <= first_fail[:, None]
    any_probe = (probe & evaluated).any(1)
    return n_eval, any_probe, first_fail


def key_stats(n_eval, any_probe, first_fail):
    n = len(n_eval)
    w = n - n % 32
    warp_iters = n_eval[:w].reshape(-1, 32).max(1)
    return {"poses": n,
            "first_failing_reach_box": {str(k + 1): round(float((first_fail == k).mean()), 4) for k in range(4)},
            "torso_evaluated": round(float((first_fail == 4).mean()), 4),
            "mean_evaluated_boxes": round(float(n_eval.mean()), 4),
            "warps_running_all_5": round(float((warp_iters == 5).mean()), 4),
            "lane_efficiency": round(float(n_eval[:w].sum() / (32 * warp_iters.sum())), 4),
            "any_probe": round(float(any_probe.mean()), 4)}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = (x.strip() for x in q.split(","))
        return {"gpu": name, "power_limit": pl, "sm_max_clock": clk}
    except Exception as ex:
        return {"gpu_query_error": repr(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--n", type=int, default=bench.POSES_PER_GPU)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--key-only", action="store_true")
    args = ap.parse_args()
    m, poses = bench.make_inputs(0, args.n)
    n_eval, any_probe, first_fail = path_key(m, poses, args.threads)
    stats = key_stats(n_eval, any_probe, first_fail)
    if args.key_only:
        print(json.dumps(stats))
        return
    order = np.lexsort((any_probe, n_eval))
    sorted_poses = np.ascontiguousarray(poses[order])

    import torch
    import art_planner_b200 as ap_
    assert torch.cuda.is_available(), "needs a CUDA device"
    chk = ap_.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    chk.setTiming(True)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    ins = {"bench_order": torch.from_numpy(poses).cuda(), "sorted_by_path": torch.from_numpy(sorted_poses).cuda()}
    outs = {k: torch.empty(args.n, dtype=torch.uint8, device="cuda") for k in ins}
    for k, d in ins.items():
        for _ in range(3):
            chk.isValidBatch(d, out=outs[k])
    torch.cuda.synchronize()
    same = bool(np.array_equal(outs["bench_order"].cpu().numpy()[order], outs["sorted_by_path"].cpu().numpy()))
    st = {k: [] for k in ins}
    for i in range(args.steps):
        for k, d in ins.items():
            flush.fill_(i & 0xFF)
            chk.isValidBatch(d, out=outs[k])
            st[k].append(chk.lastStageTimesMs())
            torch.cuda.synchronize()
    res = {"key": stats, "verdicts_equal_after_sort": same}
    for k, v in st.items():
        a = np.array(v)[:, 0]
        res[k] = {"classify_ms_median": round(float(np.median(a)), 4),
                  "classify_ms_range": [round(float(a.min()), 4), round(float(a.max()), 4)]}
    res["sorted_over_bench_order"] = round(res["sorted_by_path"]["classify_ms_median"]
                                           / res["bench_order"]["classify_ms_median"], 4)
    res.update(gpu_info())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
