"""What fills the one-warp-per-box reach queue (box_tiles_warp_kernel over the reach boxes, B) after one call, on configs[1]
(the bench step), on bench.py's rough level (c2_rough) and on configs[4] (the 4000 x 4000 map, one GPU): the lengths of
the three box queues from stats(), and the records of the reach queue read back from the device (debugReachQueue), counted
by flag class (BoxRec.flags, artp_kernels.cuh):
  non_finite      the zone holds a -inf height (REC_ALLFINITE clear, REC_NEEDS_REDUCE clear)
  needs_reduce    the range tables did not reduce the zone (REC_NEEDS_REDUCE)
  not_merge_free  the plane tables found two triangles of the zone in one plane (REC_MERGEFREE clear; a needs-reduce zone
                  never carries the flag)
  too_wide        zone wider or higher than the small tile (0 by the routing: such boxes take the big-tile queue)
Classes overlap; `movable` counts the merge-free, table-reduced records with -inf heights, the ones reach_groups_kernel
(B') takes since it handles such zones (a build that routes them there leaves none of them in this queue). Also the card,
its power limit and its max SM clock. Prints one JSON line; with --out DIR it also writes it there."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import art_planner_b200 as ap  # noqa: E402
from art_planner_b200 import synth  # noqa: E402
import bench  # noqa: E402

REC_ALLFINITE, REC_NEEDS_REDUCE, REC_MERGEFREE = 8, 16, 32


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power, clock = (x.strip() for x in (q.stdout.strip().split(",") + ["", "", ""])[:3])
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def mix(m, poses):
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    chk.isValidBatch(torch.from_numpy(poses).cuda())
    torch.cuda.synchronize()
    st = chk.stats()
    zone, fl = chk.debugReachQueue()
    n = len(fl)
    nx, nz = zone[:, 1] - zone[:, 0] + 1, zone[:, 3] - zone[:, 2] + 1
    nr = (fl & REC_NEEDS_REDUCE) != 0
    nonfin = ((fl & REC_ALLFINITE) == 0) & ~nr
    mf = (fl & REC_MERGEFREE) != 0
    movable = mf & nonfin

    def share(k):
        return {"count": int(k), "share": round(float(k) / n, 4) if n else None}
    return {
        "queued_big_tile": st["last_queued_warp_stage"], "queued_reach_warp": st["last_queued_reach_stage"],
        "queued_reach_groups": st["last_reach_plane_stage"],
        "reach_warp_records": n,
        "non_finite": share(nonfin.sum()), "needs_reduce": share(nr.sum()),
        "not_merge_free": share((~mf).sum()), "too_wide": share(0),
        "max_zone_vertices_xz": [int(nx.max()) if n else 0, int(nz.max()) if n else 0],
        "movable": share(movable.sum()),
    }


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--out", default=None, help="directory for reach_queue_mix.json")
    args = ap_.parse_args()
    assert torch.cuda.is_available(), "reach_queue_mix.py needs a CUDA device"
    n = bench.POSES_PER_GPU
    res = {"card": card()}
    m, poses = bench.make_inputs(0, n)
    res["configs[1]"] = mix(m, poses)
    m = synth.make_fbm_map(bench.MAP_N, bench.MAP_N, bench.MAP_RES, seed=bench.MAP_SEED, **bench.ROUGH_MAP)
    res["c2_rough"] = mix(m, synth.make_terrain_poses(m, n, seed=bench.POSE_SEED, **bench.ROUGH_POSES))
    m, poses = bench.make_inputs(0, n, "c5", 1)
    res["configs[4]"] = mix(m, poses)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "reach_queue_mix.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
