"""Both motion-cost networks (network_light.py and network.py) on the device, on the 256 x 256 patch (configs[3]) and
the 1000 x 1000 metric map: trunk times from artp_get_cnn_timing (3x3 stack, 15x15 layer, whole trunk), the head over
4096 queries, and the cuDNN evaluation of each module restatement in fp16 (as the reference runs it) and fp32, as
profiles/cnn_time.py does for the light network. The two networks run in alternating rounds on one handle each, so
clock drift and neighbours' load fall on both. Prints one JSON line with the card, its power limit and max SM clock.

    python profiles/cnn_networks.py [--rounds 5] [--reps 10]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
sys.path.insert(0, os.path.join(R, "tests"))

import art_planner_b200 as ap  # noqa: E402
import cases  # noqa: E402
from art_planner_b200 import costnet, synth  # noqa: E402
from oracle.cnn_oracle import CostNetOracle, cnn_input_from_layer  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, pl, clk = [x.strip() for x in q.split(",")]
    return {"name": name, "power_limit": pl, "max_sm_clock": clk}


def torch_trunk_ms(sd, E, dtype, reps):
    """CNNpart through the oracle's functional calls (the module's cuDNN convolutions) in `dtype`."""
    orc = CostNetOracle(sd)
    p = {k: v.cuda().to(dtype) for k, v in orc.p.items()}
    orc.p = p
    x = torch.as_tensor(E).cuda().to(dtype)[None, None]

    def feats():
        t = orc._conv_bn(x, "init_conv1", "init_conv1_bn")
        t = F.max_pool2d(F.leaky_relu(orc._conv_bn(t, "init_conv2", "init_conv2_bn"), 0.3), (2, 2), stride=2)
        t = F.leaky_relu(orc._conv_bn(t, "init_conv3", "init_conv3_bn"), 0.3)
        t = F.max_pool2d(F.leaky_relu(orc._conv_bn(t, "init_conv4", "init_conv4_bn"), 0.3), (3, 3), stride=1)
        t = F.leaky_relu(orc._conv_bn(t, "init_conv5", "init_conv5_bn"), 0.3)
        return F.leaky_relu(orc._conv_bn(t, "init_flatten", "init_flatten_bn"), 0.3)

    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        for _ in range(3):
            feats()
        torch.cuda.synchronize()
        s.record()
        for _ in range(reps):
            feats()
        e.record()
        torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--rounds", type=int, default=5)
    ap_.add_argument("--reps", type=int, default=10)
    a = ap_.parse_args()
    assert torch.cuda.is_available(), "needs cuda:0"
    maps = {"256": cases.c4_map(), "1000": synth.make_fbm_map(1000, 1000, 0.04, seed=2, amp=0.6)}
    nets = ("light", "full")
    sds = {n: costnet.make_state_dict(seed=5, network=n) for n in nets}
    objs = {}
    for mk, m in maps.items():
        for n in nets:
            chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
            chk.setMap(m)
            chk.updateHeightField()
            obj = ap.MotionCostObjective(chk)
            obj.setWeights(sds[n])
            obj.updateFeatures()                      # warm-up: allocation, tensor maps, kernel attributes
            objs[mk, n] = (chk, obj, torch.from_numpy(costnet.make_queries(m, 4096, seed=6)).cuda())
    trunk = {k: [] for k in objs}
    head = {k: [] for k in objs}
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.rounds):
        for k, (chk, obj, q) in objs.items():       # alternating: every round runs every (map, network)
            ts = []
            for _ in range(a.reps):
                obj.updateFeatures()
                ts.append(obj.lastTrunkTimesMs())
            trunk[k].append(np.median(np.array(ts), axis=0))
            out = torch.empty((q.shape[0], 3), device="cuda")
            for _ in range(3):
                obj.costQuery(q, out)
            torch.cuda.synchronize()
            s.record()
            for _ in range(100):
                obj.costQuery(q, out)
            e.record()
            torch.cuda.synchronize()
            head[k].append(s.elapsed_time(e) / 100)
    res = {"card": card(), "rounds": a.rounds, "reps": a.reps, "results": {}}
    for k in objs:
        mk, n = k
        t = np.array(trunk[k])
        E = cnn_input_from_layer(maps[mk].elevation)
        res["results"][f"{n}_{mk}"] = {
            "trunk_3x3_ms": [round(float(x), 4) for x in (t[:, 0].min(), np.median(t[:, 0]), t[:, 0].max())],
            "trunk_15x15_ms": [round(float(x), 4) for x in (t[:, 1].min(), np.median(t[:, 1]), t[:, 1].max())],
            "trunk_total_ms": [round(float(x), 4) for x in (t[:, 2].min(), np.median(t[:, 2]), t[:, 2].max())],
            "head_4096_ms": [round(float(x), 4) for x in (min(head[k]), np.median(head[k]), max(head[k]))],
            "torch_fp16_trunk_ms": round(torch_trunk_ms(sds[n], E, torch.float16, a.reps), 4),
            "torch_fp32_trunk_ms": round(torch_trunk_ms(sds[n], E, torch.float32, a.reps), 4),
        }
    res["note"] = "times [min, median, max] over rounds; each round the median of reps trunk runs / 100 head calls"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
