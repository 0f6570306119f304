"""What the start / goal repair costs on the GPU: StartState / GoalStateRegion::sampleGoal (start.cpp:7-41, goal.cpp:11-41)
as one artp_find_valid_near call per planning query (one start, r = 0.2 m, and one goal, r = 0.5 m, n_iter = 1000, the
shipped params.yaml values) against the reference's serial loop through this library (isValid once per candidate, stopping
at the first valid one) on the same candidates.

Maps: BASELINE configs[1] (fBm 1000x1000 @ 0.04 m, amp 0.6) and its rough level (bench.py ROUGH_MAP); yaml robot.
Regimes, chosen per map by searching seeded centres: both centres valid; first valid draw near k = 10; near k = 300; no
valid draw at all. Times: the host-buffer call (host clock, the call synchronises), the *_device call (CUDA events on the
call's stream) and the serial loop (host clock), medians. Prints one JSON line; needs a CUDA device.

    python profiles/start_goal_search.py
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

N_ITER, RADII, SEED = 1000, np.array([0.2, 0.5]), 2024
MAP_N, MAP_RES, MAP_SEED = 1000, 0.04, 2                       # bench.py: BASELINE configs[1]
ROUGH_MAP = dict(amp=1.2, wavelength=3.0, persistence=0.7)     # bench.py: the rough level
REGIMES = {"centre_valid": (0, 0), "k_near_10": (5, 20), "k_near_300": (150, 450), "none_valid": (-1, -1)}


def pick_pair(chk, m, offsets):
    """A (start, goal) centre pair whose searches end in each regime: candidates come from seeded terrain poses moved up or
    down; offsets [2, N_ITER, 2] are the stream's draws of query 0 (start) and 1 (goal)."""
    import start_goal_cases as sgc
    cand, _ = sgc.make_queries(m, 4000, SEED)
    idx = []
    for q in range(2):
        _, i = chk.findValidNear(cand, RADII[q], N_ITER, offsets=np.broadcast_to(offsets[q], (len(cand), N_ITER, 2)))
        idx.append(i)
    out = {}
    for name, (lo, hi) in REGIMES.items():
        pair = []
        for q in range(2):
            hit = np.nonzero((idx[q] >= lo) & (idx[q] <= hi))[0]
            if len(hit) == 0:
                break
            mid = 0.5 * (lo + hi)
            pair.append(cand[hit[np.argmin(np.abs(idx[q][hit] - mid))]])
        if len(pair) == 2:
            out[name] = np.stack(pair)
    return out


def serial(chk, centres, offsets):
    """The reference loop through the single-state host API, same candidates: (states, index)."""
    st, ix = centres.copy(), np.full(2, -1, np.int32)
    for q in range(2):
        s = centres[q].copy()
        if chk.isValid(s):
            ix[q] = 0
            continue
        for k in range(N_ITER):
            s[0] = centres[q, 0] + offsets[q, k, 0]
            s[1] = centres[q, 1] + offsets[q, k, 1]
            if chk.isValid(s):
                ix[q] = k + 1
                break
        st[q] = s
    return st, ix


def main() -> None:
    import torch
    import art_planner_b200 as ap
    from art_planner_b200 import build, synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    build.build()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:   # the number is still reported, without its power limit
        power = f"unavailable ({ex!r})"
    res = {"card": torch.cuda.get_device_name(0), "power_limit": power, "n_iter": N_ITER, "radii_m": RADII.tolist(),
           "queries_per_call": 2, "maps": {}}
    for level, kw in (("gentle", dict(amp=0.6)), ("rough", ROUGH_MAP)):
        m = synth.make_fbm_map(MAP_N, MAP_N, MAP_RES, seed=MAP_SEED, **kw)
        chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
        chk.setMap(m)
        chk.updateHeightField()
        off = chk.ballOffsets(SEED, 0, 2, N_ITER, RADII)
        pairs = pick_pair(chk, m, off)
        rows = {}
        for name, c in pairs.items():
            hs, hi = chk.findValidNear(c, RADII, N_ITER, seed=SEED)
            ss, si = serial(chk, c, off)
            dc, dr = torch.from_numpy(c).cuda(), torch.from_numpy(RADII).cuda()
            ds, di = chk.findValidNear(dc, dr, N_ITER, seed=SEED)
            torch.cuda.synchronize()
            same = bool(np.array_equal(hi, si) and np.array_equal(hs, ss) and np.array_equal(di.cpu().numpy(), hi)
                        and np.array_equal(ds.cpu().numpy(), hs))
            t_host = []
            for _ in range(200):
                t0 = time.perf_counter()
                chk.findValidNear(c, RADII, N_ITER, seed=SEED)
                t_host.append(time.perf_counter() - t0)
            t_dev = []
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(200):
                e0.record()
                chk.findValidNear(dc, dr, N_ITER, seed=SEED)
                e1.record()
                e1.synchronize()
                t_dev.append(e0.elapsed_time(e1) * 1e-3)
            reps = 3 if name == "none_valid" else 20
            t_ser = []
            for _ in range(reps):
                t0 = time.perf_counter()
                serial(chk, c, off)
                t_ser.append(time.perf_counter() - t0)
            rows[name] = {"index": hi.tolist(), "isValid_calls_serial": int(sum(k + 1 if k >= 0 else N_ITER + 1 for k in si)),
                          "batched_host_us": round(1e6 * float(np.median(t_host)), 1),
                          "batched_device_us": round(1e6 * float(np.median(t_dev)), 1),
                          "serial_host_us": round(1e6 * float(np.median(t_ser)), 1), "answers_equal": same}
        res["maps"][level] = rows
    print(json.dumps(res))


if __name__ == "__main__":
    main()
