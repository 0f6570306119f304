"""Time one recompute of the sampler's distribution (artp_update_sample_distribution_device: vertex histogram, Gaussian blur,
max - n, filter, unknown-space cap, CDF) for 10 k roadmap vertices on 1000^2 and 4000^2 maps at 0.04 m (yaml robot:
73-tap blur), with CUDA events, against the same chain on the CPU through cv2 (histogram, cv2.GaussianBlur, numpy cap
and CDF) on the same inputs. Prints one JSON line with the card's name and power limit.
    python profiles/sample_distribution_time.py"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import art_planner_b200 as ap  # noqa: E402
from art_planner_b200 import synth  # noqa: E402
from oracle import sample_distribution_oracle as sdo  # noqa: E402


def cpu_chain(cv2, m, v, filt, obs, dp):
    t0 = time.perf_counter()
    lx, ly = m.length
    ok = np.isfinite(v[:, 0]) & np.isfinite(v[:, 1])
    i = np.floor((m.cx + 0.5 * lx - v[ok, 0]) / m.res).astype(np.int64)
    j = np.floor((m.cy + 0.5 * ly - v[ok, 1]) / m.res).astype(np.int64)
    inside = (i >= 0) & (j >= 0) & (i < m.rows) & (j < m.cols)
    n = np.zeros((m.cols, m.rows), np.float32)                # the cols x rows image of the column-major layer
    np.add.at(n, (j[inside], i[inside]), 1.0)
    k, s = sdo.blur_size(dp.density_blur_radius, m.res)
    n = cv2.GaussianBlur(n, (k, k), s)
    p = (n.max() - n) * filt.T
    known = float(p[obs.T > 0].sum(dtype=np.float64))
    unknown = float(p[obs.T <= 0].sum(dtype=np.float64))
    km, um, _ = sdo.cap_multipliers(known, unknown, dp.max_prob_unknown_samples)
    p = p * np.where(obs.T > 0, km, um).astype(np.float32)
    rs = p.sum(axis=0)
    cum = np.cumsum(p / rs[None, :], axis=0)
    row = np.cumsum(rs / rs.sum())
    return time.perf_counter() - t0, cum, row


def main():
    try:
        import cv2
    except ImportError:
        cv2 = None
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    rp = synth.PARAMS_YAML
    dp = sdo.DistributionParams(density_blur_radius=sdo.blur_radius(rp))
    out = {"gpu": q.stdout.strip(), "vertices": 10000, "ksize": sdo.blur_size(dp.density_blur_radius, 0.04)[0]}
    for size in (1000, 4000):
        m = synth.make_flat_map(size, size, res=0.04)
        k = np.arange(size * size).reshape(size, size)
        thr = np.asfortranarray((synth.hash_uniform(3, 51, k) > 0.2).astype(np.float32))
        obs = np.asfortranarray((synth.hash_uniform(3, 52, (np.arange(size)[:, None] // 23) * 8192 + np.arange(size)[None, :] // 29)
                                 > 0.3).astype(np.float32))
        rng = np.random.default_rng(1)
        v = np.zeros((10000, 7))
        v[:, 0] = rng.uniform(-0.5, 0.5, 10000) * size * 0.04
        v[:, 1] = rng.uniform(-0.5, 0.5, 10000) * size * 0.04
        v[:, 6] = 1
        chk = ap.StateValidityChecker(rp, device=0)
        chk.setMap(m)
        chk.updateHeightField()
        filt = chk.setSampleFilter(thr, obs)
        dv = torch.from_numpy(v).cuda()
        for _ in range(3):
            chk.updateSampleDistribution(dv, dp)
        torch.cuda.synchronize()
        reps = 20
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            chk.updateSampleDistribution(dv, dp)
        e1.record()
        torch.cuda.synchronize()
        dev_ms = e0.elapsed_time(e1) / reps
        res = {"device_ms": round(dev_ms, 4)}
        if cv2 is not None:
            t = min(cpu_chain(cv2, m, v, filt, obs, dp)[0] for _ in range(3))
            res["cpu_cv2_ms"] = round(t * 1e3, 3)
            res["speedup"] = round(t * 1e3 / dev_ms, 1)
        out[f"{size}x{size}"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
