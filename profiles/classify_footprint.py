"""Is the classify stage bound by L2 misses on its range tables?

Times the classify stage (library stage events, L2 flushed before every step) on two 1M-pose inputs of the bench map
(BASELINE configs[1]) that differ only in the map area they cover: poses over the whole 1000 x 1000 map, and poses drawn
the same way over a 250 x 250-cell square in its middle. The terrain statistics are the same; the range-table footprint
shrinks 16x. The two inputs alternate step by step.

  python profiles/classify_footprint.py [--steps 30]          # GPU: stage times of both inputs, one JSON line
  python profiles/classify_footprint.py --levels [--n 200000] # CPU only: which range-table levels classify reads
  python profiles/classify_footprint.py --fallback [--n 50000] # CPU only: how often classify reads the exact tables

--levels restates the zone of each box (AABB -> vertex index range, as in classify_box) in float64 numpy over the bench
poses and counts, per layer, the table level k = floor(log2(min(nX, nZ))) and the number of windows it reads. Rounding
at cell borders can move a few boxes by one vertex; the histogram is what matters. --fallback restates the compact-table
interval tests over the same zones on the bench map, its rough level and a terraced map.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
sys.dont_write_bytecode = True

import numpy as np

import bench
from art_planner_b200 import synth

SUB = 250   # cells per side of the sub-square
CODE_MAX = 32765   # artp::kCodeMax: the largest code of a finite max in the compact range tables


def sub_square_poses(m, n):
    k = np.arange(n)
    span = SUB * m.res * 0.999
    x = m.cx + (synth.hash_uniform(bench.POSE_SEED, 1, k) - 0.5) * span
    y = m.cy + (synth.hash_uniform(bench.POSE_SEED, 2, k) - 0.5) * span
    return synth.make_terrain_poses(m, n, seed=bench.POSE_SEED, xy=(x, y))


def box_zones(m, poses, p=synth.PARAMS_YAML):
    """Per box (torso, reach0..3): layer name, zone vertex range x0, x1, z0, z1 and box bottom / top, restated in float64
    from classify_box (AABB -> vertex index range). Rounding at cell borders can move a few zones by one vertex."""
    t = poses[:, :3]
    x, y, z, w = (poses[:, i] for i in range(3, 7))
    Rm = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                   2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                   2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    lx, ly = m.length
    sW, sD = lx / (m.rows - 1), ly / (m.cols - 1)
    boxes = [("torso", "elevation", (p.torso_off_x, p.torso_off_y, p.torso_off_z - p.feet_off_z),
              (p.torso_length, p.torso_width, p.torso_height))]
    for fk in range(4):
        boxes.append((f"reach{fk}", "elevation_masked",
                      (-p.feet_off_x if fk & 2 else p.feet_off_x, -p.feet_off_y if fk & 1 else p.feet_off_y, 0.0),
                      (p.reach_x, p.reach_y, p.reach_z)))
    for name, layer, off, side in boxes:
        c = np.einsum("nij,j->ni", Rm, np.array(off)) + t
        s = np.array(side)
        xr = 0.5 * (np.abs(Rm[:, 0, :]) * s).sum(1)     # R1 row 0 = -Rb row 0
        yr = 0.5 * (np.abs(Rm[:, 2, :]) * s).sum(1)     # R1 row 1 = Rb row 2
        zr = 0.5 * (np.abs(Rm[:, 1, :]) * s).sum(1)     # R1 row 2 = Rb row 1
        P0 = -(c[:, 0] - m.cx) + 0.5 * lx
        P2 = (c[:, 1] - m.cy) + 0.5 * ly
        x0 = np.maximum(np.floor((P0 - xr) / sW), 0).astype(np.int64)
        x1 = np.minimum(np.ceil((P0 + xr) / sW), m.rows - 1).astype(np.int64)
        z0 = np.maximum(np.floor((P2 - zr) / sD), 0).astype(np.int64)
        z1 = np.minimum(np.ceil((P2 + zr) / sD), m.cols - 1).astype(np.int64)
        yield name, layer, x0, x1, z0, z1, c[:, 2] - yr, c[:, 2] + yr


def levels(m, poses):
    out = {}
    for name, layer, x0, x1, z0, z1, _, _ in box_zones(m, poses):
        nX, nZ = x1 - x0 + 1, z1 - z0 + 1
        inside = (nX >= 2) & (nZ >= 2)      # boxes clipped at the map border are left out
        nX, nZ = nX[inside], nZ[inside]
        kk = np.floor(np.log2(np.minimum(nX, nZ))).astype(np.int64)
        nw = ((nX + (1 << kk) - 1) >> kk) * ((nZ + (1 << kk) - 1) >> kk)
        key = [f"{layer}:k{a}:{b}win" for a, b in zip(kk, nw)]
        u, cnt = np.unique(key, return_counts=True)
        out[name] = {str(a): round(int(b) / len(poses), 4) for a, b in zip(u, cnt)}
    return out


def fallback_rate(m, poses):
    """Share of table-path boxes (zone at least 2 x 2 vertices) whose compact-code intervals leave one of the collider's
    early-out tests open, so that classify_box reads the exact range tables. The zone codes depend only on the exact zone
    max / min (the encodings are monotone), so they are computed here from the zone itself with the library's encoding
    in float32. Every box of every pose is counted (classify skips the boxes after a failing one)."""
    eps = np.float32(1.1920928955078125e-07)
    out = {}
    for name, layer, x0, x1, z0, z1, lo_b, hi_b in box_zones(m, poses):
        L = getattr(m, layer)
        fin_all = L[np.isfinite(L)].astype(np.float32)
        base, top = fin_all.min(), fin_all.max()
        e = -126
        while base + np.float32(CODE_MAX) * np.float32(2.0 ** e) < top:
            e += 1
        dec = base + np.arange(CODE_MAX + 3, dtype=np.float32) * np.float32(2.0 ** e)
        sel = np.nonzero((x1 - x0 >= 1) & (z1 - z0 >= 1))[0]
        mx = np.full(len(sel), -np.inf, np.float32)
        mn = np.full(len(sel), np.inf, np.float32)
        allfin = np.ones(len(sel), bool)
        for a, i in enumerate(sel):
            zone = L[x0[i]:x1[i] + 1, m.cols - 1 - z1[i]:m.cols - z0[i]]    # field vertex (x, z) = layer[x, cols-1-z]
            f = np.isfinite(zone)
            allfin[a] = f.all()
            if f.any():
                mx[a], mn[a] = zone[f].max(), zone[f].min()
        ok = np.isfinite(mx)
        cM = np.searchsorted(dec[1:CODE_MAX + 1], mx, "left") + 1
        cm = np.searchsorted(dec[:CODE_MAX + 1], mn, "right") - 1
        cM, cm = np.clip(cM, 1, CODE_MAX), np.clip(cm, 0, CODE_MAX)
        mxLo, mxHi, mnLo, mnHi = dec[cM - 1], dec[cM], dec[cm], dec[cm + 1]
        minB, maxB = lo_b[sel].astype(np.float32), hi_b[sel].astype(np.float32)
        above_t, above_f = minB - mxHi > -eps, ~(minB - mxLo > -eps)
        under_t, under_f = mnLo - maxB > -eps, ~(mnHi - maxB > -eps)
        span_t = allfin & (mnLo - minB > -eps) & (maxB - mxHi > -eps)
        span_f = ~allfin | ~((mnHi - minB > -eps) & (maxB - mxLo > -eps))
        plane_f = ~allfin | ~(mxLo - mnHi < eps)
        decided = above_t | (above_f & (under_t | (under_f & (span_t | (span_f & plane_f)))))
        out[name] = round(float(1.0 - (decided & ok).mean()), 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--levels", action="store_true")
    ap.add_argument("--fallback", action="store_true")
    ap.add_argument("--n", type=int, default=bench.POSES_PER_GPU)
    args = ap.parse_args()
    m, full = bench.make_inputs(0, args.n)
    if args.fallback:
        sys.path.insert(0, os.path.join(R, "tests"))
        import cases
        mr = synth.make_fbm_map(bench.MAP_N, bench.MAP_N, bench.MAP_RES, seed=bench.MAP_SEED, **bench.ROUGH_MAP)
        mt = cases.terraces()
        print(json.dumps({"configs[1]": fallback_rate(m, full),
                          "rough": fallback_rate(mr, synth.make_terrain_poses(mr, args.n, seed=bench.POSE_SEED, **bench.ROUGH_POSES)),
                          "terraces": fallback_rate(mt, synth.make_terrain_poses(mt, args.n, seed=bench.POSE_SEED))}))
        return
    sub = sub_square_poses(m, args.n)
    if args.levels:
        print(json.dumps({"full_map": levels(m, full), "sub_square": levels(m, sub)}))
        return

    import torch
    import art_planner_b200 as ap_
    assert torch.cuda.is_available(), "needs a CUDA device"
    chk = ap_.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    chk.setTiming(True)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    ins = {"full_map": torch.from_numpy(full).cuda(), "sub_square": torch.from_numpy(sub).cuda()}
    out = torch.empty(args.n, dtype=torch.uint8, device="cuda")
    for d in ins.values():
        for _ in range(3):
            chk.isValidBatch(d, out=out)
    torch.cuda.synchronize()
    st = {k: [] for k in ins}
    info = {}
    for i in range(args.steps):
        for k, d in ins.items():
            flush.fill_(i & 0xFF)
            chk.isValidBatch(d, out=out)
            st[k].append(chk.lastStageTimesMs())
            torch.cuda.synchronize()
            if i == 0:
                s = chk.stats()
                info[k] = {"valid_fraction": float(out.float().mean()), "queued_warp_stage": s["last_queued_warp_stage"],
                           "queued_reach_stage": s["last_queued_reach_stage"]}
    names = ("classify", "torso_queue", "reach_queue_warp", "reach_queue_groups", "group")
    res = {}
    for k, v in st.items():
        a = np.array(v)
        res[k] = {"stage_ms_median": dict(zip(names, [round(float(x), 4) for x in np.median(a, 0)])),
                  "classify_ms_range": [round(float(a[:, 0].min()), 4), round(float(a[:, 0].max()), 4)], **info[k]}
    res["classify_sub_over_full"] = round(res["sub_square"]["stage_ms_median"]["classify"]
                                          / res["full_map"]["stage_ms_median"]["classify"], 4)
    res["gpu"] = torch.cuda.get_device_name(0)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
