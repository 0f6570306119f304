"""Time inpaintMatrix on the device next to OpenCV, per hole pattern and map size (1000^2 and 4000^2 at 0.04 m):
  * device_layer_ms      one artp_inpaint_layer_device call on the elevation (CUDA events);
  * set_map_raw_ms       Planner.setMapRaw(raw elevation, raw traversability): both inpaints on the device + set_map;
  * cv2_inpaint_x2_ms    the reference's two inpaintMatrix calls through cv2 on the host CPU (where cv2 is importable);
  * set_map_ms           Planner.setMap given those two inpainted layers; cv2_route_ms = cv2_inpaint_x2_ms + set_map_ms.
Patterns (tests/inpaint_cases.profile_layer): `holes` = scattered 20 x 20-cell holes (many small interaction components),
`strip` = one unobserved strip 10 % of the map wide (one giant component), `both`. Both layers carry the same holes. Where
cv2 exists it also checks the device layer against the cv2 chain bit for bit (equals_cv2). Wall times are single calls
after one warm-up call on the 1000^2 maps. Prints one JSON line per case; with an argument, also writes them to that file."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import art_planner_b200 as ap  # noqa: E402
import inpaint_cases as ic  # noqa: E402
import planner_cases as pc  # noqa: E402
from art_planner_b200 import costnet, synth  # noqa: E402
from art_planner_b200.checker import _Handle  # noqa: E402


def checker(rp):
    chk = ap.StateValidityChecker(rp, handle=_Handle(rp, 0, risk_threshold=0.6))
    ap.MotionCostObjective(chk).setWeights(costnet.make_state_dict(seed=5))
    return chk


def wall(f):
    t = time.perf_counter()
    r = f()
    return (time.perf_counter() - t) * 1e3, r


def main():
    try:
        import cv2  # noqa: F401
        from oracle.make_golden_inpaint import cv_inpaint_matrix
    except ImportError:
        cv_inpaint_matrix = None
    rp = synth.PARAMS_YAML
    chk = checker(rp)
    rows = []
    for n in (1000, 4000):
        m = synth.make_fbm_map(n, n, seed=3)
        trav, _ = synth.make_traversability(m, seed=13)
        for pattern in ("holes", "strip", "both"):
            hole = np.isnan(ic.profile_layer(n, pattern))
            e = np.asfortranarray(np.where(hole, np.nan, m.elevation).astype(np.float32))
            t = np.asfortranarray(np.where(hole, np.nan, trav).astype(np.float32))
            d = torch.from_numpy(np.ascontiguousarray(e.T)).cuda().t()
            if n <= 1000:   # warm up once on the small maps; the large ones run once
                chk.inpaint(d)
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            got = chk.inpaint(d)
            ev[1].record()
            torch.cuda.synchronize()
            r = {"n": n, "pattern": pattern, "unknown": float(hole.mean()), "device_layer_ms": ev[0].elapsed_time(ev[1])}
            pp = ap.Planner.params(seed=1)
            pl = ap.Planner(chk, pp)
            if n <= 1000:
                pl.setMapRaw(e, t, m.res, m.cx, m.cy)
            r["set_map_raw_ms"], mi = wall(lambda: pl.setMapRaw(e, t, m.res, m.cx, m.cy))
            r["set_map_raw_bytes_h2d"] = mi["bytes_h2d"]
            if cv_inpaint_matrix is not None:
                r["cv2_inpaint_x2_ms"], (ei, ti) = wall(lambda: (cv_inpaint_matrix(e), cv_inpaint_matrix(t)))
                r["equals_cv2"] = bool(np.array_equal(got.cpu().numpy().view(np.uint32), ei.view(np.uint32)))
                if n <= 1000:
                    pl.setMap(e, t, ei, ti, m.res, m.cx, m.cy)
                r["set_map_ms"], _ = wall(lambda: pl.setMap(e, t, ei, ti, m.res, m.cx, m.cy))
                r["cv2_route_ms"] = r["cv2_inpaint_x2_ms"] + r["set_map_ms"]
            rows.append(r)
            print(json.dumps(r), flush=True)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump({"gpu": torch.cuda.get_device_name(0), "cases": rows}, f, indent=1)


if __name__ == "__main__":
    main()
