"""Time the cost server's map preparation plus the trunk on the device next to the server's own route, at 1000^2 and
4000^2 with holes (tests/inpaint_cases.profile_layer "holes": scattered 20 x 20-cell holes over an fBm map):
  * cost_map_ms          one artp_cost_map_layer_device call (CUDA events);
  * features_raw_ms      one artp_update_features_raw_device call: preparation + trunk (light network, tensor-core path);
  * host_prepare_ms      the server's preparation on the host CPU: numpy float32 + cv2.inpaint (where cv2 is importable);
  * host_route_ms        host_prepare_ms + artp_update_features on the prepared map already uploaded (the trunk alone,
                         features_ms), i.e. what a caller preparing the map on the host pays besides the upload.
Device times are medians of 5 calls after one warm-up. Prints one JSON line per size (card and power limit first); with
an argument, also writes them to that file."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import art_planner_b200 as ap  # noqa: E402
import inpaint_cases as ic  # noqa: E402
from art_planner_b200 import costnet, synth  # noqa: E402
from oracle import cost_map_oracle as cm  # noqa: E402


def device_ms(f, reps=5):
    f()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        f()
        ev[1].record()
        torch.cuda.synchronize()
        ts.append(ev[0].elapsed_time(ev[1]))
    return float(np.median(ts))


def main():
    try:
        import cv2  # noqa: F401
        have_cv2 = True
    except ImportError:
        have_cv2 = False
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    rows = [{"gpu": gpu, "cv2": have_cv2}]
    print(json.dumps(rows[0]), flush=True)
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    obj = ap.MotionCostObjective(chk)
    obj.setWeights(costnet.make_state_dict(seed=5))
    for n in (1000, 4000):
        m = synth.make_fbm_map(n, n, seed=3)
        hole = np.isnan(ic.profile_layer(n, "holes"))
        e = np.asfortranarray(np.where(hole, np.nan, m.elevation).astype(np.float32))
        d = torch.from_numpy(np.ascontiguousarray(e.T)).cuda().t()
        r = {"n": n, "unknown": float(hole.mean())}
        r["cost_map_ms"] = device_ms(lambda: obj.costMap(d))
        r["features_raw_ms"] = device_ms(lambda: obj.updateFeaturesRaw(d, m.res, m.cx, m.cy))
        out = obj.costMap(d)
        torch.cuda.synchronize()
        prepared = out.cpu().numpy()
        chk.setMap(synth.SynthMap(np.asfortranarray(prepared), np.asfortranarray(prepared), m.res, m.cx, m.cy, ""))
        chk.updateHeightField()
        r["features_ms"] = device_ms(obj.updateFeatures)
        if have_cv2:
            t = time.perf_counter()
            host = cm.cost_map_layer(e, cm.telea_cv2)
            r["host_prepare_ms"] = (time.perf_counter() - t) * 1e3
            r["host_route_ms"] = r["host_prepare_ms"] + r["features_ms"]
            r["equals_cv2"] = bool(np.array_equal(host.view(np.uint32), prepared.view(np.uint32)))
        rows.append(r)
        print(json.dumps(r), flush=True)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write("\n".join(json.dumps(r) for r in rows) + "\n")


if __name__ == "__main__":
    main()
