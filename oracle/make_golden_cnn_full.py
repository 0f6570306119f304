"""Pin the CNN oracle (oracle/cnn_oracle.py, which takes every shape from the weights) against the reference's
full-width module, network.py (imported from /root/reference, fp32, CPU), and write tests/golden/cnn_full_c4.npz:
the recipe of make_golden_cnn.py (c4 map, 4096 queries of seed 6, weights of seed 5) with network.py's widths.
Run in the build container:  python oracle/make_golden_cnn_full.py
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import cases  # noqa: E402
from art_planner_b200 import costnet  # noqa: E402
from oracle.cnn_oracle import CostNetOracle, cnn_input_from_layer  # noqa: E402

REF = "/root/reference/art_planner_motion_cost/src/art_planner_motion_cost/predictor"


def main():
    spec = importlib.util.spec_from_file_location("ref_network", os.path.join(REF, "network.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    m = cases.c4_map()
    sd = costnet.make_state_dict(seed=5, network="full")
    net = mod.network()
    assert sum(p.numel() for p in net.parameters()) == 1035779
    missing = net.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()}, strict=False)
    assert not missing.unexpected_keys and all(k.endswith("num_batches_tracked") for k in missing.missing_keys), missing
    net.eval()
    E = cnn_input_from_layer(m.elevation)
    with torch.no_grad():
        ref_feat = net.CNNpart(torch.as_tensor(E)[None, None])[0]
    orc = CostNetOracle(sd)
    feat = orc.features(E)
    assert tuple(feat.shape) == (64, 104, 104)
    err_f = float((feat - ref_feat).abs().max() / ref_feat.abs().max())
    print("feature map", tuple(feat.shape), "oracle vs reference module rel max err", err_f)
    assert err_f < 1e-6
    # FCpart through CostQuery's arithmetic (network.py:162 asks torch.ones for a CUDA tensor it never uses: patched)
    q = costnet.make_queries(m, 4096, seed=6)
    lx, ly = m.length
    t = torch.from_numpy(q.astype(np.float64)).clone()
    t[:, 0] -= m.cx; t[:, 1] -= m.cy; t[:, 3] -= m.cx; t[:, 4] -= m.cy
    t[:, :3] = t[:, :3] - t[:, 3:]
    feat_res = m.res * net.featureResDownsampleFactor
    row_bias = int((lx / m.res - 2 * net.mapClip) / net.featureResDownsampleFactor * 0.5)
    col_bias = int((ly / m.res - 2 * net.mapClip) / net.featureResDownsampleFactor * 0.5)
    row = torch.clamp(t[:, 3] / feat_res + row_bias, min=1, max=ref_feat.shape[1] - 2).long()
    col = torch.clamp(t[:, 4] / feat_res + col_bias, min=1, max=ref_feat.shape[2] - 2).long()
    f = ref_feat[None][:, :, row, col].squeeze(0).t().unsqueeze(-1).unsqueeze(-1)
    tar = torch.cat((t[:, :3], t[:, 5:6]), dim=1).unsqueeze(-1).unsqueeze(-1).float()
    real_ones = torch.ones
    torch.ones = lambda *a, **k: real_ones(*a, **{kk: vv for kk, vv in k.items() if kk not in ("device", "dtype")})
    try:
        with torch.no_grad():
            out = net.FCpart(f.float(), tar)
    finally:
        torch.ones = real_ones
    ref_cost = torch.stack((out[0][:, 0, 0, 0], out[1][:, 0, 0, 0], out[3][:, 0, 0, 0]), dim=1).numpy()
    cost = orc.query(feat, q, m.res, lx, ly, m.cx, m.cy)
    err_c = float(np.abs(cost - ref_cost).max())
    print("costs oracle vs reference module abs max err", err_c, "ranges", ref_cost.min(0), ref_cost.max(0))
    assert err_c < 1e-5
    path = os.path.join(ROOT, "tests", "golden", "cnn_full_c4.npz")
    np.savez_compressed(path, cost=ref_cost.astype(np.float32), feat_sample=ref_feat[:, ::13, ::13].numpy(),
                        feat_abs_max=np.float32(ref_feat.abs().max()),
                        blob_sum=np.float64(costnet.pack_blob(sd).astype(np.float64).sum()))
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
