"""Motion-cost network plumbing (product side): parameter naming / flat weight-blob layout of the reference's two
`network` modules (art_planner_motion_cost/src/art_planner_motion_cost/predictor/network_light.py:9-63 and
network.py:9-63) and a seeded synthetic weight generator (the shipped .pt files are Git-LFS pointers, SURVEY.md
section 8c).

The C ABI takes ONE flat fp32 blob (`artp_set_cost_weights`): for every layer of the network's table below, in this
order, the conv weight in PyTorch layout [Cout][Cin][kh][kw] followed -- for layers with a BatchNorm -- by bn.weight,
bn.bias, bn.running_mean, bn.running_var ([Cout] each), or -- for the three output convs -- by the conv bias. The two
architectures differ only in their widths, so the blob's length tells the library which one it holds. A trained model
goes straight in: `pack_blob(torch.load(path, map_location="cpu"))` (a state dict of either network).
"""
from __future__ import annotations

import numpy as np

from .synth import hash_uniform

# (conv name, bn name or None, Cout, Cin, k): network_light.py
LAYERS = [
    ("init_conv1", "init_conv1_bn", 24, 1, 3),
    ("init_conv2", "init_conv2_bn", 24, 24, 3),
    ("init_conv3", "init_conv3_bn", 48, 24, 3),
    ("init_conv4", "init_conv4_bn", 48, 48, 3),
    ("init_conv5", "init_conv5_bn", 48, 48, 3),
    ("init_flatten", "init_flatten_bn", 48, 48, 15),
    ("tar0_conv1", "tar0_conv1_bn", 16, 10, 1),
    ("out0_conv1", "out0_conv1_bn", 48, 64, 1),
    ("out1_conv1", "out1_conv1_bn", 24, 48, 1),
    ("out1_conv2", "out1_conv2_bn", 24, 48, 1),
    ("out1_conv3", "out1_conv3_bn", 36, 48, 1),
    ("out2_conv1", None, 1, 24, 1),
    ("out2_conv2", None, 1, 24, 1),
    ("out2_conv3", None, 1, 36, 1),
]
# network.py: the same layers at 32 / 64 channels in the trunk, out0 80 -> 64, out1 64 -> 32 each
LAYERS_FULL = [
    ("init_conv1", "init_conv1_bn", 32, 1, 3),
    ("init_conv2", "init_conv2_bn", 32, 32, 3),
    ("init_conv3", "init_conv3_bn", 64, 32, 3),
    ("init_conv4", "init_conv4_bn", 64, 64, 3),
    ("init_conv5", "init_conv5_bn", 64, 64, 3),
    ("init_flatten", "init_flatten_bn", 64, 64, 15),
    ("tar0_conv1", "tar0_conv1_bn", 16, 10, 1),
    ("out0_conv1", "out0_conv1_bn", 64, 80, 1),
    ("out1_conv1", "out1_conv1_bn", 32, 64, 1),
    ("out1_conv2", "out1_conv2_bn", 32, 64, 1),
    ("out1_conv3", "out1_conv3_bn", 32, 64, 1),
    ("out2_conv1", None, 1, 32, 1),
    ("out2_conv2", None, 1, 32, 1),
    ("out2_conv3", None, 1, 32, 1),
]
# network name -> (layer table, ARTP_COST_NET_* value of include/artp.h)
NETWORKS = {"light": (LAYERS, 0), "full": (LAYERS_FULL, 1)}
BN_EPS = 1e-5          # torch.nn.BatchNorm2d default
MAP_CLIP = 24          # network_light.py:16
FEATURE_DOWNSAMPLE = 2  # network_light.py:15


def blob_size(network: str = "light") -> int:
    n = 0
    for _, bn, co, ci, k in NETWORKS[network][0]:
        n += co * ci * k * k + (4 * co if bn else co)
    return n


def network_of(sd: dict) -> str:
    """"light" or "full" from a state dict: init_conv1 has 24 or 32 output channels."""
    co = int(np.shape(sd["init_conv1.weight"])[0])
    for name, (layers, _) in NETWORKS.items():
        if layers[0][2] == co:
            return name
    raise ValueError(f"init_conv1 has {co} output channels: neither network_light (24) nor network (32)")


def make_state_dict(seed: int = 5, network: str = "light") -> dict:
    """Seeded synthetic parameters (numpy fp32) keyed like the reference module's state_dict."""
    sd = {}
    stream = 0

    def u(shape, lo, hi):
        nonlocal stream
        stream += 1
        n = int(np.prod(shape))
        return (lo + (hi - lo) * hash_uniform(seed, 7000 + stream, np.arange(n))).astype(np.float32).reshape(shape)

    for conv, bn, co, ci, k in NETWORKS[network][0]:
        bound = 0.8 * np.sqrt(6.0 / (ci * k * k))
        sd[conv + ".weight"] = u((co, ci, k, k), -bound, bound)
        if bn:
            sd[bn + ".weight"] = u((co,), 0.6, 1.4)
            sd[bn + ".bias"] = u((co,), -0.2, 0.2)
            sd[bn + ".running_mean"] = u((co,), -0.2, 0.2)
            sd[bn + ".running_var"] = u((co,), 0.5, 1.5)
        else:
            sd[conv + ".bias"] = u((co,), -0.1, 0.5)
    return sd


def pack_blob(sd: dict) -> np.ndarray:
    """The flat blob of a state dict of either network (numpy arrays or CPU tensors; num_batches_tracked ignored)."""
    network = network_of(sd)
    parts = []
    for conv, bn, co, ci, k in NETWORKS[network][0]:
        assert tuple(np.shape(sd[conv + ".weight"])) == (co, ci, k, k), (conv, np.shape(sd[conv + ".weight"]))
        parts.append(np.asarray(sd[conv + ".weight"], dtype=np.float32).reshape(-1))
        if bn:
            for suffix in (".weight", ".bias", ".running_mean", ".running_var"):
                parts.append(np.asarray(sd[bn + suffix], dtype=np.float32).reshape(-1))
        else:
            parts.append(np.asarray(sd[conv + ".bias"], dtype=np.float32).reshape(-1))
    blob = np.ascontiguousarray(np.concatenate(parts), dtype=np.float32)
    assert blob.size == blob_size(network)
    return blob


def make_queries(m, n: int, seed: int = 6) -> np.ndarray:
    """C4 queries [n, 6] float32 = [target_x, target_y, target_yaw, start_x, start_y, start_yaw]
    (objectives/motion_cost_objective.h:22-23, cost_query.py:39-45): start uniform in the valid feature area,
    target = start + U(0, 0.5 m) in a random heading, yaws uniform."""
    k = np.arange(n)
    lx, ly = m.length
    inner_x, inner_y = lx - 2 * MAP_CLIP * m.res, ly - 2 * MAP_CLIP * m.res
    sx = m.cx + (hash_uniform(seed, 1, k) - 0.5) * inner_x
    sy = m.cy + (hash_uniform(seed, 2, k) - 0.5) * inner_y
    d = 0.5 * hash_uniform(seed, 3, k)
    hd = (hash_uniform(seed, 4, k) * 2 - 1) * np.pi
    tyaw = (hash_uniform(seed, 5, k) * 2 - 1) * np.pi
    syaw = (hash_uniform(seed, 6, k) * 2 - 1) * np.pi
    q = np.stack([sx + d * np.cos(hd), sy + d * np.sin(hd), tyaw, sx, sy, syaw], axis=1)
    return np.ascontiguousarray(q.astype(np.float32))
