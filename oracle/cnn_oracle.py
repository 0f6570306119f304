"""CPU oracle of the learned motion-cost path (TEST INFRASTRUCTURE ONLY), in fp32 (or float64) PyTorch functional ops,
plus the range-testing tools at the end of the file: calibrated weights, a split emulation and an error bound.

Restates, citing the reference (paths under art_planner_motion_cost/):
  * network.CNNpart            src/art_planner_motion_cost/predictor/network_light.py:78-110
  * network.FCpart             src/art_planner_motion_cost/predictor/network_light.py:113-165
  * CostQuery.setMapParams / __call__   src/art_planner_motion_cost/predictor/cost_query.py:27-69
  * the server's map orientation and query centring   scripts/cost_query_server.py:74,160-161
The reference runs the module in fp16 (`predictor.py:22`); parity is judged against the fp32 evaluation of the same
module (BASELINE.md section 3), which is what this oracle computes. oracle/make_golden_cnn.py checks this restatement
against the reference's own module (imported from /root/reference, fp32, CPU) and commits the golden costs.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

MAP_CLIP = 24          # network_light.py:16
DOWNSAMPLE = 2         # network_light.py:15
BN_EPS = 1e-5


def cnn_input_from_layer(layer: np.ndarray) -> np.ndarray:
    """grid_map layer (rows x cols, index (i,j) at -x,-y) -> network input E[r][c] = layer(rows-1-r, cols-1-c):
    np.rot90(msg.reshape(row, col), 2).transpose() of the column-major message (cost_query_server.py:74)."""
    return np.ascontiguousarray(layer[::-1, ::-1], dtype=np.float32)


class CostNetOracle:
    """dtype=torch.float64 evaluates the same module in double precision (the reference the range tests hold the
    library's fp32-accurate paths to); device: where the parameters and the feature evaluation live."""

    def __init__(self, state_dict: dict, dtype=torch.float32, device="cpu"):
        self.dtype = dtype
        self.p = {k: torch.as_tensor(np.asarray(v), dtype=torch.float32).to(device=device, dtype=dtype)
                  for k, v in state_dict.items() if not k.endswith("num_batches_tracked")}

    def _conv_bn(self, x, conv, bn):
        p = self.p
        y = F.conv2d(x, p[conv + ".weight"])
        return F.batch_norm(y, p[bn + ".running_mean"], p[bn + ".running_var"], p[bn + ".weight"], p[bn + ".bias"],
                            training=False, eps=BN_EPS)

    @torch.no_grad()
    def features(self, E: np.ndarray) -> torch.Tensor:
        """network.CNNpart (network_light.py:78-110); E [rows, cols] -> [48, (rows-48)/2, (cols-48)/2]."""
        dev = self.p["init_conv1.weight"].device
        t = torch.as_tensor(np.asarray(E, dtype=np.float32)).to(device=dev, dtype=self.dtype)[None, None]
        t = self._conv_bn(t, "init_conv1", "init_conv1_bn")
        t = F.leaky_relu(self._conv_bn(t, "init_conv2", "init_conv2_bn"), 0.3)
        t = F.max_pool2d(t, (2, 2), stride=2)
        t = F.leaky_relu(self._conv_bn(t, "init_conv3", "init_conv3_bn"), 0.3)
        t = F.leaky_relu(self._conv_bn(t, "init_conv4", "init_conv4_bn"), 0.3)
        t = F.max_pool2d(t, (3, 3), stride=1)
        t = F.leaky_relu(self._conv_bn(t, "init_conv5", "init_conv5_bn"), 0.3)
        t = F.leaky_relu(self._conv_bn(t, "init_flatten", "init_flatten_bn"), 0.3)
        return t[0]   # dropout is the identity in eval mode

    @torch.no_grad()
    def query(self, feats: torch.Tensor, edges: np.ndarray, res: float, Lx: float, Ly: float, cx: float, cy: float):
        """cost_query_server.py:160-161 + CostQuery.__call__ (cost_query.py:39-69) + network.FCpart.
        edges [n,6] = [tx,ty,tyaw,sx,sy,syaw]; returns [n,3] = (power, time, 1-prob)."""
        p = {k: v.cpu() for k, v in self.p.items()}
        feats = feats.cpu()
        t = torch.as_tensor(np.asarray(edges, dtype=np.float64))
        t = t.clone()
        t[:, 0] -= cx; t[:, 1] -= cy; t[:, 3] -= cx; t[:, 4] -= cy
        t[:, :3] = t[:, :3] - t[:, 3:]
        feat_res = res * DOWNSAMPLE
        row_bias = int((Lx / res - 2 * MAP_CLIP) / DOWNSAMPLE * 0.5)
        col_bias = int((Ly / res - 2 * MAP_CLIP) / DOWNSAMPLE * 0.5)
        Hf, Wf = feats.shape[1], feats.shape[2]
        row = torch.clamp(t[:, 3] / feat_res + row_bias, min=1, max=Hf - 2).long()
        col = torch.clamp(t[:, 4] / feat_res + col_bias, min=1, max=Wf - 2).long()
        f = feats[:, row, col].t().contiguous()                       # [n, 48]
        # [dx, dy, dyaw, syaw]: the module receives them as a float32 tensor (rounded there in either dtype)
        tar = torch.cat((t[:, :3], t[:, 5:6]), dim=1).to(torch.float32).to(self.dtype)
        ang = tar[:, 2]
        # the module compares a float32 tensor with math.pi, i.e. with float32(pi) = 3.1415927 > pi: keep those
        # branch decisions (and the float32 2*pi) in float64 too
        pi32 = float(np.float32(math.pi))
        ang = torch.where(ang > pi32, ang - 2 * pi32, ang)
        ang = torch.where(ang < -pi32, ang + 2 * pi32, ang)
        info = torch.stack((tar[:, 0], tar[:, 1], torch.sqrt(tar[:, 0] ** 2 + tar[:, 1] ** 2),
                            torch.atan2(tar[:, 1], tar[:, 0]), ang, torch.cos(ang), torch.sin(ang),
                            tar[:, 3], torch.cos(tar[:, 3]), torch.sin(tar[:, 3])), dim=1)   # [n, 10]

        def lin_bn(x, conv, bn):
            y = x @ p[conv + ".weight"].reshape(p[conv + ".weight"].shape[0], -1).t()
            s = p[bn + ".weight"] / torch.sqrt(p[bn + ".running_var"] + BN_EPS)
            return (y - p[bn + ".running_mean"]) * s + p[bn + ".bias"]

        def lin_bias(x, conv):
            return x @ p[conv + ".weight"].reshape(1, -1).t() + p[conv + ".bias"]

        tarf = lin_bn(info, "tar0_conv1", "tar0_conv1_bn")
        h = F.leaky_relu(lin_bn(torch.cat((f, tarf), dim=1), "out0_conv1", "out0_conv1_bn"), 0.3)
        power = F.relu(lin_bias(F.leaky_relu(lin_bn(h, "out1_conv1", "out1_conv1_bn"), 0.3), "out2_conv1"))
        tm = F.relu(lin_bias(F.leaky_relu(lin_bn(h, "out1_conv2", "out1_conv2_bn"), 0.3), "out2_conv2"))
        prob = torch.sigmoid(lin_bias(F.leaky_relu(lin_bn(h, "out1_conv3", "out1_conv3_bn"), 0.3), "out2_conv3"))
        return torch.cat((power, tm, 1.0 - prob), dim=1).numpy()


# ---------------------------------------------------------------------------------------------------------------------
# Range testing of the trunk: trained-like weights, an emulation of the library's fp16 split, and a per-element error
# bound. Trunk layer i = (conv, bn, LeakyReLU after it, max-pool (k, stride) after it or None).
TRUNK = [("init_conv1", "init_conv1_bn", False, None), ("init_conv2", "init_conv2_bn", True, (2, 2)),
         ("init_conv3", "init_conv3_bn", True, None), ("init_conv4", "init_conv4_bn", True, (3, 1)),
         ("init_conv5", "init_conv5_bn", True, None), ("init_flatten", "init_flatten_bn", True, None)]
FP16_OVERFLOW = 65520.0   # the smallest magnitude that rounds to fp16 infinity
U22 = 2.0 ** -22


def _calibration_input() -> np.ndarray:
    from art_planner_b200 import synth
    return cnn_input_from_layer(synth.make_fbm_map(128, 128, 0.04, seed=2, amp=0.6).elevation)


def calibrated_state_dict(seed: int = 5, network: str = "light", variant: str | None = None, value: float = 1.0,
                          layers=range(6)) -> dict:
    """costnet.make_state_dict's weights with trained-like BatchNorm statistics: layer by layer, running_mean /
    running_var are the per-channel mean and variance of that layer's conv output on a calibration map (an fBm patch
    around 0 m), as training leaves them, so every activation is O(1) on such maps. The head keeps the generator's
    statistics (its inputs are O(1) already). Deterministic, like the generator. Variants, each in the trunk layers
    `layers` (indices into TRUNK):
      "wscale"  raw conv weights times `value` before calibration;
      "gamma"   BN weights times `value` after it;
      "dead"    channel 1 near-dead: running_var 1e-8, its BN weight set so that its largest folded |w| is `value`;
      "tiny"    channel 2's BN weight set so that its largest folded |w| is `value` (e.g. 1e-6);
      "zero"    channel 3's conv weights all zero."""
    from art_planner_b200 import costnet
    sd = costnet.make_state_dict(seed, network)
    x = torch.as_tensor(_calibration_input(), dtype=torch.float64)[None, None]
    for i, (conv, bn, act, pool) in enumerate(TRUNK):
        w = torch.as_tensor(sd[conv + ".weight"], dtype=torch.float64)
        v = variant if i in layers else None
        if v == "wscale":
            w = w * value
        if v == "zero":
            w[3] = 0.0
        y = F.conv2d(x, w)
        mean, var = y.mean(dim=(0, 2, 3)), y.var(dim=(0, 2, 3), unbiased=False)
        gamma = torch.as_tensor(sd[bn + ".weight"], dtype=torch.float64).clone()
        if v == "gamma":
            gamma = gamma * value
        wmax = w.abs().amax(dim=(1, 2, 3))
        if v == "dead":
            var[1] = 1e-8
            gamma[1] = value * math.sqrt(1e-8 + BN_EPS) / float(wmax[1])
        if v == "tiny":
            gamma[2] = value * math.sqrt(float(var[2]) + BN_EPS) / float(wmax[2])
        sd[conv + ".weight"] = w.numpy().astype(np.float32)
        sd[bn + ".weight"] = gamma.numpy().astype(np.float32)
        sd[bn + ".running_mean"] = mean.numpy().astype(np.float32)
        sd[bn + ".running_var"] = var.numpy().astype(np.float32)
        p = {k: torch.as_tensor(sd[bn + k], dtype=torch.float64) for k in (".weight", ".bias", ".running_mean", ".running_var")}
        x = F.batch_norm(F.conv2d(x, torch.as_tensor(sd[conv + ".weight"], dtype=torch.float64)), p[".running_mean"],
                         p[".running_var"], p[".weight"], p[".bias"], training=False, eps=BN_EPS)
        if act:
            x = F.leaky_relu(x, 0.3)
        if pool:
            x = F.max_pool2d(x, pool[0], stride=pool[1])
    return sd


def _folded(p, conv, bn):
    """float64 BN folding: weights, bias, and |beta| + |mean * scale| (the magnitude the fp32 bias is rounded at)."""
    s = p[bn + ".weight"] / torch.sqrt(p[bn + ".running_var"] + BN_EPS)
    ms = p[bn + ".running_mean"] * s
    return p[conv + ".weight"] * s[:, None, None, None], p[bn + ".bias"] - ms, p[bn + ".bias"].abs() + ms.abs()


def channel_weight_scale(wf: torch.Tensor) -> torch.Tensor:
    """The library's per-output-channel power of two 2^k with max|w| * 2^k in [2^14, 2^15) (tc_scale_kernel)."""
    m = wf.abs().amax(dim=(1, 2, 3)).to(torch.float32)
    e = torch.frexp(m).exponent.to(torch.float64)
    return torch.pow(2.0, torch.clamp(15.0 - e, -100.0, 100.0)).to(wf.dtype)


def _split16(x):
    hi = x.to(torch.float32).to(torch.float16).to(x.dtype)
    return hi, (x.to(torch.float32) - hi.to(torch.float32)).to(torch.float16).to(x.dtype)


def trunk_features_split(state_dict: dict, E: np.ndarray, weight_scale="channel", defect: str | None = None,
                         device="cpu"):
    """Emulation of the tensor-core path's operand representation, in float64 arithmetic: init_conv1 exact (it runs in
    fp32 on CUDA cores), every later conv as a_hi*w_hi + a_hi*w_lo + a_lo*w_hi of the fp16 splits a = fp16(a) +
    fp16(a - hi) and w * scale likewise (scale: the per-channel power of two, or a constant such as the former 1024),
    the scale undone after the sum. It leaves out the tensor core's truncating accumulation. Returns the [C, Hf, Wf]
    features (inf / NaN where a split overflows fp16). `defect` injects one implementation error:
      "drop_alo_whi"  no a_lo * w_hi term;      "drop_wlo"  no w_lo at all;
      "pad_stride"    init_conv2's fp32 output stored with the pixel stride of its wgmma N (32) instead of Cout (24);
      "tap_shift"     init_flatten's tap (7, 7) reads the pixel one to the right."""
    p = {k: torch.as_tensor(np.asarray(v), dtype=torch.float32).to(device=device, dtype=torch.float64)
         for k, v in state_dict.items() if not k.endswith("num_batches_tracked")}
    x = torch.as_tensor(np.asarray(E, dtype=np.float32)).to(device=device, dtype=torch.float64)[None, None]
    for i, (conv, bn, act, pool) in enumerate(TRUNK):
        wf, b, _ = _folded(p, conv, bn)
        wf = wf.to(torch.float32).to(torch.float64)           # the library folds in fp32
        if i == 0:
            y = F.conv2d(x, wf)
        else:
            sc = channel_weight_scale(wf) if weight_scale == "channel" else torch.full((wf.shape[0],), float(weight_scale),
                                                                                        dtype=torch.float64, device=device)
            w_hi, w_lo = _split16(wf * sc[:, None, None, None])
            a_hi, a_lo = _split16(x)
            if defect == "drop_wlo":
                w_lo = torch.zeros_like(w_lo)
            y = F.conv2d(a_hi, w_hi) + F.conv2d(a_hi, w_lo)
            if defect != "drop_alo_whi":
                y = y + F.conv2d(a_lo, w_hi)
            if defect == "tap_shift" and conv == "init_flatten":
                wd = torch.zeros_like(w_hi)
                wd[:, :, 7, 8] = w_hi[:, :, 7, 7] + w_lo[:, :, 7, 7]
                wd[:, :, 7, 7] = -(w_hi[:, :, 7, 7] + w_lo[:, :, 7, 7])
                y = y + F.conv2d(x, wd)
            y = y / sc[None, :, None, None]
        x = y + b[None, :, None, None]
        if act:
            x = F.leaky_relu(x, 0.3)
        if defect == "pad_stride" and conv == "init_conv2" and x.shape[1] % 16:
            C, H, W = x.shape[1:]
            n = -(-C // 16) * 16
            buf = torch.zeros(H * W * n + n, dtype=x.dtype, device=device)
            idx = (torch.arange(H * W, device=device)[:, None] * n + torch.arange(C, device=device)[None, :]).reshape(-1)
            buf[idx] = x[0].permute(1, 2, 0).reshape(-1)
            x = buf[:H * W * C].reshape(1, H, W, C).permute(0, 3, 1, 2)
        if pool:
            x = F.max_pool2d(x, pool[0], stride=pool[1])
    return x[0]


def _chain_abs_sum(a, w, nmain, start=None):
    """sum over the steps of an accumulator chain of |partial sum| for conv(a, w): steps are the taps in row-major
    order and, inside each, 16 input channels at a time (one wgmma K step); tap t adds into accumulator t % nmain."""
    cout, cin, k, _ = w.shape
    oh, ow = a.shape[-2] - k + 1, a.shape[-1] - k + 1
    acc = [torch.zeros((cout, oh, ow), dtype=a.dtype, device=a.device) for _ in range(nmain)]
    if start is not None:
        acc[0] = acc[0] + start[:, None, None]
    total = torch.zeros_like(acc[0])
    for t in range(k * k):
        ky, kx = divmod(t, k)
        for c0 in range(0, cin, 16):
            c1 = min(cin, c0 + 16)
            acc[t % nmain] += torch.einsum("chw,oc->ohw", a[c0:c1, ky:ky + oh, kx:kx + ow], w[:, c0:c1, ky, kx])
            total += acc[t % nmain].abs()
    return total


def trunk_error_bound(state_dict: dict, E: np.ndarray, device="cpu"):
    """float64 features of the trunk and a per-element bound on the error of an fp32-accurate evaluation of it.

    Every layer adds a local error and passes on the error of its input:
        P_l = 2^-22 * (|a| (*) |w| + |beta| + |mean * s| + T_l)  +  sqrt(w^2 (*) P_{l-1}^2),
    with a = the layer's float64 input, w its float64 folded weights, (*) the layer's convolution, P_0 = 0 (the
    elevation is exact in both) and LeakyReLU / max-pool applied to P as to a (both are 1-Lipschitz per element).
      * Operands: the fp32 fold and the fp16 split a = a_hi + a_lo, w = w_hi + w_lo (a_lo, w_lo rounded once more,
        a_lo * w_lo dropped) represent each product to 4 * 2^-24 = 2^-22 of |a||w|: the |a| (*) |w| term.
      * Bias: beta - mean * s in fp32, rounded at 2^-24 of |beta| + |mean * s|, and its add in the epilogue.
      * Accumulation: each step of an accumulator chain (one wgmma K step of 16 products into the fp32 register, or
        one fma) is rounded -- truncated toward zero on the tensor core -- once when the products are aligned to the
        accumulator and once when the sum is normalised, each < 2^-23 of the partial sum: 2^-22 * T_l with
        T_l = sum over the chain's steps of |partial sum| (_chain_abs_sum, in the kernels' order: taps row-major,
        16 channels per step, the 15x15 layer's taps alternating between two accumulators). Round-to-nearest paths
        (the CUDA-core kernels, torch's fp32 conv) err by less: their per-step errors are at most half and unbiased.
      * Propagation: the input error of output element o is sum_i w_i * da_i. The da_i of distinct inputs come from
        distinct roundings, so they add in quadrature (root-sum-square) rather than in absolute value; adding them in
        absolute value would grow the bound by the square root of each layer's fan-in (~15 to ~100) per layer and
        accept any error.
    Returns (features [C, Hf, Wf], bound [C, Hf, Wf], largest |activation| at each of the five fp16 split sites)."""
    p = {k: torch.as_tensor(np.asarray(v), dtype=torch.float32).to(device=device, dtype=torch.float64)
         for k, v in state_dict.items() if not k.endswith("num_batches_tracked")}
    a = torch.as_tensor(np.asarray(E, dtype=np.float32)).to(device=device, dtype=torch.float64)[None]
    P = torch.zeros_like(a)
    site_max = []
    for i, (conv, bn, act, pool) in enumerate(TRUNK):
        wf, b, bmag = _folded(p, conv, bn)
        y = F.conv2d(a[None], wf)[0] + b[:, None, None]
        S = F.conv2d(a[None].abs(), wf.abs())[0]
        T = _chain_abs_sum(a, wf, 2 if conv == "init_flatten" else 1, b if i == 0 else None)
        P = U22 * (S + bmag[:, None, None] + T) + torch.sqrt(F.conv2d((P * P)[None], wf * wf)[0])
        a = F.leaky_relu(y, 0.3) if act else y
        if pool:
            a = F.max_pool2d(a[None], pool[0], stride=pool[1])[0]
            P = F.max_pool2d(P[None], pool[0], stride=pool[1])[0]
        if i < 5:
            site_max.append(float(a.abs().max()))
    return a, P, site_max
