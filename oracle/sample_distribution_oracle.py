"""CPU restatement of the sampler's distribution chain (TEST INFRASTRUCTURE ONLY).

Planner::setUpMapProcessors (art_planner/src/planner.cpp:39-58) with sample_from_distribution builds "sample_probability"
and its CDF with
  Basic::setTraversabilityFilter            art_planner/src/map/processors/basic.cpp:110-125
  computeInverseSampleDensity               art_planner/src/map/processors/sample_density.cpp:12-43
  applyBaseSampleDistribution               art_planner/src/map/processors/probability_distribution.cpp:9-16
  applyMaxUnknownProbability                art_planner/src/map/processors/probability_distribution.cpp:50-91
  computeCumulativeProbabilityDistribution  art_planner/src/map/processors/probability_distribution.cpp:20-46
Every function here defines the arithmetic the device runs (artp_distribution.cuh): float32 numpy operations round once
each, in the order the kernels evaluate them, so the device layers equal these bit for bit. Where the reference leaves
an order open, or OpenCV's float32 blur cannot be pinned, the restatement fixes the device's order:
  * the Gaussian blur is w0 * S0 + sum_{t=1..h} w[t] * (S[t] + S[-t]) in increasing t, first along the contiguous axis of
    the column-major layer (OpenCV's row filter on the cols x rows image of utils.cpp:93-96), then along the other;
    cv2.GaussianBlur agrees within 2e-6 x max(layer) (tests/test_sample_distribution_cpu.py);
  * the cap's double sums are per-row left-to-right sums added in row order; the reference's single row-major running
    sum (`cap_sums_reference`) gives the same multipliers on every test map.
The morphology is oracle/basic_oracle.py's (pinned against cv2 in tests/test_basic_cpu.py).
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

from oracle import basic_oracle as bo

F32 = np.float32


@dataclasses.dataclass(frozen=True)
class DistributionParams:
    """artp_sample_distribution_params; defaults: art_planner_ros/config/params.yaml:49-51, blur radius of planner.cpp:48
    for the yaml robot ((1.31 + 0.65) * 0.25)."""
    use_inverse_vertex_density: bool = True
    density_blur_radius: float = 0.49
    use_max_prob_unknown_samples: bool = True
    max_prob_unknown_samples: float = 0.1


def blur_radius(rp) -> float:
    return (rp.torso_length + rp.torso_width) * 0.25                        # planner.cpp:48


def filter_sizes(rp, res: float):
    """basic.cpp:116-122: the int size arguments of dilateAndErodeMatrix / erodeMatrix (implicit double -> int)."""
    reach = int(math.sqrt(rp.reach_x * rp.reach_x + rp.reach_y * rp.reach_y) / res)
    wall = int(min((rp.torso_length - rp.reach_x) * 0.5, (rp.torso_width - rp.reach_y) * 0.5) / res)
    return reach, wall


def sample_filter(traversability_thresholded, rp, res: float, morph=None):
    """Basic::setTraversabilityFilter -> traversability_sample_filter (float32 F-order). morph: optional (erode, dilate)."""
    er, di = morph if morph else (bo.erode, bo.dilate)
    reach, wall = filter_sizes(rp, res)
    t = np.asfortranarray(traversability_thresholded, dtype=F32)
    return np.asfortranarray(er(er(di(t, reach), reach), wall))


def effective_res(rows: int, res: float) -> float:
    """The resolution the device's index function works with: (rows * res) / rows (the map length over its size)."""
    return (rows * res) / rows


def vertex_histogram(vertex_states, rows: int, cols: int, res: float, cx: float, cy: float):
    """sample_density.cpp:21-31: +1 per vertex in the cell of grid_map getIndex (isInside + getIndexFromPosition, as
    artp_sampler.cuh's map_cell evaluates it); off-map and NaN positions are skipped."""
    s = np.asarray(vertex_states, dtype=np.float64).reshape(-1, 7)
    r = effective_res(rows, res)
    Lx, Ly = rows * r, cols * r
    px, py = s[:, 0], s[:, 1]
    with np.errstate(invalid="ignore"):
        vx = ((px - 0.5 * Lx) - cx) / r
        vy = ((py - 0.5 * Ly) - cy) / r
        tx = -((px - cx) - 0.5 * Lx)
        ty = -((py - cy) - 0.5 * Ly)
        inside = (tx >= 0.0) & (ty >= 0.0) & (tx < Lx) & (ty < Ly)
    row = np.trunc(-np.where(inside, vx, 0.0)).astype(np.int64)
    col = np.trunc(-np.where(inside, vy, 0.0)).astype(np.int64)
    inside &= (row >= 0) & (col >= 0) & (row < rows) & (col < cols)
    n = np.zeros((rows, cols), np.float64)
    np.add.at(n, (row[inside], col[inside]), 1.0)
    return np.asfortranarray(n.astype(F32))


def blur_size(radius: float, res: float):
    """sample_density.cpp:33-35: (ksize, sigma) in cells."""
    k = int(6 * radius / res)
    if k % 2 == 0:
        k += 1
    return k, radius / res


def gaussian_kernel(ksize: int, sigma: float) -> np.ndarray:
    """getGaussianKernel(ksize, sigma, CV_32F) for sigma > 0: exp(-x^2 / (2 sigma^2)) at x = i - (ksize - 1) / 2 in double,
    normalised by the double sum, cast to float."""
    sc = -0.5 / (sigma * sigma)
    v = [math.exp(sc * ((i - (ksize - 1) * 0.5) * (i - (ksize - 1) * 0.5))) for i in range(ksize)]
    tot = 0.0
    for t in v:
        tot += t
    inv = 1.0 / tot
    return np.array([t * inv for t in v], F32)


def reflect101(p: np.ndarray, n: int) -> np.ndarray:
    """cv::borderInterpolate(BORDER_REFLECT_101), reflecting as often as needed."""
    if n == 1:
        return np.zeros_like(p)
    p = p.copy()
    while True:
        bad = (p < 0) | (p >= n)
        if not bad.any():
            return p
        p = np.where(p < 0, -p, np.where(p >= n, 2 * n - 2 - p, p))


def _pass(a: np.ndarray, w: np.ndarray, axis: int) -> np.ndarray:
    h = len(w) // 2
    n = a.shape[axis]
    idx = np.arange(n)
    take = lambda off: np.take(a, reflect101(idx + off, n), axis=axis)
    s = (w[h] * a).astype(F32)
    for t in range(1, h + 1):
        s = (s + w[h + t] * (take(t) + take(-t))).astype(F32)
    return s


def gaussian_blur(n_samples, ksize: int, sigma: float) -> np.ndarray:
    """gaussianBlurMatrix (utils.cpp:90-110) restated: first along axis 0 (the contiguous one), then along axis 1."""
    w = gaussian_kernel(ksize, sigma)
    a = np.asarray(n_samples, dtype=F32)
    return np.asfortranarray(_pass(_pass(a, w, 0), w, 1))


def combine(n_blur, sample_filter_layer=None):
    """sample_density.cpp:39-42 + probability_distribution.cpp:10-15: max - n unless every |n| <= 1e-5 (Eigen's isZero at
    float precision) or there is no density (n_blur None); then 1. Times the filter when one is set."""
    if n_blur is None or not (np.abs(n_blur) > F32(1e-5)).any():
        p = np.ones(np.shape(sample_filter_layer) if n_blur is None else n_blur.shape, F32)
    else:
        p = (n_blur.max() - n_blur).astype(F32)
    if sample_filter_layer is not None:
        p = (p * np.asarray(sample_filter_layer, F32)).astype(F32)
    return np.asfortranarray(p)


def cap_sums(prob, observed):
    """(known, unknown) double sums in the device's order: per row left to right, the rows added in row order."""
    p = np.asarray(prob, F32).astype(np.float64)
    obs = np.asarray(observed, F32) > 0
    kr, ur = np.zeros(p.shape[0]), np.zeros(p.shape[0])
    for j in range(p.shape[1]):
        kr = kr + np.where(obs[:, j], p[:, j], 0.0)
        ur = ur + np.where(obs[:, j], 0.0, p[:, j])
    return float(np.cumsum(kr)[-1]), float(np.cumsum(ur)[-1])


def cap_sums_reference(prob, observed):
    """The reference's one running sum over i, then j (probability_distribution.cpp:61-71)."""
    p = np.asarray(prob, F32).astype(np.float64)
    obs = np.asarray(observed, F32) > 0
    return float(np.cumsum(np.where(obs, p, 0.0).ravel(order="C"))[-1]), float(np.cumsum(np.where(obs, 0.0, p).ravel(order="C"))[-1])


def cap_multipliers(known: float, unknown: float, max_unknown: float):
    """:73-87: (known_mult, unknown_mult, applied) as the float prob_unknown_mult layer holds them."""
    base = unknown / (known + unknown) if (known + unknown) != 0 else math.nan
    if known > 0 and unknown > 0 and base > max_unknown:
        return F32((1 - max_unknown) / known), F32(max_unknown / unknown), True
    return F32(1.0), F32(1.0), False


def apply_cap(prob, observed, max_unknown: float, sums=cap_sums):
    km, um, _ = cap_multipliers(*sums(prob, observed), max_unknown)
    obs = np.asarray(observed, F32) > 0
    return np.asfortranarray((np.asarray(prob, F32) * np.where(obs, km, um).astype(F32)).astype(F32))


def cdf(prob):
    """computeCumulativeProbabilityDistribution in the device's order (cdf_rows_kernel / cdf_rowwise_kernel): row sums
    left to right, cum = p / s + run; the row distribution sequentially. Returns (cum_prob F-order, cum_prob_rowwise)."""
    p = np.asarray(prob, F32)
    rows, cols = p.shape
    with np.errstate(invalid="ignore", divide="ignore"):
        s = p[:, 0].copy()
        for j in range(1, cols):
            s = (s + p[:, j]).astype(F32)
        cum = np.empty((rows, cols), F32, order="F")
        run = (p[:, 0] / s).astype(F32)
        cum[:, 0] = run
        for j in range(1, cols):
            run = (p[:, j] / s + run).astype(F32)
            cum[:, j] = run
        tot = F32(s[0])
        for i in range(1, rows):
            tot = F32(tot + s[i])
        row = np.empty(rows, F32)
        r = F32(s[0] / tot)
        row[0] = r
        for i in range(1, rows):
            r = F32(F32(s[i] / tot) + r)
            row[i] = r
    return cum, row


def distribution(vertex_states, m, dp: DistributionParams, sample_filter_layer=None, observed=None, blur=None, sums=cap_sums):
    """The chain after the filter: returns dict of n_samples, n_blur, sample_probability, cum_prob, cum_prob_rowwise.
    m: the map (rows, cols, res, cx, cy). blur: optional replacement of gaussian_blur (e.g. cv2's)."""
    out = {}
    n_blur = None
    if dp.use_inverse_vertex_density:
        out["n_samples"] = vertex_histogram(vertex_states, m.rows, m.cols, m.res, m.cx, m.cy)
        k, sigma = blur_size(dp.density_blur_radius, m.res)
        n_blur = (blur or gaussian_blur)(out["n_samples"], k, sigma)
        out["n_blur"] = n_blur
    prob = combine(n_blur, sample_filter_layer) if (n_blur is not None or sample_filter_layer is not None) \
        else np.ones((m.rows, m.cols), F32, order="F")
    if dp.use_max_prob_unknown_samples:
        prob = apply_cap(prob, observed, dp.max_prob_unknown_samples, sums)
    out["sample_probability"] = prob
    out["cum_prob"], out["cum_prob_rowwise"] = cdf(prob)
    return out
