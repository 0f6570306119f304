"""Layers for inpaintMatrix (oracle/inpaint_oracle.py, csrc/artp_inpaint.cuh): rows x cols float32 grid_map layers with
NaN holes. Every case is deterministic; oracle/make_golden_inpaint.py stores cv2's result of each in
tests/golden/inpaint.npz."""
import numpy as np


def _field(rows, cols, seed, noise=0.0):
    rng = np.random.default_rng(seed)
    i, j = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    a = np.sin(i * 0.31 + rng.uniform(0, 6)) * 0.8 + np.cos(j * 0.23 + rng.uniform(0, 6)) * 0.6 + 0.01 * i * j / (rows + cols)
    a = a + noise * rng.standard_normal((rows, cols))
    return np.asfortranarray(a.astype(np.float32) * np.float32(1.7) + np.float32(0.4))


def _holes(a, cells):
    a = a.copy(order="F")
    for i, j in cells:
        a[i, j] = np.nan
    return a


def single_cells():
    a = _field(23, 17, 1)
    return _holes(a, [(3, 4), (10, 10), (17, 3), (20, 14), (6, 13)])


def borders():
    a = _field(19, 21, 2, noise=0.05)
    for i, j in [(0, 0), (0, 10), (18, 20), (9, 0), (5, 20), (18, 7), (0, 20), (1, 1), (2, 5)]:
        a[i, j] = np.nan
    a[10:13, 0:2] = np.nan
    a[0:2, 14:17] = np.nan
    return a


def near_pair():   # Chebyshev gap 7 between the holes: one interaction component
    a = _field(30, 30, 3)
    a[10:13, 5:8] = np.nan
    a[10:13, 14:17] = np.nan
    return a


def far_pair():    # gap 8: two components
    a = _field(30, 30, 4)
    a[10:13, 5:8] = np.nan
    a[10:13, 15:18] = np.nan
    return a


def unobserved():
    a = _field(44, 52, 5, noise=0.02)
    a[:, 38:] = np.nan
    a[5:14, 6:15] = np.nan
    a[30:33, 20:40] = np.nan
    return a


def random_mask(frac, seed, rows=37, cols=29, noise=0.1):
    a = _field(rows, cols, seed, noise=noise)
    rng = np.random.default_rng(100 + seed)
    a[rng.random(a.shape) < frac] = np.nan
    return a


def infinities():
    a = _field(21, 26, 6)
    a[3, 3] = np.inf
    a[7, 12] = -np.inf
    a[15:17, 4:6] = np.nan
    a[8, 12] = np.nan
    a[6:9, 20] = np.inf
    a[7, 19] = np.nan
    return a


def constant():
    a = np.full((15, 18), 2.25, np.float32, order="F")
    a[4:7, 5:9] = np.nan
    return a


def non_square(rows, cols, seed):
    a = _field(rows, cols, seed, noise=0.03)
    rng = np.random.default_rng(200 + seed)
    a[rng.random(a.shape) < 0.12] = np.nan
    a[rows // 3:rows // 3 + 4, cols // 2:cols // 2 + 3] = np.nan
    return a


def giant(n=160, hole=100):   # one component of 10^4 cells: larger than any on-chip front
    a = _field(n, n, 9, noise=0.01)
    o = (n - hole) // 2
    a[o:o + hole, o:o + hole] = np.nan
    return a


CASES = {
    "single_cells": single_cells,
    "borders": borders,
    "near_pair": near_pair,
    "far_pair": far_pair,
    "unobserved": unobserved,
    "random_01": lambda: random_mask(0.01, 1),
    "random_10": lambda: random_mask(0.10, 2),
    "random_30": lambda: random_mask(0.30, 3, noise=0.5),
    "infinities": infinities,
    "constant": constant,
    "tall_odd": lambda: non_square(31, 13, 7),
    "wide_odd": lambda: non_square(13, 31, 8),
}
LARGE_CASES = {"giant": giant}   # 10^4 cells in one component: the pure-Python oracle takes seconds on it


def profile_layer(n, pattern, frac=0.14, seed=0):
    """The layers of profiles/inpaint_time.py: a smooth n x n field with `holes` = scattered 20 x 20-cell holes,
    `strip` = one unobserved strip 10 % of the map wide, or `both`."""
    rng = np.random.default_rng(seed)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    a = (np.sin(i * 0.013) + np.cos(j * 0.011) + 0.05 * rng.standard_normal((n, n))).astype(np.float32)
    m = np.zeros((n, n), bool)
    if pattern in ("holes", "both"):
        k = int(frac * n * n / 400)
        for x, y in zip(rng.integers(0, n - 20, k), rng.integers(0, n - 20, k)):
            m[x:x + 20, y:y + 20] = True
    if pattern in ("strip", "both"):
        m[:, : n // 10] = True
    a[m] = np.nan
    return np.asfortranarray(a)


# The one known divergence of the restatement from cv2 (DESIGN.md section 4.6): a 120 x 120 crop of the 8-bit image
# inpaintMatrix makes from profile_layer(1000, "holes") (image rows 0-119, columns 380-499). cv2.inpaint differs from
# oracle.inpaint_oracle.telea on 6 cells of it. The golden file stores the crop's image, mask and cv2's result.
DIVERGENCE_CROP = (slice(0, 120), slice(380, 500))
