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


# ---- map-scale layers (tests/test_inpaint_scale_gpu.py; small versions in tests/test_inpaint_components_cpu.py) ----

DIRECTIONS = {"h": (0, 1), "v": (1, 0), "d": (1, 1), "a": (1, -1)}


def hole_pair(direction, gap, block_first):
    """Cells of a one-cell hole and a 2 x 2 hole at Chebyshev distance `gap` along `direction` (the 2 x 2 hole first
    when `block_first`), shifted to start at row / column 0."""
    di, dj = DIRECTIONS[direction]
    block = [(0, 0), (0, 1), (1, 0), (1, 1)]
    if block_first:
        a = block
        b = [(di * (gap + 1) if di > 0 else 0, dj * (gap + 1) if dj > 0 else dj * gap)]
    else:
        a = [(0, 0)]
        b = [(di * gap + y, dj * gap + x - (1 if dj < 0 else 0)) for y, x in block]
    cells = np.array(a + b)
    cells -= cells.min(0)
    na = len(a)
    d = np.abs(cells[:na, None, :] - cells[None, na:, :]).max(-1).min()
    assert d == gap, (direction, gap, block_first, d)
    return cells[:na], cells[na:]


def gap_lattice(rows=1000, cols=1000, gaps=(7, 8), tile=18, seed=10, border=False):
    """Hole pairs on a tile x tile lattice, every (direction, gap, order) in turn in a seeded shuffle; one pair per
    tile at the tile's origin. A pair spans at most max(gaps) + 2 cells, so with tile >= max(gaps) + 10 pairs of
    neighbouring tiles are at least 8 apart: each pair at gap <= 7 is one interaction component, at gap >= 8 two.
    With `border`, the layer is cropped to the holes, so pairs touch all four borders.
    Returns (layer, pairs) with pairs = [(a cells, b cells, gap)] in layer (row, col) coordinates."""
    assert tile >= max(gaps) + 10
    rng = np.random.default_rng(seed)
    kinds = [(d, g, o) for d in DIRECTIONS for g in gaps for o in (False, True)]
    ti, tj = -(-rows // tile), -(-cols // tile)
    pick = rng.permutation(np.arange(ti * tj) % len(kinds))
    pairs = []
    for t in range(ti * tj):
        a, b = hole_pair(*kinds[pick[t]])
        o = np.array([(t // tj) * tile, (t % tj) * tile])
        a, b = a + o, b + o
        if np.concatenate([a, b]).max(0)[0] < rows and np.concatenate([a, b]).max(0)[1] < cols:
            pairs.append((a, b, kinds[pick[t]][1]))
    a = _field(rows, cols, seed, noise=0.2)
    for p, q, _ in pairs:
        a[p[:, 0], p[:, 1]] = np.nan
        a[q[:, 0], q[:, 1]] = np.nan
    if border:
        cells = np.concatenate([np.concatenate(p[:2]) for p in pairs])
        hi = cells.max(0) + 1
        a = np.asfortranarray(a[:hi[0], :hi[1]])
    return a, pairs


def size_ladder(rows=997, cols=613, sides=(1, 2, 6, 12, 20, 30, 50, 70, 100, 130), step=9, seed=11):
    """One square hole of each side in `sides` (interaction components of (side + 6)^2 cells: one per power-of-two
    size class from 2^5 up; side 130 is class 2^14), a one-cell hole in the corner (class 2^4, a clipped 4 x 4 region)
    and two on the borders (4 x 7), then a lattice of 1- and 2-cell holes every `step` cells on the columns right
    of the squares: several components of each small class, and more components than the march launches warps."""
    assert step >= 9
    a = _field(rows, cols, seed, noise=0.1)
    rng = np.random.default_rng(seed)
    i = 10
    for s in sides:
        a[i:i + s, 10:10 + s] = np.nan
        i += s + 10
    assert i <= rows, "the ladder does not fit"
    a[0, 0] = np.nan
    a[rows // 2, cols - 1] = np.nan
    a[rows - 1, 5] = np.nan
    j0 = 10 + max(sides) + 10
    for ii in range(0, rows - 1, step):
        for jj in range(j0, cols - 2, step):
            k = rng.integers(0, 3)
            a[ii, jj] = np.nan
            if k == 1:
                a[ii + 1, jj] = np.nan
            elif k == 2:
                a[ii, jj + 1] = np.nan
    return a


def long_thin(rows=800, cols=700, seed=12, spiral=61):
    """Long components whose bounding box is far larger than their cell count: a 1-cell diagonal line, a zig-zag
    line of 8-connected diagonal runs, and a square spiral of 1-cell arms 2 apart (a long march through many equal
    T values)."""
    a = _field(rows, cols, seed, noise=0.1)
    n = min(rows, cols) // 2 - 20
    k = np.arange(n)
    a[10 + k, 10 + k] = np.nan
    i = np.arange(10, rows - 10)
    amp = max(4, (cols - n - 60) // 2)
    tri = np.abs((i % (2 * amp)) - amp)
    a[i, cols - 10 - tri] = np.nan
    # the spiral: walk right, down, left, up with arm lengths shrinking by 2 every two turns
    y, x = rows - spiral - 10, 10
    length, d = spiral - 1, 0
    steps = [(0, 1), (1, 0), (0, -1), (-1, 0)]
    a[y, x] = np.nan
    while length > 0:
        for _ in range(length):
            y, x = y + steps[d][0], x + steps[d][1]
            a[y, x] = np.nan
        if d % 2 == 1:
            length -= 2
        d = (d + 1) % 4
    return a


def thin_layer(rows, cols, seed=13):
    """A layer 2-5 cells thin: NaN in the four corners, a hole across the whole width at both ends' second cell,
    and 1-cell holes 8 apart along the length (as many components as the width allows) with a few gaps."""
    a = _field(rows, cols, seed, noise=0.1)
    t = a if rows <= cols else a.T                     # a view: thin x long
    w, n = t.shape
    for y in (0, w - 1):
        for x in (0, n - 1):
            t[y, x] = np.nan
    t[:, 2] = np.nan
    t[:, n - 3] = np.nan
    rng = np.random.default_rng(seed)
    for x in range(12, n - 12, 8):
        if rng.random() < 0.85:
            t[rng.integers(0, w), x] = np.nan
    return np.asfortranarray(a)


def scattered(rows, cols, n_holes, seed=14):
    """Seeded 1-20-cell rectangles across the layer, plus holes in the four corners and on each border."""
    a = _field(rows, cols, seed, noise=0.1)
    rng = np.random.default_rng(seed)
    h = rng.integers(1, 5, n_holes)
    w = np.minimum(rng.integers(1, 21, n_holes), 20 // h)
    y = rng.integers(0, rows - h + 1)
    x = rng.integers(0, cols - w + 1)
    for yy, xx, hh, ww in zip(y, x, h, w):
        a[yy:yy + hh, xx:xx + ww] = np.nan
    for yy, xx in ((0, 0), (0, cols - 2), (rows - 3, 0), (rows - 1, cols - 1)):
        a[yy:yy + 3, xx:xx + 2] = np.nan
    a[0, cols // 3] = a[rows - 1, cols // 2] = a[rows // 3, 0] = a[rows // 2, cols - 1] = np.nan
    return a


def near_constant(ulps, rows=300, cols=257, seed=15, base=np.float32(37.25)):
    """A layer whose finite cells lie within `ulps` float steps above `base`, with scattered holes: the 8-bit
    conversion's multiply-add then lands near byte midpoints, where a fused and an unfused one round differently."""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, ulps + 1, (rows, cols)).astype(np.uint32)
    k[0, 0], k[-1, -1] = 0, ulps
    a = (np.uint32(np.float32(base).view(np.uint32)) + k).view(np.float32)
    a = np.asfortranarray(a)
    hole = rng.random((rows, cols)) < 0.05
    hole[0, 0] = hole[-1, -1] = False
    a[hole] = np.nan
    return a


# The one known divergence of the restatement from cv2 (DESIGN.md section 4.6): a 120 x 120 crop of the 8-bit image
# inpaintMatrix makes from profile_layer(1000, "holes") (image rows 0-119, columns 380-499). cv2.inpaint differs from
# oracle.inpaint_oracle.telea on 6 cells of it. The golden file stores the crop's image, mask and cv2's result.
DIVERGENCE_CROP = (slice(0, 120), slice(380, 500))
