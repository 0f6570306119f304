"""CPU oracle of inpaintMatrix (art_planner/src/utils.cpp:13-63) (TEST INFRASTRUCTURE ONLY).

Restates the whole chain on a column-major float layer: the finite min / max, the NaN mask (the patchNaNs 128 / 200
workaround masks NaN cells only, never +-inf), convertTo(CV_8U), cv::inpaint(radius 3, INPAINT_TELEA) on the cols x rows
image of the column-major layer, convertTo(CV_32F), the scale and offset back, and the column / row 0 copies.

`telea` is OpenCV's icvTeleaInpaintFMM written from the published algorithm (Telea 2004; the CvPriorityQueueFloat /
FastMarching_solve / icvCalcFMM structure) with every operation at the precision the library uses. Points that decide
bit equality with cv2.inpaint (4.13), each found by bisecting on one- and two-cell holes against the library:
  * the queue pops in (T, push order): equal T leave first-in first-out, the initial band in raster order;
  * the outer pass (icvCalcFMM with negated T) runs over the ring the 7 x 7 dilation adds, seeded with the band;
  * Ia reads the known pixel itself (out[k-1, l-1]); only the image gradient's reads use the clamped km / kp / lm / lp,
    and its central differences carry OpenCV's factor 2 (not 1/2);
  * dst, lev and FastMarching_solve round through double; everything else, and the final sum, is float; the result is
    saturate_cast<uchar> (round half to even).
convertTo(CV_8U) fuses the multiply and add (the library's FMA path on hosts with FMA3, which cv2 takes here); a non-finite
or out-of-int-range product converts to 0. tests/test_inpaint_cpu.py pins all of it against cv2 where it is importable.
"""
from __future__ import annotations

import heapq
from fractions import Fraction

import numpy as np

f32 = np.float32
KNOWN, BAND, INSIDE, CHANGE = 0, 1, 2, 3
RANGE = 3


def _solve(a11, f1, a22, f2):
    """FastMarching_solve: double arithmetic on the two float T values, rounded to float."""
    a11 = float(a11)
    a22 = float(a22)
    m12 = min(a11, a22)
    if f1 != INSIDE:
        if f2 != INSIDE:
            if abs(a11 - a22) >= 1.0:
                s = 1 + m12
            else:
                s = (a11 + a22 + np.sqrt(2 - (a11 - a22) * (a11 - a22))) * 0.5
        else:
            s = 1 + a11
    elif f2 != INSIDE:
        s = 1 + a22
    else:
        s = 1 + m12
    return f32(s)


def _dist4(i, j, f, t):
    def s(a, b, c, d):
        return _solve(t[a, b], f[a, b], t[c, d], f[c, d])
    return min(min(s(i - 1, j, i, j - 1), s(i + 1, j, i, j - 1)), min(s(i - 1, j, i, j + 1), s(i + 1, j, i, j + 1)))


def _dilate(m, r):
    """Binary dilation by a (2r+1)^2 square (r=1 with `cross` for the 4-neighbour cross); outside cells take no part."""
    R, C = m.shape
    p = np.zeros((R + 2 * r, C + 2 * r), bool)
    p[r:r + R, r:r + C] = m
    out = np.zeros_like(m, bool)
    for di in range(-r, r + 1):
        for dj in range(-r, r + 1):
            out |= p[r + di:r + di + R, r + dj:r + dj + C]
    return out


def _cross(m):
    R, C = m.shape
    p = np.zeros((R + 2, C + 2), bool)
    p[1:-1, 1:-1] = m
    return m | p[:-2, 1:-1] | p[2:, 1:-1] | p[1:-1, :-2] | p[1:-1, 2:]


def _fmm_outer(f, t, seeds, R, C):
    """icvCalcFMM(out, t, Out, negate=true): f holds INSIDE on the ring to march."""
    heap = [(f32(0), n, i, j) for n, (i, j) in enumerate(seeds)]
    cnt = len(heap)
    while heap:
        _, _, ii, jj = heapq.heappop(heap)
        f[ii, jj] = CHANGE
        for i, j in ((ii - 1, jj), (ii, jj - 1), (ii + 1, jj), (ii, jj + 1)):
            if i <= 0 or j <= 0 or i > R or j > C:
                continue
            if f[i, j] == INSIDE:
                d = _dist4(i, j, f, t)
                t[i, j] = d
                f[i, j] = BAND
                heapq.heappush(heap, (d, cnt, i, j))
                cnt += 1
    m = f == CHANGE
    f[m] = KNOWN
    t[m] = -t[m]


def telea(img: np.ndarray, mask: np.ndarray) -> np.ndarray:
    """cv::inpaint(img, mask, dst, 3, INPAINT_TELEA) for a uint8 single-channel image (mask != 0 = unknown)."""
    img = np.asarray(img, np.uint8)
    H, W = img.shape
    R, C = H + 2, W + 2
    out = img.astype(np.int64)
    msk = np.zeros((R, C), bool)
    msk[1:-1, 1:-1] = np.asarray(mask) != 0
    if not msk.any():
        return img.copy()
    t = np.full((R, C), f32(1e6), np.float32)
    interior = np.zeros((R, C), bool)
    interior[1:-1, 1:-1] = True
    band = _cross(msk) & ~msk & interior
    seeds = list(zip(*np.nonzero(band)))                     # raster order
    t[band] = 0
    ring = _dilate(msk, RANGE) & ~msk & ~band & interior
    fo = np.where(ring, INSIDE, KNOWN).astype(np.uint8)
    _fmm_outer(fo, t, seeds, R, C)
    f = np.where(msk, INSIDE, KNOWN).astype(np.uint8)
    heap = [(f32(0), n, i, j) for n, (i, j) in enumerate(seeds)]
    cnt = len(heap)
    rr = RANGE * RANGE
    while heap:
        _, _, ii, jj = heapq.heappop(heap)
        f[ii, jj] = KNOWN
        for i, j in ((ii - 1, jj), (ii, jj - 1), (ii + 1, jj), (ii, jj + 1)):
            if i <= 0 or j <= 0 or i > R - 1 or j > C - 1 or f[i, j] != INSIDE:
                continue
            d = _dist4(i, j, f, t)
            t[i, j] = d
            tij = t[i, j]
            if f[i, j + 1] != INSIDE:
                gx = f32(t[i, j + 1] - t[i, j - 1]) * f32(0.5) if f[i, j - 1] != INSIDE else f32(t[i, j + 1] - tij)
            else:
                gx = f32(tij - t[i, j - 1]) if f[i, j - 1] != INSIDE else f32(0)
            if f[i + 1, j] != INSIDE:
                gy = f32(t[i + 1, j] - t[i - 1, j]) * f32(0.5) if f[i - 1, j] != INSIDE else f32(t[i + 1, j] - tij)
            else:
                gy = f32(tij - t[i - 1, j]) if f[i - 1, j] != INSIDE else f32(0)
            Ia = Jx = Jy = f32(0)
            s = f32(1e-20)
            for k in range(i - RANGE, i + RANGE + 1):
                km = k - 1 + (k == 1)
                kp = k - 1 - (k == R - 2)
                for l in range(j - RANGE, j + RANGE + 1):
                    lm = l - 1 + (l == 1)
                    lp = l - 1 - (l == C - 2)
                    if not (0 < k < R - 1 and 0 < l < C - 1):
                        continue
                    if f[k, l] == INSIDE or (l - j) ** 2 + (k - i) ** 2 > rr:
                        continue
                    ry = f32(i - k)
                    rx = f32(j - l)
                    vl = f32(rx * rx + ry * ry)
                    dst = f32(1.0 / (float(vl) * np.sqrt(float(vl))))
                    lev = f32(1.0 / float(f32(1) + abs(f32(t[k, l] - tij))))
                    dr = f32(rx * gx + ry * gy)
                    if abs(float(dr)) <= 0.01:
                        dr = f32(1e-6)
                    w = abs(f32(dst * lev) * dr)
                    if f[k, l + 1] != INSIDE:
                        gix = f32(out[km, lp + 1] - out[km, lm - 1]) * f32(2) if f[k, l - 1] != INSIDE else f32(out[km, lp + 1] - out[km, lm])
                    else:
                        gix = f32(out[km, lp] - out[km, lm - 1]) if f[k, l - 1] != INSIDE else f32(0)
                    if f[k + 1, l] != INSIDE:
                        giy = f32(out[kp + 1, lm] - out[km - 1, lm]) * f32(2) if f[k - 1, l] != INSIDE else f32(out[kp + 1, lm] - out[km, lm])
                    else:
                        giy = f32(out[kp, lm] - out[km - 1, lm]) if f[k - 1, l] != INSIDE else f32(0)
                    Ia = f32(Ia + w * f32(out[k - 1, l - 1]))
                    Jx = f32(Jx - w * f32(gix * rx))
                    Jy = f32(Jy - w * f32(giy * ry))
                    s = f32(s + w)
            sat = f32(f32(Ia / s) + f32((Jx + Jy) / f32(np.sqrt(f32(Jx * Jx + Jy * Jy)) + f32(1e-20)))) + f32(0.5)
            out[i - 1, j - 1] = min(255, max(0, int(np.rint(sat))))
            f[i, j] = BAND
            heapq.heappush(heap, (d, cnt, i, j))
            cnt += 1
    return out.astype(np.uint8)


def to_u8(x: np.ndarray, alpha: np.float32, beta: np.float32) -> np.ndarray:
    """convertTo(CV_8U, alpha, beta) of float cells: saturate_cast<uchar>(fma(x, alpha, beta)) in float; a non-finite
    or out-of-int-range value (cvRound's INT_MIN) converts to 0."""
    x = np.asarray(x, np.float32)
    with np.errstate(all="ignore"):
        d = x.astype(np.float64) * np.float64(alpha) + np.float64(beta)   # product exact; one rounding to double
        v = d.astype(np.float32)
        # a double landing exactly on a float midpoint may have rounded twice: redo those exactly
        lo = np.nextafter(v, np.float32(-np.inf)); hi = np.nextafter(v, np.float32(np.inf))
        mid = np.isfinite(d) & ((d == (v.astype(np.float64) + lo) / 2) | (d == (v.astype(np.float64) + hi) / 2))
    for idx in zip(*np.nonzero(mid)):
        e = Fraction(float(x[idx])) * Fraction(float(alpha)) + Fraction(float(beta))
        c = [lo[idx], v[idx], hi[idx]]
        v[idx] = min(c, key=lambda q: (abs(Fraction(float(q)) - e), int(np.float32(q).view(np.uint32)) & 1))
    a = np.abs(v.astype(np.float64))
    ok = np.isfinite(v) & (a < 2.0 ** 31)
    r = np.rint(np.where(ok, v, 0).astype(np.float64))
    return np.where(ok, np.clip(r, 0, 255), 0).astype(np.uint8)


def interaction_components(mask: np.ndarray):
    """The interaction components of a mask: the 8-connected components of the mask dilated by the 7 x 7 square.
    Returns (labels, n) as scipy.ndimage.label does: 0 outside every component, ids 1..n."""
    from scipy import ndimage
    return ndimage.label(_dilate(np.asarray(mask) != 0, RANGE), structure=np.ones((3, 3), bool))


def telea_by_components(img: np.ndarray, mask: np.ndarray, margin: int = 4, components=None, labels=None):
    """telea(img, mask), one interaction component at a time: each component's cells come from telea run on the
    component's bounding box widened by `margin` cells (clipped to the image) with only that component's mask cells.
    Returns (result, labels); with `components` (an iterable of ids) only those components are inpainted and every
    other mask cell keeps its input byte. `labels` may pass interaction_components(mask)[0] to skip the labelling.

    Why it equals the whole-image march for any margin >= 1: the component's box already holds every cell within
    Chebyshev distance 3 of its mask. Inpainting a cell reads f, t and the image only within distance 4 of it (the
    radius-3 window, then one more cell for the image gradient's and FastMarching_solve's neighbours), and the outer
    pass marches only the ring within 3 of the mask, so with margin >= 1 every read lands inside the crop and no other
    component's cell is within reach (two components' masks are at least 8 apart). The gradient's km / kp / lm / lp
    clamps act on a window cell in the crop's first or last row or column; a window cell is within 3 of the mask, so
    that is the crop's edge only where the crop edge is the true image border. Within the crop, the queue's (T, push
    order) keeps the same relative order as the whole image's: the band is pushed in raster order in both, and the
    interleaving with other components' cells never changes what this component reads."""
    img = np.asarray(img, np.uint8)
    m = np.asarray(mask) != 0
    if labels is None:
        labels, n = interaction_components(m)
    else:
        n = int(labels.max())
    from scipy import ndimage
    boxes = ndimage.find_objects(labels)
    out = img.copy()
    H, W = img.shape
    ids = range(1, n + 1) if components is None else components
    for c in ids:
        sy, sx = boxes[c - 1]
        y0, y1 = max(sy.start - margin, 0), min(sy.stop + margin, H)
        x0, x1 = max(sx.start - margin, 0), min(sx.stop + margin, W)
        cm = m[y0:y1, x0:x1] & (labels[y0:y1, x0:x1] == c)
        res = telea(img[y0:y1, x0:x1], cm)
        out[y0:y1, x0:x1][cm] = res[cm]
    return out, labels


def to_image(layer: np.ndarray):
    """inpaintMatrix up to the march: (NaN mask, 8-bit image, both cols x rows; the finite min; the scale back;
    whether the finite cells are all equal, which skips the march). Raises ValueError for a layer without a finite cell (the C ABI's ARTP_E_INVALID)."""
    mat = np.asfortranarray(np.asarray(layer, np.float32))
    fin = np.isfinite(mat)
    if not fin.any():
        raise ValueError("layer has no finite cell")
    mn = f32(mat[fin].min())
    mx = f32(mat[fin].max())
    img_f = np.ascontiguousarray(mat.T)                      # cols x rows image of the column-major layer
    mask = np.isnan(img_f)
    with np.errstate(all="ignore"):
        rng_ = f32(mx - mn)
        alpha = f32(f32(255) / rng_)
        beta = f32(f32(f32(-mn) * f32(255)) / rng_)
        scale = f32(rng_ / f32(255))
    u8 = to_u8(img_f, alpha, beta) if mx != mn else np.zeros(img_f.shape, np.uint8)
    return mask, u8, mn, scale, mx == mn


def from_image(res: np.ndarray, mn: np.float32, scale: np.float32) -> np.ndarray:
    """inpaintMatrix after the march: the cols x rows 8-bit image back to a column-major float layer (two float
    operations), then the column / row 0 copies."""
    with np.errstate(all="ignore"):
        back = (res.astype(np.float32) * scale) + mn           # two float operations
    out = np.asfortranarray(back.T).astype(np.float32)
    out[:, 0] = out[:, 1]
    out[0, :] = out[1, :]
    return out


def inpaint_matrix(layer: np.ndarray) -> np.ndarray:
    """inpaintMatrix of a rows x cols float32 grid_map layer; returns the inpainted layer (column-major, float32).
    Raises ValueError for a layer without a finite cell (the C ABI's ARTP_E_INVALID)."""
    mask, u8, mn, scale, const = to_image(layer)
    return from_image(u8 if const else telea(u8, mask), mn, scale)


def inpaint_matrix_by_components(layer: np.ndarray, margin: int = 4, components=None, labels=None):
    """inpaint_matrix through telea_by_components. Returns (inpainted layer, labels) where labels is the interaction
    components' label image in the layer's rows x cols shape (0 outside every component). With `components`, mask
    cells of the other components keep the 8-bit conversion's byte of NaN (0), so only cells outside those
    components' masks and inside the chosen ones are inpaintMatrix's. `labels` may pass layer_components(layer)."""
    mask, u8, mn, scale, const = to_image(layer)
    lab = interaction_components(mask)[0] if labels is None else np.ascontiguousarray(np.asarray(labels).T)
    if const:
        return from_image(u8, mn, scale), lab.T
    res, lab = telea_by_components(u8, mask, margin, components, lab)
    return from_image(res, mn, scale), lab.T


def layer_components(layer: np.ndarray) -> np.ndarray:
    """The interaction components of a layer's NaN cells as a rows x cols label image (0 outside every component)."""
    return interaction_components(np.isnan(np.asarray(layer, np.float32)).T)[0].T
