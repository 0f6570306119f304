"""CPU oracle of the cost server's map preparation (TEST INFRASTRUCTURE ONLY): what
art_planner_motion_cost/scripts/cost_query_server.py's _elvMapProcess (:76-119) makes of the raw elevation before
CostPredictor.updateFeatures, restated in numpy float32 (every step one float32 operation, round to nearest):

  1. E = layer[::-1, ::-1], rows x cols: E[r][c] = layer(rows-1-r, cols-1-c) (:74, cnn_oracle.cnn_input_from_layer).
  2. No cell NaN or +-inf: the result is E itself, not quantised.
  3. Otherwise mn / mx = min / max of the finite cells (np.nanmin / nanmax once no cell is +-inf), d = mx - mn,
     q = trunc(((E - mn) * 255) / d) on the finite cells (astype(uint8) truncates; the max cell may land at 254; with
     mx == mn the quotient is 0 / 0 and its byte 0, so the map comes back as mn everywhere), and the mask is
     ~isfinite(E). A masked cell's byte is 0. Both zeros are what numpy's astype(uint8) makes of NaN on x86-64. TELEA
     reads a masked cell's byte before filling it only through its image gradient's clamped reads at the border (a
     known cell in row 0 reads row 1, and so on), so that byte matters only in components with a mask cell in the first
     or last two rows or columns.
  4. cv::inpaint(q, mask, 3, INPAINT_TELEA) in E's orientation (inpaint_oracle.telea, or cv2 itself).
  5. ((float)u * d) / 255 + mn on every cell, known cells too; no row / column 0 copies.

The server's result is NaN for a +-inf cell (the range or the offset is infinite) and for a layer without a finite cell;
for a range whose d * 255 overflows float its 8-bit cast of infinite quotients is undefined in numpy, and the result
holds inf. `refusal` names those inputs, which the C ABI refuses. `server_chain` is the same chain without the
refusals, for showing that its result is finite exactly when an input is not refused.
"""
from __future__ import annotations

import numpy as np

from oracle import inpaint_oracle as io

f32 = np.float32


def server_image(layer: np.ndarray) -> np.ndarray:
    """Step 1: the server's image E of a rows x cols grid_map layer."""
    return np.ascontiguousarray(np.asarray(layer, np.float32)[::-1, ::-1])


def range_of(E: np.ndarray):
    """(mn, d) of the finite cells of E, float32."""
    fin = E[np.isfinite(E)]
    mn, mx = f32(fin.min()), f32(fin.max())
    with np.errstate(over="ignore"):
        return mn, f32(mx - mn)


def refusal(layer: np.ndarray) -> str | None:
    """Why the server's result for this layer is not finite (the C ABI's ARTP_E_INVALID), or None."""
    E = np.asarray(layer, np.float32)
    if np.isinf(E).any():
        return "inf"
    fin = np.isfinite(E)
    if not fin.any():
        return "no finite cell"
    if fin.all():
        return None
    mn, d = range_of(E)
    with np.errstate(over="ignore"):
        if not np.isfinite(d * f32(255)):
            return "range overflows"
    return None


def quantise(E: np.ndarray, mn, d, masked=None):
    """Step 3: (q, mask). masked (optional): bytes for the masked cells instead of the server's 0."""
    mask = ~np.isfinite(E)
    with np.errstate(invalid="ignore"):
        q = (((E - f32(mn)) * f32(255)) / f32(d)).astype(np.float32)
    u = np.zeros(E.shape, np.uint8)
    ok = ~mask & np.isfinite(q)                                   # 0 / 0 when d = 0: byte 0
    u[ok] = np.trunc(q[ok]).astype(np.uint8)
    if masked is not None:
        u[mask] = np.asarray(masked, np.uint8)[mask]
    return u, mask


def dequantise(u: np.ndarray, mn, d) -> np.ndarray:
    """Step 5."""
    return ((u.astype(np.float32) * f32(d)) / f32(255) + f32(mn)).astype(np.float32)


def telea_cv2(u, mask):
    import cv2
    return cv2.inpaint(u, mask.astype(np.uint8), 3, cv2.INPAINT_TELEA)


def prepare(E: np.ndarray, inpaint=io.telea, masked=None) -> np.ndarray:
    """Steps 2-5 on the server's image E (rows x cols, E's orientation). inpaint(u8, mask) -> u8: inpaint_oracle.telea
    (default), telea_cv2, or a per-component march. Raises ValueError for a refused input."""
    E = np.asarray(E, np.float32)
    why = refusal(E)
    if why:
        raise ValueError(why)
    if np.isfinite(E).all():
        return E.copy()
    mn, d = range_of(E)
    u, mask = quantise(E, mn, d, masked)
    return dequantise(inpaint(u, mask), mn, d)


def cost_map_layer(layer: np.ndarray, inpaint=io.telea) -> np.ndarray:
    """artp_cost_map_layer: the prepared map P in grid_map layout (column-major), E'[r][c] = P(rows-1-r, cols-1-c)."""
    return np.asfortranarray(prepare(server_image(layer), inpaint)[::-1, ::-1])


def server_chain(layer: np.ndarray, inpaint=io.telea) -> np.ndarray:
    """The server's chain on the image of `layer` without the refusals (NaN and inf where float32 gives them; the bytes
    of non-finite quotients are 0, where numpy leaves them undefined). Only for small layers."""
    E = server_image(layer)
    if np.isfinite(E).all():
        return E.copy()
    with np.errstate(all="ignore"):
        fin = E[~np.isnan(E)]
        mn = f32(fin.min()) if fin.size else f32(np.nan)
        mx = f32(fin.max()) if fin.size else f32(np.nan)
        d = f32(mx - mn)
        q = ((E - mn) * f32(255)) / d
        mask = ~np.isfinite(E)
        u = np.where(np.isfinite(q) & ~mask, np.trunc(np.where(np.isfinite(q), q, 0)), 0).astype(np.uint8)
        res = inpaint(u, mask) if (~mask).any() else u
        return (res.astype(np.float32) * d) / f32(255) + mn
