"""Raw elevation layers for the cost server's map preparation (oracle/cost_map_oracle.py, artp_cost_map_layer): rows x
cols float32 grid_map layers with NaN holes, each with the map geometry (res, cx, cy) its features use. Every case is
deterministic; oracle/make_golden_cost_map.py stores what cv2 decides of each preparation in tests/golden/cost_map.npz,
and golden_case rebuilds the whole prepared map from it."""
import hashlib

import numpy as np

import inpaint_cases as ic
from art_planner_b200 import synth

f32 = np.float32


def _mm(a):
    """Heights on a 1/1024 m grid (NaN kept). The golden file stores a hash of each layer instead of the layer, and the
    grid makes the layers bit-identical on any host: a last-bit difference of a transcendental function in the
    generators would have to land exactly on a grid midpoint to show."""
    return np.asfortranarray((np.rint(np.asarray(a, np.float64) * 1024.0) / 1024.0).astype(np.float32))


def _fbm(rows, cols, seed, amp, res=0.04, cx=0.0, cy=0.0):
    return _mm(synth.make_fbm_map(rows, cols, res, seed=seed, amp=amp, cx=cx, cy=cy).elevation)


def _blobs(a, frac, seed, lo=2, hi=7):
    """Square NaN blobs of lo..hi-1 cells until `frac` of the layer is covered."""
    a = a.copy(order="F")
    rng = np.random.default_rng(seed)
    rows, cols = a.shape
    while np.isnan(a).mean() < frac:
        s = int(rng.integers(lo, hi))
        i, j = int(rng.integers(0, rows - s + 1)), int(rng.integers(0, cols - s + 1))
        a[i:i + s, j:j + s] = np.nan
    return a


def hole_free():
    return _fbm(96, 80, 21, 0.8), (0.04, 0.0, 0.0)


def fbm_blobs():
    return _blobs(_fbm(256, 256, 22, 1.5), 0.02, 22), (0.04, 0.0, 0.0)


def border_holes():
    a = _fbm(120, 90, 23, 0.6)
    a[0, 3:9] = a[-1, 40:44] = a[60:63, 0] = a[10:12, -1] = np.nan
    a[0, 0] = a[-1, -1] = a[0, -1] = a[-1, 0] = np.nan
    a[1, 20] = a[-2, 70] = np.nan
    return _blobs(a, 0.01, 23), (0.04, 0.0, 0.0)


def range_254():
    """Finite cells spread over [mn, mx], both present, for a range whose max cell converts to 254:
    trunc(((mx - mn) * 255) / (mx - mn)) = 254 in float32."""
    rng = np.random.default_rng(24)
    while True:
        mn = f32(rng.uniform(-3, 3))
        mx = f32(mn + f32(rng.uniform(0.5, 10)))
        d = f32(mx - mn)
        if int(f32(f32(d * f32(255)) / d)) == 254:
            break
    a = _fbm(100, 100, 24, 0.7)
    a = ((a - a.min()) / (a.max() - a.min())).astype(np.float32)
    a = _blobs(np.asfortranarray(np.clip(mn + a * d, mn, mx).astype(np.float32)), 0.03, 24)
    a[0, 0], a[-1, -1], a[37, 52] = mn, mx, mx
    return a, (0.04, 0.0, 0.0)


def off_origin():
    a = _blobs(_fbm(97, 143, 25, 1.0, res=0.05, cx=3.7, cy=-12.1), 0.03, 25)
    a[40:52, 60:75] = np.nan                            # one larger unknown patch
    return a, (0.05, 3.7, -12.1)


def large():
    """1000 x 1000 with more than 10 000 interaction components: square holes of 1 to 50 cells a side, and 1- and 2-cell
    holes on a 9-cell lattice."""
    return _mm(ic.size_ladder(1000, 1000, sides=(1, 2, 6, 12, 20, 30, 50), seed=26)), (0.04, 1.5, -0.5)


CASES = {"hole_free": hole_free, "fbm_blobs": fbm_blobs, "border_holes": border_holes, "range_254": range_254,
         "off_origin": off_origin}
LARGE_CASES = {"large": large}   # the CPU tests check a sample of its components against the restatement


def layer_sha256(a) -> str:
    return hashlib.sha256(np.asfortranarray(a, dtype=np.float32).tobytes(order="F")).hexdigest()


def golden_case(golden, name):
    """(layer, geometry, cv2's prepared map in grid_map layout) of a case from the golden file: the layer rebuilt from its
    seed (checked against the stored hash), its known cells' bytes from the float32 conversion and the masked cells'
    bytes from cv2."""
    from oracle import cost_map_oracle as cm
    a, _ = {**CASES, **LARGE_CASES}[name]()
    assert layer_sha256(a) == str(golden[name + "/in_sha256"]), f"{name}: the case generator changed"
    E = cm.server_image(a)
    mask = ~np.isfinite(E)
    if not mask.any():
        return a, tuple(golden[name + "/geom"]), a.copy(order="F")
    mn, d = cm.range_of(E)
    u, _ = cm.quantise(E, mn, d)
    u[mask] = golden[name + "/filled"]
    return a, tuple(golden[name + "/geom"]), np.asfortranarray(cm.dequantise(u, mn, d)[::-1, ::-1])


def refused_layers():
    """Layers whose server result is not finite (cost_map_oracle.refusal), with the reason."""
    a = _fbm(70, 66, 27, 0.5)
    out = {}
    b = a.copy(order="F"); b[3, 4] = np.inf
    out["pos_inf"] = (b, "inf")
    b = a.copy(order="F"); b[50, 60] = -np.inf; b[10, 10] = np.nan
    out["neg_inf_and_hole"] = (b, "inf")
    out["all_nan"] = (np.full((70, 66), np.nan, np.float32, order="F"), "no finite cell")
    b = (a / np.abs(a).max() * f32(3e36)).astype(np.float32, order="F"); b[20, 20] = np.nan
    out["range_overflows"] = (b, "range overflows")
    return out


def accepted_edges():
    """Layers at the edges of the refusal rules that are not refused: constant without holes (the layer itself), constant
    with holes (0 / 0 quotients: the map is the constant everywhere), one finite cell, and a range just below the
    overflow."""
    a = _fbm(70, 66, 28, 0.5)
    out = {"constant_no_hole": np.full((70, 66), f32(1.25), np.float32, order="F")}
    b = np.full((70, 66), f32(1.25), np.float32, order="F"); b[5:9, 7:9] = np.nan; b[0, 30] = np.nan
    out["constant_with_hole"] = b
    b = np.full((70, 66), np.nan, np.float32, order="F"); b[33, 12] = f32(-2.5)
    out["one_finite_cell"] = b
    b = (a / np.abs(a).max() * f32(6e35)).astype(np.float32, order="F"); b[20, 20] = np.nan
    out["range_below_overflow"] = b
    return out
