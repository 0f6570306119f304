"""CPU-only: the per-component restatement of inpaintMatrix (oracle/inpaint_oracle.telea_by_components, the oracle
of tests/test_inpaint_scale_gpu.py) against the whole-image restatement and against cv2.inpaint where cv2 is
importable: on every inpaint_cases case, on small versions of the map-scale layers, on hole pairs on both sides of
the interaction reach, and on images 2 or 3 cells thin."""
import numpy as np
import pytest

import inpaint_cases as ic
from oracle import inpaint_oracle as io


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


# Small versions of tests/test_inpaint_scale_gpu.py's layers: the whole-image restatement takes well under a second.
SMALL_LAYERS = {
    "gap_lattice": lambda: ic.gap_lattice(80, 90, tile=18)[0],
    "gap_lattice_border": lambda: ic.gap_lattice(80, 90, tile=18, border=True)[0],
    "size_ladder": lambda: ic.size_ladder(120, 70, sides=(1, 2, 6, 12)),
    "long_thin": lambda: ic.long_thin(90, 80, spiral=15),
    "thin_2xN": lambda: ic.thin_layer(2, 150),
    "thin_Nx3": lambda: ic.thin_layer(140, 3),
    "thin_4xN": lambda: ic.thin_layer(4, 90),
    "thin_Nx5": lambda: ic.thin_layer(90, 5),
    "scattered": lambda: ic.scattered(120, 97, 60),
    "near_constant": lambda: ic.near_constant(50, 40, 33),
}


@pytest.mark.parametrize("margin", [4, 5])
@pytest.mark.parametrize("name", list(ic.CASES) + list(SMALL_LAYERS))
def test_by_components_equals_whole_image(name, margin):
    a = ic.CASES[name]() if name in ic.CASES else SMALL_LAYERS[name]()
    got, labels = io.inpaint_matrix_by_components(a, margin)
    assert labels.shape == a.shape and labels.max() >= 1
    assert np.array_equal(bits(got), bits(io.inpaint_matrix(a)))


def test_by_components_restricted_to_some_components():
    a = ic.scattered(120, 97, 60)
    labels = io.layer_components(a)
    whole = io.inpaint_matrix(a)
    pick = [1, int(labels.max()), int(labels.max()) // 2]
    got, lab = io.inpaint_matrix_by_components(a, components=pick, labels=labels)
    assert np.array_equal(lab, labels)
    ours = np.isin(labels, pick) | ~np.isnan(a)
    ours[:, 0] = ours[:, 1]
    ours[0, :] = ours[1, :]
    assert np.array_equal(bits(got)[ours], bits(whole)[ours])
    assert not np.array_equal(bits(got), bits(whole))   # the other components were left at the NaN byte


def cv2_matrix(cv2, layer):
    """inpaintMatrix with cv2.inpaint in place of the restated march."""
    mask, u8, mn, scale, const = io.to_image(layer)
    return io.from_image(u8 if const else cv2.inpaint(u8, mask.astype(np.uint8), 3, cv2.INPAINT_TELEA), mn, scale)


@pytest.mark.parametrize("gap", [6, 7, 8, 9])
def test_gap_lattice_equals_cv2(gap):
    """Hole pairs in all four directions, in both orders, at gaps on both sides of the 7 / 8 reach, with pairs on all
    four borders: a pair at gap <= 7 is one component, at >= 8 two, and either way the per-component march is cv2's."""
    cv2 = pytest.importorskip("cv2")
    a, pairs = ic.gap_lattice(5 * (gap + 10), 5 * (gap + 10), gaps=(gap,), tile=gap + 10, seed=gap, border=True)
    labels = io.layer_components(a)
    holes = np.isnan(a)
    assert holes[0].any() and holes[-1].any() and holes[:, 0].any() and holes[:, -1].any()
    for p, q, g in pairs:
        la, lb = labels[p[0][0], p[0][1]], labels[q[0][0], q[0][1]]
        assert (la == lb) == (g <= 7), (p, q, g)
    assert len({(tuple(np.sign(q[0] - p[0]))) for p, q, _ in pairs}) >= 4
    got, _ = io.inpaint_matrix_by_components(a, labels=labels)
    assert np.array_equal(bits(got), bits(cv2_matrix(cv2, a)))


def test_telea_equals_cv2_on_images_two_or_three_cells_thin():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(23)
    for trial in range(80):
        thin, long_ = int(rng.integers(2, 4)), int(rng.integers(2, 60))
        H, W = (thin, long_) if trial % 2 else (long_, thin)
        img = (rng.random((H, W)) * 255).astype(np.uint8)
        m = (rng.random((H, W)) < rng.random() * 0.5).astype(np.uint8)
        if trial % 4 == 0:
            m[0, 0] = m[-1, -1] = 1
        elif trial % 4 == 1:
            m[0, -1] = m[-1, 0] = 1
        want = cv2.inpaint(img, m, 3, cv2.INPAINT_TELEA)
        assert np.array_equal(io.telea(img, m), want), (trial, H, W)
        assert np.array_equal(io.telea_by_components(img, m)[0], want), (trial, H, W)


@pytest.mark.parametrize("shape", [(2, 37), (37, 2), (2, 5), (3, 64), (64, 3)])
def test_inpaint_matrix_on_two_and_three_cell_layers(shape):
    """Holes in all four corners and one across the whole width in the middle."""
    a = ic._field(*shape, seed=sum(shape), noise=0.3)
    a[0, 0] = a[-1, -1] = a[0, -1] = a[-1, 0] = np.nan
    t = a if shape[0] <= shape[1] else a.T
    t[:, t.shape[1] // 2] = np.nan
    assert np.isfinite(a).sum() >= 2
    want = io.inpaint_matrix(a)
    assert np.array_equal(bits(io.inpaint_matrix_by_components(a)[0]), bits(want))
    cv2 = pytest.importorskip("cv2")
    assert np.array_equal(bits(cv2_matrix(cv2, a)), bits(want))


@pytest.mark.parametrize("ulps", [3, 50, 1000])
def test_near_constant_layers_separate_a_fused_from_an_unfused_conversion(ulps):
    """The near-constant layers tests/test_inpaint_scale_gpu.py uses: an unfused multiply and add would give other
    bytes on a good share of their cells, so the device's fused conversion is what those cases pin."""
    a = ic.near_constant(ulps, 300, 257, seed=ulps)
    x = a[np.isfinite(a)]
    mn, mx = np.float32(x.min()), np.float32(x.max())
    rg = np.float32(mx - mn)
    alpha = np.float32(np.float32(255) / rg)
    beta = np.float32(np.float32(np.float32(-mn) * np.float32(255)) / rg)
    unfused = np.clip(np.rint(np.float32(x * alpha) + beta), 0, 255).astype(np.uint8)
    assert (unfused != io.to_u8(x, alpha, beta)).mean() > 0.05
