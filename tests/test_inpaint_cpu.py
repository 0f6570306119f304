"""CPU-only: the restatement of inpaintMatrix (oracle/inpaint_oracle.py) against OpenCV itself where cv2 is importable,
against the golden layers made through cv2 (tests/golden/inpaint.npz), and the new entry points' argument checks."""
import ctypes as C
import os

import numpy as np
import pytest

import inpaint_cases as ic
from oracle import inpaint_oracle as io

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "inpaint.npz"))


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", list(ic.CASES))
def test_oracle_equals_golden(name, gold):
    a = ic.CASES[name]()
    assert np.array_equal(bits(gold[name + "/in"]), bits(a)), "generator drift"
    assert np.array_equal(bits(io.inpaint_matrix(a)), bits(gold[name + "/out"]))


def test_oracle_equals_golden_giant(gold):
    a = ic.LARGE_CASES["giant"]()
    assert np.array_equal(bits(gold["giant/in"]), bits(a))
    assert np.array_equal(bits(io.inpaint_matrix(a)), bits(gold["giant/out"]))


def test_telea_equals_cv2_inpaint():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    for trial in range(40):
        H, W = (int(v) for v in rng.integers(4, 28, 2))
        img = (rng.random((H, W)) * 255).astype(np.uint8)
        if trial % 2:
            img = cv2.GaussianBlur(img, (7, 7), 2)
        m = (rng.random((H, W)) < rng.random() * 0.4).astype(np.uint8)
        if trial % 3 == 0:
            a, b = rng.integers(0, H), rng.integers(0, W)
            m[a:a + rng.integers(1, 10), b:b + rng.integers(1, 10)] = 1
        assert np.array_equal(io.telea(img, m), cv2.inpaint(img, m, 3, cv2.INPAINT_TELEA)), trial


def test_telea_one_and_two_cell_holes_equal_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    img = (rng.random((12, 13)) * 255).astype(np.uint8)
    for y in range(12):                       # one hole everywhere, borders and corners included
        for x in range(13):
            m = np.zeros((12, 13), np.uint8)
            m[y, x] = 1
            assert np.array_equal(io.telea(img, m), cv2.inpaint(img, m, 3, cv2.INPAINT_TELEA)), (y, x)
    for gap in range(1, 11):                  # two holes on either side of the interaction reach
        m = np.zeros((12, 13), np.uint8)
        m[5, 1] = m[6, 1 + gap] = 1
        assert np.array_equal(io.telea(img, m), cv2.inpaint(img, m, 3, cv2.INPAINT_TELEA)), gap


def test_to_u8_equals_cv2_on_every_value_class():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    for scale in (1e-3, 1.0, 50.0, 1e4, 1e30):
        x = (rng.standard_normal(5000) * scale).astype(np.float32) + np.float32(rng.standard_normal() * 10)
        x[::37] = np.inf
        x[::41] = np.nan
        fin = x[np.isfinite(x)]
        mn, mx = np.float32(fin.min()), np.float32(fin.max())
        a = np.float32(np.float32(255) / np.float32(mx - mn))
        b = np.float32(np.float32(np.float32(-mn) * np.float32(255)) / np.float32(mx - mn))
        # convertScaleAbs shares convertTo's multiply-add and rounding; cells >= min never go negative beyond rounding
        ref = cv2.convertScaleAbs(x.reshape(1, -1), alpha=float(a), beta=float(b)).ravel()
        assert np.array_equal(io.to_u8(x, a, b), ref), scale


def test_degenerate_layers():
    a = np.full((5, 6), 1.5, np.float32, order="F")
    a[2, 3] = np.nan
    assert np.array_equal(io.inpaint_matrix(a), np.full((5, 6), 1.5, np.float32))
    with pytest.raises(ValueError):
        io.inpaint_matrix(np.full((4, 4), np.nan, np.float32))
    with pytest.raises(ValueError):
        io.inpaint_matrix(np.array([[np.inf, -np.inf], [np.nan, np.inf]], np.float32))


def test_new_symbols_and_argument_checks():
    from art_planner_b200 import capi
    lib = capi.load()
    for sym in ("artp_inpaint_layer", "artp_inpaint_layer_device", "artp_planner_set_map_raw"):
        assert hasattr(lib, sym), sym
    buf = np.zeros(16, np.float32)
    # a null handle is refused before any device work
    assert lib.artp_inpaint_layer(None, buf.ctypes.data, 4, 4, buf.ctypes.data) == capi.ARTP_E_INVALID
    assert lib.artp_inpaint_layer_device(None, buf.ctypes.data, 4, 4, buf.ctypes.data, None) == capi.ARTP_E_INVALID
    assert lib.artp_planner_set_map_raw(None, None, buf.ctypes.data, None, 4, 4, 0.1, 0.0, 0.0, None) == capi.ARTP_E_INVALID


def test_divergence_crop_golden_is_cv2():
    cv2 = pytest.importorskip("cv2")
    g = np.load(os.path.join(ROOT, "tests", "golden", "inpaint.npz"))
    assert np.array_equal(cv2.inpaint(g["divergence/u8"], g["divergence/mask"], 3, cv2.INPAINT_TELEA), g["divergence/cv2"])


@pytest.mark.xfail(strict=True, reason="known divergence from cv2 on 6 cells of this crop (DESIGN.md section 4.6)")
def test_restatement_equals_cv2_on_divergence_crop(gold):
    assert np.array_equal(io.telea(gold["divergence/u8"], gold["divergence/mask"]), gold["divergence/cv2"])
