"""CPU checks of the sampling-distribution restatement (oracle/sample_distribution_oracle.py) against OpenCV, the golden
layers made through cv2, the reference's formulas, and the new C-ABI symbols without a GPU."""
import ctypes
import math
import os

import numpy as np
import pytest

import sample_distribution_cases as sdc
from art_planner_b200 import synth
from oracle import sample_distribution_oracle as sdo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLUR_TOL = 2e-6       # x max(layer): the restated float32 blur against cv2.GaussianBlur


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "sample_distribution.npz"))


@pytest.mark.parametrize("name", sdc.GOLDEN_CASES)
def test_restatement_matches_golden(golden, name):
    import hashlib
    c = sdc.make_case(name)
    h = hashlib.sha256()
    for a in (c.m.elevation, c.thr, c.observed, c.vertices):
        h.update(np.ascontiguousarray(a).tobytes())
    assert str(golden[name + "/sha"]) == h.hexdigest(), "inputs changed: regenerate the golden file"
    filt = sdo.sample_filter(c.thr, c.rp, c.m.res)
    assert np.array_equal(np.packbits((filt > 0.5).ravel(order="F")), golden[name + "/filter"])
    assert set(np.unique(filt)) <= {0.0, 1.0}
    r = sdo.distribution(c.vertices, c.m, c.dp, filt, c.observed)
    g = golden[name + "/n_blur"]
    assert np.abs(r["n_blur"] - g).max() <= BLUR_TOL * g.max()
    gp = golden[name + "/sample_probability"]
    assert np.abs(r["sample_probability"] - gp).max() <= 4 * BLUR_TOL * max(gp.max(), 1e-30)
    assert np.abs(r["cum_prob_rowwise"] - golden[name + "/cum_prob_rowwise"]).max() <= 1e-5


@pytest.mark.parametrize("name", list(sdc.CASES))
def test_restatement_matches_cv2(name):
    cv2 = pytest.importorskip("cv2")
    from oracle import make_golden_basic as mgb
    from oracle import make_golden_sample_distribution as mg
    c = sdc.make_case(name)
    morph = (mgb.cv_morph(cv2.erode), mgb.cv_morph(cv2.dilate))
    assert np.array_equal(sdo.sample_filter(c.thr, c.rp, c.m.res), sdo.sample_filter(c.thr, c.rp, c.m.res, morph=morph))
    n = sdo.vertex_histogram(c.vertices, c.m.rows, c.m.cols, c.m.res, c.m.cx, c.m.cy)
    k, s = sdo.blur_size(c.dp.density_blur_radius, c.m.res)
    a, b = sdo.gaussian_blur(n, k, s), mg.cv_blur(n, k, s)
    assert np.abs(a - b).max() <= BLUR_TOL * b.max()


@pytest.mark.parametrize("ksize,sigma", [(1, 0.2), (3, 0.5), (7, 1.1), (49, 8.0), (61, 10.0), (73, 12.25), (101, 16.6),
                                         (301, 50.0), (1023, 170.5), (9, 40.0)])
def test_gaussian_coefficients_equal_opencv(ksize, sigma):
    cv2 = pytest.importorskip("cv2")
    assert np.array_equal(sdo.gaussian_kernel(ksize, sigma), cv2.getGaussianKernel(ksize, sigma, cv2.CV_32F).ravel())


def test_blur_size_follows_the_reference():
    assert sdo.blur_size(0.49, 0.04) == (73, 12.25)           # int(73.5) = 73, odd
    assert sdo.blur_size(0.4, 0.04)[0] == 61                  # 60 -> 61
    assert sdo.blur_size(0.4, 0.05)[0] == 49                  # 48 -> 49
    assert sdo.blur_size(0.001, 0.04)[0] == 1                 # 0 -> 1


def test_filter_sizes_follow_the_reference():
    # basic.cpp:116-122: sqrt(0.2^2 + 0.2^2) / 0.04 = 7.07 -> 7; min(0.555, 0.225) / 0.04 = 5.6 -> 5
    assert sdo.filter_sizes(synth.PARAMS_YAML, 0.04) == (7, 5)
    assert sdo.filter_sizes(synth.PARAMS_HEADER, 0.04) == (6, 5)


def _ref_index(m, x, y):
    """grid_map getIndex with the map's own resolution: checkIfPositionWithinMap, then getIndexFromPosition
    (index = (int) -((position - length / 2 - map position) / resolution))."""
    lx, ly = m.length
    if not (math.isfinite(x) and math.isfinite(y)):
        return None
    tx, ty = -((x - m.cx) - 0.5 * lx), -((y - m.cy) - 0.5 * ly)
    if not (0 <= tx < lx and 0 <= ty < ly):
        return None
    i, j = int(-(((x - 0.5 * lx) - m.cx) / m.res)), int(-(((y - 0.5 * ly) - m.cy) / m.res))
    return (i, j) if i < m.rows and j < m.cols else None


@pytest.mark.parametrize("name", list(sdc.CASES))
def test_histogram_matches_reference_index(name):
    c = sdc.make_case(name)
    n = sdo.vertex_histogram(c.vertices, c.m.rows, c.m.cols, c.m.res, c.m.cx, c.m.cy)
    ref = np.zeros((c.m.rows, c.m.cols), np.float32)
    for x, y in c.vertices[:, :2]:
        ij = _ref_index(c.m, x, y)
        if ij:
            ref[ij] += 1
    assert np.array_equal(n, ref)
    assert n.sum() < len(c.vertices)                          # NaN and off-map vertices were skipped


def test_histogram_edges_nan_and_off_map():
    m = synth.make_flat_map(10, 8, res=0.125, cx=1.0, cy=-2.0)          # binary fractions: edges exactly representable
    x0, y0 = m.cx + 0.625, m.cy + 0.5
    s = np.zeros((7, 7))
    s[:, 6] = 1
    s[:, :2] = [[x0, y0], [x0 - 0.125, y0 - 0.125], [m.cx - 0.625, m.cy], [m.cx, m.cy - 0.5], [np.nan, 0], [0, np.nan], [50, 50]]
    n = sdo.vertex_histogram(s, m.rows, m.cols, m.res, m.cx, m.cy)
    assert n[0, 0] == 1 and n[1, 1] == 1 and n.sum() == 2    # +x / +y edges inside, -x / -y edges outside
    assert sdo.vertex_histogram(s[4:], m.rows, m.cols, m.res, m.cx, m.cy).sum() == 0


def test_combine_iszero_edge():
    a = np.zeros((4, 5), np.float32, order="F")
    a[1, 2] = np.float32(1e-5)                                # |n| <= 1e-5 everywhere: isZero -> uniform 1
    assert np.array_equal(sdo.combine(a), np.ones_like(a))
    a[1, 2] = np.nextafter(np.float32(1e-5), np.float32(1))
    p = sdo.combine(a)
    assert p[1, 2] == 0 and p[0, 0] == a[1, 2]
    f = np.asfortranarray((np.arange(20).reshape(4, 5) % 2).astype(np.float32))
    assert np.array_equal(sdo.combine(None, f), f)            # no density: 1 x filter
    assert np.array_equal(sdo.combine(np.zeros_like(a), f), f)


def test_zero_vertices_and_all_off_map_give_the_uniform_layer():
    c = sdc.make_case("offorigin_header")
    filt = sdo.sample_filter(c.thr, c.rp, c.m.res)
    for v in (np.zeros((0, 7)), c.vertices[:10] + np.array([1e3, 0, 0, 0, 0, 0, 0])):
        r = sdo.distribution(v, c.m, c.dp, filt, c.observed)
        assert not r["n_blur"].any()
        assert np.array_equal(r["sample_probability"], sdo.apply_cap(filt, c.observed, 0.1))


def test_cap_branches():
    obs = np.asfortranarray(np.array([[1, 0], [1, 0]], np.float32))
    p = np.asfortranarray(np.array([[1, 1], [1, 1]], np.float32))
    km, um, on = sdo.cap_multipliers(*sdo.cap_sums(p, obs), 0.1)           # base 0.5 > 0.1: capped
    assert on and km == np.float32(0.9 / 2) and um == np.float32(0.1 / 2)
    assert np.isclose(sdo.apply_cap(p, obs, 0.1).sum(dtype=np.float64), 1.0)
    assert not sdo.cap_multipliers(*sdo.cap_sums(p, obs), 0.5)[2]          # base 0.5 <= 0.5
    assert not sdo.cap_multipliers(*sdo.cap_sums(p, np.ones_like(obs)), 0.1)[2]    # no unknown cells
    assert not sdo.cap_multipliers(*sdo.cap_sums(p, np.zeros_like(obs)), 0.1)[2]   # no known cells
    assert not sdo.cap_multipliers(0.0, 0.0, 0.1)[2]                                # no mass at all (0 / 0)
    assert np.array_equal(sdo.apply_cap(p, obs, 0.5), p)


@pytest.mark.parametrize("name", list(sdc.CASES))
def test_cap_order_gives_the_reference_multipliers(name):
    """The device's per-row sums against the reference's single row-major running sum."""
    c = sdc.make_case(name)
    filt = sdo.sample_filter(c.thr, c.rp, c.m.res)
    r = sdo.distribution(c.vertices, c.m, sdo.DistributionParams(c.dp.use_inverse_vertex_density, c.dp.density_blur_radius,
                                                                 False, 0.1), filt)
    ours = sdo.cap_multipliers(*sdo.cap_sums(r["sample_probability"], c.observed), 0.1)
    ref = sdo.cap_multipliers(*sdo.cap_sums_reference(r["sample_probability"], c.observed), 0.1)
    assert ours == ref, f"{name}: multipliers {ours} (device order) != {ref} (reference order)"


def test_reflect101_repeats():
    assert list(sdo.reflect101(np.arange(-7, 12), 4)) == [1, 0, 1, 2, 3, 2, 1, 0, 1, 2, 3, 2, 1, 0, 1, 2, 3, 2, 1]
    assert list(sdo.reflect101(np.array([-3, 0, 5]), 1)) == [0, 0, 0]


def test_cdf_restatement_matches_port_oracle(port_lib):
    c = sdc.make_case("fbm_yaml")
    p = sdo.distribution(c.vertices, c.m, c.dp, sdo.sample_filter(c.thr, c.rp, c.m.res), c.observed)
    rc, rr = port_lib.compute_cdf(p["sample_probability"])
    nan = np.isnan(rc)
    assert np.array_equal(np.isnan(p["cum_prob"]), nan)
    assert np.array_equal(p["cum_prob"][~nan].view(np.uint32), rc[~nan].view(np.uint32))
    assert np.array_equal(p["cum_prob_rowwise"].view(np.uint32), rr.view(np.uint32))


# ---- C ABI without a GPU -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import shutil
    from art_planner_b200 import build, capi
    if not os.path.exists(capi.LIB_PATH):
        if shutil.which("nvcc") is None:
            pytest.skip("libartp.so not built and nvcc absent")
        build.build()
    return capi.load()


def test_abi_symbols_and_null_handle(lib):
    from art_planner_b200 import capi
    dp = capi.ArtpSampleDistributionParams(1, 0.49, 1, 0.1)
    assert lib.artp_set_sample_filter(None, None, None, None) == capi.ARTP_E_INVALID
    assert lib.artp_update_sample_distribution(None, ctypes.byref(dp), None, 0, None, None, None) == capi.ARTP_E_INVALID
    assert lib.artp_update_sample_distribution_device(None, ctypes.byref(dp), None, 0, None) == capi.ARTP_E_INVALID
    assert ctypes.sizeof(capi.ArtpSampleDistributionParams) == 32


@pytest.mark.parametrize("ksize,sigma", [(1, 0.2), (7, 1.1), (73, 12.25), (61, 10.000000000000002), (1023, 170.5)])
def test_library_gaussian_coefficients(lib, ksize, sigma):
    out = np.zeros(ksize, np.float32)
    assert lib.artp_debug_gaussian_kernel(ksize, sigma, out.ctypes.data) == ksize
    assert np.array_equal(out, sdo.gaussian_kernel(ksize, sigma))


def test_library_gaussian_kernel_limits(lib):
    from art_planner_b200 import capi
    out = np.zeros(1025, np.float32)
    for k, s in ((1025, 100.0), (72, 12.0), (0, 1.0), (5, 0.0)):
        assert lib.artp_debug_gaussian_kernel(k, s, out.ctypes.data) == capi.ARTP_E_INVALID
