"""GPU (-m gpu): artp_inpaint_layer[_device] at map scale against the per-component restatement
(oracle/inpaint_oracle.inpaint_matrix_by_components) bit for bit, NaN compared as positions: thousands of interaction
components marched at once with hole pairs on both sides of the 7 / 8-cell reach, one component in every size class
the march hands out, more components than the launch has warps, long thin components, layers 2-5 cells thin, 4000^2
layers checked on a seeded sample of components, the layer of the known divergence from cv2, the 8-bit conversion's
edges, and the same bits on repeated calls.

Components are independent marches, so a sample of them is a sound check at any map size: every cell of a sampled
component, and every cell outside all components' holes (the 8-bit round trip), is compared; so are the column / row 0
copies of those cells. Every layer goes through both the host call and the device call on a non-default stream."""
import numpy as np
import pytest

import inpaint_cases as ic
import roadmap_cases as rc
from oracle import inpaint_oracle as io

pytestmark = pytest.mark.gpu


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def chk():
    import art_planner_b200 as ap
    return ap.StateValidityChecker(rc.make_case("gentle_inf").rp)


def on_device(chk, layer):
    """artp_inpaint_layer_device on a side stream: upload, inpaint and read back all ordered on that stream."""
    import torch
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d = torch.from_numpy(np.ascontiguousarray(np.asarray(layer, np.float32).T)).cuda().t()
        out = chk.inpaint(d).cpu().numpy()
    return out


def assert_same(got, want, where, what):
    g, w = got[where], want[where]
    gn, wn = np.isnan(g), np.isnan(w)
    assert np.array_equal(gn, wn), f"{what}: NaN at {int((gn != wn).sum())} cells the restatement does not have"
    bad = bits(g[~gn]) != bits(w[~wn])
    if bad.any():
        rows, cols = np.nonzero(where)
        k = np.flatnonzero(~gn)[np.argmax(bad)]
        raise AssertionError(f"{what}: {int(bad.sum())} of {int(where.sum())} checked cells differ, first at "
                             f"({rows[k]}, {cols[k]}): {g[k]!r} != {w[k]!r}")


def check(chk, layer, components=None, labels=None):
    """Both calls against the restatement on `components` (all when None) and on every cell outside the other
    components' holes. Returns the label image (rows x cols) and the host call's result."""
    want, labels = io.inpaint_matrix_by_components(layer, components=components, labels=labels)
    checked = np.ones(layer.shape, bool)
    if components is not None:
        checked = ~np.isnan(layer) | np.isin(labels, list(components))
    checked[:, 0] = checked[:, 1]                          # the copies read column / row 1
    checked[0, :] = checked[1, :]
    host = chk.inpaint(layer)
    assert_same(host, want, checked, "artp_inpaint_layer")
    assert_same(on_device(chk, layer), want, checked, "artp_inpaint_layer_device")
    return labels, host


def sample(labels, k, seed):
    """k seeded components plus, always: up to 8 on each border, the ones in the four corners, the largest and the
    one with the highest root (the march's root is the component's smallest column-major cell index)."""
    from scipy import ndimage
    n = int(labels.max())
    rng = np.random.default_rng(seed)
    must = set()
    for edge in (labels[0], labels[-1], labels[:, 0], labels[:, -1]):
        ids = np.unique(edge[edge > 0])
        must.update(int(c) for c in rng.choice(ids, min(8, len(ids)), replace=False))
    must.update(int(c) for c in (labels[0, 0], labels[0, -1], labels[-1, 0], labels[-1, -1]) if c)
    sizes = np.bincount(labels.ravel())
    sizes[0] = 0
    must.add(int(np.argmax(sizes)))
    idx = np.arange(labels.size, dtype=np.int64).reshape(labels.shape, order="F")
    roots = ndimage.minimum(idx, labels, np.arange(1, n + 1))
    must.add(int(np.argmax(roots)) + 1)
    return sorted(must | {int(c) + 1 for c in rng.choice(n, min(k, n), replace=False)})


def test_gap_lattice(chk):
    """About 5 k components: hole pairs at gaps 7 (one component) and 8 (two, marched side by side) in all four
    directions and both orders, with pairs touching all four borders; every component checked."""
    a, pairs = ic.gap_lattice(1000, 1000, gaps=(7, 8), tile=18)
    labels, _ = check(chk, a)
    assert labels.max() > 4000
    holes = np.isnan(a)
    assert holes[0].any() and holes[-1].any() and holes[:, 0].any() and holes[:, -1].any()
    for p, q, g in pairs:
        assert (labels[p[0][0], p[0][1]] == labels[q[0][0], q[0][1]]) == (g == 7), (p, q, g)


def test_size_class_ladder(chk):
    """One component in every power-of-two size class from 2^4 to 2^14 on a 997 x 613 layer, thousands in class
    2^5, and more components than the march launches warps (sm_count * 8 CTAs of 4), so warps take several."""
    import torch
    a = ic.size_ladder(997, 613)
    labels = io.layer_components(a)
    sizes = np.bincount(labels.ravel())[1:]
    classes = np.floor(np.log2(sizes)).astype(int)
    assert set(range(4, 15)) <= set(classes.tolist())
    assert np.bincount(classes)[4] >= 10 and np.bincount(classes)[5] > 1000
    assert len(sizes) > torch.cuda.get_device_properties(0).multi_processor_count * 8 * 4
    ladder = {int(c) + 1 for c in np.flatnonzero(sizes >= 64 * 64)}            # the large squares
    ladder |= {int(labels[0, 0]), int(labels[997 // 2, 612]), int(labels[996, 5]), int(labels[10, 10])}
    for c in range(4, 15):                                                     # one of every class
        ladder.add(int(np.flatnonzero(classes == c)[0]) + 1)
    check(chk, a, sample(labels, 300, seed=1) + sorted(ladder), labels)


def test_long_thin_components(chk):
    """A diagonal and a zig-zag 1-cell line whose bounding boxes are far larger than their cell counts, and a
    spiral hole: a long march through many equal T values; every component checked."""
    a = ic.long_thin(800, 700)
    labels, _ = check(chk, a)
    from scipy import ndimage
    boxes = ndimage.find_objects(labels)
    cells = np.bincount(labels.ravel())[1:]
    area = np.array([(b[0].stop - b[0].start) * (b[1].stop - b[1].start) for b in boxes])
    assert (area > 10 * cells).sum() >= 2                    # the two lines


@pytest.mark.parametrize("shape", [(2, 2000), (3, 1999), (4, 2000), (5, 1997),
                                   (2000, 2), (1999, 3), (2000, 4), (1997, 5)])
def test_thin_layers(chk, shape):
    """Layers 2-5 cells thin: holes in the corners, across the width near both ends, and a component every 8 cells
    along the length (the most the width allows); every component checked."""
    a = ic.thin_layer(*shape)
    labels, _ = check(chk, a)
    assert labels.max() > 200


@pytest.mark.parametrize("shape, n_holes", [((4000, 4000), 40000), ((4093, 3001), 30000)])
def test_map_scale_layers(chk, shape, n_holes):
    """Scattered 1-20-cell holes on 4000^2 and 4093 x 3001 layers: a seeded sample of components plus the ones on
    the borders and corners, the largest and the one with the highest root."""
    a = ic.scattered(*shape, n_holes)
    labels = io.layer_components(a)
    assert labels.max() > 10000
    assert labels[0, 0] and labels[0, -1] and labels[-1, 0] and labels[-1, -1]
    check(chk, a, sample(labels, 300, seed=shape[1]), labels)


def divergence_components(labels):
    """The components whose bounding box meets DIVERGENCE_CROP's window of the cols x rows image."""
    from scipy import ndimage
    (y, x) = ic.DIVERGENCE_CROP
    hit = []
    for c, (sy, sx) in enumerate(ndimage.find_objects(np.ascontiguousarray(labels.T)), 1):
        if sy.start < y.stop and sy.stop > y.start and sx.start < x.stop and sx.stop > x.start:
            hit.append(c)
    return hit


def test_known_divergence_layer(chk):
    """profile_layer(1000, "holes"), where the restatement and cv2 differ on a few cells: the device equals the
    restatement on every component near the divergence and on a sample of the others; where cv2 is importable, the
    device differs from cv2 only inside those components."""
    a = ic.profile_layer(1000, "holes")
    labels = io.layer_components(a)
    near = divergence_components(labels)
    assert near
    _, host = check(chk, a, sorted(set(near) | set(sample(labels, 20, seed=3))), labels)
    try:
        import cv2
    except ImportError:
        return
    mask, u8, mn, scale, _ = io.to_image(a)
    want = io.from_image(cv2.inpaint(u8, mask.astype(np.uint8), 3, cv2.INPAINT_TELEA), mn, scale)
    i, j = np.nonzero(bits(host) != bits(want))
    src = labels[np.maximum(i, 1), np.maximum(j, 1)]
    assert np.isin(src, near).all(), f"{int((~np.isin(src, near)).sum())} cells differ from cv2 outside them"


def conversion_layers():
    rng = np.random.default_rng(31)
    f = ic._field(300, 257, 31, noise=0.2)
    holes = rng.random(f.shape) < 0.04
    out = {}
    for u in (3, 50, 1000):                                      # fused and unfused multiply-add round apart here
        out[f"near_constant_{u}ulp"] = ic.near_constant(u, 300, 257, seed=u)
    a = f * np.float32(1e-3)
    a[a <= a.min() + np.float32(1e-4)] = np.uint32(1).view(np.float32)   # the minimum is the smallest denormal
    a[holes] = np.nan
    out["denormal_min"] = a
    a = (np.abs(f) * np.float32(1e-39)).astype(np.float32)      # a denormal range: 255 / range overflows
    a[holes] = np.nan
    out["denormal_range"] = a
    for name, z in (("neg_zero_min", -0.0), ("pos_zero_min", 0.0)):
        a = np.abs(f)
        a[a < np.float32(0.3)] = np.float32(z)
        a[holes] = np.nan
        out[name] = a
    a = np.full((300, 200), np.nan, np.float32, order="F")     # one finite cell: one component over the whole map
    a[123, 77] = np.float32(4.5)
    out["single_finite_cell"] = a
    a = np.full((61, 47), np.nan, np.float32, order="F")       # two: a real march over the whole map
    a[20, 9], a[44, 40] = np.float32(-1.25), np.float32(3.0)
    out["two_finite_cells"] = a
    a = f.copy(order="F")
    a[holes] = np.nan
    inf = np.roll(holes, 1, 0) & ~holes
    a[inf] = np.where(rng.random(int(inf.sum())) < 0.5, np.inf, -np.inf).astype(np.float32)
    out["infs_beside_holes"] = a
    a = (f / np.abs(f).max() * np.float32(3.3e38)).astype(np.float32)   # max - min overflows to inf
    a[holes] = np.nan
    out["range_overflows"] = a
    return out


CONVERSION = conversion_layers()


@pytest.mark.parametrize("name", list(CONVERSION))
def test_conversion_edges(chk, name):
    a = np.asfortranarray(CONVERSION[name])
    fin = a[np.isfinite(a)]
    if name.startswith("near_constant"):
        assert int(bits(fin.max())) - int(bits(fin.min())) == int(name.split("_")[2][:-3])
    if name == "range_overflows":
        with np.errstate(over="ignore"):
            assert np.isinf(np.float32(fin.max()) - np.float32(fin.min()))
    check(chk, a)


def test_repeated_calls_give_the_same_bits(chk):
    """More than 10 k components, whose slots and order come from atomics: three host calls and three device calls
    give identical bits."""
    a = ic.size_ladder(1000, 1000, sides=(1, 2, 6, 12, 20, 30, 50))
    assert io.layer_components(a).max() > 10000
    runs = [bits(chk.inpaint(a)) for _ in range(3)] + [bits(on_device(chk, a)) for _ in range(3)]
    assert not np.isnan(runs[0].view(np.float32)).any()
    for r in runs[1:]:
        assert np.array_equal(r, runs[0])
