"""CPU: the restatement of the cost server's map preparation (oracle/cost_map_oracle.py) against the golden maps made
through cv2 (tests/golden/cost_map.npz), the mistakes the golden cases catch (rounding instead of truncation, the 254 byte
of the max cell, inpaintMatrix's orientation, the row / column 0 copies), where the masked cells' bytes matter, the refusal
rules against the server's non-finite results, and the ctypes layout of artp_planner_params against include/artp.h."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import cost_map_cases as cc
from oracle import cost_map_oracle as cm
from oracle import inpaint_oracle as io

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "cost_map.npz"))


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def golden(name):
    a, _, want = cc.golden_case(GOLDEN, name)
    return a, want


def outside_diverging(name, a):
    """The cells of the grid_map layer outside the components where cv2 and the restatement differ (none today)."""
    div = GOLDEN[name + "/diverging"]
    if not div.size:
        return np.ones(a.shape, bool)
    labels = io.interaction_components(~np.isfinite(cm.server_image(a)))[0][::-1, ::-1]
    return ~np.isin(labels, div)


def hole_cases():
    return [n for n in cc.CASES if GOLDEN[n + "/filled"].size]


@pytest.mark.parametrize("name", list(cc.CASES) + list(cc.LARGE_CASES))
def test_cases_are_the_golden_inputs(name):
    a, geom = {**cc.CASES, **cc.LARGE_CASES}[name]()
    assert cc.layer_sha256(a) == str(GOLDEN[name + "/in_sha256"])
    assert tuple(geom) == tuple(GOLDEN[name + "/geom"])
    assert GOLDEN[name + "/filled"].size == int(np.isnan(a).sum())


@pytest.mark.parametrize("name", list(cc.CASES))
def test_oracle_equals_golden(name):
    a, want = golden(name)
    got = cm.cost_map_layer(a)
    ok = outside_diverging(name, a)
    assert np.array_equal(bits(got)[ok], bits(want)[ok])
    if name == "hole_free":
        assert np.array_equal(bits(want), bits(a))               # step 2: the layer itself, not quantised


def test_large_case_on_a_sample_of_components():
    """The 1000 x 1000 case: more than 10 000 components; the restated march on 60 seeded components equals cv2's
    bytes."""
    a, _ = cc.large()
    E = cm.server_image(a)
    mn, d = cm.range_of(E)
    u, mask = cm.quantise(E, mn, d)
    want = u.copy()
    want[mask] = GOLDEN["large/filled"]
    labels, n = io.interaction_components(mask)
    assert n > 10000
    rng = np.random.default_rng(7)
    div = set(GOLDEN["large/diverging"].tolist())
    pick = [int(c) for c in rng.choice(np.arange(1, n + 1), 60, replace=False) if int(c) not in div]
    got, _ = io.telea_by_components(u, mask, components=pick, labels=labels)
    sel = mask & np.isin(labels, pick)
    assert np.array_equal(got[sel], want[sel])


def test_truncation_and_the_254_byte():
    """The server truncates: rounding the conversion instead changes the golden result of every case with holes; and the
    max cell of range_254 lands at byte 254, so it comes back one 8-bit step below the max."""
    for name in hole_cases():
        a, want = golden(name)
        E = cm.server_image(a)
        mn, d = cm.range_of(E)
        u, mask = cm.quantise(E, mn, d)
        with np.errstate(invalid="ignore"):
            r = np.rint(((E - mn) * np.float32(255)) / d)
        rounded = u.copy()
        rounded[~mask] = r[~mask].astype(np.uint8)
        wrong = cm.dequantise(io.telea(rounded, mask), mn, d)[::-1, ::-1]
        assert not np.array_equal(bits(wrong), bits(want)), name
    a, want = golden("range_254")
    mx = a[np.isfinite(a)].max()
    E = cm.server_image(a)
    mn, d = cm.range_of(E)
    u, _ = cm.quantise(E, mn, d)
    at_max = cm.server_image(a) == mx
    assert at_max.sum() >= 2 and (u[at_max] == 254).all()
    assert (bits(want[a == mx]) == bits(cm.dequantise(np.array([254], np.uint8), mn, d))).all()
    assert (want[a == mx] < mx).all()


def test_orientation_and_copies_are_caught():
    """Marching in inpaintMatrix's orientation (the cols x rows image of the column-major layer), or adding its row /
    column 0 copies, gives a result that differs from the golden one on at least one case."""
    transposed, copies = [], []
    for name in hole_cases():
        a, want = golden(name)
        E = cm.server_image(a)
        mn, d = cm.range_of(E)
        u, mask = cm.quantise(E, mn, d)
        ul, ml = u[::-1, ::-1], mask[::-1, ::-1]                  # the layer's orientation
        t = cm.dequantise(io.telea(np.ascontiguousarray(ul.T), np.ascontiguousarray(ml.T)).T, mn, d)
        transposed.append(not np.array_equal(bits(t), bits(want)))
        c = want.copy(order="F")
        c[:, 0] = c[:, 1]
        c[0, :] = c[1, :]
        copies.append(not np.array_equal(bits(c), bits(want)))
    assert any(transposed) and any(copies)


@pytest.mark.parametrize("name", ["fbm_blobs", "border_holes", "off_origin", "range_254"])
def test_masked_cells_matter_only_at_the_border(name):
    """Random bytes on the masked cells change the result only in components with a mask cell in the first or last two
    rows or columns, where TELEA's clamped gradient reads reach a masked cell before it is filled (cv2 does the same);
    the golden maps hold the server's 0 there."""
    a, want = golden(name)
    E = cm.server_image(a)
    base = cm.prepare(E)
    assert np.array_equal(bits(base[::-1, ::-1]), bits(want))
    mask = ~np.isfinite(E)
    labels = io.interaction_components(mask)[0]
    edge = np.zeros(E.shape, bool)
    edge[:2] = edge[-2:] = True
    edge[:, :2] = edge[:, -2:] = True
    near = np.isin(labels, np.unique(labels[mask & edge]))
    rng = np.random.default_rng(3)
    for _ in range(3):
        got = cm.prepare(E, masked=rng.integers(0, 256, E.shape).astype(np.uint8))
        assert np.array_equal(bits(got)[~near], bits(base)[~near])


def test_refusals_are_the_servers_non_finite_results():
    """The refused layers are those where the server's chain yields NaN (a +-inf cell, no finite cell) or casts an
    infinite quotient to 8 bits (an overflowing range); the accepted edges give finite results, and mx == mn with holes
    comes back as the constant."""
    for name, (a, why) in cc.refused_layers().items():
        assert cm.refusal(a) == why, name
        if why == "range overflows":
            E = cm.server_image(a)
            mn, d = cm.range_of(E)
            with np.errstate(over="ignore"):
                q = ((E - mn) * np.float32(255)) / d
            assert np.isinf(q[np.isfinite(E)]).any(), name
        else:
            assert np.isnan(cm.server_chain(a)).any(), name
        with pytest.raises(ValueError):
            cm.cost_map_layer(a)
    for name, a in cc.accepted_edges().items():
        assert cm.refusal(a) is None, name
        got = cm.server_chain(a)
        assert np.isfinite(got).all(), name
        assert np.array_equal(bits(cm.cost_map_layer(a)), bits(np.asfortranarray(got[::-1, ::-1]))), name
    a = cc.accepted_edges()["constant_with_hole"]
    assert (bits(cm.cost_map_layer(a)) == bits(np.float32(1.25))).all()
    for name in cc.CASES:
        assert cm.refusal(cc.CASES[name]()[0]) is None


def test_planner_params_layout_matches_header(tmp_path):
    """capi.ArtpPlannerParams has the size and field offsets of artp_planner_params (cost_map_from_raw last)."""
    from art_planner_b200 import capi
    cc_ = shutil.which("cc") or shutil.which("gcc")
    if cc_ is None:
        pytest.skip("no C compiler")
    fields = [n for n, _ in capi.ArtpPlannerParams._fields_]
    assert fields[-1] == "cost_map_from_raw"
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "artp.h"\nint main(void) {\n'
                   '  printf("%zu\\n", sizeof(artp_planner_params));\n' +
                   "".join(f'  printf("%zu\\n", offsetof(artp_planner_params, {n}));\n' for n in fields) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc_, "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got[0] == C.sizeof(capi.ArtpPlannerParams)
    assert got[1:] == [getattr(capi.ArtpPlannerParams, n).offset for n in fields]
