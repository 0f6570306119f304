"""Golden maps of the cost server's preparation (cost_query_server.py _elvMapProcess) through OpenCV itself (cv2, the
library the server calls): run where cv2 is importable (4.13 here):
    python oracle/make_golden_cost_map.py  -> tests/golden/cost_map.npz
The layers are rebuilt from tests/cost_map_cases.py's seeds, so per case the file stores only what cv2 decides:
  <case>/in_sha256   the SHA-256 of the layer's float32 bytes (column-major), which pins the case generator;
  <case>/geom        its geometry (res, cx, cy);
  <case>/filled      cv2.inpaint's bytes of the masked cells, in E's orientation and raster order (empty without holes).
Everything else of the prepared map follows from the layer by cost_map_oracle's float32 steps: the known cells' bytes
(quantise), and the way back (dequantise); cost_map_cases.golden_case rebuilds it. Where the restated TELEA differs from
cv2 (the divergence DESIGN.md section 4.6 lists), the interaction components that hold the differing cells are stored as
<case>/diverging (labels of inpaint_oracle.interaction_components on the server's mask); the tests then hold the
library to the restatement everywhere and to cv2 outside those components."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import cost_map_cases as cc  # noqa: E402
from oracle import cost_map_oracle as cm  # noqa: E402
from oracle import inpaint_oracle as io  # noqa: E402


def main():
    out = {}
    for name, mk in {**cc.CASES, **cc.LARGE_CASES}.items():
        a, geom = mk()
        want = cm.cost_map_layer(a, cm.telea_cv2)
        E = cm.server_image(a)
        mask = ~np.isfinite(E)
        labels = io.interaction_components(mask)[0]
        restated = cm.cost_map_layer(a, lambda u, m: io.telea_by_components(u, m, labels=labels)[0])
        diff = (want.view(np.uint32) != restated.view(np.uint32))[::-1, ::-1]   # in E's orientation
        diverging = np.unique(labels[diff])
        out[name + "/in_sha256"] = np.array(cc.layer_sha256(a))
        out[name + "/geom"] = np.array(geom, np.float64)
        filled = np.zeros(0, np.uint8)
        if mask.any():
            mn, d = cm.range_of(E)
            u8 = cm.telea_cv2(*cm.quantise(E, mn, d))
            assert np.array_equal(cm.dequantise(u8, mn, d)[::-1, ::-1], want)
            filled = u8[mask]
        out[name + "/filled"] = filled
        out[name + "/diverging"] = diverging.astype(np.int32)
        print(name, a.shape, int(mask.sum()), "holes,", int(labels.max()), "components,",
              int(diff.sum()), "cells differ from the restatement in components", diverging.tolist())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "cost_map.npz"), **out)


if __name__ == "__main__":
    main()
