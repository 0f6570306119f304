"""Golden layers of inpaintMatrix (art_planner/src/utils.cpp:13-63) through OpenCV itself (cv2, the library the reference
calls): run in the build container (cv2 4.13 present):
    python oracle/make_golden_inpaint.py  -> tests/golden/inpaint.npz
Stores, per case of tests/inpaint_cases.py, the input layer and the inpainted layer."""
import os
import sys

import numpy as np
import cv2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import inpaint_cases  # noqa: E402


def cv_inpaint_matrix(layer):
    """The reference's chain with cv2's own calls. convertTo(CV_8U, a, b) has no Python binding; convertScaleAbs runs the
    same fused multiply-add and rounding and differs only on negative results, which a layer's cells (>= min) do not
    reach beyond rounding to 0; +-inf and NaN convert to 0 in both."""
    mat = np.asfortranarray(np.asarray(layer, np.float32))
    fin = np.isfinite(mat)
    mn = np.float32(mat[fin].min()); mx = np.float32(mat[fin].max())
    img = np.ascontiguousarray(mat.T)
    m1 = img.copy(); m2 = img.copy()
    cv2.patchNaNs(m1, 128); cv2.patchNaNs(m2, 200)
    mask = ((m1 == 128) & (m2 == 200)).astype(np.uint8) * 255
    with np.errstate(all="ignore"):
        alpha = np.float32(np.float32(255) / np.float32(mx - mn))
        beta = np.float32(np.float32(np.float32(-mn) * np.float32(255)) / np.float32(mx - mn))
        u8 = cv2.convertScaleAbs(img, alpha=float(alpha), beta=float(beta))
    res = cv2.inpaint(u8, mask, 3, cv2.INPAINT_TELEA)
    back = res.astype(np.float32) * np.float32(np.float32(mx - mn) / np.float32(255)) + mn
    out = np.asfortranarray(back.T).astype(np.float32)
    out[:, 0] = out[:, 1]
    out[0, :] = out[1, :]
    return out


def main():
    out = {}
    for name, mk in {**inpaint_cases.CASES, **inpaint_cases.LARGE_CASES}.items():
        a = mk()
        out[name + "/in"] = a
        out[name + "/out"] = cv_inpaint_matrix(a)
        print(name, a.shape, int(np.isnan(a).sum()), "holes")
    # the crop where the restatement still differs from cv2 (tests/inpaint_cases.py: DIVERGENCE_CROP)
    from oracle import inpaint_oracle as io
    mat = inpaint_cases.profile_layer(1000, "holes")
    fin = np.isfinite(mat)
    mn, mx = np.float32(mat[fin].min()), np.float32(mat[fin].max())
    img = np.ascontiguousarray(mat.T)
    alpha = np.float32(np.float32(255) / np.float32(mx - mn))
    beta = np.float32(np.float32(np.float32(-mn) * np.float32(255)) / np.float32(mx - mn))
    u8 = cv2.convertScaleAbs(img, alpha=float(alpha), beta=float(beta))
    assert np.array_equal(u8, io.to_u8(img, alpha, beta))
    ys, xs = inpaint_cases.DIVERGENCE_CROP
    sub, mask = np.ascontiguousarray(u8[ys, xs]), np.isnan(img[ys, xs]).astype(np.uint8)
    out["divergence/u8"], out["divergence/mask"] = sub, mask
    out["divergence/cv2"] = cv2.inpaint(sub, mask, 3, cv2.INPAINT_TELEA)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "inpaint.npz"), **out)


if __name__ == "__main__":
    main()
