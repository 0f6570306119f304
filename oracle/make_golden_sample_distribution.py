"""Golden layers of the sampler's distribution chain through OpenCV itself (cv2, the library the reference calls), the way
Planner::setUpMapProcessors chains it (planner.cpp:39-58): cv2.dilate / cv2.erode with getCircularKernel for the sample
filter (basic.cpp:110-125), cv2.GaussianBlur on the cols x rows image of the column-major layer (utils.cpp:90-110) for
the density, then applyBaseSampleDistribution / applyMaxUnknownProbability (with the reference's row-major running sums)
and the CDF. Run where cv2 is importable:
    python oracle/make_golden_sample_distribution.py  -> tests/golden/sample_distribution.npz"""
import hashlib
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import make_golden_basic as mgb  # noqa: E402
from oracle import sample_distribution_oracle as sdo  # noqa: E402
import sample_distribution_cases as sdc  # noqa: E402


def cv_blur(n_samples, ksize, sigma):
    img = np.ascontiguousarray(np.asarray(n_samples, np.float32).T)
    return np.asfortranarray(cv2.GaussianBlur(img, (ksize, ksize), sigma).T)


def main():
    out = {}
    morph = (mgb.cv_morph(cv2.erode), mgb.cv_morph(cv2.dilate))
    for name in sdc.GOLDEN_CASES:
        c = sdc.make_case(name)
        filt = sdo.sample_filter(c.thr, c.rp, c.m.res, morph=morph)
        r = sdo.distribution(c.vertices, c.m, c.dp, filt, c.observed, blur=cv_blur, sums=sdo.cap_sums_reference)
        out[name + "/filter"] = np.packbits((filt > 0.5).ravel(order="F"))
        out[name + "/n_blur"] = r["n_blur"]
        out[name + "/sample_probability"] = r["sample_probability"]
        out[name + "/cum_prob_rowwise"] = r["cum_prob_rowwise"]
        h = hashlib.sha256()
        for a in (c.m.elevation, c.thr, c.observed, c.vertices):
            h.update(np.ascontiguousarray(a).tobytes())
        out[name + "/sha"] = np.array(h.hexdigest())
        print(name, c.m.rows, "x", c.m.cols, "ksize", sdo.blur_size(c.dp.density_blur_radius, c.m.res)[0],
              "filter fraction", float((filt > 0.5).mean()))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "sample_distribution.npz"), **out)


if __name__ == "__main__":
    main()
