"""Generate tests/golden/box_verdicts.npz with the reference's own compiled ODE (oracle/_ref/liborc_ref.so): the box
verdicts (artp_box_verdicts) of the cases in tests/box_verdict_cases.py, each box decided by the reference's collider
(oracle/box_verdict_oracle.py over orc_box_collide).

Run where the reference sources are (oracle/Makefile builds the library):  python oracle/make_golden_box_verdicts.py
Inputs are regenerated from seeds; the fixture holds each case's words and a checksum of its map (so generator drift is
detected).
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import box_verdict_cases as bvc  # noqa: E402
import cases  # noqa: E402
from oracle import box_verdict_oracle as bvo  # noqa: E402
from oracle import orc  # noqa: E402
from oracle.make_golden import digest  # noqa: E402


def main() -> None:
    orc.build("ref")
    out = {}
    for mk in sorted(cases.MAPS):
        m = cases.MAPS[mk]()
        states = bvc.samples(m)
        for name, mk2, pk, u in bvc.CASES:
            if mk2 != mk:
                continue
            p = bvc.params(pk, u)
            o = orc.Oracle(p, "reference")
            o.set_map(m)
            why = bvo.box_verdicts(o, p, m, states)
            assert np.array_equal((why & 0x1F) == 0, o.check_poses(states) != 0)
            out[name + "/why"] = why
            out[name + "/sha"] = np.array(digest(m.elevation, m.elevation_masked))
            fails = [(int(((why >> k) & 1).sum())) for k in range(5)]
            print(f"{name}: valid {float(((why & 0x1F) == 0).mean()):.3f} fails per box {fails} "
                  f"outside {int((why >> 8).astype(bool).sum())} multi {int((np.bitwise_count(why & 0x1F) > 1).sum())}")
    path = os.path.join(ROOT, "tests", "golden", "box_verdicts.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
