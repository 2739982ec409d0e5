#!/usr/bin/env python
"""Record tests/golden/resize_interp_cv2.json: SHA-256 of cv2.resize's output with INTER_NEAREST and INTER_AREA on
the seeded frames of oracle.resize_interp.GOLDEN_CASES.  The hashes keep the C restatement (oracle/resize_interp.c)
pinned to OpenCV's arithmetic where cv2 is absent or has changed.  Run where cv2 is installed; the output is
committed.
"""
import hashlib
import json
import os
import sys

import cv2
import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import resize_interp as R  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "resize_interp_cv2.json")


def case_key(mode, sw, sh, dw, dh, kind):
    return f"{mode} {sw}x{sh}->{dw}x{dh} {kind}"


def case_frame(i, sw, sh, dw, dh, kind):
    return R.content(kind, 1000 + i, sh, sw, R.golden_cell(sw, sh, dw, dh))


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.uint8).tobytes()).hexdigest()


def main():
    rec = {"opencv": cv2.__version__, "frames": "oracle.resize_interp.content(kind, 1000 + case index, ...)",
           "sha256": {}}
    for i, (sw, sh, dw, dh, kind) in enumerate(R.GOLDEN_CASES):
        img = case_frame(i, sw, sh, dw, dh, kind)
        for mode in ("INTER_NEAREST", "INTER_AREA"):
            rec["sha256"][case_key(mode, sw, sh, dw, dh, kind)] = digest(
                cv2.resize(img, (dw, dh), interpolation=getattr(cv2, mode)))
    with open(OUT, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
