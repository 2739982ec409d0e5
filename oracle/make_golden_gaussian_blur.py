#!/usr/bin/env python
"""Record tests/golden/gaussian_blur_cv2.json: SHA-256 of cv2.GaussianBlur's output on the seeded frames of
oracle.gaussian_blur.GOLDEN_CASES.  The hashes keep the C restatement (oracle/gaussian_blur.c) pinned to OpenCV's
arithmetic where cv2 is absent or has changed.  Run where cv2 is installed; the output is committed.
"""
import hashlib
import json
import os
import sys

import cv2
import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import gaussian_blur as G  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "gaussian_blur_cv2.json")


def case_key(h, w, c, ksize, sx, sy, border, kind):
    return f"{w}x{h}x{c} k={ksize[0]}x{ksize[1]} sigma={sx!r},{sy!r} {border or 'BORDER_DEFAULT'} {kind}"


def case_frame(i, h, w, c, kind):
    return G.content(kind, 2000 + i, h, w, c)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.uint8).tobytes()).hexdigest()


def cv2_blur(img, ksize, sx, sy, border):
    out = cv2.GaussianBlur(img, tuple(ksize), sx, sigmaY=sy, borderType=G.BORDERS[border])
    return out.reshape(img.shape)


def main():
    rec = {"opencv": cv2.__version__, "frames": "oracle.gaussian_blur.content(kind, 2000 + case index, h, w, c)",
           "sha256": {}}
    for i, (h, w, c, ksize, sx, sy, border, kind) in enumerate(G.GOLDEN_CASES):
        img = case_frame(i, h, w, c, kind)
        rec["sha256"][case_key(h, w, c, ksize, sx, sy, border, kind)] = digest(cv2_blur(img, ksize, sx, sy, border))
    with open(OUT, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
