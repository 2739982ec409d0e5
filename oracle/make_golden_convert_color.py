#!/usr/bin/env python
"""Record tests/golden/convert_color_cv2.json: SHA-256 of cv2.cvtColor's output, for every code ConvertColor
supports, on the image that holds all 2^24 RGB triples (oracle.convert_color.all_triples; the GRAY2* codes take
its first channel).  The hashes keep the numpy restatement pinned to OpenCV's arithmetic when cv2 is absent or
changes.  Run where cv2 is installed; the output is committed.
"""
import hashlib
import json
import os
import sys

import cv2
import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import convert_color as C  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "convert_color_cv2.json")


def source(code):
    img = C.all_triples()
    return img if C.CODES[code][0] == 3 else np.ascontiguousarray(img[..., :1])


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.uint8).tobytes()).hexdigest()


def main():
    rec = {"opencv": cv2.__version__, "image": "oracle.convert_color.all_triples() (4096x4096x3)", "sha256": {}}
    for code in C.CODES:
        rec["sha256"][code] = digest(cv2.cvtColor(source(code), getattr(cv2, code)))
    with open(OUT, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
