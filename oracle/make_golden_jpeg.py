#!/usr/bin/env python
"""Record tests/golden/jpeg_cv2.json: SHA-256 of cv2.imencode('.jpg')'s output for every case of
oracle.jpeg.sweep() and for a 1080p noise frame.  The hashes keep the numpy restatement pinned to libjpeg's
bytes when cv2 is absent or changes.  Run where cv2 is installed; the output is committed.
"""
import hashlib
import json
import os
import sys

import cv2

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import jpeg as J  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "jpeg_cv2.json")


def cases():
    return J.sweep() + [("noise_1080x1920x3_q95", J.content("noise", 1080, 1920, 3, 1080), 95)]


def main():
    rec = {"opencv": cv2.__version__, "cases": "oracle.jpeg.sweep() + noise_1080x1920x3_q95", "sha256": {}}
    for name, frame, q in cases():
        rec["sha256"][name] = hashlib.sha256(J.cv2_encode(frame, q)).hexdigest()
    with open(OUT, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT, len(rec["sha256"]), "cases")


if __name__ == "__main__":
    main()
