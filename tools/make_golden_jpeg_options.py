#!/usr/bin/env python
"""Record tests/golden/jpeg_options_cv2.json: SHA-256 of cv2.imencode('.jpg')'s output, with the sampling, luma /
chroma quality and optimize options, for every case of tests/helpers/jpeg_options.sweep() and for a 1080p noise
frame in each sampling mode (and with optimised tables in two).  The hashes keep the options oracle pinned to libjpeg's bytes when cv2 is absent or changes.
Run where cv2 is installed; the output is committed.
"""
import hashlib
import json
import os
import sys

import cv2

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import jpeg_options as O  # noqa: E402
from oracle import jpeg as J  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "jpeg_options_cv2.json")


def cases():
    big = [(f"{m}_noise_1080x1920x3_q95", J.content("noise", 1080, 1920, 3, 1080), 95, {"sampling": m})
           for m in O.SAMPLING]
    big += [(f"{m}_noise_1080x1920x3_q95_opt", J.content("noise", 1080, 1920, 3, 1080), 95,
             {"sampling": m, "optimize": True}) for m in ("444", "420")]
    return O.sweep() + big


def main():
    rec = {"opencv": cv2.__version__, "cases": "helpers.jpeg_options.sweep() + <mode>_noise_1080x1920x3_q95[_opt]",
           "sha256": {}}
    for name, frame, q, opts in cases():
        rec["sha256"][name] = hashlib.sha256(O.cv2_encode(frame, q, **opts)).hexdigest()
    with open(OUT, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT, len(rec["sha256"]), "cases")


if __name__ == "__main__":
    main()
