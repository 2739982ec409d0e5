"""Runs one of the reference's tutorial scripts, UNMODIFIED, against scanner_b200.

    python tests/helpers/run_reference_tutorial.py <path/to/tutorial.py> <frames>

What is substituted is only what the machine cannot provide: the module name (`scannerpy` resolves
to scanner_b200), the example-video download (`util.download_video`, no network) and -- because this
helper is for machines without a GPU, where H.264 cannot be decoded -- the video file itself, which
becomes a raw-frame stream.  Everything else (ops, graph, run, save_mp4, delete) is the tutorial's
own code.  Run it by hand on a tutorial of a reference checkout (01, 02 and 04 need no GPU op); the
tutorial files cannot be stored in this repository, so no test runs it.  tests/test_tutorials_gpu.py replays the
tutorials' bodies.
"""
import os
import runpy
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import scanner_b200 as sp  # noqa: E402
from oracle import synth  # noqa: E402


def main():
    script, n = sys.argv[1], int(sys.argv[2])
    frames = np.stack([synth.smooth_frame(i % 50, 120, 160) for i in range(n)])
    sys.modules["scannerpy"] = sp
    util = types.ModuleType("util")
    util.download_video = lambda: "/nonexistent/example.mp4"
    sys.modules["util"] = util
    stored = sp.NamedVideoStream

    class RawFrames(stored):
        def __init__(self, sc, name, path=None, **kw):
            if path is not None:
                stored.__init__(self, sc, name, frames=frames)
            else:
                stored.__init__(self, sc, name, **kw)

    sp.NamedVideoStream = RawFrames
    os.chdir(tempfile.mkdtemp())
    runpy.run_path(script, run_name="__main__")
    for f in sorted(os.listdir(".")):
        print("wrote", f, os.path.getsize(f))


if __name__ == "__main__":
    main()
