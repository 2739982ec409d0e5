#!/usr/bin/env python
"""The headline path on an H100: H.264 -> NVDEC -> Histogram + Resize(224) on the GPU -> stored tables.

    python examples/quickstart_gpu.py [video.mp4]

Without an argument a synthetic 1080p clip is written first.  Same calls as the reference's
examples/tutorials/00_basic.py and 07_profiling.py.
"""
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import scanner_b200 as sp  # noqa: E402
from scanner_b200 import engine as E  # noqa: E402


def synthetic_clip(path, frames=120, width=1920, height=1080, gop=30):
    rng = np.random.default_rng(0)
    keys = rng.integers(16, 236, ((frames + gop - 1) // gop, width * height * 3 // 2), dtype=np.uint8)
    with open(path, "wb") as f:
        f.write(E.mp4_mux(E.h264_synth(keys, width, height, gop=gop, non_key="skip", frames=frames), 30, 1))
    return path


def main():
    work = tempfile.mkdtemp()
    video_path = sys.argv[1] if len(sys.argv) > 1 else synthetic_clip(os.path.join(work, "example.mp4"))
    with sp.Client(db_path=os.path.join(work, "db")) as sc:
        video = sp.NamedVideoStream(sc, "example", path=video_path)
        frames = sc.io.Input([video])
        hists = sc.ops.Histogram(frame=frames)
        small = sc.ops.Resize(frame=frames, width=[224], height=[224])
        hist_stream, small_stream = sp.NamedStream(sc, "example_hist"), sp.NamedVideoStream(sc, "example_224")
        job = sc.run([sc.io.Output(hists, [hist_stream]), sc.io.Output(small, [small_stream])],
                     sp.PerfParams.estimate())
        first = next(hist_stream.load())
        print("rows:", hist_stream.len(), "first histogram (R):", first[0].tolist())
        print("resized frame:", next(small_stream.load()).shape)
        sc.get_profile(job).write_trace(os.path.join(work, "quickstart.trace"))
        print(sc.summarize())
    print("database and trace under", work)


if __name__ == "__main__":
    main()
