#!/usr/bin/env python
"""Throughput of the JPEG encoder (scn_jpeg_encode_u8): 64 x 1080p RGB frames per call at quality 95, on smooth
synthetic frames and on noise.  CUDA events around `--iters` calls after `--warmup` calls (each call includes its
two read-backs of per-frame counts); the time of each stage from scn_prof over the same number of calls; output
bytes per frame; which stage bounds the encoder, with the algorithmic bytes (3 W H read + the files written) over
the call's time; cv2.imencode on every host core for the same frames; the card's name, power limit and maximum SM
clock read in the same run.  The files are checked against cv2.imencode once per content.  --sampling runs
scn_jpeg_encode_u8_opts instead, once per listed mode (cv2's IMWRITE_JPEG_SAMPLING_FACTOR, cv2 given the same);
--optimize adds optimised Huffman tables (IMWRITE_JPEG_OPTIMIZE) to every mode.

    python tools/bench_jpeg.py [--iters 50] [--warmup 10] [--sampling 444,422,420,440,411] [--optimize] [--json OUT]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import synth  # noqa: E402
from scanner_b200 import cabi, kernels  # noqa: E402

N, W, H, Q = 64, 1920, 1080, 95


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                       "-i", str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


class Encoder:
    """scn_jpeg_encode_u8 into a device buffer that is kept and grown, so calls time the encoder alone."""

    def __init__(self, frames, sampling=None, optimize=False):
        self.L = cabi.lib()
        self.opts = None if sampling is None and not optimize else kernels._jpeg_options(sampling, 0, 0, optimize)
        self.buf = torch.empty(1, dtype=torch.uint8, device="cuda")
        self.sizes = (ctypes.c_size_t * N)()
        self.src, self.keep = cabi.ptr_array([frames.data_ptr() + i * H * W * 3 for i in range(N)])
        self.cb = cabi.ALLOC_FN(self._alloc)
        self.stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def _alloc(self, _ctx, nbytes):
        if self.buf.numel() < nbytes:
            self.buf = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        return self.buf.data_ptr()

    def __call__(self):
        if self.opts is None:
            cabi.check(self.L.scn_jpeg_encode_u8(self.src, N, W, H, 3, Q, self.cb, None, self.sizes, self.stream),
                       "scn_jpeg_encode_u8")
        else:
            cabi.check(self.L.scn_jpeg_encode_u8_opts(self.src, N, W, H, 3, Q, ctypes.byref(self.opts), self.cb, None,
                                                      self.sizes, self.stream), "scn_jpeg_encode_u8_opts")

    def files(self):
        data, out, at = self.buf.cpu().numpy().tobytes(), [], 0
        for s in self.sizes:
            out.append(data[at:at + s])
            at += s
        return out


def time_calls(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def cv2_params(sampling, optimize=False):
    import cv2
    params = [cv2.IMWRITE_JPEG_QUALITY, Q] + ([cv2.IMWRITE_JPEG_OPTIMIZE, 1] if optimize else [])
    if sampling is not None:
        s = kernels.JPEG_SAMPLING[sampling]
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, (s << 16) | 0x1111]
    return params


def cv2_all_cores(frames_np, sampling=None, optimize=False, rounds=2):
    import cv2
    bgr = [np.ascontiguousarray(f[..., ::-1]) for f in frames_np]
    cores = os.cpu_count() or 1
    params = cv2_params(sampling, optimize)
    enc = lambda f: cv2.imencode(".jpg", f, params)  # noqa: E731
    with ThreadPoolExecutor(cores) as ex:  # cv2 releases the GIL inside imencode
        list(ex.map(enc, bgr))
        t = time.perf_counter()
        for _ in range(rounds):
            list(ex.map(enc, bgr))
        dt = time.perf_counter() - t
    return cores, rounds * len(bgr) / dt


def measure(args, kind, mode, host, frames):
    """one row: the encoder on `frames` (host copy `host`) with sampling `mode` (None: scn_jpeg_encode_u8)"""
    import cv2
    enc = Encoder(frames, mode, args.optimize)
    ms = time_calls(enc, args.iters, args.warmup)
    files = enc.files()
    for i in (0, N - 1):
        ok, want = cv2.imencode(".jpg", np.ascontiguousarray(host[i][..., ::-1]), cv2_params(mode, args.optimize))
        assert files[i] == want.tobytes(), f"{kind} {mode} frame {i} differs from cv2.imencode"
    L = cabi.lib()
    L.scn_prof_enable(1)
    for _ in range(args.iters):
        enc()
    stages = {k: v["ms"] / args.iters for k, v in cabi.prof_report().items()}
    L.scn_prof_enable(0)
    out_bytes = sum(len(f) for f in files)
    algo = N * 3 * W * H + out_bytes
    bound = max(stages, key=stages.get)
    cores, cv2_fps = cv2_all_cores(host, mode, args.optimize)
    row = {"content": kind, "sampling": mode or "420", "optimize": args.optimize, "ms_per_call": round(ms, 3),
           "frames_per_s": round(N / (ms * 1e-3), 1),
           "bytes_per_frame": out_bytes // N, "stages_ms": {k: round(v, 3) for k, v in stages.items()},
           "kernels_ms": round(sum(stages.values()), 3), "bound_by": bound,
           "algorithmic_GB_per_s": round(algo / (ms * 1e-3) / 1e9, 1),
           "cv2_cores": cores, "cv2_frames_per_s": round(cv2_fps, 1)}
    print(f"{kind:6s} {mode or 'default':7s} {ms:7.3f} ms/call  {row['frames_per_s']:9.1f} frames/s  "
          f"{row['bytes_per_frame']:8d} B/frame  "
          f"algorithmic {row['algorithmic_GB_per_s']:6.1f} GB/s  cv2 on {cores} cores {cv2_fps:7.1f} frames/s")
    for k, v in sorted(stages.items(), key=lambda kv: -kv[1]):
        print(f"    {k:28s} {v:7.3f} ms  {100 * v / ms:5.1f} % of the call")
    print(f"    kernels {row['kernels_ms']:.3f} ms of {ms:.3f} ms per call; bound by {bound}")
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    ap.add_argument("--sampling", default=None, help="comma-separated modes: 444, 422, 420, 440, 411")
    ap.add_argument("--optimize", action="store_true", help="optimised Huffman tables (IMWRITE_JPEG_OPTIMIZE)")
    args = ap.parse_args()
    modes = [None] if args.sampling is None else args.sampling.split(",")
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg needs a CUDA device")
    info = card()
    print(f"# {info}; {N} x {W}x{H} RGB per call, quality {Q}")
    rows = []
    for kind in ("smooth", "noise"):
        if kind == "smooth":
            host = np.stack([synth.smooth_frame(100 + i, H, W) for i in range(N)])
        else:
            host = np.random.default_rng(0).integers(0, 256, (N, H, W, 3), dtype=np.uint8)
        frames = torch.from_numpy(host).cuda()
        for mode in modes:
            rows.append(measure(args, kind, mode, host, frames))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": info, "frames_per_call": N, "width": W, "height": H, "quality": Q, "rows": rows},
                      f, indent=1)


if __name__ == "__main__":
    main()
