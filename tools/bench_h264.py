#!/usr/bin/env python
"""Throughput of the H.264 encoder (scn_h264_encode_u8): 64 x 1080p RGB frames per call at QP 23 and 35, on
smooth synthetic frames and on noise.  CUDA events around `--iters` calls after `--warmup` calls (each call includes
its two read-backs of per-frame counts); the time of each stage from scn_prof over the same number of calls; bytes
per access unit; the luma PSNR of the first frame's reconstruction against its source (the oracle's
reconstruction, which the kernel's bytes are checked to encode); the card's name, power limit and maximum SM clock
read in the same run.  Frames 0 and 63 of each call are checked against oracle/h264_enc.py.

A second section runs the engine on a 1080p clip (decode -> Blur -> Output into a database) with the output stored
lossless() and with compress_video() (QP 23, an IDR every 120 pictures): frames per second of the run (wall clock,
best of --runs) and the bytes the table holds.

    python tools/bench_h264.py [--iters 50] [--warmup 10] [--clip-frames 240] [--runs 3] [--json OUT]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import h264_enc as HE  # noqa: E402
from oracle import synth  # noqa: E402
from scanner_b200 import cabi  # noqa: E402

N, W, H, KD = 64, 1920, 1080, 120


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                       "-i", str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


class Encoder:
    """scn_h264_encode_u8 into a device buffer that is kept and grown, so calls time the encoder alone."""

    def __init__(self, frames, qp):
        self.L, self.qp = cabi.lib(), qp
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
        cabi.check(self.L.scn_h264_encode_u8(self.src, N, W, H, self.qp, None, KD, self.cb, None, self.sizes,
                                             self.stream), "scn_h264_encode_u8")

    def access_units(self):
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


def engine_section(frames, runs):
    """decode -> Blur -> Output with lossless() and with compress_video(): frames/s and stored bytes of each"""
    import scanner_b200 as sp
    from scanner_b200 import engine as E
    rgb = np.stack([synth.smooth_frame(500 + i, H, W) for i in range(frames)]).astype(np.int64)
    r, g, b = rgb[..., 0], rgb[..., 1], rgb[..., 2]
    y = ((66 * r + 129 * g + 25 * b + 128) >> 8) + 16
    cb = (((-38 * r - 74 * g + 112 * b + 128) >> 8) + 128)[:, ::2, ::2]
    cr = (((112 * r - 94 * g - 18 * b + 128) >> 8) + 128)[:, ::2, ::2]
    yuv = np.concatenate([p.reshape(frames, -1) for p in (y, cb, cr)], 1).astype(np.uint8)
    out = []
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "clip.mp4")
        open(path, "wb").write(E.mp4_mux(E.h264_synth(yuv, W, H, gop=30), 30, 1))
        sc = sp.Client(gpus=[torch.cuda.current_device()], db_path=os.path.join(tmp, "db"))
        video = sp.NamedVideoStream(sc, "clip", path=path)
        for label, store in (("lossless", lambda c: c.lossless()), ("compress_video", lambda c: c.compress_video())):
            best = None
            for k in range(runs + 1):  # the first run warms up
                name = f"{label}_{k}"
                blurred = sc.ops.Blur(frame=sc.io.Input([video]), kernel_size=3, sigma=0.5)
                t = time.perf_counter()
                sc.run(sc.io.Output(store(blurred), [sp.NamedVideoStream(sc, name)]), sp.PerfParams.estimate())
                dt = time.perf_counter() - t
                d = os.path.join(sc._db.path, "tables", str(sc._db.table_info(name)["id"]))
                stored = sum(os.path.getsize(os.path.join(d, f)) for f in os.listdir(d)
                             if f.startswith("1_") and f.endswith(".bin") and "metadata" not in f)
                if k and (best is None or dt < best):
                    best = dt
                sc._db.delete_table(name)
            row = {"output": label, "frames": frames, "frames_per_s": round(frames / best, 1),
                   "bytes_written": stored, "bytes_per_frame": stored // frames}
            out.append(row)
            print(f"engine {label:15s} {row['frames_per_s']:8.1f} frames/s  {stored:12d} bytes written "
                  f"({row['bytes_per_frame']} per frame)")
        sc.stop()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--clip-frames", type=int, default=240)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_h264 needs a CUDA device")
    info = card()
    print(f"# {info}; {N} x {W}x{H} RGB per call, keyframe_distance {KD}")
    rows = []
    for kind in ("smooth", "noise"):
        if kind == "smooth":
            host = np.stack([synth.smooth_frame(100 + i, H, W) for i in range(N)])
        else:
            host = np.random.default_rng(0).integers(0, 256, (N, H, W, 3), dtype=np.uint8)
        frames = torch.from_numpy(host).cuda()
        for qp in (23, 35):
            enc = Encoder(frames, qp)
            ms = time_calls(enc, args.iters, args.warmup)
            aus = enc.access_units()
            for i in (0, N - 1):
                want, rec = HE.encode_frame(host[i], qp, i, KD)
                assert aus[i] == want, f"{kind} QP {qp} frame {i} differs from the oracle"
                if i == 0:
                    psnr = HE.psnr(rec[0], HE.rgb_to_planes(host[0])[0][:H, :W])
            L = cabi.lib()
            L.scn_prof_enable(1)
            for _ in range(args.iters):
                enc()
            stages = {k: v["ms"] / args.iters for k, v in cabi.prof_report().items()}
            L.scn_prof_enable(0)
            out_bytes = sum(len(a) for a in aus)
            bound = max(stages, key=stages.get)
            row = {"content": kind, "qp": qp, "ms_per_call": round(ms, 3), "frames_per_s": round(N / (ms * 1e-3), 1),
                   "bytes_per_frame": out_bytes // N, "luma_psnr_db": round(psnr, 2),
                   "stages_ms": {k: round(v, 3) for k, v in stages.items()},
                   "kernels_ms": round(sum(stages.values()), 3), "bound_by": bound}
            rows.append(row)
            print(f"{kind:6s} QP {qp}  {ms:8.3f} ms/call  {row['frames_per_s']:9.1f} frames/s  "
                  f"{row['bytes_per_frame']:8d} B/frame  Y-PSNR {psnr:5.2f} dB")
            for k, v in sorted(stages.items(), key=lambda kv: -kv[1]):
                print(f"    {k:28s} {v:8.3f} ms  {100 * v / ms:5.1f} % of the call")
            print(f"    kernels {row['kernels_ms']:.3f} ms of {ms:.3f} ms per call; bound by {bound}")
    engine = engine_section(args.clip_frames, args.runs)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": info, "frames_per_call": N, "width": W, "height": H, "keyframe_distance": KD,
                       "rows": rows, "engine": engine}, f, indent=1)


if __name__ == "__main__":
    main()
