#!/usr/bin/env python
"""Kernel time of GaussianBlur: 64 x 1080p frames per launch, k x k kernels for k in 3, 5, 7, 15, 31 (sigma 0, the
default border), from dense RGB24, from gray (HxWx1) and from packed NV12 elements (the decode stage's format).  CUDA
events around `--iters` launches after `--warmup` launches; prints one line per case with the algorithmic bytes
(source read once, output written once: 2 C WH from frames, 1.5 WH + 3 WH from NV12) over kernel time, the share of
the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), and the card's name, power limit and clock read in the same run.

    python tools/bench_gaussian_blur.py [--iters 50] [--warmup 10] [--json OUT]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from scanner_b200 import cabi, kernels  # noqa: E402

HBM_PEAK = 3.35e12
N, W, H = 64, 1920, 1080
KS = (3, 5, 7, 15, 31)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def time_launches(fn, iters, warmup):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gaussian_blur needs a CUDA device")
    L = cabi.lib()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    gen = torch.Generator(device="cuda").manual_seed(0)
    rgb = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, device="cuda", generator=gen)
    gray = torch.randint(0, 256, (N, H, W, 1), dtype=torch.uint8, device="cuda", generator=gen)
    nv12 = torch.randint(0, 256, (N, H * 3 // 2, W), dtype=torch.uint8, device="cuda", generator=gen)
    out = torch.empty((N, H, W, 3), dtype=torch.uint8, device="cuda")
    info = card()
    print(f"# {info}; {N} x {W}x{H} per launch")
    ms = time_launches(lambda: out.copy_(rgb), args.iters, args.warmup)
    copy_gbs = 2 * rgb.numel() / (ms * 1e-3) / 1e9
    print(f"{'copy (torch)':14s} rgb24  {ms:7.3f} ms/launch  {copy_gbs:7.1f} GB/s  "
          f"{100 * copy_gbs * 1e9 / HBM_PEAK:5.1f} % of 3.35 TB/s")
    rows = [{"k": 0, "from": "copy", "ms_per_launch": round(ms, 4), "GB_per_s": round(copy_gbs, 1),
             "share_of_hbm_peak": round(copy_gbs * 1e9 / HBM_PEAK, 3)}]
    lp, k_l = cabi.ptr_array([nv12.data_ptr() + i * H * W * 3 // 2 for i in range(N)])
    cp, k_c = cabi.ptr_array([nv12.data_ptr() + i * H * W * 3 // 2 + H * W for i in range(N)])
    for k in KS:
        plan = kernels.gaussian_blur_plan((k, k), 0.0)
        pp = plan.ctypes.data
        for kind, c in (("rgb24", 3), ("gray", 1), ("nv12", 3)):
            dst, k_d = cabi.ptr_array([out.data_ptr() + i * H * W * c for i in range(N)])
            if kind == "nv12":
                frame_bytes = (3 * W * H) // 2 + 3 * W * H
                fn = lambda: cabi.check(L.scn_gaussian_blur_nv12(pp, lp, cp, W, N, W, H, dst, stream), "nv12")  # noqa
            else:
                src = rgb if c == 3 else gray
                sp_, k_s = cabi.ptr_array([src.data_ptr() + i * H * W * c for i in range(N)])
                frame_bytes = 2 * c * W * H
                fn = lambda: cabi.check(L.scn_gaussian_blur_u8(pp, sp_, N, W, H, c, dst, stream), "u8")  # noqa
            ms = time_launches(fn, args.iters, args.warmup)
            gbs = N * frame_bytes / (ms * 1e-3) / 1e9
            rows.append({"k": k, "from": kind, "ms_per_launch": round(ms, 4), "bytes_per_frame": frame_bytes,
                         "GB_per_s": round(gbs, 1), "share_of_hbm_peak": round(gbs * 1e9 / HBM_PEAK, 3)})
            print(f"k={k:<3d} from {kind:5s}  {ms:7.3f} ms/launch  {gbs:7.1f} GB/s  "
                  f"{100 * gbs * 1e9 / HBM_PEAK:5.1f} % of 3.35 TB/s")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": info, "frames_per_launch": N, "width": W, "height": H, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
