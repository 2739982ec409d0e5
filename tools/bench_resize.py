#!/usr/bin/env python
"""Kernel time of Resize per interpolation mode: 64 frames per launch, 1080p and 2160p to 224 x 224 with
INTER_NEAREST, INTER_LINEAR and INTER_AREA, from dense RGB24 and from packed NV12 elements (the decode stage's format),
plus 224 x 224 to 1080p with INTER_AREA (resize_linear_kernel with area taps).  CUDA events around `--iters` launches
after `--warmup` launches.  Each line gives the algorithmic bytes over kernel time and their share of the H100 SXM
data-sheet HBM3 bandwidth (3.35 TB/s); the card's name and power limit are read in the same run.

Byte model: INTER_AREA downscales read every source byte once (3 WH from RGB24, 1.5 WH from NV12) and write the
destination (3 dw dh).  INTER_NEAREST and INTER_LINEAR read only the pixels their taps touch, so for them the same
figure is an upper bound on useful traffic, given for comparison; upscales count source plus destination.

    python tools/bench_resize.py [--iters 50] [--warmup 10] [--json OUT]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from scanner_b200 import cabi  # noqa: E402

HBM_PEAK = 3.35e12
N = 64
MODES = {"INTER_NEAREST": 0, "INTER_LINEAR": 1, "INTER_AREA": 3}
CASES = [(1920, 1080, 224, 224, m) for m in MODES] + [(3840, 2160, 224, 224, m) for m in MODES] + \
        [(224, 224, 1920, 1080, "INTER_AREA")]


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


def plan(mode, sw, sh, dw, dh):
    L = cabi.lib()
    host = np.zeros(L.scn_resize_interp_plan_bytes(MODES[mode], sw, sh, dw, dh), np.uint8)
    cabi.check(L.scn_resize_interp_plan_fill(MODES[mode], sw, sh, dw, dh, host.ctypes.data), "plan_fill")
    return torch.from_numpy(host).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resize needs a CUDA device")
    L = cabi.lib()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    gen = torch.Generator(device="cuda").manual_seed(0)
    info = card()
    print(f"# {info}; {N} frames per launch")
    rows = []
    for (sw, sh, dw, dh, mode) in CASES:
        rgb = torch.randint(0, 256, (N, sh, sw, 3), dtype=torch.uint8, device="cuda", generator=gen)
        nv12 = torch.randint(0, 256, (N, sh * 3 // 2, sw), dtype=torch.uint8, device="cuda", generator=gen)
        out = torch.empty((N, dh, dw, 3), dtype=torch.uint8, device="cuda")
        p = plan(mode, sw, sh, dw, dh)
        sp_, k1 = cabi.ptr_array([rgb.data_ptr() + i * sh * sw * 3 for i in range(N)])
        lp, k2 = cabi.ptr_array([nv12.data_ptr() + i * sh * sw * 3 // 2 for i in range(N)])
        cp, k3 = cabi.ptr_array([nv12.data_ptr() + i * sh * sw * 3 // 2 + sh * sw for i in range(N)])
        dp, k4 = cabi.ptr_array([out.data_ptr() + i * dh * dw * 3 for i in range(N)])
        code = MODES[mode]
        cases = [("rgb24", 3 * sw * sh + 3 * dw * dh,
                  lambda: cabi.check(L.scn_resize_interp_u8c3(code, sp_, N, sw, sh, dp, dw, dh, p.data_ptr(), stream),
                                     mode)),
                 ("nv12", 3 * sw * sh // 2 + 3 * dw * dh,
                  lambda: cabi.check(L.scn_resize_interp_nv12(code, lp, cp, sw, N, sw, sh, dp, dw, dh, p.data_ptr(),
                                                              stream), mode))]
        for src_kind, frame_bytes, fn in cases:
            ms = time_launches(fn, args.iters, args.warmup)
            gbs = N * frame_bytes / (ms * 1e-3) / 1e9
            rows.append({"mode": mode, "from": src_kind, "src": [sw, sh], "dst": [dw, dh],
                         "ms_per_launch": round(ms, 4), "bytes_per_frame": frame_bytes, "GB_per_s": round(gbs, 1),
                         "share_of_hbm_peak": round(gbs * 1e9 / HBM_PEAK, 3)})
            print(f"{mode:14s} {sw}x{sh}->{dw}x{dh:<5d} from {src_kind:5s}  {ms:7.3f} ms/launch  {gbs:7.1f} GB/s  "
                  f"{100 * gbs * 1e9 / HBM_PEAK:5.1f} % of 3.35 TB/s")
        del rgb, nv12, out
        torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": info, "frames_per_launch": N, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
