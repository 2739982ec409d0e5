"""Measure TV-L1 (scn_tvl1_u8) on 1080p pairs, and the OpticalFlowTVL1 op in an engine run of configs[3]'s shape.

    python tools/bench_tvl1.py [--reps 3]

Prints the card (name, power limit, SM clock), then per (n pairs, epsilon): ms per call and per pair (CUDA
events around the call, median of --reps after a warm-up call), the iterations each (level, warp) ran, the
bytes the byte model below says the call moves and that over the time against the 3.35 TB/s data-sheet HBM3
bandwidth.  epsilon = -1 (no early stop) runs 50 iterations per warp: the iteration-bound case.  Last, one engine
run (synthetic 1080p H.264 clip -> NV12 elements -> OpticalFlowTVL1 stencil [0, 1], one GPU) in frames/s.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import tvl1 as T  # noqa: E402
from scanner_b200 import engine as E  # noqa: E402
from scanner_b200 import kernels  # noqa: E402

HBM_TBS = 3.35
W, H = 1920, 1080


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "nvidia-smi unavailable"


def level_sizes(w, h, nscales=5, step=0.8):
    sizes = [(w, h)]
    while len(sizes) < nscales:
        nw, nh = int(np.floor(sizes[-1][0] * step + 0.5)), int(np.floor(sizes[-1][1] * step + 0.5))
        if nw < 16 or nh < 16:
            break
        sizes.append((nw, nh))
    return sizes


# Byte model, per pixel of a level (float32 planes; neighbour taps assumed to hit in cache):
#   iteration, v/u phase:  reads wx, wy, rho_c, u1, u2, p11, p12, p21, p22; writes u1, u2       44 B
#   iteration, p phase:    reads u1, u2, p11, p12, p21, p22; writes p11, p12, p21, p22          40 B
#   warp step:             reads u1, u2, I0 + I1, Ix, Iy (once); writes wx, wy, rho_c           36 B
#                          median of u1, u2: reads 2, writes 2 planes                           16 B
#   level:                 Ix, Iy from I1 (read 1, write 2) and p = 0 (write 4)                 28 B
#                          u upsample (write 2; the coarse read is small)                        8 B
ITER_B, WARP_B, LEVEL_B = 84, 52, 36


def model_bytes(iters, sizes, warps):
    """iters: int [n][nscales][warps] from return_iterations"""
    total = 0
    for pair in iters:
        for s, (w, h) in enumerate(sizes):
            px = w * h
            total += px * (ITER_B * int(pair[s].sum()) + WARP_B * warps + LEVEL_B)
    return total + len(iters) * W * H * (2 * 1 + 2 * 4 + 8)  # u8 in, float level 0 out, the flow out


def time_calls(prev, nxt, reps, **kw):
    kernels.tvl1_flow(prev, nxt, **kw)  # warm-up (module load, workspace)
    ws = torch.empty(kernels.tvl1_workspace_bytes(W, H, prev.shape[0]), dtype=torch.uint8, device="cuda")
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        kernels.tvl1_flow(prev, nxt, workspace=ws, **kw)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    _, iters = kernels.tvl1_flow(prev, nxt, workspace=ws, return_iterations=True, **kw)
    return float(np.median(ts)), iters


def engine_run(frames=48):
    rng = np.random.default_rng(1)
    yy, xx = np.mgrid[0:H, 0:W]
    ys = [(128 + 60 * np.sin(0.05 * (xx - 2 * i)) * np.cos(0.04 * yy) + rng.normal(0, 2, (H, W))).clip(0, 255)
          .astype(np.uint8).reshape(-1) for i in range(frames)]
    uv = np.full(W * H // 2, 128, np.uint8)
    yuv = np.stack([np.concatenate([y, uv]) for y in ys])
    E.load_stdlib()
    eng = E.Engine(gpus=[0], instances_per_gpu=1)
    try:
        sid = eng.add_h264(E.h264_synth(yuv, W, H, gop=24))
        g = E.Graph()
        src = g.add_source(True)
        fl = g.add_op("OpticalFlowTVL1", [(src, "frame")], device=1)
        g.add_sink((g.add_op("FrameDigest", [(fl, "flow")], device=1), "digest"))
        j = E.Job()
        j.bind_source(src, sid)
        eng.run(g, [j], 8, 24)  # warm-up
        t = time.perf_counter()
        eng.run(g, [j], 8, 24)
        return frames / (time.perf_counter() - t)
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print("card:", card())
    pairs = [T.flow_pair_known(s, H, W, "shift")[:2] for s in range(4)]
    sizes = level_sizes(W, H)
    results = []
    for n in (1, 4, 16):
        prev = torch.from_numpy(np.stack([pairs[i % 4][0] for i in range(n)])).cuda()
        nxt = torch.from_numpy(np.stack([pairs[i % 4][1] for i in range(n)])).cuda()
        for eps, its in ((0.01, 300), (-1.0, 50)):
            ms, iters = time_calls(prev, nxt, a.reps, epsilon=eps, iterations=its)
            nbytes = model_bytes(iters, sizes, 5)
            r = dict(n=n, epsilon=eps, iterations=its, ms_per_call=round(ms, 2), ms_per_pair=round(ms / n, 2),
                     iterations_run_pair0=iters[0, :len(sizes)].tolist(),
                     model_GB=round(nbytes / 1e9, 2), achieved_TBs=round(nbytes / ms / 1e9, 3),
                     share_of_hbm=round(nbytes / ms / 1e9 / HBM_TBS, 3))
            print(json.dumps(r))
            results.append(r)
    print(json.dumps({"engine_1080p_tvl1_frames_per_s": round(engine_run(), 2)}))
    print("card:", card())


if __name__ == "__main__":
    main()
