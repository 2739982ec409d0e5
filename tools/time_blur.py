#!/usr/bin/env python
"""CUDA-event timing of the box filter at BASELINE configs[2] size (16 x 4K frames) for several kernel sizes.
One JSON line."""
import json
import sys

import torch

sys.path.insert(0, ".")
from scanner_b200 import cabi, kernels  # noqa: E402

g = torch.Generator(device="cuda").manual_seed(3)
n, h, w = 16, 2160, 3840
frames = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda", generator=g)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
out = {}
for k in (3, 5, 7, 9, 15, 16, 17, 23, 31):
    kernels.blur(frames, k)
    ts = []
    for _ in range(7):
        flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        kernels.blur(frames, k)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    ms = ts[len(ts) // 2]
    out[f"k{k}"] = {"ms": round(ms, 4), "TBs": round(n * h * w * 6 / ms / 1e9, 3)}
print(json.dumps(out))
