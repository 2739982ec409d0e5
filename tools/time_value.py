#!/usr/bin/env python
"""The value leg's step of bench.py, repeated: NV12 surfaces in HBM -> Histogram + Resize(224), --batch 1080p
surfaces per step (pitch 2048, two seeded batches alternating, as bench.py builds them).

    python tools/time_value.py [--windows 5] [--steps 200] [--batch 256]

Prints one JSON line: frames/s of each window (CUDA events around --steps steps), their median, the same windows
with the Histogram alone (time per streaming-kernel launch, memset and launch gaps included), the per-launch time
of every kernel with each kernel launched on its own (scn_prof_*, as bench.py's roofline leg), and a SHA-256 of the
last step's outputs.  SCN_KERNELS_LIB selects the library, so two builds can be alternated in one session:

    for i in 1 2 3; do SCN_KERNELS_LIB=old.so python tools/time_value.py; python tools/time_value.py; done
"""
import argparse
import hashlib
import json
import statistics
import sys
import threading
import time

import torch

sys.path.insert(0, ".")
from scanner_b200 import cabi, kernels  # noqa: E402

W, H, PITCH, DW, DH = 1920, 1080, 2048, 224, 224


class Nvml:
    """SM clock (MHz) and board power (W) of GPU 0, sampled every 2 ms from a thread between start() and stop()."""

    def __init__(self):
        import pynvml as nv
        nv.nvmlInit()
        self.nv, self.h = nv, nv.nvmlDeviceGetHandleByIndex(0)
        self.mhz, self.watts, self.run = [], [], False

    def _loop(self):
        nv = self.nv
        while self.run:
            self.mhz.append(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
            self.watts.append(nv.nvmlDeviceGetPowerUsage(self.h) / 1000)
            time.sleep(0.002)

    def start(self):
        self.mhz, self.watts, self.run = [], [], True
        self.t = threading.Thread(target=self._loop, daemon=True)
        self.t.start()

    def stop(self):
        self.run = False
        self.t.join()
        return {"sm_mhz_median": statistics.median(self.mhz), "sm_mhz_min": min(self.mhz),
                "power_w_median": round(statistics.median(self.watts))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--prof-steps", type=int, default=50)
    args = ap.parse_args()
    B = args.batch
    g = torch.Generator(device="cuda").manual_seed(1000)
    batches = [torch.randint(0, 256, (B, H * 3 // 2, PITCH), dtype=torch.uint8, device="cuda", generator=g)
               for _ in range(2)]
    plan = kernels.ResizePlan(W, H, DW, DH, "cuda")

    def step(i):
        return kernels.nv12_hist_resize(batches[i & 1], W, H, DW, DH, plan)

    for i in range(10):
        step(i)
    torch.cuda.synchronize()
    nvml = Nvml()
    fps, clocks = [], []
    for _ in range(args.windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        nvml.start()
        e0.record()
        for i in range(args.steps):
            last = step(i)
        e1.record()
        e1.synchronize()
        clocks.append(nvml.stop())
        fps.append(B * args.steps / (e0.elapsed_time(e1) * 1e-3))
    digest = hashlib.sha256()
    for t in last:
        digest.update(t.cpu().numpy().tobytes())

    # the same windows with the Histogram alone: one memset + ceil(B / 64) nv12_stream_kernel launches per step
    launches = -(-B // 64)
    hist_ms, hist_clocks = [], []
    for _ in range(args.windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        nvml.start()
        e0.record()
        for i in range(args.steps):
            kernels.nv12_hist_resize(batches[i & 1], W, H, DW, DH, plan, want_resize=False)
        e1.record()
        e1.synchronize()
        hist_clocks.append(nvml.stop())
        hist_ms.append(e0.elapsed_time(e1) / (args.steps * launches))

    L = cabi.lib()
    L.scn_prof_enable(1)
    nvml.start()
    for i in range(args.prof_steps):
        kernels.nv12_hist_resize(batches[i & 1], W, H, DW, DH, plan, want_resize=False)
        kernels.nv12_hist_resize(batches[i & 1], W, H, DW, DH, plan, want_hist=False)
    torch.cuda.synchronize()
    prof_clock = nvml.stop()
    prof = cabi.prof_report()
    L.scn_prof_enable(0)

    print(json.dumps({"lib": cabi.LIB_PATH, "gpu": torch.cuda.get_device_name(0), "batch": B,
                      "steps_per_window": args.steps, "fps_windows": [round(v) for v in fps],
                      "fps_median": round(statistics.median(fps)), "clocks_windows": clocks,
                      "hist_only_ms_per_launch_windows": [round(v, 5) for v in hist_ms],
                      "hist_only_ms_per_launch_median": round(statistics.median(hist_ms), 5),
                      "hist_only_clocks_windows": hist_clocks,
                      "kernel_ms_per_launch": {k: round(v["ms"] / v["launches"], 5) for k, v in prof.items()},
                      "clocks_kernels": prof_clock,
                      "outputs_sha256": digest.hexdigest()}))


if __name__ == "__main__":
    main()
