#!/usr/bin/env python
"""How do decode sessions land on the NVDEC engines, and does dropping slow sessions fix a bad placement?

For `trials` fresh engines (7 pipeline instances = 7 decode sessions on one H100): four runs of the bench's
end-to-end workload (56 clips x 120 frames 1080p, GOP 30) each; per run the frames/s and every session's
picture rate (frames decoded / host time spent waiting on its engine).  One JSON line per run.
usage: python tools/nvdec_placement.py [trials]"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, ".")
from scanner_b200 import engine as E  # noqa: E402
from scanner_b200 import protolite  # noqa: E402

STD = protolite.parse_proto(open("scanner_b200/csrc/ops/stdlib_args.proto").read())


def clip(seed, n, gop=30):
    rng = np.random.default_rng(seed)
    yuv = rng.integers(0, 256, ((n + gop - 1) // gop, 1080 * 1920 * 3 // 2), dtype=np.uint8)
    return E.h264_synth(yuv, 1920, 1080, gop=gop, non_key="skip", frames=n)


class Sampler:
    """NVML clocks / utilisation while a run is in flight (50 ms period)."""

    def __init__(self):
        import threading
        import pynvml as nv
        nv.nvmlInit()
        self.nv, self.h = nv, nv.nvmlDeviceGetHandleByIndex(0)
        self.rows, self.stop = [], False
        self.t = threading.Thread(target=self.loop, daemon=True)
        self.t.start()

    def loop(self):
        nv = self.nv
        while not self.stop:
            try:
                dec = nv.nvmlDeviceGetDecoderUtilization(self.h)[0]
            except Exception:
                dec = -1
            self.rows.append((nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM), nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_VIDEO),
                              nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_MEM), nv.nvmlDeviceGetPerformanceState(self.h),
                              nv.nvmlDeviceGetPowerUsage(self.h) // 1000, dec))
            time.sleep(0.05)

    def take(self):
        rows, self.rows = self.rows, []
        if not rows:
            return None
        med = lambda k: sorted(r[k] for r in rows)[len(rows) // 2]
        return {"sm_mhz": med(0), "video_mhz": med(1), "video_mhz_min": min(r[1] for r in rows), "mem_mhz": med(2),
                "pstate": med(3), "power_w": med(4), "dec_util": med(5), "samples": len(rows)}


def cpu_stat():
    """cgroup v2 CPU accounting of this container: usage and CFS-throttling counters"""
    out = {}
    try:
        for line in open("/sys/fs/cgroup/cpu.stat"):
            k, v = line.split()
            out[k] = int(v)
    except Exception:
        pass
    return out


def main():
    import resource
    E.load_stdlib()
    sampler = Sampler()
    trials = int(sys.argv[1]) if len(sys.argv) > 1 else 6
    uniq = [clip(2000 + i, 120) for i in range(4)]
    for t in range(trials):
        eng = E.Engine(gpus=[0], instances_per_gpu=7)
        sids = [eng.add_h264(uniq[i % 4]) for i in range(56)]
        g = E.Graph()
        src = g.add_source(True)
        hs = g.add_op("Histogram", [(src, "frame")], device=1)
        rz = g.add_op("Resize", [(src, "frame")], device=1)
        g.add_sink((hs, "histogram"))
        g.add_sink((rz, "frame"))
        jobs = []
        for s in sids:
            j = E.Job()
            j.bind_source(src, s)
            j.set_stream_args(rz, protolite.encode(STD["ResizeArgs"], {"width": 224, "height": 224}))
            jobs.append(j)
        for run in range(4):
            sampler.take()
            c0, r0 = cpu_stat(), resource.getrusage(resource.RUSAGE_SELF)
            t0 = time.time()
            eng.run(g, jobs, 30, 60)
            dt = time.time() - t0
            c1, r1 = cpu_stat(), resource.getrusage(resource.RUSAGE_SELF)
            clocks = sampler.take()
            host = {"process_cpu_cores": round(((r1.ru_utime - r0.ru_utime) + (r1.ru_stime - r0.ru_stime)) / dt, 2),
                    "cgroup_cpu_cores": round((c1.get("usage_usec", 0) - c0.get("usage_usec", 0)) / 1e6 / dt, 2),
                    "cgroup_nr_throttled": c1.get("nr_throttled", 0) - c0.get("nr_throttled", 0),
                    "cgroup_throttled_ms": round((c1.get("throttled_usec", 0) - c0.get("throttled_usec", 0)) / 1e3, 1)}
            c = eng.stats()["counters"]
            rates = [round(c[f"inst{i}_frames_decoded"] * 1e6 / max(c[f"inst{i}_decode_busy_us"], 1)) for i in range(c["instances"])]
            print(json.dumps({"trial": t, "run": run, "fps": round(56 * 120 / dt), "session_pictures_per_s": rates,
                              "tasks": [c[f"inst{i}_tasks"] for i in range(c["instances"])],
                              "nvml": clocks, "host": host,
                              "host_us": {k: c[k] for k in ("nvdec_parse_us", "nvdec_map_us", "nvdec_decode_call_us", "nvdec_release_wait_us")}}),
                  flush=True)
        eng.close()


if __name__ == "__main__":
    main()
