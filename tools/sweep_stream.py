#!/usr/bin/env python3
"""Build-variant sweep of the NV12 streaming kernel (nv12_stream.cuh): warps per CTA, ring depth, chroma
conversion pipe.

    python tools/sweep_stream.py build     # here (no GPU): build/variants/<tag>/libscn_kernels.so
    python tools/sweep_stream.py run OUT   # on a GPU: time + check every variant, one JSON line each, all in OUT
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILDS = {"w8": "-DNVS_WARPS=8", "w12": "-DNVS_WARPS=12", "w16": "-DNVS_WARPS=16"}
# (build, SCN_NV12_RESIZE): how Histogram + Resize of the same surfaces run (fused.cu)
RUNS = [("w12", "fused"), ("w12", "split"), ("w12", "overlap"), ("w8", "fused"), ("w8", "split"), ("w8", "overlap"),
        ("w16", "split")]


def build():
    for tag, extra in BUILDS.items():
        out = os.path.join(ROOT, "build", "variants", tag)
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "scanner_b200", "csrc"), "-j8", f"OBJ={out}/obj", f"OUT={out}",
                               f"EXTRA={extra}"], stdout=subprocess.DEVNULL)
        log = open(os.path.join(out, "obj", "fused.ptxas.log")).read()
        i = log.index("nv12_stream_kernelILb0")
        print(tag, [l.strip() for l in log[i:].splitlines()[1:4]])


CHILD = r'''
import json, sys, torch
sys.path.insert(0, ".")
from scanner_b200 import cabi, kernels
g = torch.Generator(device="cuda").manual_seed(5)
L = cabi.lib()
n, h, w, pitch = 64, 1080, 1920, 2048
surf = torch.randint(0, 256, (n, h * 3 // 2, pitch), dtype=torch.uint8, device="cuda", generator=g)
plan = kernels.ResizePlan(w, h, 224, 224)
rgb = kernels.nv12_to_rgb(surf, w, h)
ref_h = kernels.histogram(rgb)
ref_r = kernels.resize(rgb, 224, 224)
out = {}
for name, want_resize in (("hist", False), ("hist+resize", True)):
    hist, res = kernels.nv12_hist_resize(surf, w, h, 224, 224, plan, want_resize=want_resize)
    ok = bool((hist == ref_h).all()) and (not want_resize or bool((res == ref_r).all()))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ts = []
    for _ in range(12):
        flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        kernels.nv12_hist_resize(surf, w, h, 224, 224, plan, want_resize=want_resize)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    us = ts[len(ts) // 2]
    out[name] = {"ok": ok, "us": round(us, 1), "TBs": round(n * (h * w * 1.5) / us / 1e6, 3)}
print(json.dumps(out))
'''


def run(out_path):
    res = {}
    for build_tag, mode in RUNS:
        tag = f"{build_tag}_{mode}"
        so = os.path.join(ROOT, "build", "variants", build_tag, "libscn_kernels.so")
        env = dict(os.environ, SCN_KERNELS_LIB=so, SCN_NV12_RESIZE=mode)
        r = subprocess.run([sys.executable, "-c", CHILD], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        line = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ""
        try:
            res[tag] = json.loads(line)
        except Exception:
            res[tag] = {"error": r.stdout[-400:]}
        print(tag, res[tag], flush=True)
    json.dump(res, open(out_path, "w"), indent=1)


if __name__ == "__main__":
    build() if sys.argv[1] == "build" else run(sys.argv[2])
