#!/usr/bin/env python
"""BASELINE.json configs[2..4] on one GPU (SURVEY 8d: two numbers per config -- the kernel stage
on device-resident batches against the HBM roofline, and end to end through the pipeline with the
decode-bound ceiling stated).  configs[1] is bench.py's headline.  Prints one JSON object per config.

    python tools/bench_configs.py [--steps 3] [--gpu 0]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scanner_b200 import cabi, kernels, protolite  # noqa: E402
from scanner_b200 import engine as E  # noqa: E402

PEAK = 6567.4  # GB/s, MEASURED_PEAKS.json copy bandwidth (bench.py reads the file; same number)
STD = protolite.parse_proto(open(os.path.join(os.path.dirname(E.ENGINE_PATH), "..", "csrc", "ops",
                                              "stdlib_args.proto")).read())


def clip(seed, w, h, frames, gop=30):
    rng = np.random.default_rng(seed)
    k = (frames + gop - 1) // gop
    yuv = rng.integers(0, 256, (k, h * w * 3 // 2), dtype=np.uint8)
    return E.h264_synth(yuv, w, h, gop=gop, non_key="skip", frames=frames)


def inst(args, tuned):
    """pipeline instances per GPU: --instances, else the value tuned for the config (the reference's
    pipeline_instances_per_node knob): P_Skip-heavy 1080p decode is best at one session per NVDEC
    engine (7), IDR-heavy or 4K decode at two (14)."""
    return args.instances if args.instances > 0 else tuned


def gpu_list(args):
    return [args.gpu] if args.ngpus <= 1 else list(range(args.ngpus))


def timed(fn, steps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def run_engine(eng, graph, jobs, wps, ios, steps):
    for _ in range(2):
        eng.run(graph, jobs, wps, ios)
    t0 = time.perf_counter()
    for _ in range(steps):
        eng.run(graph, jobs, wps, ios)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def config2(args):
    """4K decode + Blur(3) + Histogram."""
    w, h, n = 3840, 2160, 16
    g = torch.Generator(device="cuda").manual_seed(2)
    batches = [torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda", generator=g) for _ in range(2)]
    i = [0]

    def step():
        i[0] += 1
        return kernels.histogram(kernels.blur(batches[i[0] & 1], 3))
    ms = timed(step, 10)
    alg = n * (3 * w * h * 2 + 3 * w * h + 192)  # blur reads + writes a frame, histogram reads it again
    L = cabi.lib()
    L.scn_prof_enable(1)
    for _ in range(5):
        step()
    torch.cuda.synchronize()
    prof = {k: v["ms"] / v["launches"] for k, v in cabi.prof_report().items()}
    L.scn_prof_enable(0)
    clips, frames = 4 * args.ngpus * args.clip_mult, 60
    eng = E.Engine(gpus=gpu_list(args), instances_per_gpu=inst(args, 14))
    data = [clip(300 + k, w, h, frames) for k in range(2)]
    sids = [eng.add_h264(data[k % 2]) for k in range(clips)]
    graph = E.Graph()
    src = graph.add_source(True)
    bl = graph.add_op("Blur", [(src, "frame")], device=1,
                      args=protolite.encode(STD["BlurArgs"], {"kernel_size": 3, "sigma": 0.5}))
    hs = graph.add_op("Histogram", [(bl, "frame")], device=1)
    sink = graph.add_sink((hs, "histogram"))
    jobs = []
    for sid in sids:
        j = E.Job()
        j.bind_source(src, sid)
        jobs.append(j)
    sec = run_engine(eng, graph, jobs, 15, 30, args.steps)
    assert jobs[0].output_rows(sink) == frames
    eng.close()
    return {"config": "configs[2]: 4K H.264 decode + Blur(3) + Histogram", "kernel_stage": {
        "frames_per_s": n / (ms * 1e-3), "ms_per_16_frames": ms, "alg_bytes_per_frame": alg // n,
        "achieved_GBs": alg / (ms * 1e-3) / 1e9, "frac_of_hbm_peak": alg / (ms * 1e-3) / 1e9 / PEAK,
        "kernels_ms": prof}, "e2e": {"frames_per_s": clips * frames / sec, "clips": clips, "frames_per_clip": frames, "n_gpus": args.ngpus,
                                     "bound": "NVDEC (4K: ~4x the pixels of 1080p per picture)"}}


def config3(args):
    """1080p dense OpticalFlow, stencil [0, 1] (Farneback: the in-tree op; TV-L1 does not exist upstream)."""
    w, h, n = 1920, 1080, 4
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda", generator=g)
    b = torch.roll(a, shifts=(1, 2), dims=(1, 2)).contiguous()
    ms = timed(lambda: kernels.optical_flow(a, b), 5) / n
    clips, frames = 2 * args.ngpus, 60
    eng = E.Engine(gpus=gpu_list(args), instances_per_gpu=inst(args, 7))
    sids = [eng.add_h264(clip(400 + k, w, h, frames)) for k in range(clips)]
    graph = E.Graph()
    src = graph.add_source(True)
    fl = graph.add_op("OpticalFlow", [(src, "frame")], device=1)
    sink = graph.add_sink((fl, "flow"))
    jobs = []
    for sid in sids:
        j = E.Job()
        j.bind_source(src, sid)
        jobs.append(j)
    sec = run_engine(eng, graph, jobs, 10, 30, args.steps)
    assert jobs[0].output_rows(sink) == frames
    if os.environ.get("SCN_BENCH_STATS"):
        print(json.dumps(eng.stats()), file=sys.stderr)
    eng.close()
    lower = 2 * w * h * 3 + 8 * w * h  # two RGB frames in, one flow field out
    return {"config": "configs[3]: 1080p OpticalFlow (Farneback) stencil [0,1]", "kernel_stage": {
        "pairs_per_s": 1e3 / ms, "ms_per_pair": ms, "lower_bound_bytes_per_pair": lower,
        "frac_of_hbm_peak_at_lower_bound": lower / (ms * 1e-3) / 1e9 / PEAK},
        "e2e": {"frames_per_s": clips * frames / sec, "clips": clips, "frames_per_clip": frames,
                "d2h_bytes_per_frame": w * h * 8, "bound": "flow kernels + 16.6 MB/frame D2H of the flow field"}}


def config4(args):
    """Stride(30) over many 1080p clips, GOP 30: only IDR pictures are needed -- decode-bound."""
    w, h = 1920, 1080
    clips, frames = 56 * args.ngpus, 300
    eng = E.Engine(gpus=gpu_list(args), instances_per_gpu=inst(args, 14))
    data = [clip(500 + k, w, h, frames) for k in range(2)]
    sids = [eng.add_h264(data[k % 2]) for k in range(clips)]
    graph = E.Graph()
    src = graph.add_source(True)
    smp = graph.add_sample((src, "frame"))
    hs = graph.add_op("Histogram", [(smp, "frame")], device=1)
    sink = graph.add_sink((hs, "histogram"))
    jobs = []
    for sid in sids:
        j = E.Job()
        j.bind_source(src, sid)
        j.set_sampler(smp, "Strided", protolite.encode(protolite.SAMPLER_ARGS["StridedSamplerArgs"], {"stride": 30}))
        jobs.append(j)
    sec = run_engine(eng, graph, jobs, 10, 10, args.steps)
    c = eng.stats()["counters"]
    assert jobs[0].output_rows(sink) == frames // 30
    eng.close()
    used = clips * (frames // 30)
    return {"config": "configs[4]: Stride(30) Histogram over 1080p clips (GOP 30)", "e2e": {
        "frames_used_per_s": used / sec, "source_frames_covered_per_s": clips * frames / sec, "clips": clips,
        "frames_per_clip": frames, "n_gpus": args.ngpus, "frames_decoded_last_run": c["frames_decoded"], "frames_used_last_run": c["frames_used"],
        "bound": "NVDEC: one ~3 MB I_PCM IDR picture per used frame; nothing else of a GOP is fed"}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--gpu", type=int, default=0)
    ap.add_argument("--instances", type=int, default=0, help="pipeline instances per GPU (0: one per NVDEC engine)")
    ap.add_argument("--only", default="")
    ap.add_argument("--clip-mult", type=int, default=1, help="multiply the number of clips of the e2e legs")
    ap.add_argument("--ngpus", type=int, default=1, help="GPUs driven by ONE engine (tasks sharded over all of them)")
    args = ap.parse_args()
    E.load_stdlib()
    torch.cuda.set_device(args.gpu)
    for name, fn in (("2", config2), ("3", config3), ("4", config4)):
        if args.only and name not in args.only.split(","):
            continue
        print(json.dumps(fn(args)), flush=True)


if __name__ == "__main__":
    main()
