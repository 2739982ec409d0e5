#!/usr/bin/env python
"""bench.py -- BASELINE.json configs[1]: 1080p H.264 decode + Resize(224) + Histogram, frames/s.

    python bench.py --gpus N --steps K --warmup W                    # our arm (one rank per GPU)
    python bench.py --impl reference --gpus N --steps K --warmup W   # CPU reference arm (rank 0)
    python bench.py --config 3 --gpus N ...                          # configs[3]: OpticalFlow, one clip over N GPUs

A "step" is one pass of the hot path over one batch of `--batch` decoded 1080p surfaces (NV12,
NVDEC layout, pitch 2048): surfaces -> RGB -> {Histogram 3x16 int32, Resize 224x224 RGB24}.
  value   frames/s over all ranks with the surfaces already resident in HBM (CUDA events, max
          over ranks); inputs rotate between two batches, each larger than the 50 MB L2.
  e2e     same metric end to end through the public pipeline API as configs[1] states it, on a stream with a real
          encoder's structure (scanner_b200/synth_h264.py; `e2e_ipcm_stream` repeats it on r01's lossless stream): the clips are
          TABLES of a database directory shared by all ranks (ingested H.264 + stored index); every step
          each rank binds its shard of the table list, runs scn_engine_run (host H.264 -> NVDEC ->
          Histogram + Resize(224) GPU ops -> host rows) with the save stage writing every finished task
          into output tables of the same database, and commits them.  Timed per step (barrier, wall clock,
          max over ranks), the steps summed; h2d/d2h bytes are the encoded bytes fed and the rows returned.
  roofline  the one kernel of the value leg (nv12_stream_kernel: histogram + resize in one pass over the
          surfaces): algorithmic bytes / its CUDA-event duration (scn_prof_*), against MEASURED_PEAKS.json's
          HBM copy bandwidth when that file exists, else the H100 SXM data-sheet figure (3.35 TB/s).
  cpu_baseline  the reference's CPU path restated with the libraries it calls (FFmpeg H.264
          decode through cv2.VideoCapture, cv2.calcHist x3, cv2.resize; one clip per process, as
          the reference runs one pipeline instance per core) on a bounded sample of the same
          clips on this box's host cores (rank 0, N=1 only).  The clips of the reference arm come from
          oracle/h264_writer.py (pure numpy): that arm loads no product library.
configs[0] (Histogram on one 640x480 H.264 clip, CPU pipeline_instances=1, no GPU) is run beside it on rank 0 at N=1
as `config0_cpu`: the engine's CPU instance decodes with FFmpeg (libavcodec + libswscale through dlopen,
scanner_b200/csrc/engine/swdec.h -- what the reference's SoftwareVideoDecoder is) and the stdlib Histogram runs on
the CPU; a second or two, sampled rows checked against cv2 + the oracle.  Not part of `value` / `e2e`.
Prints ONE JSON line on rank 0.  --dump-outputs DIR writes what the value leg's last timed step computed (rank 0) as
float32 .npy files: hist.npy (batch, 3, 16) and resize_sample.npy, the Resize(224) rows of a fixed seeded sample of
at most 64 of its frames, with their indices in resize_sample_frames.npy.  Inputs are seeded: the same arguments give
the same inputs on every run.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

W, H, PITCH = 1920, 1080, 2048
DW, DH = 224, 224
SURF_ROWS = H * 3 // 2
B_ALG_FUSED = W * H * 3 // 2 + DW * DH * 3 + 192      # SURVEY 8(d): 3,261,120 B / frame
B_ALG_HIST_NV12 = W * H * 3 // 2 + 192                  # the histogram kernel alone
METRIC = "frames/sec (1080p H.264 decode+resize+histogram)"


def config0_cpu(frames=720):
    """BASELINE configs[0] as stated (SURVEY 8d "Config 1": one 640x480 clip of 720 frames, GOP 24, CPU Histogram,
    pipeline_instances = 1, work_packet 10, io_packet 100; pass = every row equal to the oracle's histogram of the same
    decoded RGB), on this box's host."""
    import cv2
    import numpy as np
    import oracle
    from scanner_b200 import engine as E, synth_h264
    caps = E.swdec_caps()
    if not caps["available"]:
        return {"unavailable": caps.get("error", "")}
    data, _ = synth_h264.write(640, 480, frames, gop=24, seed=9)
    E.load_stdlib()
    eng = E.Engine(gpus=[], cpu_instances=1)
    sid = eng.add_h264(data)
    g = E.Graph()
    src = g.add_source(True)
    sink = g.add_sink((g.add_op("Histogram", [(src, "frame")], device=0), "histogram"))
    j = E.Job()
    j.bind_source(src, sid)
    eng.run(g, [j], 10, 100)                     # warm: libraries loaded, codec opened
    t0 = time.perf_counter()
    eng.run(g, [j], 10, 100)
    dt = time.perf_counter() - t0
    hist = j.output_array(sink, 192, np.int32).reshape(frames, 3, 16)
    dec_threads = int(os.environ.get("SCN_SWDEC_THREADS", "1"))
    tmp = tempfile.mkdtemp(prefix="scn_c0_")
    try:
        path = os.path.join(tmp, "c.h264")
        open(path, "wb").write(data)
        cap = cv2.VideoCapture(path)
        checked = 0
        for i in range(frames):
            ok, f = cap.read()
            assert ok
            assert (hist[i] == oracle.hist16(np.ascontiguousarray(f[..., ::-1]))).all(), i   # every row
            checked += 1
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    eng.close()
    return {"workload": "configs[0]: Histogram on one 640x480 H.264 clip, CPU pipeline_instances=1 (no GPU)",
            "value": frames / dt, "unit": "frames/s", "frames": frames, "pipeline_instances": 1,
            "decoder_threads": dec_threads,
            "decoder": f"libavcodec {caps['avcodec']} / libswscale {caps['swscale']} via dlopen ({os.path.basename(caps['where'])})",
            "rows_checked_against_cv2_and_oracle": checked}


H100_HBM_GBS = 3350.0   # NVIDIA H100 SXM data sheet, HBM3


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return json.load(open(p)).get("hbm_gbs", H100_HBM_GBS), "measured (burst copy, MEASURED_PEAKS.json)"
    return H100_HBM_GBS, "H100 SXM data sheet"


class ClockSampler(threading.Thread):
    """Samples SM / video clocks, decoder utilisation and throttle reasons of one GPU (pynvml)."""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.samples, self.video, self.dec, self.reasons, self.stop_flag = index, [], [], [], set(), False
        self.max_mhz = None

    def setup(self):
        import pynvml as nv
        nv.nvmlInit()
        self.nv = nv
        self.h = nv.nvmlDeviceGetHandleByIndex(self.index)
        self.max_mhz = nv.nvmlDeviceGetMaxClockInfo(self.h, nv.NVML_CLOCK_SM)
        self.names = {nv.nvmlClocksThrottleReasonHwSlowdown: "hw_slowdown",
                      nv.nvmlClocksThrottleReasonHwThermalSlowdown: "hw_thermal_slowdown",
                      nv.nvmlClocksThrottleReasonSwThermalSlowdown: "sw_thermal_slowdown",
                      nv.nvmlClocksThrottleReasonSwPowerCap: "sw_power_cap",
                      nv.nvmlClocksThrottleReasonHwPowerBrakeSlowdown: "hw_power_brake"}

    def sample_now(self):
        """One sample from the calling thread (used while the timed steps are in flight)."""
        try:
            if not hasattr(self, "h"):
                self.setup()
            nv = self.nv
            self.samples.append(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
            try:
                self.video.append(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_VIDEO))
                self.dec.append(nv.nvmlDeviceGetDecoderUtilization(self.h)[0])
            except Exception:
                pass
            r = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
            for bit, name in self.names.items():
                if r & bit:
                    self.reasons.add(name)
        except Exception as e:  # clocks are evidence, not a dependency
            self.reasons.add(f"nvml_unavailable:{type(e).__name__}")

    def run(self):
        while not self.stop_flag:
            self.sample_now()
            time.sleep(0.005)

    def reset(self):
        self.samples, self.video, self.dec = [], [], []

    @staticmethod
    def _med(v):
        v = sorted(v)
        return v[len(v) // 2] if v else None

    def result(self):
        return {"sm_mhz": self._med(self.samples), "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons),
                "samples": len(self.samples)}

    def video_result(self):
        return {"video_mhz": self._med(self.video), "decoder_util_pct": self._med(self.dec), "samples": len(self.video)}


def usable_cores():
    """Host cores this process may actually use: scheduler affinity capped by the cgroup CPU quota
    (a container can see every host CPU and still run under a cgroup quota of a few cores)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if quota != "max":
            n = min(n, max(1, -(-int(quota) // int(period))))
    except Exception:
        pass
    return max(1, n)


# ------------------------------------------------------------------------------------------
def clip_yuv(seed, frames, gop=30, w=W, h=H):
    import numpy as np
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, ((frames + gop - 1) // gop, h * w * 3 // 2), dtype=np.uint8)


def make_clip_bytes(seed, frames, gop=30, w=W, h=H):
    """Synthetic H.264 (SURVEY 7: no encoder offline): I_PCM IDR every `gop` frames with uniform-random
    planes, the pictures in between P_Skip -> ~105 KB/frame at 1080p.  Product writer (scn_h264_synth)."""
    from scanner_b200 import engine as E
    return E.h264_synth(clip_yuv(seed, frames, gop, w, h), w, h, gop=gop, non_key="skip", frames=frames)


def make_clip_cavlc(seed, frames, gop=30):
    """A stream a real encoder could have produced (scanner_b200/synth_h264.py, pure numpy: Intra16x16 + CAVLC key
    pictures, motion-compensated P pictures; ~35 KB per key picture, ~5 KB per P picture) -> (bytes, expected I420)."""
    from scanner_b200 import synth_h264
    return synth_h264.write(W, H, frames, gop=gop, seed=seed, mv=(2, -2))


def make_clip_bytes_ref(seed, frames, gop=30):
    """The same stream (byte for byte, tests/test_storage_cpu.py) from the pure-numpy writer: the CPU
    reference arm must not load product libraries."""
    from oracle import h264_writer
    return h264_writer.h264_synth_skip(clip_yuv(seed, frames, gop), W, H, gop=gop, frames=frames)


def _ref_worker(path):
    """One reference pipeline instance: decode a clip and run Histogram + Resize on every frame
    (reference software_video_decoder.cpp:98-219 + tests/test_ops.cpp:13-59,114-170)."""
    import cv2
    cv2.setNumThreads(1)
    cap = cv2.VideoCapture(path)
    n = 0
    while True:
        ok, frame = cap.read()
        if not ok:
            break
        for c in range(3):
            cv2.calcHist([frame], [c], None, [16], [0, 256])
        cv2.resize(frame, (DW, DH))
        n += 1
    return n


def cpu_reference_fps(clip_bytes, n_clips, steps, warmup):
    """frames/s of the CPU path on all host cores; clips are written to /dev/shm once."""
    import multiprocessing as mp
    cores = usable_cores()
    tmpdir = tempfile.mkdtemp(prefix="scn_ref_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    paths = []
    for i in range(n_clips):
        p = os.path.join(tmpdir, f"clip{i}.h264")
        with open(p, "wb") as f:
            f.write(clip_bytes[i % len(clip_bytes)])
        paths.append(p)
    ctx = mp.get_context("fork")
    try:
        with ctx.Pool(min(cores, n_clips)) as pool:
            for _ in range(warmup):
                pool.map(_ref_worker, paths[:min(cores, n_clips)])
            t0 = time.perf_counter()
            frames = 0
            for _ in range(steps):
                frames += sum(pool.map(_ref_worker, paths))
            dt = time.perf_counter() - t0
    finally:
        shutil.rmtree(tmpdir, ignore_errors=True)
    return frames / dt, dt / steps, cores, frames // steps


def cv2_note():
    try:
        import cv2
        v = cv2.__version__
    except Exception:
        v = "unavailable"
    return f"opencv-python-headless {v} with its bundled FFmpeg (the reference pins OpenCV 4.2.0 / FFmpeg n4.2, deps.sh:643,725)"


def run_reference(args, rank, world):
    """CPU arm (rank 0 only): FFmpeg decode + OpenCV Histogram/Resize, one clip per core.  Loads no
    product library: the clips come from oracle/h264_writer.py."""
    if rank != 0:
        return 0
    cores = usable_cores()
    frames_per_clip = 60
    n_clips = max(2 * cores, 8)
    realistic = [make_clip_cavlc(500 + i, frames_per_clip)[0] for i in range(min(n_clips, 4))]
    fps, s_per_step, cores, sample = cpu_reference_fps(realistic, n_clips, args.steps, max(1, min(args.warmup, 1)))
    clips = [make_clip_bytes_ref(500 + i, frames_per_clip) for i in range(min(n_clips, 4))]
    fps_ipcm = cpu_reference_fps(clips, n_clips, max(1, min(args.steps, 3)), 1)[0]
    desc = (f"{n_clips} clips x {frames_per_clip} frames per step ({sample} frames, Intra16x16/CAVLC + motion-compensated "
            f"stream), cv2.VideoCapture (FFmpeg) decode + "
            f"cv2.calcHist x3 + cv2.resize(224), one process per core; {cv2_note()}")
    line = {"impl": "reference", "metric": METRIC, "value": fps, "unit": "frames/s", "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": s_per_step * 1e3,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
            "config": workload_config(args, sample),
            "cpu_baseline": {"value": fps, "unit": "frames/s", "cores": cores, "kind": "port", "sample": desc,
                             "ipcm_stream": {"value": fps_ipcm, "unit": "frames/s"}},
            "e2e": {"value": fps, "unit": "frames/s", "stream": "cavlc", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "e2e_ipcm_stream": {"value": fps_ipcm, "unit": "frames/s", "stream": "pcm"}}
    emit(line)
    return 0


def workload_config(args, batch):
    return {"workload": "configs[1]: 1080p H.264 decode + Resize(224x224) + Histogram",
            "frame": [H, W], "pitch": PITCH, "resize": [DH, DW], "frames_per_step": batch,
            "value_leg": "decoded NV12 surfaces resident in HBM -> streaming Histogram kernel + Resize kernel "
                         "(two rotating input batches, each > the 50 MB L2)",
            "e2e_leg": "clips are tables of one database directory shared by all ranks (H.264: Intra16x16 + CAVLC key picture "
                       "every 30, motion-compensated P pictures, ~6 KB/frame; e2e_ipcm_stream: I_PCM IDR + P_Skip, ~105 KB/frame) "
                       "-> NVDEC -> GPU ops -> save stage into output tables, through scn_engine_run",
            "goldens": "OpenCV 4.13.0 (the reference pins 4.2.0); NV12->RGB pinned to the reference's own image.cu"}


# ------------------------------------------------------------------------------------------
_REAL_STDOUT = None


def protect_stdout():
    """The contract is ONE JSON line on stdout.  NCCL (and anything else native) prints banners such
    as "NCCL version ..." straight to fd 1, so fd 1 is pointed at stderr for the whole run and the
    result line is written to the saved descriptor."""
    global _REAL_STDOUT
    if _REAL_STDOUT is None:
        sys.stdout.flush()
        _REAL_STDOUT = os.fdopen(os.dup(1), "w")
        os.dup2(2, 1)


def emit(line):
    out = _REAL_STDOUT or sys.stdout
    out.write(json.dumps(line) + "\n")
    out.flush()


class Ranks:
    """torch.distributed plumbing: barrier, max over ranks, object broadcast / gather."""

    def __init__(self, rank, local_rank, world):
        import torch
        self.torch, self.rank, self.local_rank, self.world = torch, rank, local_rank, world
        self.dev = torch.device("cuda", local_rank)
        self.dist = None
        if world > 1:
            import torch.distributed as dist
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            dist.init_process_group("nccl", device_id=self.dev)
            self.dist = dist

    def barrier(self):
        if self.dist is not None:
            self.dist.barrier()
        self.torch.cuda.synchronize()

    def max(self, values):
        if self.dist is None:
            return list(values)
        t = self.torch.tensor(list(values), device=self.dev, dtype=self.torch.float64)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return t.tolist()

    def bcast(self, obj):
        if self.dist is None:
            return obj
        box = [obj]
        self.dist.broadcast_object_list(box, src=0)
        return box[0]

    def gather(self, obj):
        if self.dist is None:
            return [obj]
        parts = [None] * self.world
        self.dist.all_gather_object(parts, obj)
        return parts

    def close(self):
        if self.dist is not None:
            self.dist.destroy_process_group()


def default_instances(args, local_rank, world):
    from scanner_b200 import engine as E
    if args.instances > 0:
        return args.instances
    # one decode session per NVDEC engine (7 on an H100), but never more threads than the rank's share of the host
    # cores can keep fed
    engines = E.nvdec_caps(local_rank).get("engines", 7) or 7
    return max(2, min(engines, 2 * usable_cores() // world))


def session_rates(counters):
    n = counters.get("instances", 0)
    return [round(counters[f"inst{i}_frames_decoded"] * 1e6 / max(1, counters[f"inst{i}_decode_busy_us"]))
            for i in range(n) if f"inst{i}_frames_decoded" in counters]


# ------------------------------------------------------------------------------------------
def e2e_config1(args, R, sampler, stream_kind="pcm", steps=None):
    """configs[1] end to end: one database of ingested clips shared by all ranks, the table list sharded
    over the ranks (scanner_b200/shard.py), sinks saved into output tables inside the timed region."""
    import numpy as np
    import oracle
    from scanner_b200 import engine as E
    from scanner_b200 import protolite, shard
    rank, world, local_rank = R.rank, R.world, R.local_rank
    E.load_stdlib()
    std = protolite.parse_proto(open(os.path.join(ROOT, "scanner_b200", "csrc", "ops", "stdlib_args.proto")).read())
    clips_per_rank, frames = args.e2e_clips, args.e2e_frames
    steps = steps or args.steps
    total = clips_per_rank * world
    if getattr(args, "e2e_total_clips", 0):       # strong scaling: ONE table list of fixed size split over the ranks
        total = args.e2e_total_clips
        clips_per_rank = (total + world - 1) // world
    root = R.bcast(tempfile.mkdtemp(prefix="scn_bench_db_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
                   if rank == 0 else None)
    db = E.Database(root)
    # ingest: every rank ingests the tables it will NOT necessarily process (strided), all into the one catalogue
    n_unique = 4
    uniq_seed = lambda i: 2000 + (i % (n_unique * world))
    cache = {}
    t_ing = time.perf_counter()
    for i in range(rank, total, world):
        s = uniq_seed(i)
        if s not in cache:
            cache[s] = make_clip_bytes(s, frames) if stream_kind == "pcm" else make_clip_cavlc(s, frames)[0]
        db.ingest_h264(f"clip_{i:05d}", cache[s])
    ingest_s = time.perf_counter() - t_ing
    R.barrier()
    mine = shard.shard_indices(total, rank, world)            # ONE table list, split over the ranks
    instances = default_instances(args, local_rank, world)
    eng = E.Engine(gpus=[local_rank], instances_per_gpu=instances)
    graph = E.Graph()
    src = graph.add_source(True)
    op_h = graph.add_op("Histogram", [(src, "frame")], device=1)
    op_r = graph.add_op("Resize", [(src, "frame")], device=1)
    sink_h = graph.add_sink((op_h, "histogram"))
    sink_r = graph.add_sink((op_r, "frame"))
    # N > 1: the ranks PULL tasks of the one job list from a queue they share (scn_engine_share_task_queue; the
    # reference's workers pull from the master), so a rank whose NVDEC sessions are in a slow spell takes fewer
    # tasks instead of holding the step up.  --static-shards gives every rank a fixed share of the tables instead.
    dynamic = world > 1 and not getattr(args, "static_shards", False)
    listed = list(range(total)) if dynamic else mine
    sids = {i: db.add_video_stream(eng, f"clip_{i:05d}") for i in listed}
    h2d = sum(db.table_info(f"clip_{i:05d}").get("bytes", 0) or 0 for i in listed) // (world if dynamic else 1)
    resize_args = protolite.encode(std["ResizeArgs"], {"width": DW, "height": DH})
    if dynamic:
        eng.share_task_queue(os.path.join(root, "task_queue"))
    phases = []   # per step: seconds for {reserve tables, scn_engine_run, commit}

    def one_step(tag):
        # the output tables of the step's jobs are reserved and committed with ONE catalogue lock each
        # (scn_db_new_tables / scn_db_commit_job_tables): ranks sharing the directory do not queue per table
        specs = ([(f"hist_{tag}_{i:05d}", "histogram", False, "Histogram", i) for i in listed] +
                 [(f"small_{tag}_{i:05d}", "frame", True, "", i) for i in listed])
        t_a = time.perf_counter()
        if dynamic:
            # rank 0 reserves (and later commits) the tables of the whole list under ONE catalogue lock each and
            # broadcasts the ids; the items of a table are written by whichever ranks pull its tasks.  (Every rank
            # reserving its own share was tried: eight ranks queue on the catalogue lock twice per step, ~3 ms each.)
            ids = R.bcast(db.new_tables(specs) if rank == 0 else None)
        else:
            ids = db.new_tables(specs)
        jobs = []
        for k, i in enumerate(listed):
            j = E.Job()
            j.bind_source(src, sids[i])
            j.set_stream_args(op_r, resize_args)
            j.set_sink_table(sink_h, ids[k], keep_rows=False)
            j.set_sink_table(sink_r, ids[len(listed) + k], keep_rows=False)
            jobs.append(j)
        if dynamic:
            if rank == 0:
                eng.reset_task_queue()
            R.barrier()
        t_b = time.perf_counter()
        eng.run(graph, jobs, 30, 60, out_dir=root)
        t_c = time.perf_counter()
        if dynamic:
            R.barrier()          # every rank's items are on disk
        if not dynamic or rank == 0:
            db.commit_job_tables([(ids[k], jobs[k % len(listed)]) for k in range(2 * len(listed))])
        phases.append([t_b - t_a, t_c - t_b, time.perf_counter() - t_c])
        return jobs

    def drop(tag):
        if not dynamic or rank == 0:
            db.delete_tables([f"hist_{tag}_{i:05d}" for i in listed] + [f"small_{tag}_{i:05d}" for i in listed])

    for k in range(2):
        one_step(f"w{k}")  # warm-up: decoder creation, memory pools
        drop(f"w{k}")
    step_s, rates, video, done_frames = [], [], [], []
    for k in range(steps):
        R.barrier()
        sampler.reset()
        t0 = time.perf_counter()
        one_step(f"s{k}")
        R.torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        sampler.sample_now()
        step_s.append(dt)
        rates.append(session_rates(eng.stats()["counters"]))
        done_frames.append(int(eng.stats()["counters"].get("frames_used", 0)))
        video.append(sampler.video_result())
        if k + 1 < steps:
            drop(f"s{k}")  # untimed: the next step writes fresh tables
    stats = eng.stats()["counters"]
    # parity on what the save stage stored (last step): rows of one of this rank's clips against the oracle
    last = f"s{steps - 1}"
    R.barrier()               # (dynamic: rank 0 has committed the last step's tables)
    i0 = mine[0]
    yuv = clip_yuv(uniq_seed(i0), frames) if stream_kind == "pcm" else make_clip_cavlc(uniq_seed(i0), frames)[1]
    check_rows = sorted({0, 1, min(frames - 1, 31), frames - 1})
    got_h = db.read_rows(f"hist_{last}_{i0:05d}", "histogram", check_rows)
    got_r = db.read_rows(f"small_{last}_{i0:05d}", "frame", check_rows)
    for row, gh, gr in zip(check_rows, got_h, got_r):
        src_pic = yuv[row // 30] if stream_kind == "pcm" else yuv[row]
        y = src_pic[:H * W].reshape(H, W)
        chroma = np.empty((H // 2, W), np.uint8)
        chroma[:, 0::2] = src_pic[H * W:H * W * 5 // 4].reshape(H // 2, W // 2)
        chroma[:, 1::2] = src_pic[H * W * 5 // 4:].reshape(H // 2, W // 2)
        want = oracle.nv12_to_rgb(y, chroma)
        assert (np.frombuffer(gh, np.int32).reshape(3, 16) == oracle.hist16(want)).all(), f"stored histogram row {row}"
        assert (gr == oracle.resize(want, DW, DH)).all(), f"stored resize row {row}"
    n_rows = db.table_info(f"hist_{last}_{i0:05d}")["rows"]
    assert n_rows == frames, (n_rows, frames)
    eng.close()
    R.barrier()
    per_rank = R.gather({"rank": rank, "step_s": step_s, "frames_per_step": sum(done_frames) / max(1, len(done_frames)),
                         "frames_done_per_step": done_frames, "session_pictures_per_s": rates,
                         "phase_ms": [[round(x * 1e3, 2) for x in ph] for ph in phases[-len(step_s):]],
                         "nvml": video, "numa_pinned_cpus": stats.get("numa_pinned_cpus")})
    step_max = R.max(step_s)
    if rank == 0:
        shutil.rmtree(root, ignore_errors=True)
    frames_per_step_all = total * frames
    return {"value": frames_per_step_all * steps / sum(step_max), "unit": "frames/s", "stream": stream_kind, "steps": steps,
            "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": len(mine) * frames * (192 + DH * DW * 3),
            "frames_per_step": frames_per_step_all, "clips": total, "frames_per_clip": frames,
            "pipeline_instances": instances, "frames_decoded_last_step": stats.get("frames_decoded"),
            "ingest_s": ingest_s,
            "timing": "per step: barrier, host wall clock around {new output tables, scn_engine_run with the save stage "
                      "writing every task into them, commit}, max over ranks; the steps summed",
            "stored_rows_checked_against_oracle": len(check_rows) * 2,
            "step_fps": [frames_per_step_all / s for s in step_max],
            "task_assignment": "ranks pull tasks from one shared queue (scn_engine_share_task_queue)" if dynamic
                               else "static: every rank owns a fixed share of the tables",
            "per_rank": [{"rank": p["rank"], "fps": sum(p["frames_done_per_step"]) / sum(p["step_s"]),
                          "frames_done_per_step": p["frames_done_per_step"],
                          "reserve_run_commit_ms_per_step": p["phase_ms"],
                          "step_fps_min_median_max": _mmm([f / s for f, s in zip(p["frames_done_per_step"], p["step_s"])]),
                          "session_pictures_per_s_last_step": p["session_pictures_per_s"][-1],
                          "session_rate_spread_worst_step": max((max(r) - min(r)) / max(1, max(r)) for r in p["session_pictures_per_s"] if r),
                          "nvml_last_step": p["nvml"][-1], "numa_pinned_cpus": p["numa_pinned_cpus"]} for p in per_rank],
            "decoder": ("FFmpeg on the host (the GPU exposes no NVDEC engine to this process)"
                        if stats.get("gpu_software_decode_sessions") else "NVDEC"),
            "bound": "decode: session_pictures_per_s is the decode rate of every pipeline instance"}


def dump_outputs(out_dir, hist, res):
    """The last step's outputs as float32 .npy: every histogram, and the Resize rows of a fixed seeded sample of at
    most 64 frames (all of them would be 4x the batch's uint8 bytes)."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    n = hist.shape[0]
    pick = np.sort(np.random.default_rng(0).choice(n, min(n, 64), replace=False))
    sample = res.index_select(0, torch.from_numpy(pick).to(res.device))
    np.save(os.path.join(out_dir, "hist.npy"), hist.cpu().numpy().astype(np.float32))
    np.save(os.path.join(out_dir, "resize_sample.npy"), sample.cpu().numpy().astype(np.float32))
    np.save(os.path.join(out_dir, "resize_sample_frames.npy"), pick.astype(np.float32))


def _mmm(v):
    v = sorted(v)
    return [v[0], v[len(v) // 2], v[-1]]


# ------------------------------------------------------------------------------------------
def run_config1(args, R):
    import torch
    from scanner_b200 import cabi, kernels
    rank, world, local_rank, dev = R.rank, R.world, R.local_rank, R.dev
    B = args.batch
    L = cabi.lib()

    # --- device-resident inputs: two batches of B surfaces, seeded per rank (different "clips")
    g = torch.Generator(device=dev).manual_seed(1000 + rank)
    batches = [torch.randint(0, 256, (B, SURF_ROWS, PITCH), dtype=torch.uint8, device=dev, generator=g)
               for _ in range(2)]
    plan = kernels.ResizePlan(W, H, DW, DH, dev)

    def step(i):
        return kernels.nv12_hist_resize(batches[i & 1], W, H, DW, DH, plan)

    for i in range(max(args.warmup, 3)):
        step(i)
    R.barrier()
    sampler = ClockSampler(local_rank)
    sampler.sample_now()
    sampler.reset()
    sampler.start()
    l0 = L.scn_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    R.barrier()
    e0.record()
    for i in range(args.steps):
        last = step(i)
    e1.record()
    sampler.sample_now()  # the steps are still executing: a sample under load even for short runs
    R.barrier()
    ms = e0.elapsed_time(e1)
    launches = L.scn_launch_count() - l0
    clocks = sampler.result()
    sampler.stop_flag = True
    sampler.join(timeout=2)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, *last)

    # --- roofline leg: the same kernels on the same batches with per-kernel events (scn_prof_*), not used for
    # `value`.  In the value leg the Resize kernel runs on a forked stream next to the Histogram kernel; here each
    # is launched on its own (Histogram-only call, then Resize-only call) so that a launch's duration is that
    # kernel's and nothing else's.
    L.scn_prof_enable(1)
    for i in range(args.steps):
        kernels.nv12_hist_resize(batches[i & 1], W, H, DW, DH, plan, want_resize=False)
        kernels.nv12_hist_resize(batches[i & 1], W, H, DW, DH, plan, want_hist=False)
    torch.cuda.synchronize()
    prof = cabi.prof_report()
    L.scn_prof_enable(0)
    del batches
    torch.cuda.empty_cache()

    # headline: a stream with a real encoder's structure and bitrate (CAVLC intra + motion-compensated pictures);
    # the lossless I_PCM / P_Skip stream r01 reported (105 KB per frame, nothing an encoder would produce) beside it
    e2e = e2e_config1(args, R, ClockSampler(local_rank), stream_kind="cavlc")
    e2e_ipcm = e2e_config1(args, R, ClockSampler(local_rank), stream_kind="pcm", steps=min(args.steps, 5))
    ms = R.max([ms])[0]

    if rank == 0:
        frames = B * args.steps * world
        value = frames / (ms * 1e-3)
        peak, peak_kind = peaks()
        kname = max(prof, key=lambda k: prof[k]["ms"]) if prof else None
        roof = None
        if kname:
            per_launch_s = prof[kname]["ms"] * 1e-3 / prof[kname]["launches"]
            per_launch = min(B, 64)  # SCN_MAX_PTRS surfaces per launch
            # the streaming kernel alone reads the surface and writes the histogram; when the Resize rows are produced
            # in the same pass (SCN_NV12_RESIZE=fused) there is no separate Resize kernel and its output counts too
            separate_resize = True  # (SCN_NV12_RESIZE=fused would produce the Resize rows inside the streaming pass)
            alg = (B_ALG_HIST_NV12 if separate_resize else B_ALG_FUSED) * per_launch
            ach = alg / per_launch_s / 1e9
            roof = {"kernel": kname, "achieved": ach, "peak": peak, "unit": "GB/s",
                    "frac": ach / peak, "peak_kind": peak_kind,
                    "alg_bytes_per_launch": alg, "ms_per_launch": per_launch_s * 1e3,
                    "launch_mode": "Histogram by the streaming kernel, Resize by nv12_resize_kernel on a forked stream next to it"
                                   if separate_resize else
                                   "one kernel per 64 surfaces does Histogram and Resize in one pass",
                    "kernel_share_of_step": prof[kname]["ms"] / sum(v["ms"] for v in prof.values()),
                    "note": "kernels timed one at a time; in the value leg they overlap (ms_per_step / launches < their sum)",
                    "all_kernels_ms": {k: v["ms"] / v["launches"] for k, v in prof.items()}}
        line = {"metric": METRIC, "value": value, "unit": "frames/s", "n_gpus": world, "steps": args.steps,
                "warmup": max(args.warmup, 3), "ms_per_step": ms / args.steps, "higher_is_better": True,
                "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
                "config": workload_config(args, B), "clocks": clocks, "e2e": e2e, "e2e_ipcm_stream": e2e_ipcm,
                "gpu_launches": int(launches), "roofline": roof,
                "whole_step_roofline_frac": value / world * B_ALG_FUSED / 1e9 / peak}
        if world == 1:
            line["cpu_baseline"] = cpu_baseline(args)
            line["config0_cpu"] = config0_cpu()
        emit(line)
    return 0


def cpu_baseline(args):
    """The reference's CPU path (FFmpeg decode + OpenCV ops) on a bounded sample, all host cores."""
    cores = usable_cores()
    n_clips = max(2 * cores, 8)
    realistic = [make_clip_cavlc(700 + i, 60)[0] for i in range(min(n_clips, 4))]
    fps, s_per_step, cores, sample = cpu_reference_fps(realistic, n_clips, 1, 1)
    clips = [make_clip_bytes_ref(700 + i, 60) for i in range(min(n_clips, 4))]
    fps2 = cpu_reference_fps(clips, n_clips, 1, 1)[0]
    return {"value": fps, "unit": "frames/s", "cores": cores, "kind": "port",
            "sample": f"{sample} frames ({n_clips} clips x 60, Intra16x16/CAVLC + motion-compensated stream), cv2.VideoCapture "
                      f"(FFmpeg) decode + cv2.calcHist x3 + cv2.resize(224), one process per core; {cv2_note()}",
            "ipcm_stream": {"value": fps2, "unit": "frames/s", "sample": "the same sample on the I_PCM / P_Skip stream"}}


# ------------------------------------------------------------------------------------------
def run_config3(args, R):
    """configs[3]: dense OpticalFlow (stencil {0,1}) over clips whose rows are split into N contiguous
    intervals, one per GPU; the boundary frame of every interval comes from the neighbouring GPU as a
    decoded NV12 element over NCCL (scn_engine_comm_init / scn_job_set_shard), inside scn_engine_run.
    Flow fields are 16.6 MB per 1080p frame, so the sink is a per-frame checksum of the field's bytes
    (FrameDigest op): the sharded run's digests must equal the single-GPU run's, bit for bit."""
    import numpy as np
    import torch
    from scanner_b200 import engine as E
    from scanner_b200 import halo
    rank, world, local_rank = R.rank, R.world, R.local_rank
    E.load_stdlib()
    n_clips, frames = args.flow_clips, args.flow_frames
    # realistic streams (CAVLC key pictures, motion-compensated P pictures): decode must not be what is measured
    clips = [make_clip_cavlc(300 + c, frames)[0] for c in range(min(n_clips, 2))]
    eng = E.Engine(gpus=[local_rank], instances_per_gpu=default_instances(args, local_rank, world))
    if world > 1:
        eng.init_comm(local_rank)
    graph = E.Graph()
    src = graph.add_source(True)
    op_f = graph.add_op("OpticalFlow", [(src, "frame")], device=1)
    op_d = graph.add_op("FrameDigest", [(op_f, "flow")], device=1)
    sink = graph.add_sink((op_d, "digest"))
    sids = [eng.add_h264(clips[c % len(clips)]) for c in range(n_clips)]
    bounds = [halo.interval_of(frames, r, world)[0] for r in range(world)] + [frames]

    def jobs_for(sharded):
        out = []
        for s in sids:
            j = E.Job()
            j.bind_source(src, s)
            if sharded:
                j.set_shard(rank, bounds, list(range(world)))
            out.append(j)
        return out

    jobs = jobs_for(world > 1)
    for _ in range(max(1, min(args.warmup, 2))):
        eng.run(graph, jobs, 8, 24)
    step_s = []
    for _ in range(args.steps):
        R.barrier()
        t0 = time.perf_counter()
        eng.run(graph, jobs, 8, 24)
        torch.cuda.synchronize()
        step_s.append(time.perf_counter() - t0)
    st = eng.stats()["counters"]
    a, b = bounds[rank], bounds[rank + 1]
    mine = [jobs[c].output_array(sink, 16, np.uint64, row0=a) for c in range(n_clips)]
    # the single-GPU answer for this rank's rows of the first clip (same engine, unsharded job restricted by a Range sampler
    # would change the stencil edges: run the whole first clip once on rank 0 only and compare every rank's rows)
    gathered = R.gather((a, b, [m.tolist() for m in mine[:1]]))
    identical = None
    if rank == 0:
        ref_job = E.Job()
        ref_job.bind_source(src, sids[0])
        eng.run(graph, [ref_job], 8, 24)
        full = ref_job.output_array(sink, 16, np.uint64)
        identical = all((np.array(rows[0], np.uint64).reshape(-1, 2) == full[lo:hi]).all() for lo, hi, rows in gathered)
        assert identical, "sharded OpticalFlow differs from the single-GPU run"
    eng.close()
    step_max = R.max(step_s)
    if rank == 0:
        total = n_clips * frames * args.steps
        fps = total / sum(step_max)
        line = {"metric": "frames/sec (1080p dense OpticalFlow, clips split into contiguous intervals over N GPUs)",
                "value": fps, "unit": "frames/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
                "ms_per_step": sum(step_max) / args.steps * 1e3, "higher_is_better": True, "scaling": "strong",
                "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                "config": {"workload": "configs[3]: 1080p dense OpticalFlow (Farneback, the in-tree op; TV-L1 has no reference), "
                                       "stencil {0,1}, every clip split into N contiguous intervals, halo over NCCL",
                           "clips": n_clips, "frames_per_clip": frames, "intervals": bounds},
                "e2e": {"value": fps, "unit": "frames/s", "h2d_bytes_per_step": sum(len(clips[c % len(clips)]) for c in range(n_clips)),
                        "d2h_bytes_per_step": n_clips * (b - a) * 16},
                "halo": {"bytes_sent_rank0": st.get("halo_bytes_sent"), "bytes_received_rank0": st.get("halo_bytes_received"),
                         "exchange_us_rank0": st.get("halo_exchange_us"), "element": "packed NV12 surface (3.1 MB per 1080p frame)",
                         "identical_to_single_gpu": identical,
                         "note": "exchange_us covers decoding the boundary rows, the NCCL group and the wait for the slowest peer"},
                "step_fps": [n_clips * frames / s_ for s_ in step_max]}
        emit(line)
    return 0


def _i420_to_rgb(yuv, w, h):
    """Expected picture of the synthetic writers (planar I420) -> RGB24 through the oracle's NV12 -> RGB."""
    import numpy as np
    import oracle
    luma = yuv[:w * h].reshape(h, w)
    chroma = np.empty((h // 2, w), np.uint8)
    chroma[:, 0::2] = yuv[w * h:w * h * 5 // 4].reshape(h // 2, w // 2)
    chroma[:, 1::2] = yuv[w * h * 5 // 4:].reshape(h // 2, w // 2)
    return oracle.nv12_to_rgb(np.ascontiguousarray(luma), chroma, w)


def run_config2(args, R):
    """configs[2]: 4K H.264 decode + Blur + Histogram (shot-boundary features), every clip split into N contiguous
    intervals, one per GPU (no stencil: no halo).  As stated: 64 clips x 600 frames on 8 GPUs; default here 16 x 120.
    Strong scaling: the clip list is fixed, N GPUs split every clip's rows."""
    import numpy as np
    import torch
    import oracle
    from scanner_b200 import engine as E, halo, protolite, synth_h264
    rank, world, local_rank = R.rank, R.world, R.local_rank
    E.load_stdlib()
    std = protolite.parse_proto(open(os.path.join(ROOT, "scanner_b200", "csrc", "ops", "stdlib_args.proto")).read())
    W4, H4 = 3840, 2160
    n_clips, frames = args.clips or 16, args.frames or 120
    unit = 120 if frames % 120 == 0 else frames          # a 600-frame clip is the 120-frame stream five times over
    made = synth_h264.write(W4, H4, unit, gop=30, seed=41, mv=(2, -2)) if rank == 0 else None   # ~0.2 s per 4K picture
    made = R.bcast(made)
    clip, expect = made[0] * (frames // unit), made[1]
    eng = E.Engine(gpus=[local_rank], instances_per_gpu=default_instances(args, local_rank, world))
    if world > 1:
        eng.init_comm(local_rank)
    graph = E.Graph()
    src = graph.add_source(True)
    op_b = graph.add_op("Blur", [(src, "frame")], device=1,
                        args=protolite.encode(std["BlurArgs"], {"kernel_size": 3, "sigma": 0.5}))
    op_h = graph.add_op("Histogram", [(op_b, "frame")], device=1)
    sink = graph.add_sink((op_h, "histogram"))
    sids = [eng.add_h264(clip) for _ in range(n_clips)]
    # interval bounds on key pictures (GOP 30) when the clip has at least one GOP per rank: an interval that starts
    # inside a GOP would decode that GOP's head only to throw it away
    gops = frames // 30
    bounds = ([gops * r // world * 30 for r in range(world)] + [frames] if gops >= world and frames % 30 == 0 else
              [halo.interval_of(frames, r, world)[0] for r in range(world)] + [frames])
    jobs = []
    for sid in sids:
        j = E.Job()
        j.bind_source(src, sid)
        if world > 1:
            j.set_shard(rank, bounds, list(range(world)))
        jobs.append(j)
    for _ in range(max(1, min(args.warmup, 2))):
        eng.run(graph, jobs, 10, 30)    # tasks of one GOP: no task starts inside a GOP
    step_s = []
    for _ in range(args.steps):
        R.barrier()
        t0 = time.perf_counter()
        eng.run(graph, jobs, 10, 30)    # tasks of one GOP: no task starts inside a GOP
        torch.cuda.synchronize()
        step_s.append(time.perf_counter() - t0)
    st = eng.stats()["counters"]
    a, b = bounds[rank], bounds[rank + 1]
    hist = jobs[-1].output_array(sink, 192, np.int32, row0=a).reshape(b - a, 3, 16)
    checked = 0
    for row in sorted({a, a + 1, (a + b) // 2, b - 1}):   # this rank's rows of the last clip against the oracle
        want = oracle.hist16(oracle.blur(_i420_to_rgb(expect[row % unit], W4, H4), 3))
        assert (hist[row - a] == want).all(), f"configs[2] row {row} differs from the oracle"
        checked += 1
    eng.close()
    step_max = R.max(step_s)
    decoded = R.gather(int(st.get("frames_decoded", 0)))
    if rank == 0:
        fps = n_clips * frames * args.steps / sum(step_max)
        emit({"metric": "frames/sec (4K H.264 decode + Blur + Histogram, clips split into contiguous intervals over N GPUs)",
              "value": fps, "unit": "frames/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
              "ms_per_step": sum(step_max) / args.steps * 1e3, "higher_is_better": True, "scaling": "strong",
              "vs_baseline": None, "dtype": "u8", "data": "synthetic",
              "config": {"workload": "configs[2]: 4K H.264 decode + Blur(3) + Histogram, interval-sharded", "clips": n_clips,
                         "frames_per_clip": frames, "intervals": bounds, "frame": [H4, W4],
                         "stream": "Intra16x16/CAVLC key pictures + motion-compensated P pictures, GOP 30"},
              "e2e": {"value": fps, "unit": "frames/s", "h2d_bytes_per_step": n_clips * len(clip) // world,
                      "d2h_bytes_per_step": n_clips * (b - a) * 192},
              "frames_decoded_per_rank_last_run": decoded, "rows_checked_against_oracle_per_rank": checked,
              "step_fps": [n_clips * frames / s_ for s_ in step_max]})
    return 0


def run_config4(args, R):
    """configs[4]: Strided sampling (1 frame of every 30) + Histogram across many clips, decode-bound: with GOP 30 every
    wanted row is a key picture and the decode stage feeds NVDEC only those samples (slice_into_intervals).  The clips
    are tables of ONE database split over the ranks (shard.shard_indices); as stated 10,000 clips on 8 GPUs, default
    here 1,000 x 300 frames.  `value` counts SOURCE frames covered per second (clips x frames / time), `sampled_rows_per_s`
    the histogram rows produced."""
    import numpy as np
    import oracle
    from scanner_b200 import engine as E, protolite, shard
    rank, world, local_rank = R.rank, R.world, R.local_rank
    E.load_stdlib()
    total, frames, stride = args.clips or 1000, args.frames or 300, 30
    root = R.bcast(tempfile.mkdtemp(prefix="scn_bench_c4_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
                   if rank == 0 else None)
    db = E.Database(root)
    uniq = {}
    t_ing = time.perf_counter()
    for i in range(rank, total, world):                  # every rank ingests a strided share into the one catalogue
        s = 2500 + i % 4
        if s not in uniq:
            uniq[s] = make_clip_cavlc(s, frames)
        db.ingest_h264(f"clip_{i:05d}", uniq[s][0])
    ingest_s = time.perf_counter() - t_ing
    R.barrier()
    mine = shard.shard_indices(total, rank, world)
    eng = E.Engine(gpus=[local_rank], instances_per_gpu=default_instances(args, local_rank, world))
    graph = E.Graph()
    src = graph.add_source(True)
    samp = graph.add_sample((src, "frame"))
    op_h = graph.add_op("Histogram", [(samp, "frame")], device=1)
    sink = graph.add_sink((op_h, "histogram"))
    strided = protolite.encode(protolite.SAMPLER_ARGS["StridedSamplerArgs"], {"stride": stride})
    jobs = []
    for i in mine:
        j = E.Job()
        j.bind_source(src, db.add_video_stream(eng, f"clip_{i:05d}"))
        j.set_sampler(samp, "Strided", strided)
        jobs.append(j)
    rows_per_clip = (frames + stride - 1) // stride
    for _ in range(max(1, min(args.warmup, 2))):
        eng.run(graph, jobs, 10, 10)
    step_s = []
    for _ in range(args.steps):
        R.barrier()
        t0 = time.perf_counter()
        eng.run(graph, jobs, 10, 10)
        R.torch.cuda.synchronize()
        step_s.append(time.perf_counter() - t0)
    st = eng.stats()["counters"]
    i0 = mine[0]
    hist = jobs[0].output_array(sink, 192, np.int32).reshape(rows_per_clip, 3, 16)
    exp = make_clip_cavlc(2500 + i0 % 4, frames)[1] if (2500 + i0 % 4) not in uniq else uniq[2500 + i0 % 4][1]
    for k in (0, rows_per_clip // 2, rows_per_clip - 1):
        assert (hist[k] == oracle.hist16(_i420_to_rgb(exp[k * stride], W, H))).all(), f"configs[4] row {k} differs"
    eng.close()
    db.close()
    step_max = R.max(step_s)
    decoded = R.gather((int(st.get("frames_decoded", 0)), int(st.get("frames_used", 0))))
    R.barrier()
    if rank == 0:
        shutil.rmtree(root, ignore_errors=True)
        t = sum(step_max)
        emit({"metric": "frames/sec (1080p H.264, 1 frame of every 30 sampled + Histogram; source frames covered per second)",
              "value": total * frames * args.steps / t, "unit": "frames/s", "n_gpus": world, "steps": args.steps,
              "warmup": args.warmup, "ms_per_step": t / args.steps * 1e3, "higher_is_better": True, "scaling": "strong",
              "vs_baseline": None, "dtype": "u8", "data": "synthetic",
              "config": {"workload": "configs[4]: Strided(30) sampling + Histogram over a table list, decode-bound",
                         "clips": total, "frames_per_clip": frames, "stride": stride, "gop": 30,
                         "stream": "Intra16x16/CAVLC key pictures + motion-compensated P pictures"},
              "sampled_rows_per_s": total * rows_per_clip * args.steps / t,
              "e2e": {"value": total * frames * args.steps / t, "unit": "frames/s", "h2d_bytes_per_step": 0,
                      "d2h_bytes_per_step": total * rows_per_clip * 192 // world},
              "frames_decoded_used_per_rank_last_run": decoded, "ingest_s_rank0": ingest_s,
              "step_fps": [total * frames / s_ for s_ in step_max]})
    return 0


def main():
    protect_stdout()
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", type=int, default=1, choices=[1, 2, 3, 4])
    ap.add_argument("--batch", type=int, default=256,
                    help="surfaces per step (kernels take 64 per launch: a step of 256 is 4 launches)")
    ap.add_argument("--clips", type=int, default=0, help="--config 2 / 4: total clips (0 = that config's default)")
    ap.add_argument("--frames", type=int, default=0, help="--config 2 / 4: frames per clip (0 = that config's default)")
    ap.add_argument("--static-shards", action="store_true",
                    help="e2e leg at N > 1: give every rank a fixed share of the tables instead of the shared task queue")
    ap.add_argument("--e2e-total-clips", type=int, default=0,
                    help="e2e leg: total clips over ALL ranks (strong scaling; configs[1] as stated: 1000); overrides --e2e-clips")
    ap.add_argument("--e2e-clips", type=int, default=56, help="clips (tables) per rank in the e2e leg; configs[1] as stated: 1000")
    ap.add_argument("--e2e-frames", type=int, default=120, help="frames per clip in the e2e leg; configs[1] as stated: 300")
    ap.add_argument("--flow-clips", type=int, default=8, help="--config 3: clips; configs[3] as stated: 16")
    ap.add_argument("--flow-frames", type=int, default=96, help="--config 3: frames per clip; configs[3] as stated: 1200")
    ap.add_argument("--dump-outputs", default="", metavar="DIR",
                    help="--config 1: write the value leg's last-step outputs to DIR/<name>.npy (float32)")
    ap.add_argument("--instances", type=int, default=0,
                    help="pipeline instances per GPU for the e2e leg (0 = one per NVDEC engine, capped by the host cores)")
    args = ap.parse_args()
    if args.dump_outputs and (args.config != 1 or args.impl != "ours"):
        ap.error("--dump-outputs is implemented for --config 1 of this implementation")
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.impl == "reference":
        return run_reference(args, rank, world)

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (there is no CPU fallback)")
    torch.cuda.set_device(local_rank)
    R = Ranks(rank, local_rank, world)
    try:
        return {1: run_config1, 2: run_config2, 3: run_config3, 4: run_config4}[args.config](args, R)
    finally:
        R.close()


if __name__ == "__main__":
    sys.exit(main())
