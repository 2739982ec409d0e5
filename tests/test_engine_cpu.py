"""The C++ host pipeline (libscn_engine.so) driven through its C ABI on the CPU: row algebra,
stencils, batching, state ops, samplers, liveness, args, column files.  Kernels come from the
test plugin tests/cpp/test_plugin_ops.cpp, built against the public plugin headers.

Pins taken from the reference's own tests: bounded-state warmup values [0,3,3,4,5]
(tests/py_test.py:407-423), stencil row counts (py_test.py:459-520), sampler row counts
(py_test.py:274-336)."""
import os
import struct
import subprocess

import numpy as np
import pytest

import oracle
from oracle import synth
from scanner_b200 import engine as E
from scanner_b200 import protolite

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TEST_ARGS = protolite.parse_proto(open(os.path.join(ROOT, "tests", "cpp", "test_args.proto")).read())


@pytest.fixture(scope="module", autouse=True)
def plugin():
    oracle.build()
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "cpp")], stdout=subprocess.DEVNULL)
    so = os.path.join(ROOT, "build", "tests", "libtest_plugin_ops.so")
    if "TestWindow" not in E.list_ops():
        E.load_op_library(so)
    return so


@pytest.fixture()
def eng():
    e = E.Engine(gpus=[], cpu_instances=3)
    yield e
    e.close()


def i64_rows(n, start=0):
    return [struct.pack("<q", start + i) for i in range(n)]


def unpack_rows(job, sink, fmt="<q"):
    return [struct.unpack(fmt, job.output_row(sink, i)) for i in range(job.output_rows(sink))]


def run_simple(eng, n, build, wps=5, ios=10, samplers=None, stream_args=None, out_dir=None):
    sid = eng.add_bytes(i64_rows(n))
    g = E.Graph()
    src = g.add_source(False)
    sinks, bind = build(g, src)
    j = E.Job()
    j.bind_source(src, sid)
    for op, (fn, args) in (samplers or {}).items():
        j.set_sampler(bind[op], fn, args)
    for op, args in (stream_args or {}).items():
        j.set_stream_args(bind[op], args)
    eng.run(g, [j], wps, ios, out_dir)
    return j, sinks


# ------------------------------------------------------------------------------------------------
def test_stencil_window_repeat_edge_across_tasks_and_packets(eng):
    def build(g, src):
        w = g.add_op("TestWindow", [(src, "column")])
        return g.add_sink((w, "window")), {}
    for (wps, ios) in [(5, 10), (1, 1), (23, 23), (3, 9), (10, 100)]:
        j, sink = run_simple(eng, 23, build, wps, ios)
        got = unpack_rows(j, sink, "<3q")
        assert got == [(max(i - 1, 0), i, min(i + 1, 22)) for i in range(23)], (wps, ios)


def test_custom_stencil_overrides_op_default(eng):
    def build(g, src):
        w = g.add_op("TestWindow", [(src, "column")], stencil=[0, 2])
        return g.add_sink((w, "window")), {}
    j, sink = run_simple(eng, 12, build, 4, 4)
    assert unpack_rows(j, sink, "<2q") == [(i, min(i + 2, 11)) for i in range(12)]


def test_stencil_requires_op_support(eng):
    g = E.Graph()
    src = g.add_source(False)
    b = g.add_op("TestBatch", [(src, "column")], stencil=[0, 1])
    g.add_sink((b, "pair"))
    j = E.Job()
    j.bind_source(src, eng.add_bytes(i64_rows(4)))
    with pytest.raises(E.EngineError, match="stencil"):
        eng.run(g, [j], 2, 2)


def test_batching_full_batches_then_short_tail(eng):
    # kernel batch 4; a task of 10 rows -> batches 4,4 then the task tail as one short batch of 2
    # (reference evaluate_worker.cpp:899-908 + :1058-1060)
    def build(g, src):
        b = g.add_op("TestBatch", [(src, "column")])
        return g.add_sink((b, "pair")), {}
    j, sink = run_simple(eng, 10, build, wps=10, ios=10)
    got = unpack_rows(j, sink, "<2q")
    assert [g[0] for g in got] == list(range(10))
    assert [g[1] for g in got] == [4] * 8 + [2, 2]
    # explicit batch override
    def build2(g, src):
        b = g.add_op("TestBatch", [(src, "column")], batch=3)
        return g.add_sink((b, "pair")), {}
    j, sink = run_simple(eng, 7, build2, wps=7, ios=7)
    assert [g[1] for g in unpack_rows(j, sink, "<2q")] == [3, 3, 3, 3, 3, 3, 1]


def test_bounded_state_warmup_matches_reference_test(eng):
    """reference tests/py_test.py:407-423: Gather [0,10,25,26,27], warmup 3 -> [0,3,3,4,5]."""
    def build(g, src):
        inc = g.add_op("TestIncrementBounded", [(src, "column")], warmup=3)
        s = g.add_sample((inc, "integer"))
        return g.add_sink((s, "integer")), {"gather": s}
    args = protolite.encode(protolite.SAMPLER_ARGS["GatherSamplerArgs"], {"rows": [0, 10, 25, 26, 27]})
    for (wps, ios) in [(10, 100), (1, 5), (5, 5)]:  # one task, as PerfParams.estimate gives the reference
        j, sink = run_simple(eng, 40, build, wps, ios, samplers={"gather": ("Gather", args)})
        assert [v[0] for v in unpack_rows(j, sink)] == [0, 3, 3, 4, 5], (wps, ios)
    # one task per output row: every task warms up on its own 3 predecessors and drops them
    j, sink = run_simple(eng, 40, build, 1, 1, samplers={"gather": ("Gather", args)})
    assert [v[0] for v in unpack_rows(j, sink)] == [0, 3, 3, 3, 3]


def test_unbounded_state_recomputes_from_row_zero(eng):
    def build(g, src):
        inc = g.add_op("TestIncrementUnbounded", [(src, "column")])
        return g.add_sink((inc, "integer")), {}
    j, sink = run_simple(eng, 25, build, wps=5, ios=10)
    assert [v[0] for v in unpack_rows(j, sink)] == list(range(25))


@pytest.mark.parametrize("fn,msg,args,n,expect", [
    ("Strided", "StridedSamplerArgs", {"stride": 8}, 100, list(range(0, 100, 8))),
    ("Strided", "StridedSamplerArgs", {"stride": 1}, 7, list(range(7))),
    ("Gather", "GatherSamplerArgs", {"rows": [0, 1, 2, 3, 4, 5, 20, 50, 51]}, 60, [0, 1, 2, 3, 4, 5, 20, 50, 51]),
    ("StridedRanges", "StridedRangeSamplerArgs", {"stride": 1, "starts": [0], "ends": [30]}, 100, list(range(30))),
    ("StridedRanges", "StridedRangeSamplerArgs", {"stride": 10, "starts": [0, 50], "ends": [25, 80]}, 100,
     [0, 10, 20, 50, 60, 70]),
    ("All", None, {}, 9, list(range(9))),
])
def test_samplers(eng, fn, msg, args, n, expect):
    def build(g, src):
        s = g.add_sample((src, "column"))
        return g.add_sink((s, "column")), {"s": s}
    enc = protolite.encode(protolite.SAMPLER_ARGS[msg], args) if msg else b""
    j, sink = run_simple(eng, n, build, wps=4, ios=8, samplers={"s": (fn, enc)})
    assert [v[0] for v in unpack_rows(j, sink)] == expect


def test_space_null_and_repeat(eng):
    def build(g, src):
        s = g.add_space((src, "column"))
        return g.add_sink((s, "column")), {"s": s}
    for fn, msg in [("SpaceNull", "SpaceNullSamplerArgs"), ("SpaceRepeat", "SpaceRepeatSamplerArgs")]:
        enc = protolite.encode(protolite.SAMPLER_ARGS[msg], {"spacing": 3})
        j, sink = run_simple(eng, 5, build, wps=2, ios=6, samplers={"s": (fn, enc)})
        assert j.output_rows(sink) == 15
        rows = [j.output_row(sink, i) for i in range(15)]
        for i, r in enumerate(rows):
            if i % 3 == 0 or fn == "SpaceRepeat":
                assert struct.unpack("<q", r)[0] == i // 3
            else:
                assert r is None  # null element


def test_sampler_errors_surface(eng):
    j = E.Job()
    with pytest.raises(E.EngineError, match="stride"):
        j.set_sampler(1, "Strided", protolite.encode(protolite.SAMPLER_ARGS["StridedSamplerArgs"], {"stride": 0}))
    with pytest.raises(E.EngineError, match="not found"):
        j.set_sampler(1, "NoSuchSampler", b"")


def test_two_consumers_and_unused_output_column(eng):
    # one source feeds two ops; TestTwoOut's second column is never read (freed immediately)
    def build(g, src):
        two = g.add_op("TestTwoOut", [(src, "column")])
        win = g.add_op("TestWindow", [(src, "column")])
        return (g.add_sink((two, "twice")), g.add_sink((win, "window"))), {}
    j, (s1, s2) = run_simple(eng, 17, build, wps=4, ios=8)
    assert [v[0] for v in unpack_rows(j, s1)] == [2 * i for i in range(17)]
    assert unpack_rows(j, s2, "<3q") == [(max(i - 1, 0), i, min(i + 1, 16)) for i in range(17)]


def test_init_args_and_stream_args(eng):
    def build(g, src):
        a = g.add_op("TestAffine", [(src, "column")], args=protolite.encode(TEST_ARGS["TestScaleArgs"], {"scale": 3}))
        return g.add_sink((a, "out")), {"a": a}
    j, sink = run_simple(eng, 6, build, stream_args={"a": protolite.encode(TEST_ARGS["TestOffsetArgs"], {"offset": 7})})
    assert [v[0] for v in unpack_rows(j, sink)] == [3 * i + 7 for i in range(6)]
    # missing init args -> validate() failure is reported, not a crash (reference test_ops.cpp:244-247)
    def build_bad(g, src):
        a = g.add_op("TestAffine", [(src, "column")])
        return g.add_sink((a, "out")), {}
    with pytest.raises(E.EngineError, match="Could not parse"):
        run_simple(eng, 3, build_bad)


def test_many_jobs_share_the_task_queue(eng):
    g = E.Graph()
    src = g.add_source(False)
    w = g.add_op("TestWindow", [(src, "column")])
    sink = g.add_sink((w, "window"))
    jobs = []
    for k in range(7):
        j = E.Job()
        j.bind_source(src, eng.add_bytes(i64_rows(10 + k, start=100 * k)))
        jobs.append(j)
    eng.run(g, jobs, 3, 6)
    for k, j in enumerate(jobs):
        n = 10 + k
        base = 100 * k
        assert unpack_rows(j, sink, "<3q") == [(base + max(i - 1, 0), base + i, base + min(i + 1, n - 1))
                                               for i in range(n)]
    assert eng.stats()["counters"]["tasks"] == sum((10 + k + 5) // 6 for k in range(7))


def test_no_buffers_leak_across_runs(eng):
    """Every element the pipeline allocates is released by the end of the run (refcounted blocks,
    stencil caches, dropped warmup rows, unused output columns, sampled-away rows)."""
    def build(g, src):
        two = g.add_op("TestTwoOut", [(src, "column")])
        win = g.add_op("TestWindow", [(two, "twice")])
        inc = g.add_op("TestIncrementBounded", [(src, "column")], warmup=2)
        s = g.add_sample((inc, "integer"))
        s2 = g.add_sample((win, "window"))
        return (g.add_sink((s2, "window")), g.add_sink((s, "integer"))), {"s": s, "s2": s2}
    enc = protolite.encode(protolite.SAMPLER_ARGS["StridedSamplerArgs"], {"stride": 3})
    for _ in range(3):
        run_simple(eng, 30, build, wps=4, ios=12, samplers={"s": ("Strided", enc), "s2": ("Strided", enc)})
        c = eng.stats()["counters"]
        assert c["cpu_bytes_live"] == 0, c
        assert c["cpu_bytes_peak"] > 0


def test_errors(eng):
    with pytest.raises(E.EngineError, match="not registered"):
        E.Graph().add_op("NoSuchOp", [(0, "column")])
    g = E.Graph()
    src = g.add_source(False)
    b = g.add_op("TestBadCount", [(src, "column")])
    g.add_sink((b, "out"))
    j = E.Job()
    j.bind_source(src, eng.add_bytes(i64_rows(6)))
    with pytest.raises(E.EngineError, match="Expected 3 outputs"):
        eng.run(g, [j], 6, 6)
    with pytest.raises(E.EngineError, match="multiple of work packet"):
        eng.run(g, [j], 4, 6)
    # GPU kernel requested for an op that only has a CPU kernel
    g2 = E.Graph()
    s2 = g2.add_source(False)
    g2.add_sink((g2.add_op("TestWindow", [(s2, "column")], device=1), "window"))
    with pytest.raises(E.EngineError, match="no such kernel"):
        eng.run(g2, [j], 2, 2)
    # column that does not exist
    g3 = E.Graph()
    s3 = g3.add_source(False)
    g3.add_sink((g3.add_op("TestWindow", [(s3, "nope")]), "window"))
    with pytest.raises(E.EngineError, match="does not have the requested column"):
        eng.run(g3, [j], 2, 2)
    # the failed runs released what their kernels produced
    g4 = E.Graph()
    s4 = g4.add_source(False)
    g4.add_sink((s4, "column"))
    j4 = E.Job()
    j4.bind_source(s4, eng.add_bytes(i64_rows(2)))
    eng.run(g4, [j4], 2, 2)
    assert eng.stats()["counters"]["cpu_bytes_live"] == 0


# ------------------------------------------------------------------------------------------------
def test_config0_cpu_plumbing_histogram_640x480(eng, tmp_path):
    """BASELINE.json configs[0] analogue (no GPU): 640x480 frames -> Histogram on the CPU with one
    pipeline instance; every row equals the oracle bit-for-bit; column files use the reference's
    layout (column_sink.cpp:159-195)."""
    n = 30
    frames = np.stack([synth.smooth_frame(1 + i, 480, 640) for i in range(n)])
    e1 = E.Engine(gpus=[], cpu_instances=1)
    sid = e1.add_raw_frames(frames)
    assert e1.stream_info(sid)["width"] == 640 and e1.stream_rows(sid) == n
    g = E.Graph()
    src = g.add_source(True)
    h = g.add_op("TestHistogramOracle", [(src, "frame")])
    sink = g.add_sink((h, "histogram"))
    j = E.Job()
    j.bind_source(src, sid)
    e1.run(g, [j], 10, 20, str(tmp_path))
    hist = j.output_array(sink, 192, np.int32).reshape(n, 3, 16)
    for i in range(n):
        assert (hist[i] == oracle.hist16(frames[i])).all()
    # files: task 0 has 20 rows, task 1 has 10
    d = tmp_path / "tables" / "0"
    for task, rows in [(0, 20), (1, 10)]:
        meta = np.fromfile(d / f"1_{task}_metadata.bin", "<u8")
        assert meta[0] == rows and (meta[1:] == 192).all() and len(meta) == rows + 1
        data = np.fromfile(d / f"1_{task}.bin", "<i4").reshape(rows, 3, 16)
        assert (data == hist[task * 20: task * 20 + rows]).all()
        idx = np.fromfile(d / f"0_{task}.bin", "<i8")
        assert (idx == np.arange(task * 20, task * 20 + rows)).all()
        assert (idx.tobytes() == oracle.index_column(task * 20, rows).tobytes())
    e1.close()


def test_frame_ops_chain_resize_then_histogram_and_stride(eng):
    n = 12
    frames = np.stack([synth.rand_frame(50 + i, 60, 80) for i in range(n)])
    sid = eng.add_raw_frames(frames)
    g = E.Graph()
    src = g.add_source(True)
    samp = g.add_sample((src, "frame"))
    rz = g.add_op("TestResizeOracle", [(samp, "frame")])
    hs = g.add_op("TestHistogramOracle", [(rz, "frame")])
    s_frames = g.add_sink((rz, "frame"))
    s_hist = g.add_sink((hs, "histogram"))
    j = E.Job()
    j.bind_source(src, sid)
    j.set_sampler(samp, "Strided", protolite.encode(protolite.SAMPLER_ARGS["StridedSamplerArgs"], {"stride": 3}))
    j.set_stream_args(rz, protolite.encode(TEST_ARGS["TestSizeArgs"], {"width": 32, "height": 24}))
    eng.run(g, [j], 2, 4)
    assert j.output_rows(s_frames) == 4
    for k in range(4):
        want = oracle.resize(frames[3 * k], 32, 24)
        got = j.output_row(s_frames, k)
        assert got.shape == (24, 32, 3) and (got == want).all()
        assert (np.frombuffer(j.output_row(s_hist, k), np.int32).reshape(3, 16) == oracle.hist16(want)).all()


def test_frame_stencil_0_1_row_counts(eng):
    """reference py_test.py:459-520 checks only row counts for stencil [0,1]; here values too."""
    n = 9
    frames = np.stack([synth.rand_frame(70 + i, 16, 20) for i in range(n)])
    sid = eng.add_raw_frames(frames)
    g = E.Graph()
    src = g.add_source(True)
    d = g.add_op("TestFrameDiff", [(src, "frame")])
    sink = g.add_sink((d, "diff"))
    j = E.Job()
    j.bind_source(src, sid)
    for (wps, ios) in [(1, 1), (4, 8)]:
        eng.run(g, [j], wps, ios)
        assert j.output_rows(sink) == n
        got = [struct.unpack("<d", j.output_row(sink, i))[0] for i in range(n)]
        want = [float(np.abs(frames[i].astype(int) - frames[min(i + 1, n - 1)].astype(int)).sum()) for i in range(n)]
        assert got == want


def _cv2_rgb_frames(path):
    import cv2
    cap = cv2.VideoCapture(path)
    out = []
    while True:
        ok, f = cap.read()
        if not ok:
            return out
        out.append(f[..., ::-1].copy())


def test_config0_as_stated_h264_clip_histogram_on_a_cpu_instance(tmp_path):
    """BASELINE configs[0] as written: Histogram on one 640x480 H.264 clip, CPU pipeline_instances=1, no GPU.
    The CPU instance decodes with libavcodec + libswscale (swdec.h -- what the reference's SoftwareVideoDecoder
    is), so the frames must equal what FFmpeg gives through an independent caller (cv2.VideoCapture, BGR
    swapped); the op is the stdlib Histogram placed on the CPU.  The stream has Intra16x16/CAVLC key pictures
    and motion-compensated P pictures (scanner_b200/synth_h264.py)."""
    from scanner_b200 import synth_h264
    caps = E.swdec_caps()
    assert caps["available"], caps
    n = 24
    data, _ = synth_h264.write(640, 480, n, gop=8, seed=5)
    path = str(tmp_path / "clip.h264")
    open(path, "wb").write(data)
    want = _cv2_rgb_frames(path)
    assert len(want) == n
    E.load_stdlib()
    e1 = E.Engine(gpus=[], cpu_instances=1)
    sid = e1.add_h264(data)
    g = E.Graph()
    src = g.add_source(True)
    hs = g.add_op("Histogram", [(src, "frame")], device=0)
    s_h, s_f = g.add_sink((hs, "histogram")), g.add_sink((src, "frame"))
    j = E.Job()
    j.bind_source(src, sid)
    e1.run(g, [j], 5, 10, str(tmp_path))
    hist = j.output_array(s_h, 192, np.int32).reshape(n, 3, 16)
    for i in range(n):
        got = j.output_row(s_f, i)
        assert got.shape == (480, 640, 3) and (got == want[i]).all(), i
        assert (hist[i] == oracle.hist16(want[i])).all(), i
    st = e1.stats()["counters"]
    # tasks of 10 rows over GOPs of 8: tasks 1 and 2 start inside a GOP and decode from its key picture (2 + 4 extra)
    assert st["frames_used"] == n and st["frames_decoded"] == n + 6
    e1.close()


@pytest.mark.parametrize("mode,gop", [("pcm", 4), ("skip", 5), ("bidir", 6)])
def test_cpu_instance_decodes_sampled_rows_of_every_stream_kind(tmp_path, mode, gop):
    """Gather over keyframe intervals on the software path: only the intervals that hold wanted rows are fed, B
    pictures come out in display order (reference DecoderAutomata + SoftwareVideoDecoder semantics)."""
    n, h, w = 23, 48, 64
    rng = np.random.default_rng(21)
    k = n if mode == "pcm" else (n + gop - 1) // gop if mode == "skip" else n
    yuv = rng.integers(0, 256, (k, h * w * 3 // 2), dtype=np.uint8)
    data = E.h264_synth(yuv, w, h, gop=gop, non_key=mode, frames=n)
    path = str(tmp_path / "s.h264")
    open(path, "wb").write(data)
    want = _cv2_rgb_frames(path)
    assert len(want) == n
    e1 = E.Engine(gpus=[], cpu_instances=2)
    sid = e1.add_h264(data)
    g = E.Graph()
    src = g.add_source(True)
    samp = g.add_sample((src, "frame"))
    sink = g.add_sink((samp, "frame"))
    rows = [0, 3, 4, 11, 17, 22]
    j = E.Job()
    j.bind_source(src, sid)
    j.set_sampler(samp, "Gather", protolite.encode(protolite.SAMPLER_ARGS["GatherSamplerArgs"], {"rows": rows}))
    e1.run(g, [j], 2, 4)
    for i, r in enumerate(rows):
        assert (j.output_row(sink, i) == want[r]).all(), (mode, r)
    assert e1.stats()["counters"]["frames_decoded"] < n or mode == "bidir" or gop >= n
    e1.close()


def test_cpu_instance_says_why_when_no_ffmpeg_can_be_loaded(tmp_path):
    """No silent path: without libavcodec an H.264 source on a CPU instance is an error naming the cause."""
    code = (
        "import sys, numpy as np; sys.path.insert(0, '.');"
        "from scanner_b200 import engine as E;"
        "yuv = np.zeros((2, 48 * 64 * 3 // 2), np.uint8);"
        "e = E.Engine(gpus=[], cpu_instances=1); sid = e.add_h264(E.h264_synth(yuv, 64, 48, gop=2));"
        "g = E.Graph(); src = g.add_source(True); g.add_sink((src, 'frame'));"
        "j = E.Job(); j.bind_source(src, sid);"
        "\ntry:\n    e.run(g, [j], 2, 2)\n    print('RAN')\nexcept E.EngineError as x:\n    print('ERR', x)")
    empty = tmp_path / "nothing"
    empty.mkdir()
    out = subprocess.run([os.sys.executable, "-c", code], env=dict(os.environ, SCN_FFMPEG_DIR=str(empty)),
                         cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))), capture_output=True, text=True)
    assert "ERR" in out.stdout and "software H.264 decoder unavailable" in out.stdout, out.stdout + out.stderr


def test_shared_task_queue_refuses_interval_sharded_jobs(tmp_path):
    """One queue indexes one task list: scn_job_set_shard gives every rank its own, so the combination is an error."""
    e1 = E.Engine(gpus=[], cpu_instances=1)
    e1.share_task_queue(str(tmp_path / "queue"))
    g = E.Graph()
    src = g.add_source(True)
    g.add_sink((g.add_op("TestHistogramOracle", [(src, "frame")]), "histogram"))
    j = E.Job()
    j.bind_source(src, e1.add_raw_frames(np.zeros((8, 4, 4, 3), np.uint8)))
    j.set_shard(0, [0, 4, 8], [0, 1])
    with pytest.raises(E.EngineError, match="shared task queue"):
        e1.run(g, [j], 2, 4)
    e1.share_task_queue(None)                      # back to the private queue: the sharded job runs
    e1.close()


def test_trace_file_has_one_event_per_interval_and_instance_ids(eng, tmp_path):
    """scn_engine_write_trace: Chrome trace events of the last run (reference Profiler records +
    scannerpy Profile.write_trace)."""
    import json
    eng.set_trace(True)

    def build(g, src):
        w = g.add_op("TestWindow", [(src, "column")])
        return (g.add_sink((w, "window")),), {}
    run_simple(eng, 40, build, wps=5, ios=10)
    path = str(tmp_path / "run.trace")
    eng.write_trace(path)
    ev = json.load(open(path))["traceEvents"]
    st = eng.stats()
    names = {e["name"] for e in ev}
    assert {"task", "op:TestWindow", "evaluate:TestWindow"} <= names
    assert sum(1 for e in ev if e["name"] == "task") == st["counters"]["tasks"] == 4
    for k, n in st["interval_counts"].items():
        assert sum(1 for e in ev if e["name"] == k) == n
    assert all(e["ph"] == "X" and e["dur"] >= 0 and e["pid"] == -1 and 0 <= e["tid"] < 3 for e in ev)
    # an op interval lies inside a task interval of the same instance
    tasks = [(e["tid"], e["ts"], e["ts"] + e["dur"]) for e in ev if e["name"] == "task"]
    for e in ev:
        if e["name"] == "op:TestWindow":
            assert any(t == e["tid"] and a <= e["ts"] and e["ts"] + e["dur"] <= b + 1e-3 for t, a, b in tasks)
    eng.set_trace(False)
    run_simple(eng, 10, build, wps=5, ios=10)
    eng.write_trace(path)
    assert json.load(open(path))["traceEvents"] == []


def test_random_pipelines_match_a_python_model(eng):
    """Differential test of the row algebra: random chains of samplers, space ops, element-wise ops and a
    stencil op over an int64 column, random packet sizes, against a list-based Python model
    (REPEAT_EDGE windows over the op's own input domain, Gather/Stride/Range/Repeat semantics of
    reference sampler.cpp:78-454)."""
    rng = np.random.default_rng(1234)
    S = protolite.SAMPLER_ARGS

    def random_case():
        n = int(rng.integers(5, 60))
        stages, cur = [], n
        for _ in range(int(rng.integers(1, 5))):
            kind = rng.choice(["stride", "gather", "range", "repeat", "twice", "affine"])
            if cur < 2 and kind in ("stride", "gather", "range"):
                kind = "twice"
            if kind == "stride":
                s = int(rng.integers(1, 5))
                stages.append(("stride", s))
                cur = (cur + s - 1) // s
            elif kind == "gather":
                rows = sorted(set(int(x) for x in rng.integers(0, cur, int(rng.integers(1, cur + 1)))))
                stages.append(("gather", rows))
                cur = len(rows)
            elif kind == "range":
                a = int(rng.integers(0, cur))
                b = int(rng.integers(a + 1, cur + 1))
                stages.append(("range", a, b))
                cur = b - a
            elif kind == "repeat":
                k = int(rng.integers(2, 4))
                stages.append(("repeat", k))
                cur *= k
            elif kind == "twice":
                stages.append(("twice",))
            else:
                stages.append(("affine", int(rng.choice([-3, -2, -1, 1, 2, 3])), int(rng.integers(-50, 50))))
        if rng.random() < 0.6:
            stages.append(("window",))
            if rng.random() < 0.5 and cur >= 2:
                s = int(rng.integers(1, 4))
                stages.append(("stride", s))
        if rng.random() < 0.3:
            stages.append(("null", int(rng.integers(2, 4))))
        wps = int(rng.choice([1, 2, 3, 5]))
        return n, stages, wps, wps * int(rng.integers(1, 4))

    def model(n, stages):
        vals = list(range(n))
        for st in stages:
            if st[0] == "stride":
                vals = vals[::st[1]]
            elif st[0] == "gather":
                vals = [vals[i] for i in st[1]]
            elif st[0] == "range":
                vals = vals[st[1]:st[2]]
            elif st[0] == "repeat":
                vals = [v for v in vals for _ in range(st[1])]
            elif st[0] == "null":
                vals = [x for v in vals for x in [v] + [None] * (st[1] - 1)]
            elif st[0] == "twice":
                vals = [v * 2 for v in vals]
            elif st[0] == "affine":
                vals = [v * st[1] + st[2] for v in vals]
            elif st[0] == "window":
                m = len(vals)
                vals = [(vals[max(i - 1, 0)], vals[i], vals[min(i + 1, m - 1)]) for i in range(m)]
        return vals

    for case in range(200):
        n, stages, wps, ios = random_case()
        sid = eng.add_bytes(i64_rows(n))
        g = E.Graph()
        src = g.add_source(False)
        j = E.Job()
        j.bind_source(src, sid)
        cur = (src, "column")
        for st in stages:
            if st[0] in ("stride", "gather", "range"):
                op = g.add_sample(cur)
                if st[0] == "stride":
                    j.set_sampler(op, "Strided", protolite.encode(S["StridedSamplerArgs"], {"stride": st[1]}))
                elif st[0] == "gather":
                    j.set_sampler(op, "Gather", protolite.encode(S["GatherSamplerArgs"], {"rows": st[1]}))
                else:
                    j.set_sampler(op, "StridedRanges", protolite.encode(
                        S["StridedRangeSamplerArgs"], {"stride": 1, "starts": [st[1]], "ends": [st[2]]}))
                cur = (op, cur[1])
            elif st[0] in ("repeat", "null"):
                op = g.add_space(cur)
                name = "SpaceRepeat" if st[0] == "repeat" else "SpaceNull"
                j.set_sampler(op, name, protolite.encode(S[name + "SamplerArgs"], {"spacing": st[1]}))
                cur = (op, cur[1])
            elif st[0] == "twice":
                cur = (g.add_op("TestTwoOut", [cur]), "twice")
            elif st[0] == "affine":
                op = g.add_op("TestAffine", [cur], args=protolite.encode(TEST_ARGS["TestScaleArgs"], {"scale": st[1]}))
                j.set_stream_args(op, protolite.encode(TEST_ARGS["TestOffsetArgs"], {"offset": st[2]}))
                cur = (op, "out")
            elif st[0] == "window":
                cur = (g.add_op("TestWindow", [cur]), "window")
        sink = g.add_sink(cur)
        eng.run(g, [j], wps, ios)
        want = model(n, stages)
        assert j.output_rows(sink) == len(want), (case, n, stages, wps, ios)
        for i, w in enumerate(want):
            row = j.output_row(sink, i)
            if w is None:
                assert row is None, (case, i, stages)
            elif isinstance(w, tuple):
                assert struct.unpack("<3q", row) == w, (case, i, n, stages, wps, ios)
            else:
                assert struct.unpack("<q", row)[0] == w, (case, i, n, stages, wps, ios)
