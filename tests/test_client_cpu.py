"""The scannerpy-shaped surface (scanner_b200.client) on the CPU with the test op library:
the same call shapes as the reference's tests/py_test.py and examples/tutorials/00_basic.py."""
import os
import struct
import subprocess

import numpy as np
import pytest

import oracle
from oracle import synth
import scanner_b200 as sp
from scanner_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sc():
    oracle.build()
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "cpp")], stdout=subprocess.DEVNULL)
    c = sp.Client(gpus=[], cpu_instances=2)
    so = os.path.join(ROOT, "build", "tests", "libtest_plugin_ops.so")
    # Client.load_op(so_path, proto_path) (reference client.py:514-537): the argument messages of the
    # ops are the ones they registered with (.protobuf_name / .stream_protobuf_name), found in the file
    c.load_op(so, os.path.join(ROOT, "tests", "cpp", "test_args.proto"))
    assert sorted(c._op_protos["TestAffine"]) == ["init", "stream"] and list(c._op_protos["TestResizeOracle"]) == ["stream"]
    yield c
    c.stop()


def test_basic_tutorial_shape(sc):
    """examples/tutorials/00_basic.py:27-80 -- two videos, Histogram, len(hist)==3, 16 bins."""
    clips = [np.stack([synth.smooth_frame(10 * k + i, 48, 64) for i in range(9 + k)]) for k in range(2)]
    v1 = sp.NamedVideoStream(sc, "example1", frames=clips[0])
    v2 = sp.NamedVideoStream(sc, "example2", frames=clips[1])
    frames = sc.io.Input([v1, v2])
    hists = sc.ops.TestHistogramOracle(frame=frames)
    o1, o2 = sp.NamedStream(sc, "example1_hist"), sp.NamedStream(sc, "example2_hist")
    sc.run(sc.io.Output(hists, [o1, o2]), sp.PerfParams.estimate())
    for clip, out, v in zip(clips, (o1, o2), (v1, v2)):
        num_rows = 0
        for i, hist in enumerate(out.load()):
            assert len(hist) == 3 and hist[0].shape[0] == 16
            assert (np.stack(hist) == oracle.hist16(clip[i])).all()
            num_rows += 1
        assert num_rows == v.len() == out.len()


def test_streams_and_per_stream_args(sc):
    rows = [struct.pack("<q", i) for i in range(40)]
    a, b = sp.NamedStream(sc, "ints_a", rows=rows), sp.NamedStream(sc, "ints_b", rows=rows[:20])
    col = sc.io.Input([a, b])
    sampled = sc.streams.Stride(col, [4, 5])
    aff = sc.ops.TestAffine(col=sampled, scale=2, offset=[100, 200])
    oa, ob = sp.NamedStream(sc, "oa"), sp.NamedStream(sc, "ob")
    sc.run(sc.io.Output(aff, [oa, ob]), sp.PerfParams.manual(2, 4))
    assert [struct.unpack("<q", r)[0] for r in oa.load()] == [2 * i + 100 for i in range(0, 40, 4)]
    assert [struct.unpack("<q", r)[0] for r in ob.load()] == [2 * i + 200 for i in range(0, 20, 5)]


def test_gather_range_and_bounded_state(sc):
    """reference py_test.py:407-423."""
    rows = [struct.pack("<q", i) for i in range(40)]
    a = sp.NamedStream(sc, "ints_c", rows=rows)
    col = sc.io.Input([a])
    inc = sc.ops.TestIncrementBounded(ignore=col, bounded_state=3)
    g = sc.streams.Gather(inc, indices=[[0, 10, 25, 26, 27]])
    out = sp.NamedStream(sc, "test_bounded_state")
    sc.run(sc.io.Output(g, [out]), sp.PerfParams.estimate())
    assert [struct.unpack("=q", buf)[0] for buf in out.load()] == [0, 3, 3, 4, 5]
    r = sc.streams.Range(col, [(0, 30)])
    out2 = sp.NamedStream(sc, "range")
    sc.run(sc.io.Output(r, [out2]), sp.PerfParams.estimate())
    assert out2.len() == 30


def test_errors_are_scanner_exceptions(sc):
    with pytest.raises(sp.ScannerException):
        sc.ops.NoSuchOp
    rows = [struct.pack("<q", i) for i in range(4)]
    a = sp.NamedStream(sc, "ints_d", rows=rows)
    with pytest.raises(sp.ScannerException, match="does not take argument"):
        sc.ops.TestAffine(col=sc.io.Input([a]), bogus=1)


# ------------------------------------------------------------------------------------------------
def _db_client(path):
    c = sp.Client(gpus=[], cpu_instances=2, db_path=str(path))
    c.load_op(os.path.join(ROOT, "build", "tests", "libtest_plugin_ops.so"),
              os.path.join(ROOT, "tests", "cpp", "test_args.proto"))
    return c


def test_database_backed_streams_persist_and_cache_modes(sc, tmp_path):
    """Outputs are committed as tables (reference storage.py NamedStream / CacheMode, client.py:1325-1370)
    and a later session loads them without re-running."""
    rows = [struct.pack("<q", i) for i in range(30)]
    c1 = _db_client(tmp_path / "db")
    src = sp.NamedStream(c1, "ints", rows=rows)
    out = sp.NamedStream(c1, "ints_scaled")
    assert not out.exists()
    aff = c1.ops.TestAffine(col=c1.io.Input([src]), scale=3, offset=[7])
    assert c1.run(c1.io.Output(aff, [out]), sp.PerfParams.manual(4, 8)) == 1
    want = [3 * i + 7 for i in range(30)]
    assert [struct.unpack("<q", r)[0] for r in out.load()] == want
    assert c1.table_names() == ["ints_scaled"] and out.exists()
    # the same output again: Error refuses, Ignore skips the job, Overwrite recomputes
    with pytest.raises(sp.ScannerException, match="already exists"):
        c1.run(c1.io.Output(aff, [out]), sp.PerfParams.manual(4, 8))
    assert c1.run(c1.io.Output(aff, [out]), sp.PerfParams.manual(4, 8), cache_mode=sp.CacheMode.Ignore) == 0
    assert [struct.unpack("<q", r)[0] for r in out.load(rows=[0, 29])] == [want[0], want[29]]
    aff2 = c1.ops.TestAffine(col=c1.io.Input([src]), scale=5, offset=[1])
    assert c1.run(c1.io.Output(aff2, [out]), sp.PerfParams.manual(4, 8), cache_mode=sp.CacheMode.Overwrite) == 1
    assert [struct.unpack("<q", r)[0] for r in out.load()] == [5 * i + 1 for i in range(30)]
    c1.stop()

    c2 = _db_client(tmp_path / "db")          # a later session
    t = c2.table("ints_scaled")
    assert t.num_rows() == 30 and t.column_names() == ["index", "out"] and "ints_scaled" in c2.summarize()
    assert [struct.unpack("<q", r)[0] for r in t.column("out").load(rows=[3])] == [16]
    assert [struct.unpack("<q", r)[0] for r in t.column("index").load(rows=[29])] == [29]
    again = sp.NamedStream(c2, "ints_scaled")
    assert again.exists() and again.len() == 30
    assert [struct.unpack("<q", r)[0] for r in again.load()] == [5 * i + 1 for i in range(30)]
    again.delete()
    assert c2.table_names() == [] and not sp.NamedStream(c2, "ints_scaled").exists()
    with pytest.raises(sp.ScannerException, match="without db_path"):
        sc.has_table("x")
    c2.stop()


def test_ingest_videos_from_mp4_and_h264_files(tmp_path):
    """Client.ingest_videos (reference client.py:1009-1078): tables appear, failures are reported per
    file, a stored video re-binds by name in a later session (decode itself needs a GPU)."""
    rng = np.random.default_rng(8)
    n, h, w = 8, 48, 64
    yuv = rng.integers(0, 256, (n, h * w * 3 // 2), dtype=np.uint8)
    stream = E.h264_synth(yuv, w, h, gop=4)
    mp4, raw = tmp_path / "a.mp4", tmp_path / "b.h264"
    mp4.write_bytes(E.mp4_mux(stream, 25, 1))
    raw.write_bytes(stream)
    c = sp.Client(gpus=[], cpu_instances=1, db_path=str(tmp_path / "db"), load_stdlib=False)
    done, failed = c.ingest_videos([("a", str(mp4)), ("b", str(raw)), ("c", str(tmp_path / "nope.mp4"))])
    assert [v.name() for v in done] == ["a", "b"] and len(failed) == 1 and "nope.mp4" in failed[0][0]
    assert all(v.len() == n and v.info()["width"] == w for v in done)
    _, failed = c.ingest_videos([("a", str(mp4))])
    assert "already exists" in failed[0][1]
    done, failed = c.ingest_videos([("a", str(raw))], force=True)
    assert not failed and done[0].len() == n
    # inplace=True: the table points at the file instead of holding a copy (py_test.py 'test1_inplace')
    done, failed = c.ingest_videos([("a_inplace", str(mp4))], inplace=True)
    assert not failed and done[0].len() == n and done[0].info()["keyframes"] == 2
    assert not os.path.exists(os.path.join(str(tmp_path / "db"), "tables", str(c.table("a_inplace").id()), "1_0.bin"))
    assert sp.NamedVideoStream(c, "v_inplace", path=str(raw), inplace=True).len() == n
    for name in ("a_inplace", "v_inplace"):
        c.delete_table(name)
    c.stop()
    c2 = sp.Client(gpus=[], cpu_instances=1, db_path=str(tmp_path / "db"), load_stdlib=False)
    assert sorted(c2.table_names()) == ["a", "b"]
    v = sp.NamedVideoStream(c2, "b")       # by name only: bound from the stored descriptor
    assert v.len() == n and v.info()["keyframes"] == 2
    # export the stored table as .mp4 again: FFmpeg reads it, and it demuxes to the ingested stream
    out = v.save_mp4(str(tmp_path / "exported"))
    import cv2
    cap = cv2.VideoCapture(out)
    assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == n and abs(cap.get(cv2.CAP_PROP_FPS) - 25) < 1e-6
    assert E.mp4_demux(open(out, "rb").read())[0] == stream
    missing = sp.NamedVideoStream(c2, "zzz")      # allowed: it may become the target of an Output
    assert not missing.exists()
    with pytest.raises(sp.ScannerException, match="does not exist"):
        missing.len()
    c2.stop()


# ------------------------------------------------------------------------------------------------
def _ints(sc, name, n):
    return sp.NamedStream(sc, name, rows=[struct.pack("<q", i) for i in range(n)])


def _load_ints(stream):
    return [struct.unpack("<q", r)[0] for r in stream.load()]


def test_reference_tutorial_00_on_the_cpu_with_a_real_video(tmp_path):
    """examples/tutorials/00_basic.py of the reference with device=CPU: ingest an .mp4, Histogram every frame, load
    the rows.  No GPU anywhere: the CPU instance decodes with FFmpeg (swdec.h) and runs the CPU Histogram kernel."""
    import cv2
    from scanner_b200 import synth_h264
    from scanner_b200.client import Client, DeviceType, NamedStream, NamedVideoStream, PerfParams
    data, _ = synth_h264.write(320, 240, 20, gop=5, seed=1)
    mp4 = str(tmp_path / "a.mp4")
    open(mp4, "wb").write(E.mp4_mux(data, 30, 1))
    cl = Client(gpus=[], db_path=str(tmp_path / "db"))   # CPU instances only, also where a GPU is present
    frames = cl.io.Input([NamedVideoStream(cl, "clip", path=mp4)])
    hist = cl.ops.Histogram(frame=frames, device=DeviceType.CPU)
    out = NamedStream(cl, "hists")
    cl.run(cl.io.Output(hist, [out]), PerfParams.manual(5, 10))
    rows = list(out.load())
    cap = cv2.VideoCapture(mp4)
    assert len(rows) == 20
    for r in rows:
        ok, f = cap.read()
        assert ok and (np.asarray(r).reshape(3, 16) == oracle.hist16(np.ascontiguousarray(f[..., ::-1]))).all()


def test_slice_unslice_keeps_every_row(sc):
    """reference tests/py_test.py:350-358 test_slice: Slice(all(50)) -> Unslice gives the input back."""
    src = _ints(sc, "slice_in", 130)
    col = sc.io.Input([src])
    sliced = sc.streams.Slice(col, partitions=[sc.partitioner.all(50)])
    out = sp.NamedStream(sc, "slice_out")
    sc.run(sc.io.Output(sc.streams.Unslice(sliced), [out]), sp.PerfParams.manual(4, 16))
    assert out.len() == src.len() == 130 and _load_ints(out) == list(range(130))


def test_overlapping_slices_with_a_sampler_per_group(sc):
    """py_test.py:361-375 test_overlapping_slice: three overlapping ranges, a Range per slice group
    (SliceList), 30 rows out -- here the values are checked too."""
    src = _ints(sc, "ovl_in", 40)
    col = sc.io.Input([src])
    sliced = sc.streams.Slice(col, partitions=[sc.partitioner.strided_ranges([(0, 15), (5, 25), (15, 35)], 1)])
    sampled = sc.streams.Range(sliced, ranges=[sp.SliceList([{"start": 0, "end": 10}, {"start": 5, "end": 15},
                                                             {"start": 5, "end": 15}])])
    out = sp.NamedStream(sc, "ovl_out")
    sc.run(sc.io.Output(sc.streams.Unslice(sampled), [out]), sp.PerfParams.manual(3, 6))
    want = list(range(0, 10)) + list(range(10, 20)) + list(range(20, 30))
    assert out.len() == 30 and _load_ints(out) == want


def test_state_and_stencils_restart_at_slice_boundaries(sc):
    """Inside a Slice every group is an independent stream: an unbounded-state counter restarts at 0
    in every group, a stencil window clamps at the group's edges instead of reading its neighbour."""
    src = _ints(sc, "st_in", 23)
    col = sc.io.Input([src])
    sliced = sc.streams.Slice(col, partitions=[sc.partitioner.all(10)])
    counted = sc.ops.TestIncrementUnbounded(ignore=sliced)
    window = sc.ops.TestWindow(col=sliced)
    o1, o2 = sp.NamedStream(sc, "st_cnt"), sp.NamedStream(sc, "st_win")
    sc.run([sc.io.Output(sc.streams.Unslice(counted), [o1]), sc.io.Output(sc.streams.Unslice(window), [o2])],
           sp.PerfParams.manual(2, 4))
    assert _load_ints(o1) == list(range(10)) + list(range(10)) + list(range(3))
    got = [struct.unpack("<3q", r) for r in o2.load()]
    want = []
    for lo, hi in ((0, 10), (10, 20), (20, 23)):
        for i in range(lo, hi):
            want.append((max(lo, i - 1), i, min(hi - 1, i + 1)))
    assert got == want


def test_per_slice_stream_args_and_gather_partitioner(sc):
    """py_test.py:393-404 test_slice_args: one new_stream argument per slice group (SliceList)."""
    src = _ints(sc, "args_in", 12)
    col = sc.io.Input([src])
    sliced = sc.streams.Slice(col, [sc.partitioner.gather([[0, 1, 2], [3, 7], [11]])])
    aff = sc.ops.TestAffine(col=sliced, scale=10, offset=[sp.SliceList([1, 2, 3])])
    out = sp.NamedStream(sc, "args_out")
    sc.run(sc.io.Output(sc.streams.Unslice(aff), [out]), sp.PerfParams.manual(2, 2))
    assert _load_ints(out) == [1, 11, 21, 32, 72, 113]
    with pytest.raises(sp.ScannerException, match="ascending"):
        bad = sc.streams.Slice(col, [sc.partitioner.gather([[5, 2]])])
        sc.run(sc.io.Output(sc.streams.Unslice(bad), [sp.NamedStream(sc, "args_bad")]), sp.PerfParams.manual(2, 2))


def test_slice_errors(sc):
    src = _ints(sc, "err_in", 10)
    col = sc.io.Input([src])
    sliced = sc.streams.Slice(col, partitions=[sc.partitioner.all(5)])
    with pytest.raises(sp.ScannerException, match="must be unsliced"):
        sc.run(sc.io.Output(sliced, [sp.NamedStream(sc, "e1")]), sp.PerfParams.manual(2, 2))
    with pytest.raises(sp.ScannerException, match="not been sliced"):
        sc.run(sc.io.Output(sc.streams.Unslice(col), [sp.NamedStream(sc, "e2")]), sp.PerfParams.manual(2, 2))
    un = sc.streams.Unslice(sliced)
    with pytest.raises(sp.ScannerException, match="only supports Output"):
        sc.run(sc.io.Output(sc.ops.TestAffine(col=un, scale=1, offset=[0]), [sp.NamedStream(sc, "e3")]),
               sp.PerfParams.manual(2, 2))
    with pytest.raises(sp.ScannerException, match="3 samplers but there are 2 slice groups"):
        bad = sc.streams.Range(sliced, ranges=[sp.SliceList([{"start": 0, "end": 2}] * 3)])
        sc.run(sc.io.Output(sc.streams.Unslice(bad), [sp.NamedStream(sc, "e4")]), sp.PerfParams.manual(2, 2))


def test_frame_outputs_into_a_named_video_stream(sc, tmp_path):
    """An Output may target a NamedVideoStream (reference storage.py): frames are stored (uncompressed --
    there is no encoder here) and load() yields them, in memory and from the database."""
    frames = np.stack([synth.rand_frame(400 + i, 24, 32) for i in range(7)])
    for client in (sc, _db_client(tmp_path / "db")):
        vin = sp.NamedVideoStream(client, "vs_in", frames=frames)
        small = client.ops.TestResizeOracle(frame=client.io.Input([vin]), width=[16], height=[12])
        vout = sp.NamedVideoStream(client, "vs_out")
        assert not vout.exists()
        client.run(client.io.Output(small, [vout]), sp.PerfParams.manual(2, 4), cache_mode=sp.CacheMode.Overwrite)
        assert vout.exists() and vout.len() == 7
        for i, f in enumerate(vout.load()):
            assert (f == oracle.resize(frames[i], 16, 12)).all()
        if client is not sc:
            client.stop()


def test_new_table_from_python_rows(tmp_path):
    """Reference tests/py_test.py:209-217 (test_new_table) plus nulls, force and the catalogue."""
    c = sp.Client(gpus=[], cpu_instances=1, db_path=str(tmp_path / "db"), load_stdlib=False)
    t = c.new_table("test", ["col1", "col2"], [[b"r00", b"r01"], [b"r10", b"r11"], [b"", None]])
    assert t.num_rows() == 3 and t.column_names() == ["index", "col1", "col2"]
    assert next(t.column("col2").load()) == b"r01"
    assert list(t.column("col1").load()) == [b"r00", b"r10", None]  # NullElement() == None
    got = list(t.column("col2").load(rows=[1, 2]))
    assert got[0] == b"r11" and isinstance(got[1], sp.NullElement)
    assert [struct.unpack("<q", r)[0] for r in t.column("index").load()] == [0, 1, 2]
    with pytest.raises(sp.ScannerException, match="existing name"):
        c.new_table("test", ["a"], [[b"x"]])
    t = c.new_table("test", ["a"], [[b"x"]], force=True)
    assert t.column_names() == ["index", "a"] and t.num_rows() == 1
    with pytest.raises(sp.ScannerException, match="every row must have 2 elements"):
        c.new_table("bad", ["a", "b"], [[b"x"]])
    assert not c.has_table("bad")
    # the table is a normal stored stream: a job can read its column
    src = sp.NamedStream(c, "test")
    assert src.exists() and list(src.load()) == [b"x"]
    with sp.Client(gpus=[], cpu_instances=1, db_path=str(tmp_path / "db"), load_stdlib=False) as c2:
        assert c2.table("test").num_rows() == 1
        assert list(c2.sequence("test").load()) == [b"x"] and c2.get_active_jobs() == []
        c2.new_table("other", ["v"], [[b"1"]])
        c2.delete_tables(["test", "other"])
        assert c2.table_names() == []
    c.stop()


def test_sampler_arguments_in_every_form_the_reference_accepts(sc):
    """py_test.py:274-336 test_sample / test_space call the samplers with keyword `input=` and with
    dict arguments ({'stride': 8}, {'start': 0, 'end': 30}, {'start':, 'end':, 'stride':}); the
    tutorials use plain numbers and tuples.  Both must select the same rows."""
    src = _ints(sc, "samp_in", 60)

    def rows(make):
        out = sp.NamedStream(sc, "samp_out")
        sc.run(sc.io.Output(make(sc.io.Input([src])), [out]), sp.PerfParams.manual(4, 8),
               cache_mode=sp.CacheMode.Overwrite)
        return list(out.load())

    def ints(make):
        return [struct.unpack("<q", r)[0] for r in rows(make)]

    assert ints(lambda c: sc.streams.Stride(input=c, strides=[{"stride": 8}])) == list(range(0, 60, 8)) \
        == ints(lambda c: sc.streams.Stride(c, [8]))
    assert ints(lambda c: sc.streams.Range(input=c, ranges=[{"start": 0, "end": 30}])) == list(range(30)) \
        == ints(lambda c: sc.streams.Range(c, [(0, 30)]))
    assert ints(lambda c: sc.streams.StridedRange(input=c, ranges=[{"start": 0, "end": 50, "stride": 10}])) \
        == [0, 10, 20, 30, 40] == ints(lambda c: sc.streams.StridedRange(c, [(0, 50, 10)]))
    assert ints(lambda c: sc.streams.StridedRanges(c, [[(0, 10), (30, 40)]], stride=5)) == [0, 5, 30, 35]
    assert ints(lambda c: sc.streams.Gather(input=c, indices=[[0, 15, 37, 50]])) == [0, 15, 37, 50]
    rep = ints(lambda c: sc.streams.Repeat(input=sc.streams.Range(c, [(0, 3)]), spacings=[4]))
    assert rep == [0] * 4 + [1] * 4 + [2] * 4
    nulls = rows(lambda c: sc.streams.RepeatNull(input=sc.streams.Range(c, [(0, 3)]), spacings=[{"spacing": 4}]))
    assert len(nulls) == 12
    for i, r in enumerate(nulls):
        if i % 4 == 0:
            assert not isinstance(r, sp.NullElement) and struct.unpack("<q", r)[0] == i // 4
        else:
            assert isinstance(r, sp.NullElement)
    with pytest.raises(sp.ScannerException, match="lacks 'end'"):
        sc.streams.StridedRange(sc.io.Input([src]), [{"start": 0, "stride": 2}])


def test_cpp_kernel_reports_bad_data_without_aborting(sc):
    """scanner::report_kernel_error (scanner/api/kernel.h) from a C++ plugin kernel: the run fails
    with the kernel's message; the same client then runs the next job."""
    src = _ints(sc, "refuse_in", 20)
    col = sc.io.Input([src])
    out = sp.NamedStream(sc, "refuse_out")
    sc.run(sc.io.Output(sc.ops.TestRefuseValue(col=col, scale=99), [out]), sp.PerfParams.manual(2, 4))
    live = sc.stats()["counters"]["cpu_bytes_live"]
    with pytest.raises(sp.ScannerException, match=r"Op TestRefuseValue failed: .*cannot process the value 13 \(row 13\)"):
        sc.run(sc.io.Output(sc.ops.TestRefuseValue(col=col, scale=13), [out]), sp.PerfParams.manual(2, 4),
               cache_mode=sp.CacheMode.Overwrite)
    # the failed packet released what it owned (rows handed in, rows of earlier batches, sink rows)
    assert sc.stats()["counters"]["cpu_bytes_live"] == live
    sc.run(sc.io.Output(sc.ops.TestRefuseValue(col=col, scale=99), [out]), sp.PerfParams.manual(2, 4),
           cache_mode=sp.CacheMode.Overwrite)
    assert _load_ints(out) == list(range(20))


# ---- regressions for the round-1 advisor findings -------------------------------------------------
def test_null_only_tasks_of_a_video_table_stay_video_items(tmp_path):
    """A task whose rows are all null (RepeatNull spacing) must still be written as a video item of a
    Video column: the item kind comes from the declared column type, not from the rows."""
    c = _db_client(tmp_path / "db")
    frames = np.stack([synth.rand_frame(900 + i, 16, 24) for i in range(3)])
    vin = sp.NamedVideoStream(c, "nul_in", frames=frames)
    spaced = c.streams.RepeatNull(c.io.Input([vin]), [8])
    vout = sp.NamedVideoStream(c, "nul_out")
    c.run(c.io.Output(spaced, [vout]), sp.PerfParams.manual(2, 4), cache_mode=sp.CacheMode.Overwrite)
    got = list(vout.load())
    assert len(got) == 24
    for i, f in enumerate(got):
        if i % 8 == 0:
            assert (f == frames[i // 8]).all()
        else:
            assert isinstance(f, sp.NullElement)
    c.stop()


def test_large_pass_through_rows_survive_engine_teardown():
    """Sink rows >= 64 KB that pass an input stream through unchanged pointed into the stream's adopted
    storage; destroying the engine before the job's outputs aborted the process ("not a live buffer")."""
    import gc
    c = sp.Client(gpus=[], cpu_instances=1)
    frames = np.stack([synth.rand_frame(950 + i, 200, 200) for i in range(6)])
    vin = sp.NamedVideoStream(c, "big_in", frames=frames)
    strided = c.streams.Stride(c.io.Input([vin]), [2])
    vout = sp.NamedVideoStream(c, "big_out")
    c.run(c.io.Output(strided, [vout]), sp.PerfParams.manual(2, 4), cache_mode=sp.CacheMode.Overwrite)
    got = [np.array(f) for f in vout.load()]
    c.stop()
    del c, vin, vout, strided
    gc.collect()
    assert len(got) == 3 and all((got[i] == frames[2 * i]).all() for i in range(3))


def test_gather_rows_must_ascend(sc):
    rows = [struct.pack("<q", i) for i in range(20)]
    a = sp.NamedStream(sc, "ints_g", rows=rows)
    g = sc.streams.Gather(sc.io.Input([a]), indices=[[5, 3, 10]])
    with pytest.raises((sp.ScannerException, E.EngineError), match="strictly ascending"):
        sc.run(sc.io.Output(g, [sp.NamedStream(sc, "g_out")]), sp.PerfParams.manual(2, 4), cache_mode=sp.CacheMode.Overwrite)
    g2 = sc.streams.Gather(sc.io.Input([a]), indices=[[3, 3, 10]])
    with pytest.raises((sp.ScannerException, E.EngineError), match="strictly ascending"):
        sc.run(sc.io.Output(g2, [sp.NamedStream(sc, "g_out2")]), sp.PerfParams.manual(2, 4), cache_mode=sp.CacheMode.Overwrite)
