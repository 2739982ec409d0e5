"""The pipeline on a real GPU: NVDEC decode of synthetic (lossless I_PCM) H.264 into device frames,
the stdlib GPU ops behind REGISTER_KERNEL, results brought back through the save stage.
Every comparison is bit-exact: I_PCM decodes to the source planes, so the expected RGB is the
oracle's NV12->RGB of the planes the stream was made from."""
import os

import numpy as np
import pytest

import oracle
from oracle import synth
from scanner_b200 import engine as E
from scanner_b200 import protolite

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STD_ARGS = protolite.parse_proto(open(os.path.join(ROOT, "scanner_b200", "csrc", "ops", "stdlib_args.proto")).read())


@pytest.fixture(scope="module", autouse=True)
def stdlib():
    E.load_stdlib()


@pytest.fixture()
def eng():
    e = E.Engine(gpus=[0], instances_per_gpu=3)
    yield e
    e.close()


def make_clip(seed, n, h, w, gop, non_key="pcm"):
    """-> (stream bytes, expected RGB frames (n,h,w,3)) ; planes are uniform random bytes."""
    rng = np.random.default_rng(seed)
    y = rng.integers(0, 256, (n, h, w), dtype=np.uint8)
    u = rng.integers(0, 256, (n, h // 2, w // 2), dtype=np.uint8)
    v = rng.integers(0, 256, (n, h // 2, w // 2), dtype=np.uint8)
    yuv = np.concatenate([y.reshape(n, -1), u.reshape(n, -1), v.reshape(n, -1)], axis=1)
    if non_key == "skip":
        data = E.h264_synth(yuv[::gop], w, h, gop=gop, non_key="skip", frames=n)
    elif non_key == "bidir":
        # odd GOP positions are B pictures coded after their later anchor; what is displayed there
        # is the rounded mean of the two anchors (validated against FFmpeg in test_storage_cpu.py)
        data = E.h264_synth(yuv, w, h, gop=gop, non_key="bidir")
        shown = E.bidir_expected(yuv, gop)
        y = shown[:, :h * w].reshape(n, h, w)
        u = shown[:, h * w:h * w + h * w // 4].reshape(n, h // 2, w // 2)
        v = shown[:, h * w + h * w // 4:].reshape(n, h // 2, w // 2)
    else:
        data = E.h264_synth(yuv, w, h, gop=gop)
    rgb = []
    for i in range(n):
        src = (i // gop) * gop if non_key == "skip" else i  # P_Skip repeats the last key picture
        chroma = np.empty((h // 2, w), np.uint8)
        chroma[:, 0::2], chroma[:, 1::2] = u[src], v[src]
        rgb.append(oracle.nv12_to_rgb(y[src], chroma))
    return data, np.stack(rgb)


def test_nvdec_is_present():
    caps = E.nvdec_caps(0)
    if not caps["available"]:
        # a container started without the driver's video capability: the engine decodes with FFmpeg (nvdec.h)
        pytest.skip(f"the GPU exposes no NVDEC engine to this process: {caps}")
    assert caps["h264"] and caps["engines"] >= 1, caps


@pytest.mark.parametrize("h,w,n,gop,mode", [(96, 128, 11, 4, "pcm"), (480, 640, 9, 5, "pcm"), (1080, 1920, 7, 3, "pcm"),
                                            (112, 200, 8, 8, "pcm"), (96, 128, 10, 5, "skip"),
                                            (96, 128, 13, 6, "bidir"), (480, 640, 9, 9, "bidir")])
def test_decode_all_frames_bit_exact(eng, h, w, n, gop, mode):
    data, want = make_clip(11, n, h, w, gop, mode)
    sid = eng.add_h264(data)
    info = eng.stream_info(sid)
    assert (info["width"], info["height"]) == (w, h) and eng.stream_rows(sid) == n
    g = E.Graph()
    src = g.add_source(True)
    sink = g.add_sink((src, "frame"))
    j = E.Job()
    j.bind_source(src, sid)
    for (wps, ios) in [(4, 8), (1, 1), (16, 16)]:
        eng.run(g, [j], wps, ios)
        assert j.output_rows(sink) == n
        for i in range(n):
            got = j.output_row(sink, i)
            assert got.shape == (h, w, 3)
            assert (got == want[i]).all(), (i, wps, ios)
    st = eng.stats()["counters"]
    assert st["frames_used"] == n


def test_gather_decodes_only_needed_gops(eng):
    n, gop = 40, 8
    data, want = make_clip(12, n, 96, 128, gop)
    sid = eng.add_h264(data)
    g = E.Graph()
    src = g.add_source(True)
    s = g.add_sample((src, "frame"))
    sink = g.add_sink((s, "frame"))
    rows = [3, 4, 17, 39]
    j = E.Job()
    j.bind_source(src, sid)
    j.set_sampler(s, "Gather", protolite.encode(protolite.SAMPLER_ARGS["GatherSamplerArgs"], {"rows": rows}))
    eng.run(g, [j], 2, 4)
    for k, r in enumerate(rows):
        assert (j.output_row(sink, k) == want[r]).all()
    c = eng.stats()["counters"]
    assert c["frames_used"] == 4
    # rows 3,4 need frames 0..4 of GOP 0; 17 needs 16..17; 39 needs 32..39: 5 + 2 + 8 decoded
    assert c["frames_decoded"] == 15


def test_b_pictures_rows_are_display_order_and_sparse_rows_feed_past_the_target(eng):
    """A stream whose coding order differs from its display order (I0 P2 B1 P4 B3 ...): table rows are
    display positions, and a wanted B picture needs the anchor coded AFTER it -- the decode stage must
    not stop feeding at the wanted position (it does for streams whose SPS rules reordering out)."""
    n, gop = 24, 8
    data, want = make_clip(21, n, 96, 128, gop, "bidir")
    sid = eng.add_h264(data)
    assert eng.stream_may_reorder(sid)
    plain, _ = make_clip(21, 4, 96, 128, 2)
    assert not eng.stream_may_reorder(eng.add_h264(plain))
    g = E.Graph()
    src = g.add_source(True)
    s = g.add_sample((src, "frame"))
    sink = g.add_sink((s, "frame"))
    for rows in ([1], [3, 4, 9, 17, 23], [5, 6, 7], list(range(0, n, 3))):
        j = E.Job()
        j.bind_source(src, sid)
        j.set_sampler(s, "Gather", protolite.encode(protolite.SAMPLER_ARGS["GatherSamplerArgs"], {"rows": rows}))
        eng.run(g, [j], 2, 4)
        assert j.output_rows(sink) == len(rows)
        for k, r in enumerate(rows):
            assert (j.output_row(sink, k) == want[r]).all(), (rows, r)
    got = eng.decode_to_device(sid, [1, 2, 15, 16, 21]).cpu().numpy()
    assert (got == want[[1, 2, 15, 16, 21]]).all()


def strip_repeated_parameter_sets(stream):
    """Drop the SPS / PPS NAL units of every GOP but the first: what encoders write unless asked to
    repeat headers (x264 without --repeat-headers, most .mp4 -> Annex-B conversions of one avcC)."""
    sc = b"\x00\x00\x00\x01"
    parts = stream.split(sc)[1:]
    out, seen = [], set()
    for nal in parts:
        t = nal[0] & 0x1F
        if t in (7, 8):
            if t in seen:
                continue
            seen.add(t)
        out.append(sc + nal)
    return b"".join(out)


def test_seeking_into_a_stream_whose_parameter_sets_appear_once(eng):
    """A decode that starts at a later IDR gets SPS / PPS from the index's metadata packets (the
    reference replays them the same way after a seek, decoder_automata.cpp:299-318)."""
    n, gop = 24, 6
    data, want = make_clip(31, n, 96, 128, gop)
    lean = strip_repeated_parameter_sets(data)
    assert len(lean) < len(data) and lean.count(b"\x00\x00\x00\x01\x67") == 1
    sid = eng.add_h264(lean)
    assert eng.stream_rows(sid) == n and eng.stream_info(sid)["keyframes"] == n // gop
    got = eng.decode_to_device(sid, [20, 21]).cpu().numpy()
    assert (got == want[[20, 21]]).all()
    g = E.Graph()
    src = g.add_source(True)
    s = g.add_sample((src, "frame"))
    sink = g.add_sink((s, "frame"))
    rows = [7, 13, 14, 23]
    j = E.Job()
    j.bind_source(src, sid)
    j.set_sampler(s, "Gather", protolite.encode(protolite.SAMPLER_ARGS["GatherSamplerArgs"], {"rows": rows}))
    eng.run(g, [j], 2, 4)
    for k, r in enumerate(rows):
        assert (j.output_row(sink, k) == want[r]).all(), r


def test_stride_30_only_keyframes(eng):
    """configs[4] shape: Stride(gop) touches exactly the IDR of every GOP."""
    n, gop = 60, 6
    data, want = make_clip(13, n, 96, 128, gop)
    sid = eng.add_h264(data)
    g = E.Graph()
    src = g.add_source(True)
    s = g.add_sample((src, "frame"))
    h = g.add_op("Histogram", [(s, "frame")], device=1)
    sink = g.add_sink((h, "histogram"))
    j = E.Job()
    j.bind_source(src, sid)
    j.set_sampler(s, "Strided", protolite.encode(protolite.SAMPLER_ARGS["StridedSamplerArgs"], {"stride": gop}))
    eng.run(g, [j], 5, 10)
    hist = j.output_array(sink, 192, np.int32).reshape(-1, 3, 16)
    assert len(hist) == n // gop
    for k in range(n // gop):
        assert (hist[k] == oracle.hist16(want[k * gop])).all()
    c = eng.stats()["counters"]
    assert c["frames_used"] == c["frames_decoded"] == n // gop


@pytest.mark.parametrize("force_rgb", [False, True])
def test_c2_dag_histogram_and_resize_on_decoded_frames(eng, force_rgb, monkeypatch):
    """BASELINE configs[1] DAG through the engine: decode -> {Histogram, Resize(224)}.  Both consumers
    registered for NV12 surfaces, so the decode stage hands them the decoder's own format and RGB24 is
    never written; SCN_DECODE_RGB=1 forces the reference's RGB24 elements.  Same bits either way."""
    if force_rgb:
        monkeypatch.setenv("SCN_DECODE_RGB", "1")
    else:
        monkeypatch.delenv("SCN_DECODE_RGB", raising=False)
    n = 10
    data, want = make_clip(14, n, 1080, 1920, 5)
    sid = eng.add_h264(data)
    g = E.Graph()
    src = g.add_source(True)
    hs = g.add_op("Histogram", [(src, "frame")], device=1)
    rz = g.add_op("Resize", [(src, "frame")], device=1)
    s_h = g.add_sink((hs, "histogram"))
    s_r = g.add_sink((rz, "frame"))
    j = E.Job()
    j.bind_source(src, sid)
    j.set_stream_args(rz, protolite.encode(STD_ARGS["ResizeArgs"], {"width": 224, "height": 224}))
    eng.run(g, [j], 4, 8)
    hist = j.output_array(s_h, 192, np.int32).reshape(n, 3, 16)
    for i in range(n):
        assert (hist[i] == oracle.hist16(want[i])).all()
        assert (j.output_row(s_r, i) == oracle.resize(want[i], 224, 224)).all()
    assert eng.stats()["counters"]["frames_delivered_nv12"] == (0 if force_rgb else n)


def test_mixed_consumers_keep_rgb_elements(eng):
    """One consumer (Blur) only takes dense RGB24 -> the column is delivered as RGB24 to everyone."""
    n = 5
    data, want = make_clip(31, n, 96, 128, 5)
    sid = eng.add_h264(data)
    g = E.Graph()
    src = g.add_source(True)
    hs = g.add_op("Histogram", [(src, "frame")], device=1)
    bl = g.add_op("Blur", [(src, "frame")], device=1,
                  args=protolite.encode(STD_ARGS["BlurArgs"], {"kernel_size": 3, "sigma": 0.5}))
    s_h = g.add_sink((hs, "histogram"))
    s_b = g.add_sink((bl, "frame"))
    j = E.Job()
    j.bind_source(src, sid)
    eng.run(g, [j], 5, 5)
    hist = j.output_array(s_h, 192, np.int32).reshape(n, 3, 16)
    for i in range(n):
        assert (hist[i] == oracle.hist16(want[i])).all()
        got = j.output_row(s_b, i).reshape(96, 128, 3)
        assert (got[1:-1, 1:-1] == oracle.blur(want[i], 3)[1:-1, 1:-1]).all()
    assert eng.stats()["counters"]["frames_delivered_nv12"] == 0


def test_nv12_elements_through_sampler_and_small_unaligned_frames(eng):
    """Stride sampler between source and Histogram keeps NV12 delivery; 200x112 (width % 16 != 0)
    takes the generic NV12 histogram kernel."""
    n, gop = 12, 3
    data, want = make_clip(32, n, 112, 200, gop)
    sid = eng.add_h264(data)
    g = E.Graph()
    src = g.add_source(True)
    smp = g.add_sample((src, "frame"))
    hs = g.add_op("Histogram", [(smp, "frame")], device=1)
    sink = g.add_sink((hs, "histogram"))
    j = E.Job()
    j.bind_source(src, sid)
    j.set_sampler(smp, "Strided", protolite.encode(protolite.SAMPLER_ARGS["StridedSamplerArgs"], {"stride": gop}))
    eng.run(g, [j], 2, 4)
    hist = j.output_array(sink, 192, np.int32).reshape(n // gop, 3, 16)
    for k in range(n // gop):
        assert (hist[k] == oracle.hist16(want[k * gop])).all()
    assert eng.stats()["counters"]["frames_delivered_nv12"] == n // gop


def test_c3_dag_blur_then_histogram(eng):
    n = 6
    data, want = make_clip(15, n, 480, 640, 3)
    sid = eng.add_h264(data)
    g = E.Graph()
    src = g.add_source(True)
    bl = g.add_op("Blur", [(src, "frame")], device=1,
                  args=protolite.encode(STD_ARGS["BlurArgs"], {"kernel_size": 3, "sigma": 0.5}))
    hs = g.add_op("Histogram", [(bl, "frame")], device=1)
    sink = g.add_sink((hs, "histogram"))
    j = E.Job()
    j.bind_source(src, sid)
    eng.run(g, [j], 3, 3)
    hist = j.output_array(sink, 192, np.int32).reshape(n, 3, 16)
    for i in range(n):
        assert (hist[i] == oracle.hist16(oracle.blur(want[i], 3))).all()


def test_blur_without_args_fails_validation(eng):
    g = E.Graph()
    src = g.add_source(True)
    g.add_sink((g.add_op("Blur", [(src, "frame")], device=1), "frame"))
    j = E.Job()
    j.bind_source(src, eng.add_raw_frames(np.zeros((2, 8, 8, 3), np.uint8)))
    with pytest.raises(E.EngineError, match="Could not parse BlurArgs"):
        eng.run(g, [j], 1, 1)


def test_raw_frames_host_to_device_marshalling(eng):
    """The reference's only GPU input path (host frames copied to the device per packet,
    runtime.cpp:141-189): RAW frame column -> GPU Histogram / Resize(preserve_aspect)."""
    n = 13
    frames = np.stack([synth.rand_frame(80 + i, 360, 640) for i in range(n)])
    sid = eng.add_raw_frames(frames)
    g = E.Graph()
    src = g.add_source(True)
    hs = g.add_op("Histogram", [(src, "frame")], device=1, batch=5)
    rz = g.add_op("Resize", [(src, "frame")], device=1)
    s_h, s_r = g.add_sink((hs, "histogram")), g.add_sink((rz, "frame"))
    j = E.Job()
    j.bind_source(src, sid)
    j.set_stream_args(rz, protolite.encode(STD_ARGS["ResizeArgs"], {"width": 0, "height": 90, "preserve_aspect": True}))
    eng.run(g, [j], 4, 8)
    hist = j.output_array(s_h, 192, np.int32).reshape(n, 3, 16)
    for i in range(n):
        assert (hist[i] == oracle.hist16(frames[i])).all()
        got = j.output_row(s_r, i)
        assert got.shape == (90, 160, 3) and (got == oracle.resize(frames[i], 160, 90)).all()


def test_no_device_memory_leaks(eng):
    data, want = make_clip(16, 14, 96, 128, 4)
    sid = eng.add_h264(data)
    g = E.Graph()
    src = g.add_source(True)
    bl = g.add_op("Blur", [(src, "frame")], device=1, args=protolite.encode(STD_ARGS["BlurArgs"], {"kernel_size": 3}))
    hs = g.add_op("Histogram", [(bl, "frame")], device=1)
    rz = g.add_op("Resize", [(src, "frame")], device=1)
    g.add_sink((hs, "histogram"))
    g.add_sink((rz, "frame"))
    j = E.Job()
    j.bind_source(src, sid)
    j.set_stream_args(rz, protolite.encode(STD_ARGS["ResizeArgs"], {"width": 32, "height": 24}))
    for _ in range(2):
        eng.run(g, [j], 3, 6)
        c = eng.stats()["counters"]
        assert c["gpu0_bytes_live"] == 0 and c["cpu_bytes_live"] == 0, c
        assert c["gpu0_bytes_peak"] >= 3 * 96 * 128 * 3


def test_many_clips_sharded_over_instances(eng):
    clips = [make_clip(100 + k, 12 + k, 96, 128, 4) for k in range(6)]
    g = E.Graph()
    src = g.add_source(True)
    hs = g.add_op("Histogram", [(src, "frame")], device=1)
    sink = g.add_sink((hs, "histogram"))
    jobs = []
    for data, _ in clips:
        j = E.Job()
        j.bind_source(src, eng.add_h264(data))
        jobs.append(j)
    eng.run(g, jobs, 4, 8)
    for (data, want), j in zip(clips, jobs):
        hist = j.output_array(sink, 192, np.int32).reshape(-1, 3, 16)
        assert len(hist) == len(want)
        for i in range(len(want)):
            assert (hist[i] == oracle.hist16(want[i])).all()
    assert eng.stats()["counters"]["instances"] == 3


def test_client_surface_on_gpu_like_tutorial_00():
    """The scannerpy-shaped API end to end on the GPU: H.264 in, Stride, GPU Histogram + Resize."""
    import scanner_b200 as sp
    data, want = make_clip(21, 24, 96, 128, 6)
    sc = sp.Client(gpus=[0], instances_per_gpu=2)
    video = sp.NamedVideoStream(sc, "clip", data=data)
    assert video.len() == 24
    frames = sc.io.Input([video])
    strided = sc.streams.Stride(frames, [3])
    hists = sc.ops.Histogram(frame=strided, device=sp.DeviceType.GPU)
    small = sc.ops.Resize(frame=strided, device=sp.DeviceType.GPU, width=[64], height=[48])
    o_h, o_r = sp.NamedStream(sc, "clip_hist"), sp.NamedStream(sc, "clip_small")
    sc.run([sc.io.Output(hists, [o_h]), sc.io.Output(small, [o_r])], sp.PerfParams.manual(4, 8))
    got = list(o_h.load())
    assert len(got) == 8
    for k, hist in enumerate(got):
        assert len(hist) == 3 and hist[0].shape[0] == 16
        assert (np.stack(hist) == oracle.hist16(want[3 * k])).all()
    for k, fr in enumerate(o_r.load()):
        assert (fr == oracle.resize(want[3 * k], 64, 48)).all()
    sc.stop()


def test_mp4_ingest_to_stored_histograms_through_the_database(tmp_path):
    """The whole path on disk formats: .mp4 file -> Client.ingest_videos (demux + index + video table)
    -> NVDEC decode from the stored stream -> GPU Histogram / Resize -> output tables -> a later
    session loads them.  Every value equals the oracle on the source planes."""
    import scanner_b200 as sp
    n, gop = 20, 5
    data, want = make_clip(41, n, 96, 128, gop)
    (tmp_path / "clip.mp4").write_bytes(E.mp4_mux(data, 30, 1))
    sc = sp.Client(gpus=[0], instances_per_gpu=2, db_path=str(tmp_path / "db"))
    done, failed = sc.ingest_videos([("clip", str(tmp_path / "clip.mp4"))])
    assert not failed and done[0].len() == n
    frames = sc.io.Input([sp.NamedVideoStream(sc, "clip")])
    gathered = sc.streams.Gather(frames, [[1, 4, 5, 13, 19]])
    hists = sc.ops.Histogram(frame=gathered, device=sp.DeviceType.GPU)
    small = sc.ops.Resize(frame=gathered, device=sp.DeviceType.GPU, width=[32], height=[24])
    o_h, o_r = sp.NamedStream(sc, "clip_hist"), sp.NamedStream(sc, "clip_small")
    sc.run([sc.io.Output(hists, [o_h]), sc.io.Output(small, [o_r])], sp.PerfParams.manual(2, 4))
    assert sc.stats()["counters"]["frames_delivered_nv12"] == 5
    sc.stop()
    sc2 = sp.Client(gpus=[], cpu_instances=1, db_path=str(tmp_path / "db"), load_stdlib=False)
    assert sorted(sc2.table_names()) == ["clip", "clip_hist", "clip_small"]
    hist = list(sp.NamedStream(sc2, "clip_hist").load())
    small = list(sp.NamedStream(sc2, "clip_small").load())
    assert len(hist) == len(small) == 5
    for k, row in enumerate([1, 4, 5, 13, 19]):
        assert (np.stack(hist[k]) == oracle.hist16(want[row])).all()
        assert (small[k] == oracle.resize(want[row], 32, 24)).all()
    sc2.stop()


def test_decode_to_device_matches_engine_path(eng):
    data, want = make_clip(31, 20, 96, 128, 6)
    sid = eng.add_h264(data)
    rows = [0, 1, 5, 6, 7, 13, 19]
    got = eng.decode_to_device(sid, rows, 0)
    assert got.shape == (len(rows), 96, 128, 3) and got.is_cuda
    for k, r in enumerate(rows):
        assert (got[k].cpu().numpy() == want[r]).all()
    with pytest.raises(E.EngineError, match="ascending"):
        eng.decode_to_device(sid, [3, 2], 0)


def test_single_rank_sharded_flow_equals_direct():
    """halo.sharded_optical_flow with world size 1 == decode + optical_flow with the edge repeated."""
    from scanner_b200 import halo
    data, want = make_clip(32, 6, 96, 128, 3)
    e = E.Engine(gpus=[0])
    sid = e.add_h264(data)
    a, flows = halo.sharded_optical_flow(e, sid, 0)
    assert a == 0 and flows.shape == (6, 96, 128, 2)
    for i in range(6):
        ref = oracle.optical_flow(want[i], want[min(i + 1, 5)])
        d = np.abs(flows[i].cpu().numpy() - ref)
        assert np.quantile(d, 0.999) <= 5e-2 and d.mean() <= 1e-3   # uniform-noise frames: ill-conditioned
    e.close()


def test_random_gathers_across_gops_both_element_layouts(eng):
    """Random row subsets (seeks into the middle of GOPs, adjacent GOPs, the last frame) over two clips
    at once, the sampled frames going both to a frame sink (which keeps the column RGB24 for every
    consumer) and to Histogram: both equal the oracle on the source planes."""
    rng = np.random.default_rng(99)
    clips = [make_clip(50 + k, 45, 96, 128, 7) for k in range(2)]
    sids = [eng.add_h264(c[0]) for c in clips]
    g = E.Graph()
    src = g.add_source(True)
    smp = g.add_sample((src, "frame"))
    hs = g.add_op("Histogram", [(smp, "frame")], device=1)
    s_f = g.add_sink((smp, "frame"))
    s_h = g.add_sink((hs, "histogram"))
    for trial in range(4):
        jobs, picks = [], []
        for sid in sids:
            rows = sorted(set(int(x) for x in rng.integers(0, 45, int(rng.integers(1, 20)))) | ({44} if trial == 0 else set()))
            j = E.Job()
            j.bind_source(src, sid)
            j.set_sampler(smp, "Gather", protolite.encode(protolite.SAMPLER_ARGS["GatherSamplerArgs"], {"rows": rows}))
            jobs.append(j)
            picks.append(rows)
        eng.run(g, jobs, 2, 4)
        for (data, want), rows, j in zip(clips, picks, jobs):
            assert j.output_rows(s_f) == len(rows)
            hist = j.output_array(s_h, 192, np.int32).reshape(len(rows), 3, 16)
            for k, r in enumerate(rows):
                assert (j.output_row(s_f, k) == want[r]).all(), (trial, r)
                assert (hist[k] == oracle.hist16(want[r])).all(), (trial, r)


@pytest.mark.parametrize("h,w,n,gop,mv", [(96, 128, 12, 5, (2, -2)), (1080, 1920, 9, 4, (-4, 6)), (270, 480, 10, 10, (0, 2))])
def test_decode_cavlc_intra_and_motion_compensated_pictures_bit_exact(eng, h, w, n, gop, mv):
    """Streams a real encoder could have produced (scanner_b200/synth_h264.py: Intra16x16 DC prediction +
    CAVLC residuals, P_L0_16x16 macroblocks with a motion vector) through the indexer and NVDEC: every
    picture equals the writer's integer model of the decoder -- the same model FFmpeg is held to on the CPU
    (tests/test_storage_cpu.py).  Histogram / Gather rows on such a stream are checked too."""
    from scanner_b200 import synth_h264
    data, yuv = synth_h264.write(w, h, n, gop=gop, seed=h + w, mv=mv)
    sid = eng.add_h264(data)
    info = eng.stream_info(sid)
    assert (info["width"], info["height"]) == (w, h) and eng.stream_rows(sid) == n
    assert info["keyframes"] == (n + gop - 1) // gop
    want = []
    for i in range(n):
        y = yuv[i, :h * w].reshape(h, w)
        chroma = np.empty((h // 2, w), np.uint8)
        chroma[:, 0::2] = yuv[i, h * w:h * w * 5 // 4].reshape(h // 2, w // 2)
        chroma[:, 1::2] = yuv[i, h * w * 5 // 4:].reshape(h // 2, w // 2)
        want.append(oracle.nv12_to_rgb(y, chroma))
    g = E.Graph()
    src = g.add_source(True)
    sink = g.add_sink((src, "frame"))
    hs = g.add_op("Histogram", [(src, "frame")], device=1)
    sink_h = g.add_sink((hs, "histogram"))
    j = E.Job()
    j.bind_source(src, sid)
    for (wps, ios) in [(4, 8), (1, 1)]:
        eng.run(g, [j], wps, ios)
        assert j.output_rows(sink) == n
        for i in range(n):
            got = j.output_row(sink, i)
            assert (got == want[i]).all(), (i, wps, ios, np.abs(got.astype(int) - want[i]).max())
            assert (np.frombuffer(j.output_row(sink_h, i), np.int32).reshape(3, 16) == oracle.hist16(want[i])).all()
    # seeking into the middle of a GOP decodes from its IDR through the motion-compensated pictures
    g2 = E.Graph()
    src2 = g2.add_source(True)
    s2 = g2.add_sample((src2, "frame"))
    sink2 = g2.add_sink((s2, "frame"))
    rows = sorted({n - 1, gop + 1 if gop + 1 < n else 0})
    j2 = E.Job()
    j2.bind_source(src2, sid)
    j2.set_sampler(s2, "Gather", protolite.encode(protolite.SAMPLER_ARGS["GatherSamplerArgs"], {"rows": rows}))
    eng.run(g2, [j2], 2, 2)
    for k, r in enumerate(rows):
        assert (j2.output_row(sink2, k) == want[r]).all(), r
