"""ConvertColor on the GPU, byte for byte against the numpy restatement of cv::cvtColor (oracle/convert_color.py,
itself held to cv2 on all 2^24 RGB triples by tests/test_convert_color_cpu.py):
  * scn_convert_color_u8 on the image of all 2^24 triples, for every code;
  * batches over 64 frames, runs of mixed geometry, odd widths and unaligned frame bases, over outputs pre-filled
    with 0 and with 255 so that a byte never written cannot pass;
  * scn_convert_color_nv12 against scn_nv12_to_rgb24 (pinned to the reference's own kernel by test_ref_pin_gpu.py)
    followed by scn_convert_color_u8;
  * the ConvertColor op through the engine, with NV12 and with RGB24 decode elements, next to Histogram;
  * its errors, and the reference's grayscale walkthrough replayed through the client.
"""
import ctypes

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import oracle  # noqa: E402
import scanner_b200 as sp  # noqa: E402
from oracle import convert_color as C  # noqa: E402
from oracle import synth  # noqa: E402
from scanner_b200 import cabi, kernels  # noqa: E402
from scanner_b200 import engine as E  # noqa: E402

pytestmark = pytest.mark.gpu

CODES = list(C.CODES)
RGB_CODES = [c for c in CODES if C.CODES[c][0] == 3]


def _code(name):
    return cabi.lib().scn_convert_color_code(name.encode())


def _convert_into(srcs, dsts, w, h, code):
    """scn_convert_color_u8 from the CUDA tensors (or raw device addresses) `srcs` into `dsts`."""
    addr = lambda t: t if isinstance(t, int) else t.data_ptr()  # noqa: E731
    sp_, k1 = cabi.ptr_array([addr(t) for t in srcs])
    dp, k2 = cabi.ptr_array([addr(t) for t in dsts])
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    cabi.check(cabi.lib().scn_convert_color_u8(sp_, len(srcs), w, h, _code(code), dp, stream), "scn_convert_color_u8")


@pytest.fixture(scope="module")
def triples():
    return C.all_triples()


@pytest.mark.parametrize("code", CODES)
def test_all_rgb_triples_equal_the_oracle(code, triples):
    src = triples if C.CODES[code][0] == 3 else np.ascontiguousarray(triples[..., :1])
    got = kernels.convert_color(torch.from_numpy(src).cuda()[None], code)[0]
    want = C.convert_color(src, code)
    assert got.shape == want.shape
    assert torch.equal(got, torch.from_numpy(want).cuda())


@pytest.mark.parametrize("fill", [0, 255])
@pytest.mark.parametrize("n", [65, 130])
@pytest.mark.parametrize("code", ["COLOR_RGB2GRAY", "COLOR_BGR2HSV", "COLOR_GRAY2RGB"])
def test_batches_over_64_frames_into_prefilled_outputs(code, n, fill):
    cin, cout = C.CODES[code]
    h, w = 21, 35  # 735 pixels: frame i of the dense batch starts at i * 735 * C bytes, mostly unaligned
    src = np.random.default_rng(n).integers(0, 256, (n, h, w, cin), dtype=np.uint8)
    d_src = torch.from_numpy(src).cuda()
    out = torch.full((n, h, w, cout), fill, dtype=torch.uint8, device="cuda")
    _convert_into(list(d_src), list(out), w, h, code)
    assert (out.cpu().numpy() == C.convert_color(src, code)).all()


@pytest.mark.parametrize("fill", [0, 255])
@pytest.mark.parametrize("w", [1, 3, 17, 4095])
@pytest.mark.parametrize("code", ["COLOR_BGR2GRAY", "COLOR_RGB2YCrCb", "COLOR_RGB2HSV_FULL", "COLOR_BGR2RGB",
                                  "COLOR_GRAY2BGR"])
def test_narrow_and_odd_widths_at_every_base_alignment(code, w, fill):
    """Frames of a dense batch at offsets 1..16 bytes into the allocation, outputs at offset 0: the source and
    destination reach 16-byte alignment at the same pixel only when the two offsets agree mod 16, else the
    frame goes pixel by pixel.  Each frame's output sits between guard bytes that must stay untouched."""
    cin, cout = C.CODES[code]
    h, n = 5, 7
    src = np.random.default_rng(w).integers(0, 256, (n, h, w, cin), dtype=np.uint8)
    want = C.convert_color(src, code)
    fb_in, fb_out = h * w * cin, h * w * cout
    for off in range(1, 17):
        d_in = torch.zeros(off + n * fb_in, dtype=torch.uint8, device="cuda")
        d_in[off:] = torch.from_numpy(src.reshape(-1)).cuda()
        d_out = torch.full((n * fb_out + 64,), fill, dtype=torch.uint8, device="cuda")
        _convert_into([d_in.data_ptr() + off + i * fb_in for i in range(n)],
                      [d_out.data_ptr() + i * fb_out for i in range(n)], w, h, code)
        got = d_out.cpu().numpy()
        assert (got[:n * fb_out].reshape(want.shape) == want).all(), off
        assert (got[n * fb_out:] == fill).all(), off


def test_runs_of_mixed_geometry_in_one_list():
    rng = np.random.default_rng(3)
    shapes = [(48, 64), (48, 64), (17, 33), (48, 64), (1, 1), (1, 1), (1080, 1920)]
    frames = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]
    for code in RGB_CODES:
        got = kernels.convert_color([torch.from_numpy(f).cuda() for f in frames], code)
        assert len(got) == len(frames)
        for g, f in zip(got, frames):
            assert (g.cpu().numpy() == C.convert_color(f, code)).all(), (code, f.shape)


def _nv12_then_u8(surf, w, h, code):
    return kernels.convert_color(kernels.nv12_to_rgb(surf, w, h), code)


@pytest.mark.parametrize("code", RGB_CODES)
def test_nv12_path_equals_nv12_to_rgb_then_convert_on_all_yuv_triples(code):
    w, h = synth.EXH_W, synth.EXH_H
    for f0 in range(0, synth.EXH_FRAMES, 16):
        surf = np.stack([np.concatenate(synth.nv12_exhaustive(f), 0) for f in range(f0, f0 + 16)])
        d = torch.from_numpy(surf).cuda()
        assert torch.equal(kernels.convert_color(d, code, w, h), _nv12_then_u8(d, w, h, code)), f0


@pytest.mark.parametrize("fill", [0, 255])
@pytest.mark.parametrize("h,w,pitch", [(270, 480, 480), (270, 480, 512), (90, 136, 160), (6, 34, 34), (2, 2, 2)])
def test_nv12_path_on_seeded_surfaces_of_odd_chroma_height(h, w, pitch, fill):
    """h / 2 odd: the last chroma row has no partner; w % 16 != 0 or pitch > w take the per-pixel path."""
    n = 66
    surf = np.zeros((n, h * 3 // 2, pitch), np.uint8)
    for i in range(n):
        luma, chroma = synth.nv12_surface(500 + i, h, w, pitch)
        surf[i, :h], surf[i, h:] = luma, chroma
    d = torch.from_numpy(surf).cuda()
    lum, chr_, _ = kernels._surface_ptrs(d, h)
    for code in RGB_CODES:
        cout = C.CODES[code][1]
        out = torch.full((n, h, w, cout), fill, dtype=torch.uint8, device="cuda")
        lp, k1 = cabi.ptr_array(lum)
        cp, k2 = cabi.ptr_array(chr_)
        op, k3 = cabi.ptr_array([out.data_ptr() + i * h * w * cout for i in range(n)])
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        cabi.check(cabi.lib().scn_convert_color_nv12(lp, cp, pitch, n, w, h, _code(code), op, stream), "nv12")
        assert torch.equal(out, _nv12_then_u8(d, w, h, code)), code


# ---- through the engine ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def std_args():
    import os
    from scanner_b200 import protolite
    E.load_stdlib()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return protolite.parse_proto(open(os.path.join(root, "scanner_b200", "csrc", "ops", "stdlib_args.proto")).read())


def _clip(seed, n, h, w, gop):
    """-> (H.264 bytes of I_PCM pictures, the RGB frames a decoder shows for them)"""
    rng = np.random.default_rng(seed)
    y = rng.integers(0, 256, (n, h, w), dtype=np.uint8)
    u = rng.integers(0, 256, (n, h // 2, w // 2), dtype=np.uint8)
    v = rng.integers(0, 256, (n, h // 2, w // 2), dtype=np.uint8)
    yuv = np.concatenate([y.reshape(n, -1), u.reshape(n, -1), v.reshape(n, -1)], axis=1)
    rgb = []
    for i in range(n):
        chroma = np.empty((h // 2, w), np.uint8)
        chroma[:, 0::2], chroma[:, 1::2] = u[i], v[i]
        rgb.append(oracle.nv12_to_rgb(y[i], chroma))
    return E.h264_synth(yuv, w, h, gop=gop), np.stack(rgb)


def _run_convert(std_args, data, code, with_hist):
    from scanner_b200 import protolite
    eng = E.Engine(gpus=[0], instances_per_gpu=2)
    try:
        sid = eng.add_h264(data)
        g = E.Graph()
        src = g.add_source(True)
        cc = g.add_op("ConvertColor", [(src, "frame")], device=1)
        s_c = g.add_sink((cc, "frame"))
        s_h = g.add_sink((g.add_op("Histogram", [(src, "frame")], device=1), "histogram")) if with_hist else None
        j = E.Job()
        j.bind_source(src, sid)
        j.set_stream_args(cc, protolite.encode(std_args["ConvertColorArgs"], {"conversion": code}))
        eng.run(g, [j], 4, 8)
        frames = [j.output_row(s_c, i) for i in range(j.output_rows(s_c))]
        hist = j.output_array(s_h, 192, np.int32).reshape(-1, 3, 16) if with_hist else None
        return frames, hist, eng.stats()["counters"]["frames_delivered_nv12"]
    finally:
        eng.close()


@pytest.mark.parametrize("code", ["COLOR_RGB2GRAY", "COLOR_BGR2YCrCb", "COLOR_RGB2HSV"])
def test_op_gives_the_same_bytes_from_nv12_and_from_rgb24_elements(std_args, code, monkeypatch):
    n, h, w = 10, 360, 640
    data, shown = _clip(21, n, h, w, 5)
    monkeypatch.delenv("SCN_DECODE_RGB", raising=False)
    nv12, _, delivered = _run_convert(std_args, data, code, False)
    assert delivered == n
    monkeypatch.setenv("SCN_DECODE_RGB", "1")
    rgb, _, delivered = _run_convert(std_args, data, code, False)
    assert delivered == 0
    assert len(nv12) == len(rgb) == n
    for i in range(n):
        want = C.convert_color(shown[i], code)
        assert nv12[i].shape == want.shape and (nv12[i] == want).all() and (rgb[i] == want).all(), i


def test_histogram_keeps_its_nv12_path_and_results_next_to_convert_color(std_args, monkeypatch):
    monkeypatch.delenv("SCN_DECODE_RGB", raising=False)
    n, h, w = 8, 270, 480
    data, shown = _clip(22, n, h, w, 4)
    gray, hist, delivered = _run_convert(std_args, data, "COLOR_RGB2GRAY", True)
    assert delivered == n
    for i in range(n):
        assert (hist[i] == oracle.hist16(shown[i])).all()
        assert (gray[i] == C.convert_color(shown[i], "COLOR_RGB2GRAY")).all()


# ---- through the client -----------------------------------------------------------------------------------------
@pytest.fixture()
def sc(tmp_path):
    c = sp.Client(db_path=str(tmp_path / "scanner_db"))
    yield c
    c.stop()


def test_unknown_code_fails_the_run_naming_it(sc):
    frames = sc.io.Input([sp.NamedVideoStream(sc, "raw", frames=np.zeros((3, 8, 8, 3), np.uint8))])
    out = sp.NamedVideoStream(sc, "lab")
    with pytest.raises(sp.ScannerException, match=r"'COLOR_RGB2Lab'.*supported: COLOR_RGB2GRAY"):
        sc.run(sc.io.Output(sc.ops.ConvertColor(frame=frames, conversion=["COLOR_RGB2Lab"]), [out]),
               sp.PerfParams.estimate())


def test_wrong_channel_count_fails_the_run_and_the_process_survives(sc):
    rgb = np.random.default_rng(5).integers(0, 256, (4, 6, 10, 3), dtype=np.uint8)
    frames = sc.io.Input([sp.NamedVideoStream(sc, "rgb", frames=rgb)])
    with pytest.raises(sp.ScannerException, match=r"COLOR_GRAY2RGB takes 1-channel frames, got 3 channels"):
        sc.run(sc.io.Output(sc.ops.ConvertColor(frame=frames, conversion=["COLOR_GRAY2RGB"]),
                            [sp.NamedVideoStream(sc, "bad")]), sp.PerfParams.estimate())
    # the same client goes on: gray and back
    frames = sc.io.Input([sp.NamedVideoStream(sc, "rgb")])
    gray = sc.ops.ConvertColor(frame=frames, conversion=["COLOR_RGB2GRAY"])
    back = sc.ops.ConvertColor(frame=gray, conversion=["COLOR_GRAY2RGB"])
    out = sp.NamedVideoStream(sc, "good")
    sc.run(sc.io.Output(back, [out]), sp.PerfParams.estimate())
    got = list(out.load())
    assert len(got) == 4
    for i in range(4):
        assert (got[i] == C.convert_color(C.convert_color(rgb[i], "COLOR_RGB2GRAY"), "COLOR_GRAY2RGB")).all()


W, H, FRAMES, GOP = 320, 240, 24, 6


@pytest.fixture(scope="module")
def sample_clip(tmp_path_factory):
    """-> (path of a synthetic .mp4, the frames a decoder shows for it)"""
    data, shown = _clip(40, FRAMES, H, W, GOP)
    path = str(tmp_path_factory.mktemp("video") / "sample-clip.mp4")
    open(path, "wb").write(E.mp4_mux(data, 24, 1))
    return path, shown


@sp.register_python_op()
def CloneChannels(config, frame: sp.FrameType) -> sp.FrameType:
    return np.dstack([frame for _ in range(config.args['replications'])])


def test_grayscale_walkthrough(sc, sample_clip, tmp_path):
    """examples/apps/walkthroughs/grayscale_conversion.py with the clip replaced by a synthetic one."""
    import cv2
    path, shown = sample_clip
    input_stream = sp.NamedVideoStream(sc, 'sample-clip', path=path)
    frames = sc.io.Input([input_stream])
    sampled_frames = sc.streams.Stride(frames, [2])
    resized_frames = sc.ops.Resize(frame=sampled_frames, width=[640], height=[480])
    grayscale_frames = sc.ops.ConvertColor(frame=resized_frames, conversion=['COLOR_RGB2GRAY'])
    grayscale3_frames = sc.ops.CloneChannels(frame=grayscale_frames, replications=3)
    output_stream = sp.NamedVideoStream(sc, 'sample-grayscale')
    output = sc.io.Output(grayscale3_frames, [output_stream])
    sc.run(output, sp.PerfParams.manual(50, 250))
    saved = output_stream.save_mp4(str(tmp_path / 'sample-grayscale'))

    got = list(output_stream.load())
    assert len(got) == FRAMES // 2
    for k, frame in enumerate(got):
        gray = cv2.cvtColor(oracle.resize(shown[2 * k], 640, 480), cv2.COLOR_RGB2GRAY)
        assert frame.shape == (480, 640, 3) and (frame == np.dstack([gray] * 3)).all(), k
    cap = cv2.VideoCapture(saved)
    assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == FRAMES // 2
    ok, first = cap.read()
    assert ok and first.shape == (480, 640, 3)
    input_stream.delete(sc)
    output_stream.delete(sc)
