"""JPEG output of ImageEncoder on the GPU: scn_jpeg_encode_u8 and the op's GPU kernel, byte for byte against the
oracle (oracle/jpeg.py, itself held to cv2.imencode in tests/test_jpeg_cpu.py) and against live cv2.  Also the
reference's tutorial 05_sources_sinks.py, replayed with the import changed and the two image ops placed on the
GPU."""
import os

import cv2
import numpy as np
import pytest
import torch

import oracle
import scanner_b200 as sp
from oracle import jpeg as J
from scanner_b200 import cabi, kernels
from scanner_b200 import engine as E

pytestmark = pytest.mark.gpu


def _check(frames, quality, got):
    assert len(got) == len(frames)
    for i, (f, g) in enumerate(zip(frames, got)):
        f = np.asarray(f)
        want = J.encode(f, quality)
        assert g == want, (i, f.shape, quality, len(g), len(want))
        assert g == J.cv2_encode(f, quality), i
        h, w, c = f.shape
        assert len(g) <= kernels.jpeg_encode_bound(w, h, c)


# ---- kernel level -----------------------------------------------------------------------------------------------
def test_the_sweep_equals_the_oracle():
    for name, frame, q in J.sweep():
        got = kernels.jpeg_encode(torch.from_numpy(frame[None]).cuda(), q)
        assert got[0] == J.encode(frame, q), name
        assert got[0] == J.cv2_encode(frame, q), name


@pytest.mark.parametrize("h,w", [(1080, 1920), (2160, 3840)])
@pytest.mark.parametrize("kind", ["noise", "smooth"])
def test_full_hd_and_4k_frames(h, w, kind):
    from oracle import synth
    frame = J.content("noise", h, w, 3, h) if kind == "noise" else synth.smooth_frame(h, h, w)
    gray = np.ascontiguousarray(frame[..., 1:2])
    for f, q in ((frame, 95), (gray, 90)):
        got = kernels.jpeg_encode(torch.from_numpy(f[None]).cuda(), q)
        _check([f], q, got)
        if kind == "noise":
            assert got[0][600:].count(b"\xff\x00") > 1000  # the stuffing path ran


@pytest.mark.parametrize("n", [65, 130])
def test_batches_over_64_frames(n):
    rng = np.random.default_rng(n)
    frames = rng.integers(0, 256, (n, 37, 53, 3), dtype=np.uint8)
    frames[::3] //= 16  # smoother frames too: sizes differ between frames
    _check(frames, 75, kernels.jpeg_encode(torch.from_numpy(frames).cuda(), 75))
    gray = np.ascontiguousarray(frames[..., :1])
    _check(gray, 50, kernels.jpeg_encode(torch.from_numpy(gray).cuda(), 50))


def test_runs_of_mixed_geometry_in_one_list():
    rng = np.random.default_rng(3)
    shapes = [(24, 40, 3), (24, 40, 3), (9, 70, 3), (24, 40, 3), (31, 17, 1), (31, 17, 1), (1, 1, 3)]
    frames = [rng.integers(0, 256, s, dtype=np.uint8) for s in shapes]
    _check(frames, 95, kernels.jpeg_encode([torch.from_numpy(f).cuda() for f in frames], 95))


@pytest.mark.parametrize("c", [3, 1])
def test_frames_at_odd_base_offsets(c):
    rng = np.random.default_rng(c)
    h, w = 21, 35
    buf = torch.from_numpy(rng.integers(0, 256, 8 * h * w * c + 64, dtype=np.uint8)).cuda()
    offs = [1, 3 + 2 * h * w * c, 5 + 4 * h * w * c, 7 + 6 * h * w * c]
    views = [buf[o:o + h * w * c].view(h, w, c) for o in offs]
    assert all(v.data_ptr() % 2 == 1 for v in views)
    frames = [v.cpu().numpy() for v in views]
    _check(frames, 85, kernels.jpeg_encode(views, 85))
    # a dense batch whose frames are only byte-aligned (odd W * C)
    dense = buf[1:1 + 5 * h * w * c].view(5, h, w, c)
    _check(dense.cpu().numpy(), 30, kernels.jpeg_encode(dense, 30))


def test_refusals_launch_nothing():
    L = cabi.lib()
    before = L.scn_launch_count()
    for shape in [(1, 8, 8, 2), (1, 8, 8, 4)]:
        with pytest.raises(cabi.ScnError, match="argument error -2"):
            kernels.jpeg_encode(torch.zeros(shape, dtype=torch.uint8, device="cuda"))
    with pytest.raises(cabi.ScnError, match="argument error -1"):
        kernels.jpeg_encode(torch.zeros((1, 8, 8, 3), dtype=torch.uint8, device="cuda"), quality=0)
    assert L.scn_launch_count() == before


# ---- op level ---------------------------------------------------------------------------------------------------
@pytest.fixture()
def sc(tmp_path):
    c = sp.Client(db_path=str(tmp_path / "scanner_db"))
    yield c
    c.stop()


def _encode_op(sc, frames, name, **kw):
    inp = sc.io.Input([sp.NamedVideoStream(sc, name, frames=frames)])
    enc = sc.ops.ImageEncoder(frame=inp, device=sp.DeviceType.GPU, **kw)
    out = sp.NamedStream(sc, name + "_jpg")
    sc.run(sc.io.Output(enc, [out]), sp.PerfParams.manual(8, 16))
    return list(out.load())


def test_op_encodes_host_frames_with_default_and_given_quality(sc):
    rng = np.random.default_rng(11)
    frames = rng.integers(0, 256, (20, 45, 61, 3), dtype=np.uint8)
    frames[::2] //= 8
    _check(frames, 95, _encode_op(sc, frames, "rgb", format="jpg"))
    _check(frames, 40, _encode_op(sc, frames, "rgb40", format="jpeg", quality=40))
    gray = np.ascontiguousarray(frames[:5, ..., :1])
    _check(gray, 100, _encode_op(sc, gray, "gray", format="JPEG", quality=100))


def test_png_on_the_gpu_kernel_equals_the_cpu_kernel(sc):
    rng = np.random.default_rng(12)
    frames = rng.integers(0, 256, (6, 30, 41, 3), dtype=np.uint8)
    gpu = _encode_op(sc, frames, "png_gpu", format="png")
    inp = sc.io.Input([sp.NamedVideoStream(sc, "png_cpu", frames=frames)])
    out = sp.NamedStream(sc, "png_cpu_out")
    sc.run(sc.io.Output(sc.ops.ImageEncoder(frame=inp, format="png"), [out]), sp.PerfParams.manual(8, 16))
    cpu = list(out.load())
    assert len(gpu) == 6 and gpu == cpu
    assert (cv2.imdecode(np.frombuffer(gpu[2], np.uint8), cv2.IMREAD_UNCHANGED)[..., ::-1] == frames[2]).all()


@pytest.mark.parametrize("shape,dtype,why", [((4, 8, 8, 2), np.uint8, "got 2 channels"),
                                             ((4, 8, 8, 4), np.uint8, "got 4 channels"),
                                             ((4, 8, 8, 3), np.uint16, "needs uint8 frames")])
def test_unsupported_frames_fail_the_run_and_the_engine_goes_on(sc, shape, dtype, why):
    bad = np.zeros(shape, dtype)
    with pytest.raises(sp.ScannerException, match=r"ImageEncoder, row 0: JPEG .*" + why):
        _encode_op(sc, bad, "bad", format="jpg")
    good = np.full((3, 8, 8, 3), 77, np.uint8)
    _check(good, 95, _encode_op(sc, good, "good", format="jpg"))


def test_bad_quality_and_format_fail_validation(sc):
    frames = np.zeros((2, 8, 8, 3), np.uint8)
    with pytest.raises(sp.ScannerException, match=r"quality 101 is outside \[1, 100\]"):
        _encode_op(sc, frames, "q", format="jpg", quality=101)
    with pytest.raises(sp.ScannerException, match="Valid types are: png, jpg"):
        _encode_op(sc, frames, "f", format="webp")


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


def test_decoded_clip_feeds_histogram_and_the_encoder(sc, tmp_path):
    data, shown = _clip(21, 18, 144, 176, 6)
    path = str(tmp_path / "clip.mp4")
    open(path, "wb").write(E.mp4_mux(data, 24, 1))
    frames = sc.io.Input([sp.NamedVideoStream(sc, "clip", path=path)])
    hists = sc.ops.Histogram(frame=frames)
    jpgs = sc.ops.ImageEncoder(frame=frames, format="jpg", quality=90, device=sp.DeviceType.GPU)
    h_out, j_out = sp.NamedStream(sc, "clip_hist"), sp.NamedStream(sc, "clip_jpg")
    sc.run([sc.io.Output(hists, [h_out]), sc.io.Output(jpgs, [j_out])], sp.PerfParams.manual(8, 16))
    hs, js = list(h_out.load()), list(j_out.load())
    assert len(hs) == len(js) == len(shown)
    for i, f in enumerate(shown):
        assert (np.stack(hs[i]) == oracle.hist16(f)).all(), i
    _check(shown, 90, js)


# ---- tutorial 05_sources_sinks.py ------------------------------------------------------------------------------
def test_05_sources_sinks(sc, tmp_path):
    from oracle import synth
    rng = np.random.default_rng(5)
    image_paths = []
    for i, (h, w) in enumerate([(480, 720), (360, 500), (533, 800)]):  # the tutorial's downloaded images
        img = synth.smooth_frame(50 + i, h, w)
        img = np.clip(img.astype(np.int32) + rng.integers(-6, 7, img.shape), 0, 255).astype(np.uint8)
        p = str(tmp_path / f"sample-frame-{i + 1}.jpg")
        assert cv2.imwrite(p, img[..., ::-1])
        image_paths.append(p)

    # -- the tutorial, with the two image ops placed on the GPU --
    image_stream = sp.FilesStream(image_paths)
    compressed_images = sc.io.Input([image_stream])
    frames = sc.ops.ImageDecoder(img=compressed_images, device=sp.DeviceType.GPU)
    resized_frames = sc.ops.Resize(frame=frames, width=[640], height=[360])
    encoded_frames = sc.ops.ImageEncoder(frame=resized_frames, format='jpg', device=sp.DeviceType.GPU)
    resized_paths = [str(tmp_path / f"resized-{i}.jpg") for i in (1, 2, 3)]
    resized_stream = sp.FilesStream(resized_paths)
    output = sc.io.Output(encoded_frames, [resized_stream])
    sc.run(output, sp.PerfParams.estimate(), cache_mode=sp.CacheMode.Overwrite)

    # -- what it wrote: cv2.imencode of the oracle resize of the frames the GPU decoder gives (one run per
    # image: the frames of one stored item share a shape) --
    shown = []
    for i, p in enumerate(image_paths):
        decoded = sc.ops.ImageDecoder(img=sc.io.Input([sp.FilesStream([p])]), device=sp.DeviceType.GPU)
        dec_out = sp.NamedVideoStream(sc, f"decoded{i}")
        sc.run(sc.io.Output(decoded, [dec_out]), sp.PerfParams.estimate())
        shown += list(dec_out.load())
    assert len(shown) == 3
    for p, f in zip(resized_paths, shown):
        assert os.path.exists(p)
        want = J.cv2_encode(oracle.resize(f, 640, 360), 95)
        assert open(p, "rb").read() == want == J.encode(oracle.resize(f, 640, 360), 95)
