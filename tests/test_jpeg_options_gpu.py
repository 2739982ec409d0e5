"""cv2's JPEG options (sampling factor, optimised Huffman tables, luma and chroma quality) on the GPU: scn_jpeg_encode_u8_opts and the
ImageEncoder op's GPU kernel, byte for byte against the options oracle (tests/helpers/jpeg_options.py, itself held
to cv2.imencode in tests/test_jpeg_options_cpu.py) and against live cv2:
  * the sweep: every residue of W and H mod each mode's MCU, content kinds, qualities, the luma / chroma pairs;
  * 1080p and 2160p noise and smooth frames in every mode;
  * sides of 65,500 in every mode, within the bound for those options;
  * batches of 65 and 130 frames, frames at odd base offsets;
  * outputs pre-filled with 0x00 and 0xFF and followed by guard bytes, back-to-back calls on dirty scratch;
  * optimised tables: 1080p and 2160p in every mode, batches of 65 and 130 whose neighbouring frames get different
    tables and header lengths, the table kernel on synthetic frequencies against the oracle's builder;
  * the op with each option, and its refusals failing the run before anything is written."""
import ctypes

import numpy as np
import pytest
import torch

import scanner_b200 as sp
from helpers import guarded_output
from helpers import jpeg_options as O
from oracle import jpeg as J
from scanner_b200 import cabi, kernels

pytestmark = pytest.mark.gpu

MODES = tuple(O.SAMPLING)


def encode_raw(frames, quality, fill, **opts):
    """scn_jpeg_encode_u8_opts of equal-shape frames into an output pre-filled with `fill` and followed by guard
    bytes -> the files."""
    frames = [np.ascontiguousarray(f) for f in frames]
    h, w = frames[0].shape[:2]
    c = 1 if frames[0].ndim == 2 else frames[0].shape[2]
    dev = [torch.from_numpy(f).cuda() for f in frames]
    pp, _keep = cabi.ptr_array([t.data_ptr() for t in dev])
    o = kernels._jpeg_options(opts.get("sampling"), opts.get("luma_quality", 0), opts.get("chroma_quality", 0),
                              opts.get("optimize", False))
    L = cabi.lib()
    return guarded_output.encode_raw("scn_jpeg_encode_u8_opts", len(frames), fill, lambda cb, sizes, stream:
                                     L.scn_jpeg_encode_u8_opts(pp, len(frames), w, h, c, quality, ctypes.byref(o), cb,
                                                               None, sizes, stream))


def check(frames, quality, got, cv2=True, **opts):
    assert len(got) == len(frames)
    for i, (f, g) in enumerate(zip(frames, got)):
        f = np.asarray(f)
        want = O.encode(f, quality, **opts)
        assert g == want, (i, f.shape, quality, opts, len(g), len(want))
        if cv2:
            assert g == O.cv2_encode(f, quality, **opts), (i, f.shape, quality, opts)
        h, w = f.shape[:2]
        c = 1 if f.ndim == 2 else f.shape[2]
        assert len(g) <= kernels.jpeg_encode_bound(w, h, c, **opts)


# ---- kernel level -----------------------------------------------------------------------------------------------
def test_the_sweep_equals_the_oracle_and_cv2():
    for i, (name, frame, q, opts) in enumerate(O.sweep()):
        if i % 3 == 0:
            got = encode_raw([frame], q, 0xFF if i & 1 else 0x00, **opts)[0]
        else:
            got = kernels.jpeg_encode(torch.from_numpy(frame[None]).cuda(), q, **opts)[0]
        assert got == O.encode(frame, q, **opts), name
        assert got == O.cv2_encode(frame, q, **opts), name


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("h,w", [(1080, 1920), (2160, 3840)])
@pytest.mark.parametrize("kind", ["noise", "smooth"])
def test_full_hd_and_4k_frames(mode, h, w, kind):
    from oracle import synth
    frame = J.content("noise", h, w, 3, h) if kind == "noise" else synth.smooth_frame(h, h, w)
    got = kernels.jpeg_encode(torch.from_numpy(frame[None]).cuda(), 95, sampling=mode)
    assert got[0] == O.cv2_encode(frame, 95, sampling=mode)
    if h == 1080:  # the numpy oracle as well (at 2160p it would dominate the test's time)
        assert got[0] == O.encode(frame, 95, sampling=mode)
    assert len(got[0]) <= kernels.jpeg_encode_bound(w, h, 3, sampling=mode)
    if kind == "noise":
        assert got[0][600:].count(b"\xff\x00") > 1000  # the stuffing path ran


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("h,w", [(16, 65500), (65500, 16), (1, 65500), (65500, 1)])
def test_65500_sides_within_the_bound(mode, h, w):
    f = J.content("noise", h, w, 3, h + len(mode))
    got = encode_raw([f], 100, 0xFF, sampling=mode)
    check([f], 100, got, sampling=mode)


@pytest.mark.parametrize("n", [65, 130])
def test_batches_over_64_frames(n):
    rng = np.random.default_rng(n)
    frames = rng.integers(0, 256, (n, 37, 53, 3), dtype=np.uint8)
    frames[::3] //= 16  # smoother frames too: sizes differ between frames
    for opts in ({"sampling": "444"}, {"sampling": "411"}, {"sampling": "422", "luma_quality": 60,
                                                            "chroma_quality": 30}):
        check(frames, 75, kernels.jpeg_encode(torch.from_numpy(frames).cuda(), 75, **opts), cv2=False, **opts)
    check(frames[:3], 75, kernels.jpeg_encode(torch.from_numpy(frames[:3]).cuda(), 75, sampling="440"),
          sampling="440")


@pytest.mark.parametrize("mode", MODES)
def test_frames_at_odd_base_offsets(mode):
    rng = np.random.default_rng(len(mode))
    h, w, c = 21, 35, 3
    buf = torch.from_numpy(rng.integers(0, 256, 8 * h * w * c + 64, dtype=np.uint8)).cuda()
    offs = [1, 3 + 2 * h * w * c, 5 + 4 * h * w * c, 7 + 6 * h * w * c]
    views = [buf[o:o + h * w * c].view(h, w, c) for o in offs]
    frames = [v.cpu().numpy() for v in views]
    check(frames, 85, kernels.jpeg_encode(views, 85, sampling=mode), sampling=mode)
    dense = buf[1:1 + 5 * h * w * c].view(5, h, w, c)
    check(dense.cpu().numpy(), 30, kernels.jpeg_encode(dense, 30, sampling=mode), cv2=False, sampling=mode)


@pytest.mark.parametrize("fill", [0x00, 0xFF])
@pytest.mark.parametrize("mode", MODES)
def test_prefilled_outputs_and_guards(fill, mode):
    frames = [J.content("noise", 80, 112, 3, s) for s in range(4)]
    frames[2] = J.content("checker", 80, 112, 3, 0)
    check(frames, 100, encode_raw(frames, 100, fill, sampling=mode), sampling=mode)


def test_back_to_back_calls_reuse_dirty_scratch():
    big = J.content("noise", 2160, 3840, 3, 4)
    tiny = [J.content("noise", 9, 13, 3, s) for s in range(3)]
    for _ in range(2):
        for mode in ("444", "411"):
            got = kernels.jpeg_encode(torch.from_numpy(big[None]).cuda(), 100, sampling=mode)
            assert got[0] == O.cv2_encode(big, 100, sampling=mode)
            assert encode_raw(tiny, 100, 0x00, sampling="440") == [O.encode(f, 100, sampling="440") for f in tiny]
        # and the default encoder after them
        assert kernels.jpeg_encode([torch.from_numpy(f).cuda() for f in tiny], 100) == [J.encode(f, 100) for f in tiny]


def test_refusals_launch_nothing():
    L = cabi.lib()
    before = L.scn_launch_count()
    f = torch.zeros((1, 8, 8, 3), dtype=torch.uint8, device="cuda")
    for kw in ({"sampling": "423"}, {"luma_quality": 101}, {"chroma_quality": -3}):
        with pytest.raises(cabi.ScnError, match="argument error -1"):
            kernels.jpeg_encode(f, **kw)
    assert L.scn_launch_count() == before


# ---- optimised tables ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("h,w", [(1080, 1920), (2160, 3840)])
def test_optimised_full_hd_and_4k_frames(mode, h, w):
    from oracle import synth
    for frame in (J.content("noise", h, w, 3, h), synth.smooth_frame(h, h, w)):
        got = kernels.jpeg_encode(torch.from_numpy(frame[None]).cuda(), 95, sampling=mode, optimize=True)[0]
        assert got == O.cv2_encode(frame, 95, sampling=mode, optimize=True)
        assert len(got) <= kernels.jpeg_encode_bound(w, h, 3, sampling=mode, optimize=True)
        if h == 1080 and mode in ("420", "444"):
            assert got == O.encode(frame, 95, sampling=mode, optimize=True)


@pytest.mark.parametrize("n", [65, 130])
def test_optimised_batches_over_64_frames(n):
    """neighbouring frames of different content: different tables, DHT segments and header lengths in one launch and
    across the 64-frame split"""
    kinds = [J.content(k, 37, 53, 3, i) for i, k in enumerate(J.KINDS)]
    frames = np.stack([kinds[i % 4] if i % 5 else J.content("noise", 37, 53, 3, 100 + i) for i in range(n)])
    for opts in ({"optimize": True}, {"sampling": "411", "optimize": True}):
        got = encode_raw(frames, 75, 0xFF if n == 65 else 0x00, **opts)
        check(frames, 75, got, cv2=False, **opts)
        heads = {g.index(b"\xff\xda") for g in got}
        assert len(heads) >= 3  # header lengths differ between frames
    gray = np.ascontiguousarray(frames[..., :1])
    check(gray, 50, kernels.jpeg_encode(torch.from_numpy(gray).cuda(), 50, optimize=True), cv2=False, optimize=True)
    for i in (0, 1, 63, 64, n - 1):
        assert got[i] == O.cv2_encode(frames[i], 75, sampling="411", optimize=True), i


@pytest.mark.parametrize("h,w", [(16, 65500), (65500, 1)])
def test_optimised_65500_sides(h, w):
    f = J.content("noise", h, w, 3, h)
    check([f], 100, encode_raw([f], 100, 0x00, optimize=True), optimize=True)


def test_table_kernel_on_synthetic_frequencies():
    from test_jpeg_options_cpu import synthetic_frequencies
    L = cabi.lib()
    for name, freq in sorted(synthetic_frequencies().items()):
        f = (ctypes.c_uint64 * 256)(*freq)
        bits, vals = (ctypes.c_uint8 * 16)(), (ctypes.c_uint8 * 256)()
        cabi.check(L.scn_jpeg_optimal_table(f, bits, vals), "scn_jpeg_optimal_table")
        want_bits, want_vals = O.gen_optimal_table(freq)
        assert list(bits) == want_bits, name
        assert list(vals)[:len(want_vals)] == want_vals, name


def test_optimised_back_to_back_calls_reuse_dirty_scratch():
    frames = [J.content(k, 40, 72, 3, 3) for k in J.KINDS]
    for _ in range(2):
        for k in range(len(frames)):  # each call's symbol counts start from the last call's dirty scratch
            assert encode_raw([frames[k]], 90, 0x00, optimize=True)[0] == O.encode(frames[k], 90, optimize=True)


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


def test_op_with_each_option(sc):
    rng = np.random.default_rng(13)
    frames = rng.integers(0, 256, (10, 45, 61, 3), dtype=np.uint8)
    frames[::2] //= 8
    for mode in MODES:
        check(frames, 95, _encode_op(sc, frames, "s" + mode, format="jpg", sampling=mode), sampling=mode)
    check(frames, 80, _encode_op(sc, frames, "lq", format="jpg", quality=80, luma_quality=50), luma_quality=50)
    check(frames, 80, _encode_op(sc, frames, "cq", format="jpg", quality=80, chroma_quality=50), chroma_quality=50)
    check(frames, 95, _encode_op(sc, frames, "opt", format="jpg", optimize=True), optimize=True)
    opts = {"sampling": "420", "luma_quality": 70, "chroma_quality": 30, "optimize": True}
    check(frames, 95, _encode_op(sc, frames, "lcq", format="jpg", **opts), **opts)
    gray = np.ascontiguousarray(frames[:4, ..., :1])
    check(gray, 95, _encode_op(sc, gray, "gray", format="jpg", sampling="411", luma_quality=60), sampling="411",
          luma_quality=60)


@pytest.mark.parametrize("kw,why", [
    ({"format": "jpg", "sampling": "423"}, "sampling 423 is not one of 444, 422, 420, 440, 411"),
    ({"format": "jpg", "luma_quality": 101}, r"luma / chroma quality 101 is outside \[1, 100\]"),
    ({"format": "jpg", "chroma_quality": -1}, r"luma / chroma quality -1 is outside \[1, 100\]"),
    ({"format": "png", "sampling": "444"}, "are JPEG options; format is png"),
    ({"format": "png", "optimize": True}, "are JPEG options; format is png"),
    ({"sampling": "444"}, "are JPEG options; format is png")])
def test_refusals_fail_the_run_and_write_nothing(sc, kw, why):
    frames = np.zeros((2, 8, 8, 3), np.uint8)
    with pytest.raises(sp.ScannerException, match=why):
        _encode_op(sc, frames, "bad", **kw)
    assert not sp.NamedStream(sc, "bad_jpg").committed()
    # and the engine goes on
    good = np.full((3, 8, 8, 3), 77, np.uint8)
    check(good, 95, _encode_op(sc, good, "good", format="jpg", sampling="444"), sampling="444")


def test_png_options_refused_on_the_cpu_kernel(sc):
    frames = np.zeros((2, 8, 8, 3), np.uint8)
    inp = sc.io.Input([sp.NamedVideoStream(sc, "cpu", frames=frames)])
    out = sp.NamedStream(sc, "cpu_png")
    with pytest.raises(sp.ScannerException, match="are JPEG options; format is png"):
        sc.run(sc.io.Output(sc.ops.ImageEncoder(frame=inp, format="png", luma_quality=50), [out]),
               sp.PerfParams.manual(8, 16))
