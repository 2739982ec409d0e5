"""GaussianBlur on the GPU: scn_gaussian_blur_u8 and scn_gaussian_blur_nv12 byte for byte against the C restatement
(oracle/gaussian_blur.c, itself held to cv2 by tests/test_gaussian_blur_cpu.py) and against live cv2, and the
GaussianBlur op through the engine and the client."""
import ctypes
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import oracle  # noqa: E402
import scanner_b200 as sp  # noqa: E402
from oracle import gaussian_blur as G  # noqa: E402
from oracle import synth  # noqa: E402
from scanner_b200 import cabi, kernels, protolite  # noqa: E402
from scanner_b200 import engine as E  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GAP = 37  # guard bytes after every output frame
KSIZES = tuple(range(1, 32, 2))
BORDERS = ("BORDER_REFLECT_101", "BORDER_REPLICATE", "BORDER_REFLECT")


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _blur_into(src_ptrs, dst_ptrs, w, h, c, ksize, sx, sy=0.0, border=""):
    plan = kernels.gaussian_blur_plan(ksize, sx, sy, border)
    sp_, k1 = cabi.ptr_array(src_ptrs)
    dp, k2 = cabi.ptr_array(dst_ptrs)
    return cabi.lib().scn_gaussian_blur_u8(plan.ctypes.data, sp_, len(src_ptrs), w, h, c, dp, _stream())


def _carve_out(n, fb, fill):
    """n output frames of fb bytes in one buffer, each followed by GAP guard bytes, all pre-filled with `fill`."""
    buf = torch.full((n * (fb + GAP),), fill, dtype=torch.uint8, device="cuda")
    return buf, [buf.data_ptr() + i * (fb + GAP) for i in range(n)]


def _frames_of(buf, n, fb, fill):
    """The n frames of a _carve_out buffer, after checking that every guard byte still holds `fill`."""
    a = buf.cpu().numpy().reshape(n, fb + GAP)
    assert (a[:, fb:] == fill).all(), "bytes written past the end of a frame"
    return a[:, :fb]


def test_case_sweep_equals_the_oracle_and_cv2():
    """Every odd (kw, kh), every border, C = 1 and 3, explicit and derived sigmas, frames down to 1 x 1."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(1)
    cases = [((kw, kh), 0.0, 0.0) for kw in KSIZES for kh in KSIZES]
    cases += [((0, 0), s, 0.0) for s in (0.2, 0.7, 1.1, 2.5, 4.9)] + [((0, 0), 1.5, 4.0), ((5, 9), 2.0, 0.0),
                                                                      ((31, 3), 7.0, 0.2), ((0, 13), 1.0, 0.0)]
    for i, (ksize, sx, sy) in enumerate(cases):
        h, w = (int(rng.integers(1, 90)), int(rng.integers(1, 200))) if i % 4 else (int(rng.integers(1, 9)),
                                                                                    int(rng.integers(1, 9)))
        c = (1, 3)[i % 2]
        border = BORDERS[i % 3]
        kind = ("noise", "gradient", "noise", "full", "noise", "zero")[i % 6]
        img = G.content(kind, 50 + i, h, w, c)
        got = kernels.gaussian_blur(torch.from_numpy(img[None]).cuda(), ksize, sx, sy, border)[0].cpu().numpy()
        want = G.gaussian_blur(img, ksize, sx, sy, border)
        assert (got == want).all(), (ksize, sx, sy, border, h, w, c)
        assert (got == cv2.GaussianBlur(img, ksize, sx, sigmaY=sy,
                                        borderType=G.BORDERS[border]).reshape(img.shape)).all()


@pytest.mark.parametrize("h,w", [(1080, 1920), (2160, 3840)])
@pytest.mark.parametrize("c", [1, 3])
def test_1080p_and_2160p_equal_cv2(h, w, c):
    cv2 = pytest.importorskip("cv2")
    n = 2
    frames = np.stack([G.content("noise", 900 + i, h, w, c) for i in range(n)])
    d = torch.from_numpy(frames).cuda()
    for ksize, sx, border in (((3, 3), 0, ""), ((7, 7), 0, "BORDER_REPLICATE"), ((15, 15), 3.0, "BORDER_REFLECT"),
                              ((31, 31), 0, ""), ((5, 9), 2.0, "")):
        got = kernels.gaussian_blur(d, ksize, sx, 0, border).cpu().numpy()
        for i in range(n):
            want = cv2.GaussianBlur(frames[i], ksize, sx, borderType=G.BORDERS[border]).reshape(h, w, c)
            assert (got[i] == want).all(), (ksize, sx, border, i)


def test_widths_1_to_4095_at_every_base_alignment():
    """Every width 1-4095 (3 channels; 1 channel on every 7th), 16 copies at base offsets 0-15 of one buffer into
    outputs at offsets 15-0, with every kernel width across the widths so that every tile edge meets every kernel."""
    h = 5
    for w in range(1, 4096):
        for c in ((3, 1) if w % 7 == 0 else (3,)):
            fb = h * w * c
            img = G.content("noise", w, h, w, c)
            ksize = (KSIZES[w % 16], KSIZES[(w // 16) % 3])
            border = BORDERS[w % 3]
            host = np.zeros(16 * (fb + 16) + 16, np.uint8)
            for o in range(16):
                host[o * (fb + 16) + o:][:fb] = img.reshape(-1)
            src = torch.from_numpy(host).cuda()
            dst = torch.full((16 * (fb + 16) + 16,), 0xA5, dtype=torch.uint8, device="cuda")
            sps = [src.data_ptr() + o * (fb + 16) + o for o in range(16)]
            dps = [dst.data_ptr() + o * (fb + 16) + 15 - o for o in range(16)]
            assert _blur_into(sps, dps, w, h, c, ksize, 0.0, 0.0, border) == 0
            want = G.gaussian_blur(img, ksize, 0.0, 0.0, border).reshape(-1)
            out = dst.cpu().numpy()
            untouched = np.ones(out.size, bool)
            for o in range(16):
                at = o * (fb + 16) + 15 - o
                assert (out[at:at + fb] == want).all(), (w, c, o, ksize)
                untouched[at:at + fb] = False
            assert (out[untouched] == 0xA5).all(), (w, c)


@pytest.mark.parametrize("n", [65, 130])
@pytest.mark.parametrize("fill", [0x00, 0xFF])
def test_batches_over_64_frames_into_prefilled_guarded_outputs(n, fill):
    h, w = 37, 61
    for c, ksize, sx, border in ((3, (7, 5), 0.0, ""), (1, (0, 0), 2.2, "BORDER_REFLECT"),
                                 (3, (31, 1), 6.0, "BORDER_REPLICATE")):
        fb = h * w * c
        frames = np.stack([G.content("noise", 3000 + i, h, w, c) for i in range(n)])
        frames[3] = 255
        frames[4] = 0
        d = torch.from_numpy(frames).cuda()
        buf, dps = _carve_out(n, fb, fill)
        assert _blur_into([d.data_ptr() + i * fb for i in range(n)], dps, w, h, c, ksize, sx, 0.0, border) == 0
        got = _frames_of(buf, n, fb, fill)
        for i in range(n):
            assert (got[i] == G.gaussian_blur(frames[i], ksize, sx, 0.0, border).reshape(-1)).all(), (c, i)


def test_mixed_shapes_in_one_list():
    frames = [G.content("noise", i, h, w, c) for i, (h, w, c) in
              enumerate([(9, 17, 3), (9, 17, 3), (40, 3, 1), (1, 1, 3), (64, 64, 1), (64, 64, 1)])]
    got = kernels.gaussian_blur([torch.from_numpy(f).cuda() for f in frames], (5, 3), 0.9)
    for g, f in zip(got, frames):
        assert (g.cpu().numpy() == G.gaussian_blur(f, (5, 3), 0.9)).all(), f.shape


def _nv12_then_u8(surf, w, h, ksize, sx, sy=0.0, border=""):
    return kernels.gaussian_blur(kernels.nv12_to_rgb(surf, w, h), ksize, sx, sy, border)


def test_nv12_equals_nv12_to_rgb_then_blur_on_all_yuv_triples():
    w, h = synth.EXH_W, synth.EXH_H
    args = (((3, 3), 0.0, ""), ((7, 7), 0.0, "BORDER_REPLICATE"), ((31, 9), 4.0, "BORDER_REFLECT"), ((0, 0), 1.3, ""))
    for f0 in range(0, synth.EXH_FRAMES, 16):
        surf = np.stack([np.concatenate(synth.nv12_exhaustive(f), 0) for f in range(f0, f0 + 16)])
        d = torch.from_numpy(surf).cuda()
        ksize, sx, border = args[(f0 // 16) % len(args)]
        got = kernels.nv12_gaussian_blur(d, w, h, ksize, sx, 0.0, border)
        assert torch.equal(got, _nv12_then_u8(d, w, h, ksize, sx, 0.0, border)), f0


@pytest.mark.parametrize("fill", [0x00, 0xFF])
@pytest.mark.parametrize("h,w,pitch", [(270, 480, 480), (270, 480, 512), (90, 136, 160), (6, 34, 34), (2, 2, 2)])
def test_nv12_on_seeded_surfaces_into_guarded_outputs(h, w, pitch, fill):
    n = 66
    surf = np.zeros((n, h * 3 // 2, pitch), np.uint8)
    for i in range(n):
        luma, chroma = synth.nv12_surface(700 + i, h, w, pitch)
        surf[i, :h], surf[i, h:] = luma, chroma
    d = torch.from_numpy(surf).cuda()
    lum, chr_, _ = kernels._surface_ptrs(d, h)
    for ksize, sx, border in (((5, 5), 0.0, ""), ((0, 0), 3.0, "BORDER_REFLECT")):
        fb = h * w * 3
        buf, dps = _carve_out(n, fb, fill)
        plan = kernels.gaussian_blur_plan(ksize, sx, 0.0, border)
        lp, k1 = cabi.ptr_array(lum)
        cp, k2 = cabi.ptr_array(chr_)
        op, k3 = cabi.ptr_array(dps)
        assert cabi.lib().scn_gaussian_blur_nv12(plan.ctypes.data, lp, cp, pitch, n, w, h, op, _stream()) == 0
        got = _frames_of(buf, n, fb, fill)
        want = _nv12_then_u8(d, w, h, ksize, sx, 0.0, border).cpu().numpy().reshape(n, -1)
        assert (got == want).all(), (ksize, sx)


def test_refusals_launch_and_write_nothing():
    l = cabi.lib()
    h, w = 8, 8
    src = torch.zeros((2, h, w, 3), dtype=torch.uint8, device="cuda")
    dst = torch.full((2, h, w, 3), 0x5A, dtype=torch.uint8, device="cuda")
    sps = [src.data_ptr(), src.data_ptr() + h * w * 3]
    dps = [dst.data_ptr(), dst.data_ptr() + h * w * 3]
    plan = kernels.gaussian_blur_plan((5, 5), 0.0)
    before = l.scn_launch_count()
    s, k1 = cabi.ptr_array(sps)
    d, k2 = cabi.ptr_array(dps)
    assert l.scn_gaussian_blur_u8(plan.ctypes.data, s, 2, w, h, 2, d, _stream()) == -1
    assert l.scn_gaussian_blur_u8(plan.ctypes.data, s, -2, w, h, 3, d, _stream()) == -1
    assert l.scn_gaussian_blur_u8(None, s, 2, w, h, 3, d, _stream()) == -3
    bad = plan.copy()
    bad[4] = 3  # kernel width 5 -> 3: its first three taps no longer sum to 256
    assert l.scn_gaussian_blur_u8(bad.ctypes.data, s, 2, w, h, 3, d, _stream()) == -3
    assert l.scn_gaussian_blur_nv12(plan.ctypes.data, s, s, w, 2, w - 1, h, d, _stream()) == -1
    for args in (((4, 4), 1.0), ((0, 0), 0.0), ((33, 3), 1.0), ((0, 0), 6.0)):
        with pytest.raises(cabi.ScnError):
            kernels.gaussian_blur(src, *args)
    with pytest.raises(cabi.ScnError, match="BORDER_CONSTANT.*not supported; supported: BORDER_DEFAULT"):
        kernels.gaussian_blur(src, (3, 3), 0.0, border="BORDER_CONSTANT")
    torch.cuda.synchronize()
    assert l.scn_launch_count() == before
    assert (dst == 0x5A).all()


# ---- through the engine -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def std_args():
    E.load_stdlib()
    return protolite.parse_proto(open(os.path.join(ROOT, "scanner_b200", "csrc", "ops", "stdlib_args.proto")).read())


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


def test_engine_pipeline_from_nv12_elements_equals_cv2(std_args, monkeypatch):
    """synthetic H.264 clip -> NV12 frame elements -> GaussianBlur -> sink, every row against cv2."""
    cv2 = pytest.importorskip("cv2")
    monkeypatch.delenv("SCN_DECODE_RGB", raising=False)
    n, h, w = 10, 270, 480
    data, shown = _clip(31, n, h, w, 5)
    args = {"kernel_width": 9, "kernel_height": 5, "sigma_x": 1.7, "sigma_y": 0.0, "border": "BORDER_REFLECT"}
    eng = E.Engine(gpus=[0], instances_per_gpu=2)
    try:
        g = E.Graph()
        src = g.add_source(True)
        gb = g.add_op("GaussianBlur", [(src, "frame")], device=1,
                      args=protolite.encode(std_args["GaussianBlurArgs"], args))
        s = g.add_sink((gb, "frame"))
        j = E.Job()
        j.bind_source(src, eng.add_h264(data))
        eng.run(g, [j], 4, 8)
        assert eng.stats()["counters"]["frames_delivered_nv12"] == n
        assert j.output_rows(s) == n
        for i in range(n):
            want = cv2.GaussianBlur(shown[i], (9, 5), 1.7, borderType=cv2.BORDER_REFLECT)
            assert np.array_equal(j.output_row(s, i), want), i
    finally:
        eng.close()


@pytest.fixture()
def sc(tmp_path):
    c = sp.Client(db_path=str(tmp_path / "scanner_db"))
    yield c
    c.stop()


def _run_op(sc, name, frames, make):
    inp = sc.io.Input([sp.NamedVideoStream(sc, name, frames=frames)])
    out = sp.NamedVideoStream(sc, name + "_out")
    sc.run(sc.io.Output(make(inp), [out]), sp.PerfParams.estimate())
    return list(out.load())


def test_client_gray_pipeline_equals_cv2_and_bad_ksize_fails_the_run(sc):
    """ConvertColor(COLOR_RGB2GRAY) -> GaussianBlur per row against cv2; a bad ksize fails the run with its message
    and the same client then runs a good job."""
    cv2 = pytest.importorskip("cv2")
    GPU = sp.DeviceType.GPU
    rgb = np.random.default_rng(8).integers(0, 256, (6, 45, 70, 3), dtype=np.uint8)

    def gray_blur(f, **kw):
        return sc.ops.GaussianBlur(frame=sc.ops.ConvertColor(frame=f, conversion=["COLOR_RGB2GRAY"]), device=GPU, **kw)

    with pytest.raises(sp.ScannerException, match=r"GaussianBlur, row 0: bad ksize 4x5"):
        _run_op(sc, "bad", rgb, lambda f: gray_blur(f, kernel_width=4, kernel_height=5, sigma_x=1.0))
    with pytest.raises(sp.ScannerException, match=r"GaussianBlur, row 0: unsupported border 'BORDER_WRAP'"):
        _run_op(sc, "bad_border", rgb, lambda f: gray_blur(f, kernel_width=3, kernel_height=3, border="BORDER_WRAP"))
    got = _run_op(sc, "good", rgb, lambda f: gray_blur(f, kernel_width=0, kernel_height=7, sigma_x=1.4, sigma_y=2.0))
    assert len(got) == 6
    for i in range(6):
        want = cv2.GaussianBlur(cv2.cvtColor(rgb[i], cv2.COLOR_RGB2GRAY), (0, 7), 1.4, sigmaY=2.0)
        assert got[i].size == 45 * 70 and (got[i].reshape(45, 70) == want).all(), i
    rgb_out = _run_op(sc, "rgb", rgb, lambda f: sc.ops.GaussianBlur(frame=f, kernel_width=5, kernel_height=5,
                                                                    device=GPU))
    for i in range(6):
        assert (rgb_out[i] == cv2.GaussianBlur(rgb[i], (5, 5), 0)).all(), i
