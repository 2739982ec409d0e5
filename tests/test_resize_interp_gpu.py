"""Resize's INTER_NEAREST and INTER_AREA on the GPU: scn_resize_interp_u8c3 and scn_resize_interp_nv12 byte for byte
against the C restatement (oracle/resize_interp.c, itself held to cv2 by tests/test_resize_interp_cpu.py), INTER_LINEAR
through the new entry points against the existing ones, and the Resize op's `interpolation` argument."""
import ctypes

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import oracle  # noqa: E402
import scanner_b200 as sp  # noqa: E402
from oracle import resize_interp as R  # noqa: E402
from oracle import synth  # noqa: E402
from scanner_b200 import cabi, kernels, protolite  # noqa: E402
from scanner_b200 import engine as E  # noqa: E402

pytestmark = pytest.mark.gpu

MODE = {"INTER_NEAREST": 0, "INTER_LINEAR": 1, "INTER_AREA": 3}
ORACLE = {"INTER_NEAREST": R.resize_nearest, "INTER_AREA": R.resize_area, "INTER_LINEAR": oracle.resize}
GAP = 37  # guard bytes after every output frame

GRID = {  # (sw, sh, dw, dh): every INTER_AREA regime, odd widths, degenerate cells
    "1080p_224": (1920, 1080, 224, 224), "4k_224": (3840, 2160, 224, 224), "4k_1x1": (3840, 2160, 1, 1),
    "1080p_div4": (1920, 1080, 480, 270), "div3x2": (99, 60, 33, 30), "div2x1": (130, 40, 65, 40),
    "div1x2": (65, 80, 65, 40), "div2x2": (130, 80, 65, 40), "identity": (33, 17, 33, 17), "div8": (256, 128, 32, 16),
    "frac": (97, 61, 40, 25), "frac_odd": (301, 199, 223, 150), "frac_wide": (1919, 9, 257, 4),
    "up": (224, 224, 1920, 1080), "up_odd": (17, 3, 45, 31), "mixed": (64, 48, 32, 96), "mixed2": (1920, 1080, 224, 2000),
    "col": (1, 1079, 1, 224), "row": (1079, 1, 224, 1), "wide_tiles": (2000, 30, 700, 7),
}


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _plan(mode, sw, sh, dw, dh):
    l = cabi.lib()
    host = np.zeros(max(l.scn_resize_interp_plan_bytes(MODE[mode], sw, sh, dw, dh), 1), np.uint8)
    assert l.scn_resize_interp_plan_fill(MODE[mode], sw, sh, dw, dh, host.ctypes.data) == 0
    return torch.from_numpy(host).cuda()


def _carve_out(n, dw, dh, fill):
    """n output frames in one buffer, each followed by GAP guard bytes, all pre-filled with `fill`."""
    fb = dh * dw * 3
    buf = torch.full((n * (fb + GAP),), fill, dtype=torch.uint8, device="cuda")
    return buf, [buf.data_ptr() + i * (fb + GAP) for i in range(n)], fb


def _outputs(buf, n, fb, fill, dw, dh):
    data = buf.cpu().numpy().reshape(n, fb + GAP)
    assert (data[:, fb:] == fill).all(), "bytes written outside a frame"
    return data[:, :fb].reshape(n, dh, dw, 3)


def _sources(frames, offset):
    """frames (n, h, w, 3) on the GPU at byte `offset` into a buffer, each after the previous one at an odd stride."""
    n, h, w, _ = frames.shape
    fb = h * w * 3
    stride = fb + 5
    buf = torch.zeros((offset + n * stride,), dtype=torch.uint8, device="cuda")
    for i in range(n):
        buf[offset + i * stride:offset + i * stride + fb] = torch.from_numpy(frames[i].reshape(-1)).cuda()
    return buf, [buf.data_ptr() + offset + i * stride for i in range(n)]


def _run_rgb(mode, frames, dw, dh, fill, offset=0, plan=None):
    n, sh, sw, _ = frames.shape
    src, sptr = _sources(frames, offset)
    out, dptr, fb = _carve_out(n, dw, dh, fill)
    plan = _plan(mode, sw, sh, dw, dh) if plan is None else plan
    sp_, k1 = cabi.ptr_array(sptr)
    dp, k2 = cabi.ptr_array(dptr)
    rc = cabi.lib().scn_resize_interp_u8c3(MODE[mode], sp_, n, sw, sh, dp, dw, dh, plan.data_ptr(), _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    return _outputs(out, n, fb, fill, dw, dh)


def _frames(seed, n, h, w):
    f = np.stack([synth.rand_frame(seed + i, h, w) for i in range(n)])
    if n > 2:
        f[1], f[2] = 0, 255
    return f


@pytest.mark.parametrize("mode", ["INTER_AREA", "INTER_NEAREST"])
@pytest.mark.parametrize("name", sorted(GRID))
def test_rgb_grid_equals_oracle(mode, name):
    sw, sh, dw, dh = GRID[name]
    n = 2 if sw * sh > 2_000_000 else 3
    frames = _frames(100, n, sh, sw)
    for fill, offset in ((0x00, 0), (0xFF, 3)):
        got = _run_rgb(mode, frames, dw, dh, fill, offset)
        for i in range(n):
            assert (got[i] == ORACLE[mode](frames[i], dw, dh)).all(), (name, fill, offset, i)


def test_rgb_half_cells_and_every_alignment():
    """Exact .5 cells (2 x 2 rounds half up, other factors half to even) from every 16-byte phase of the source."""
    for (kx, ky) in ((2, 2), (4, 2), (3, 2), (2, 1), (8, 8)):
        w, h = kx * 41, ky * 9
        frames = np.stack([R.content("half", kx + ky + i, h, w, (kx, ky)) for i in range(2)])
        for offset in range(16):
            got = _run_rgb("INTER_AREA", frames, w // kx, h // ky, 0xFF, offset)
            for i in range(2):
                assert (got[i] == R.resize_area(frames[i], w // kx, h // ky)).all(), (kx, ky, offset, i)


@pytest.mark.parametrize("mode", ["INTER_AREA", "INTER_NEAREST"])
def test_rgb_seeded_sweep(mode):
    big = synth.rand_frame(7, 1080, 1920)
    for (sw, sh, dw, dh) in synth.resize_geometries(71, 120):
        if dw * dh > 1_500_000:
            continue
        frame = np.ascontiguousarray(big[:sh, :sw])[None]
        got = _run_rgb(mode, frame, dw, dh, 0x00, (sw + dh) % 16)
        assert (got[0] == ORACLE[mode](frame[0], dw, dh)).all(), (sw, sh, dw, dh)


@pytest.mark.parametrize("n", [65, 130])
@pytest.mark.parametrize("mode,geom", [("INTER_AREA", (97, 61, 40, 25)), ("INTER_AREA", (96, 60, 24, 20)),
                                       ("INTER_AREA", (30, 20, 45, 31)), ("INTER_NEAREST", (97, 61, 40, 25))])
def test_batches_over_64_frames(n, mode, geom):
    sw, sh, dw, dh = geom
    frames = np.stack([synth.rand_frame(300 + i, sh, sw) for i in range(n)])
    got = _run_rgb(mode, frames, dw, dh, 0xFF, 1)
    for i in range(n):
        assert (got[i] == ORACLE[mode](frames[i], dw, dh)).all(), i


def test_linear_through_the_new_entry_equals_scn_resize_bilinear():
    for (sw, sh, dw, dh) in [(1920, 1080, 224, 224), (130, 80, 65, 40), (17, 3, 45, 31), (97, 61, 40, 25)]:
        frames = _frames(500, 3, sh, sw)
        got = _run_rgb("INTER_LINEAR", frames, dw, dh, 0x00, 0)
        t = torch.from_numpy(frames).cuda()
        want = kernels.resize(t, dw, dh).cpu().numpy()
        assert (got == want).all(), (sw, sh, dw, dh)


# ---------------------------------------------------------------------------------------------- NV12
def _surfaces(seed, n, w, h, pitch):
    surf = np.zeros((n, h * 3 // 2, pitch), np.uint8)
    for i in range(n):
        l, c = synth.nv12_surface(seed + i, h, w, pitch)
        surf[i, :h], surf[i, h:] = l, c
    return surf


def _run_nv12(mode, surf, w, h, dw, dh, fill):
    n, _, pitch = surf.shape
    d = torch.from_numpy(surf).cuda()
    lum = [d.data_ptr() + i * d[0].numel() for i in range(n)]
    chroma = [p + h * pitch for p in lum]
    out, dptr, fb = _carve_out(n, dw, dh, fill)
    plan = _plan(mode, w, h, dw, dh)
    lp, k1 = cabi.ptr_array(lum)
    cp, k2 = cabi.ptr_array(chroma)
    dp, k3 = cabi.ptr_array(dptr)
    rc = cabi.lib().scn_resize_interp_nv12(MODE[mode], lp, cp, pitch, n, w, h, dp, dw, dh, plan.data_ptr(), _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    return _outputs(out, n, fb, fill, dw, dh), kernels.nv12_to_rgb(d, w, h)


NV12_GRID = [(1920, 1080, 224, 224), (3840, 2160, 224, 224), (1920, 1080, 480, 270), (98, 60, 33, 30),
             (96, 60, 48, 30), (98, 62, 40, 25), (224, 224, 1920, 1080), (64, 48, 32, 96), (2, 2, 1, 1), (30, 46, 15, 23)]


@pytest.mark.parametrize("mode", ["INTER_AREA", "INTER_NEAREST", "INTER_LINEAR"])
@pytest.mark.parametrize("pitch_kind", ["packed", "odd", "four", "sixty_four"])
def test_nv12_equals_rgb24_path(mode, pitch_kind):
    """scn_resize_interp_nv12 == scn_nv12_to_rgb24 + scn_resize_interp_u8c3 (== the oracle), at four pitches."""
    for (w, h, dw, dh) in NV12_GRID:
        pitch = {"packed": w, "odd": w + 1, "four": (w + 3) // 4 * 4 + 4, "sixty_four": (w + 63) // 64 * 64}[pitch_kind]
        n = 2
        surf = _surfaces(900, n, w, h, pitch)
        for fill in (0x00, 0xFF):
            got, rgb = _run_nv12(mode, surf, w, h, dw, dh, fill)
            rgb_np = rgb.cpu().numpy()
            via_rgb = _run_rgb(mode, rgb_np, dw, dh, fill)
            assert (got == via_rgb).all(), (w, h, dw, dh, pitch, fill)
            assert (got[0] == ORACLE[mode](rgb_np[0], dw, dh)).all(), (w, h, dw, dh, pitch)
        if mode == "INTER_LINEAR":
            _, want = kernels.nv12_hist_resize(torch.from_numpy(surf).cuda(), w, h, dw, dh, want_hist=False)
            assert (got == want.cpu().numpy()).all(), (w, h, dw, dh, pitch)


def test_nv12_batch_of_130_and_the_binding():
    w, h, dw, dh = 98, 62, 40, 25
    surf = _surfaces(1300, 130, w, h, 128)
    got, rgb = _run_nv12("INTER_AREA", surf, w, h, dw, dh, 0xFF)
    rgb_np = rgb.cpu().numpy()
    for i in range(130):
        assert (got[i] == R.resize_area(rgb_np[i], dw, dh)).all(), i
    hist, res = kernels.nv12_hist_resize(torch.from_numpy(surf).cuda(), w, h, dw, dh, interpolation="INTER_AREA")
    assert (res.cpu().numpy() == got).all()
    assert (hist.cpu().numpy() == kernels.histogram(rgb).cpu().numpy()).all()
    assert (kernels.resize(rgb, dw, dh, interpolation="INTER_AREA").cpu().numpy() == got).all()


def test_refusals_launch_nothing_and_write_nothing():
    l = cabi.lib()
    frames = _frames(5, 2, 16, 16)
    src, sptr = _sources(frames, 0)
    out, dptr, fb = _carve_out(2, 8, 8, 0x5A)
    plan = _plan("INTER_AREA", 16, 16, 8, 8)
    sp_, k1 = cabi.ptr_array(sptr)
    dp, k2 = cabi.ptr_array(dptr)
    torch.cuda.synchronize()
    before = l.scn_launch_count()
    for mode, rc in ((2, -2), (4, -2), (5, -2), (6, -2), (9, -1)):
        assert l.scn_resize_interp_u8c3(mode, sp_, 2, 16, 16, dp, 8, 8, plan.data_ptr(), _stream()) == rc
        assert l.scn_resize_interp_nv12(mode, sp_, sp_, 16, 2, 16, 16, dp, 8, 8, plan.data_ptr(), _stream()) == rc
    for mode in (0, 3):
        assert l.scn_resize_interp_u8c3(mode, sp_, 2, 16, 16, dp, 5, 5, None, _stream()) == -3
        assert l.scn_resize_interp_u8c3(mode, sp_, 2, 16, 16, dp, 65536, 32768, plan.data_ptr(), _stream()) == -1
        assert l.scn_resize_interp_nv12(mode, sp_, sp_, 16, 2, 16, 15, dp, 8, 8, plan.data_ptr(), _stream()) == -1
    torch.cuda.synchronize()
    assert l.scn_launch_count() == before
    assert (out.cpu().numpy() == 0x5A).all()


# ---------------------------------------------------------------------------------------------- the op
@pytest.fixture(scope="module")
def std_args():
    import os
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


OP_ARGS = {
    "area_224": {"width": 224, "height": 224, "interpolation": "INTER_AREA"},
    "area_div4": {"width": 160, "height": 90, "interpolation": "INTER_AREA"},
    "area_2x": {"width": 320, "height": 180, "interpolation": "INTER_AREA"},
    "area_up": {"width": 700, "height": 400, "interpolation": "INTER_AREA"},
    "nearest": {"width": 100, "height": 37, "interpolation": "INTER_NEAREST"},
    "linear": {"width": 100, "height": 37, "interpolation": "INTER_LINEAR"},
    "default": {"width": 100, "height": 37},
}


def _run_ops(std_args, add_source, args):
    eng = E.Engine(gpus=[0], instances_per_gpu=2)
    try:
        sid = add_source(eng)
        g = E.Graph()
        src = g.add_source(True)
        ops = {k: g.add_op("Resize", [(src, "frame")], device=1) for k in args}
        sinks = {k: g.add_sink((op, "frame")) for k, op in ops.items()}
        j = E.Job()
        j.bind_source(src, sid)
        for k, a in args.items():
            j.set_stream_args(ops[k], protolite.encode(std_args["ResizeArgs"], a))
        eng.run(g, [j], 4, 8)
        return {k: [j.output_row(s, i) for i in range(j.output_rows(s))] for k, s in sinks.items()}
    finally:
        eng.close()


def _check_ops(got, frames):
    for k, a in OP_ARGS.items():
        want = ORACLE[a.get("interpolation") or "INTER_LINEAR"]
        assert len(got[k]) == len(frames), k
        for i, f in enumerate(got[k]):
            assert (f == want(frames[i], a["width"], a["height"])).all(), (k, i)


def test_op_modes_on_host_frames_and_on_nv12_elements(std_args, monkeypatch):
    n = 5
    data, shown = _clip(62, n, 360, 640, 3)
    monkeypatch.delenv("SCN_DECODE_RGB", raising=False)
    nv12 = _run_ops(std_args, lambda eng: eng.add_h264(data), OP_ARGS)
    monkeypatch.setenv("SCN_DECODE_RGB", "1")
    rgb = _run_ops(std_args, lambda eng: eng.add_h264(data), OP_ARGS)
    host = _run_ops(std_args, lambda eng: eng.add_raw_frames(shown), OP_ARGS)
    for got in (nv12, rgb, host):
        _check_ops(got, shown)
    for k in OP_ARGS:
        for a, b in zip(nv12[k], host[k]):
            assert (a == b).all(), k


def test_plan_cache_keeps_modes_of_one_geometry_apart(std_args):
    """Streams of one geometry and target with different modes through a single pipeline instance: a cache key
    without the mode would hand the second stream the first one's plan."""
    frames = np.stack([synth.rand_frame(710 + i, 48, 97) for i in range(3)])
    eng = E.Engine(gpus=[0], instances_per_gpu=1)
    try:
        g = E.Graph()
        src = g.add_source(True)
        rz = g.add_op("Resize", [(src, "frame")], device=1)
        sink = g.add_sink((rz, "frame"))
        sid = eng.add_raw_frames(frames)
        modes = ["INTER_AREA", "INTER_NEAREST", "INTER_LINEAR", "INTER_AREA", ""]
        jobs = []
        for m in modes:
            j = E.Job()
            j.bind_source(src, sid)
            j.set_stream_args(rz, protolite.encode(std_args["ResizeArgs"], {"width": 40, "height": 30,
                                                                          "interpolation": m}))
            jobs.append(j)
        eng.run(g, jobs, 4, 8)
        assert eng.stats()["counters"]["instances"] == 1
        for m, j in zip(modes, jobs):
            for i in range(3):
                assert (j.output_row(sink, i) == ORACLE[m or "INTER_LINEAR"](frames[i], 40, 30)).all(), (m, i)
    finally:
        eng.close()


@pytest.fixture()
def sc(tmp_path):
    c = sp.Client(db_path=str(tmp_path / "scanner_db"))
    yield c
    c.stop()


def _resize_op(sc, name, frames, **kw):
    inp = sc.io.Input([sp.NamedVideoStream(sc, name, frames=frames)])
    out = sp.NamedVideoStream(sc, name + "_out")
    sc.run(sc.io.Output(sc.ops.Resize(frame=inp, device=sp.DeviceType.GPU, **kw), [out]), sp.PerfParams.estimate())
    return list(out.load())


def test_client_pipeline_with_inter_area_and_refused_modes(sc):
    rgb = np.random.default_rng(11).integers(0, 256, (4, 90, 160, 3), dtype=np.uint8)
    for bad, kind in (("INTER_CUBIC", "unsupported"), ("bogus", "unknown")):
        with pytest.raises(sp.ScannerException, match=rf"Resize, row 0: {kind} interpolation '{bad}'; supported: "
                                                      r"INTER_NEAREST, INTER_LINEAR, INTER_AREA"):
            _resize_op(sc, "bad_" + bad, rgb, width=[40], height=[30], interpolation=[bad])
    # the same client goes on
    got = _resize_op(sc, "area", rgb, width=[37], height=[23], interpolation=["INTER_AREA"])
    assert len(got) == 4
    for i in range(4):
        assert (got[i] == R.resize_area(rgb[i], 37, 23)).all(), i
    got = _resize_op(sc, "nearest", rgb, width=[37], height=[23], interpolation=["INTER_NEAREST"])
    for i in range(4):
        assert (got[i] == R.resize_nearest(rgb[i], 37, 23)).all(), i
