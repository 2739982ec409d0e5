"""Both Resize kernel families and the Resize op, byte for byte against oracle.resize (itself held to live cv2.resize
over the same geometry sweep by tests/test_oracle_golden.py) and, on a subset, against live cv2:
  * resize_linear_kernel / resize_area2x_kernel (resize.cu) on a grid of scale factors and edge geometries (1-pixel
    sources and destinations, 1 x N and N x 1, 2x on one axis only, integer 3x and 4x, large upscales) and a seeded
    sweep over synth.RESIZE_SIDES, with the kernel that ran checked by the profiler;
  * pointer lists at odd byte offsets and over 64 frames, outputs separated by sentinel gaps;
  * nv12_resize_kernel (fused.cu) on the even part of the grid at four pitches, with and without the histogram (which
    sends the Resize to the side stream), over outputs pre-filled with 0 and with 255;
  * refusals, which launch nothing and write nothing;
  * the Resize op through the engine and the client: target rules, NV12 and RGB24 elements, the per-geometry plan
    cache, and bad input, which fails the run and leaves the process and the client usable.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
cv2 = pytest.importorskip("cv2")

import oracle  # noqa: E402
import scanner_b200 as sp  # noqa: E402
from oracle import synth  # noqa: E402
from scanner_b200 import cabi, kernels, protolite  # noqa: E402
from scanner_b200 import engine as E  # noqa: E402

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5

GRID = {                                 # name: (src_w, src_h, dst_w, dst_h)
    "identity": (64, 48, 64, 48),
    "2x": (1920, 1080, 960, 540),
    "2x_small": (2, 2, 1, 1),
    "2x_w_only": (64, 48, 32, 48),
    "2x_h_only": (64, 48, 64, 24),
    "2x_w_3x_h": (64, 48, 32, 16),
    "3x": (192, 144, 64, 48),
    "4x": (256, 192, 64, 48),
    "non_integer_down": (1000, 702, 333, 257),
    "up_1px": (1, 1, 224, 224),
    "up_2px": (2, 2, 224, 224),
    "up_3px": (3, 3, 224, 224),
    "up_7px": (7, 7, 224, 224),
    "up_4x6": (6, 4, 224, 224),
    "dst_1x1": (64, 48, 1, 1),
    "dst_1xN": (64, 48, 1, 37),
    "dst_Nx1": (64, 48, 37, 1),
    "src_1xN": (1, 100, 17, 50),
    "src_Nx1": (100, 1, 50, 17),
    "1080p_224": (1920, 1080, 224, 224),
    "4k_360p": (3840, 2160, 640, 360),
    "224_1080p": (224, 224, 1920, 1080),
    "area_odd_dst": (46, 30, 23, 15),
    "area_odd_1918": (1918, 1080, 959, 540),
}
SWEEP = synth.resize_geometries(31, 200)


def _area2x(sw, sh, dw, dh):
    return sw == 2 * dw and sh == 2 * dh


def _ran(fn):
    """fn() and the {kernel: launches} it caused."""
    L = cabi.lib()
    L.scn_prof_enable(1)
    try:
        out = fn()
        torch.cuda.synchronize()
        rep = cabi.prof_report()
    finally:
        L.scn_prof_enable(0)
    return out, {k: v["launches"] for k, v in rep.items()}


def _frames(seed, n, h, w):
    """n random frames, then (when n > 2) a constant 0 and a constant 255 frame."""
    f = np.stack([synth.rand_frame(seed + i, h, w) for i in range(n)])
    if n > 2:
        f[-2], f[-1] = 0, 255
    return f


def _check_rgb(sw, sh, dw, dh, n, seed, with_cv2):
    frames = _frames(seed, n, sh, sw)
    got, ran = _ran(lambda: kernels.resize(torch.from_numpy(frames).cuda(), dw, dh))
    kernel = "resize_area2x_kernel" if _area2x(sw, sh, dw, dh) else "resize_linear_kernel"
    assert ran == {kernel: 1}, (sw, sh, dw, dh, ran)
    got = got.cpu().numpy()
    for i in range(n):
        want = oracle.resize(frames[i], dw, dh)
        assert (got[i] == want).all(), (sw, sh, dw, dh, i)
        if with_cv2:
            live = cv2.resize(frames[i], (dw, dh), interpolation=cv2.INTER_LINEAR)
            assert (got[i] == live).all(), ("cv2", sw, sh, dw, dh, i)


@pytest.mark.parametrize("name", list(GRID))
def test_rgb_grid_equals_oracle_and_cv2(name):
    sw, sh, dw, dh = GRID[name]
    _check_rgb(sw, sh, dw, dh, 2 if sw * sh > 1 << 20 else 4, 100, True)


@pytest.mark.parametrize("part", range(4))
def test_rgb_seeded_sweep(part):
    for k, (sw, sh, dw, dh) in enumerate(SWEEP[part::4]):
        _check_rgb(sw, sh, dw, dh, 1, 200 + k, k % 4 == 0)


# ---------------------------------------------------------------------------------------------- pointer lists
def _carve(n, sw, sh, dw, dh, fill):
    """Sources at odd byte offsets of one buffer; outputs in one buffer behind, between and after 5-byte gaps that
    hold SENTINEL, the outputs themselves filled with `fill`."""
    sb, db, gap = sw * sh * 3, dw * dh * 3, 5
    sstride = sb + (1 if sb % 2 else 2)          # even: every source starts at an odd offset
    frames = _frames(7 * n, n, sh, sw)
    src = torch.zeros(1 + n * sstride, dtype=torch.uint8, device="cuda")
    for i in range(n):
        src[1 + i * sstride:1 + i * sstride + sb] = torch.from_numpy(frames[i].reshape(-1)).cuda()
    out = torch.full((gap + n * (db + gap),), SENTINEL, dtype=torch.uint8, device="cuda")
    doffs = [gap + i * (db + gap) for i in range(n)]
    for o in doffs:
        out[o:o + db] = fill
    return frames, src, [src.data_ptr() + 1 + i * sstride for i in range(n)], out, doffs


@pytest.mark.parametrize("n", [65, 130])
@pytest.mark.parametrize("sw,sh,dw,dh", [(37, 23, 29, 17), (34, 22, 17, 11), (5, 3, 224, 1)])
def test_pointer_lists_write_their_frames_and_nothing_else(sw, sh, dw, dh, n):
    # the plan with one zeroed spare tap behind it, so that a thread past the last pixel reads defined memory
    host = kernels.ResizePlan(sw, sh, dw, dh).host
    plan = torch.from_numpy(np.concatenate([host, np.zeros(16, np.uint8)])).cuda()
    want = None
    for fill in (0, 255):
        frames, src, sptrs, out, doffs = _carve(n, sw, sh, dw, dh, fill)
        if want is None:
            want = [oracle.resize(f, dw, dh) for f in frames]
        sp_, k1 = cabi.ptr_array(sptrs)
        dp, k2 = cabi.ptr_array([out.data_ptr() + o for o in doffs])
        _, ran = _ran(lambda: cabi.check(cabi.lib().scn_resize_bilinear_u8c3(sp_, n, sw, sh, dp, dw, dh,
                                                                             plan.data_ptr(), kernels._stream()),
                                                       "resize"))
        kernel = "resize_area2x_kernel" if _area2x(sw, sh, dw, dh) else "resize_linear_kernel"
        assert ran == {kernel: (n + 63) // 64}, ran
        host = out.cpu().numpy()
        db = dw * dh * 3
        keep = np.ones(host.size, bool)
        for i, o in enumerate(doffs):
            assert (host[o:o + db] == want[i].reshape(-1)).all(), (fill, i)
            keep[o:o + db] = False
        assert (host[keep] == SENTINEL).all(), (fill, np.nonzero(keep & (host != SENTINEL))[0][:8])


# ---------------------------------------------------------------------------------------------- NV12
def _pitches(w):
    return {"packed": w, "odd": w + 1, "4-aligned": (w + 3) // 4 * 4 + 4, "64-aligned": (w + 64) // 64 * 64}


def _nv12_resize(surf, w, h, dw, dh, want_hist, fill):
    """scn_nv12_hist_resize on (N, H*3/2, pitch) surfaces into outputs filled with `fill`."""
    n, _, pitch = surf.shape
    lum, chr_, _ = kernels._surface_ptrs(surf, h)
    lp, k1 = cabi.ptr_array(lum)
    cp, k2 = cabi.ptr_array(chr_)
    hist = torch.full((n, 3, 16), -1, dtype=torch.int32, device="cuda") if want_hist else None
    plan = kernels.ResizePlan(w, h, dw, dh)
    res = torch.full((n, dh, dw, 3), fill, dtype=torch.uint8, device="cuda")
    op, k3 = cabi.ptr_array([res.data_ptr() + i * dh * dw * 3 for i in range(n)])
    rc = cabi.lib().scn_nv12_hist_resize(lp, cp, pitch, n, w, h, hist.data_ptr() if want_hist else None, op, dw, dh,
                                         plan.ptr, kernels._stream())
    cabi.check(rc, "scn_nv12_hist_resize")
    torch.cuda.synchronize()
    return hist, res


def _check_nv12(w, h, dw, dh, pitch, seed, runs=((False, 0), (False, 255), (True, 0), (True, 255))):
    n = 2 if w * h > 1 << 20 else 3
    g = torch.Generator(device="cuda").manual_seed(seed)
    surf = torch.randint(0, 256, (n, h * 3 // 2, pitch), dtype=torch.uint8, device="cuda", generator=g)
    rgb = kernels.nv12_to_rgb(surf, w, h)
    want = kernels.resize(rgb, dw, dh)
    host = surf.cpu().numpy()
    oh, orr = oracle.nv12_hist_resize(host[0, :h], host[0, h:], dw, dh, w)
    assert (want[0].cpu().numpy() == orr).all()
    kernel = "nv12_resize_kernel"
    for want_hist, fill in runs:
        (hist, res), ran = _ran(lambda: _nv12_resize(surf, w, h, dw, dh, want_hist, fill))
        assert ran.get(kernel) == 1, ran
        bad = (res != want).flatten(1).any(1).nonzero().flatten().tolist()
        assert not bad, (want_hist, fill, bad)
        if want_hist:
            assert (hist[0].cpu().numpy() == oh).all()
    return surf


NV12_GRID = {k: v for k, v in GRID.items() if v[0] % 2 == 0 and v[1] % 2 == 0}
NV12_GRID.update({"up_2x2_to_5x3": (2, 2, 5, 3), "up_6x4_to_1x9": (6, 4, 1, 9), "2x2_identity": (2, 2, 2, 2)})


@pytest.mark.parametrize("pitch_kind", ["packed", "odd", "4-aligned", "64-aligned"])
@pytest.mark.parametrize("name", list(NV12_GRID))
def test_nv12_grid_equals_rgb_path_and_oracle(name, pitch_kind):
    w, h, dw, dh = NV12_GRID[name]
    _check_nv12(w, h, dw, dh, _pitches(w)[pitch_kind], 300)


def test_nv12_seeded_sweep():
    even = tuple(s for s in synth.RESIZE_SIDES if s % 2 == 0)
    for k, (w, h, dw, dh) in enumerate(synth.resize_geometries(41, 40, even)):
        pitch = list(_pitches(w).values())[k % 4]
        _check_nv12(w, h, dw, dh, pitch, 400 + k, runs=((k % 2 == 1, 255 * (k % 3 == 0)),))


def test_nv12_packed_elements_equal_pitched_surfaces():
    """The FrameLayout::NV12 element kernels.nv12_pack makes, on the odd-destination area path and on a linear one."""
    for (w, h, dw, dh) in [(46, 30, 23, 15), (46, 30, 224, 7)]:
        surf = _check_nv12(w, h, dw, dh, 51, 500)
        packed = kernels.nv12_pack(surf, w, h)
        _check_nv12(w, h, dw, dh, w, 500)
        assert torch.equal(packed, surf[:, :, :w])
        for want_hist in (False, True):
            _, a = _nv12_resize(packed, w, h, dw, dh, want_hist, 0)
            _, b = _nv12_resize(surf, w, h, dw, dh, want_hist, 255)
            assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------- refusals
def test_refusals_launch_nothing_and_write_nothing():
    L = cabi.lib()
    src = torch.randint(0, 256, (4096,), dtype=torch.uint8, device="cuda")
    dst = torch.full((4096,), SENTINEL, dtype=torch.uint8, device="cuda")
    plan = torch.zeros(4096, dtype=torch.uint8, device="cuda")   # never read: every call below is refused
    sp_, k1 = cabi.ptr_array([src.data_ptr()] * 2)
    cp, k2 = cabi.ptr_array([src.data_ptr() + 64] * 2)
    dp, k3 = cabi.ptr_array([dst.data_ptr()] * 2)
    st = kernels._stream()
    torch.cuda.synchronize()
    before = L.scn_launch_count()

    def rgb(n, sw, sh, dw, dh, p):
        return L.scn_resize_bilinear_u8c3(sp_, n, sw, sh, dp, dw, dh, p, st)

    def nv12(n, w, h, pitch, dw, dh, p):
        return L.scn_nv12_hist_resize(sp_, cp, pitch, n, w, h, None, dp, dw, dh, p, st)

    cases = [
        ("rgb n < 0", rgb(-1, 8, 8, 4, 4, plan.data_ptr()), -1),
        ("rgb zero src", rgb(2, 0, 8, 4, 4, plan.data_ptr()), -1),
        ("rgb zero dst", rgb(2, 8, 8, 4, 0, plan.data_ptr()), -1),
        ("rgb no plan", rgb(2, 8, 8, 3, 3, None), -3),
        ("rgb no plan 2x on one axis", rgb(2, 8, 8, 4, 8, None), -3),
        ("rgb dst over INT_MAX pixels", rgb(2, 8, 8, 65536, 32768, plan.data_ptr()), -1),
        ("strided n < 0", L.scn_resize_bilinear_u8c3_strided(src.data_ptr(), 192, -1, 8, 8, dst.data_ptr(), 48, 4, 4,
                                                             plan.data_ptr(), st), -1),
        ("nv12 n < 0", nv12(-1, 8, 8, 8, 4, 4, plan.data_ptr()), -1),
        ("nv12 zero dst", nv12(2, 8, 8, 8, 0, 4, plan.data_ptr()), -1),
        ("nv12 no plan", nv12(2, 8, 8, 8, 3, 3, None), -3),
        ("nv12 no plan 2x on one axis", nv12(2, 8, 8, 8, 8, 4, None), -3),
        ("nv12 odd width", nv12(2, 7, 8, 8, 3, 3, plan.data_ptr()), -1),
        ("nv12 odd height", nv12(2, 8, 7, 8, 3, 3, plan.data_ptr()), -1),
        ("nv12 dst over INT_MAX pixels", nv12(2, 8, 8, 8, 65536, 32768, plan.data_ptr()), -1),
    ]
    torch.cuda.synchronize()
    for what, rc, want in cases:
        assert rc == want, (what, rc)
    assert L.scn_launch_count() == before
    assert (dst.cpu().numpy() == SENTINEL).all()
    # the 2x path needs no plan, on both entry points
    assert rgb(1, 8, 8, 4, 4, None) == 0 and nv12(1, 8, 8, 8, 4, 4, None) == 0


# ---------------------------------------------------------------------------------------------- the op
@pytest.fixture(scope="module")
def std_args():
    import os
    E.load_stdlib()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return protolite.parse_proto(open(os.path.join(root, "scanner_b200", "csrc", "ops", "stdlib_args.proto")).read())


TARGETS = {                                  # ResizeArgs for a 640 x 360 source
    "given": {"width": 100, "height": 37},
    "aspect_w0": {"width": 0, "height": 90, "preserve_aspect": True},
    "aspect_h0": {"width": 200, "height": 0, "preserve_aspect": True},
    "min_smaller_source": {"width": 1000, "height": 1000, "min": True},
    "min_larger_source": {"width": 320, "height": 200, "min": True},
}


def _target(sw, sh, a):
    return oracle.resize_target(sw, sh, a.get("width", 0), a.get("height", 0), a.get("min", False),
                                a.get("preserve_aspect", False))


def _run_targets(std_args, add_source, targets):
    """One graph: the source feeding one Resize per ResizeArgs of `targets` -> {name: [frames]}."""
    eng = E.Engine(gpus=[0], instances_per_gpu=2)
    try:
        sid = add_source(eng)
        g = E.Graph()
        src = g.add_source(True)
        ops = {k: g.add_op("Resize", [(src, "frame")], device=1) for k in targets}
        sinks = {k: g.add_sink((op, "frame")) for k, op in ops.items()}
        j = E.Job()
        j.bind_source(src, sid)
        for k, a in targets.items():
            j.set_stream_args(ops[k], protolite.encode(std_args["ResizeArgs"], a))
        eng.run(g, [j], 4, 8)
        return {k: [j.output_row(s, i) for i in range(j.output_rows(s))] for k, s in sinks.items()}, \
            eng.stats()["counters"]["frames_delivered_nv12"]
    finally:
        eng.close()


def _check_targets(got, frames):
    h, w = frames.shape[1:3]
    for k, a in TARGETS.items():
        tw, th = _target(w, h, a)
        assert len(got[k]) == len(frames), k
        for i, f in enumerate(got[k]):
            assert f.shape == (th, tw, 3) and (f == oracle.resize(frames[i], tw, th)).all(), (k, i)
    for i, f in enumerate(got["min_smaller_source"]):
        assert (f == frames[i]).all(), i


def test_op_targets_on_host_frames(std_args):
    frames = np.stack([synth.rand_frame(600 + i, 360, 640) for i in range(5)])
    frames[3], frames[4] = 0, 255
    got, _ = _run_targets(std_args, lambda eng: eng.add_raw_frames(frames), TARGETS)
    _check_targets(got, frames)


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


def test_op_gives_the_same_bytes_from_nv12_and_from_rgb24_elements(std_args, monkeypatch):
    n = 6
    data, shown = _clip(61, n, 360, 640, 3)
    monkeypatch.delenv("SCN_DECODE_RGB", raising=False)
    nv12, delivered = _run_targets(std_args, lambda eng: eng.add_h264(data), TARGETS)
    assert delivered >= n
    monkeypatch.setenv("SCN_DECODE_RGB", "1")
    rgb, delivered = _run_targets(std_args, lambda eng: eng.add_h264(data), TARGETS)
    assert delivered == 0
    _check_targets(nv12, shown)
    _check_targets(rgb, shown)


def test_plan_cache_keeps_geometries_of_streams_apart(std_args):
    """Streams of different source sizes and one target through a single pipeline instance: each run of the op must
    use the plan of its own source size, so a cache key without the source width or without its height fails.  The
    streams grow, so a plan of an earlier stream never addresses past a later stream's frames."""
    streams = [np.stack([synth.rand_frame(700 + 10 * k + i, h, w) for i in range(3)])
               for k, (h, w) in enumerate([(48, 64), (48, 96), (72, 96)])]
    eng = E.Engine(gpus=[0], instances_per_gpu=1)
    try:
        g = E.Graph()
        src = g.add_source(True)
        rz = g.add_op("Resize", [(src, "frame")], device=1)
        sink = g.add_sink((rz, "frame"))
        jobs = []
        for frames in streams:
            j = E.Job()
            j.bind_source(src, eng.add_raw_frames(frames))
            j.set_stream_args(rz, protolite.encode(std_args["ResizeArgs"], {"width": 40, "height": 30}))
            jobs.append(j)
        eng.run(g, jobs, 4, 8)
        assert eng.stats()["counters"]["instances"] == 1
        for frames, j in zip(streams, jobs):
            assert j.output_rows(sink) == len(frames)
            for i in range(len(frames)):
                assert (j.output_row(sink, i) == oracle.resize(frames[i], 40, 30)).all(), (frames.shape, i)
    finally:
        eng.close()


def test_unparsable_args_fail_the_run_and_the_engine_goes_on(std_args):
    frames = np.stack([synth.rand_frame(800 + i, 24, 32) for i in range(3)])
    eng = E.Engine(gpus=[0], instances_per_gpu=1)
    try:
        sid = eng.add_raw_frames(frames)
        g = E.Graph()
        src = g.add_source(True)
        rz = g.add_op("Resize", [(src, "frame")], device=1)
        sink = g.add_sink((rz, "frame"))
        j = E.Job()
        j.bind_source(src, sid)
        j.set_stream_args(rz, b"\x08\xff")   # field 1, a varint that never ends
        with pytest.raises(E.EngineError, match=r"Resize, row 0: could not parse ResizeArgs"):
            eng.run(g, [j], 4, 8)
        j = E.Job()
        j.bind_source(src, sid)
        j.set_stream_args(rz, protolite.encode(std_args["ResizeArgs"], {"width": 16, "height": 12}))
        eng.run(g, [j], 4, 8)
        for i in range(3):
            assert (j.output_row(sink, i) == oracle.resize(frames[i], 16, 12)).all(), i
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


def test_bad_targets_and_gray_frames_fail_the_run_and_the_client_goes_on(sc):
    big = np.random.default_rng(9).integers(0, 256, (2, 1080, 1920, 3), dtype=np.uint8)
    with pytest.raises(sp.ScannerException, match=r"Resize, row 0: invalid target size 1x0 for a 1920x1080 frame"):
        _resize_op(sc, "aspect", big, width=[1], height=[0], preserve_aspect=[True])
    with pytest.raises(sp.ScannerException, match=r"Resize, row 0: invalid target size 0x0"):
        _resize_op(sc, "zero", big[:1], width=[0], height=[0])
    rgb = np.random.default_rng(10).integers(0, 256, (4, 6, 10, 3), dtype=np.uint8)
    frames = sc.io.Input([sp.NamedVideoStream(sc, "rgb", frames=rgb)])
    gray = sc.ops.ConvertColor(frame=frames, conversion=["COLOR_RGB2GRAY"])
    with pytest.raises(sp.ScannerException, match=r"Resize, row 0: expects HxWx3 uint8 frames, got 6x10x1"):
        sc.run(sc.io.Output(sc.ops.Resize(frame=gray, device=sp.DeviceType.GPU, width=[5], height=[3]),
                            [sp.NamedVideoStream(sc, "gray_small")]), sp.PerfParams.estimate())
    # the same client goes on
    got = _resize_op(sc, "good", rgb, width=[7], height=[13])
    assert len(got) == 4
    for i in range(4):
        assert (got[i] == oracle.resize(rgb[i], 7, 13)).all(), i
