"""The three Blur kernels (blur.cu) and the Blur op, byte for byte against oracle.blur_sat (the summed-area-table
restatement of the box filter, held to oracle.blur for every kernel size by tests/test_blur_cpu.py), border included:
  * box_packed_kernel<K> at every combination of halo R in {1, 2, 3} and strip height in {32, 64, 128}, which the
    launcher picks from the grid size and the device's SM count (restated here and asserted to be reached on the
    device the test runs on), at heights 0, 1 and -1 mod the strip, at heights k and k + 1, at the Blur op's own call
    (16 frames of 1080p and of 4K) and in a 66-frame call whose two chunks get different strip heights;
  * its warp and CTA edges: widths whose quad count lies around multiples of the output quads per warp and per CTA,
    a last CTA with 1 to 4 active warps, a row narrower than the halo;
  * lane content that drives one packed u16 lane to 255 K (vertically) or 255 K^2 (horizontally) beside a zero lane,
    and bands that saturate one 8-term group above K = 16;
  * box3_kernel at widths 4, 8 and 12 mod 16, on both sides of its 256-thread CTA, at 4-byte offsets, at heights
    around its 64-row strips; box_generic_kernel at byte offsets 1-15, around its 64 x 32 tile, at k 1, 2, 4, 30, 31;
  * the kernel each 64-frame chunk of one call takes, and the height that makes a frame eligible for the packed kernel;
  * refusals, which launch nothing and write nothing.
Every call writes into outputs pre-filled with 0x00 in one run and 0xFF in another, laid out in one buffer with
guard bytes between frames that must stay untouched.  The Blur and Histogram ops then run through the engine at the
op's 16-frame calls, and bad input fails the run with the op, the row and the reason while the client goes on."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import oracle  # noqa: E402
import scanner_b200 as sp  # noqa: E402
from scanner_b200 import cabi, protolite  # noqa: E402
from scanner_b200 import engine as E  # noqa: E402

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
GUARD = 64  # bytes after every frame (and before it, when it sits at an offset) that a call must not touch
FILLS = (0x00, 0xFF)
CHUNK = 64  # frames per launch


# ----------------------------------------------------------------------------- the launcher, restated
def halo(k):
    """R: halo quads on each side of a box_packed_kernel<K> thread's quad."""
    return (3 * (k // 2) + 15) // 16


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def strip_rows(w, h, k, cnt, sms):
    """Rows per strip of box_packed_kernel<K> for a chunk of `cnt` frames: 128, halved down to 32 while the grid has
    fewer than two CTAs per SM; a CTA is 4 warps of 32 - 2R output quads (16 bytes)."""
    out_quads = 32 - 2 * halo(k)
    gx = -(-(w * 3 // 16) // (4 * out_quads))
    rows = 128
    while rows > 32 and gx * -(-h // rows) * cnt < 2 * sms:
        rows //= 2
    return rows


def last_cta_warps(w, k):
    warps = -(-(w * 3 // 16) // (32 - 2 * halo(k)))
    return (warps - 1) % 4 + 1


def chunk_rows(w, h, k, n, sms):
    return [strip_rows(w, h, k, min(CHUNK, n - i0), sms) for i0 in range(0, n, CHUNK)]


# ----------------------------------------------------------------------------- calls
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


def _offsets(off, n):
    return [off] * n if isinstance(off, int) else list(off)


def blur_list(frames, k, fill, src_off=0, dst_off=0):
    """scn_box_blur_u8c3 over pointer lists into one device buffer per side: frame i at byte i * stride + offset
    (offset 0 is 16-byte aligned), every output pre-filled with `fill` and surrounded by SENTINEL bytes that must
    survive.  -> (outputs (n, h, w, 3), {kernel: launches})."""
    n, h, w, _ = frames.shape
    fb = h * w * 3
    stride = (fb + GUARD + 16 + 15) // 16 * 16
    so, do = _offsets(src_off, n), _offsets(dst_off, n)
    host = np.zeros((n, stride), np.uint8)
    want_dst = np.full((n, stride), SENTINEL, np.uint8)
    for i in range(n):
        host[i, so[i]:so[i] + fb] = frames[i].reshape(-1)
        want_dst[i, do[i]:do[i] + fb] = fill
    src = torch.from_numpy(host).cuda()
    dst = torch.from_numpy(want_dst).cuda()
    base_s, base_d = src.data_ptr(), dst.data_ptr()
    ps, keep_s = cabi.ptr_array([base_s + i * stride + so[i] for i in range(n)])
    pd, keep_d = cabi.ptr_array([base_d + i * stride + do[i] for i in range(n)])
    rc, ran = _ran(lambda: cabi.lib().scn_box_blur_u8c3(ps, n, w, h, k, pd, None))
    assert rc == 0, rc
    got = dst.cpu().numpy()
    outs = np.empty_like(frames)
    for i in range(n):
        outs[i] = got[i, do[i]:do[i] + fb].reshape(h, w, 3)
        got[i, do[i]:do[i] + fb] = SENTINEL
    bad = np.argwhere(got != SENTINEL)
    assert bad.size == 0, f"bytes outside the frames written: (frame, byte) {bad[:8].tolist()}"
    return outs, ran


def check(frames, k, want=None, kernel=None, launches=None, **offsets):
    """blur_list at both fills, every frame == oracle.blur_sat, and (optionally) the kernel that ran."""
    if want is None:
        want = oracle.blur_sat(frames, k)
    for fill in FILLS:
        got, ran = blur_list(frames, k, fill, **offsets)
        for i in range(len(frames)):
            if not np.array_equal(got[i], want[i]):
                bad = np.argwhere(got[i] != want[i])
                pytest.fail(f"k={k} {frames.shape[1]}x{frames.shape[2]} frame {i} fill {fill:#x}: {len(bad)} samples "
                            f"differ, first (y, x, c) {bad[:4].tolist()}")
        if kernel is not None:
            assert set(ran) == {kernel}, ran
        if launches is not None:
            assert ran.get(kernel) == launches, ran
    return ran


def rand_frames(seed, n, h, w):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


# ----------------------------------------------------------------------------- strip heights
# (k, h, w, n): each halo R in {1, 2, 3} (k <= 11, <= 21, <= 31) at each strip height on 132 SMs, at heights 0, 1 and
# -1 mod the strip, and at heights k and k + 1
STRIP_CASES = (
    [(k, h, 1920, 16) for k, h in [(3, 768), (7, 769), (11, 767), (12, 768), (16, 769), (21, 767),
                                     (22, 768), (27, 769), (31, 767)]] +
    [(k, h, 1920, 4) for k, h in [(3, 1408), (7, 1409), (11, 1407), (12, 1088), (16, 1089), (21, 1087),
                                    (22, 1088), (27, 1089), (31, 1087)]] +
    [(k, h, 1920, 2) for k, h in [(3, 256), (7, 257), (11, 255), (12, 256), (16, 257), (21, 255),
                                    (22, 256), (27, 257), (31, 255)]] +
    [(k, h, 1920, 2) for k in (2, 3, 11, 12, 21, 22, 31) for h in (k, k + 1)]
)
OP_CALLS = [(3, 1080, 1920, 16), (3, 2160, 3840, 16)]   # the Blur op's batch of 16 at 1080p and 4K
SPLIT_CALLS = [(3, 1024, 1024, 66), (31, 1024, 1024, 66)]  # a 64-frame chunk and a 2-frame chunk in one call


def test_strip_height_coverage_holds_on_this_device():
    """The geometries below reach every halo x strip-height combination, and the 66-frame calls get two different
    strip heights, on the device the suite runs on."""
    sms = sm_count()
    seen = {(halo(k), strip_rows(w, h, k, n, sms)) for (k, h, w, n) in STRIP_CASES + OP_CALLS}
    want = {(r, rows) for r in (1, 2, 3) for rows in (32, 64, 128)}
    assert want <= seen, f"on {sms} SMs the strip cases miss (R, rows) {sorted(want - seen)}"
    for (k, h, w, n) in SPLIT_CALLS:
        rows = chunk_rows(w, h, k, n, sms)
        assert len(set(rows)) == 2, f"on {sms} SMs the {n}-frame call at k = {k} gets strip heights {rows}"
    for (k, h, w, n) in OP_CALLS:
        assert strip_rows(w, h, k, n, sms) == 128, f"on {sms} SMs the Blur op's call {n} x {w}x{h} is not 128 rows"
    # and the heights sit at 0, 1 and -1 modulo the strips they get
    for rows in (32, 64, 128):
        mods = {h % rows for (k, h, w, n) in STRIP_CASES if strip_rows(w, h, k, n, sms) == rows}
        assert {0, 1, rows - 1} <= mods, (sms, rows, sorted(mods))


@pytest.mark.parametrize("k,h,w,n", STRIP_CASES)
def test_packed_kernel_at_every_strip_height(k, h, w, n):
    frames = rand_frames(100 * k + h, n, h, w)
    frames[-1, : h // 2] = 255  # a saturated upper half
    check(frames, k, kernel="box_packed_kernel", launches=1)


@pytest.mark.parametrize("k,h,w,n", OP_CALLS)
def test_packed_kernel_at_the_blur_ops_call(k, h, w, n):
    check(rand_frames(7 + h, n, h, w), k, kernel="box_packed_kernel", launches=1)


@pytest.mark.parametrize("k,h,w,n", SPLIT_CALLS)
def test_packed_kernel_chunks_of_different_strip_heights_in_one_call(k, h, w, n):
    frames = rand_frames(31 + k, n, h, w)
    frames[CHUNK - 1] = 255
    frames[CHUNK] = 255
    check(frames, k, kernel="box_packed_kernel", launches=2)


# ----------------------------------------------------------------------------- warp and CTA edges, lane content
EDGE_WIDTHS = {  # quad counts 3W/16 below, at and above multiples of 32 - 2R and of 4 (32 - 2R)
    1: [16, 144, 160, 176, 320, 336, 480, 496, 640, 656],
    2: [16, 160, 320, 448, 480, 592, 640],
    3: [16, 144, 320, 416, 448, 480, 544, 560, 592],
}
EDGE_KS = {1: (3, 11), 2: (12, 21), 3: (22, 31)}


def test_edge_widths_reach_every_last_cta_size():
    for r, widths in EDGE_WIDTHS.items():
        assert {last_cta_warps(w, EDGE_KS[r][0]) for w in widths} == {1, 2, 3, 4}, r


@pytest.mark.parametrize("r,k", [(r, k) for r, ks in EDGE_KS.items() for k in ks])
def test_packed_kernel_warp_and_cta_edges(r, k):
    assert halo(k) == r
    for w in EDGE_WIDTHS[r]:
        h = k + 37
        frames = rand_frames(w + k, 3, h, w)
        frames[1] = 255
        frames[2, :, :] = patterned(h, w, 3, 0)
        check(frames, k, kernel="box_packed_kernel", launches=1)


def patterned(h, w, period, phase):
    """255 at the bytes whose index in the row is `phase` mod `period`, 0 elsewhere."""
    row = np.where(np.arange(w * 3) % period == phase, 255, 0).astype(np.uint8)
    return np.broadcast_to(row.reshape(w, 3), (h, w, 3)).copy()


def lane_frames(k, h, w):
    f = [np.full((h, w, 3), 255, np.uint8), rand_frames(k, 1, h, w)[0]]
    alt = np.zeros((h, w, 3), np.uint8)
    alt[::2] = 255
    f += [alt, 255 - alt]
    f += [patterned(h, w, 3, p) for p in range(3)] + [patterned(h, w, 4, p) for p in range(4)]
    # patterns that also alternate by row: one lane at 255 K vertically only on every other window row
    f += [np.where(alt == 255, patterned(h, w, 4, 1), 0).astype(np.uint8)]
    x = np.arange(w)[None, :, None]
    # bands of 8 saturated pixels: above K = 16 one 8-term group of a window sums to 8 x 255 K beside empty groups
    f += [np.broadcast_to(np.where(x % 16 < 8, 255, 0), (h, w, 3)).astype(np.uint8),
          np.broadcast_to(np.where(x % k < 8, 255, 0), (h, w, 3)).astype(np.uint8),
          np.broadcast_to(np.where((x + k // 2) % (2 * k) < 8, 255, 0), (h, w, 3)).astype(np.uint8)]
    return np.stack(f)


@pytest.mark.parametrize("k", range(2, 32))
def test_packed_kernel_lane_content(k):
    check(lane_frames(k, 2 * k + 35, 656), k, kernel="box_packed_kernel", launches=1)


# ----------------------------------------------------------------------------- box3_kernel
B3_WIDTHS = [4, 20, 24, 28, 76, 340, 344, 1036]  # 4, 8, 12 mod 16; 340 / 344: 255 / 258 words per row
B3_HEIGHTS = [3, 4, 5, 6, 64, 65, 66, 67, 128, 129, 130, 131]


@pytest.mark.parametrize("w", B3_WIDTHS)
def test_box3_kernel_widths_and_heights(w):
    assert w % 16 and w % 4 == 0
    for h in B3_HEIGHTS:
        frames = rand_frames(w * 1000 + h, 2, h, w)
        frames[1, ::2] = 255
        check(frames, 3, kernel="box3_kernel", launches=1)


@pytest.mark.parametrize("src_off,dst_off", [(4, 0), (0, 4), (4, 12), (8, 8)])
def test_box3_kernel_at_4_byte_offsets(src_off, dst_off):
    for h in (3, 64, 67, 131):
        frames = rand_frames(h, 3, h, 1024)
        frames[2] = patterned(h, 1024, 4, 1)
        check(frames, 3, kernel="box3_kernel", launches=1, src_off=src_off, dst_off=dst_off)


# ----------------------------------------------------------------------------- box_generic_kernel
@pytest.mark.parametrize("k", [1, 2, 4, 30, 31])
def test_generic_kernel_around_its_tile_at_byte_offsets(k):
    cases = [(h, w) for h in (31, 32, 33) for w in (63, 64, 65)] + [(k - 1, 70), (70, k - 1), (k, k), (1, 1),
                                                                     (2, 129), (97, 2)]
    for j, (h, w) in enumerate(c for c in cases if c[0] > 0 and c[1] > 0):
        frames = rand_frames(k * 100 + j, 3, h, w)
        frames[1] = 255
        offs = [(j + 1 + 5 * i) % 15 + 1 for i in range(3)]  # 1..15
        check(frames, k, kernel="box_generic_kernel", launches=1, src_off=offs, dst_off=offs[::-1])
    # widths that are not a multiple of 4 take the generic kernel at any alignment
    for w in (5, 7, 18, 66, 130):
        frames = rand_frames(k + w, 2, 40, w)
        check(frames, k, kernel="box_generic_kernel", launches=1)


# ----------------------------------------------------------------------------- kernel choice
def test_each_chunk_takes_its_own_kernel():
    """130 frames at k = 3 (W = 48, a multiple of 16): the chunks of frames 0-63 and 128-129 are 16-byte aligned and
    take box_packed_kernel; the chunk of frames 64-127 holds one frame that is only 4-byte aligned and takes
    box3_kernel."""
    frames = rand_frames(130, 130, 32, 48)
    offs = [0] * 130
    offs[100] = 4
    ran = check(frames, 3, src_off=offs)
    assert ran == {"box_packed_kernel": 2, "box3_kernel": 1}, ran
    ran = check(frames, 3, dst_off=offs)
    assert ran == {"box_packed_kernel": 2, "box3_kernel": 1}, ran


@pytest.mark.parametrize("k", [2, 3, 5, 16, 17, 31])
def test_packed_kernel_eligibility_starts_at_height_k(k):
    check(rand_frames(k, 2, k - 1, 64), k, kernel="box_generic_kernel", launches=1)  # h = k - 1: all border, generic kernel
    check(rand_frames(k + 1, 2, k, 64), k, kernel="box_packed_kernel", launches=1)


# ----------------------------------------------------------------------------- refusals
REFUSALS = [  # (n, width, height, kernel_size, return code)
    (-1, 16, 16, 3, -1), (1, 16, 16, 0, -1), (1, 16, 16, 32, -1), (1, (1 << 29) + 1, 1, 3, -1),
    (1, 2**31 - 1, 1, 1, -1), (1, 1, 65535 * 32 + 1, 3, -2), (2, 16, 2**31 - 1, 3, -2),
]


def test_refusals_launch_nothing_and_write_nothing():
    L = cabi.lib()
    src = torch.randint(0, 256, (2, 16 * 16 * 3), dtype=torch.uint8, device="cuda")
    dst = torch.full((2, 16 * 16 * 3), SENTINEL, dtype=torch.uint8, device="cuda")
    ps, keep_s = cabi.ptr_array([src[i].data_ptr() for i in range(2)])
    pd, keep_d = cabi.ptr_array([dst[i].data_ptr() for i in range(2)])
    torch.cuda.synchronize()
    before = L.scn_launch_count()
    for (n, w, h, k, rc) in REFUSALS:
        assert L.scn_box_blur_u8c3(ps, n, w, h, k, pd, None) == rc, (n, w, h, k)
        assert L.scn_box_blur_u8c3_strided(src.data_ptr(), 768, n, w, h, k, dst.data_ptr(), None) == rc, (n, w, h, k)
    assert L.scn_box_blur_u8c3(None, 1, 16, 16, 3, pd, None) == -1
    assert L.scn_box_blur_u8c3(ps, 1, 16, 16, 3, None, None) == -1
    assert L.scn_box_blur_u8c3_strided(None, 768, 1, 16, 16, 3, dst.data_ptr(), None) == -1
    assert L.scn_box_blur_u8c3(ps, 0, 16, 16, 3, pd, None) == 0
    torch.cuda.synchronize()
    assert L.scn_launch_count() == before
    assert (dst == SENTINEL).all()


# ----------------------------------------------------------------------------- the ops through the engine
@pytest.fixture(scope="module")
def std_args():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    E.load_stdlib()
    return protolite.parse_proto(open(os.path.join(root, "scanner_b200", "csrc", "ops", "stdlib_args.proto")).read())


def test_blur_op_and_blur_then_histogram_at_16_frame_calls(std_args):
    """32 raw 1080p frames in packets of 16: two Blur calls of 16 frames, each one box_packed_kernel<3> launch of
    128-row strips; every frame whole (border included) and Blur -> Histogram against the restatement."""
    n, h, w = 32, 1080, 1920
    assert strip_rows(w, h, 3, 16, sm_count()) == 128
    frames = rand_frames(1080, n, h, w)
    frames[5] = 255
    want = oracle.blur_sat(frames, 3)
    eng = E.Engine(gpus=[0], instances_per_gpu=1)
    try:
        g = E.Graph()
        src = g.add_source(True)
        bl = g.add_op("Blur", [(src, "frame")], device=1,
                      args=protolite.encode(std_args["BlurArgs"], {"kernel_size": 3, "sigma": 0.5}))
        hs = g.add_op("Histogram", [(bl, "frame")], device=1)
        s_b, s_h = g.add_sink((bl, "frame")), g.add_sink((hs, "histogram"))
        j = E.Job()
        j.bind_source(src, eng.add_raw_frames(frames))
        _, ran = _ran(lambda: eng.run(g, [j], 16, 16))
        assert ran.get("box_packed_kernel") == 2, ran
        assert not {"box3_kernel", "box_generic_kernel"} & set(ran), ran
        assert j.output_rows(s_b) == n and j.output_rows(s_h) == n
        hist = j.output_array(s_h, 192, np.int32).reshape(n, 3, 16)
        for i in range(n):
            assert np.array_equal(j.output_row(s_b, i), want[i]), i
            assert (hist[i] == oracle.hist16(want[i])).all(), i
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


def test_bad_blur_and_histogram_input_fails_the_run_and_the_client_goes_on(sc):
    G = sp.DeviceType.GPU
    rgb = rand_frames(11, 4, 16, 24)

    def gray(inp):
        return sc.ops.ConvertColor(frame=inp, conversion=["COLOR_RGB2GRAY"])

    with pytest.raises(sp.ScannerException, match=r"Histogram, row 0: expects HxWx3 uint8 frames, got 16x24x1"):
        _run_op(sc, "g1", rgb, lambda f: sc.ops.Histogram(frame=gray(f), device=G))
    with pytest.raises(sp.ScannerException, match=r"Blur, row 0: expects HxWx3 uint8 frames, got 16x24x1"):
        _run_op(sc, "g2", rgb, lambda f: sc.ops.Blur(frame=gray(f), kernel_size=3, sigma=0.5, device=G))
    with pytest.raises(sp.ScannerException, match=r"Blur, row 0: expects HxWx3 uint8 frames, got 16x24x2 type 1"):
        _run_op(sc, "flow", rgb, lambda f: sc.ops.Blur(frame=sc.ops.OpticalFlow(frame=f, device=G), kernel_size=3,
                                                       sigma=0.5, device=G))
    tall = rand_frames(3, 1, 65535 * 32 + 1, 1)  # 6.3 MB; one row past what the launcher takes
    with pytest.raises(sp.ScannerException, match=r"Blur, row 0: scn_box_blur_u8c3 failed with code -2"):
        _run_op(sc, "tall", tall, lambda f: sc.ops.Blur(frame=f, kernel_size=3, sigma=0.5, device=G))
    # the same client goes on
    got = _run_op(sc, "good", rgb, lambda f: sc.ops.Blur(frame=f, kernel_size=5, sigma=0.5, device=G))
    assert len(got) == 4
    for i in range(4):
        assert np.array_equal(got[i], oracle.blur(rgb[i], 5)), i
    hist = _run_op(sc, "good_h", rgb, lambda f: sc.ops.Histogram(frame=f, device=G))
    assert len(hist) == 4
    for i in range(4):
        assert (np.stack(hist[i]) == oracle.hist16(rgb[i])).all(), i
