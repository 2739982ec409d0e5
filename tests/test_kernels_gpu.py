"""Parity of the sm_90a kernels (called through the C ABI) against the oracle and the
committed golden vectors.  Integer / byte work: every comparison is bit-exact."""
import os

import numpy as np
import pytest
import torch

import oracle
from oracle import synth
from scanner_b200 import cabi, kernels

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _cases(npz):
    return sorted(k[:-5] for k in npz.files if k.endswith("_meta"))


# ----------------------------------------------------------------------------- histogram
def test_hist_golden_cv2(golden_dir):
    g = np.load(os.path.join(golden_dir, "hist_cv2.npz"))
    for k in _cases(g):
        meta = g[k + "_meta"]
        if meta[3] == 2:
            img = np.full((meta[1], meta[2], 3), meta[0], np.uint8)
        else:
            img = synth.frame(int(meta[0]), int(meta[1]), int(meta[2]), int(meta[3]))
        got = kernels.histogram(dev(img[None]))[0].cpu().numpy()
        assert (got == g[k + "_hist"]).all(), k


@pytest.mark.parametrize("h,w,n", [(480, 640, 5), (1080, 1920, 3), (17, 31, 4), (1, 1, 2), (2, 3, 70),
                                   (240, 1, 3), (333, 77, 2)])
def test_hist_vs_oracle_batches(h, w, n):
    frames = np.stack([synth.rand_frame(10 + i, h, w) for i in range(n)])
    got = kernels.histogram(dev(frames)).cpu().numpy()
    for i in range(n):
        assert (got[i] == oracle.hist16(frames[i])).all(), i
    assert (got.sum(axis=(1, 2)) == 3 * h * w).all()


def test_hist_pointer_list_and_misaligned_frames():
    # frames carved at odd byte offsets out of one buffer -> generic (unaligned) path
    h, w = 37, 53
    raw = np.random.default_rng(3).integers(0, 256, 5 + 3 * (h * w * 3 + 7), dtype=np.uint8)
    buf = dev(raw)
    offs = [5 + i * (h * w * 3 + 7) for i in range(3)]
    views = [buf[o:o + h * w * 3].view(h, w, 3) for o in offs]
    got = kernels.histogram(views).cpu().numpy()
    for i, o in enumerate(offs):
        assert (got[i] == oracle.hist16(raw[o:o + h * w * 3].reshape(h, w, 3))).all()


def test_hist_empty_batch_and_overwrite():
    l = cabi.lib()
    assert l.scn_hist16_u8c3_strided(None, 0, 0, 4, 4, None, None) == 0
    # `out` is fully overwritten even if it held garbage
    frames = dev(synth.rand_frame(1, 8, 8)[None])
    out = torch.full((1, 3, 16), 12345, dtype=torch.int32, device="cuda")
    rc = l.scn_hist16_u8c3_strided(frames.data_ptr(), 8 * 8 * 3, 1, 8, 8, out.data_ptr(), None)
    torch.cuda.synchronize()
    assert rc == 0 and out.sum().item() == 3 * 64


def test_hist_full_size_property():
    """1080p x 64 (BASELINE size): sum of bins == 3*W*H per frame and linear in concatenation."""
    g = torch.Generator(device="cuda").manual_seed(5)
    frames = torch.randint(0, 256, (64, 1080, 1920, 3), dtype=torch.uint8, device="cuda", generator=g)
    hist = kernels.histogram(frames)
    assert (hist.sum(dim=(1, 2)) == 3 * 1080 * 1920).all()
    ref = torch.stack([torch.bincount((frames[:, :, :, c] >> 4).flatten().int() +
                                      16 * torch.arange(64, device="cuda").repeat_interleave(1080 * 1920).int(),
                                      minlength=64 * 16).view(64, 16) for c in range(3)], 1)
    assert (hist == ref.int()).all()


# ----------------------------------------------------------------------------- resize
def test_resize_golden_cv2(golden_dir):
    g = np.load(os.path.join(golden_dir, "resize_cv2.npz"))
    for k in _cases(g):
        seed, h, w, dh, dw, kind = [int(x) for x in g[k + "_meta"]]
        img = synth.frame(seed, h, w, kind)
        got = kernels.resize(dev(img[None]), dw, dh)[0].cpu().numpy()
        assert (got == g[k + "_out"]).all(), (k, h, w, dh, dw)


@pytest.mark.parametrize("h,w,dh,dw,n", [(1080, 1920, 224, 224, 4), (480, 640, 224, 224, 3), (50, 70, 25, 35, 2),
                                         (33, 47, 99, 120, 2), (5, 1, 3, 4, 1)])
def test_resize_vs_oracle_batches(h, w, dh, dw, n):
    frames = np.stack([synth.rand_frame(20 + i, h, w) for i in range(n)])
    got = kernels.resize(dev(frames), dw, dh).cpu().numpy()
    for i in range(n):
        assert (got[i] == oracle.resize(frames[i], dw, dh)).all()


def test_resize_missing_plan_is_an_error():
    f = dev(synth.rand_frame(1, 8, 8)[None])
    out = torch.empty((1, 3, 3, 3), dtype=torch.uint8, device="cuda")
    rc = cabi.lib().scn_resize_bilinear_u8c3_strided(f.data_ptr(), 192, 1, 8, 8, out.data_ptr(), 27, 3, 3, None, None)
    assert rc == -3


# ----------------------------------------------------------------------------- blur
def test_blur_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "blur_np.npz"))
    for k in _cases(g):
        seed, h, w, ks = [int(x) for x in g[k + "_meta"]]
        img = synth.rand_frame(seed, h, w)
        got = kernels.blur(dev(img[None]), ks)[0].cpu().numpy()
        assert (got == g[k + "_out"]).all(), (k, h, w, ks)


@pytest.mark.parametrize("h,w,k,n", [(480, 640, 3, 2), (2160, 3840, 3, 1), (100, 70, 7, 3), (65, 129, 31, 1),
                                     (10, 10, 12, 1), (33, 50, 3, 2), (3, 4, 3, 1), (70, 1028, 3, 2), (64, 64, 2, 1)])
def test_blur_vs_oracle(h, w, k, n):
    frames = np.stack([synth.rand_frame(30 + i, h, w) for i in range(n)])
    got = kernels.blur(dev(frames), k).cpu().numpy()
    for i in range(n):
        assert (got[i] == oracle.blur(frames[i], k)).all()


@pytest.mark.parametrize("h,w,k,kernel", [(64, 64, 3, "box_packed_kernel"), (64, 64, 5, "box_packed_kernel"),
                                          (70, 1028, 3, "box3_kernel"), (70, 1028, 5, "box_generic_kernel"),
                                          (33, 50, 3, "box_generic_kernel")])
def test_blur_kernel_selection(h, w, k, kernel):
    """16-byte aligned rows at least k tall take box_packed_kernel<K>, k = 3 included; otherwise k = 3 on 4-byte
    aligned rows takes box3_kernel; everything else takes box_generic_kernel."""
    frames = np.stack([synth.rand_frame(50 + i, h, w) for i in range(2)])
    src = dev(frames)
    L = cabi.lib()
    L.scn_prof_enable(1)
    try:
        got = kernels.blur(src, k)
        torch.cuda.synchronize()
        ran = {name: v["launches"] for name, v in cabi.prof_report().items()}
    finally:
        L.scn_prof_enable(0)
    assert ran == {kernel: 1}
    got = got.cpu().numpy()
    for i in range(2):
        assert (got[i] == oracle.blur(frames[i], k)).all()


def test_div9_multiply_shift_is_exact():
    """box3_kernel divides by 9 with (v * 7282) >> 16: exact for every reachable sum (<= 9*255)."""
    v = np.arange(0, 9 * 255 + 1, dtype=np.uint64)
    assert ((v * 7282) >> 16 == v // 9).all()


# ----------------------------------------------------------------------------- nv12
def _surfaces(seed, n, h, w, pitch):
    out = np.zeros((n, h * 3 // 2, pitch), np.uint8)
    for i in range(n):
        l, c = synth.nv12_surface(seed + i, h, w, pitch)
        out[i, :h], out[i, h:] = l, c
    return out


def test_nv12_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "nv12_np.npz"))
    for k in _cases(g):
        seed, h, w, pitch = [int(x) for x in g[k + "_meta"]]
        l, c = synth.nv12_surface(seed, h, w, pitch)
        surf = np.concatenate([l, c])[None]
        got = kernels.nv12_to_rgb(dev(surf), w, h)[0].cpu().numpy()
        assert (got == g[k + "_out"]).all(), (k, h, w, pitch)


@pytest.mark.parametrize("h,w,pitch,n", [(1080, 1920, 2048, 2), (480, 640, 640, 3), (30, 50, 64, 2), (2, 2, 4, 1),
                                         (16, 18, 18, 2)])
def test_nv12_vs_oracle(h, w, pitch, n):
    surf = _surfaces(40, n, h, w, pitch)
    got = kernels.nv12_to_rgb(dev(surf), w, h).cpu().numpy()
    for i in range(n):
        assert (got[i] == oracle.nv12_to_rgb(surf[i, :h], surf[i, h:], w)).all()


# ----------------------------------------------------------------------------- fused C2 DAG
@pytest.mark.parametrize("h,w,pitch,dh,dw,n", [(1080, 1920, 2048, 224, 224, 3), (480, 640, 640, 224, 224, 2),
                                               (48, 64, 64, 24, 32, 2), (30, 50, 64, 45, 70, 2)])
def test_fused_nv12_hist_resize_vs_oracle(h, w, pitch, dh, dw, n):
    surf = _surfaces(50, n, h, w, pitch)
    hist, res = kernels.nv12_hist_resize(dev(surf), w, h, dw, dh)
    hist, res = hist.cpu().numpy(), res.cpu().numpy()
    for i in range(n):
        oh, orr = oracle.nv12_hist_resize(surf[i, :h], surf[i, h:], dw, dh, w)
        assert (hist[i] == oh).all()
        assert (res[i] == orr).all()


@pytest.mark.parametrize("h,w,pitch,n", [(1080, 1920, 1920, 8), (2160, 3840, 4096, 3)])
def test_fused_equals_three_pass_composition(h, w, pitch, n):
    g = torch.Generator(device="cuda").manual_seed(9)
    surf = torch.randint(0, 256, (n, h * 3 // 2, pitch), dtype=torch.uint8, device="cuda", generator=g)
    hist, res = kernels.nv12_hist_resize(surf, w, h, 224, 224)
    rgb = kernels.nv12_to_rgb(surf, w, h)
    assert (hist == kernels.histogram(rgb)).all()
    assert (res == kernels.resize(rgb, 224, 224)).all()


@pytest.mark.parametrize("h,w,pitch,n", [(1080, 1920, 2048, 3), (30, 50, 64, 2), (48, 64, 80, 2), (2, 2, 4, 1)])
def test_nv12_pack_is_a_byte_copy_and_ops_accept_packed_elements(h, w, pitch, n):
    """The FrameLayout::NV12 element: surface rows without the pitch; Histogram-only / Resize-only
    entry points on it give what the fused call gives on the pitched surface."""
    surf = _surfaces(60, n, h, w, pitch)
    packed = kernels.nv12_pack(dev(surf), w, h)
    assert (packed.cpu().numpy() == surf[:, :, :w]).all()
    dh, dw = max(1, h // 3), max(1, w // 3)
    hist, res = kernels.nv12_hist_resize(dev(surf), w, h, dw, dh)
    h_only, none = kernels.nv12_hist_resize(packed, w, h, dw, dh, want_resize=False)
    none2, r_only = kernels.nv12_hist_resize(packed, w, h, dw, dh, want_hist=False)
    assert none is None and none2 is None
    assert (h_only == hist).all() and (r_only == res).all()


def test_launch_counter_counts():
    before = cabi.lib().scn_launch_count()
    kernels.histogram(dev(synth.rand_frame(1, 8, 8)[None]))
    assert cabi.lib().scn_launch_count() > before


def test_generic_nv12_paths_small_and_ragged():
    """Sizes that miss every vector fast path (odd pitch, width % 4 != 0): the scalar conversion used
    by the generic NV12 histogram / resize kernels and the ragged tails, against the oracle."""
    for (h, w, pitch) in [(18, 22, 23), (34, 46, 51), (66, 130, 131)]:
        surf = _surfaces(70, 2, h, w, pitch)
        rgb = kernels.nv12_to_rgb(dev(surf), w, h).cpu().numpy()
        hist, res = kernels.nv12_hist_resize(dev(surf), w, h, 16, 12)
        for i in range(2):
            want = oracle.nv12_to_rgb(surf[i, :h], surf[i, h:], w)
            assert (rgb[i] == want).all()
            assert (hist[i].cpu().numpy() == oracle.hist16(want)).all()
            assert (res[i].cpu().numpy() == oracle.resize(want, 16, 12)).all()


def test_4k_blur_then_histogram_properties():
    """BASELINE configs[2] at full size: every pixel is counted once per channel, the blurred interior
    equals the oracle on one frame, and Blur -> Histogram equals the histogram of the oracle's blur."""
    h, w, n = 2160, 3840, 2
    g = torch.Generator(device="cuda").manual_seed(21)
    frames = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda", generator=g)
    blurred = kernels.blur(frames, 3)
    hist = kernels.histogram(blurred).cpu().numpy()
    assert (hist.sum(axis=2) == h * w).all()
    f0 = frames[0].cpu().numpy()
    want = oracle.blur(f0, 3)
    got = blurred[0].cpu().numpy()
    assert (got[1:-1, 1:-1] == want[1:-1, 1:-1]).all() and (got[0] == 0).all() and (got[:, 0] == 0).all()
    assert (hist[0] == oracle.hist16(got)).all()


def test_frame_digest_matches_numpy():
    g = torch.Generator(device="cuda").manual_seed(9)
    for shape, dt in (((5, 37, 53, 2), torch.float32), ((3, 270, 480, 3), torch.uint8), ((70, 64, 4), torch.int32)):
        if dt == torch.float32:
            x = torch.randn(shape, device="cuda", generator=g)
        else:
            x = torch.randint(0, 200, shape, device="cuda", generator=g).to(dt)
        if (x[0].numel() * x.element_size()) % 4:
            continue
        got = kernels.frame_digest(x).cpu().numpy().view(np.uint64)
        for i in range(shape[0]):
            w = np.frombuffer(x[i].cpu().numpy().tobytes(), "<u4").astype(np.uint64)
            k = (np.arange(w.size, dtype=np.uint64) % np.uint64(65521)) + np.uint64(1)
            with np.errstate(over="ignore"):
                want = np.array([w.sum(dtype=np.uint64), (w * k).sum(dtype=np.uint64)], np.uint64)
            assert (got[i] == want).all(), (shape, i)


def test_sharded_job_windows_on_one_gpu_equal_the_whole_clip():
    """scn_job_set_shard with every interval owned by this rank (no transport): each job computes its window,
    decoding the stencil rows beyond it itself; the windows together equal the unsharded job.  (The NCCL
    exchange between ranks is exercised by `bench.py --config 3 --gpus N` and, on the CPU, by the gloo test.)"""
    from scanner_b200 import engine as E
    E.load_stdlib()
    w, h, n = 128, 96, 25
    rng = np.random.default_rng(4)
    yuv = rng.integers(0, 256, (n, h * w * 3 // 2), dtype=np.uint8)
    eng = E.Engine(gpus=[0], instances_per_gpu=2)
    sid = eng.add_h264(E.h264_synth(yuv, w, h, gop=6, non_key="pcm"))
    g = E.Graph()
    src = g.add_source(True)
    fl = g.add_op("OpticalFlow", [(src, "frame")], device=1)
    dg = g.add_op("FrameDigest", [(fl, "flow")], device=1)
    sink = g.add_sink((dg, "digest"))
    whole = E.Job()
    whole.bind_source(src, sid)
    eng.run(g, [whole], 4, 8)
    full = whole.output_array(sink, 16, np.uint64)
    assert full.shape == (n, 2)
    bounds = [0, 7, 7, 19, n]  # one empty interval
    parts = []
    for q in range(4):
        j = E.Job()
        j.bind_source(src, sid)
        j.set_shard(q, bounds, [0, 0, 0, 0])
        eng.run(g, [j], 4, 8)
        assert j.output_rows(sink) == bounds[q + 1] - bounds[q]
        parts.append(j.output_array(sink, 16, np.uint64, row0=bounds[q]))
    assert (np.concatenate(parts) == full).all()
    eng.close()


@pytest.mark.parametrize("h,w,k,n", [(480, 640, 5, 2), (2160, 3840, 5, 1), (1080, 1920, 9, 2), (70, 3088, 7, 2), (40, 1040, 31, 1),
                                     (129, 1024, 4, 1), (257, 2064, 6, 2), (131, 48, 2, 3), (31, 16, 31, 1), (200, 1920, 16, 1),
                                     (90, 1040, 5, 2)])
def test_blur_aligned_rows_vs_oracle(h, w, k, n):
    """box_packed_kernel<K> on 16-byte aligned rows: several warps / strips / row ranges, even and odd kernel sizes
    (fl != fr), windows as tall as the frame."""
    assert w % 16 == 0
    frames = np.stack([synth.rand_frame(60 + i, h, w) for i in range(n)])
    l0 = cabi.lib().scn_launch_count()
    got = kernels.blur(dev(frames), k).cpu().numpy()
    assert cabi.lib().scn_launch_count() > l0
    for i in range(n):
        want = oracle.blur(frames[i], k)
        assert (got[i] == want).all(), (i, np.argwhere(got[i] != want)[:4])


@pytest.mark.parametrize("k", list(range(2, 32)))
def test_blur_packed_kernel_every_size_vs_oracle(k):
    """box_packed_kernel<K> (u16x2 lanes): every kernel size it serves, a row narrower than one warp's span and one
    that needs several warps with a ragged tail, strips that end inside the frame, and all-255 frames (the lane sums
    reach 255 k^2 -- 65280 at k = 16 -- and must not carry into the neighbouring lane; above 16 the terms are summed
    in groups of 8 and the groups unpacked)."""
    for (h, w, n) in [(67, 144, 2), (140, 2064, 1), (k + 1, 16, 1)]:
        frames = np.stack([synth.rand_frame(90 + k + i, h, w) for i in range(n)])
        frames[-1, : h // 2] = 255
        got = kernels.blur(dev(frames), k).cpu().numpy()
        for i in range(n):
            want = oracle.blur(frames[i], k)
            assert (got[i] == want).all(), (k, h, w, i, np.argwhere(got[i] != want)[:4])
    sat = np.full((1, 40, 64, 3), 255, np.uint8)
    got = kernels.blur(dev(sat), k).cpu().numpy()[0]
    assert (got == oracle.blur(sat[0], k)).all()


@pytest.mark.parametrize("k", [17, 18, 21, 24, 27, 30, 31])
def test_blur_packed_kernel_large_sizes_vs_oracle(k):
    """Kernel sizes above 16, where box_packed_kernel<K> sums the terms in groups of 8 (a u16 lane no longer holds K
    terms), on frames several warps wide with a saturated band."""
    frames = np.stack([synth.rand_frame(400 + k + i, 90, 1040) for i in range(2)])
    frames[1, 20:70] = 255
    got = kernels.blur(dev(frames), k).cpu().numpy()
    for i in range(2):
        want = oracle.blur(frames[i], k)
        assert (got[i] == want).all(), (k, i, np.argwhere(got[i] != want)[:4])


def test_blur_division_by_multiply_shift_is_exact():
    """box_packed_kernel<K> divides a window sum by k*k with umulhi(v, floor(2^32 / k^2) + 1)."""
    for k in range(2, 32):
        d = k * k
        v = np.arange(0, 255 * d + 1, dtype=np.uint64)
        m = np.uint64((1 << 32) // d + 1)
        assert (((v * m) >> np.uint64(32)) == v // np.uint64(d)).all(), k
