"""scn_h264_encode_u8 on the GPU, byte for byte against oracle/h264_enc.py (itself held to FFmpeg in
tests/test_h264_encode_cpu.py): the CPU sweep, 1080p and 2160p frames, batches over 64 frames, unaligned frames,
outputs pre-filled with 0x00 and 0xFF and followed by guard bytes.  The engine's decoder then reads the kernel's
streams back to exactly the oracle's reconstruction, chroma included."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from helpers import guarded_output
from helpers.h264_cases import epb_seam_frames
from oracle import h264_enc as H
from scanner_b200 import cabi, kernels
from scanner_b200 import engine as E

pytestmark = pytest.mark.gpu


def _check(frames, qp, kd=120, positions=None):
    got = kernels.h264_encode(torch.from_numpy(np.ascontiguousarray(frames)).cuda(), qp, kd, positions)
    want, recs = H.encode(frames, qp, kd, positions)
    assert len(got) == len(want)
    h, w = frames.shape[1:3]
    for i, (g, o) in enumerate(zip(got, want)):
        assert g == o, (i, frames.shape, qp, len(g), len(o))
        assert len(g) <= kernels.h264_encode_bound(w, h)
    return got, recs


def test_the_sweep_equals_the_oracle():
    for name, frames, qp in H.sweep():
        got = kernels.h264_encode(torch.from_numpy(frames).cuda(), qp, 2)
        assert got == H.encode(frames, qp, 2)[0], name


@pytest.mark.parametrize("h,w,kind", [(1080, 1920, "noise"), (1080, 1920, "smooth"), (2160, 3840, "noise"),
                                      (2160, 3840, "smooth")])
def test_large_frames_equal_the_oracle(h, w, kind):
    if kind == "noise":
        f = np.random.default_rng(h).integers(0, 256, (1, h, w, 3), dtype=np.uint8)
    else:
        yy, xx = np.mgrid[0:h, 0:w]
        f = np.stack([(xx // 8) % 256, (yy // 9) % 256, ((xx + 2 * yy) // 17) % 256], -1).astype(np.uint8)[None]
    for qp in (23, 35) if kind == "smooth" else (23,):
        _check(f, qp)


@pytest.mark.parametrize("n", [65, 130])
def test_batches_over_64_frames_equal_the_oracle(n):
    rng = np.random.default_rng(n)
    frames = rng.integers(0, 256, (n, 32, 48, 3), dtype=np.uint8)
    frames[::3] //= 16  # some quiet pictures among the noisy ones
    _check(frames, 27, kd=7)
    _check(frames[:n - 1], 30, kd=5, positions=list(range(9, 9 + n - 1)))


def test_unaligned_frames_equal_the_oracle():
    h, w = 34, 50
    frames = np.stack([H.content("gradient", h, w, i) for i in range(3)])
    buf = torch.zeros(3 * h * w * 3 + 64, dtype=torch.uint8, device="cuda")
    views = []
    for i, off in enumerate((1, 3 + h * w * 3, 7 + 2 * h * w * 3)):
        views.append(buf[off:off + h * w * 3].view(h, w, 3))
        views[-1].copy_(torch.from_numpy(frames[i]))
    assert kernels.h264_encode(views, 20, 2) == H.encode(frames, 20, 2)[0]


def _encode_raw(frames, qp, kd, fill):
    """scn_h264_encode_u8 into an output pre-filled with `fill` and followed by guard bytes (helpers.guarded_output)
    -> the access units."""
    frames = np.ascontiguousarray(frames)
    n, h, w = frames.shape[:3]
    dev = torch.from_numpy(frames).cuda()
    pp, _keep = cabi.ptr_array([dev.data_ptr() + i * h * w * 3 for i in range(n)])
    L = cabi.lib()
    return guarded_output.encode_raw("scn_h264_encode_u8", n, fill, lambda cb, sizes, stream:
                                     L.scn_h264_encode_u8(pp, n, w, h, qp, None, kd, cb, None, sizes, stream))


@pytest.mark.parametrize("fill", [0x00, 0xFF])
def test_prefilled_outputs_and_guards(fill):
    """the emulation-prevention seam frames, whose payloads carry escapes at lane and chunk edges; and 70 frames at
    keyframe_distance 3, so that IDR and non-IDR prefixes alternate within each launch and across the 64-frame
    split"""
    seams = epb_seam_frames()
    assert _encode_raw(seams, 0, 120, fill) == H.encode(seams, 0)[0]
    frames = np.random.default_rng(70).integers(0, 256, (70, 32, 48, 3), dtype=np.uint8)
    frames[::4] //= 16
    assert _encode_raw(frames, 27, 3, fill) == H.encode(frames, 27, 3)[0]


def test_the_decoder_reads_the_kernels_stream_back_to_the_reconstruction():
    n, h, w, kd = 12, 96, 160, 5
    frames = np.stack([H.content("noise" if i % 2 else "stripes", h, w, i) for i in range(n)])
    got, recs = _check(frames, 26, kd)
    eng = E.Engine(gpus=[0], instances_per_gpu=1)
    sid = eng.add_h264(b"".join(got))
    assert eng.stream_info(sid)["keyframes"] == (n + kd - 1) // kd and eng.stream_rows(sid) == n
    rows = [0, 1, 4, 5, 6, 11]
    dec = eng.decode_to_device(sid, rows).cpu().numpy()
    for k, r in enumerate(rows):
        y, c = H.to_nv12(recs[r])
        assert (dec[k] == oracle.nv12_to_rgb(y, c)).all(), r
    eng.close()


@pytest.mark.parametrize("w,h,qp,kd,rc", [(31, 16, 23, 1, -2), (16, 30 + 1, 23, 1, -2), (4098, 16, 23, 1, -2),
                                          (4096, 2320, 23, 1, -2), (16, 16, 52, 1, -1), (16, 16, 23, 0, -1)])
def test_refusals(w, h, qp, kd, rc):
    L = cabi.lib()
    sizes = (ctypes.c_size_t * 1)()
    pp, keep = cabi.ptr_array([0])
    cb = cabi.ALLOC_FN(lambda _c, _n: 0)
    assert L.scn_h264_encode_u8(pp, 1, w, h, qp, None, kd, cb, None, sizes, None) == rc
    with pytest.raises(cabi.ScnError, match="odd|beyond|QP|keyframe_distance"):
        kernels.h264_encode(torch.zeros((1, h, w, 3), dtype=torch.uint8, device="cuda"), qp, kd)
