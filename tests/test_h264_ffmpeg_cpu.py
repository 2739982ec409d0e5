"""oracle/h264_enc.py held to FFmpeg in all three planes (oracle/lavc.py decodes each access unit to Y, Cb and Cr)
and its colour stage held to float64 BT.601.  tests/test_h264_encode_cpu.py compares only the luma plane with
FFmpeg; a mistake shared by the oracle and the kernel that touches only chroma samples (a chroma-QP entry, a
chroma-DC prediction rule) or the colour conversion (a coefficient row, a rounding term) shows up only here.
The GPU kernel equals the oracle byte for byte (tests/test_h264_encode_gpu.py, tests/test_h264_ffmpeg_gpu.py)."""
import re

import numpy as np
import pytest

from oracle import h264_enc as H
from oracle import lavc


def _decode(aus, w, h):
    try:
        return lavc.decode(aus, (w, h))
    except lavc.Unavailable as e:
        pytest.skip(f"FFmpeg is not available: {e}")


def _assert_planes_equal(got, recs, what):
    assert len(got) == len(recs), what
    for i, (g, r) in enumerate(zip(got, recs)):
        for p, name in enumerate(("Y", "Cb", "Cr")):
            assert g[p].shape == r[p].shape, (what, i, name, g[p].shape, r[p].shape)
            bad = np.argwhere(g[p] != r[p])
            assert not len(bad), (what, i, name, f"{len(bad)} samples differ, first at {tuple(bad[0])}",
                                  int(g[p][tuple(bad[0])]), int(r[p][tuple(bad[0])]))


def test_the_decoder_wrapper_refuses_what_it_cannot_vouch_for():
    frames = np.stack([H.content("gradient", 32, 48, i) for i in range(2)])
    aus, recs = H.encode(frames, 20, keyframe_distance=2)
    _assert_planes_equal(_decode(aus, 48, 32), recs, "plain")
    with pytest.raises(RuntimeError, match="not 46x32"):
        lavc.decode(aus, (46, 32))
    with pytest.raises(RuntimeError, match="access unit 0"):   # a non-IDR picture without its parameter sets
        lavc.decode(aus[1:], (48, 32))


# ---- (a) the sweep, every plane -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sweep():
    """every sweep item encoded once as tests/test_h264_encode_cpu.py does: (name, w, h, access units, recs)"""
    items = []
    for name, frames, qp in H.sweep():
        aus, recs = H.encode(frames, qp, keyframe_distance=2)
        items.append((name, frames.shape[2], frames.shape[1], aus, recs))
    return items


def test_ffmpeg_decodes_every_plane_of_the_sweep_to_the_oracles_reconstruction(sweep):
    for name, w, h, aus, recs in sweep:
        _assert_planes_equal(_decode(aus, w, h), recs, name)


def test_the_sweep_codes_chroma_residuals_at_every_qp():
    """the chroma comparison above tests the chroma-QP table at a QP only if chroma levels are coded there: every
    sweep QP codes macroblocks with chroma DC only (cbp 1) and with chroma AC (cbp 2)"""
    for qp in H.SWEEP_QPS:
        cbpc = set()
        for name, frames, q in H.sweep():
            if q != qp or not name.startswith(("noise", "checkerboard")):
                continue
            _, m = H._reconstruct(H.rgb_to_planes(frames[0]), qp, H.new_stats())
            cbpc |= set(np.unique(m["cbpc"]).tolist())
        assert {1, 2} <= cbpc, (qp, cbpc)


# ---- (b) long items: frame_num wrapping, idr_pic_id, positions ---------------------------------------------------
def _slice_fields(au):
    """(nal_unit_type, frame_num, idr_pic_id or None) of the slice in one access unit, parsed from the bytes"""
    nal = au[au.rfind(b"\x00\x00\x00\x01") + 4:]
    kind = nal[0] & 31
    bits = "".join(format(b, "08b") for b in re.sub(b"\x00\x00\x03", b"\x00\x00", nal[1:64]))
    at = 0

    def ue():
        nonlocal at
        z = bits.index("1", at) - at
        v = int(bits[at + z:at + 2 * z + 1], 2) - 1
        at += 2 * z + 1
        return v
    ue(), ue(), ue()                         # first_mb_in_slice, slice_type, pic_parameter_set_id
    frame_num = int(bits[at:at + 4], 2)      # log2_max_frame_num = 4
    at += 4
    return kind, frame_num, ue() if kind == 5 else None


def _frames(n, h=32, w=48):
    kinds = ("noise", "gradient", "stripes", "saturated")
    return np.stack([H.content(kinds[i % 4], h, w, 77 + i) for i in range(n)])


@pytest.mark.parametrize("kd", [1, 2, 16, 17, 120])
def test_long_items_decode_to_every_picture(kd):
    n = 40
    frames = _frames(n)
    aus, recs = H.encode(frames, 24, keyframe_distance=kd)
    _assert_planes_equal(_decode(aus, 48, 32), recs, kd)
    # 7.4.3: frame_num is 0 at an IDR and counts every (reference) picture after it modulo MaxFrameNum = 16;
    # two IDRs in a row differ in idr_pic_id
    prev = None
    for i, au in enumerate(aus):
        kind, frame_num, idr_id = _slice_fields(au)
        assert kind == (5 if i % kd == 0 else 1), (kd, i)
        assert frame_num == (0 if kind == 5 else (prev[1] + 1) % 16), (kd, i, frame_num, prev)
        if kind == 5 and prev is not None and prev[0] == 5:
            assert idr_id != prev[2], (kd, i)
        prev = (kind, frame_num, idr_id)


@pytest.mark.parametrize("k,kd", [(16, 16), (21, 16), (1, 120), (35, 17)])
def test_an_item_continued_with_positions_is_one_stream(k, kd):
    n = 36
    frames = _frames(n)
    whole, recs = H.encode(frames, 30, keyframe_distance=kd)
    head, _ = H.encode(frames[:k], 30, keyframe_distance=kd)
    tail, _ = H.encode(frames[k:], 30, keyframe_distance=kd, positions=list(range(k, n)))
    assert head + tail == whole
    _assert_planes_equal(_decode(head + tail, 48, 32), recs, (k, kd))


# ---- (c) the colour stage against float64 BT.601 ----------------------------------------------------------------
# Measured on these inputs (max / mean): Y over all 2^24 triples 0.759 / 0.262; Cb and Cr on the random blocks
# 0.827 / 0.260 and 0.762 / 0.256, on the extremes 0.652 / 0.274 and 0.660 / 0.269, one off them 0.956 / 0.275 and
# 0.852 / 0.264.  A dropped rounding term moves every sample by about 0.5 and breaks both bounds; swapped
# coefficient rows break them by far.
COLOUR_MAX, COLOUR_MEAN = 1.0, 0.3


def test_luma_of_every_rgb_triple_is_within_one_of_bt601():
    v = np.arange(256, dtype=np.uint8)
    gb = np.stack(np.meshgrid(v, v, indexing="ij"), -1).reshape(256, 256, 2)
    worst, total = 0.0, 0.0
    for r in range(256):
        rgb = np.concatenate([np.full((256, 256, 1), r, np.uint8), gb], -1)
        y = H.rgb_to_planes(rgb)[0][:256, :256]
        e = np.abs(y - H.bt601_float(rgb)[0])
        worst, total = max(worst, float(e.max())), total + float(e.sum())
    assert worst < COLOUR_MAX and total / 2 ** 24 < COLOUR_MEAN, (worst, total / 2 ** 24)


def _chroma_blocks():
    rng = np.random.default_rng(601)
    random = rng.integers(0, 256, (1 << 18, 2, 2, 3), dtype=np.uint8)
    # every 2x2 block whose 12 samples are each 0 or 255: the primaries, black, white and every mix of them
    extremes = (((np.arange(4096)[:, None] >> np.arange(12)) & 1) * 255).astype(np.uint8).reshape(4096, 2, 2, 3)
    # one sample off the extremes, where a floor and a round part
    near = np.clip(extremes.astype(np.int64) + rng.choice([-1, 1], extremes.shape), 0, 255).astype(np.uint8)
    return {"random": random, "extremes": extremes, "near extremes": near}


@pytest.mark.parametrize("which", ["random", "extremes", "near extremes"])
def test_chroma_of_2x2_blocks_is_within_one_of_bt601(which):
    blocks = _chroma_blocks()[which]
    n = len(blocks)
    frame = blocks.transpose(1, 0, 2, 3).reshape(2, 2 * n, 3)   # the blocks side by side in a 2-row frame
    _, cb, cr = H.rgb_to_planes(frame)
    _, fcb, fcr = H.bt601_float(blocks.astype(np.float64).mean((1, 2)))
    for name, got, want in (("Cb", cb[0, :n], fcb), ("Cr", cr[0, :n], fcr)):
        e = np.abs(got - want)
        assert e.max() < COLOUR_MAX and e.mean() < COLOUR_MEAN, (which, name, e.max(), e.mean(), blocks[e.argmax()])


# ---- (d) the round trip: source -> oracle -> FFmpeg against float BT.601 -----------------------------------------
# Bounds per plane, measured on H.natural(144, 176, 3) through FFmpeg 8 (max / mean over Y, Cb, Cr):
#   QP 0   1.62 / 0.268   1.59 / 0.268   1.53 / 0.265
#   QP 6   1.84 / 0.427   2.07 / 0.429   1.99 / 0.421
#   QP 12  3.56 / 0.725   3.31 / 0.695   3.34 / 0.710
ROUND_TRIP = {0: (1.9, 0.30), 6: (2.4, 0.47), 12: (3.9, 0.78)}


@pytest.mark.parametrize("qp", sorted(ROUND_TRIP))
def test_ffmpeg_decodes_smooth_content_close_to_bt601(qp):
    frame = H.natural(144, 176, 3)
    aus, recs = H.encode(frame[None], qp)
    (got,) = _decode(aus, 176, 144)
    _assert_planes_equal([got], recs, qp)
    max_bound, mean_bound = ROUND_TRIP[qp]
    for name, g, want in zip(("Y", "Cb", "Cr"), got, H.bt601_planes(frame)):
        e = np.abs(g - want)
        assert e.max() < max_bound and e.mean() < mean_bound, (qp, name, e.max(), e.mean())
