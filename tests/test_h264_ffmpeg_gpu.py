"""scn_h264_encode_u8's own streams straight into FFmpeg (oracle/lavc.py, all three planes), and byte for byte
against oracle/h264_enc.py: the sweep, the geometries at the limits the kernel enforces (level 5.1's 36,864
macroblocks, 4096-sample sides, a one-macroblock wavefront, the level 4.1 / 5.1 switch at 8,192 macroblocks) in
QP 0 noise, the largest payloads, and in smooth content at QP 23; batches over 64 frames continuing an item; and
emulation-prevention bytes at the seams of the kernel's 16-byte lanes and 4096-byte chunks."""
import re

import numpy as np
import pytest
import torch

from helpers.h264_cases import epb_seam_frames
from oracle import h264_enc as H
from oracle import lavc
from scanner_b200 import kernels

pytestmark = pytest.mark.gpu

LANE, CHUNK = 16, 4096   # bytes per thread and per CTA of the escape passes (kLane, kChunk in bitstream.cuh)


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
            assert not len(bad), (what, i, name, f"{len(bad)} samples differ, first at {tuple(bad[0])}")


def _check(frames, qp, kd=120, positions=None, decode=True):
    """the kernel's access units equal the oracle's, and FFmpeg decodes them to the oracle's reconstruction (when
    they start with an IDR picture: `decode`)"""
    got = kernels.h264_encode(torch.from_numpy(np.ascontiguousarray(frames)).cuda(), qp, kd, positions)
    want, recs = H.encode(frames, qp, kd, positions)
    assert len(got) == len(want)
    for i, (g, o) in enumerate(zip(got, want)):
        assert g == o, (i, frames.shape, qp, len(g), len(o))
    if decode:
        _assert_planes_equal(_decode(got, frames.shape[2], frames.shape[1]), recs, (frames.shape, qp))
    return got


def test_ffmpeg_decodes_the_kernels_sweep_to_the_oracles_reconstruction():
    for name, frames, qp in H.sweep():
        _check(frames, qp, 2)


# ---- the limits --------------------------------------------------------------------------------------------------
LIMITS = [(4096, 2304), (4094, 2302), (4096, 16), (16, 4096), (4096, 2), (2, 4096), (2048, 1024), (2048, 1040)]


@pytest.mark.parametrize("kind,qp", [("noise", 0), ("smooth", 23)])
@pytest.mark.parametrize("w,h", LIMITS)
def test_limit_geometries(w, h, kind, qp):
    if kind == "noise":
        frame = np.random.default_rng(w * h).integers(0, 256, (h, w, 3), dtype=np.uint8)
    else:
        frame = H.natural(h, w, w + h)
    (au,) = _check(frame[None], qp)
    mbs = ((w + 15) // 16) * ((h + 15) // 16)
    # Table A-1: MaxFS 8,192 macroblocks at level 4.1 and 36,864 at level 5.1
    assert au[:8] == b"\x00\x00\x00\x01\x67\x42\xc0" + bytes([41 if mbs <= 8192 else 51]), au[:8]
    bound = kernels.h264_encode_bound(w, h)
    assert len(au) <= bound
    print(f"\n{w}x{h} {kind} QP {qp}: {len(au)} bytes, {len(au) / bound:.3f} of scn_h264_encode_bound ({bound})")


# ---- batches over 64 frames that continue an item -----------------------------------------------------------------
@pytest.mark.parametrize("n", [65, 130])
def test_batches_over_64_frames_continue_an_item_as_one_stream(n):
    rng = np.random.default_rng(n)
    frames = rng.integers(0, 256, (n + 3, 32, 48, 3), dtype=np.uint8)
    frames[::3] //= 16
    head = _check(frames[:3], 24, kd=16)
    tail = _check(frames[3:], 24, kd=16, positions=list(range(3, n + 3)), decode=False)
    _assert_planes_equal(_decode(head + tail, 48, 32), H.encode(frames, 24, 16)[1], n)


# ---- emulation prevention at the kernel's seams ------------------------------------------------------------------
def _rbsp(au):
    nal = au[au.rfind(b"\x00\x00\x00\x01") + 5:]
    return re.sub(b"\x00\x00\x03", b"\x00\x00", nal)


def _epb_pairs(rbsp):
    """offsets of the zero pairs that get an emulation-prevention byte (7.4.1): a payload byte <= 3 after an even,
    nonzero run of payload zeros"""
    out, z = [], 0
    for i, b in enumerate(rbsp):
        if b <= 3 and z >= 2 and z % 2 == 0:
            out.append(i - 2)
        z = 0 if b else z + 1
    return out


def test_emulation_prevention_at_lane_and_chunk_seams():
    frames = epb_seam_frames()
    pairs = [p for au in H.encode(frames, 0)[0] for p in _epb_pairs(_rbsp(au))]
    assert any(p % LANE == LANE - 1 and p % CHUNK != CHUNK - 1 for p in pairs), "no pair across a lane seam"
    assert any(p % CHUNK == CHUNK - 1 for p in pairs), "no pair across a chunk seam"
    assert any(p % CHUNK == 0 and p > 0 for p in pairs), "no pair starting a chunk"
    _check(frames, 0)
