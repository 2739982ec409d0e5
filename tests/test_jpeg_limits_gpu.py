"""The JPEG kernels at their limits on the GPU, byte for byte against the oracle (oracle/jpeg.py) and live cv2:
  * every quality 1-100, and the corpus that codes every Huffman symbol of both tables (tests/golden/jpeg_symbols.npz);
  * outputs pre-filled with 0x00 and with 0xFF and followed by guard bytes, so that a byte the encoder never writes
    and a byte written past the end both fail;
  * scans whose length or 0xFF bytes fall on the edges of the 4 KiB chunks and 16-byte lanes of the 0xFF passes,
    and a scan whose last byte is 0xFF (its stuffed 0x00 sits just before the EOI);
  * sides of 65500, MCU counts around multiples of the MCU kernels' 128 threads and of jpeg_scan_kernel's 1024,
    a frame of more than 2^20 MCUs;
  * one-chunk frames beside frames of over a hundred chunks, in one launch and across the 64-frame split, and calls of
    very different sizes back to back on one stream;
  * the ImageEncoder op at the 65500-wide limit and one pixel past it."""
import os

import numpy as np
import pytest
import torch

import scanner_b200 as sp
from helpers import guarded_output
from oracle import jpeg as J
from scanner_b200 import cabi, kernels

pytestmark = pytest.mark.gpu

CORPUS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_symbols.npz")


def encode_raw(frames, quality, fill):
    """scn_jpeg_encode_u8 of equal-shape frames into an output pre-filled with `fill` and followed by guard bytes
    (helpers.guarded_output) -> the files."""
    frames = [np.ascontiguousarray(f) for f in frames]
    h, w = frames[0].shape[:2]
    c = 1 if frames[0].ndim == 2 else frames[0].shape[2]
    dev = [torch.from_numpy(f).cuda() for f in frames]
    pp, _keep = cabi.ptr_array([t.data_ptr() for t in dev])
    L = cabi.lib()
    return guarded_output.encode_raw("scn_jpeg_encode_u8", len(frames), fill, lambda cb, sizes, stream:
                                     L.scn_jpeg_encode_u8(pp, len(frames), w, h, c, quality, cb, None, sizes, stream))


def check(frames, quality, got, cv2=True):
    assert len(got) == len(frames)
    for i, (f, g) in enumerate(zip(frames, got)):
        want = J.encode(f, quality)
        assert g == want, (i, f.shape, quality, len(g), len(want))
        if cv2:
            assert g == J.cv2_encode(f, quality), (i, f.shape, quality)


# ---- tables ------------------------------------------------------------------------------------------------------
def test_every_quality():
    for q in range(1, 101):
        fill = 0xFF if q & 1 else 0x00
        for c, (h, w) in ((3, (21, 35)), (1, (19, 27))):
            frames = [J.content(k, h, w, c, q)[..., 0] if c == 1 else J.content(k, h, w, c, q)
                      for k in ("noise", "gradient", "saturated")]
            check(frames, q, encode_raw(frames, q, fill))


def test_the_symbol_corpus():
    with np.load(CORPUS) as z:
        frames = J.symbol_corpus_frames({k: z[k] for k in z.files})
    assert {q for _, _, q in frames} == {100, 98}
    for name, frame, q in frames:
        for fill in (0x00, 0xFF):
            assert encode_raw([frame], q, fill)[0] == J.encode(frame, q) == J.cv2_encode(frame, q), (name, fill)


# ---- the caller's output -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("fill", [0x00, 0xFF])
@pytest.mark.parametrize("c", [3, 1])
def test_prefilled_outputs_and_guards(fill, c):
    frames = [J.content("noise", 80, 112, c, s) for s in range(5)]
    frames[2] = J.content("checker", 80, 112, c, 0)
    got = encode_raw(frames, 100, fill)
    check(frames, 100, got)
    assert sum(g.count(b"\xff\x00") for g in got) > 500  # dense stuffing


# ---- the 0xFF passes: chunk and lane edges -----------------------------------------------------------------------
CHUNK = 4096


def _search(width, seeds, want):
    """seeded 8 x width gray noise at quality 100 -> {name: (frame, scan)} for the first seed meeting each test of
    `want` ({name: predicate(scan)})."""
    found = {}
    for seed in range(seeds):
        f = J.content("noise", 8, width, 1, seed)[..., 0]
        s = J.scan(f, 100)
        for name, pred in want.items():
            if name not in found and pred(s):
                found[name] = (f, s)
        if len(found) == len(want):
            break
    assert set(found) == set(want), sorted(set(want) - set(found))
    return found


@pytest.fixture(scope="module")
def edge_frames():
    """gray frames whose scans (before stuffing) end at and around chunk and lane edges, or carry a 0xFF at them"""
    cases = {}
    for k, width in ((1, 325), (2, 650)):  # about 12.6 bytes of scan per column of 8 x 8 noise blocks
        cases.update(_search(width, 1500, {f"len {CHUNK * k + d}": (lambda s, n=CHUNK * k + d: len(s) == n)
                                           for d in (-1, 0, 1)}))
    cases.update(_search(88, 2000, {"last byte 0xFF": lambda s: s[-1] == 0xFF,
                                    "len 16k - 1": lambda s: len(s) % 16 == 15,
                                    "len 16k + 1": lambda s: len(s) % 16 == 1}))
    edges = range(CHUNK, 4 * CHUNK, CHUNK)
    cases.update(_search(1300, 1500, {
        "0xFF ends a chunk": lambda s: any(len(s) > e and s[e - 1] == 0xFF for e in edges),
        "0xFF starts a chunk": lambda s: any(len(s) > e and s[e] == 0xFF for e in edges),
        "0xFF ends a lane": lambda s: 0xFF in s[15::16],
        "0xFF starts a lane": lambda s: 0xFF in s[16::16]}))
    return cases


@pytest.mark.parametrize("fill", [0x00, 0xFF])
def test_chunk_and_lane_edges(edge_frames, fill):
    for name, (frame, s) in edge_frames.items():
        got = encode_raw([frame], 100, fill)[0]
        want = J.encode(frame, 100)
        assert got == want, (name, len(s))
        if name == "last byte 0xFF":
            assert got.endswith(b"\xff\x00\xff\xd9")
    # the frames of one geometry in one call too
    for w in sorted({f.shape[1] for f, _ in edge_frames.values()}):
        group = [f for f, _ in edge_frames.values() if f.shape[1] == w]
        check(group, 100, encode_raw(group, 100, fill), cv2=False)


# ---- geometry ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(16, 65500), (65500, 16), (1, 65500), (65500, 1)])
@pytest.mark.parametrize("c", [3, 1])
def test_65500_sides(h, w, c):
    f = J.content("noise", h, w, c, h + c)
    check([f], 100, encode_raw([f], 100, 0xFF if c == 3 else 0x00))


@pytest.mark.parametrize("mcus", [127, 128, 129, 255, 256, 257, 1023, 1024, 1025, 2047, 2048, 2049])
def test_mcu_counts_at_cta_and_scan_splits(mcus):
    """MCU counts around multiples of the MCU kernels' 128-thread CTA and of jpeg_scan_kernel's 1024 threads, where
    each thread's share of MCUs (ceil(mcus / 1024)) changes."""
    for c, m in ((1, 8), (3, 16)):
        f = J.content("noise", m, m * mcus, c, mcus)
        check([f], 90, encode_raw([f], 90, 0x00))
    # two-dimensional grids of the same counts
    rows = next(r for r in (33, 31, 25, 23, 17, 16, 9, 8, 7, 3, 1) if mcus % r == 0)
    f = J.content("noise", 8 * rows, 8 * (mcus // rows), 1, mcus)[..., 0]
    check([f], 75, encode_raw([f], 75, 0xFF), cv2=False)


def test_frame_of_more_than_2_20_mcus():
    """8200 x 8200 gray: 1,050,625 MCUs, each jpeg_scan_kernel thread summing 1027 of them (against cv2 only: the
    oracle would need several GB here)."""
    f = np.random.default_rng(20).integers(0, 256, (8200, 8200), dtype=np.uint8)
    got = kernels.jpeg_encode(torch.from_numpy(f[None, ..., None]).cuda(), 95)
    assert got[0] == J.cv2_encode(f, 95)


# ---- stream sizes ------------------------------------------------------------------------------------------------
def test_one_chunk_frames_beside_many_chunk_frames():
    """66 RGB frames of one geometry: 0 and 64 constant, the rest quality-100 noise; frames 64 and 65 make the
    second launch.  An MCU of 128s codes in 32 bits, so 512 x 512 is the largest colour frame whose constant scan
    fits one chunk (exactly 4096 bytes); its noise scans take over 120 chunks."""
    h, w = 512, 512
    distinct = [np.full((h, w, 3), 128, np.uint8)] + [J.content("noise", h, w, 3, s) for s in range(4)]
    which = [0 if i in (0, 64) else 1 + i % 4 for i in range(66)]
    wants = [J.encode(f, 100) for f in distinct]
    assert len(J.scan(distinct[0], 100)) == CHUNK and min(len(J.scan(f, 100)) for f in distinct[1:]) > 120 * CHUNK
    got = encode_raw([distinct[j] for j in which], 100, 0xFF)
    for i, j in enumerate(which):
        assert got[i] == wants[j], i
    assert wants[1] == J.cv2_encode(distinct[1], 100)


def test_back_to_back_calls_of_very_different_sizes():
    """The scratch pool hands the second call the first call's dirty memory."""
    big = J.content("noise", 2160, 3840, 3, 4)
    tiny = [J.content("noise", 9, 13, 3, s) for s in range(3)]
    tiny_want = [J.encode(f, 100) for f in tiny]
    for _ in range(2):
        got = kernels.jpeg_encode(torch.from_numpy(big[None]).cuda(), 100)
        assert got[0] == J.cv2_encode(big, 100)
        assert kernels.jpeg_encode([torch.from_numpy(f).cuda() for f in tiny], 100) == tiny_want
        assert encode_raw(tiny, 100, 0x00) == tiny_want


# ---- op level ----------------------------------------------------------------------------------------------------
@pytest.fixture()
def sc(tmp_path):
    c = sp.Client(db_path=str(tmp_path / "scanner_db"))
    yield c
    c.stop()


def _encode_op(sc, frames, name):
    inp = sc.io.Input([sp.NamedVideoStream(sc, name, frames=frames)])
    enc = sc.ops.ImageEncoder(frame=inp, device=sp.DeviceType.GPU, format="jpg", quality=100)
    out = sp.NamedStream(sc, name + "_jpg")
    sc.run(sc.io.Output(enc, [out]), sp.PerfParams.manual(8, 16))
    return list(out.load())


def test_op_at_the_65500_limit_and_past_it(sc):
    wide = np.stack([J.content("noise", 8, 65500, 3, s) for s in range(2)])
    got = _encode_op(sc, wide, "wide")
    assert got == [J.cv2_encode(f, 100) for f in wide] == [J.encode(f, 100) for f in wide]
    with pytest.raises(sp.ScannerException, match="JPEG frames are at most 65500 x 65500, got 65501 x 8"):
        _encode_op(sc, np.zeros((2, 8, 65501, 3), np.uint8), "too_wide")
    good = np.stack([J.content("gradient", 24, 40, 3, 1)] * 3)
    assert _encode_op(sc, good, "good") == [J.cv2_encode(f, 100) for f in good]
