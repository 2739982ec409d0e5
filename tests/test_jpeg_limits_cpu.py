"""The JPEG oracle at its limits, host side: every quality 1-100 against live cv2 (files and quantisation tables);
a corpus of frames that codes every Huffman symbol of both tables (tests/golden/jpeg_symbols.npz, made by
oracle/make_golden_jpeg_symbols.py); the arithmetic jpeg.cu's quantiser relies on, exhaustively; and
scn_jpeg_encode_bound against the densest files.  tests/test_jpeg_limits_gpu.py holds the kernels to the same cases."""
import os

import numpy as np
import pytest

from oracle import jpeg as J
from scanner_b200 import cabi

CORPUS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_symbols.npz")


def corpus_frames():
    with np.load(CORPUS) as z:
        return J.symbol_corpus_frames({k: z[k] for k in z.files})


def _segments(data, marker):
    """payloads of every `marker` segment before the scan"""
    out, at = [], 2
    while data[at + 1] != 0xDA:
        n = int.from_bytes(data[at + 2:at + 4], "big")
        if data[at + 1] == marker:
            out.append(data[at + 4:at + 2 + n])
        at += 2 + n
    return out


def quality_frames(q):
    return [J.content("noise", 13, 21, 3, q), J.content("gradient", 19, 11, 3, q),
            J.content("noise", 11, 17, 1, q), J.content("gradient", 9, 23, 1, q)]


def test_every_quality_equals_live_cv2_in_file_and_tables():
    pytest.importorskip("cv2")
    for q in range(1, 101):
        for f in quality_frames(q):
            want = J.cv2_encode(f, q)
            assert J.encode(f, q) == want, (q, f.shape)
            h, w, c = f.shape
            dqt = _segments(J.header(w, h, c, q), 0xDB)
            assert dqt == _segments(want, 0xDB) and len(dqt) == (2 if c == 3 else 1), (q, c)
            for t, base in enumerate((J.LUMA_Q, J.CHROMA_Q)[:len(dqt)]):
                assert list(dqt[t][1:]) == J.quant_table(base, q)[J.ZIGZAG].tolist(), (q, t)


def test_corpus_codes_every_symbol_of_both_tables():
    seen = set()
    for _, frame, q in corpus_frames():
        seen |= set(J.symbols(frame, q))
    for t in (0, 1):
        assert {s for c, tt, s in seen if (c, tt) == (0, t)} == set(J.DC_SYMBOLS), t
        assert {s for c, tt, s in seen if (c, tt) == (1, t)} == set(J.AC_SYMBOLS), t
    assert len(J.AC_SYMBOLS) == 162 and {0x00, 0xF0, 0xFA, 0xF1, 0x0A} <= set(J.AC_SYMBOLS)


def test_corpus_frames_equal_live_cv2():
    pytest.importorskip("cv2")
    frames = corpus_frames()
    assert {name.split("_")[0] for name, _, _ in frames} == {"luma", "chroma"}
    for name, frame, q in frames:
        assert J.encode(frame, q) == J.cv2_encode(frame, q), name


def test_corpus_chroma_frames_carry_their_blocks_as_cb():
    """The layout the corpus relies on: pixels (255 - X, 255 - X, X) have Cb = X exactly, and a 2 x 2 doubled
    plane downsamples to itself."""
    x = np.arange(256, dtype=np.uint8)
    _, cb, _ = J.rgb_ycc(np.stack([255 - x, 255 - x, x], -1))
    assert (cb == x).all()
    plane = np.random.default_rng(0).integers(0, 256, (8, 8)).repeat(2, 0).repeat(2, 1)
    assert (J.downsample(plane, 8, 8) == plane[::2, ::2]).all()


def test_scan_and_symbols_restate_the_file():
    for name, frame, q in corpus_frames() + [("noise", J.content("noise", 40, 56, 3, 1), 100)]:
        data = J.encode(frame, q)
        h, w = frame.shape[:2]
        hdr = J.header(w, h, frame.shape[2] if frame.ndim == 3 else 1, q)
        s = J.scan(frame, q)
        assert data == hdr + J.stuff(s) + b"\xFF\xD9", name
        blocks = -(-h // 16) * -(-w // 16) * 6 if frame.ndim == 3 else -(-h // 8) * -(-w // 8)
        syms = J.symbols(frame, q)
        assert sum(n for (c, _, _), n in syms.items() if c == 0) == blocks, name


def test_quantiser_multiply_shift_is_exact():
    """fdct_quant in jpeg.cu divides |coef| + 4q by 8q as umulhi(x, ceil(2^32 / 8q)), exact for every x < 2^17 and
    every q in 1..255; x stays below 2^17 because no islow output comes near 2^17 - 4 * 255."""
    x = np.arange(1 << 17, dtype=np.uint64)
    for q in range(1, 256):
        d = 8 * q
        m = np.uint64(((1 << 32) + d - 1) // d)
        assert (((x * m) >> np.uint64(32)) == x // np.uint64(d)).all(), q
    # the extreme of each coefficient: samples 127 where its basis function is positive, -128 where negative
    u = np.arange(8)
    cos = np.cos((2 * u[None] + 1) * u[:, None] * np.pi / 16)  # (frequency, position), never 0
    sign = np.einsum("ux,vy->uvxy", cos, cos).reshape(64, 8, 8) > 0
    pats = np.concatenate([np.where(sign, 255, 0), np.where(sign, 0, 255)]).astype(np.uint8)
    out = np.abs(J.fdct(pats)).reshape(2, 64, 64)
    largest = int(out.max())
    assert largest == 8192 and out[:, 0, 0].max() == 8192  # the DC of an all-0 block
    # no block reaches more on any coefficient: random blocks of 0 / 255 stay at or below these extremes
    rnd = np.random.default_rng(1).integers(0, 2, (20000, 8, 8)).astype(np.uint8) * 255
    per_coef = np.abs(J.fdct(rnd)).reshape(-1, 64).max(0)
    assert (per_coef <= out.max(0).diagonal()).all()
    assert largest + 4 * 255 < 1 << 17


def test_bound_covers_the_densest_files():
    L = cabi.lib()
    frames = [(name, f, q) for name, f, q in corpus_frames()]
    for c in (3, 1):
        for kind in ("noise", "checker", "saturated"):
            frames.append((f"{kind}{c}", J.content(kind, 64, 80, c, 7), 100))
    worst = 0.0
    for name, frame, q in frames:
        h, w = frame.shape[:2]
        c = frame.shape[2] if frame.ndim == 3 else 1
        data = J.encode(frame, q)
        assert len(data) <= L.scn_jpeg_encode_bound(w, h, c), name
        blocks = -(-h // 16) * -(-w // 16) * 6 if c == 3 else -(-h // 8) * -(-w // 8)
        worst = max(worst, 8 * len(J.scan(frame, q)) / blocks)
    # single blocks: the bits one block can take, DC difference from 0 included
    rng = np.random.default_rng(5)
    singles = [rng.integers(0, 256, (8, 8)).astype(np.uint8) for _ in range(200)]
    singles += [J.content("checker", 8, 8, 1, 0)[..., 0], np.where(np.indices((8, 8)).sum(0) % 2, 0, 255)]
    for b in singles:
        worst = max(worst, 8 * len(J.scan(np.ascontiguousarray(b, np.uint8), 100)))
    print(f"largest bits per block seen: {worst:.0f} of the bound's 1660")
    assert worst < 1660
