"""The oracle (oracle/scn_oracle.c) against the committed golden vectors.

hist_cv2 / resize_cv2 come from OpenCV itself (cv2.calcHist / cv2.resize called the way
tests/test_ops.cpp:38-43,156 of the reference calls them); blur_np / nv12_np come from the
independent numpy restatement in oracle/make_golden.py.  CPU only.
"""
import os

import numpy as np

import oracle
from oracle import synth


def _cases(npz):
    keys = sorted(k[:-5] for k in npz.files if k.endswith("_meta"))
    return keys


def test_hist_matches_cv2_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "hist_cv2.npz"))
    for k in _cases(g):
        meta = g[k + "_meta"]
        if meta[3] == 2:
            img = np.full((meta[1], meta[2], 3), meta[0], np.uint8)
        else:
            img = synth.frame(int(meta[0]), int(meta[1]), int(meta[2]), int(meta[3]))
        got = oracle.hist16(img)
        assert got.dtype == np.int32 and got.shape == (3, 16)
        assert (got == g[k + "_hist"]).all(), k
        assert got.sum() == 3 * meta[1] * meta[2]


def test_resize_matches_cv2_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "resize_cv2.npz"))
    for k in _cases(g):
        seed, h, w, dh, dw, kind = [int(x) for x in g[k + "_meta"]]
        img = synth.frame(seed, h, w, kind)
        got = oracle.resize(img, dw, dh)
        assert (got == g[k + "_out"]).all(), (k, h, w, dh, dw)


def test_blur_matches_numpy_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "blur_np.npz"))
    for k in _cases(g):
        seed, h, w, ks = [int(x) for x in g[k + "_meta"]]
        img = synth.rand_frame(seed, h, w)
        assert (oracle.blur(img, ks) == g[k + "_out"]).all(), (k, h, w, ks)


def test_nv12_matches_numpy_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "nv12_np.npz"))
    for k in _cases(g):
        seed, h, w, pitch = [int(x) for x in g[k + "_meta"]]
        luma, chroma = synth.nv12_surface(seed, h, w, pitch)
        assert (oracle.nv12_to_rgb(luma, chroma, w) == g[k + "_out"]).all(), (k, h, w, pitch)


def test_nv12_exhaustive_yuv_triples():
    """All 2^24 (Y,Cb,Cr) triples on even rows equal the float formula evaluated in numpy."""
    # even rows only use the co-sited chroma sample: build a surface where each 2x2 block has
    # one (Cb,Cr) and two distinct Y on the even row.
    cb, cr = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8))
    for y0 in (0, 1, 16, 127, 128, 235, 254, 255):
        w = 2 * 256
        luma = np.full((2 * 256, w), y0, np.uint8)
        chroma = np.zeros((256, w), np.uint8)
        chroma[:, 0::2] = cb
        chroma[:, 1::2] = cr
        rgb = oracle.nv12_to_rgb(luma, chroma)[0::2, 0::2]
        lf = np.float32(y0 * 4) * np.float32(1.1644)
        fcb = (cb.astype(np.int32) * 4 - 512).astype(np.float64)
        fcr = (cr.astype(np.int32) * 4 - 512).astype(np.float64)
        r = (fcr * np.float64(np.float32(1.596)) + np.float64(lf)).astype(np.float32)
        r = (np.clip(r, 0, 1023).astype(np.uint32) >> 2).astype(np.uint8)
        assert (rgb[..., 0] == r).all()


def test_resize_equals_live_cv2_over_a_sweep():
    """oracle.resize against cv2.resize itself on the ~2000 seeded geometries test_cabi_host.py holds the product's
    plan to, random and constant 0 / 255 frames."""
    import pytest
    cv2 = pytest.importorskip("cv2")
    big = synth.rand_frame(23, 1920, 1920)
    for k, (sw, sh, dw, dh) in enumerate(synth.resize_geometries(5, 2000)):
        img = big[:sh, :sw] if k % 2 else np.full((sh, sw, 3), 255 * (k % 4 == 0), np.uint8)
        want = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR)
        assert (oracle.resize(img, dw, dh) == want).all(), (sw, sh, dw, dh)


def test_resize_target_rules():
    # tests/test_ops.cpp:126-147
    assert oracle.resize_target(1920, 1080, 224, 224) == (224, 224)
    assert oracle.resize_target(1920, 1080, 0, 540, preserve_aspect=True) == (960, 540)
    assert oracle.resize_target(1920, 1080, 640, 0, preserve_aspect=True) == (640, 360)
    assert oracle.resize_target(640, 480, 1000, 1000, min=True) == (640, 480)
    assert oracle.resize_target(640, 480, 320, 1000, min=True) == (320, 1000)


def test_index_column():
    b = oracle.index_column(5, 4)
    assert (np.frombuffer(b.tobytes(), "<i8") == np.arange(5, 9)).all()


def test_blur_interior_only_and_border_zero():
    img = synth.rand_frame(1, 12, 14)
    out = oracle.blur(img, 3)
    ys, xs = oracle.blur_interior(12, 14, 3)
    mask = np.ones((12, 14), bool)
    mask[ys, xs] = False
    assert (out[mask] == 0).all()
    # k=1 is the identity on the whole frame (fl=fr=0)
    assert (oracle.blur(img, 1) == img).all()


def test_flow_matches_cv2_golden(golden_dir):
    """Farneback is float: the restatement sums in a different order than OpenCV's SIMD code.
    Stated tolerance vs cv2.FarnebackOpticalFlow(3,0.5,False,15,3,5,1.2,0): max |d| <= 1e-4 px
    (measured 2e-6 on smooth motion, 8e-6 on noise)."""
    g = np.load(os.path.join(golden_dir, "flow_cv2.npz"))
    for k in _cases(g):
        seed, h, w, kind = [int(x) for x in g[k + "_meta"]]
        a, b = synth.flow_pair(seed, h, w, "shift" if kind == 0 else "noise")
        assert (oracle.bgr2gray(a) == g[k + "_gray0"]).all()      # gray conversion is bit-exact
        got = oracle.optical_flow(a, b)
        assert got.shape == (h, w, 2) and got.dtype == np.float32
        assert np.abs(got - g[k + "_flow"]).max() <= 1e-4, (k, np.abs(got - g[k + "_flow"]).max())
        if kind == 0 and h >= 64:  # the pair moves by (+1.5, -0.75): direction and rough size come out
            inner = got[16:-16, 16:-16].reshape(-1, 2).mean(0)
            assert 0.5 < inner[0] < 2.0 and -1.2 < inner[1] < -0.2, inner


def test_flow_1080p_matches_cv2_run_here():
    """configs[3]'s frame size, against cv2 itself (no stored golden: 16 MB of floats): max |d| <= 1e-4 px
    (measured 3.8e-5)."""
    import cv2
    a, b = synth.flow_pair(941, 1080, 1920, "shift")
    g0, g1 = cv2.cvtColor(a, cv2.COLOR_BGR2GRAY), cv2.cvtColor(b, cv2.COLOR_BGR2GRAY)
    assert (oracle.bgr2gray(a) == g0).all()
    ref = cv2.FarnebackOpticalFlow_create(3, 0.5, False, 15, 3, 5, 1.2, 0).calc(g0, g1, None)
    assert np.abs(oracle.optical_flow(a, b) - ref).max() <= 1e-4


def test_nv12_matches_the_reference_kernels_own_output(golden_dir):
    """tests/golden/nv12_ref.npz holds what the reference's OWN kernel (scanner/util/image.cu compiled
    unmodified, oracle/_ref) produced on an H100 (oracle/make_golden_ref.py): seeded surfaces (the output, or its
    SHA-256 where it is large), and the SHA-256 of its output over an input set that presents every (Y,Cb,Cr) triple
    (synth.nv12_exhaustive).  The restatement must reproduce both -- this is what pins the oracle's FMA contraction
    order."""
    import hashlib
    g = np.load(os.path.join(golden_dir, "nv12_ref.npz"))
    for k in _cases(g):
        seed, h, w, pitch = [int(x) for x in g[k + "_meta"]]
        luma, chroma = synth.nv12_surface(seed, h, w, pitch)
        got = oracle.nv12_to_rgb(luma, chroma, w)
        if k + "_out" in g.files:
            assert (got == g[k + "_out"]).all(), (k, h, w, pitch)
        else:
            assert hashlib.sha256(got.tobytes()).digest() == g[k + "_sha256"].tobytes(), (k, h, w, pitch)
    sha = hashlib.sha256()
    for f in range(synth.EXH_FRAMES):
        luma, chroma = synth.nv12_exhaustive(f)
        sha.update(oracle.nv12_to_rgb(luma, chroma, synth.EXH_W).tobytes())
    assert sha.digest() == g["exhaustive_sha256"].tobytes()
