"""GaussianBlur without a GPU: the C restatement of cv2's 8-bit fixed-point path (oracle/gaussian_blur.c) against
live cv2.GaussianBlur and against recorded cv2 4.13 hashes, the product's host plans against cv2's own kernels, and
the refusals of the C ABI."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import gaussian_blur as G
from scanner_b200 import cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BORDERS = ("BORDER_REFLECT_101", "BORDER_REPLICATE", "BORDER_REFLECT")
KSIZES = tuple(range(1, 32, 2))


def _cv2_blur(cv2, img, ksize, sx, sy, border):
    return cv2.GaussianBlur(img, tuple(ksize), sx, sigmaY=sy, borderType=G.BORDERS[border]).reshape(img.shape)


def _plan(ksize, sx, sy=0.0, border=4):
    l = cabi.lib()
    host = np.zeros(l.scn_gaussian_blur_plan_bytes(), np.uint8)
    rc = l.scn_gaussian_blur_plan_fill(ksize[0], ksize[1], sx, sy, border, host.ctypes.data)
    return rc, host.view(np.int32)


def _plan_taps(ksize, sx, sy=0.0):
    rc, p = _plan(ksize, sx, sy)
    assert rc == 0
    kw, kh = p[1], p[2]
    return p[4:4 + kw], p[36:36 + kh]


@pytest.mark.parametrize("border", BORDERS)
@pytest.mark.parametrize("c", (1, 3))
def test_oracle_equals_live_cv2_on_every_ksize_pair(border, c):
    """Every odd (kw, kh) in 1-31 with sigma 0, on noise frames that are taller and wider than the kernel."""
    cv2 = pytest.importorskip("cv2")
    img = G.content("noise", 7 + c, 41, 37, c)
    for kw in KSIZES:
        for kh in KSIZES:
            want = _cv2_blur(cv2, img, (kw, kh), 0, 0, border)
            assert (G.gaussian_blur(img, (kw, kh), 0, 0, border) == want).all(), (kw, kh)


def test_oracle_equals_live_cv2_with_explicit_sigmas():
    """Explicit, anisotropic and ksize-0 sigmas on every ksize, all borders, C = 1 and 3."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    cases = [(k, k, s, 0.0) for k in KSIZES for s in (0.3, 0.8, 1.1, 2.0, 3.0, 5.5, 12.0)]
    cases += [(kw, kh, sx, sy) for kw, kh, sx, sy in [(5, 9, 2.0, 0), (9, 5, 1.0, 3.0), (0, 0, 1.5, 4.0), (0, 7, 2.2, 0),
                                                     (13, 0, 0, 1.7), (0, 0, 0.4, 0), (0, 0, 4.9, 0), (31, 3, 7.0, 0.2)]]
    cases += [(int(rng.choice((0,) + KSIZES)), int(rng.choice((0,) + KSIZES)), float(rng.uniform(0.05, 5)),
               float(rng.choice([0, rng.uniform(0.05, 5)]))) for _ in range(120)]
    n = 0
    for i, (kw, kh, sx, sy) in enumerate(cases):
        try:
            G.taps((kw, kh), sx, sy)
        except ValueError:
            continue  # a derived size above 31
        c = (1, 3)[i % 2]
        border = BORDERS[i % 3]
        img = G.content("noise", 100 + i, 29 + i % 7, 33 + i % 5, c)
        assert (G.gaussian_blur(img, (kw, kh), sx, sy, border) == _cv2_blur(cv2, img, (kw, kh), sx, sy, border)).all(), \
            (kw, kh, sx, sy, border, c)
        n += 1
    assert n > 200


@pytest.mark.parametrize("kind", ("noise", "zero", "full", "gradient"))
def test_oracle_equals_live_cv2_on_frames_smaller_than_the_kernel(kind):
    """Sides 1-9 against kernels up to 31, so every border reflects more than once."""
    cv2 = pytest.importorskip("cv2")
    i = 0
    for h in range(1, 10):
        for w in range(1, 10):
            for ksize, sx in (((3, 3), 0), ((31, 31), 0), ((7, 31), 0), ((0, 0), 2.0), ((17, 5), 1.2)):
                border = BORDERS[i % 3]
                c = (1, 3)[i % 2]
                img = G.content(kind, 300 + i, h, w, c)
                want = _cv2_blur(cv2, img, ksize, sx, 0, border)
                assert (G.gaussian_blur(img, ksize, sx, 0, border) == want).all(), (h, w, ksize, sx, border, c)
                i += 1


def test_oracle_equals_live_cv2_at_1080p():
    cv2 = pytest.importorskip("cv2")
    for c, ksize, sx, border in ((3, (7, 7), 0, ""), (1, (15, 15), 3.0, "BORDER_REPLICATE"),
                                 (3, (0, 0), 1.1, "BORDER_REFLECT")):
        img = G.content("noise", 5 + c, 1080, 1920, c)
        assert (G.gaussian_blur(img, ksize, sx, 0, border) == _cv2_blur(cv2, img, ksize, sx, 0, border)).all()


def test_oracle_equals_recorded_cv2_hashes():
    from oracle.make_golden_gaussian_blur import case_frame, case_key
    with open(os.path.join(ROOT, "tests", "golden", "gaussian_blur_cv2.json")) as f:
        rec = json.load(f)["sha256"]
    assert len(rec) == len(G.GOLDEN_CASES)
    for i, (h, w, c, ksize, sx, sy, border, kind) in enumerate(G.GOLDEN_CASES):
        got = G.gaussian_blur(case_frame(i, h, w, c, kind), ksize, sx, sy, border)
        assert hashlib.sha256(got.tobytes()).hexdigest() == rec[case_key(h, w, c, ksize, sx, sy, border, kind)], i


def _cv2_fixed_taps(cv2, n, sigma):
    """The 8-bit taps from cv2's own double kernel (cv2.getGaussianKernel is the bit-exact soft-float one), with
    the error-diffusion rounding of the fixed-point path."""
    k = cv2.getGaussianKernel(n, sigma, cv2.CV_64F).ravel()
    out, err, s = np.zeros(n, np.int32), 0.0, 0
    for i in range(n // 2):
        adj = k[i] * 256.0 + err
        v = int(np.rint(adj))
        err = adj - v
        out[i] = out[n - 1 - i] = v
        s += v
    out[n // 2] = 256 - 2 * s
    return out


def test_plan_taps_equal_the_taps_of_cv2s_own_kernel_on_a_sigma_sweep():
    """The plan computes the Gaussian with libm's exp; cv2 uses a soft-float exp whose doubles differ in the last
    bits.  No 8-bit tap may differ: every ksize on 1,500 sigmas spread from 0.01 to 50, plus sigma 0."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    sigmas = np.concatenate([[0.0], np.exp(rng.uniform(np.log(0.01), np.log(50), 1000)), np.arange(1, 501) * 0.05])
    for n in KSIZES:
        for s in sigmas:
            kx, ky = _plan_taps((n, n), float(s))
            want = _cv2_fixed_taps(cv2, n, float(s))
            assert (kx == want).all() and (ky == want).all(), (n, s)


def test_plan_taps_sum_to_one_and_are_symmetric():
    rng = np.random.default_rng(4)
    for kw in (0,) + KSIZES:
        for kh in (0,) + KSIZES:
            sx, sy = float(rng.uniform(0.1, 4.5)), float(rng.choice([0.0, rng.uniform(0.1, 4.5)]))
            rc, p = _plan((kw, kh), sx, sy)
            assert rc == 0, (kw, kh, sx, sy)
            for taps in _plan_taps((kw, kh), sx, sy):
                assert taps.sum() == 256 and (taps == taps[::-1]).all() and (taps >= 0).all()
            ox, oy = G.taps((kw, kh), sx, sy)
            px, py = _plan_taps((kw, kh), sx, sy)
            assert (px == ox).all() and (py == oy).all()


def test_ksize_derivation_and_sigma_defaults():
    # ksize 0 from sigma: cvRound(sigma * 6 + 1) | 1
    for s, k in ((0.1, 3), (0.5, 5), (1.0, 7), (1.1, 9), (2.0, 13), (4.9, 31)):
        rc, p = _plan((0, 0), s)
        assert rc == 0 and p[1] == k and p[2] == k, (s, p[1])
    # sigma_y 0 (or negative) means sigma_x
    assert (_plan((9, 9), 1.7, 0.0)[1] == _plan((9, 9), 1.7, 1.7)[1]).all()
    assert (_plan((9, 9), 1.7, -3.0)[1] == _plan((9, 9), 1.7, 1.7)[1]).all()
    # sigma <= 0 on a ksize <= 9 takes cv2's fixed tables
    for n, want in ((3, [64, 128, 64]), (5, [16, 64, 96, 64, 16]), (7, [8, 28, 56, 72, 56, 28, 8]),
                    (9, [4, 13, 30, 51, 60, 51, 30, 13, 4])):
        assert list(_plan_taps((n, n), 0.0)[0]) == want


def test_border_names():
    l = cabi.lib()
    for name, code in (("", 4), ("BORDER_DEFAULT", 4), ("BORDER_REFLECT_101", 4), ("BORDER_REFLECT101", 4),
                       ("BORDER_REPLICATE", 1), ("BORDER_REFLECT", 2)):
        assert l.scn_gaussian_blur_border_code(name.encode()) == code, name
    for name in ("BORDER_CONSTANT", "BORDER_WRAP", "BORDER_TRANSPARENT", "BORDER_ISOLATED"):
        assert l.scn_gaussian_blur_border_code(name.encode()) == -2, name
    assert l.scn_gaussian_blur_border_code(b"reflect") == -1
    supported = l.scn_gaussian_blur_borders().decode()
    for name in ("BORDER_DEFAULT", "BORDER_REFLECT_101", "BORDER_REPLICATE", "BORDER_REFLECT"):
        assert name in supported


def test_bad_arguments_are_refused_without_a_gpu():
    """Refusals return SCN_E_* before anything reaches the device: scn_launch_count() stays where it was."""
    l = cabi.lib()
    before = l.scn_launch_count()
    BAD, UNSUP, PLAN = -1, -2, -3
    for args, want in ((((4, 3), 1.0, 0.0), BAD), (((3, -1), 1.0, 0.0), BAD), (((0, 3), 0.0, 0.0), BAD),
                       (((0, 0), -1.0, 0.0), BAD), (((3, 3), float("nan"), 0.0), BAD),
                       (((3, 3), 1.0, float("inf")), BAD), (((33, 3), 1.0, 0.0), UNSUP),
                       (((0, 0), 5.5, 0.0), UNSUP), (((3, 35), 0.0, 0.0), UNSUP)):
        assert _plan(*args)[0] == want, args
    assert _plan((3, 3), 1.0, 0.0, border=0)[0] == BAD  # BORDER_CONSTANT's number
    assert _plan((3, 3), 1.0, 0.0, border=3)[0] == BAD
    assert l.scn_gaussian_blur_plan_fill(3, 3, 1.0, 0.0, 4, None) == BAD

    rc, plan = _plan((5, 5), 1.0)
    assert rc == 0
    pp = plan.ctypes.data
    fake = (ctypes.c_void_p * 2)(0x1000, 0x2000)
    for c in (0, 2, 4):
        assert l.scn_gaussian_blur_u8(pp, fake, 2, 16, 16, c, fake, None) == BAD, c
    assert l.scn_gaussian_blur_u8(pp, fake, -1, 16, 16, 3, fake, None) == BAD
    assert l.scn_gaussian_blur_u8(pp, fake, 2, -16, 16, 3, fake, None) == BAD
    assert l.scn_gaussian_blur_u8(pp, None, 2, 16, 16, 3, fake, None) == BAD
    assert l.scn_gaussian_blur_u8(pp, fake, 2, 16, 16, 3, None, None) == BAD
    assert l.scn_gaussian_blur_u8(pp, fake, 2, 65536, 32769, 1, fake, None) == BAD  # over INT_MAX pixels
    assert l.scn_gaussian_blur_u8(None, fake, 2, 16, 16, 3, fake, None) == PLAN
    broken = plan.copy()
    broken[4] += 1  # taps no longer sum to 256
    assert l.scn_gaussian_blur_u8(broken.ctypes.data, fake, 2, 16, 16, 3, fake, None) == PLAN
    assert l.scn_gaussian_blur_u8(np.zeros_like(plan).ctypes.data, fake, 2, 16, 16, 3, fake, None) == PLAN
    assert l.scn_gaussian_blur_u8(pp, fake, 0, 16, 16, 3, fake, None) == 0  # nothing to do

    assert l.scn_gaussian_blur_nv12(pp, fake, fake, 16, 2, 15, 16, fake, None) == BAD  # odd width
    assert l.scn_gaussian_blur_nv12(pp, fake, fake, 16, 2, 16, 15, fake, None) == BAD  # odd height
    assert l.scn_gaussian_blur_nv12(pp, fake, fake, 8, 2, 16, 16, fake, None) == BAD  # pitch below width
    assert l.scn_gaussian_blur_nv12(pp, fake, fake, 16, -1, 16, 16, fake, None) == BAD
    assert l.scn_gaussian_blur_nv12(pp, None, fake, 16, 2, 16, 16, fake, None) == BAD
    assert l.scn_gaussian_blur_nv12(pp, fake, None, 16, 2, 16, 16, fake, None) == BAD
    assert l.scn_gaussian_blur_nv12(pp, fake, fake, 16, 2, 16, 16, None, None) == BAD
    assert l.scn_gaussian_blur_nv12(None, fake, fake, 16, 2, 16, 16, fake, None) == PLAN
    assert l.scn_launch_count() == before
