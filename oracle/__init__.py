"""CPU oracle for the scanner hot path -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
reference legs may import this package.  The product (scanner_b200/) never does.

The arithmetic lives in scn_oracle.c (plain C, gcc); this module is a ctypes
shim returning numpy arrays.  Each wrapper names the reference file:line its C
function restates.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force=False):
    so = os.path.join(_HERE, "liborc.so")
    src = os.path.join(_HERE, "scn_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-B", "liborc.so"],
                              stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build())
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def hist16(frame):
    """tests/test_ops.cpp:13-59 -> int32[3,16]."""
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    h, w, c = frame.shape
    assert c == 3
    out = np.zeros((3, 16), np.int32)
    lib().orc_hist16_u8c3(_p(frame), ctypes.c_int(w), ctypes.c_int(h), _p(out))
    return out


def resize_target(src_w, src_h, width=0, height=0, min=False, preserve_aspect=False):
    """tests/test_ops.cpp:126-147."""
    ow, oh = ctypes.c_int(), ctypes.c_int()
    lib().orc_resize_target(src_w, src_h, width, height, int(min), int(preserve_aspect),
                            ctypes.byref(ow), ctypes.byref(oh))
    return ow.value, oh.value


def resize(frame, dw, dh):
    """tests/test_ops.cpp:156 (cv::resize INTER_LINEAR, u8)."""
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    h, w, c = frame.shape
    out = np.zeros((dh, dw, c), np.uint8)
    lib().orc_resize_bilinear_u8(_p(frame), w, h, c, _p(out), dw, dh)
    return out


def blur(frame, kernel_size):
    """tests/test_ops.cpp:239-310 (border defined as 0)."""
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    h, w, c = frame.shape
    assert c == 3
    out = np.zeros_like(frame)
    lib().orc_blur_u8c3(_p(frame), w, h, int(kernel_size), _p(out))
    return out


def blur_sat(frame, kernel_size):
    """blur() restated with a summed-area table, O(1) per sample: fl = ceil(k/2) - 1, fr = k/2; an interior sample
    is the sum of its (fl + fr + 1)^2 window integer-divided by (fl + fr + 1)^2, every other sample is 0 (so is the
    whole frame when a side is shorter than the window).  Sums are uint32 with wrap-around: a window sum is below
    31^2 * 255 < 2^32, so differences of wrapped prefix sums are exact.  Takes (H, W, 3) or (N, H, W, 3)."""
    frame = np.asarray(frame, dtype=np.uint8)
    h, w = frame.shape[-3], frame.shape[-2]
    fl, fr = (kernel_size + 1) // 2 - 1, kernel_size // 2
    k = fl + fr + 1
    out = np.zeros_like(frame)
    if h < k or w < k:
        return out
    s = np.zeros(frame.shape[:-3] + (h + 1, w + 1, frame.shape[-1]), np.uint32)
    np.cumsum(frame, axis=-3, dtype=np.uint32, out=s[..., 1:, 1:, :])
    np.cumsum(s[..., 1:, 1:, :], axis=-2, dtype=np.uint32, out=s[..., 1:, 1:, :])
    win = s[..., k:, k:, :] - s[..., :-k, k:, :]
    win -= s[..., k:, :-k, :]
    win += s[..., :-k, :-k, :]
    out[..., fl:h - fr, fl:w - fr, :] = win // np.uint32(k * k)
    return out


def blur_interior(h, w, kernel_size):
    """Slices of the region the reference actually writes (test_ops.cpp:278-279)."""
    import math
    fl = int(math.ceil(kernel_size / 2.0)) - 1
    fr = kernel_size // 2
    return slice(fl, h - fr), slice(fl, w - fr)


def nv12_to_rgb(luma, chroma, width=None):
    """scanner/util/image.cu:67-200.  luma: (H,P) u8, chroma: (H/2,P) u8 interleaved CbCr."""
    luma = np.ascontiguousarray(luma, dtype=np.uint8)
    chroma = np.ascontiguousarray(chroma, dtype=np.uint8)
    h, pitch = luma.shape
    w = pitch if width is None else width
    assert chroma.shape == (h // 2, pitch)
    out = np.zeros((h, w, 3), np.uint8)
    lib().orc_nv12_to_rgb24(_p(luma), _p(chroma), ctypes.c_size_t(pitch), w, h, _p(out),
                            ctypes.c_size_t(w * 3))
    return out


def nv12_hist_resize(luma, chroma, dw, dh, width=None):
    """configs[1] DAG on one surface: NV12 -> RGB -> {Histogram, Resize}."""
    luma = np.ascontiguousarray(luma, dtype=np.uint8)
    chroma = np.ascontiguousarray(chroma, dtype=np.uint8)
    h, pitch = luma.shape
    w = pitch if width is None else width
    hist = np.zeros((3, 16), np.int32)
    res = np.zeros((dh, dw, 3), np.uint8)
    scratch = np.zeros((h, w, 3), np.uint8)
    lib().orc_nv12_hist_resize(_p(luma), _p(chroma), ctypes.c_size_t(pitch), w, h, _p(hist),
                               _p(res), dw, dh, _p(scratch))
    return hist, res


def index_column(start, n):
    """scanner/engine/ingest.cpp:337-345."""
    out = np.zeros(n * 8, np.uint8)
    lib().orc_index_column(ctypes.c_int64(start), ctypes.c_int64(n), _p(out))
    return out


def bgr2gray(frame):
    """cv::cvtColor(COLOR_BGR2GRAY) as the reference applies it to its RGB frames
    (tests/test_ops.cpp:91-92): 15-bit fixed point, first channel weighted 0.114."""
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    h, w, c = frame.shape
    assert c == 3
    out = np.zeros((h, w), np.uint8)
    lib().orc_bgr2gray_u8c3(_p(frame), w, h, _p(out))
    return out


def farneback(gray0, gray1, num_levels=3, pyr_scale=0.5, win_size=15, num_iters=3, poly_n=5, poly_sigma=1.2):
    """cv::FarnebackOpticalFlow(3, 0.5, false, 15, 3, 5, 1.2, 0)->calc (tests/test_ops.cpp:68-69,94)."""
    gray0 = np.ascontiguousarray(gray0, dtype=np.uint8)
    gray1 = np.ascontiguousarray(gray1, dtype=np.uint8)
    h, w = gray0.shape
    out = np.zeros((h, w, 2), np.float32)
    lib().orc_farneback_u8(_p(gray0), _p(gray1), w, h, int(num_levels), ctypes.c_double(pyr_scale), int(win_size),
                           int(num_iters), int(poly_n), ctypes.c_double(poly_sigma), _p(out))
    return out


def optical_flow(frame0, frame1):
    """The reference's OpticalFlow op on one stencil window {0,1} of RGB frames -> (H,W,2) float32."""
    return farneback(bgr2gray(frame0), bgr2gray(frame1))
