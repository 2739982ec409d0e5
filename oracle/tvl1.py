"""CPU oracle for TV-L1 dense optical flow -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The arithmetic lives in tvl1.c (plain C, gcc, -ffp-contract=off); this module is a ctypes shim returning numpy
arrays, plus flow_pair_known, the known-motion test pairs.  DESIGN.md section 11 is the specification.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libtvl1.so")
_SRC = os.path.join(_HERE, "tvl1.c")
# the flags of liborc.so (oracle/Makefile): every float expression rounds as written
CFLAGS = ["-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]
_LIB = None

DEFAULTS = dict(tau=0.25, lambda_=0.15, theta=0.3, nscales=5, warps=5, epsilon=0.01, iterations=300,
                scale_step=0.8, median_filtering=5)


def build(force=False):
    """Compile tvl1.c into libtvl1.so when it is missing or older than its source."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        fd, tmp = tempfile.mkstemp(suffix=".so", dir=_HERE)
        os.close(fd)
        try:
            subprocess.check_call([os.environ.get("CC", "gcc"), *CFLAGS, "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, _SO)
        finally:
            if os.path.exists(tmp):
                os.unlink(tmp)
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build())
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def gray_u8(frame):
    """(H, W) or (H, W, 1) u8 as it is; (H, W, 3) RGB through cv2's COLOR_RGB2GRAY (oracle/convert_color.py)."""
    frame = np.asarray(frame, np.uint8)
    if frame.ndim == 3 and frame.shape[2] == 3:
        from .convert_color import convert_color
        return np.ascontiguousarray(convert_color(frame, "COLOR_RGB2GRAY")[..., 0])
    if frame.ndim == 3 and frame.shape[2] == 1:
        frame = frame[..., 0]
    assert frame.ndim == 2, frame.shape
    return np.ascontiguousarray(frame)


def levels(width, height, nscales=5, scale_step=0.8):
    """[(w, h), ...] of a TV-L1 pyramid, level 0 first."""
    ws, hs = (ctypes.c_int * 16)(), (ctypes.c_int * 16)()
    n = lib().orc_tvl1_levels(width, height, int(nscales), ctypes.c_float(scale_step), ws, hs)
    return [(ws[i], hs[i]) for i in range(n)]


def resize(img, dw, dh):
    """cv2.resize(float32 img, (dw, dh), interpolation=INTER_LINEAR), as the pyramid and the flow upsampling
    apply it."""
    img = np.ascontiguousarray(img, np.float32)
    h, w = img.shape
    out = np.zeros((dh, dw), np.float32)
    lib().orc_tvl1_resize_f32(_p(img), w, h, _p(out), int(dw), int(dh))
    return out


def median(img, k):
    """cv2.medianBlur(float32 img, k), k = 3 or 5."""
    img = np.ascontiguousarray(img, np.float32)
    h, w = img.shape
    out = np.zeros_like(img)
    lib().orc_tvl1_median_f32(_p(img), w, h, int(k), _p(out))
    return out


def tile_sum(terms):
    """The sum of float32 terms in the order of tvl1_iterate_kernel's stop error (orc_tvl1_tile_sum), as a float."""
    terms = np.ascontiguousarray(terms, np.float32).ravel()
    L = lib()
    L.orc_tvl1_tile_sum.restype = ctypes.c_double
    return L.orc_tvl1_tile_sum(_p(terms), int(terms.size))


def flow(frame0, frame1, return_iterations=False, error_sum="sequential", **params):
    """TV-L1 dense flow of one pair -> (H, W, 2) float32 (dx, dy).  Frames are u8 gray (H, W) or RGB (H, W, 3).
    Keyword parameters as DEFAULTS.  With return_iterations, also int32 [nscales][warps]: the iterations each
    (level, warp) ran, level 0 (finest) first, 0 for levels the pyramid stops before.  error_sum: "sequential"
    sums the stop error in double pixel by pixel (the specification); "tiles" sums the same float terms in the
    order of the GPU kernel (tile_sum), so that a warp step stops after the same iteration as on the GPU."""
    assert error_sum in ("sequential", "tiles"), error_sum
    p = dict(DEFAULTS)
    unknown = set(params) - set(p)
    assert not unknown, unknown
    p.update(params)
    g0, g1 = gray_u8(frame0), gray_u8(frame1)
    assert g0.shape == g1.shape
    h, w = g0.shape
    out = np.zeros((h, w, 2), np.float32)
    iters = np.zeros((int(p["nscales"]), int(p["warps"])), np.int32)
    f = ctypes.c_float
    lib().orc_tvl1_u8(_p(g0), _p(g1), w, h, f(p["tau"]), f(p["lambda_"]), f(p["theta"]), int(p["nscales"]),
                      int(p["warps"]), f(p["epsilon"]), int(p["iterations"]), f(p["scale_step"]),
                      int(p["median_filtering"]), int(error_sum == "tiles"), _p(out), _p(iters))
    return (out, iters) if return_iterations else out


# ---- known-motion pairs -------------------------------------------------------------------------------------------
def tex_gray(seed, x, y):
    """The analytic sum-of-sinusoids texture of synth.flow_pair (its first channel), unclipped float, at (x, y)."""
    acc = np.zeros(np.broadcast(x, y).shape)
    r2 = np.random.default_rng(seed * 10)
    for _ in range(6):
        fx, fy, ph = r2.uniform(0.02, 0.25), r2.uniform(0.02, 0.25), r2.uniform(0, 6.28)
        acc += np.sin(fx * x + fy * y + ph)
    return 127.5 + 20 * acc


def flow_pair_known(seed, h, w, kind="shift"):
    """(frame0, frame1, true_flow): two u8 gray frames and the float32 (h, w, 2) flow (dx, dy) with
    frame1(x + u(x)) = frame0(x) holding exactly for the analytic texture (frame1 is sampled at the inverse map).
      "shift":  the synth.flow_pair translation (1.5, -0.75) everywhere.
      "affine": a rotation by 0.02 rad and a zoom of 1.02 about the centre (|u| <= 8 px up to ~270 x 480).
      "square": a textured square (a second texture, side min(h, w) / 3, centred) moved by (1.25, -0.6) over the
                static texture; the true flow is zero outside the square.
    Frames are rounded to u8 after the exact relation, so it holds up to that rounding."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    q = lambda v: np.clip(np.rint(v), 0, 255).astype(np.uint8)  # noqa: E731
    if kind == "shift":
        dx, dy = 1.5, -0.75
        f0, f1 = tex_gray(seed, xx, yy), tex_gray(seed, xx - dx, yy - dy)
        fl = np.stack([np.full((h, w), dx), np.full((h, w), dy)], -1)
    elif kind == "affine":
        cx, cy, a, z = (w - 1) / 2, (h - 1) / 2, 0.02, 1.02
        c, s = z * np.cos(a), z * np.sin(a)
        # forward map T(x) = C + A (x - C); u = T(x) - x; frame1(y) = frame0(T^-1 y)
        X, Y = xx - cx, yy - cy
        fl = np.stack([(c - 1) * X - s * Y, s * X + (c - 1) * Y], -1)
        det = c * c + s * s
        xi, yi = (c * X + s * Y) / det + cx, (-s * X + c * Y) / det + cy
        f0, f1 = tex_gray(seed, xx, yy), tex_gray(seed, xi, yi)
    elif kind == "square":
        dx, dy = 1.25, -0.6
        side = min(h, w) // 3
        x0, y0 = (w - side) / 2, (h - side) / 2
        inside = lambda x, y: (x >= x0) & (x < x0 + side) & (y >= y0) & (y < y0 + side)  # noqa: E731
        f0 = np.where(inside(xx, yy), tex_gray(seed + 7, xx, yy), tex_gray(seed, xx, yy))
        # frame1: the square has moved by (dx, dy); where it is not, the static background shows
        f1 = np.where(inside(xx - dx, yy - dy), tex_gray(seed + 7, xx - dx, yy - dy), tex_gray(seed, xx, yy))
        m = inside(xx, yy)
        fl = np.stack([np.where(m, dx, 0.0), np.where(m, dy, 0.0)], -1)
    else:
        raise ValueError(kind)
    return q(f0), q(f1), fl.astype(np.float32)
