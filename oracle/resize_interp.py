"""CPU oracle for Resize's INTER_NEAREST and INTER_AREA -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The arithmetic lives in resize_interp.c (plain C, gcc, -ffp-contract=off), which documents cv2's rules; this module
is a ctypes shim returning numpy arrays.  INTER_LINEAR is oracle.resize.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libresize_interp.so")
_SRC = os.path.join(_HERE, "resize_interp.c")
# the flags of liborc.so (oracle/Makefile): every float expression rounds as written
CFLAGS = ["-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]
_LIB = None


def build(force=False):
    """Compile resize_interp.c into libresize_interp.so when it is missing or older than its source."""
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


def _run(fn, frame, dw, dh):
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    if frame.ndim == 2:
        frame = frame[..., None]
    h, w, c = frame.shape
    out = np.zeros((dh, dw, c), np.uint8)
    fn(frame.ctypes.data_as(ctypes.c_void_p), w, h, c, out.ctypes.data_as(ctypes.c_void_p), dw, dh)
    return out


def resize_nearest(frame, dw, dh):
    """cv2.resize(frame, (dw, dh), interpolation=cv2.INTER_NEAREST) on a u8 (H, W, C) frame."""
    return _run(lib().orc_resize_nearest_u8, frame, dw, dh)


def resize_area(frame, dw, dh):
    """cv2.resize(frame, (dw, dh), interpolation=cv2.INTER_AREA) on a u8 (H, W, C) frame."""
    return _run(lib().orc_resize_area_u8, frame, dw, dh)


def resize(frame, dw, dh, interpolation="INTER_LINEAR"):
    """The oracle of Resize's `interpolation` argument: "" and INTER_LINEAR are oracle.resize."""
    if interpolation in ("", "INTER_LINEAR"):
        from . import resize as linear
        return linear(frame, dw, dh)
    return {"INTER_NEAREST": resize_nearest, "INTER_AREA": resize_area}[interpolation](frame, dw, dh)


def area_regime(sw, sh, dw, dh):
    """Which INTER_AREA regime cv2 takes: 'up' (a scale below 1: linear arithmetic with area taps), 'int2x2',
    'int' (integer factors) or 'float' (fractional downscale)."""
    sx, sy = 1.0 / (dw / sw), 1.0 / (dh / sh)
    if sx < 1 or sy < 1:
        return "up"
    if sw % dw == 0 and sh % dh == 0:
        return "int2x2" if (sw // dw, sh // dh) == (2, 2) else "int"
    return "float"


def content(kind, seed, h, w, cell=(2, 2)):
    """Test frames: 'noise', 'zero', 'full' (255), 'gradient', or 'half': every (kx, ky) = `cell` box of the frame
    averages to an exact .5 (multiples of kx * ky, plus 1 on even rows when ky is even, else on even columns), so that
    the 2 x 2 case's half-up rounding and the other factors' half-to-even rounding both show."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind in ("zero", "full"):
        return np.full((h, w, 3), 255 if kind == "full" else 0, np.uint8)
    if kind == "gradient":
        yy, xx = np.mgrid[0:h, 0:w]
        return np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx + yy) % 256], -1).astype(np.uint8)
    assert kind == "half", kind
    kx, ky = cell
    k = kx * ky
    img = (rng.integers(0, 256 // k, (h, w, 3)) * k).astype(np.uint8)
    if ky % 2 == 0:
        img[::2] += 1
    elif kx % 2 == 0:
        img[:, ::2] += 1
    return img


# (src_w, src_h, dst_w, dst_h, content) of the recorded cv2 hashes (tests/golden/resize_interp_cv2.json)
GOLDEN_CASES = [
    (1920, 1080, 224, 224, "noise"), (3840, 2160, 224, 224, "noise"), (1920, 1080, 224, 224, "gradient"),
    (1920, 1080, 480, 270, "noise"), (1920, 1080, 960, 540, "half"), (1920, 1080, 480, 270, "half"),
    (3840, 2160, 1, 1, "full"), (3840, 2160, 1, 1, "noise"), (97, 61, 40, 25, "noise"), (300, 200, 224, 150, "noise"),
    (64, 48, 23, 17, "noise"), (224, 224, 1920, 1080, "noise"), (64, 48, 32, 96, "noise"),
    (1920, 1080, 224, 2000, "noise"), (17, 3, 5, 9, "noise"), (128, 80, 64, 80, "half"), (128, 80, 128, 40, "half"),
    (192, 160, 32, 40, "half"), (480, 270, 480, 270, "noise"), (255, 255, 37, 37, "zero"), (1079, 1919, 224, 224, "noise"),
]


def golden_cell(sw, sh, dw, dh):
    return (max(sw // dw, 1), max(sh // dh, 1))
