"""CPU oracle for the GaussianBlur op -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The arithmetic lives in gaussian_blur.c (plain C, gcc, -ffp-contract=off), which documents cv2's rules; this module
is a ctypes shim returning numpy arrays.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libgaussian_blur.so")
_SRC = os.path.join(_HERE, "gaussian_blur.c")
# the flags of liborc.so (oracle/Makefile): every float expression rounds as written
CFLAGS = ["-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]
_LIB = None

# cv2's BorderTypes numbers of the supported borders
BORDERS = {"": 4, "BORDER_DEFAULT": 4, "BORDER_REFLECT_101": 4, "BORDER_REPLICATE": 1, "BORDER_REFLECT": 2}


def build(force=False):
    """Compile gaussian_blur.c into libgaussian_blur.so when it is missing or older than its source."""
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
        L = ctypes.CDLL(build())
        L.orc_gaussian_taps.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.orc_gaussian_blur_u8.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                           ctypes.c_double, ctypes.c_int]
        _LIB = L
    return _LIB


def _border(border):
    return BORDERS[border] if isinstance(border, str) else int(border)


def taps(ksize, sigma_x, sigma_y=0.0):
    """(kx, ky) int32 arrays: the 8-fraction-bit taps cv2 uses for ksize (kw, kh) and the sigmas."""
    kx, ky = np.zeros(31, np.int32), np.zeros(31, np.int32)
    kw, kh = ctypes.c_int(), ctypes.c_int()
    rc = lib().orc_gaussian_taps(int(ksize[0]), int(ksize[1]), float(sigma_x), float(sigma_y), kx.ctypes.data,
                                 ctypes.byref(kw), ky.ctypes.data, ctypes.byref(kh))
    if rc:
        raise ValueError(f"GaussianBlur arguments refused ({rc}): ksize={ksize} sigma=({sigma_x}, {sigma_y})")
    return kx[:kw.value].copy(), ky[:kh.value].copy()


def gaussian_blur(frame, ksize, sigma_x, sigma_y=0.0, border=""):
    """cv2.GaussianBlur(frame, ksize, sigma_x, sigmaY=sigma_y, borderType=border) on a u8 (H, W) or (H, W, C) frame
    -> (H, W, C)."""
    frame = np.ascontiguousarray(frame, dtype=np.uint8)
    if frame.ndim == 2:
        frame = frame[..., None]
    h, w, c = frame.shape
    out = np.zeros((h, w, c), np.uint8)
    rc = lib().orc_gaussian_blur_u8(frame.ctypes.data, w, h, c, out.ctypes.data, int(ksize[0]), int(ksize[1]),
                                    float(sigma_x), float(sigma_y), _border(border))
    if rc:
        raise ValueError(f"GaussianBlur arguments refused ({rc}): ksize={ksize} sigma=({sigma_x}, {sigma_y})")
    return out


def content(kind, seed, h, w, c=3):
    """Test frames: 'noise', 'zero', 'full' (255) or 'gradient'."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, c), dtype=np.uint8)
    if kind in ("zero", "full"):
        return np.full((h, w, c), 255 if kind == "full" else 0, np.uint8)
    assert kind == "gradient", kind
    yy, xx = np.mgrid[0:h, 0:w]
    g = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx * 7 + yy * 3) % 256], -1)
    return g[..., :c].astype(np.uint8)


# (h, w, c, (kw, kh), sigma_x, sigma_y, border, content) of the recorded cv2 hashes (tests/golden/gaussian_blur_cv2.json)
GOLDEN_CASES = [
    (1080, 1920, 3, (3, 3), 0, 0, "", "noise"), (1080, 1920, 3, (5, 5), 1.1, 0, "", "noise"),
    (1080, 1920, 3, (7, 7), 0, 0, "", "noise"), (1080, 1920, 3, (15, 15), 3, 0, "", "noise"),
    (1080, 1920, 3, (31, 31), 0, 0, "", "noise"), (1080, 1920, 3, (5, 9), 2, 0, "", "noise"),
    (1080, 1920, 1, (9, 9), 0, 0, "", "noise"), (1080, 1920, 1, (0, 0), 2.5, 0, "BORDER_REPLICATE", "gradient"),
    (720, 1280, 3, (0, 0), 1.5, 4.0, "BORDER_REFLECT", "noise"), (720, 1280, 3, (11, 3), 0, 0, "BORDER_REPLICATE", "noise"),
    (480, 640, 3, (31, 1), 7.0, 0, "BORDER_REFLECT", "gradient"), (480, 640, 1, (1, 31), 0, 0.7, "", "noise"),
    (97, 61, 3, (21, 13), 4.5, 1.3, "BORDER_REFLECT_101", "noise"), (17, 5, 3, (31, 31), 0, 0, "", "noise"),
    (5, 17, 1, (29, 3), 0, 0, "BORDER_REFLECT", "noise"), (3, 2, 3, (31, 31), 9.0, 9.0, "BORDER_REPLICATE", "noise"),
    (1, 1, 3, (31, 31), 0, 0, "", "noise"), (1, 40, 3, (7, 7), 0, 0, "", "noise"), (40, 1, 1, (7, 7), 0, 0, "", "noise"),
    (256, 256, 3, (13, 13), 0, 0, "", "full"), (256, 256, 3, (13, 13), 0, 0, "", "zero"),
    (256, 256, 3, (0, 0), 4.9, 0, "", "gradient"),
]
