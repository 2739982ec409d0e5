"""Kernel-ordered CPU oracle for Farneback dense optical flow -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The arithmetic lives in farneback_k.c (plain C, gcc, -ffp-contract=off): scanner_b200/csrc/flow.cu restated in its
own order of operations, so that the kernels equal it bit for bit.  oracle.farneback (orc_farneback_u8) stays the
specification held to cv2; tests/test_flow_exact_cpu.py holds this oracle within that specification's tolerance.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libfarneback_k.so")
_SRC = os.path.join(_HERE, "farneback_k.c")
# the flags of liborc.so (oracle/Makefile): every float expression rounds as written
CFLAGS = ["-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-shared"]
_LIB = None

DEFAULTS = dict(num_levels=3, pyr_scale=0.5, win_size=15, num_iters=3, poly_n=5, poly_sigma=1.2)
BOXES = {"f32": 0, "f64_slide": 1, "f64": 2}


def build(force=False):
    """Compile farneback_k.c into libfarneback_k.so when it is missing or older than its source."""
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
        _LIB.fbk_flow_u8c3.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                       ctypes.c_double, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                       ctypes.c_int, ctypes.c_void_p]
        _LIB.fbk_levels.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_void_p]
    return _LIB


def box_for(win_size, unfused=False, box_f64=False):
    """The box + solve variant scn_farneback_u8c3 launches: the float tree (box_solve_f32_kernel) for windows of
    half-width 7 (win_size 14 or 15), the sliding double sums (box_solve_fused_kernel) there under SCN_FLOW_BOX=f64,
    and the two-pass double box otherwise and under SCN_FLOW_UNFUSED=1."""
    if unfused or win_size // 2 != 7:
        return "f64"
    return "f64_slide" if box_f64 else "f32"


def levels(width, height, num_levels=3, pyr_scale=0.5):
    """[(w, h), ...] of the pyramid scn_farneback_u8c3 runs, level 0 first."""
    wh = (ctypes.c_int * 32)()
    n = lib().fbk_levels(width, height, int(num_levels), float(pyr_scale), wh)
    return [(wh[2 * i], wh[2 * i + 1]) for i in range(n)]


def flow(frame0, frame1, box=None, **params):
    """scn_farneback_u8c3 of one pair of RGB24 frames (H, W, 3) u8 -> (H, W, 2) float32 (dx, dy).  Keyword parameters
    as DEFAULTS; box is "f32", "f64_slide" or "f64", by default the one box_for(win_size) picks."""
    p = dict(DEFAULTS)
    unknown = set(params) - set(p)
    assert not unknown, unknown
    p.update(params)
    f0, f1 = (np.ascontiguousarray(f, np.uint8) for f in (frame0, frame1))
    assert f0.shape == f1.shape and f0.ndim == 3 and f0.shape[2] == 3, (f0.shape, f1.shape)
    h, w = f0.shape[:2]
    box = box or box_for(p["win_size"])
    out = np.zeros((h, w, 2), np.float32)
    rc = lib().fbk_flow_u8c3(f0.ctypes.data, f1.ctypes.data, w, h, int(p["num_levels"]), float(p["pyr_scale"]),
                             int(p["win_size"]), int(p["num_iters"]), int(p["poly_n"]), float(p["poly_sigma"]),
                             BOXES[box], out.ctypes.data)
    if rc:
        raise ValueError(f"fbk_flow_u8c3 refused {p} box={box}: {rc}")
    return out
