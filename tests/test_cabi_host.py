"""CPU-side checks of the C-ABI library: it loads, exports every symbol include/scn_kernels.h
declares, and its host-only entry points (resize target rule, resize plan) agree with the
oracle.  No compute launches here -- there is no GPU in the build container."""
import ctypes
import os
import re

import numpy as np
import pytest

import oracle
from oracle import synth
from scanner_b200 import cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    return sorted(set(re.findall(r"SCN_API\s+[\w\s\*]+?\b(scn_\w+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    names = _declared_symbols("scn_kernels.h")
    assert len(names) >= 13
    l = ctypes.CDLL(cabi.LIB_PATH)
    for n in names:
        assert hasattr(l, n), f"libscn_kernels.so does not export {n}"
    # and the Python binding table covers the header exactly
    assert sorted(cabi.SIGNATURES) == names


def test_abi_version_and_launch_counter():
    l = cabi.lib()
    assert l.scn_abi_version() == 1
    assert l.scn_launch_count() == 0  # nothing launched on a CPU-only run


def test_resize_target_matches_oracle():
    l = cabi.lib()
    fixed = [(1920, 1080, 224, 224, 0, 0), (1920, 1080, 0, 540, 0, 1), (1920, 1080, 640, 0, 0, 1),
             (640, 480, 1000, 1000, 1, 0), (640, 480, 320, 1000, 1, 0), (640, 480, 0, 0, 0, 0), (33, 77, 100, 0, 1, 1),
             (1920, 1080, 1, 0, 0, 1), (1920, 1080, 0, 0, 0, 1), (1080, 1920, 0, 1, 0, 1)]
    rng = np.random.default_rng(17)
    sides = (0,) + synth.RESIZE_SIDES
    sweep = [tuple(int(x) for x in rng.choice(sides, 4)) + (int(rng.integers(2)), int(rng.integers(2)))
             for _ in range(3000)]
    zero = 0
    for (sw, sh, w, h, mn, pa) in fixed + [g for g in sweep if g[0] and g[1]]:
        ow, oh = ctypes.c_int(), ctypes.c_int()
        l.scn_resize_target(sw, sh, w, h, mn, pa, ctypes.byref(ow), ctypes.byref(oh))
        assert (ow.value, oh.value) == oracle.resize_target(sw, sh, w, h, bool(mn), bool(pa)), (sw, sh, w, h, mn, pa)
        zero += ow.value <= 0 or oh.value <= 0
    # the zero targets the Resize op refuses: 1920 x 1080 at width 1 with preserve_aspect is 1 x 0
    assert oracle.resize_target(1920, 1080, 1, 0, preserve_aspect=True) == (1, 0)
    assert oracle.resize_target(1920, 1080, 0, 0, preserve_aspect=True) == (0, 0)
    assert zero > 100


def _apply_plan_numpy(img, plan_bytes, dw, dh):
    """Apply the PRODUCT's plan with numpy -- checks the host table logic against the oracle."""
    p = plan_bytes.view(np.int32)
    hdr, taps = p[:8], p[8:].reshape(-1, 4)
    assert hdr[3] == dw and hdr[4] == dh
    xt, yt = taps[:dw], taps[dw:dw + dh]
    s = img.astype(np.int32)
    hb = s[:, xt[:, 0], :] * xt[None, :, 2, None] + s[:, xt[:, 1], :] * xt[None, :, 3, None]
    h0, h1 = hb[yt[:, 0]], hb[yt[:, 1]]
    b0, b1 = yt[:, 2][:, None, None], yt[:, 3][:, None, None]
    return ((((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2).astype(np.uint8)


@pytest.mark.parametrize("h,w,dh,dw", [(48, 64, 20, 30), (100, 130, 333, 257), (7, 9, 224, 224),
                                       (1080, 1920, 224, 224), (37, 53, 37, 53), (64, 64, 1, 1),
                                       (5, 1, 3, 4)])
def test_resize_plan_matches_oracle(h, w, dh, dw):
    l = cabi.lib()
    n = l.scn_resize_plan_bytes(dw, dh)
    assert n == 32 + 16 * (dw + dh)
    buf = np.zeros(n, np.uint8)
    assert l.scn_resize_plan_fill(w, h, dw, dh, buf.ctypes.data) == 0
    img = synth.rand_frame(7, h, w)
    assert (_apply_plan_numpy(img, buf, dw, dh) == oracle.resize(img, dw, dh)).all()


def _cv2_taps(ssz, dsz, clamp_x):
    """cv::resize's INTER_LINEAR table for one axis restated in float32 numpy (OpenCV imgproc/src/resize.cpp):
    f = (float)((d + 0.5) * scale - 0.5), s = floor(f), weights saturate_cast<short>((1 - f, f) * 2048).  On x a tap
    left of 0 or at/after the last pixel becomes (edge, weight 2048, 0); on y the weights stay and the rows clamp."""
    scale = 1.0 / (dsz / ssz)
    f = ((np.arange(dsz) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = f - s.astype(np.float32)
    if clamp_x:
        f[s < 0], s[s < 0] = 0, 0
        last = s >= ssz - 1
        f[last], s[last] = 0, ssz - 1
    w0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    w1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return np.stack([np.clip(s, 0, ssz - 1), np.clip(s + 1, 0, ssz - 1), w0, w1], 1)


def test_resize_plan_equals_cv2_over_a_sweep():
    """The product's plan over ~2000 seeded geometries (every side from synth.RESIZE_SIDES): the header, every tap
    and weight against cv2's table, and the plan applied with numpy against live cv2.resize.  Exact-2x geometries
    take INTER_AREA in cv2 and in the kernels, so there only the header flag and the table are checked."""
    cv2 = pytest.importorskip("cv2")
    l = cabi.lib()
    big = synth.rand_frame(23, 1920, 1920)
    area = 0
    for k, (sw, sh, dw, dh) in enumerate(synth.resize_geometries(5, 2000)):
        buf = np.zeros(l.scn_resize_plan_bytes(dw, dh), np.uint8)
        assert l.scn_resize_plan_fill(sw, sh, dw, dh, buf.ctypes.data) == 0
        hdr, taps = buf.view(np.int32)[:8], buf.view(np.int32)[8:].reshape(-1, 4)
        area2x = sw == 2 * dw and sh == 2 * dh
        assert list(hdr[1:6]) == [sw, sh, dw, dh, int(area2x)], (sw, sh, dw, dh)
        assert (taps[:dw] == _cv2_taps(sw, dw, True)).all(), ("x", sw, sh, dw, dh)
        assert (taps[dw:] == _cv2_taps(sh, dh, False)).all(), ("y", sw, sh, dw, dh)
        area += area2x
        if area2x:
            continue
        img = big[:sh, :sw] if k % 2 else np.full((sh, sw, 3), 255 * (k % 4 == 0), np.uint8)
        want = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR)
        assert (_apply_plan_numpy(img, buf, dw, dh) == want).all(), (sw, sh, dw, dh)
    assert area >= 200


def test_bad_arguments_are_rejected_without_a_gpu():
    l = cabi.lib()
    assert l.scn_resize_plan_fill(0, 10, 4, 4, None) == -1
    assert l.scn_resize_plan_bytes(0, 5) == 0
    assert l.scn_hist16_u8c3(None, -1, 4, 4, None, None) == -1
    assert l.scn_hist16_u8c3(None, 0, 4, 4, None, None) == 0  # n == 0 is a no-op
    assert l.scn_box_blur_u8c3(None, 1, 4, 4, 0, None, None) == -1  # kernel_size < 1
    assert l.scn_nv12_to_rgb24(None, None, 8, 1, 7, 8, None, 24, None) == -1  # odd width


BLUR_REFUSALS = [  # (n, width, height, kernel_size, expected return code)
    (-1, 16, 16, 3, -1), (1, 16, 16, 0, -1), (1, 16, 16, 32, -1), (1, 0, 16, 3, -1), (1, 16, 0, 3, -1),
    (1, (1 << 29) + 1, 1, 3, -1), (1, 2**31 - 1, 1, 1, -1), (0, 2**31 - 1, 1, 1, -1),
    (1, 1, 65535 * 32 + 1, 3, -2), (2, 16, 2**31 - 1, 3, -2), (1, 1 << 29, 2**31 - 1, 31, -2),
]


def test_blur_refusals_launch_nothing_and_write_nothing():
    """scn_box_blur_u8c3 refuses before any launch: n < 0, kernel sizes 0 and 32, null pointer lists, a width past
    2^29 (row offsets are int arithmetic), and, with SCN_E_UNSUPPORTED, frames taller than 2,097,120 rows (the
    generic kernel's grid), INT_MAX included, whose rounding up to a strip would overflow int.  The pointers name
    host buffers: a refusal never dereferences them."""
    l = cabi.lib()
    src, dst = np.arange(64, dtype=np.uint8), np.full(64, 0x5A, np.uint8)
    before = l.scn_launch_count()
    for (n, w, h, k, rc) in BLUR_REFUSALS:
        ps, keep_s = cabi.ptr_array([src.ctypes.data] * max(n, 1))
        pd, keep_d = cabi.ptr_array([dst.ctypes.data] * max(n, 1))
        assert l.scn_box_blur_u8c3(ps, n, w, h, k, pd, None) == rc, (n, w, h, k)
        assert l.scn_box_blur_u8c3_strided(src.ctypes.data, 0, n, w, h, k, dst.ctypes.data, None) == rc, (n, w, h, k)
    for n in (1, 3):
        ps, keep_s = cabi.ptr_array([src.ctypes.data] * n)
        assert l.scn_box_blur_u8c3(None, n, 16, 16, 3, ps, None) == -1
        assert l.scn_box_blur_u8c3(ps, n, 16, 16, 3, None, None) == -1
        assert l.scn_box_blur_u8c3_strided(None, 48, n, 16, 16, 3, dst.ctypes.data, None) == -1
        assert l.scn_box_blur_u8c3_strided(src.ctypes.data, 48, n, 16, 16, 3, None, None) == -1
    assert l.scn_box_blur_u8c3(None, 0, 16, 16, 3, None, None) == 0  # n == 0 is a no-op
    assert l.scn_launch_count() == before
    assert (dst == 0x5A).all() and (src == np.arange(64)).all()


def test_nv12_stream_unit_division_by_multiply_shift_is_exact():
    """nv12_stream_kernel splits a unit index u (16 pixels x 2 rows) into row pair and column with
    (u * (floor(2^32 / upr) + 1)) >> 32, upr = width / 16 (nvs::launch, nvs::Params::upr_recip).  Exhaustive over every
    width the kernel takes up to 8192 and every unit index a frame up to 8192 rows tall reaches, padding lanes of the
    last step included.  The multiplier needs 33 bits at width 16: truncated to 32 it is 1 and every quotient is 0."""
    for upr in range(1, 8192 // 16 + 1):
        m = np.uint64((1 << 32) // upr + 1)
        v = np.arange(upr * (8192 // 2) + 32, dtype=np.uint64)
        q = (v * m) >> np.uint64(32)
        assert ((v - q * np.uint64(upr)) < np.uint64(upr)).all(), upr * 16


def test_no_silent_cpu_fallback():
    """On a box without CUDA the torch wrappers must raise, not compute on the CPU."""
    import torch
    from scanner_b200 import kernels
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(cabi.ScnError):
        kernels.histogram(torch.zeros((1, 4, 4, 3), dtype=torch.uint8))


def test_engine_library_exports_every_declared_symbol():
    import re as _re
    from scanner_b200 import engine as E
    src = open(os.path.join(ROOT, "include", "scn_engine.h")).read()
    names = sorted(set(_re.findall(r"SCN_ENGINE_API\s+[\w\s\*]+?\b(scn_\w+)\s*\(", src)))
    assert len(names) >= 30
    l = ctypes.CDLL(E.ENGINE_PATH)
    for n in names:
        assert hasattr(l, n), f"libscn_engine.so does not export {n}"
    assert sorted(E.SIGNATURES) == names
    # the stdlib plugin loads and registers the three GPU ops without touching a GPU
    E.load_stdlib()
    ops = E.list_ops()
    for op in ("Histogram", "Resize", "Blur"):
        assert op in ops and E.lib().scn_kernel_registered(op.encode(), 1) == 1
