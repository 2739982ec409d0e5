"""Resize's interpolation modes without a GPU: the C restatement of cv2's INTER_NEAREST and INTER_AREA
(oracle/resize_interp.c) against live cv2.resize and against recorded cv2 4.13 hashes, the product's host tables, the
name table and the refusals of the C ABI."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

import oracle
from oracle import resize_interp as R
from oracle import synth
from scanner_b200 import cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("INTER_NEAREST", "INTER_AREA")
ORACLES = {"INTER_NEAREST": R.resize_nearest, "INTER_AREA": R.resize_area}
SIDES = synth.RESIZE_SIDES + (2160, 3840)


def _cv2_resize(cv2, img, dw, dh, mode):
    out = cv2.resize(img, (dw, dh), interpolation=getattr(cv2, mode))
    return out if out.ndim == 3 else out[..., None]


def sweep_geometries():
    """~2000 seeded geometries with sides from synth.RESIZE_SIDES plus 2160 and 3840, and the fixed cases: 1080p and
    4K to 224, integer factors 1-8 on each axis, upscales and geometries that grow one axis and shrink the other."""
    fixed = [(1920, 1080, 224, 224), (3840, 2160, 224, 224), (1080, 1920, 224, 224), (2160, 3840, 224, 224),
             (224, 224, 1920, 1080), (64, 48, 32, 96), (1920, 1080, 224, 2000), (17, 3, 5, 9), (3840, 2160, 1, 1)]
    fixed += [(8 * 7 * 5 * 3, 8 * 7 * 5 * 3 // 2, 8 * 7 * 5 * 3 // kx, 8 * 7 * 5 * 3 // 2 // ky)
              for kx in range(1, 9) for ky in range(1, 9) if (8 * 7 * 5 * 3 // 2) % ky == 0]
    return fixed + synth.resize_geometries(31, 2000, SIDES)


@pytest.mark.parametrize("mode", MODES)
def test_oracle_equals_live_cv2_on_every_small_geometry(mode):
    """Every (sw, dw) x (sh, dh) with sides 1-16, on noise."""
    cv2 = pytest.importorskip("cv2")
    img = synth.rand_frame(41, 16, 16)
    for sw in range(1, 17):
        for sh in range(1, 17):
            src = np.ascontiguousarray(img[:sh, :sw])
            for dw in range(1, 17):
                for dh in range(1, 17):
                    assert (ORACLES[mode](src, dw, dh) == _cv2_resize(cv2, src, dw, dh, mode)).all(), (sw, sh, dw, dh)


@pytest.mark.parametrize("mode", MODES)
def test_oracle_equals_live_cv2_on_a_seeded_sweep(mode):
    """The sweep on noise, constant 0 and 255 and gradients; the regimes of INTER_AREA are all reached."""
    cv2 = pytest.importorskip("cv2")
    big = synth.rand_frame(43, 3840, 3840)
    grad = R.content("gradient", 0, 3840, 3840)
    regimes = {}
    for k, (sw, sh, dw, dh) in enumerate(sweep_geometries()):
        if k % 4 == 0:
            img = np.ascontiguousarray(big[:sh, :sw])
        elif k % 4 == 1:
            img = np.ascontiguousarray(grad[:sh, :sw])
        else:
            img = np.full((sh, sw, 3), 255 * (k % 4 == 2), np.uint8)
        assert (ORACLES[mode](img, dw, dh) == _cv2_resize(cv2, img, dw, dh, mode)).all(), (sw, sh, dw, dh)
        r = R.area_regime(sw, sh, dw, dh)
        regimes[r] = regimes.get(r, 0) + 1
    assert min(regimes.get(r, 0) for r in ("up", "int2x2", "int", "float")) >= 50, regimes


@pytest.mark.parametrize("kx,ky", [(2, 2), (2, 1), (1, 2), (4, 2), (2, 4), (4, 4), (6, 4), (8, 8)])
def test_half_cells_round_half_up_at_2x2_only(kx, ky):
    """Content whose every box averages to an exact .5: the 2 x 2 box rounds half up, every other integer factor
    half to even, as cv2 does."""
    cv2 = pytest.importorskip("cv2")
    w, h = kx * 48, ky * 30
    img = R.content("half", kx * 10 + ky, h, w, (kx, ky))
    got = R.resize_area(img, w // kx, h // ky)
    assert (got == _cv2_resize(cv2, img, w // kx, h // ky, "INTER_AREA")).all()
    s = img.astype(np.int64).reshape(h // ky, ky, w // kx, kx, 3).sum(axis=(1, 3))
    assert ((2 * s) % (kx * ky) == 0).all() and ((2 * s // (kx * ky)) % 2 == 1).all()  # every cell is m + .5
    half_up = (s + kx * ky // 2) // (kx * ky)
    half_even = np.rint(s / (kx * ky)).astype(np.int64)
    assert (half_up != half_even).any()
    assert (got == (half_up if (kx, ky) == (2, 2) else half_even)).all()


def _golden():
    with open(os.path.join(ROOT, "tests", "golden", "resize_interp_cv2.json")) as f:
        return json.load(f)


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.uint8).tobytes()).hexdigest()


def _golden_cases():
    for i, (sw, sh, dw, dh, kind) in enumerate(R.GOLDEN_CASES):
        yield f"{sw}x{sh}->{dw}x{dh} {kind}", R.content(kind, 1000 + i, sh, sw, R.golden_cell(sw, sh, dw, dh)), dw, dh


@pytest.mark.parametrize("mode", MODES)
def test_oracle_equals_recorded_cv2_hashes(mode):
    rec = _golden()["sha256"]
    n = 0
    for key, img, dw, dh in _golden_cases():
        assert _sha(ORACLES[mode](img, dw, dh)) == rec[f"{mode} {key}"], key
        n += 1
    assert n == len(R.GOLDEN_CASES) and len(rec) == 2 * n


@pytest.mark.parametrize("mode", MODES)
def test_live_cv2_still_equals_the_recorded_hashes(mode):
    """A cv2 whose INTER_NEAREST or INTER_AREA has drifted from 4.13's shows up here, instead of being followed."""
    cv2 = pytest.importorskip("cv2")
    rec = _golden()["sha256"]
    for key, img, dw, dh in _golden_cases():
        assert _sha(_cv2_resize(cv2, img, dw, dh, mode)) == rec[f"{mode} {key}"], key


def _plan(mode, sw, sh, dw, dh):
    l = cabi.lib()
    n = l.scn_resize_interp_plan_bytes(mode, sw, sh, dw, dh)
    assert n > 0
    buf = np.zeros(n, np.uint8)
    assert l.scn_resize_interp_plan_fill(mode, sw, sh, dw, dh, buf.ctypes.data) == 0
    return buf


def _apply_linear_plan(img, plan, dw, dh):
    """A kPlanLinearTaps plan applied with numpy: INTER_LINEAR's 11-bit fixed point."""
    p = plan.view(np.int32)
    taps = p[8:].reshape(-1, 4)
    xt, yt = taps[:dw], taps[dw:dw + dh]
    s = img.astype(np.int32)
    hb = s[:, xt[:, 0], :] * xt[None, :, 2, None] + s[:, xt[:, 1], :] * xt[None, :, 3, None]
    h0, h1 = hb[yt[:, 0]], hb[yt[:, 1]]
    b0, b1 = yt[:, 2][:, None, None], yt[:, 3][:, None, None]
    return ((((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2).astype(np.uint8)


def test_area_upscale_plan_applied_with_numpy_equals_the_oracle():
    """INTER_AREA with a scale below 1 is INTER_LINEAR's arithmetic with the plan's area taps."""
    big = synth.rand_frame(47, 1080, 1920)
    n = 0
    for (sw, sh, dw, dh) in sweep_geometries():
        if R.area_regime(sw, sh, dw, dh) != "up" or sw > 1920 or sh > 1080 or dw * dh > 4_000_000:
            continue
        plan = _plan(3, sw, sh, dw, dh)
        hdr = plan.view(np.int32)[:8]
        assert list(hdr[1:7]) == [sw, sh, dw, dh, 0, 0], (sw, sh, dw, dh)  # kPlanLinearTaps
        img = np.ascontiguousarray(big[:sh, :sw])
        assert (_apply_linear_plan(img, plan, dw, dh) == R.resize_area(img, dw, dh)).all(), (sw, sh, dw, dh)
        n += 1
    assert n >= 200


def test_linear_plan_through_the_new_entry_is_scn_resize_plan_fill_byte_for_byte():
    l = cabi.lib()
    for (sw, sh, dw, dh) in sweep_geometries()[:300]:
        old = np.zeros(l.scn_resize_plan_bytes(dw, dh), np.uint8)
        assert l.scn_resize_plan_fill(sw, sh, dw, dh, old.ctypes.data) == 0
        assert (_plan(1, sw, sh, dw, dh) == old).all(), (sw, sh, dw, dh)


def test_nearest_and_area_plans_hold_cv2s_tables():
    """The NEAREST plan's indices, and the AREA plan's tables applied in the oracle's order with numpy."""
    for (sw, sh, dw, dh) in [(1920, 1080, 224, 224), (97, 61, 40, 25), (7, 5, 16, 3), (3840, 2160, 1, 1)]:
        p = _plan(0, sw, sh, dw, dh).view(np.int32)
        assert list(p[1:7]) == [sw, sh, dw, dh, 0, 1]
        fx, fy = 1.0 / (dw / sw), 1.0 / (dh / sh)
        assert list(p[8:8 + dw]) == [min(int(np.floor(x * fx)), sw - 1) for x in range(dw)]
        assert list(p[8 + dw:8 + dw + dh]) == [min(int(np.floor(y * fy)), sh - 1) for y in range(dh)]
    img = synth.rand_frame(53, 61, 97)
    for (sw, sh, dw, dh) in [(97, 61, 40, 25), (97, 61, 13, 61), (96, 60, 24, 20), (97, 61, 97, 61)]:
        src = np.ascontiguousarray(img[:sh, :sw])
        b = _plan(3, sw, sh, dw, dh)
        i32, f32 = b.view(np.int32), b.view(np.float32)
        assert list(i32[1:7]) == [sw, sh, dw, dh, 0, 2]
        xo, yo = i32[8:9 + dw], i32[9 + dw:10 + dw + dh]
        at = (32 + 4 * (dw + 1) + 4 * (dh + 1) + 7) // 8 * 2  # int32 index of the column table
        xs, xa = i32[at:at + 2 * xo[-1]:2], f32[at + 1:at + 2 * xo[-1]:2]
        ys, ya = i32[at + 2 * xo[-1]::2], f32[at + 2 * xo[-1] + 1::2]
        assert len(ys) == yo[-1]
        S = src.astype(np.float32)
        out = np.zeros((dh, dw, 3), np.uint8)
        for y in range(dh):
            acc = None
            for j in range(yo[y], yo[y + 1]):
                buf = np.zeros((dw, 3), np.float32)
                for x in range(dw):
                    for e in range(xo[x], xo[x + 1]):
                        buf[x] = buf[x] + S[ys[j], xs[e]] * xa[e]
                acc = ya[j] * buf if acc is None else acc + ya[j] * buf
            out[y] = np.clip(np.rint(acc), 0, 255)
        if R.area_regime(sw, sh, dw, dh) == "float":
            assert (out == R.resize_area(src, dw, dh)).all(), (sw, sh, dw, dh)
        else:  # integer factors: the table lists each box's pixels
            assert all(xo[x + 1] - xo[x] == sw // dw for x in range(dw)), (sw, sh, dw, dh)


def test_interp_code_maps_every_cv2_name():
    l = cabi.lib()
    want = {"INTER_NEAREST": 0, "INTER_LINEAR": 1, "INTER_AREA": 3, "INTER_CUBIC": -2, "INTER_LANCZOS4": -2,
            "INTER_LINEAR_EXACT": -2, "INTER_NEAREST_EXACT": -2}
    for name, code in want.items():
        assert l.scn_resize_interp_code(name.encode()) == code, name
    assert l.scn_resize_interp_code(b"") == 1
    for bad in (b"bogus", b"inter_area", b"INTER_AREA ", b"INTER_MAX", b"INTER_BITS", b"WARP_FILL_OUTLIERS"):
        assert l.scn_resize_interp_code(bad) == -1, bad
    assert l.scn_resize_interp_code(None) == -1
    assert l.scn_resize_interp_supported() == b"INTER_NEAREST, INTER_LINEAR, INTER_AREA"
    cv2 = pytest.importorskip("cv2")
    for name in dir(cv2):
        if name.startswith("INTER_"):
            code = l.scn_resize_interp_code(name.encode())
            assert code == want.get(name, -1), name
            if code >= 0:
                assert code == getattr(cv2, name), name


def test_binding_names_the_supported_modes():
    from scanner_b200 import kernels
    assert kernels.resize_interp_code("") == 1 and kernels.resize_interp_code("INTER_AREA") == 3
    for bad in ("INTER_CUBIC", "bogus"):
        with pytest.raises(cabi.ScnError, match="INTER_NEAREST, INTER_LINEAR, INTER_AREA"):
            kernels.resize_interp_code(bad)


def test_bad_arguments_are_refused_without_a_gpu():
    """Before any launch: unsupported (-2) and unknown (-1) modes, bad sizes, a destination over INT_MAX pixels,
    n < 0, null pointer lists, odd NV12 sides or a short pitch, and a missing plan (-3) where one is needed.  The
    pointers name host buffers, so nothing may be dereferenced or launched."""
    l = cabi.lib()
    src, dst = np.arange(64, dtype=np.uint8), np.full(64, 0x5A, np.uint8)
    ps, k1 = cabi.ptr_array([src.ctypes.data] * 2)
    pd, k2 = cabi.ptr_array([dst.ctypes.data] * 2)
    plan = np.zeros(4096, np.uint8)
    before = l.scn_launch_count()
    for mode, rc in ((2, -2), (4, -2), (5, -2), (6, -2), (7, -1), (-1, -1), (8, -1)):
        assert l.scn_resize_interp_plan_bytes(mode, 8, 8, 4, 4) == 0
        assert l.scn_resize_interp_plan_fill(mode, 8, 8, 4, 4, plan.ctypes.data) == rc
        assert l.scn_resize_interp_u8c3(mode, ps, 2, 8, 8, pd, 4, 4, plan.ctypes.data, None) == rc
        assert l.scn_resize_interp_nv12(mode, ps, ps, 8, 2, 8, 8, pd, 4, 4, plan.ctypes.data, None) == rc
    for mode in (0, 1, 3):
        for (sw, sh, dw, dh) in ((0, 8, 4, 4), (8, 0, 4, 4), (8, 8, 0, 4), (8, 8, 4, -1), (8, 8, 65536, 32768)):
            assert l.scn_resize_interp_plan_bytes(mode, sw, sh, dw, dh) == 0
            assert l.scn_resize_interp_plan_fill(mode, sw, sh, dw, dh, plan.ctypes.data) == -1
            assert l.scn_resize_interp_u8c3(mode, ps, 1, sw, sh, pd, dw, dh, plan.ctypes.data, None) == -1
            assert l.scn_resize_interp_nv12(mode, ps, ps, 8, 1, sw, sh, pd, dw, dh, plan.ctypes.data, None) == -1
        assert l.scn_resize_interp_plan_fill(mode, 8, 8, 4, 4, None) == -1
        assert l.scn_resize_interp_u8c3(mode, ps, -1, 8, 8, pd, 3, 3, plan.ctypes.data, None) == -1
        assert l.scn_resize_interp_u8c3(mode, None, 1, 8, 8, pd, 3, 3, plan.ctypes.data, None) == -1
        assert l.scn_resize_interp_u8c3(mode, ps, 1, 8, 8, None, 3, 3, plan.ctypes.data, None) == -1
        assert l.scn_resize_interp_u8c3(mode, None, 0, 8, 8, None, 3, 3, None, None) == 0  # n == 0 is a no-op
        assert l.scn_resize_interp_u8c3(mode, ps, 1, 8, 8, pd, 3, 3, None, None) == -3
        assert l.scn_resize_interp_nv12(mode, ps, ps, 8, 1, 7, 8, pd, 3, 3, plan.ctypes.data, None) == -1  # odd
        assert l.scn_resize_interp_nv12(mode, ps, ps, 8, 1, 8, 7, pd, 3, 3, plan.ctypes.data, None) == -1
        assert l.scn_resize_interp_nv12(mode, ps, ps, 6, 1, 8, 8, pd, 3, 3, plan.ctypes.data, None) == -1  # pitch
        assert l.scn_resize_interp_nv12(mode, ps, None, 8, 1, 8, 8, pd, 3, 3, plan.ctypes.data, None) == -1
        assert l.scn_resize_interp_nv12(mode, ps, ps, 8, 1, 8, 8, pd, 3, 3, None, None) == -3
    assert l.scn_launch_count() == before
    assert (dst == 0x5A).all()
