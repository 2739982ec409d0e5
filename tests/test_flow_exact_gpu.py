"""Every Farneback kernel of flow.cu against its kernel-ordered restatement (oracle/farneback_k.c), bit for bit.

flow.cu is built with -fmad=false and writes every fused multiply-add out; farneback_k.c evaluates the same
expressions in the same order, so the flow fields must be equal: finite values `==`, NaN where the oracle has NaN.
tests/test_flow_exact_cpu.py holds farneback_k to the cv2-pinned specification (orc_farneback_u8).

The ladder adds kernels rung by rung, so the first failing rung names the culprit; the path switches (read once per
process, so run in subprocesses) select the other kernel families; the geometries sit at the tile edges of each
kernel (Gaussian and expansion 64 x 32, update_matrices 32 x 8, float box 88 x 32, double box 64 x 16) and where the
pyramid's level count or lrint's rounding changes."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from oracle import farneback_k as K
from oracle import synth
from scanner_b200 import engine as E
from scanner_b200 import kernels

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _eq(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    if not same.all():
        d = np.abs(np.nan_to_num(got) - np.nan_to_num(want))
        ys, xs = np.nonzero(~same.all(-1))
        raise AssertionError(f"{what}: {(~same.all(-1)).sum()} of {got.shape[0] * got.shape[1]} pixels differ, "
                             f"max |d| {d.max():.3e}, first at (y, x) = ({ys[0]}, {xs[0]})")


def _gpu(f0, f1, **a):
    return kernels.optical_flow(dev(f0[None]), dev(f1[None]), **a)[0].cpu().numpy()


def _exact(f0, f1, what, **a):
    _eq(_gpu(f0, f1, **a), K.flow(f0, f1, **a), what)


# ---- the ladder ----------------------------------------------------------------------------------------------------
LADDER = [
    ("1-levels0-iters1", dict(num_levels=0, num_iters=1)),        # gray, Gaussian r 1, expansion, UM at 0, box + solve
    ("2-levels0-iters2", dict(num_levels=0, num_iters=2)),        # update_matrices on a nonzero flow, both branches
    ("3-levels1-iters2", dict(num_levels=1, num_iters=2)),        # both resize_f32 instances, a computed Gaussian
    ("4-defaults", dict()),                                       # radii 4 and 9
    ("5-levels4", dict(num_levels=4)),                            # radius 19: gauss_fused_kernel<0>
    ("6-poly3", dict(poly_n=3, poly_sigma=0.9)),                  # poly_fused_kernel<0>
    ("6-poly7", dict(poly_n=7, poly_sigma=1.5)),
    ("7-win2", dict(win_size=2)),                                 # the two-pass double box
    ("7-win9", dict(win_size=9)),
    ("7-win16", dict(win_size=16)),
    ("7-win14", dict(win_size=14)),                               # float box at an even window (scale 1 / 196)
]


@pytest.mark.parametrize("name,over", LADDER, ids=[n for n, _ in LADDER])
def test_ladder(name, over):
    # odd sizes: at 270 x 480 level 1 is exactly half, the resize's coordinates are exact in float as well, and a
    # resize_f32_kernel that dropped its double coordinate chain would pass rung 3
    h, w = (541, 961) if over.get("num_levels") == 4 else (271, 481)
    f0, f1 = synth.flow_pair(3000 + h, h, w, "shift")
    _exact(f0, f1, name, **over)


# ---- every path, at the defaults and one point off them ------------------------------------------------------------
PATH_CASES = [(270, 480, {}), (97, 131, dict(num_levels=2, num_iters=2, poly_n=7, poly_sigma=1.5, win_size=14))]
PATHS = [("fused-f32", {}), ("fused-f64_slide", dict(SCN_FLOW_BOX="f64")),
         ("unfused", dict(SCN_FLOW_UNFUSED="1")), ("no-pyramid-cache", dict(SCN_FLOW_NO_PYRAMID_CACHE="1"))]


@pytest.mark.parametrize("name,env", PATHS, ids=[n for n, _ in PATHS])
def test_every_path(name, env):
    code = (
        "import sys, numpy as np, torch; sys.path.insert(0, '.');"
        "from scanner_b200 import kernels; from oracle import synth;"
        f"outs = []; cases = {PATH_CASES!r}"
        "\nfor (h, w, kw) in cases:"
        "\n    a, b = synth.flow_pair(3100 + h, h, w, 'shift')"
        "\n    d = torch.from_numpy(np.stack([a, b, np.roll(b, (1, 2), (0, 1))])).cuda()"
        "\n    outs.append(kernels.optical_flow(d[:2], d[1:], **kw).cpu().numpy())"
        "\nnp.savez(sys.argv[1], *outs)")
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "o.npz")
        base = {k: v for k, v in os.environ.items() if k not in ("SCN_FLOW_BOX", "SCN_FLOW_UNFUSED",
                                                                   "SCN_FLOW_NO_PYRAMID_CACHE")}
        subprocess.check_call([sys.executable, "-c", code, out], cwd=ROOT, env=dict(base, **env))
        got = np.load(out)
        got = [got[f"arr_{i}"] for i in range(len(PATH_CASES))]
    box = lambda ws: K.box_for(ws, unfused="SCN_FLOW_UNFUSED" in env, box_f64="SCN_FLOW_BOX" in env)  # noqa: E731
    for (h, w, kw), g in zip(PATH_CASES, got):
        a, b = synth.flow_pair(3100 + h, h, w, "shift")
        frames = [a, b, np.roll(b, (1, 2), (0, 1))]
        for i in range(2):
            _eq(g[i], K.flow(frames[i], frames[i + 1], box=box(kw.get("win_size", 15)), **kw), (name, h, w, kw, i))


# ---- geometry ------------------------------------------------------------------------------------------------------
GEOM = [(1, 1), (2, 2), (1, 97), (97, 1), (3, 200),
        (32, 64), (33, 65), (31, 63),      # Gaussian / expansion tile
        (8, 32), (9, 33), (16, 96),        # update_matrices tile
        (32, 88), (33, 89), (64, 176),     # float box tile
        (16, 64), (17, 65),                # double box tile
        (63, 63), (64, 64), (65, 65),      # 0 / 1 coarser level at pyr_scale 0.5
        (129, 129), (131, 257)]            # lrint(64.5) = 64, lrint(128.5) = 128


@pytest.mark.parametrize("h,w", GEOM, ids=[f"{h}x{w}" for h, w in GEOM])
def test_geometry(h, w):
    f0, f1 = synth.flow_pair(3200 + h + w, h, w, "shift")
    _exact(f0, f1, (h, w))
    if h >= 16 and w >= 16:
        _exact(f0, f1, (h, w, "win9"), win_size=9)


@pytest.mark.parametrize("over", [{}, dict(num_levels=4)], ids=["defaults", "levels4"])
def test_1080p(over):
    """At num_levels=4 a pixel near (0, 566) sits on UpdateMatrices' range test by 1.6e-8 px in orc_farneback_u8, which
    needs an 8 x 15 exemption against cv2; against the kernel-ordered oracle there is none."""
    f0, f1 = synth.flow_pair(942 if over else 941, 1080, 1920, "shift")
    _exact(f0, f1, ("1080p", over), **over)


# ---- content -------------------------------------------------------------------------------------------------------
def _content(kind, h=96, w=128):
    rng = np.random.default_rng(5)
    if kind == "constant":
        return np.full((h, w, 3), 117, np.uint8), np.full((h, w, 3), 118, np.uint8)
    if kind == "saturated":
        a, b = synth.flow_pair(3300, h, w, "shift")
        return np.maximum(a, 128).astype(np.uint8), np.maximum(b, 128).astype(np.uint8)
    if kind == "checker":
        yy, xx = np.mgrid[0:h, 0:w]
        a = np.where(((yy // 4) + (xx // 4)) % 2 == 0, 255, 0).astype(np.uint8)
        a = np.repeat(a[..., None], 3, -1)
        return a, np.roll(a, (1, 2), (0, 1))
    if kind == "noise":
        a = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        return a, rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["constant", "saturated", "checker", "noise"])
def test_content(kind):
    f0, f1 = _content(kind)
    _exact(f0, f1, kind)
    _exact(f0, f1, (kind, "win5"), win_size=5)


def test_large_motion_takes_the_out_of_range_branch_for_a_band():
    """A 9 px pan: along the right edge a band of pixels has x + dx past the last column in the final field, so
    UpdateMatrices takes the branch that drops the warped R1 there (the final field is what its last call saw, one
    box + solve later)."""
    h, w = 120, 160
    base = synth.flow_pair(3400, h, w + 16, "shift")[0]
    f0, f1 = np.ascontiguousarray(base[:, 9:9 + w]), np.ascontiguousarray(base[:, :w])
    want = K.flow(f0, f1)
    _eq(_gpu(f0, f1), want, "pan 9 px")
    xx = np.arange(w)[None, :] + want[..., 0]
    out = (np.floor(xx) >= w - 1) | (np.floor(xx) < 0)
    assert out.sum() >= h, out.sum()              # a band as tall as the frame


# ---- batches and chaining ------------------------------------------------------------------------------------------
def test_mixed_batch_and_identity():
    frames = np.stack([synth.flow_pair(700, 96, 128, "shift")[i] for i in (0, 1, 0)])
    out = kernels.optical_flow(dev(frames[:2]), dev(frames[1:])).cpu().numpy()
    for i in range(2):
        _eq(out[i], K.flow(frames[i], frames[i + 1]), ("batch", i))
    _eq(_gpu(frames[0], frames[0]), K.flow(frames[0], frames[0]), "identical frames")


@pytest.mark.parametrize("step", [None, 2, 1], ids=["one-call", "2-per-call", "1-per-call"])
def test_sequence_pairs(step):
    n, h, w = 5, 96, 128
    a, b = synth.flow_pair(3500, h, w, "shift")
    rng = np.random.default_rng(3)
    frames = np.stack([a, b] + [np.roll(a, (i, 2 * i), (0, 1)) + rng.integers(0, 2, a.shape, dtype=np.uint8)
                                for i in range(1, n - 1)])
    got = kernels.optical_flow_sequence(dev(frames), pairs_per_call=step).cpu().numpy()
    for i in range(n - 1):
        _eq(got[i], K.flow(frames[i], frames[i + 1]), (step, i))


# ---- the OpticalFlow op --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("force_rgb", [False, True], ids=["nv12", "rgb24"])
def test_optical_flow_op_rows(force_rgb, monkeypatch):
    """Every row of the OpticalFlow op (stencil [0, 1], last row clamped) equals the oracle on the frames the decoder
    shows, whether the op receives NV12 elements or dense RGB24 ones."""
    if force_rgb:
        monkeypatch.setenv("SCN_DECODE_RGB", "1")
    else:
        monkeypatch.delenv("SCN_DECODE_RGB", raising=False)
    n, h, w = 6, 96, 128
    base = synth.flow_pair(3600, h + n, w + n, "shift")[0]
    gray = (base[..., 0].astype(np.int32) * 3 + base[..., 1] * 5 + base[..., 2] * 2) // 10
    y = np.stack([gray[i // 2:i // 2 + h, i:i + w] for i in range(n)]).astype(np.uint8)
    u = np.stack([y[i, ::2, ::2] // 4 + 96 for i in range(n)]).astype(np.uint8)
    v = np.stack([160 - y[i, 1::2, 1::2] // 4 for i in range(n)]).astype(np.uint8)
    data = E.h264_synth(np.concatenate([y.reshape(n, -1), u.reshape(n, -1), v.reshape(n, -1)], axis=1), w, h, gop=4)
    E.load_stdlib()
    eng = E.Engine(gpus=[0], instances_per_gpu=2)
    try:
        sid = eng.add_h264(data)
        g = E.Graph()
        src = g.add_source(True)
        fl = g.add_op("OpticalFlow", [(src, "frame")], device=1)
        sink = g.add_sink((fl, "flow"))
        j = E.Job()
        j.bind_source(src, sid)
        eng.run(g, [j], 2, 2)
        rows = [j.output_row(sink, i) for i in range(j.output_rows(sink))]
        shown = eng.decode_to_device(eng.add_h264(data), range(n), 0).cpu().numpy()
    finally:
        eng.close()
    assert len(rows) == n
    for i in range(n):
        _eq(rows[i], K.flow(shown[i], shown[min(i + 1, n - 1)]), ("op row", force_rgb, i))
