"""TV-L1 on the CPU: the oracle's pieces against live cv2, the oracle against known motion, and the C ABI's
refusals (which happen before any CUDA call)."""
import ctypes
import math

import cv2
import numpy as np
import pytest

from oracle import synth
from oracle import tvl1 as T
from scanner_b200 import cabi


def test_levels_follow_the_rounding_rule_and_stop_below_16():
    assert T.levels(480, 270) == [(480, 270), (384, 216), (307, 173), (246, 138), (197, 110)]
    assert T.levels(200, 24) == [(200, 24), (160, 19)]
    assert T.levels(2, 2, nscales=5) == [(2, 2)]
    assert T.levels(53, 37, nscales=10, scale_step=0.5) == [(53, 37), (27, 19)]


@pytest.mark.parametrize("step", [0.5, 0.6, 0.8, 0.9])
def test_pyramid_and_flow_resize_match_cv2(step):
    rng = np.random.default_rng(int(step * 10))
    for h, w in [(270, 480), (37, 53), (120, 160), (1080, 1920), (17, 16)]:
        levels = T.levels(w, h, nscales=6, scale_step=step)
        for (sw, sh), (dw, dh) in zip(levels, levels[1:]):
            src = (rng.random((sh, sw)) * 255).astype(np.float32)
            for a, b in (((sw, sh), (dw, dh)), ((dw, dh), (sw, sh))):  # pyramid down, flow upsampling up
                s = src if a == (sw, sh) else cv2.resize(src, (dw, dh))
                want = cv2.resize(s, b, interpolation=cv2.INTER_LINEAR)
                got = T.resize(s, *b)
                assert np.abs(got - want).max() <= 1e-4 * max(np.abs(want).max(), 1.0), (a, b)


@pytest.mark.parametrize("k", [3, 5])
def test_median_matches_cv2_exactly(k):
    rng = np.random.default_rng(k)
    for h, w in [(2, 2), (3, 7), (37, 53), (120, 160)]:
        img = (rng.standard_normal((h, w)) * 3).astype(np.float32)
        img[rng.random((h, w)) < 0.2] = 0.5  # ties
        assert np.array_equal(T.median(img, k), cv2.medianBlur(img, k))


def test_gray_matches_cv2_exactly():
    frame = synth.rand_frame(3, 64, 96)
    assert np.array_equal(T.gray_u8(frame), cv2.cvtColor(frame, cv2.COLOR_RGB2GRAY))


def test_identical_frames_give_exact_zero():
    f = T.flow_pair_known(4, 60, 90, "affine")[0]
    flow, it = T.flow(f, f, return_iterations=True)
    assert (flow == 0).all()
    assert set(it[it > 0].tolist()) == {1}
    assert (T.flow(f, f, epsilon=-1, iterations=20) == 0).all()


def test_known_pairs_relation_holds():
    """frame1(x + u(x)) = frame0(x): an integer shift of the same texture is exact up to the u8 rounding."""
    yy, xx = np.mgrid[0:40, 0:60].astype(np.float64)
    t0, t1 = T.tex_gray(5, xx, yy), T.tex_gray(5, xx - 2, yy + 1)
    assert np.allclose(t1[:-1, 2:], t0[1:, :-2])
    f0, f1, flow = T.flow_pair_known(5, 40, 60, "shift")
    assert flow.shape == (40, 60, 2) and (flow[..., 0] == 1.5).all() and (flow[..., 1] == -0.75).all()
    _, _, fa = T.flow_pair_known(5, 270, 480, "affine")
    assert np.abs(fa).max() <= 8
    _, _, fs = T.flow_pair_known(5, 120, 160, "square")
    assert (fs[0, 0] == 0).all() and (fs[60, 80] != 0).all()


def interior(a, b=8):
    return a[b:-b, b:-b]


def test_oracle_recovers_known_motion():
    """The oracle's own CPU run at the defaults (recorded when this test was written):
         120 x 160  shift   interior median (1.4947, -0.7418)  |  affine mean EPE 0.069 px  |  square 0.077 px
         270 x 480  shift   interior median (1.4962, -0.7447)  |  affine mean EPE 0.036 px  |  square 0.028 px
    ("square": outside a 3 px band around the square's edges).  Bounds: median within 0.02 px of (1.5, -0.75),
    mean EPE <= 0.1 px.  For information, the oracle's Farneback (the reference's arguments) on the same gray
    pairs: shift median (1.227, -0.593) and (1.254, -0.599); affine mean EPE 0.54 and 1.08 px; square 0.22 and
    0.067 px (120 x 160 and 270 x 480; not asserted)."""
    for h, w in [(120, 160), (270, 480)]:
        f0, f1, tf = T.flow_pair_known(3, h, w, "shift")
        med = np.median(interior(T.flow(f0, f1)).reshape(-1, 2), axis=0)
        assert abs(med[0] - 1.5) <= 0.02 and abs(med[1] + 0.75) <= 0.02, (h, w, med)
        f0, f1, tf = T.flow_pair_known(3, h, w, "affine")
        epe = np.sqrt(((T.flow(f0, f1) - tf) ** 2).sum(-1))
        assert interior(epe).mean() <= 0.1, (h, w, interior(epe).mean())
        f0, f1, tf = T.flow_pair_known(3, h, w, "square")
        epe = np.sqrt(((T.flow(f0, f1) - tf) ** 2).sum(-1))
        m = tf[..., 0] != 0
        ys, xs = np.nonzero(m)
        band = np.zeros_like(m)
        band[max(ys.min() - 3, 0):ys.max() + 4, max(xs.min() - 3, 0):xs.max() + 4] = True
        band[ys.min() + 4:ys.max() - 3, xs.min() + 4:xs.max() - 3] = False
        keep = interior(~band)
        assert interior(epe)[keep].mean() <= 0.1, (h, w, interior(epe)[keep].mean())


DEFAULTS = dict(tau=0.25, lambda_=0.15, theta=0.3, nscales=5, warps=5, epsilon=0.01, iterations=300,
                scale_step=0.8, median_filtering=5)
BAD = [dict(tau=0.0), dict(tau=-1.0), dict(lambda_=0.0), dict(theta=-0.3), dict(nscales=0), dict(nscales=11),
       dict(warps=0), dict(warps=21), dict(iterations=0), dict(iterations=10001), dict(scale_step=0.0),
       dict(scale_step=1.0), dict(scale_step=1.5), dict(median_filtering=0), dict(median_filtering=2),
       dict(median_filtering=7), dict(tau=math.nan), dict(lambda_=math.inf), dict(theta=math.nan),
       dict(epsilon=math.nan), dict(epsilon=-math.inf), dict(scale_step=math.nan), dict(width=1), dict(height=1),
       dict(n=-1), dict(workspace_bytes=-1), dict(workspace=0)]


@pytest.mark.parametrize("bad", BAD, ids=lambda b: ",".join(f"{k}={v}" for k, v in b.items()))
def test_refusals_return_badarg_and_launch_nothing(bad):
    L = cabi.lib()
    a = dict(DEFAULTS, width=64, height=48, n=2)
    a.update({k: v for k, v in bad.items() if k not in ("workspace_bytes", "workspace")})
    need = L.scn_tvl1_workspace_bytes(64, 48, 2)
    wsb = need - 1 if bad.get("workspace_bytes") == -1 else need
    ws = 0 if bad.get("workspace") == 0 else 1 << 20  # never dereferenced: the call refuses before any launch
    fake, keep = cabi.ptr_array([1 << 21, 1 << 22])
    before = L.scn_launch_count()
    f = ctypes.c_float
    rc = L.scn_tvl1_u8(fake, fake, a["n"], a["width"], a["height"], fake, f(a["tau"]), f(a["lambda_"]),
                       f(a["theta"]), a["nscales"], a["warps"], f(a["epsilon"]), a["iterations"], f(a["scale_step"]),
                       a["median_filtering"], None, ws, wsb, None)
    assert rc == -1  # SCN_E_BADARG
    assert L.scn_launch_count() == before


def test_workspace_size_covers_chunks_of_64_pairs():
    L = cabi.lib()
    one = L.scn_tvl1_workspace_bytes(1920, 1080, 1)
    assert L.scn_tvl1_workspace_bytes(1920, 1080, 64) == L.scn_tvl1_workspace_bytes(1920, 1080, 500)
    assert L.scn_tvl1_workspace_bytes(1920, 1080, 64) > 60 * one
    assert L.scn_tvl1_workspace_bytes(1, 1080, 1) == 0
