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


# ---- the stop error in the GPU kernel's order (oracle.tvl1.flow(error_sum="tiles")) ----------------------------
def lane_tree(v):
    """lane 0 of __shfl_down_sync at offsets 16, 8, 4, 2, 1, for each row of 32 lanes"""
    v = v.copy()
    o = 16
    while o:
        v[..., :o] = v[..., :o] + v[..., o:2 * o]
        o >>= 1
    return v[..., 0]


def tile_sum_numpy(terms, warp_order=range(8)):
    """tvl1_iterate_kernel's error sum: 1024-pixel tiles, thread x of 256 adding pixels 1024 t + 256 j + x in
    float, the lane tree per warp, the 8 warp sums in order; then per pair, thread x adding tiles x, x + 256, ...
    in double, and the same tree and warp order."""
    terms = np.asarray(terms, np.float32).ravel()
    tiles = -(-terms.size // 1024)
    pad = np.zeros(tiles * 1024, np.float32)
    pad[:terms.size] = terms
    e = np.zeros((tiles, 256), np.float32)
    for j in range(4):
        e = e + pad.reshape(tiles, 4, 256)[:, j]
    warp = lane_tree(e.reshape(tiles, 8, 32))
    s = np.zeros(tiles, np.float32)
    for k in warp_order:
        s = s + warp[:, k]
    rounds = np.zeros(-(-tiles // 256) * 256)
    rounds[:tiles] = s
    acc = np.zeros(256)
    for r in rounds.reshape(-1, 256):
        acc = acc + r
    warp = lane_tree(acc.reshape(8, 32))
    t = 0.0
    for k in warp_order:
        t = t + warp[k]
    return t


@pytest.mark.parametrize("n", [1, 31, 255, 256, 257, 1023, 1024, 1025, 2047, 2048, 2049, 5000,
                               256 * 1024 - 1, 256 * 1024, 256 * 1024 + 1, 300_001])
def test_tile_sum_follows_the_kernel_tree(n):
    """orc_tvl1_tile_sum equals the numpy emulation of the kernel's tree bit for bit, at the tile edges (1024
    pixels) and where a thread's double sum takes a second round of tiles (256 tiles)."""
    rng = np.random.default_rng(n)
    # squared steps over a wide range of scales, so that the order of the additions shows in the last bits
    terms = (rng.standard_normal(n) * np.exp(rng.uniform(-8, 4, n))).astype(np.float32) ** 2
    got = T.tile_sum(terms)
    assert got == tile_sum_numpy(terms)
    if n >= 2048:  # the float tile sums round: the tree is not the exact sum
        assert got != math.fsum(terms.astype(np.float64))


def test_tile_error_changes_nothing_at_fixed_iterations():
    """With epsilon <= 0 the error decides nothing: both error sums give the same flow, bit for bit."""
    f0, f1, _ = T.flow_pair_known(8, 72, 96, "affine")
    kw = dict(epsilon=-1.0, iterations=15, nscales=3, warps=3)
    a, ia = T.flow(f0, f1, return_iterations=True, **kw)
    b, ib = T.flow(f0, f1, return_iterations=True, error_sum="tiles", **kw)
    assert np.array_equal(a, b) and np.array_equal(ia, ib)


# ---- the specification in float64, written from DESIGN.md section 11 alone ------------------------------------
def forward_grad(u):
    """forward differences, 0 at the last column (a) and the last row (b)"""
    a, b = np.zeros_like(u), np.zeros_like(u)
    a[:, :-1] = u[:, 1:] - u[:, :-1]
    b[:-1, :] = u[1:, :] - u[:-1, :]
    return a, b


def divergence(p1, p2):
    """div(p1, p2) = p1(x, y) - p1(x-1, y) + p2(x, y) - p2(x, y-1), terms outside the frame 0"""
    d = p1 + p2
    d[:, 1:] -= p1[:, :-1]
    d[1:, :] -= p2[:-1, :]
    return d


def centred_grad(img):
    """0.5 (I[x+1] - I[x-1]); 0.5 times the one-sided difference at the first and last column and row"""
    gx, gy = np.empty_like(img), np.empty_like(img)
    gx[:, 1:-1] = 0.5 * (img[:, 2:] - img[:, :-2])
    gx[:, 0], gx[:, -1] = 0.5 * (img[:, 1] - img[:, 0]), 0.5 * (img[:, -1] - img[:, -2])
    gy[1:-1] = 0.5 * (img[2:] - img[:-2])
    gy[0], gy[-1] = 0.5 * (img[1] - img[0]), 0.5 * (img[-1] - img[-2])
    return gx, gy


def catmull_rom(v0, v1, v2, v3, t):
    """Keys' cubic with a = -0.5, written as its four weights"""
    return (v0 * ((-0.5 * t + 1.0) * t - 0.5) * t + v1 * ((1.5 * t - 2.5) * t * t + 1.0) +
            v2 * ((-1.5 * t + 2.0) * t + 0.5) * t + v3 * ((0.5 * t - 0.5) * t * t))


def bicubic(img, px, py):
    """rows first, then columns; every tap clamped into the frame"""
    h, w = img.shape
    ix, iy = np.floor(px).astype(np.int64), np.floor(py).astype(np.int64)
    tx, ty = px - ix, py - iy
    rows = []
    for j in range(4):
        r = np.clip(iy - 1 + j, 0, h - 1)
        rows.append(catmull_rom(*(img[r, np.clip(ix - 1 + k, 0, w - 1)] for k in range(4)), tx))
    return catmull_rom(*rows, ty)


def tvl1_level_float64(f0, f1, tau=0.25, lambda_=0.15, theta=0.3, warps=5, iterations=300, median_filtering=5):
    """One pyramid level (nscales = 1) at fixed iterations, in float64."""
    from scipy import ndimage
    I0, I1 = f0.astype(np.float64), f1.astype(np.float64)
    h, w = I0.shape
    Ix, Iy = centred_grad(I1)
    u1, u2 = np.zeros((h, w)), np.zeros((h, w))
    p11, p12, p21, p22 = (np.zeros((h, w)) for _ in range(4))
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    l_t, taut = lambda_ * theta, tau / theta
    for _ in range(warps):
        px, py = xx + u1, yy + u2
        I1w, gx, gy = bicubic(I1, px, py), bicubic(Ix, px, py), bicubic(Iy, px, py)
        grad = gx * gx + gy * gy
        rho_c = I1w - gx * u1 - gy * u2 - I0
        for _ in range(iterations):
            rho = rho_c + gx * u1 + gy * u2
            with np.errstate(divide="ignore", invalid="ignore"):
                fi = np.where(grad < 1e-10, 0.0, -rho / grad)
            fi = np.where(rho < -l_t * grad, l_t, np.where(rho > l_t * grad, -l_t, fi))
            u1 = u1 + fi * gx + theta * divergence(p11, p12)
            u2 = u2 + fi * gy + theta * divergence(p21, p22)
            a1, b1 = forward_grad(u1)
            a2, b2 = forward_grad(u2)
            n1, n2 = 1 + taut * np.hypot(a1, b1), 1 + taut * np.hypot(a2, b2)
            p11, p12 = (p11 + taut * a1) / n1, (p12 + taut * b1) / n1
            p21, p22 = (p21 + taut * a2) / n2, (p22 + taut * b2) / n2
        if median_filtering > 1:
            u1 = ndimage.median_filter(u1, median_filtering, mode="nearest")
            u2 = ndimage.median_filter(u2, median_filtering, mode="nearest")
    return np.stack([u1, u2], -1)


# (warps, iterations, median_filtering) -> max |oracle - float64| bound.  Measured on x86-64 (gcc -O2, the oracle's
# flags) over the three kinds below: 1.1e-7, 3.3e-5, 1.8e-4 and 6.0e-4 px; mean |d| at most 4.1e-6 px.
SPEC_CASES = {(1, 1, 1): 5e-7, (2, 5, 1): 1e-4, (3, 10, 5): 1e-3, (5, 30, 5): 2e-3}


@pytest.mark.parametrize("kind,h,w", [("affine", 72, 96), ("shift", 60, 80), ("square", 72, 96)])
def test_oracle_matches_a_float64_restatement_of_the_spec(kind, h, w):
    """The kernels and the oracle were written from each other, so a mistake they share would pass every GPU
    test; this float64 restatement of one level follows DESIGN.md section 11 with its own algebra (Keys' weights,
    whole-array numpy, scipy's median)."""
    f0, f1, _ = T.flow_pair_known(13, h, w, kind)
    for (warps, iterations, med), bound in SPEC_CASES.items():
        kw = dict(warps=warps, iterations=iterations, median_filtering=med)
        got = T.flow(f0, f1, nscales=1, epsilon=-1.0, **kw)
        want = tvl1_level_float64(f0, f1, **kw)
        d = np.abs(got - want)
        assert d.max() <= bound and d.mean() <= 2e-5, (kw, d.max(), d.mean())


def test_divergence_is_minus_the_adjoint_of_the_forward_gradient():
    """<grad+ u, p> = -<u, div p> for p that is 0 at the last column (p1) and the last row (p2): the border rules
    of the spec.  The p update keeps those entries 0, since the forward gradient is 0 there."""
    rng = np.random.default_rng(1)
    for h, w in [(2, 2), (5, 9), (37, 53)]:
        u, p1, p2 = rng.standard_normal((3, h, w))
        p1[:, -1] = 0.0
        p2[-1, :] = 0.0
        a, b = forward_grad(u)
        lhs, rhs = (a * p1 + b * p2).sum(), -(u * divergence(p1, p2)).sum()
        assert abs(lhs - rhs) <= 1e-12 * (np.abs(a * p1).sum() + np.abs(b * p2).sum() + 1), (h, w, lhs, rhs)
        assert (a[:, -1] == 0).all() and (b[-1, :] == 0).all()
