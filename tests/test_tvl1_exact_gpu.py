"""TV-L1 kernels (scn_tvl1_u8) equal to their C restatement oracle.tvl1.flow bit for bit.

tvl1.cu is built with -fmad=false and evaluates every per-pixel expression in orc_tvl1_u8's order, so the only
expression the two do not share is the error sum that stops a warp step.  With epsilon <= 0 that sum decides
nothing, and with error_sum="tiles" the oracle sums it in the kernel's order.  Every comparison here is therefore
`==` on finite values (which takes -0 and +0 as equal: fminf / fmaxf in the median kernel and the oracle's
insertion sort may return either zero), and iteration counts are equal.

The ladder adds one kernel per rung, so the first rung that fails names the kernel at fault."""
import numpy as np
import pytest
import torch

from oracle import synth
from oracle import tvl1 as T
from scanner_b200 import kernels

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_flow(f0, f1, **kw):
    out = kernels.tvl1_flow(dev(f0[None]), dev(f1[None]), return_iterations=True, **kw)
    return out[0][0].cpu().numpy(), out[1][0]


def assert_exact(got, it, want, wit):
    assert np.isfinite(want).all() and np.isfinite(got).all()
    assert np.array_equal(it, wit), (it, wit)
    bad = got != want
    assert not bad.any(), (f"{int(bad.sum())} of {bad.size} values differ, first at {tuple(np.argwhere(bad)[0])}, "
                           f"max |d| {np.abs(got.astype(np.float64) - want).max():.3g}")


def check(f0, f1, **kw):
    got, it = gpu_flow(f0, f1, **kw)
    want, wit = T.flow(f0, f1, return_iterations=True, error_sum="tiles", **kw)
    assert_exact(got, it, want, wit)
    return want


FIXED = dict(epsilon=-1.0)

LADDER = [
    ("warp-at-integer-positions", dict(nscales=1, warps=1, iterations=1, median_filtering=1)),
    ("div-and-p", dict(nscales=1, warps=1, iterations=2, median_filtering=1)),
    ("bicubic-at-fractions", dict(nscales=1, warps=2, iterations=2, median_filtering=1)),
    ("median3", dict(nscales=1, warps=2, iterations=2, median_filtering=3)),
    ("median5", dict(nscales=1, warps=2, iterations=2, median_filtering=5)),
    ("pyramid-and-upsample", dict(nscales=2, warps=2, iterations=2, median_filtering=5)),
]


@pytest.mark.parametrize("params", [p for _, p in LADDER], ids=[n for n, _ in LADDER])
def test_ladder(params):
    f0, f1, _ = T.flow_pair_known(31, 72, 96, "affine")
    check(f0, f1, **FIXED, **params)


# (h, w, params): pyramids of one level (under 16 at the next level), npx at the 1024-pixel tile edges, thin
# frames, all ten levels packed in the workspace, the largest warp count
GEOMETRY = [
    (2, 2, {}), (2, 37, {}), (37, 2, {}), (15, 15, {}), (16, 16, {}), (17, 16, {}),
    (31, 33, {}), (32, 32, {}), (25, 41, {}), (3, 683, {}),
    (2, 4096, {}), (4096, 2, {}),
    (120, 160, dict(nscales=10, scale_step=0.95)), (120, 160, dict(nscales=10, scale_step=0.99)),
    (48, 64, dict(warps=20, nscales=2)),
]


@pytest.mark.parametrize("h,w,params", GEOMETRY,
                         ids=[f"{h}x{w}" + "".join(f",{k}={v}" for k, v in p.items()) for h, w, p in GEOMETRY])
def test_geometry_fixed_iterations(h, w, params):
    f0, f1, _ = T.flow_pair_known(800 + h + w, h, w, "shift")
    kw = dict(FIXED, iterations=5, warps=3)
    kw.update(params)
    if kw.get("nscales") == 10:  # all ten levels are packed into the workspace
        assert len(T.levels(w, h, nscales=10, scale_step=kw["scale_step"])) == 10
    check(f0, f1, **kw)


def test_1080p_fixed_iterations():
    f0, f1, _ = T.flow_pair_known(5, 1080, 1920, "affine")
    check(f0, f1, **FIXED, iterations=5, nscales=2, warps=2)


def test_2160p_fixed_iterations():
    """3840 x 2160 (8.3 M pixels, 8100 error tiles) at one level, which keeps the oracle's CPU time near 20 s."""
    f0, f1, _ = T.flow_pair_known(6, 2160, 3840, "shift")
    check(f0, f1, **FIXED, iterations=3, nscales=1, warps=2, median_filtering=3)


def checkerboard(h, w, cell, dx=0, dy=0):
    yy, xx = np.mgrid[0:h, 0:w]
    return np.where((((xx - dx) // cell) + ((yy - dy) // cell)) % 2 == 0, 255, 0).astype(np.uint8)


def half_constant(seed, h, w):
    f0, f1, _ = T.flow_pair_known(seed, h, w, "shift")
    f0, f1 = f0.copy(), f1.copy()
    f0[:, : w // 2] = 90
    f1[:, : w // 2] = 90
    return f0, f1


CONTENT = {
    # grad = 0 and rho = 0 everywhere: every pixel takes the grad < 1e-10 branch
    "constant-equal": lambda h, w: (np.full((h, w), 77, np.uint8), np.full((h, w), 77, np.uint8)),
    # grad = 0 and rho > 0: the threshold branch with a zero gradient
    "constant-step": lambda h, w: (np.full((h, w), 77, np.uint8), np.full((h, w), 78, np.uint8)),
    "half-constant": lambda h, w: half_constant(12, h, w),
    "checkerboard": lambda h, w: (checkerboard(h, w, 6), checkerboard(h, w, 6, 2, 1)),
}


@pytest.mark.parametrize("kind", list(CONTENT))
def test_content_fixed_iterations(kind):
    f0, f1 = CONTENT[kind](60, 84)
    want = check(f0, f1, **FIXED, iterations=6, nscales=3, warps=3)
    if kind == "constant-equal":
        assert (want == 0).all()


def test_flow_that_leaves_the_frame():
    """A 6 px shift on a 40 x 48 frame: the flow at the last columns points past x = w + 1, so the warp clamps
    sample positions to [-2, w + 1] (measured with the oracle: max x + u1 - (w + 1) = 5.2 px)."""
    h, w = 40, 48
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    f0 = np.clip(np.rint(T.tex_gray(3, xx, yy)), 0, 255).astype(np.uint8)
    f1 = np.clip(np.rint(T.tex_gray(3, xx - 6.0, yy - 1.0)), 0, 255).astype(np.uint8)
    want = check(f0, f1, **FIXED, iterations=30, nscales=3, warps=3)
    px = xx + want[..., 0]
    assert px.max() > w + 1 + 2.0, px.max()


# ---- the stop decision, at the last bit of the error sum ----
# (seed, h, w) of affine pairs whose first-iteration error lies where a different order of the float sums (for
# example the 8 warp sums of a tile added last to first) would round to the other side of epsilon^2
PROBES = [(1, 40, 60), (7, 40, 60), (9, 32, 32), (13, 40, 60), (17, 72, 96), (18, 32, 32), (25, 40, 60),
          (28, 40, 60), (31, 40, 60), (35, 72, 96), (3, 512, 520)]


@pytest.mark.parametrize("seed,h,w", PROBES, ids=[f"seed{s}-{h}x{w}" for s, h, w in PROBES])
def test_stop_decision_at_the_last_bit(seed, h, w):
    """One warp of one level.  The first iteration starts from u = 0, so its error terms are u1^2 + u2^2 of the
    flow after one iteration, and the error is tile_sum(terms) / npx.  epsilon = the smallest float with
    epsilon^2 >= error must stop after that iteration; the float just below must run a second."""
    f0, f1, _ = T.flow_pair_known(seed, h, w, "affine")
    P = dict(nscales=1, warps=1, median_filtering=1)
    one = T.flow(f0, f1, epsilon=-1.0, iterations=1, **P)
    terms = one[..., 0] * one[..., 0] + one[..., 1] * one[..., 1]
    err = T.tile_sum(terms) / (h * w)
    eps = np.float32(np.sqrt(err))
    while float(eps) * float(eps) < err:
        eps = np.nextafter(eps, np.float32(np.inf))
    while float(np.nextafter(eps, np.float32(0))) ** 2 >= err:
        eps = np.nextafter(eps, np.float32(0))
    below = np.nextafter(eps, np.float32(0))
    for e, n in ((eps, 1), (below, 2)):
        got, it = gpu_flow(f0, f1, epsilon=float(e), iterations=3, **P)
        want, wit = T.flow(f0, f1, return_iterations=True, error_sum="tiles", epsilon=float(e), iterations=3, **P)
        assert wit[0, 0] == n, (e, wit)
        assert_exact(got, it, want, wit)


def test_noise_defaults():
    f0, f1 = synth.rand_frame(15, 90, 120, 1)[..., 0], synth.rand_frame(16, 90, 120, 1)[..., 0]
    check(f0, f1)
