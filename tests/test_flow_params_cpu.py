"""The Farneback oracle (orc_farneback_u8) against live cv2.calcOpticalFlowFarneback over the argument space
scn_farneback_u8c3 accepts, not only the reference's (3, 0.5, 15, 3, 5, 1.2).  The GPU tests
(tests/test_flow_params_gpu.py) use the oracle as their reference for these arguments, so it is held to cv2 at
the oracle's stated bound, max |d| <= 1e-4 px, here.

Each case names the GPU path it stands for (flow.cu): a generic Gaussian radius, a generic poly_n, the two-pass
double box for win_size != 15, the per-level expansion without the pyramid cache, 2 or 4 pyramid levels, one
iteration, and frames smaller than the window.

win_size = 1 is not in the grid: cv2 and the oracle disagree there (OpenCV's FarnebackUpdateFlow_Blur starts its
running sums from (m + 2) rows at m = 0), and scn_farneback_u8c3 refuses it -- see
test_flow_params_gpu.py::test_refusals_leave_output_and_launch_count_untouched."""
import cv2
import numpy as np
import pytest

import oracle
from oracle import synth

DEFAULTS = dict(num_levels=3, pyr_scale=0.5, win_size=15, num_iters=3, poly_n=5, poly_sigma=1.2)

# (h, w, overrides of DEFAULTS): what each case stands for in flow.cu
GRID = [
    (96, 128, {}),
    (540, 960, dict(num_levels=4)),                          # Gaussian radius 19 (generic); levels == 4
    (270, 480, dict(pyr_scale=0.7)),                         # radius 2 at level 3 (generic)
    (96, 128, dict(pyr_scale=0.3)),
    (96, 128, dict(poly_n=7, poly_sigma=1.5)),               # generic poly_n
    (96, 128, dict(poly_n=3, poly_sigma=0.9)),
    (96, 128, dict(poly_n=1, poly_sigma=0.6)),
    (96, 128, dict(win_size=2)),                             # double two-pass box (win_size != 15)
    (96, 128, dict(win_size=3)),
    (96, 128, dict(win_size=4)),
    (96, 128, dict(win_size=9)),
    (96, 128, dict(win_size=16)),
    (96, 128, dict(win_size=21)),
    (270, 480, dict(pyr_scale=0.8, num_levels=8)),           # pyramid over 2 W H pixels: no cache
    (540, 960, dict(pyr_scale=0.7, num_levels=8, poly_n=7, poly_sigma=1.5)),
    (540, 960, dict(pyr_scale=0.8, num_levels=8)),
    (200, 300, {}),                                          # levels == 2
    (96, 128, dict(num_iters=1)),                            # no update_matrices_kernel between iterations
    (96, 128, dict(num_iters=6)),
    (96, 128, dict(num_levels=0)),
    (1, 1, {}), (2, 2, {}), (1, 64, {}), (64, 1, {}), (4, 4, {}), (14, 14, {}),   # smaller than the window
    (33, 89, {}),
]


def _cv2(g0, g1, a):
    return cv2.calcOpticalFlowFarneback(g0, g1, None, a["pyr_scale"], a["num_levels"], a["win_size"], a["num_iters"],
                                        a["poly_n"], a["poly_sigma"], 0)


def _check(h, w, over, seed):
    a = dict(DEFAULTS, **over)
    f0, f1 = synth.flow_pair(seed, h, w, "shift")
    g0, g1 = oracle.bgr2gray(f0), oracle.bgr2gray(f1)
    got = oracle.farneback(g0, g1, **a)
    want = _cv2(g0, g1, a)
    assert got.shape == want.shape == (h, w, 2)
    d = np.abs(got - want)
    assert d.max() <= 1e-4, (h, w, over, d.max(), d.mean())
    return want


@pytest.mark.parametrize("h,w,over", GRID, ids=[f"{h}x{w}-" + "-".join(f"{k}{v}" for k, v in o.items())
                                                for h, w, o in GRID])
def test_oracle_matches_cv2_off_the_default_arguments(h, w, over):
    _check(h, w, over, 1000 + h + w)


def test_oracle_matches_cv2_with_a_79_tap_gaussian():
    """num_levels=5 at 1080p: level 5's Gaussian has ksize 79 (the GPU refuses this with SCN_E_UNSUPPORTED; the
    oracle used to overrun fixed 64-entry tap arrays here).  The field still follows the synthetic motion."""
    want = _check(1080, 1920, dict(num_levels=5), 941)
    med = np.median(want[200:-200, 200:-200].reshape(-1, 2), axis=0)
    assert 1.0 < med[0] < 1.6 and -0.8 < med[1] < -0.5, med
