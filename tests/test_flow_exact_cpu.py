"""The kernel-ordered Farneback oracle (oracle/farneback_k.c) against the specification (orc_farneback_u8, itself held
to cv2 within 1e-4 px by test_flow_params_cpu.py).

tests/test_flow_exact_gpu.py holds the CUDA kernels to farneback_k with `==`; this file carries the cv2 anchor over:
over the argument grid and the edge geometries of test_flow_params_gpu.py, every box variant stays within the bounds
the kernels were held to against orc_farneback_u8 before (max |d| <= 2e-3 px, mean <= 1e-4 px; win_size 2, whose
3 x 3 window at scale 1/4 leaves ill-conditioned systems, within 0.1 px with at most 130 pixels over 2e-3 px).  The
two double box variants agree, and the float one is within 5e-4 px of them on smooth pairs."""
import numpy as np
import pytest

import oracle
from oracle import farneback_k as K
from oracle import synth

from helpers.flow_cases import DEFAULTS, EDGES, GRID


def _check(got, want, what, max_d=2e-3, outliers=0):
    d = np.abs(got - want)
    n_out = int((d.max(-1) > 2e-3).sum())
    assert np.isfinite(got).all(), what
    assert d.max() <= max_d and d.mean() <= 1e-4 and n_out <= outliers, (what, d.max(), d.mean(), n_out)


def _pair(h, w, seed):
    return synth.flow_pair(seed, h, w, "shift")


def _spec(f0, f1, a):
    return oracle.farneback(oracle.bgr2gray(f0), oracle.bgr2gray(f1), **a)


@pytest.mark.parametrize("h,w,over", GRID, ids=[f"{h}x{w}-" + "-".join(f"{k}{v}" for k, v in o.items())
                                                for h, w, o in GRID])
def test_kernel_ordered_oracle_within_the_specification_over_the_grid(h, w, over):
    a = dict(DEFAULTS, **over)
    f0, f1 = _pair(h, w, 2000 + h + w)
    want = _spec(f0, f1, a)
    bound = dict(max_d=0.1, outliers=130) if a["win_size"] == 2 else {}
    boxes = ["f32", "f64_slide", "f64"] if a["win_size"] // 2 == 7 else ["f64"]
    got = {b: K.flow(f0, f1, box=b, **a) for b in boxes}
    for b, g in got.items():
        _check(g, want, (h, w, over, b), **bound)
    if "f32" in got:
        assert np.abs(got["f64_slide"] - got["f64"]).max() <= 1e-6, (h, w, over)
        assert np.abs(got["f32"] - got["f64"]).max() <= 5e-4, (h, w, over)


@pytest.mark.parametrize("h,w", EDGES, ids=[f"{h}x{w}" for h, w in EDGES])
def test_kernel_ordered_oracle_within_the_specification_at_edge_geometries(h, w):
    f0, f1 = _pair(h, w, 2300 + h + w)
    want = _spec(f0, f1, DEFAULTS)
    got = {b: K.flow(f0, f1, box=b) for b in ("f32", "f64_slide", "f64")}
    for b, g in got.items():
        _check(g, want, (h, w, b))
    assert np.abs(got["f64_slide"] - got["f64"]).max() <= 1e-6
    assert np.abs(got["f32"] - got["f64"]).max() <= 5e-4


def test_level_plan_and_box_choice():
    """The level plan of scn_farneback_u8c3: the 32-px stop (63 / 64 / 65 px at pyr_scale 0.5) and lrint's half to
    even (129 * 0.5 = 64.5 -> 64); the box variant per win_size and switch."""
    assert K.levels(63, 63) == [(63, 63)]
    assert K.levels(64, 64) == [(64, 64), (32, 32)]
    assert K.levels(65, 65) == [(65, 65), (32, 32)]          # 32.5 -> 32
    assert K.levels(129, 129) == [(129, 129), (64, 64), (32, 32)]
    assert K.levels(1920, 1080, 4) == [(1920, 1080), (960, 540), (480, 270), (240, 135), (120, 68)]
    assert K.box_for(15) == "f32" and K.box_for(14) == "f32" and K.box_for(16) == "f64" and K.box_for(2) == "f64"
    assert K.box_for(15, box_f64=True) == "f64_slide" and K.box_for(15, unfused=True) == "f64"
    with pytest.raises(ValueError):
        K.flow(*_pair(8, 8, 1), box="f32", win_size=9)
    with pytest.raises(ValueError):
        K.flow(*_pair(8, 8, 1), win_size=1)
