"""TV-L1 (scn_tvl1_u8, kernels.tvl1_flow) on the GPU against its C restatement oracle.tvl1.flow.

The kernels evaluate every per-pixel expression in the oracle's order and are built with -fmad=false, so
apart from the error sum that stops a warp step (a fixed tree of float tile sums on the GPU, a running double
sum in the oracle) the two round alike.  Bounds: at fixed iterations mean |d| <= 2e-4 px, 99.9th percentile
<= 5e-3 px, max <= 5e-2 px; at the defaults iteration counts within 1 of the oracle's and, on textured pairs,
mean |d| <= 2e-3 px, 99.9th percentile <= 5e-2 px."""
import numpy as np
import pytest
import torch

from oracle import synth
from oracle import tvl1 as T
from scanner_b200 import cabi, kernels

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def textured(seed, h, w):
    f0, f1, _ = T.flow_pair_known(seed, h, w, "shift")
    return f0, f1


def gpu_flow(f0, f1, **kw):
    out = kernels.tvl1_flow(dev(f0[None]), dev(f1[None]), return_iterations=True, **kw)
    return out[0][0].cpu().numpy(), out[1][0]


def check_close(got, want, mean=2e-4, p999=5e-3, mx=5e-2):
    assert np.isfinite(got).all()
    d = np.abs(got.astype(np.float64) - want)
    stats = (d.mean(), np.percentile(d, 99.9), d.max())
    assert stats[0] <= mean and stats[1] <= p999 and stats[2] <= mx, stats


@pytest.mark.parametrize("h,w", [(37, 53), (120, 160), (270, 480), (24, 200)])
def test_fixed_iterations_match_oracle(h, w):
    """epsilon = -1: every warp runs all `iterations` (30 here, to keep the oracle's CPU time short).  24 x 200
    stops its pyramid after two levels (19 x 160, then 15 < 16)."""
    f0, f1 = textured(700 + h, h, w)
    kw = dict(epsilon=-1.0, iterations=30)
    got, it = gpu_flow(f0, f1, **kw)
    want, wit = T.flow(f0, f1, return_iterations=True, **kw)
    assert (it == wit).all(), (it, wit)
    check_close(got, want)


@pytest.mark.parametrize("kind", ["shift", "affine", "square", "noise"])
def test_defaults_match_oracle(kind):
    h, w = 120, 160
    if kind == "noise":
        f0, f1 = synth.rand_frame(5, h, w, 1)[..., 0], synth.rand_frame(6, h, w, 1)[..., 0]
    else:
        f0, f1, _ = T.flow_pair_known(11, h, w, kind)
    got, it = gpu_flow(f0, f1)
    want, wit = T.flow(f0, f1, return_iterations=True)
    assert np.abs(it - wit).max() <= 1, (it, wit)
    if kind == "noise":
        assert np.isfinite(got).all()
        assert np.abs(got - want).mean() <= 2e-2
    else:
        check_close(got, want, mean=2e-3, p999=5e-2, mx=np.inf)


def test_1080p_shift_defaults():
    f0, f1, _ = T.flow_pair_known(3, 1080, 1920, "shift")
    got, it = gpu_flow(f0, f1)
    want, wit = T.flow(f0, f1, return_iterations=True)
    assert np.abs(it - wit).max() <= 1, (it, wit)
    check_close(got, want, mean=2e-3, p999=5e-2, mx=np.inf)
    med = np.median(got[16:-16, 16:-16].reshape(-1, 2), axis=0)
    assert abs(med[0] - 1.5) <= 0.02 and abs(med[1] + 0.75) <= 0.02, med


GRID = [dict(nscales=s) for s in (1, 2, 3, 4, 6)] + [dict(warps=k) for k in (1, 2, 3, 6)] + \
       [dict(scale_step=v) for v in (0.5, 0.6, 0.7, 0.9)] + [dict(median_filtering=m) for m in (1, 3)] + \
       [dict(tau=0.125), dict(lambda_=0.05), dict(lambda_=0.4), dict(theta=0.1), dict(theta=0.6),
        dict(tau=0.2, lambda_=0.3, theta=0.5, nscales=3, warps=2, median_filtering=3)]


@pytest.mark.parametrize("params", GRID, ids=lambda p: ",".join(f"{k}={v}" for k, v in p.items()))
def test_parameter_grid_matches_oracle(params):
    f0, f1, _ = T.flow_pair_known(21, 72, 96, "affine")
    kw = dict(epsilon=-1.0, iterations=20, **params)
    got, it = gpu_flow(f0, f1, **kw)
    want, wit = T.flow(f0, f1, return_iterations=True, **kw)
    assert (it == wit).all()
    check_close(got, want)


def mixed_batch(h, w):
    """8 pairs: identical frames (stop after 1 iteration per step), noise, and shifts (which run longer)."""
    pairs = []
    for i in range(8):
        if i % 3 == 0:
            f = T.flow_pair_known(40 + i, h, w, "shift")[0]
            pairs.append((f, f))
        elif i % 3 == 1:
            pairs.append((synth.rand_frame(50 + i, h, w, 1)[..., 0], synth.rand_frame(60 + i, h, w, 1)[..., 0]))
        else:
            pairs.append(T.flow_pair_known(70 + i, h, w, "affine" if i % 2 else "shift")[:2])
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])


def test_deterministic_and_isolated_in_a_batch():
    a, b = mixed_batch(64, 96)
    A, B = dev(a), dev(b)
    f1, it1 = kernels.tvl1_flow(A, B, return_iterations=True)
    f2 = kernels.tvl1_flow(A, B)
    assert torch.equal(f1, f2)
    assert len({int(x) for x in it1[:, 0, 0]}) > 1  # pairs stop at different iterations within one call
    for i in range(8):
        alone, ita = kernels.tvl1_flow(A[i:i + 1], B[i:i + 1], return_iterations=True)
        assert torch.equal(alone[0], f1[i]), i
        assert (ita[0] == it1[i]).all()
        if i % 3 == 0:
            assert (alone == 0).all() and (ita[0][ita[0] > 0] == 1).all()


def test_identical_frames_give_exact_zero_at_fixed_iterations():
    f = T.flow_pair_known(9, 90, 130, "affine")[0]
    got = kernels.tvl1_flow(dev(f[None]), dev(f[None]), epsilon=-1.0, iterations=40)
    assert (got == 0).all()


def test_pointer_lists_over_64_pairs():
    n, h, w = 70, 24, 40
    rng = np.random.default_rng(5)
    base = [T.flow_pair_known(int(s), h, w, "shift")[:2] for s in rng.integers(0, 1000, 5)]
    a = np.stack([base[i % 5][0] for i in range(n)])
    b = np.stack([base[i % 5][1] if i % 7 else base[i % 5][0] for i in range(n)])
    got, it = kernels.tvl1_flow(dev(a), dev(b), return_iterations=True)
    for i in (0, 1, 7, 63, 64, 65, 69):
        want, wit = T.flow(a[i], b[i], return_iterations=True)
        assert np.abs(it[i] - wit).max() <= 1
        check_close(got[i].cpu().numpy(), want, mean=2e-3, p999=5e-2, mx=np.inf)


def test_rgb_input_goes_through_rgb2gray():
    a, b = synth.flow_pair(12, 48, 64, "shift")
    got = kernels.tvl1_flow(dev(a[None]), dev(b[None]), epsilon=-1.0, iterations=10)[0].cpu().numpy()
    want = T.flow(a, b, epsilon=-1.0, iterations=10)
    check_close(got, want)


def test_refusals_on_device_launch_nothing():
    f = dev(np.zeros((1, 8, 8), np.uint8))
    L = cabi.lib()
    before = L.scn_launch_count()
    for kw in (dict(tau=0.0), dict(iterations=0), dict(scale_step=1.0), dict(median_filtering=4),
               dict(epsilon=float("nan"))):
        with pytest.raises(cabi.ScnError):
            kernels.tvl1_flow(f, f, **kw)
    assert L.scn_launch_count() == before
