"""TV-L1 (scn_tvl1_u8, kernels.tvl1_flow) on the GPU against its C restatement oracle.tvl1.flow.

The kernels evaluate every per-pixel expression in the oracle's order and are built with -fmad=false, so the two
round alike.  The only expression they do not share by default is the error sum that stops a warp step (a fixed
tree of float tile sums on the GPU, a running double sum in the oracle); oracle.tvl1.flow(error_sum="tiles") sums
it in the kernel's order.  So every comparison here is exact: equal iteration counts and `==` flows, at fixed
iterations and at the defaults.  test_tvl1_exact_gpu.py holds the kernels to the same bar across geometries,
content and the stop decision itself."""
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


def oracle_flow(f0, f1, **kw):
    return T.flow(f0, f1, return_iterations=True, error_sum="tiles", **kw)


def check_exact(got, it, want, wit):
    """Equal iteration counts and bit-equal finite flows (== takes -0 and +0 as equal)."""
    assert np.isfinite(want).all() and np.isfinite(got).all()
    assert np.array_equal(it, wit), (it, wit)
    bad = got != want
    assert not bad.any(), (f"{int(bad.sum())} of {bad.size} values differ, first at {tuple(np.argwhere(bad)[0])}, "
                           f"max |d| {np.abs(got.astype(np.float64) - want).max():.3g}")


@pytest.mark.parametrize("h,w", [(37, 53), (120, 160), (270, 480), (24, 200)])
def test_fixed_iterations_match_oracle(h, w):
    """epsilon = -1: every warp runs all `iterations` (30 here, to keep the oracle's CPU time short).  24 x 200
    stops its pyramid after two levels (19 x 160, then 15 < 16)."""
    f0, f1 = textured(700 + h, h, w)
    kw = dict(epsilon=-1.0, iterations=30)
    got, it = gpu_flow(f0, f1, **kw)
    check_exact(got, it, *oracle_flow(f0, f1, **kw))


@pytest.mark.parametrize("kind", ["shift", "affine", "square", "noise"])
def test_defaults_match_oracle(kind):
    h, w = 120, 160
    if kind == "noise":
        f0, f1 = synth.rand_frame(5, h, w, 1)[..., 0], synth.rand_frame(6, h, w, 1)[..., 0]
    else:
        f0, f1, _ = T.flow_pair_known(11, h, w, kind)
    got, it = gpu_flow(f0, f1)
    check_exact(got, it, *oracle_flow(f0, f1))


def test_1080p_shift_defaults():
    f0, f1, _ = T.flow_pair_known(3, 1080, 1920, "shift")
    got, it = gpu_flow(f0, f1)
    check_exact(got, it, *oracle_flow(f0, f1))
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
    check_exact(got, it, *oracle_flow(f0, f1, **kw))


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
    for i in range(8):  # every pair, each stopping on its own, equals its oracle run
        check_exact(f1[i].cpu().numpy(), it1[i], *oracle_flow(a[i], b[i]))


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
        check_exact(got[i].cpu().numpy(), it[i], *oracle_flow(a[i], b[i]))


def test_rgb_input_goes_through_rgb2gray():
    a, b = synth.flow_pair(12, 48, 64, "shift")
    got, it = gpu_flow(a, b, epsilon=-1.0, iterations=10)
    check_exact(got, it, *oracle_flow(a, b, epsilon=-1.0, iterations=10))


def test_refusals_on_device_launch_nothing():
    f = dev(np.zeros((1, 8, 8), np.uint8))
    L = cabi.lib()
    before = L.scn_launch_count()
    for kw in (dict(tau=0.0), dict(iterations=0), dict(scale_step=1.0), dict(median_filtering=4),
               dict(epsilon=float("nan"))):
        with pytest.raises(cabi.ScnError):
            kernels.tvl1_flow(f, f, **kw)
    assert L.scn_launch_count() == before
