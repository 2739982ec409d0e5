"""nv12_stream_kernel's two prefetch paths and its two step loops, on geometries where they alternate.

The kernel counts most steps in blocks of 4, whose prefetch moves every lane's pointers on by one select per step,
and the rest one at a time, locating every lane's unit from scratch: the last steps of a frame (the last chroma row,
padding lanes), the steps up to the next multiple of 4 after them, and the last ns mod 4 steps of every span.  Which
steps take which path depends on the row width in 16-pixel units (a step moves a lane 32 units on: 32 / units_per_row
row pairs plus one where its column wraps), the frame height and where each warp's range starts and ends.  The
geometries below vary all three; each histogram is compared exactly with torch.bincount of v >> 4 of
kernels.nv12_to_rgb (pinned to the reference's own kernel by test_ref_pin_gpu.py)."""
import pytest
import torch

from scanner_b200 import cabi, kernels

pytestmark = pytest.mark.gpu

# (n, h, w, pitch), commented with units per row, steps per frame, padding lanes in a frame's last step.  These
# launches give each warp about 8 steps, so most ranges hold a frame boundary or a partial block.
GEOMETRIES = [
    (9, 4098, 16, 32),        # 1 unit per row (a step spans 32 row pairs), 65 steps, 31 padding lanes
    (5, 2050, 32, 48),        # 2, 65, 30
    (7, 1640, 80, 96),        # 5 (32 = 6 * 5 + 2), 129, 28
    (11, 1172, 112, 128),     # 7, 129, 26
    (13, 270, 496, 512),      # 31 (a wrap in nearly every step), 131, 7
    (6, 252, 528, 544),       # 33, 130, 2
    (17, 330, 912, 912),      # 57 (pitch == width), 294, 3
    (64, 98, 1936, 1952),     # 121, 186, 23
    (64, 360, 640, 656),      # 40, 225, 0
    (3, 1080, 1920, 2048),    # the benchmark's frame: 120, 2025, 0
]


def _ref_hist(surf, w, h, chunk=4):
    off = torch.arange(0, 48, 16, device=surf.device)
    out = []
    for i in range(0, surf.shape[0], chunk):
        rgb = kernels.nv12_to_rgb(surf[i:i + chunk], w, h)
        out += [torch.bincount(((f.reshape(-1, 3) >> 4).long() + off).flatten(), minlength=48).view(3, 16) for f in rgb]
    return torch.stack(out)


@pytest.mark.parametrize("n,h,w,pitch", GEOMETRIES)
def test_nv12_stream_prefetch_paths(n, h, w, pitch):
    g = torch.Generator(device="cuda").manual_seed(n * 7919 + h * 31 + w)
    surf = torch.randint(0, 256, (n, h * 3 // 2, pitch), dtype=torch.uint8, device="cuda", generator=g)
    surf[n // 2, : h // 3, :w] = 16             # a bar of one colour: counters far from uniform
    surf[n // 2, h: h + h // 6, :w] = 128
    L = cabi.lib()
    L.scn_prof_enable(1)
    try:
        got, _ = kernels.nv12_hist_resize(surf, w, h, 224, 224, want_resize=False)
        torch.cuda.synchronize()
        ran = {k: v["launches"] for k, v in cabi.prof_report().items()}
    finally:
        L.scn_prof_enable(0)
    assert ran.get("nv12_stream_kernel") == 1, ran
    want = _ref_hist(surf, w, h)
    bad = (got.long() != want).flatten(1).any(1).nonzero().flatten().tolist()
    assert not bad, bad[:8]
