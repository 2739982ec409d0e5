"""oracle.blur_sat, the summed-area-table restatement of the box filter that tests/test_blur_gpu.py holds the Blur
kernels to at sizes where oracle.blur (O(k^2) per sample) is too slow, against oracle.blur itself (which
tests/test_reference_ops_cpu.py pins to the reference's own compiled BlurKernel): every kernel size, frames smaller
than the window, exactly the window, one row or one column, batched and saturated."""
import numpy as np
import pytest

import oracle
from oracle import synth

SHAPES = [(1, 1), (1, 40), (40, 1), (2, 3), (5, 5), (7, 33), (33, 7), (31, 31), (32, 30), (45, 52)]


@pytest.mark.parametrize("k", range(1, 32))
def test_blur_sat_equals_the_oracle(k):
    shapes = SHAPES + [(k, k), (k - 1, 40), (40, k - 1), (k, 40), (40, k), (k + 1, k + 2), (k + 1, 1)]
    for j, (h, w) in enumerate(s for s in shapes if s[0] > 0 and s[1] > 0):
        img = synth.rand_frame(1000 + 37 * k + j, h, w)
        assert (oracle.blur_sat(img, k) == oracle.blur(img, k)).all(), (k, h, w)
    sat = np.full((k + 3, 2 * k + 5, 3), 255, np.uint8)
    assert (oracle.blur_sat(sat, k) == oracle.blur(sat, k)).all(), k
    # a batch is each frame on its own
    batch = np.stack([synth.rand_frame(2000 + k + i, 23, 41) for i in range(3)])
    got = oracle.blur_sat(batch, k)
    for i in range(3):
        assert (got[i] == oracle.blur(batch[i], k)).all(), (k, i)


def test_blur_sat_border_and_window_edges():
    img = synth.rand_frame(5, 12, 14)
    out = oracle.blur_sat(img, 4)  # fl = 1, fr = 2
    assert (out[:1] == 0).all() and (out[-2:] == 0).all() and (out[:, :1] == 0).all() and (out[:, -2:] == 0).all()
    assert out[1, 1, 0] == img[0:4, 0:4, 0].astype(np.int64).sum() // 16
    assert (oracle.blur_sat(img, 1) == img).all()
    assert not oracle.blur_sat(img[:3], 4).any()  # shorter than the window: all border
