"""Pin of the NV12 -> RGB arithmetic to the REFERENCE'S OWN KERNEL.

tests/golden/nv12_ref.npz holds what scanner::convertNV12toRGBA (image.cu:229-239 -> NV12_to_RGB :109-200 of the
reference, compiled unmodified: oracle/make_golden_ref.py) produced on an H100: the SHA-256 of its output over an input
set that presents every one of the 2^24 (Y,Cb,Cr) triples on an even row, the averaged-chroma odd rows and every
frame's last-chroma-row case (oracle/synth.py nv12_exhaustive), the SHA-256 of its output on seeded random surfaces,
and its output on the seeded surfaces of make_golden_ref.CASES.  Against it, byte for byte:
  * the product's colour conversion (scn_nv12_to_rgb24) must reproduce it,
  * the oracle restatement (oracle.nv12_to_rgb) must equal the product,
and the histogram / resize the product computes straight from the NV12 surface (scn_nv12_hist_resize:
nv12_hist kernels + nv12_resize_kernel) must equal the histogram / resize of that RGB.
"""
import hashlib
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import oracle  # noqa: E402
from oracle import synth  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "nv12_ref.npz"))


def _hist_of_rgb(rgb):  # (H,W,3) u8 cuda -> (3,16) int64, bin = v >> 4 (tests/test_ops.cpp:38-43)
    bins = (rgb >> 4).to(torch.int64).reshape(-1, 3)
    return torch.stack([torch.bincount(bins[:, c], minlength=16) for c in range(3)])


def test_reference_kernel_equals_oracle_and_product_on_all_yuv_triples(golden):
    from scanner_b200 import kernels
    w, h = synth.EXH_W, synth.EXH_H
    seen = torch.zeros(1 << 24, dtype=torch.bool, device="cuda")
    sha = hashlib.sha256()
    for f in range(synth.EXH_FRAMES):
        luma, chroma = synth.nv12_exhaustive(f)
        surf_h = np.concatenate([luma, chroma], 0)
        surf = torch.from_numpy(surf_h).cuda()
        # 1. the product's conversion kernel; the reference kernel's output over all frames is held by its SHA-256
        got_p = kernels.nv12_to_rgb(surf[None], w, h)[0]
        got_h = got_p.cpu().numpy()
        sha.update(got_h.tobytes())
        # coverage bookkeeping: the triples presented on even rows of this frame
        ly = surf[0:h:2, :w].to(torch.int64)
        cb = surf[h:, 0:w:2].to(torch.int64).repeat_interleave(2, dim=1)
        cr = surf[h:, 1:w:2].to(torch.int64).repeat_interleave(2, dim=1)
        seen[(ly << 16 | cb << 8 | cr).reshape(-1)] = True
        # 2. the oracle restatement
        bad = (got_h != oracle.nv12_to_rgb(luma, chroma, w))
        assert not bad.any(), f"frame {f}: oracle differs from the product at {bad.sum()} bytes, first {np.argwhere(bad)[0]}"
        # 3. histogram + resize computed from the NV12 surface without materialising RGB
        hist, res = kernels.nv12_hist_resize(surf[None], w, h, 224, 224)
        assert torch.equal(hist[0].to(torch.int64), _hist_of_rgb(got_p)), f"frame {f}: fused histogram"
        assert torch.equal(res[0], kernels.resize(got_p[None], 224, 224)[0]), f"frame {f}: fused resize"
    assert bool(seen.all()), "the input set must present every (Y,Cb,Cr) triple on an even row"
    assert sha.digest() == golden["exhaustive_sha256"].tobytes(), "scn_nv12_to_rgb24 differs from the reference kernel"


@pytest.mark.parametrize("seed,h,w,pitch", [(1, 1080, 1920, 2048), (2, 270, 480, 512), (3, 34, 70, 128), (4, 2, 2, 64),
                                            (5, 18, 30, 32), (6, 1088, 1920, 1920)])
def test_reference_kernel_on_random_surfaces(golden, seed, h, w, pitch):
    from scanner_b200 import kernels
    luma, chroma = synth.nv12_surface(seed, h, w, pitch)
    surf = torch.from_numpy(np.concatenate([luma, chroma], 0)).cuda()
    got = kernels.nv12_to_rgb(surf[None], w, h)[0]
    assert hashlib.sha256(got.cpu().numpy().tobytes()).digest() == golden[f"rand{seed}_sha256"].tobytes()
    assert (got.cpu().numpy() == oracle.nv12_to_rgb(luma, chroma, w)).all()
    hist, _ = kernels.nv12_hist_resize(surf[None], w, h, 0, 0, want_resize=False)
    assert torch.equal(hist[0].to(torch.int64), _hist_of_rgb(got))


def test_committed_reference_goldens_reproduce(golden):
    from scanner_b200 import kernels
    for k in sorted(x[:-5] for x in golden.files if x.endswith("_meta")):
        seed, h, w, pitch = [int(x) for x in golden[k + "_meta"]]
        luma, chroma = synth.nv12_surface(seed, h, w, pitch)
        surf = torch.from_numpy(np.concatenate([luma, chroma], 0)).cuda()
        got = kernels.nv12_to_rgb(surf[None], w, h)[0].cpu().numpy()
        if k + "_out" in golden.files:
            assert (got == golden[k + "_out"]).all(), k
        else:
            assert hashlib.sha256(got.tobytes()).digest() == golden[k + "_sha256"].tobytes(), k
