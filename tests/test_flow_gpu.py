"""OpticalFlow (Farneback) on the GPU against cv2 and against the kernel-ordered oracle (oracle/farneback_k.c).
Against cv2 (and its restatement orc_farneback_u8, pinned to cv2 within 1e-4 px) the CUDA kernels sum in a different
order and keep the polynomial expansion in float32.  Stated tolerance: max |d| <= 2e-3 px and mean |d| <= 1e-4 px on
well-conditioned (smooth, textured) input; on pure noise (ill-conditioned 2x2 systems) mean |d| <= 1e-3 px.  Against
farneback_k, which restates the kernels' own order, they are equal bit for bit."""
import os

import numpy as np
import pytest
import torch

import oracle
from oracle import farneback_k
from oracle import synth
from scanner_b200 import engine as E
from scanner_b200 import kernels

pytestmark = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("h,w", [(96, 128), (64, 80), (120, 160), (37, 53), (270, 480)])
def test_flow_vs_oracle_smooth_motion(h, w):
    a, b = synth.flow_pair(600 + h, h, w, "shift")
    got = kernels.optical_flow(dev(a[None]), dev(b[None]))[0].cpu().numpy()
    assert np.array_equal(got, farneback_k.flow(a, b))


def test_flow_vs_cv2_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "flow_cv2.npz"))
    for k in sorted(x[:-5] for x in g.files if x.endswith("_meta")):
        seed, h, w, kind = [int(x) for x in g[k + "_meta"]]
        a, b = synth.flow_pair(seed, h, w, "shift" if kind == 0 else "noise")
        got = kernels.optical_flow(dev(a[None]), dev(b[None]))[0].cpu().numpy()
        d = np.abs(got - g[k + "_flow"])
        if kind == 0:
            assert d.max() <= 2e-3 and d.mean() <= 1e-4, (k, d.max(), d.mean())
        else:
            assert d.mean() <= 1e-3 and np.quantile(d, 0.999) <= 5e-2, (k, d.max(), d.mean())


def test_flow_1080p_vs_cv2_and_the_oracle():
    """configs[3]'s size.  cv2 (the library the reference's op calls, optical_flow_kernel_cpu.cpp:27-47 /
    tests/test_ops.cpp:68-94) is run HERE on the same pair, so this is a direct comparison, not a stored golden;
    the oracle is run beside it so its own distance to cv2 at this size is on record too.
    Tolerance (float32 sums in another order): max |d| <= 2e-3 px, mean |d| <= 1e-4 px, both against cv2."""
    import cv2
    a, b = synth.flow_pair(941, 1080, 1920, "shift")
    got = kernels.optical_flow(dev(a[None]), dev(b[None]))[0].cpu().numpy()
    g0, g1 = cv2.cvtColor(a, cv2.COLOR_BGR2GRAY), cv2.cvtColor(b, cv2.COLOR_BGR2GRAY)
    ref = cv2.FarnebackOpticalFlow_create(3, 0.5, False, 15, 3, 5, 1.2, 0).calc(g0, g1, None)
    d = np.abs(got - ref)
    assert d.max() <= 2e-3 and d.mean() <= 1e-4, (d.max(), d.mean())
    want = oracle.optical_flow(a, b)
    assert np.abs(want - ref).max() <= 1e-3                 # the oracle's own pin at this size
    assert np.array_equal(got, farneback_k.flow(a, b))   # and the kernel-ordered oracle, bit for bit
    # all three agree on a field that follows the synthetic motion (1.5, -0.75) (3 levels x 3 iterations
    # under-estimate it: cv2 itself gives a median of (1.13, -0.56))
    med = np.median(got[200:-200, 200:-200].reshape(-1, 2), axis=0)
    assert 1.0 < med[0] < 1.6 and -0.8 < med[1] < -0.5, med


def test_flow_batch_and_identity():
    frames = np.stack([synth.flow_pair(700, 96, 128, "shift")[i] for i in (0, 1, 0)])
    out = kernels.optical_flow(dev(frames[:2]), dev(frames[1:])).cpu().numpy()
    assert np.array_equal(out[0], farneback_k.flow(frames[0], frames[1]))
    assert np.array_equal(out[1], farneback_k.flow(frames[1], frames[2]))
    # identical frames: NOT zero flow -- the last row/column take OpenCV's out-of-range branch of
    # UpdateMatrices (r2 = r3 = 0) and the coarse levels spread that inwards; same as the oracle
    same = kernels.optical_flow(dev(frames[:1]), dev(frames[:1]))[0].cpu().numpy()
    assert np.abs(same).max() > 0
    assert np.array_equal(same, farneback_k.flow(frames[0], frames[0]))


def test_optical_flow_op_stencil_through_the_engine():
    """reference py_test.py:459-520 runs OpticalFlow with stencil [0,1] and checks row counts;
    here every row is also compared with the kernel-ordered oracle, bit for bit (last row: window clamps to the last
    frame)."""
    E.load_stdlib()
    n, h, w = 7, 64, 96
    base = synth.flow_pair(800, h, w + n, "shift")[0]
    frames = np.stack([np.ascontiguousarray(base[:, i:i + w]) for i in range(n)])  # pans 1 px / frame
    eng = E.Engine(gpus=[0], instances_per_gpu=2)
    g = E.Graph()
    src = g.add_source(True)
    fl = g.add_op("OpticalFlow", [(src, "frame")], device=1)
    sink = g.add_sink((fl, "flow"))
    j = E.Job()
    j.bind_source(src, eng.add_raw_frames(frames))
    for (wps, ios) in [(1, 1), (4, 4)]:
        eng.run(g, [j], wps, ios)
        assert j.output_rows(sink) == n
        for i in range(n):
            got = j.output_row(sink, i)
            assert got.shape == (h, w, 2) and got.dtype == np.float32
            want = farneback_k.flow(frames[i], frames[min(i + 1, n - 1)])
            assert np.array_equal(got, want), (i, wps)
    eng.close()


def test_sequence_reuses_every_frames_expansion_and_changes_nothing():
    """scn_farneback_u8c3_chain: walking a clip pair by pair (one call, several calls, one pair per call like the
    op) gives the bits of independent pairs; sizes include one whose pyramid stops early (40 x 70: 1 level)."""
    for (n, h, w) in [(6, 96, 128), (4, 40, 70), (3, 270, 480)]:
        a, b = synth.flow_pair(810 + h, h, w, "shift")
        rng = np.random.default_rng(h)
        frames = np.stack([a, b] + [np.roll(a, (i, 2 * i), (0, 1)) + rng.integers(0, 2, a.shape, dtype=np.uint8)
                                    for i in range(1, n - 1)])
        d = dev(frames)
        want = kernels.optical_flow(d[:-1], d[1:])
        for step in (None, 2, 1):
            got = kernels.optical_flow_sequence(d, pairs_per_call=step)
            assert torch.equal(got, want), (n, h, w, step)


def test_float_window_sums_stay_close_to_the_double_ones():
    """box_solve_f32_kernel (default) against SCN_FLOW_BOX=f64 on the same pairs: the 2x2 solve stays in double,
    the 15 x 15 sums are float32 trees.  Stated: max |d| <= 5e-4 px on smooth motion."""
    import subprocess
    import sys
    import tempfile
    code = (
        "import sys, numpy as np, torch; sys.path.insert(0, '.');"
        "from scanner_b200 import kernels; from oracle import synth;"
        "outs = [];"
        "\nfor (h, w) in [(270, 480), (1080, 1920)]:"
        "\n    a, b = synth.flow_pair(77 + h, h, w, 'shift')"
        "\n    outs.append(kernels.optical_flow(torch.from_numpy(a[None]).cuda(), torch.from_numpy(b[None]).cuda()).cpu().numpy())"
        "\nnp.savez(sys.argv[1], *outs)")
    with tempfile.TemporaryDirectory() as d:
        for mode in ("f32", "f64"):
            subprocess.check_call([sys.executable, "-c", code, os.path.join(d, mode + ".npz")],
                                  env=dict(os.environ, SCN_FLOW_BOX=mode),
                                  cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        f, g = np.load(os.path.join(d, "f32.npz")), np.load(os.path.join(d, "f64.npz"))
        for k in f.files:
            dd = np.abs(f[k] - g[k])
            assert 0 < dd.max() <= 5e-4 and dd.mean() <= 2e-5, (k, dd.max(), dd.mean())


def test_fused_tiled_kernels_equal_the_two_pass_kernels_bit_for_bit():
    """The shared-memory tiled Gaussian / polynomial-expansion / box+solve kernels keep the summation
    order of the per-row two-pass kernels (SCN_FLOW_UNFUSED=1): same bits, including at image borders
    and for sizes that are not multiples of the tiles."""
    import subprocess
    import sys
    code = (
        "import sys, numpy as np, torch; sys.path.insert(0, '.');"
        "from scanner_b200 import kernels;"
        "g = torch.Generator(device='cuda').manual_seed(11);"
        "outs = [];"
        "\nfor (h, w) in [(270, 480), (97, 131), (1080, 1920)]:"
        "\n    a = torch.randint(0, 256, (2, h, w, 3), dtype=torch.uint8, device='cuda', generator=g)"
        "\n    b = torch.roll(a, shifts=(1, 2), dims=(1, 2)).contiguous()"
        "\n    outs.append(kernels.optical_flow(a, b).cpu().numpy())"
        "\nnp.savez(sys.argv[1], *outs)")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        for mode, name in (("0", "fused.npz"), ("1", "unfused.npz")):
            env = dict(os.environ, SCN_FLOW_UNFUSED=mode, SCN_FLOW_BOX="f64")   # the double box kernel keeps the order
            subprocess.check_call([sys.executable, "-c", code, os.path.join(d, name)], env=env,
                                  cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        f, u = np.load(os.path.join(d, "fused.npz")), np.load(os.path.join(d, "unfused.npz"))
        for k in f.files:
            assert f[k].shape == u[k].shape and np.array_equal(f[k], u[k]), k
