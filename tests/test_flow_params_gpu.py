"""Every Farneback kernel path of flow.cu against the oracle, and the OpticalFlow op's frame reuse, exactly.

tests/test_flow_gpu.py holds the kernels at the reference's arguments (3, 0.5, 15, 3, 5, 1.2).  scn_farneback_u8c3
accepts more, and several code paths run only off those defaults: the generic-radius Gaussian, the generic-poly_n
expansion, the double two-pass box for win_size != 15, the per-level expansion without the pyramid cache, 2 or 4
pyramid levels, a single iteration.  The oracle is held to cv2 over the same arguments by
tests/test_flow_params_cpu.py, so it is the reference here.  Bounds are those of test_flow_gpu.py: max |d| <= 2e-3
px and mean |d| <= 1e-4 px on smooth motion."""
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import oracle
from oracle import synth
from scanner_b200 import cabi, kernels, protolite
from scanner_b200 import engine as E

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCN_E_BADARG, SCN_E_UNSUPPORTED = -1, -2
DEFAULTS = dict(num_levels=3, pyr_scale=0.5, win_size=15, num_iters=3, poly_n=5, poly_sigma=1.2)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ran(fn):
    """fn() and the {kernel: launches} it caused."""
    L = cabi.lib()
    L.scn_prof_enable(1)
    try:
        out = fn()
        torch.cuda.synchronize()
        rep = cabi.prof_report()
    finally:
        L.scn_prof_enable(0)
    return out, {k: v["launches"] for k, v in rep.items()}


def _check(got, want, what, max_d=2e-3, outliers=0):
    """max |d| <= max_d, mean |d| <= 1e-4 px, and at most `outliers` pixels beyond the usual 2e-3 px."""
    d = np.abs(got - want)
    n_out = int((d.max(-1) > 2e-3).sum())
    print(f"{what}: max {d.max():.3e} mean {d.mean():.3e} pixels over 2e-3: {n_out}")
    assert d.max() <= max_d and d.mean() <= 1e-4 and n_out <= outliers, (what, d.max(), d.mean(), n_out)


def _vs_oracle(h, w, over, seed, **bound):
    a = dict(DEFAULTS, **over)
    f0, f1 = synth.flow_pair(seed, h, w, "shift")
    got, ran = _ran(lambda: kernels.optical_flow(dev(f0[None]), dev(f1[None]), **a)[0].cpu().numpy())
    want = oracle.farneback(oracle.bgr2gray(f0), oracle.bgr2gray(f1), **a)
    _check(got, want, f"{h}x{w} {over}", **bound)
    return ran


# ---- a. the argument grid against the oracle ------------------------------------------------------------------------
GRID = [
    (540, 960, dict(num_levels=4)),                          # Gaussian radius 19: gauss_fused_kernel<0>; 4 levels
    (270, 480, dict(pyr_scale=0.7)),                         # radius 2 at level 3: gauss_fused_kernel<0>
    (96, 128, dict(pyr_scale=0.3)),
    (270, 480, dict(poly_n=7, poly_sigma=1.5)),              # poly_fused_kernel<0>
    (270, 480, dict(poly_n=3, poly_sigma=0.9)),
    (96, 128, dict(poly_n=1, poly_sigma=0.6)),
    (270, 480, dict(win_size=2)),                            # box_v_kernel + box_h_solve_kernel (double); bound below
    (96, 128, dict(win_size=3)),
    (96, 128, dict(win_size=4)),
    (270, 480, dict(win_size=9)),
    (96, 128, dict(win_size=16)),
    (270, 480, dict(win_size=21)),
    (270, 480, dict(pyr_scale=0.8, num_levels=8)),           # pyramid over 2 W H pixels: per-level expansion
    (540, 960, dict(pyr_scale=0.7, num_levels=8, poly_n=7, poly_sigma=1.5)),
    (540, 960, dict(pyr_scale=0.8, num_levels=8)),
    (270, 480, dict(num_iters=1)),                           # no update_matrices_kernel between iterations
    (96, 128, dict(num_iters=6)),
    (96, 128, dict(num_levels=0)),
]


@pytest.mark.parametrize("h,w,over", GRID, ids=[f"{h}x{w}-" + "-".join(f"{k}{v}" for k, v in o.items())
                                                for h, w, o in GRID])
def test_kernels_match_the_oracle_off_the_default_arguments(h, w, over):
    bound = {}
    if over == dict(win_size=2):
        # A 3 x 3 window (at scale 1/4) leaves ill-conditioned 2x2 systems: the worst pixel's flow is (11.6, -13.2) px
        # where the motion is (1.5, -0.75), and there cv2 and the oracle already differ by 2.1e-2 px.  Measured on an
        # H100: max 7.3e-2, mean 1.1e-5, 59 of 129600 pixels over 2e-3; the same with SCN_FLOW_BOX=f64 and unfused.
        bound = dict(max_d=0.1, outliers=130)
    ran = _vs_oracle(h, w, over, 2000 + h + w, **bound)
    if over.get("win_size", 15) != 15:   # the f32 box kernel is instantiated for win_size 15 only
        assert ran.get("flow_box_v_kernel", 0) > 0 and ran.get("flow_box_h_solve_kernel", 0) > 0, ran
        assert "flow_box_solve_f32_kernel" not in ran, ran
    else:
        assert "flow_box_v_kernel" not in ran, ran


def _poly_launches(frames, monkeypatch, no_cache):
    if no_cache:
        monkeypatch.setenv("SCN_FLOW_NO_PYRAMID_CACHE", "1")
    else:
        monkeypatch.delenv("SCN_FLOW_NO_PYRAMID_CACHE", raising=False)
    out, ran = _ran(lambda: kernels.optical_flow_sequence(frames))
    return out, ran.get("flow_poly_fused_kernel", 0)


def test_pyramid_cache_and_per_level_expansion_give_the_same_bits(monkeypatch):
    """A 6-frame clip through optical_flow_sequence: with the pyramid cache every frame is expanded once at each of
    its L + 1 levels, (L + 1) n expansions; SCN_FLOW_NO_PYRAMID_CACHE=1 expands both frames of every pair at every
    level, 2 (L + 1)(n - 1).  270 x 480 has L = 3.  The two give the same bits, and the oracle's flow."""
    n, h, w = 6, 270, 480
    a, b = synth.flow_pair(2100, h, w, "shift")
    frames = np.stack([a, b] + [np.roll(b, (i, 2 * i), (0, 1)) for i in range(1, n - 1)])
    d = dev(frames)
    cached, k_cached = _poly_launches(d, monkeypatch, False)
    plain, k_plain = _poly_launches(d, monkeypatch, True)
    assert k_cached == 4 * n and k_plain == 2 * 4 * (n - 1), (k_cached, k_plain)
    assert torch.equal(cached, plain)
    for i in (0, n - 2):
        want = oracle.optical_flow(frames[i], frames[i + 1])
        assert np.abs(cached[i].cpu().numpy() - want).max() <= 2e-3, i


def test_tiny_frames_take_the_per_level_expansion(monkeypatch):
    """Each level of the cache is rounded up to 64 pixels, so a 4 x 4 clip has no room for it."""
    monkeypatch.delenv("SCN_FLOW_NO_PYRAMID_CACHE", raising=False)
    n = 4
    frames = np.stack([synth.flow_pair(2200, 4, 4 + n, "shift")[0][:, i:i + 4] for i in range(n)])
    got, ran = _ran(lambda: kernels.optical_flow_sequence(dev(frames)))
    assert ran.get("flow_poly_fused_kernel", 0) == 2 * (n - 1), ran
    for i in range(n - 1):
        assert np.abs(got[i].cpu().numpy() - oracle.optical_flow(frames[i], frames[i + 1])).max() <= 2e-3, i


# ---- b. edge geometries at the default arguments --------------------------------------------------------------------
# frames smaller than the window; widths and heights at the tiles' edges (f32 box 88 x 32, Gaussian and polynomial
# 64 x 32, update_matrices_kernel 32 x 8); 200 x 300 has two pyramid levels
EDGES = [(1, 1), (2, 2), (1, 64), (64, 1), (4, 4), (14, 14),
         (31, 87), (32, 88), (33, 89), (33, 87), (31, 89), (32, 64), (200, 300)]


@pytest.mark.parametrize("h,w", EDGES, ids=[f"{h}x{w}" for h, w in EDGES])
def test_edge_geometries_match_the_oracle(h, w):
    _vs_oracle(h, w, {}, 2300 + h + w)


def test_1080p_four_levels_vs_cv2():
    """num_levels=4 at 1080p runs the generic-radius Gaussian (radius 19) at full resolution; cv2 is run here.

    One pixel sits on a branch of UpdateMatrices: at (0, 566), in level 0's third call, the oracle's y + dy is
    -1.6e-8, so floor() takes it out of range; the GPU's float-order difference puts it at or above 0.  The 15 x 15
    box spreads that pixel over rows 0-7, columns 559-573.  Measured on an H100: max 4.8e-3, mean 1.1e-6, 104 pixels
    over 2e-3, all in that block (the same with SCN_FLOW_BOX=f64 and unfused); everywhere else <= 1e-5 px.  So the
    bound is widened for this block alone: at most one 8 x 15 footprint over 2e-3 px."""
    import cv2
    a, b = synth.flow_pair(942, 1080, 1920, "shift")
    got = kernels.optical_flow(dev(a[None]), dev(b[None]), num_levels=4)[0].cpu().numpy()
    g0, g1 = cv2.cvtColor(a, cv2.COLOR_BGR2GRAY), cv2.cvtColor(b, cv2.COLOR_BGR2GRAY)
    ref = cv2.calcOpticalFlowFarneback(g0, g1, None, 0.5, 4, 15, 3, 5, 1.2, 0)
    _check(got, ref, "1080p num_levels=4 vs cv2", max_d=6e-3, outliers=120)
    d = np.abs(got - ref)
    d[:8, 559:574] = 0
    assert d.max() <= 2e-3, d.max()


# ---- c. bit-for-bit: the fused kernels against the two-pass ones at a generic radius and poly_n --------------------
def test_fused_equals_two_pass_at_generic_radius_and_poly_n():
    """SCN_FLOW_UNFUSED=1 against the fused kernels, both with the double box (whose order both keep), where the
    generic instantiations gauss_fused_kernel<0> / poly_fused_kernel<0> run: radius 19 (num_levels=4), radius 2
    (pyr_scale=0.7), poly_n=7 and poly_n=3.  Both environment switches are read once per process."""
    code = (
        "import sys, numpy as np, torch; sys.path.insert(0, '.');"
        "from scanner_b200 import kernels;"
        "g = torch.Generator(device='cuda').manual_seed(12);"
        "outs = [];"
        "\nfor (h, w, kw) in [(540, 960, dict(num_levels=4)), (270, 480, dict(pyr_scale=0.7)),"
        "                     (97, 131, dict(poly_n=7, poly_sigma=1.5)), (97, 131, dict(poly_n=3, poly_sigma=0.9))]:"
        "\n    a = torch.randint(0, 256, (1, h, w, 3), dtype=torch.uint8, device='cuda', generator=g)"
        "\n    b = torch.roll(a, shifts=(1, 2), dims=(1, 2)).contiguous()"
        "\n    outs.append(kernels.optical_flow(a, b, **kw).cpu().numpy())"
        "\nnp.savez(sys.argv[1], *outs)")
    with tempfile.TemporaryDirectory() as d:
        for mode in ("0", "1"):
            subprocess.check_call([sys.executable, "-c", code, os.path.join(d, mode + ".npz")], cwd=ROOT,
                                  env=dict(os.environ, SCN_FLOW_UNFUSED=mode, SCN_FLOW_BOX="f64"))
        f, u = np.load(os.path.join(d, "0.npz")), np.load(os.path.join(d, "1.npz"))
        assert len(f.files) == 4
        for k in f.files:
            assert f[k].shape == u[k].shape and np.array_equal(f[k], u[k]), k


# ---- d. refusals ----------------------------------------------------------------------------------------------------
REFUSED = [(1080, 1920, dict(num_levels=5), SCN_E_UNSUPPORTED),   # level 5's Gaussian: ksize 79 > 65
           (96, 128, dict(poly_n=8), SCN_E_BADARG),
           (96, 128, dict(poly_n=0), SCN_E_BADARG),
           (96, 128, dict(win_size=1), SCN_E_BADARG),               # cv2's m = 0 box is not a 1 x 1 box
           (96, 128, dict(win_size=0), SCN_E_BADARG)]


@pytest.mark.parametrize("h,w,over,rc", REFUSED, ids=[f"{h}x{w}-" + "-".join(f"{k}{v}" for k, v in o.items())
                                                      for h, w, o, _ in REFUSED])
def test_refusals_leave_output_and_launch_count_untouched(h, w, over, rc):
    a = dict(DEFAULTS, **over)
    L = cabi.lib()
    frames = torch.zeros((2, h, w, 3), dtype=torch.uint8, device="cuda")
    out = torch.full((1, h, w, 2), 7.25, dtype=torch.float32, device="cuda")
    ws = torch.empty(L.scn_farneback_workspace_bytes(w, h), dtype=torch.uint8, device="cuda")
    pp, k1 = cabi.ptr_array([frames[0].data_ptr()])
    np_, k2 = cabi.ptr_array([frames[1].data_ptr()])
    op, k3 = cabi.ptr_array([out.data_ptr()])
    args = (a["num_levels"], a["pyr_scale"], a["win_size"], a["num_iters"], a["poly_n"], a["poly_sigma"],
            ws.data_ptr(), ws.numel())
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    before = L.scn_launch_count()
    assert L.scn_farneback_u8c3(pp, np_, 1, w, h, op, *args, stream) == rc
    chain = ctypes.c_int(1)
    assert L.scn_farneback_u8c3_chain(pp, np_, 1, w, h, op, *args, 1, ctypes.byref(chain), stream) == rc
    torch.cuda.synchronize()
    assert L.scn_launch_count() == before
    assert bool((out == 7.25).all())


# ---- e. the OpticalFlow op, exactly ---------------------------------------------------------------------------------
N, H, W, GOP = 17, 144, 192, 4   # 144 x 192: two pyramid levels, the whole pyramid cached


@pytest.fixture(scope="module")
def clip():
    """A smooth texture panning 1 px right and 1 px down every other frame, as lossless I_PCM H.264 (4:2:0)."""
    base = synth.flow_pair(2400, H + N, W + N, "shift")[0]
    gray = (base[..., 0].astype(np.int32) * 3 + base[..., 1] * 5 + base[..., 2] * 2) // 10
    y = np.stack([gray[i // 2:i // 2 + H, i:i + W] for i in range(N)]).astype(np.uint8)
    u = np.stack([y[i, ::2, ::2] // 4 + 96 for i in range(N)]).astype(np.uint8)
    v = np.stack([160 - y[i, 1::2, 1::2] // 4 for i in range(N)]).astype(np.uint8)
    yuv = np.concatenate([y.reshape(N, -1), u.reshape(N, -1), v.reshape(N, -1)], axis=1)
    return E.h264_synth(yuv, W, H, gop=GOP)


SAMPLINGS = [("gather", [0, 1, 2, 5, 6, 11, 12, 13, 16]),   # gaps, ends on the last row
             ("strided", 3),                                 # rows 0, 3, ..., 15
             ("all", None)]


def _run_op(data, sampling, placement, packets):
    """Decode through the engine -> (Sample ->) OpticalFlow (-> Sample) -> sink; -> (rows, frames delivered as
    NV12).  With the sampler before the op the op's windows are consecutive rows of the sampled domain; after it,
    the op computes only the windows of the rows that are kept, so consecutive calls skip rows."""
    eng = E.Engine(gpus=[0], instances_per_gpu=2)
    try:
        sid = eng.add_h264(data)
        kind, arg = sampling
        g = E.Graph()
        src = g.add_source(True)
        col = (src, "frame")
        smp = None
        if kind != "all" and placement == "before":
            smp = g.add_sample(col)
            col = (smp, "frame")
        fl = g.add_op("OpticalFlow", [col], device=1)
        col = (fl, "flow")
        if kind != "all" and placement == "after":
            smp = g.add_sample(col)
            col = (smp, "flow")
        sink = g.add_sink(col)
        j = E.Job()
        j.bind_source(src, sid)
        if kind == "gather":
            j.set_sampler(smp, "Gather", protolite.encode(protolite.SAMPLER_ARGS["GatherSamplerArgs"], {"rows": arg}))
        elif kind == "strided":
            j.set_sampler(smp, "Strided", protolite.encode(protolite.SAMPLER_ARGS["StridedSamplerArgs"],
                                                           {"stride": arg}))
        out = {}
        for wps, ios in packets:
            eng.run(g, [j], wps, ios)
            out[(wps, ios)] = [j.output_row(sink, i) for i in range(j.output_rows(sink))]
        return out, eng.stats()["counters"]["frames_delivered_nv12"], eng
    except BaseException:
        eng.close()
        raise


def _want(eng, data, sampling, placement):
    """kernels.optical_flow on the frames the decoder shows, window {0, 1} clamped at the last row."""
    sid = eng.add_h264(data)
    kind, arg = sampling
    rows = arg if kind == "gather" else list(range(0, N, arg)) if kind == "strided" else list(range(N))
    if placement == "before":   # f = the sampled frames; the window is {i, i + 1} in the sampled domain
        f = eng.decode_to_device(sid, rows, 0)
        cur, nxt = list(range(len(rows))), [min(i + 1, len(rows) - 1) for i in range(len(rows))]
    else:                       # f = every frame; row r of the op is kept when r is sampled
        f = eng.decode_to_device(sid, range(N), 0)
        cur, nxt = rows, [min(r + 1, N - 1) for r in rows]
    return kernels.optical_flow(f[cur], f[nxt]).cpu().numpy()


# (work packet, io packet): io packet 1 puts a task boundary between every pair of rows
PACKETS = [(1, 1), (2, 2), (1, 4), (3, 6), (4, 8)]


OP_CASES = [(s, p) for s in SAMPLINGS for p in ("before", "after") if s[0] != "all" or p == "before"]


@pytest.mark.parametrize("sampling,placement", OP_CASES, ids=[f"{s[0]}-{p}" for s, p in OP_CASES])
def test_optical_flow_op_is_bit_exact_on_nv12_and_rgb_elements(clip, sampling, placement, monkeypatch):
    """Row i of the op's output is kernels.optical_flow of the frames of its window, bit for bit: the op's pyramid
    reuse (window[0] == the last call's window[1]) and its per-row RGB cache of NV12 elements change nothing, under
    samplers, across task boundaries and on two pipeline instances.  SCN_DECODE_RGB=1 (dense RGB24 elements) gives
    the same bits."""
    E.load_stdlib()
    for force_rgb in (False, True):
        if force_rgb:
            monkeypatch.setenv("SCN_DECODE_RGB", "1")
        else:
            monkeypatch.delenv("SCN_DECODE_RGB", raising=False)
        got, nv12, eng = _run_op(clip, sampling, placement, PACKETS)
        try:
            want = _want(eng, clip, sampling, placement)
        finally:
            eng.close()
        assert (nv12 == 0) if force_rgb else (nv12 > 0), nv12
        for packets, rows in got.items():
            assert len(rows) == len(want), (packets, len(rows), len(want))
            for i, r in enumerate(rows):
                assert r.shape == (H, W, 2) and r.dtype == np.float32
                assert np.array_equal(r, want[i]), (force_rgb, packets, i, float(np.abs(r - want[i]).max()))
