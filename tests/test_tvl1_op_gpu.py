"""The OpticalFlowTVL1 op (stencil [0, 1], batch 8) through the engine and the client: every row bit-identical to
kernels.tvl1_flow on the same frames, across packet sizes, instances, a Strided sampler and NV12 elements."""
import os

import numpy as np
import pytest
import torch

import scanner_b200 as sp
from oracle import convert_color as C
from oracle import synth
from scanner_b200 import engine as E
from scanner_b200 import kernels, protolite

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(epsilon=-1.0, iterations=15, nscales=3, warps=2)


@pytest.fixture(scope="module")
def std():
    E.load_stdlib()
    return protolite.parse_proto(open(os.path.join(ROOT, "scanner_b200", "csrc", "ops", "stdlib_args.proto")).read())


def args(std, **kw):
    return protolite.encode(std["OpticalFlowTVL1Args"], kw)


def panning(n, h, w, seed=800):
    base = synth.flow_pair(seed, h, w + 2 * n, "shift")[0]
    return np.stack([np.ascontiguousarray(base[:, 2 * i:2 * i + w]) for i in range(n)])  # 2 px per frame


def expected(gray, rows, **kw):
    """kernels.tvl1_flow of windows (r, min(r + 1, last)) over the gray frames of the sampled rows"""
    g = torch.from_numpy(np.ascontiguousarray(gray)).cuda()
    nxt = [min(i + 1, len(rows) - 1) for i in range(len(rows))]
    return kernels.tvl1_flow(g[list(range(len(rows)))], g[nxt], **kw).cpu().numpy()


def run(eng, std, source_id, n_rows, wps, ios, stride=None, convert=False, op_args=None):
    g = E.Graph()
    src = g.add_source(True)
    inp = (src, "frame")
    if stride:
        smp = g.add_sample(inp)
        inp = (smp, "frame")
    cc = None
    if convert:
        cc = g.add_op("ConvertColor", [inp], device=1)
        inp = (cc, "frame")
    fl = g.add_op("OpticalFlowTVL1", [inp], device=1, args=op_args if op_args is not None else args(std, **{
        "epsilon": -1.0, "iterations": 15, "nscales": 3, "warps": 2}))
    sink = g.add_sink((fl, "flow"))
    j = E.Job()
    j.bind_source(src, source_id)
    if stride:
        j.set_sampler(smp, "Strided", protolite.encode(protolite.SAMPLER_ARGS["StridedSamplerArgs"], {"stride": stride}))
    if convert:
        j.set_stream_args(cc, protolite.encode(std["ConvertColorArgs"], {"conversion": "COLOR_RGB2GRAY"}))
    eng.run(g, [j], wps, ios)
    assert j.output_rows(sink) == n_rows
    return [j.output_row(sink, i) for i in range(n_rows)]


@pytest.mark.parametrize("instances", [1, 2])
def test_rgb_and_gray_frames_rows_equal_the_kernel(std, instances):
    n, h, w = 11, 48, 64
    frames = panning(n, h, w)
    gray = np.stack([C.convert_color(f, "COLOR_RGB2GRAY")[..., 0] for f in frames])
    want = expected(gray, range(n), **KW)
    eng = E.Engine(gpus=[0], instances_per_gpu=instances)
    try:
        sid = eng.add_raw_frames(frames)
        for wps, ios in [(1, 1), (4, 8), (3, 9)]:
            for convert in (False, True):
                rows = run(eng, std, sid, n, wps, ios, convert=convert)
                for i in range(n):
                    assert rows[i].shape == (h, w, 2) and rows[i].dtype == np.float32
                    assert np.array_equal(rows[i], want[i]), (wps, ios, convert, i)
        assert (want[-1] == 0).all()  # the last window clamps to (last, last)
        sid = eng.add_raw_frames(frames[::3])
        rows = run(eng, std, sid, len(frames[::3]), 2, 4)
        w3 = expected(gray[::3], range(len(frames[::3])), **KW)
        for i in range(len(rows)):
            assert np.array_equal(rows[i], w3[i])
    finally:
        eng.close()


def _clip(seed, n, h, w, gop):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    y = np.stack([(128 + 60 * np.sin(0.21 * (xx - 2 * i)) * np.cos(0.17 * yy) + rng.normal(0, 2, (h, w))).clip(0, 255)
                  for i in range(n)]).astype(np.uint8)
    u = np.full((n, h // 2, w // 2), 120, np.uint8)
    v = np.full((n, h // 2, w // 2), 136, np.uint8)
    yuv = np.concatenate([y.reshape(n, -1), u.reshape(n, -1), v.reshape(n, -1)], axis=1)
    import oracle
    rgb = []
    for i in range(n):
        chroma = np.empty((h // 2, w), np.uint8)
        chroma[:, 0::2], chroma[:, 1::2] = u[i], v[i]
        rgb.append(oracle.nv12_to_rgb(y[i], chroma))
    return E.h264_synth(yuv, w, h, gop=gop), np.stack(rgb)


def test_nv12_elements_and_a_strided_sampler(std):
    n, h, w = 12, 64, 96
    data, shown = _clip(3, n, h, w, 4)
    gray = np.stack([C.convert_color(f, "COLOR_RGB2GRAY")[..., 0] for f in shown])
    eng = E.Engine(gpus=[0], instances_per_gpu=2)
    try:
        sid = eng.add_h264(data)
        want = expected(gray, range(n), **KW)
        for wps, ios in [(2, 4), (4, 12)]:
            rows = run(eng, std, sid, n, wps, ios)
            for i in range(n):
                assert np.array_equal(rows[i], want[i]), (wps, i)
        rows = run(eng, std, sid, n // 2, 2, 4, stride=2)
        w2 = expected(gray[::2], range(n // 2), **KW)
        for i in range(n // 2):
            assert np.array_equal(rows[i], w2[i]), i
    finally:
        eng.close()


def test_bad_input_fails_the_run_naming_the_op_and_the_engine_goes_on(std):
    eng = E.Engine(gpus=[0], instances_per_gpu=1)
    try:
        frames = panning(4, 32, 40)
        sid = eng.add_raw_frames(frames)
        with pytest.raises(Exception, match="OpticalFlowTVL1"):
            run(eng, std, sid, 4, 2, 4, op_args=args(std, median_filtering=4))
        with pytest.raises(Exception, match="OpticalFlowTVL1"):
            run(eng, std, sid, 4, 2, 4, op_args=args(std, scale_step=1.5))
        two = eng.add_raw_frames(np.zeros((4, 16, 16, 2), np.uint8))
        with pytest.raises(Exception, match="OpticalFlowTVL1"):
            run(eng, std, two, 4, 2, 4)
        tiny = eng.add_raw_frames(np.zeros((4, 1, 16, 3), np.uint8))
        with pytest.raises(Exception, match="OpticalFlowTVL1"):
            run(eng, std, tiny, 4, 2, 4)
        rows = run(eng, std, sid, 4, 2, 4)
        gray = np.stack([C.convert_color(f, "COLOR_RGB2GRAY")[..., 0] for f in frames])
        want = expected(gray, range(4), **KW)
        assert all(np.array_equal(rows[i], want[i]) for i in range(4))
    finally:
        eng.close()


def test_through_the_client(tmp_path):
    sc = sp.Client(db_path=str(tmp_path / "db"))
    try:
        n, h, w = 6, 40, 56
        frames = panning(n, h, w, seed=31)
        inp = sc.io.Input([sp.NamedVideoStream(sc, "clip", frames=frames)])
        out = sp.NamedVideoStream(sc, "flow")
        sc.run(sc.io.Output(sc.ops.OpticalFlowTVL1(frame=inp, epsilon=-1, iterations=15, nscales=3, warps=2), [out]),
               sp.PerfParams.estimate())
        got = list(out.load())
        gray = np.stack([C.convert_color(f, "COLOR_RGB2GRAY")[..., 0] for f in frames])
        want = expected(gray, range(n), **KW)
        assert len(got) == n and all(np.array_equal(np.asarray(got[i]), want[i]) for i in range(n))
        # defaults: 0 / absent fields mean the documented defaults
        out2 = sp.NamedVideoStream(sc, "flow2")
        sc.run(sc.io.Output(sc.ops.OpticalFlowTVL1(frame=sc.io.Input([sp.NamedVideoStream(sc, "clip")])), [out2]),
               sp.PerfParams.estimate())
        want2 = expected(gray, range(n))
        assert all(np.array_equal(np.asarray(r), want2[i]) for i, r in enumerate(out2.load()))
        with pytest.raises(sp.ScannerException, match="OpticalFlowTVL1"):
            sc.run(sc.io.Output(sc.ops.OpticalFlowTVL1(frame=sc.io.Input([sp.NamedVideoStream(sc, "clip")]),
                                                       warps=99), [sp.NamedVideoStream(sc, "bad")]),
                   sp.PerfParams.estimate())
        out3 = sp.NamedVideoStream(sc, "flow3")
        sc.run(sc.io.Output(sc.ops.OpticalFlowTVL1(frame=sc.io.Input([sp.NamedVideoStream(sc, "clip")]), epsilon=-1,
                                                   iterations=15, nscales=3, warps=2), [out3]),
               sp.PerfParams.estimate())
        assert all(np.array_equal(np.asarray(r), want[i]) for i, r in enumerate(out3.load()))
    finally:
        sc.stop()
