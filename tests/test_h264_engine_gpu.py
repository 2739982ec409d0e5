"""compress_video() outputs end to end on the GPU: the reference's tutorial 06 flow (decode -> Blur -> Output) on a
1080p clip, with the column stored as H.264 by the save stage.  Each picture is intra-coded, so any stored picture
can be checked alone: the oracle (oracle/h264_enc.py) encodes the lossless run's frame at its position in its task,
and the decode of the stored column must equal the oracle's reconstruction bit for bit."""
import os

import cv2
import numpy as np
import pytest

import oracle
import scanner_b200 as sp
from oracle import h264_enc as HE
from oracle import synth
from scanner_b200 import engine as E

pytestmark = pytest.mark.gpu

W, H, N = 1920, 1080, 30


@pytest.fixture(scope="module")
def clip(tmp_path_factory):
    rgb = np.stack([synth.smooth_frame(70 + i, H, W) for i in range(N)]).astype(np.int64)
    r, g, b = rgb[..., 0], rgb[..., 1], rgb[..., 2]
    y = ((66 * r + 129 * g + 25 * b + 128) >> 8) + 16
    cb = (((-38 * r - 74 * g + 112 * b + 128) >> 8) + 128)[:, ::2, ::2]
    cr = (((112 * r - 94 * g - 18 * b + 128) >> 8) + 128)[:, ::2, ::2]
    yuv = np.concatenate([p.reshape(N, -1) for p in (y, cb, cr)], 1).astype(np.uint8)
    path = str(tmp_path_factory.mktemp("video") / "clip.mp4")
    open(path, "wb").write(E.mp4_mux(E.h264_synth(yuv, W, H, gop=10), 30, 1))
    return path


@pytest.fixture()
def sc(tmp_path):
    c = sp.Client(db_path=str(tmp_path / "scanner_db"))
    yield c
    c.stop()


def _blur_job(sc, path, name, store, perf=None, after=None):
    video = sp.NamedVideoStream(sc, "clip", path=path)
    frames = sc.ops.Blur(frame=sc.io.Input([video]), kernel_size=3, sigma=0.5)
    if after:
        frames = after(frames)
    out = sp.NamedVideoStream(sc, name)
    sc.run(sc.io.Output(store(frames), [out]), perf or sp.PerfParams.estimate())
    return out


def _oracle_decode(frame, qp, pos, kd):
    _, rec = HE.encode_frame(frame, qp, pos, kd)
    return oracle.nv12_to_rgb(*HE.to_nv12(rec))


def _stored_bytes(sc, name):
    d = os.path.join(sc._db.path, "tables", str(sc._db.table_info(name)["id"]))
    return sum(os.path.getsize(os.path.join(d, f)) for f in os.listdir(d) if f.startswith("1_") and
               f.endswith(".bin") and "metadata" not in f)


def test_tutorial_06_stores_h264_and_reads_it_back(sc, clip, tmp_path):
    raw = np.stack(list(_blur_job(sc, clip, "lossless_video", lambda c: c.lossless()).load()))
    low = _blur_job(sc, clip, "low_quality_video", lambda c: c.compress_video(quality=35))
    info = sc._db.table_info("low_quality_video")
    assert info["keyframes"] == 1 and info["rows"] == N
    stored = _stored_bytes(sc, "low_quality_video")
    assert stored < N * W * H * 3 // 10, stored
    got = np.stack(list(low.load()))
    for r in (0, 7, 29):
        assert (got[r] == _oracle_decode(raw[r], 35, r, 120)).all(), r
    part = list(low.load(rows=[29, 7]))
    assert (part[0] == got[29]).all() and (part[1] == got[7]).all()
    mp4 = low.save_mp4(str(tmp_path / "low_quality_video"))
    assert int(cv2.VideoCapture(mp4).get(cv2.CAP_PROP_FRAME_COUNT)) == N
    assert stored <= os.path.getsize(mp4) <= stored + 64 * 1024
    # the lossless column is unchanged: raw frames, no keyframes
    assert sc._db.table_info("lossless_video")["keyframes"] == -1


def test_tasks_become_items_that_read_as_one_stream(sc, clip):
    raw = np.stack(list(_blur_job(sc, clip, "raw", lambda c: c.lossless(), sp.PerfParams.manual(8, 8)).load()))
    out = _blur_job(sc, clip, "items", lambda c: c.compress_video(quality=30, keyframe_distance=7),
                    sp.PerfParams.manual(8, 8))
    info = sc._db.table_info("items")
    assert info["items"] == 4
    assert info["keyframes"] == 2 + 2 + 2 + 1  # tasks of 8, 8, 8 and 6 rows, an IDR every 7 pictures of each
    got = np.stack(list(out.load()))
    assert got.shape == raw.shape
    for r in (0, 7, 8, 13, 29):
        assert (got[r] == _oracle_decode(raw[r], 30, r % 8, 7)).all(), r
    # a next job reads the compressed column as its input
    hist_out = sp.NamedStream(sc, "hist")
    sc.run(sc.io.Output(sc.ops.Histogram(frame=sc.io.Input([out])), [hist_out]), sp.PerfParams.estimate())
    for r, h in enumerate(hist_out.load()):
        assert all((np.asarray(a) == b).all() for a, b in zip(h, oracle.hist16(got[r]))), r


def test_frames_from_a_python_op_are_encoded_too(sc, clip):
    @sp.register_python_op(name="Invert")
    def invert(config, frame: sp.FrameType) -> sp.FrameType:
        return 255 - frame

    raw = np.stack(list(_blur_job(sc, clip, "raw", lambda c: c.lossless(), after=lambda f: sc.ops.Invert(frame=f))
                        .load(rows=range(3))))
    out = _blur_job(sc, clip, "inverted", lambda c: c.compress_video(quality=20),
                    after=lambda f: sc.ops.Invert(frame=f))
    assert sc._db.table_info("inverted")["keyframes"] == 1
    got = list(out.load(rows=[0, 2]))
    assert (got[0] == _oracle_decode(raw[0], 20, 0, 120)).all()
    assert (got[1] == _oracle_decode(raw[2], 20, 2, 120)).all()


@pytest.mark.parametrize("after,match", [
    (lambda sc: lambda f: sc.ops.ConvertColor(frame=f, conversion=["COLOR_RGB2GRAY"]), "1 channel"),
    (lambda sc: lambda f: sc.ops.Resize(frame=f, width=[33], height=[24]), "odd size"),
])
def test_frames_h264_cannot_hold_fail_the_run(sc, clip, after, match):
    with pytest.raises(sp.ScannerException, match=match + ".*lossless"):
        _blur_job(sc, clip, "bad", lambda c: c.compress_video(), after=after(sc))
    assert not sc._db.has_table("bad")
    ok = _blur_job(sc, clip, "good", lambda c: c.compress_video(), sp.PerfParams.manual(8, 8),
                   after=lambda f: sc.ops.Resize(frame=f, width=[64], height=[48]))
    assert len(list(ok.load())) == N


def test_quality_out_of_range_is_refused_when_the_job_is_built(sc, clip):
    with pytest.raises(sp.ScannerException, match="quality"):
        _blur_job(sc, clip, "q99", lambda c: c.compress_video(quality=99))
