"""The H.264 encoder's model, oracle/h264_enc.py, held to an independent decoder: FFmpeg (through cv2, raw output =
the luma plane) must output exactly the oracle's reconstruction of every picture of the sweep -- even sizes over
every residue mod 16, QP 0-51, six kinds of content -- and the sweep must take every prediction mode and every
CAVLC path.  The GPU kernel is held to the oracle byte for byte in tests/test_h264_encode_gpu.py, where the
chroma planes are checked through a decode as well."""
import numpy as np
import pytest

from oracle import h264_enc as H
from scanner_b200 import engine as E


def _ffmpeg_luma(tmp_path, stream, n):
    import cv2
    path = str(tmp_path / "s.h264")
    open(path, "wb").write(stream)
    cap = cv2.VideoCapture(path)
    if not cap.set(cv2.CAP_PROP_CONVERT_RGB, 0):
        pytest.skip("this OpenCV build cannot return undecorated decoder output")
    out = []
    for _ in range(n):
        ok, y = cap.read()
        assert ok
        out.append(y)
    assert not cap.read()[0]
    return out


@pytest.fixture(scope="module")
def sweep(tmp_path_factory):
    """every sweep item encoded once: (name, frames, qp, access units, reconstructions), and the path counters"""
    st = H.new_stats()
    items = []
    for name, frames, qp in H.sweep():
        aus, recs = H.encode(frames, qp, keyframe_distance=2, stats=st)
        items.append((name, frames, qp, aus, recs))
    return items, st, tmp_path_factory.mktemp("h264")


def test_ffmpeg_decodes_the_sweep_to_the_oracles_reconstruction(sweep):
    items, _, tmp = sweep
    for name, frames, qp, aus, recs in items:
        got = _ffmpeg_luma(tmp, b"".join(aus), len(aus))
        for i, (y, rec) in enumerate(zip(got, recs)):
            assert y.shape == rec[0].shape and (y == rec[0]).all(), (name, i)


def test_the_sweep_takes_every_mode_and_cavlc_path(sweep):
    _, st, _ = sweep
    assert all(st["luma_mode"]), st           # V, H, DC, Plane
    assert all(st["chroma_mode"]), st         # DC, H, V, Plane
    assert all(st["nc_class"]), st            # nC 0-1, 2-3, 4-7, 8+, and -1 (chroma DC)
    assert st["level_prefix_14"] and st["level_prefix_15"] and st["total_coeff_16"], st
    assert st["emulation_prevention"], st


def test_ffmpeg_decodes_1080p_noise_to_the_oracles_reconstruction(tmp_path):
    rng = np.random.default_rng(5)
    frames = rng.integers(0, 256, (1, 1080, 1920, 3), dtype=np.uint8)
    aus, recs = H.encode(frames, 23)
    (y,) = _ffmpeg_luma(tmp_path, aus[0], 1)
    assert (y == recs[0][0]).all()


def test_size_and_psnr_fall_as_qp_rises(tmp_path):
    frame = H.natural(144, 176, 3)
    src = H.rgb_to_planes(frame)[0][:144, :176]
    sizes, psnrs = [], []
    for qp in (0, 12, 23, 35, 51):
        aus, recs = H.encode(frame[None], qp)
        (y,) = _ffmpeg_luma(tmp_path, aus[0], 1)
        assert (y == recs[0][0]).all()
        sizes.append(len(aus[0]))
        psnrs.append(H.psnr(recs[0][0], src))
    assert psnrs[0] >= 45, psnrs
    assert all(a > b for a, b in zip(sizes[1:], sizes[2:])), sizes
    assert all(a > b for a, b in zip(psnrs[1:], psnrs[2:])), psnrs


@pytest.mark.parametrize("n,kd", [(10, 3), (7, 1), (5, 120)])
def test_the_index_finds_every_picture_and_keyframe(n, kd):
    frames = np.stack([H.content("gradient", 48, 64, i) for i in range(n)])
    aus, _ = H.encode(frames, 30, keyframe_distance=kd)
    assert [au.startswith(b"\x00\x00\x00\x01\x67") for au in aus] == [i % kd == 0 for i in range(n)]
    eng = E.Engine(gpus=[], cpu_instances=1)
    sid = eng.add_h264(b"".join(aus))
    info = eng.stream_info(sid)
    assert (info["width"], info["height"], info["keyframes"]) == (64, 48, (n + kd - 1) // kd)
    assert eng.stream_rows(sid) == n and not eng.stream_may_reorder(sid)
    eng.close()


def test_positions_continue_an_item():
    frames = np.stack([H.content("noise", 32, 48, i) for i in range(6)])
    whole, _ = H.encode(frames, 28, keyframe_distance=4)
    tail, _ = H.encode(frames[3:], 28, keyframe_distance=4, positions=[3, 4, 5])
    assert whole[3:] == tail


def test_vlc_tables_are_prefix_free():
    def prefix_free(codes):
        s = sorted(format(b, f"0{n}b") for n, b in codes if n)
        return all(not b.startswith(a) for a, b in zip(s, s[1:]))
    for cls in range(5):
        valid = [i for i in range(len(H.COEFF_TOKEN_LEN[cls])) if i % 4 <= i // 4]   # TrailingOnes <= TotalCoeff
        assert prefix_free((H.COEFF_TOKEN_LEN[cls][i], H.COEFF_TOKEN_BITS[cls][i]) for i in valid), cls
    for lens, bits in ((H.TOTAL_ZEROS_LEN, H.TOTAL_ZEROS_BITS), (H.CDC_TOTAL_ZEROS_LEN, H.CDC_TOTAL_ZEROS_BITS),
                       (H.RUN_LEN, H.RUN_BITS)):
        for row_l, row_b in zip(lens, bits):
            assert prefix_free(zip(row_l, row_b))


@pytest.mark.parametrize("w,h,qp", [(31, 16, 23), (16, 31, 23), (4098, 16, 23), (4096, 2320, 23), (16, 16, 52),
                                    (16, 16, -1)])
def test_the_oracle_refuses_what_the_kernel_refuses(w, h, qp):
    with pytest.raises(ValueError):
        H.check_args(w, h, qp)


# ---- client options -------------------------------------------------------------------------------------------
def test_compress_video_options_map_to_qp_and_keyframe_distance():
    import scanner_b200 as sp
    from scanner_b200.client import OpColumn, _h264_encoding
    col = OpColumn(None, "frame", True)
    assert _h264_encoding(col) is None
    assert _h264_encoding(col.lossless()) is None and _h264_encoding(col.compress("default")) is None
    assert _h264_encoding(col.compress_video()) == (23, 120)
    assert _h264_encoding(col.compress_video(quality=0, bitrate=5000, keyframe_distance=1)) == (0, 1)
    assert _h264_encoding(col.compress("video", quality=51, keyframe_distance=30)) == (51, 30)
    for bad in (dict(quality=99), dict(quality=-2), dict(quality=1.5), dict(keyframe_distance=0)):
        with pytest.raises(sp.ScannerException):
            _h264_encoding(col.compress_video(**bad))
    job = E.Job()
    job.set_sink_encoding(0, 35, 7)
    for qp, kd in ((52, 1), (-1, 1), (23, 0)):
        with pytest.raises(E.EngineError):
            job.set_sink_encoding(0, qp, kd)


def _video(tmp_path, w=64, h=48, n=6):
    rng = np.random.default_rng(3)
    yuv = rng.integers(0, 256, (n, w * h * 3 // 2), dtype=np.uint8)
    path = str(tmp_path / "v.mp4")
    open(path, "wb").write(E.mp4_mux(E.h264_synth(yuv, w, h, gop=3), 24, 1))
    return path


def test_cpu_only_clients_store_compress_video_outputs_raw(tmp_path):
    import scanner_b200 as sp
    sc = sp.Client(gpus=[], db_path=str(tmp_path / "db"))
    video = sp.NamedVideoStream(sc, "v", path=_video(tmp_path))
    frames = sc.io.Input([video])
    lossless, compressed = sp.NamedVideoStream(sc, "lossless"), sp.NamedVideoStream(sc, "compressed")
    sc.run(sc.io.Output(frames.lossless(), [lossless]), sp.PerfParams.estimate())
    sc.run(sc.io.Output(sc.io.Input([video]).compress_video(quality=30), [compressed]), sp.PerfParams.estimate())
    assert sc._db.table_info("compressed")["keyframes"] == -1
    assert all((a == b).all() for a, b in zip(lossless.load(), compressed.load()))
    with pytest.raises(sp.ScannerException, match="quality"):
        sc.run(sc.io.Output(sc.io.Input([video]).compress_video(quality=99), [sp.NamedVideoStream(sc, "q")]),
               sp.PerfParams.estimate())
    assert not sc._db.has_table("q")
    sc.stop()


def test_clients_without_a_database_keep_compress_video_outputs_in_memory(tmp_path):
    import scanner_b200 as sp
    sc = sp.Client(gpus=[])
    video = sp.NamedVideoStream(sc, "v", path=_video(tmp_path))
    out = sp.NamedVideoStream(sc, "out")
    sc.run(sc.io.Output(sc.io.Input([video]).compress_video(), [out]), sp.PerfParams.estimate())
    got = list(out.load())
    assert len(got) == 6 and got[0].shape == (48, 64, 3)
    sc.stop()
